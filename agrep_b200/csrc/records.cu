/* agrep_b200/csrc/records.cu -- stage 2, the forms that start from record boundaries (records_kernel.cuh): the
 * instantiations for 32- and 64-bit rows, and the launchers of every row width */
#include "records_kernel.cuh"

template <bool SET>
static int launch_dense_any(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st)
{
	if (d.wide) return launch_dense_wide(d.nrows, P, grid, st, SET);
	const bool costs = d.engine == AGB_ENGINE_ASEARCH1, narrow = d.M <= 31;
	if (costs) return narrow ? launch_dense_t<uint32_t, true, SET>(d.nrows, P, grid, st) : launch_dense_t<uint64_t, true, SET>(d.nrows, P, grid, st);
	return narrow ? launch_dense_t<uint32_t, false, SET>(d.nrows, P, grid, st) : launch_dense_t<uint64_t, false, SET>(d.nrows, P, grid, st);
}
int launch_dense(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st) { return launch_dense_any<false>(d, P, grid, st); }
int launch_dense_set(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st) { return launch_dense_any<true>(d, P, grid, st); }

int launch_records_list(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st)
{
	if (d.wide) return launch_records_list_wide(d.nrows, P, grid, st);
	const bool costs = d.engine == AGB_ENGINE_ASEARCH1, narrow = d.M <= 31;
	if (costs) return narrow ? launch_records_list_t<uint32_t, true>(d.nrows, P, grid, st) : launch_records_list_t<uint64_t, true>(d.nrows, P, grid, st);
	return narrow ? launch_records_list_t<uint32_t, false>(d.nrows, P, grid, st) : launch_records_list_t<uint64_t, false>(d.nrows, P, grid, st);
}

