/* agrep_b200/csrc/records.cu -- stage 2, the forms that start from record boundaries (records_kernel.cuh): the
 * instantiations for 32- and 64-bit rows, and the launchers of every row width */
#include "records_kernel.cuh"

template <typename T, bool COSTS, bool SET>
static int launch_dense_t(int nrows, const RecParams &P, unsigned grid, cudaStream_t st)
{
	switch (nrows) {
	case 1: launch_dense_one<T, 1, COSTS, SET>(P, grid, st); break;
	case 2: launch_dense_one<T, 2, COSTS, SET>(P, grid, st); break;
	case 3: launch_dense_one<T, 3, COSTS, SET>(P, grid, st); break;
	case 4: launch_dense_one<T, 4, COSTS, SET>(P, grid, st); break;
	case 5: launch_dense_one<T, 5, COSTS, SET>(P, grid, st); break;
	case 6: launch_dense_one<T, 6, COSTS, SET>(P, grid, st); break;
	case 7: launch_dense_one<T, 7, COSTS, SET>(P, grid, st); break;
	case 8: launch_dense_one<T, 8, COSTS, SET>(P, grid, st); break;
	case 9: launch_dense_one<T, 9, COSTS, SET>(P, grid, st); break;
	default: return -1;
	}
	g_launches++;
	return 0;
}
template <bool SET>
static int launch_dense_any(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st)
{
	if (d.wide) return launch_dense_wide(P, grid, st, SET);
	const bool costs = d.engine == AGB_ENGINE_ASEARCH1, narrow = d.M <= 31;
	if (costs) return narrow ? launch_dense_t<uint32_t, true, SET>(d.nrows, P, grid, st) : launch_dense_t<uint64_t, true, SET>(d.nrows, P, grid, st);
	return narrow ? launch_dense_t<uint32_t, false, SET>(d.nrows, P, grid, st) : launch_dense_t<uint64_t, false, SET>(d.nrows, P, grid, st);
}
int launch_dense(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st) { return launch_dense_any<false>(d, P, grid, st); }
int launch_dense_set(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st) { return launch_dense_any<true>(d, P, grid, st); }

template <typename T, bool COSTS>
static int launch_records_list_t(int nrows, const RecParams &P, unsigned grid, cudaStream_t st)
{
	switch (nrows) {
	case 1: k_records_list<T, 1, COSTS><<<grid, REC_THREADS, LIST_SMEM, st>>>(P); break;
	case 2: k_records_list<T, 2, COSTS><<<grid, REC_THREADS, LIST_SMEM, st>>>(P); break;
	case 3: k_records_list<T, 3, COSTS><<<grid, REC_THREADS, LIST_SMEM, st>>>(P); break;
	case 4: k_records_list<T, 4, COSTS><<<grid, REC_THREADS, LIST_SMEM, st>>>(P); break;
	case 5: k_records_list<T, 5, COSTS><<<grid, REC_THREADS, LIST_SMEM, st>>>(P); break;
	case 6: k_records_list<T, 6, COSTS><<<grid, REC_THREADS, LIST_SMEM, st>>>(P); break;
	case 7: k_records_list<T, 7, COSTS><<<grid, REC_THREADS, LIST_SMEM, st>>>(P); break;
	case 8: k_records_list<T, 8, COSTS><<<grid, REC_THREADS, LIST_SMEM, st>>>(P); break;
	case 9: k_records_list<T, 9, COSTS><<<grid, REC_THREADS, LIST_SMEM, st>>>(P); break;
	default: return -1;
	}
	g_launches++;
	return 0;
}

int launch_records_list(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st)
{
	if (d.wide) return launch_records_list_wide(P, grid, st);
	const bool costs = d.engine == AGB_ENGINE_ASEARCH1, narrow = d.M <= 31;
	if (costs) return narrow ? launch_records_list_t<uint32_t, true>(d.nrows, P, grid, st) : launch_records_list_t<uint64_t, true>(d.nrows, P, grid, st);
	return narrow ? launch_records_list_t<uint32_t, false>(d.nrows, P, grid, st) : launch_records_list_t<uint64_t, false>(d.nrows, P, grid, st);
}

