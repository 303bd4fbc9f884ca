/* agrep_b200/csrc/records_wide.cu -- stage 2 for 320-bit rows: simple literals of more than 63 positions, k = 0..8
 * (agb_wide).  The dense tile and list forms of records_kernel.cuh at 1..9 rows, unit costs; there is no slices form for
 * them (slices_usable). */
#include "records_kernel.cuh"

int launch_dense_wide(int nrows, const RecParams &P, unsigned grid, cudaStream_t st, bool set)
{
	return set ? launch_dense_t<Wide, false, true>(nrows, P, grid, st) : launch_dense_t<Wide, false, false>(nrows, P, grid, st);
}

int launch_records_list_wide(int nrows, const RecParams &P, unsigned grid, cudaStream_t st)
{
	return launch_records_list_t<Wide, false>(nrows, P, grid, st);
}
