/* agrep_b200/csrc/records_wide.cu -- stage 2 for 320-bit rows: simple literals of more than 63 positions at k = 0
 * (agb_wide).  The dense tile and list forms of records_kernel.cuh at one row; there is no slices form for them
 * (slices_usable). */
#include "records_kernel.cuh"

int launch_dense_wide(const RecParams &P, unsigned grid, cudaStream_t st, bool set)
{
	if (set) launch_dense_one<Wide, 1, false, true>(P, grid, st);
	else launch_dense_one<Wide, 1, false, false>(P, grid, st);
	g_launches++;
	return 0;
}

int launch_records_list_wide(const RecParams &P, unsigned grid, cudaStream_t st)
{
	k_records_list<Wide, 1, false><<<grid, REC_THREADS, LIST_SMEM, st>>>(P);
	g_launches++;
	return 0;
}
