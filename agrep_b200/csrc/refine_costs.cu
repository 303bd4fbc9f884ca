/* agrep_b200/csrc/refine_costs.cu -- instantiations of stage 1.5 (refine_kernel.cuh); the 64-bit rows are in
 * refine_costs_u64.cu, so that the two halves compile in parallel */
#include "refine_kernel.cuh"

int refine_launch_costs_u64(int nrows, const RefineParams &P, unsigned &grid, cudaStream_t st);

int refine_launch_costs(bool narrow, int nrows, const RefineParams &P, unsigned &grid, cudaStream_t st)
{
	if (!narrow) return refine_launch_costs_u64(nrows, P, grid, st);
	switch (nrows) {
	case 1: launch_refine_one<uint32_t, 1, true>(P, grid, st); break;
	case 2: launch_refine_one<uint32_t, 2, true>(P, grid, st); break;
	case 3: launch_refine_one<uint32_t, 3, true>(P, grid, st); break;
	case 4: launch_refine_one<uint32_t, 4, true>(P, grid, st); break;
	case 5: launch_refine_one<uint32_t, 5, true>(P, grid, st); break;
	case 6: launch_refine_one<uint32_t, 6, true>(P, grid, st); break;
	case 7: launch_refine_one<uint32_t, 7, true>(P, grid, st); break;
	case 8: launch_refine_one<uint32_t, 8, true>(P, grid, st); break;
	case 9: launch_refine_one<uint32_t, 9, true>(P, grid, st); break;
	default: return -1;
	}
	return 0;
}
