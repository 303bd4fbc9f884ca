// tools/front_bench.cu -- development microbenchmark (not product): inner-compare variants of the stage-1
// anchor kernel on synthetic text, to pick the instruction mix with measurements instead of guesses.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o tools/front_bench tools/front_bench.cu
// run:   tools/front_bench [GiB]
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>
#include <algorithm>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

struct P { const uint4 *text; uint32_t *bitmap; uint64_t n_chunks, n_words; uint32_t anchor[8]; uint32_t coef[8]; uint32_t one, scale; };

__device__ __forceinline__ uint4 ld16(const uint4 *p) {
	uint4 v; asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p)); return v; }

template <int V, int NA> __device__ __forceinline__ uint32_t win(uint32_t lo, uint32_t hi, const P &p, uint32_t acc)
{
	uint32_t w0 = lo, w1 = __funnelshift_r(lo, hi, 8), w2 = __funnelshift_r(lo, hi, 16), w3 = __funnelshift_r(lo, hi, 24);
#pragma unroll
	for (int a = 0; a < NA; a++) {
		uint32_t A = p.anchor[a];
		if (V == 0) { acc = __vimin3_u32(acc, w0 - A, w1 - A); acc = __vimin3_u32(acc, w2 - A, w3 - A); }
		if (V == 1) { acc |= (w0 == A) | (w1 == A) | (w2 == A) | (w3 == A); }
		if (V == 2) { acc = __vimin3_u32(acc, w0 ^ A, w1 ^ A); acc = __vimin3_u32(acc, w2 ^ A, w3 ^ A); }
		if (V == 3) {
			uint32_t d0, d1, d2, d3, nA = 0u - A;
			asm volatile("mad.lo.u32 %0, %1, 1, %2;" : "=r"(d0) : "r"(w0), "r"(nA));
			asm volatile("mad.lo.u32 %0, %1, 1, %2;" : "=r"(d1) : "r"(w1), "r"(nA));
			asm volatile("mad.lo.u32 %0, %1, 1, %2;" : "=r"(d2) : "r"(w2), "r"(nA));
			asm volatile("mad.lo.u32 %0, %1, 1, %2;" : "=r"(d3) : "r"(w3), "r"(nA));
			acc = __vimin3_u32(acc, d0, d1); acc = __vimin3_u32(acc, d2, d3);
		}
		if (V == 4) { acc = min(acc, min(min(w0 - A, w1 - A), min(w2 - A, w3 - A))); }
	}
	return acc;
}

// polynomial test: f(w) = prod_i (w - A_i) mod 2^32 by Horner on the FMA pipe (IMAD); zero iff (almost surely) w is an anchor
template <int NA> __device__ __forceinline__ uint32_t poly(uint32_t w, const P &p)
{
	uint32_t r = w * p.one + p.coef[NA - 1];
#pragma unroll
	for (int i = NA - 2; i >= 0; i--) r = r * w + p.coef[i];
	return r;
}
template <int NA, bool SC> __device__ __forceinline__ uint32_t winpoly(uint32_t lo, uint32_t hi, const P &p, uint32_t acc)
{
	uint32_t w0 = lo, w1 = __funnelshift_r(lo, hi, 8), w2 = __funnelshift_r(lo, hi, 16), w3 = __funnelshift_r(lo, hi, 24);
	uint32_t p0 = poly<NA>(w0, p), p1 = poly<NA>(w1, p), p2 = poly<NA>(w2, p), p3 = poly<NA>(w3, p);
	if (SC) { p0 *= p.scale; p1 *= p.scale; p2 *= p.scale; p3 *= p.scale; }
	acc = __vimin3_u32(acc, p0, p1); acc = __vimin3_u32(acc, p2, p3);
	return acc;
}

// V==9: no compare at all (pure streaming read + ballot): the load-path ceiling of this kernel shape
template <int V, int NA, int U, int T>
__global__ void __launch_bounds__(T) k(const P p)
{
	const uint32_t lane = threadIdx.x & 31;
	const uint64_t warp = ((uint64_t)blockIdx.x * T + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * T) >> 5;
	const uint64_t n_groups = (p.n_words + U - 1) / U;
	for (uint64_t g = warp; g < n_groups; g += nwarps) {
		const uint64_t w0 = g * U;
		uint4 v[U + 1];
#pragma unroll
		for (int u = 0; u < U; u++) { uint64_t c = (w0 + u) * 32 + lane; v[u] = (c < p.n_chunks) ? ld16(p.text + c) : make_uint4(0, 0, 0, 0); }
		{ uint64_t c = (w0 + U) * 32; uint32_t nx = 0; if (lane == 0 && c < p.n_chunks) nx = __ldg((const uint32_t *)(p.text + c)); v[U] = make_uint4(nx, 0, 0, 0); }
#pragma unroll
		for (int u = 0; u < U; u++) {
			if (w0 + u >= p.n_words) break;
			uint32_t give = (lane == 0) ? v[u + 1].x : v[u].x;
			uint32_t x4 = __shfl_sync(0xffffffffu, give, (lane + 1) & 31);
			uint32_t x0 = v[u].x, x1 = v[u].y, x2 = v[u].z, x3 = v[u].w;
			bool flag;
			if (V == 9) flag = ((x0 ^ x1 ^ x2 ^ x3 ^ x4) == p.anchor[0]);
			else {
				uint32_t acc = (V == 1) ? 0u : 0xffffffffu;
				if (V == 5) { acc = winpoly<NA, false>(x0, x1, p, acc); acc = winpoly<NA, false>(x1, x2, p, acc); acc = winpoly<NA, false>(x2, x3, p, acc); acc = winpoly<NA, false>(x3, x4, p, acc); }
				else if (V == 6) { acc = winpoly<NA, false>(x0, x1, p, acc); acc = winpoly<NA, false>(x1, x2, p, acc); acc = winpoly<NA, false>(x2, x3, p, acc); acc = win<0, NA>(x3, x4, p, acc); }
				else if (V == 7) { acc = winpoly<NA, false>(x0, x1, p, acc); acc = win<0, NA>(x1, x2, p, acc); acc = winpoly<NA, false>(x2, x3, p, acc); acc = win<0, NA>(x3, x4, p, acc); }
				else if (V == 8) { acc = winpoly<NA, true>(x0, x1, p, acc); acc = winpoly<NA, true>(x1, x2, p, acc); acc = winpoly<NA, true>(x2, x3, p, acc); acc = winpoly<NA, true>(x3, x4, p, acc); }
				else { acc = win<V, NA>(x0, x1, p, acc); acc = win<V, NA>(x1, x2, p, acc); acc = win<V, NA>(x2, x3, p, acc); acc = win<V, NA>(x3, x4, p, acc); }
				flag = (V == 1) ? (acc != 0) : (acc == 0);
			}
			uint32_t word = __ballot_sync(0xffffffffu, flag);
			if (lane == 0) p.bitmap[w0 + u] = word;
		}
	}
}


static void set_coef(P &p, int NA);
// ---- V10: bulk-async (TMA) staged pipeline: one thread streams 16 KiB stages into shared memory through
// mbarriers, all threads consume from shared memory (LDS.128), so the load depth no longer depends on registers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *b, int cnt) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(b)), "r"(cnt)); }
__device__ __forceinline__ void mbar_expect(uint64_t *b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *b) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(b)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t *b, uint32_t parity) {
	asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@!p bra W_%=;\n}" :: "r"(smem_u32(b)), "r"(parity) : "memory"); }

template <int NA, int NST, int T, int CH, int XMODE>
__global__ void __launch_bounds__(T) k_tma(const P p, uint64_t total_bytes_readable)
{
	extern __shared__ __align__(128) uint8_t smem[];
	constexpr uint32_t SB = T * CH * 16, SS = SB + 16;
	__shared__ uint64_t bar[NST];
	const uint32_t tid = threadIdx.x, lane = tid & 31;
	const uint64_t n_stages = (p.n_chunks + (uint64_t)T * CH - 1) / ((uint64_t)T * CH);
	if (tid == 0) { for (int i = 0; i < NST; i++) mbar_init(&bar[i], 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
	__syncthreads();
	auto issue = [&](uint64_t it) {
		uint64_t sg = blockIdx.x + it * gridDim.x;
		if (sg >= n_stages) return;
		uint32_t slot = (uint32_t)(it % NST);
		uint64_t off = sg * SB, avail = total_bytes_readable - off;
		uint32_t bytes = (uint32_t)(avail < SS ? (avail & ~15ull) : SS);
		mbar_expect(&bar[slot], bytes);
		bulk_g2s(smem + slot * SS, (const uint8_t *)p.text + off, bytes, &bar[slot]);
	};
	if (tid == 0) for (int i = 0; i < NST; i++) issue(i);
	for (uint64_t it = 0;; it++) {
		uint64_t sg = blockIdx.x + it * gridDim.x;
		if (sg >= n_stages) break;
		uint32_t slot = (uint32_t)(it % NST), parity = (uint32_t)((it / NST) & 1);
		mbar_wait(&bar[slot], parity);
		const uint8_t *st = smem + slot * SS;
#pragma unroll
		for (int c = 0; c < CH; c++) {
			uint32_t idx = c * T + tid;
			uint4 v = *reinterpret_cast<const uint4 *>(st + idx * 16);
			uint32_t x4;
			if (XMODE == 0) x4 = *reinterpret_cast<const uint32_t *>(st + idx * 16 + 16);
			else if (XMODE == 1) { x4 = __shfl_down_sync(0xffffffffu, v.x, 1); if (lane == 31) x4 = *reinterpret_cast<const uint32_t *>(st + idx * 16 + 16); }
			else { uint32_t a, b, c2, d; asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(c2), "=r"(d) : "r"(smem_u32(st + idx * 16 + 16))); x4 = a; }
			uint32_t acc = 0xffffffffu;
			acc = winpoly<NA, false>(v.x, v.y, p, acc); acc = winpoly<NA, false>(v.y, v.z, p, acc);
			acc = winpoly<NA, false>(v.z, v.w, p, acc); acc = winpoly<NA, false>(v.w, x4, p, acc);
			uint64_t chunk = sg * (uint64_t)T * CH + idx;
			bool flag = chunk < p.n_chunks && acc == 0;
			uint32_t word = __ballot_sync(0xffffffffu, flag);
			if (lane == 0 && chunk < p.n_chunks) p.bitmap[chunk >> 5] = word;
		}
		__syncthreads();
		if (tid == 0) issue(it + NST);
	}
}

template <int NA, int NST, int T, int CH, int XMODE = 0>
static void run_tma(const char *name, P p, uint64_t bytes, int sms, int bps)
{
	set_coef(p, NA);
	cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
	int smem = NST * (T * CH * 16 + 16);
	CK(cudaFuncSetAttribute(k_tma<NA, NST, T, CH, XMODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
	std::vector<float> ms;
	for (int it = 0; it < 6; it++) {
		CK(cudaEventRecord(e0));
		k_tma<NA, NST, T, CH, XMODE><<<sms * bps, T, smem>>>(p, bytes + 64);
		CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
		float t; CK(cudaEventElapsedTime(&t, e0, e1)); if (it >= 2) ms.push_back(t);
	}
	CK(cudaGetLastError());
	std::sort(ms.begin(), ms.end());
	printf("%-28s NA=%d NST=%d T=%d CH=%d X=%d grid=%dx%d smem=%d  %8.3f ms  %8.1f GB/s\n", name, NA, NST, T, CH, XMODE, sms, bps, smem, ms[0], bytes / ms[0] / 1e6);
	fflush(stdout);
}

__global__ void fill(uint32_t *t, uint64_t nwords, uint32_t seed)
{
	uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (uint64_t)gridDim.x * blockDim.x;
	for (; i < nwords; i += stride) {
		uint64_t z = (i + seed) * 0x9E3779B97F4A7C15ull; z ^= z >> 29; z *= 0xBF58476D1CE4E5B9ull; z ^= z >> 32;
		uint32_t w = 0;
		for (int b = 0; b < 4; b++) { uint32_t r = (z >> (b * 8)) & 31; w |= (r < 26 ? 'a' + r : (r < 31 ? ' ' : '\n')) << (8 * b); }
		t[i] = w;
	}
}

static void set_coef(P &p, int NA)
{
	// expand prod (x - A_i) mod 2^32: c[0..NA-1] low-order first, leading coefficient 1 implied
	uint32_t c[9] = {1, 0, 0, 0, 0, 0, 0, 0, 0}; int deg = 0;
	for (int i = 0; i < NA; i++) { uint32_t a = 0u - p.anchor[i]; for (int j = deg + 1; j >= 1; j--) c[j] = c[j - 1] + c[j] * a; c[0] = c[0] * a; deg++; }
	for (int i = 0; i < NA; i++) p.coef[i] = c[i];
	p.one = 1; p.scale = 256;
}

template <int V, int NA, int U, int T>
static void run(const char *name, P p, uint64_t bytes, int sms, int bps)
{
	set_coef(p, NA);
	cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
	int grid = sms * bps;
	std::vector<float> ms;
	for (int it = 0; it < 6; it++) {
		CK(cudaEventRecord(e0));
		k<V, NA, U, T><<<grid, T>>>(p);
		CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
		float t; CK(cudaEventElapsedTime(&t, e0, e1)); if (it >= 2) ms.push_back(t);
	}
	CK(cudaGetLastError());
	std::sort(ms.begin(), ms.end());
	printf("%-28s NA=%d U=%d T=%d grid=%dx%d  %8.3f ms  %8.1f GB/s\n", name, NA, U, T, sms, bps, ms[0], bytes / ms[0] / 1e6);
	fflush(stdout);
}

int main(int argc, char **argv)
{
	double gib = argc > 1 ? atof(argv[1]) : 4.0;
	uint64_t bytes = (uint64_t)(gib * (1ull << 30)) & ~511ull;
	uint32_t *text, *bitmap; CK(cudaMalloc(&text, bytes + 64)); CK(cudaMalloc(&bitmap, bytes / 128 + 64));
	cudaDeviceProp pr; CK(cudaGetDeviceProperties(&pr, 0));
	int sms = pr.multiProcessorCount;
	fill<<<sms * 8, 256>>>(text, bytes / 4, 1); CK(cudaDeviceSynchronize());
	printf("device %s, %d SMs, %.2f GiB text\n", pr.name, sms, gib);
	P p; p.text = (const uint4 *)text; p.bitmap = bitmap; p.n_chunks = bytes / 16; p.n_words = p.n_chunks / 32;
	const char *a[8] = { "beca", "use ", "each", "gove", "rnme", "ntal", "xyzw", "qqqq" };
	for (int i = 0; i < 8; i++) p.anchor[i] = *(const uint32_t *)a[i];
	run_tma<3, 4, 256, 4, 0>("tma-poly", p, bytes, sms, 3);
	run_tma<3, 4, 256, 4, 1>("tma-poly", p, bytes, sms, 3);
	run_tma<3, 4, 256, 4, 2>("tma-poly", p, bytes, sms, 3);
	run_tma<3, 3, 256, 4, 0>("tma-poly", p, bytes, sms, 4);
	run_tma<3, 3, 256, 4, 2>("tma-poly", p, bytes, sms, 4);
	run_tma<3, 2, 256, 4, 0>("tma-poly", p, bytes, sms, 6);
	run_tma<3, 4, 256, 2, 0>("tma-poly", p, bytes, sms, 5);
	run_tma<3, 8, 256, 2, 0>("tma-poly", p, bytes, sms, 3);
	run_tma<3, 4, 384, 4, 0>("tma-poly", p, bytes, sms, 2);
	run_tma<3, 4, 128, 8, 0>("tma-poly", p, bytes, sms, 3);
	run_tma<3, 4, 128, 4, 0>("tma-poly", p, bytes, sms, 6);
	run_tma<1, 4, 256, 4, 0>("tma-poly", p, bytes, sms, 3);
	run_tma<2, 4, 256, 4, 0>("tma-poly", p, bytes, sms, 3);
	run_tma<4, 4, 256, 4, 0>("tma-poly", p, bytes, sms, 3);
	run_tma<5, 4, 256, 4, 0>("tma-poly", p, bytes, sms, 3);
	return 0;
	run_tma<1, 6, 256, 4>("tma-poly", p, bytes, sms, 2);
	run_tma<3, 6, 256, 4>("tma-poly", p, bytes, sms, 2);
	run_tma<3, 4, 256, 4>("tma-poly", p, bytes, sms, 3);
	run_tma<3, 3, 512, 4>("tma-poly", p, bytes, sms, 1);
	run_tma<3, 6, 512, 2>("tma-poly", p, bytes, sms, 2);
	run_tma<3, 8, 128, 4>("tma-poly", p, bytes, sms, 4);
	run_tma<3, 4, 1024, 2>("tma-poly", p, bytes, sms, 1);
	run_tma<5, 6, 256, 4>("tma-poly", p, bytes, sms, 2);
	run_tma<2, 6, 256, 4>("tma-poly", p, bytes, sms, 2);
	// verify bitmaps agree between the register path and the TMA path
	{
		P q = p; set_coef(q, 3);
		std::vector<uint32_t> a(p.n_words), b(p.n_words);
		k<5, 3, 4, 256><<<sms * 8, 256>>>(q); CK(cudaMemcpy(a.data(), bitmap, p.n_words * 4, cudaMemcpyDeviceToHost));
		CK(cudaMemset(bitmap, 0xAA, p.n_words * 4));
		int smem = 6 * (256 * 4 * 16 + 16);
		CK(cudaFuncSetAttribute(k_tma<3, 6, 256, 4, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
		k_tma<3, 6, 256, 4, 0><<<sms * 2, 256, smem>>>(q, bytes + 64); CK(cudaMemcpy(b.data(), bitmap, p.n_words * 4, cudaMemcpyDeviceToHost));
		uint64_t diff = 0, set = 0; for (uint64_t i = 0; i < p.n_words; i++) { diff += a[i] != b[i]; set += __builtin_popcount(a[i]); }
		printf("bitmap check: %llu differing words of %llu, %llu bits set\n", (unsigned long long)diff, (unsigned long long)p.n_words, (unsigned long long)set);
	}
	run<9, 1, 4, 256>("stream-only", p, bytes, sms, 4);
	run<9, 1, 4, 256>("stream-only", p, bytes, sms, 4);
	run<0, 1, 4, 256>("viaddmnmx", p, bytes, sms, 8);
	run<0, 2, 4, 256>("viaddmnmx", p, bytes, sms, 8);
	run<0, 3, 4, 256>("viaddmnmx", p, bytes, sms, 8);
	run<0, 4, 4, 256>("viaddmnmx", p, bytes, sms, 8);
	run<0, 5, 4, 256>("viaddmnmx", p, bytes, sms, 8);
	run<1, 1, 4, 256>("isetp-or", p, bytes, sms, 8);
	run<1, 2, 4, 256>("isetp-or", p, bytes, sms, 8);
	run<1, 3, 4, 256>("isetp-or", p, bytes, sms, 8);
	run<1, 4, 4, 256>("isetp-or", p, bytes, sms, 8);
	run<1, 5, 4, 256>("isetp-or", p, bytes, sms, 8);
	run<2, 3, 4, 256>("xor+vimin3", p, bytes, sms, 8);
	run<3, 1, 4, 256>("imad-sub+vimin3", p, bytes, sms, 8);
	run<3, 3, 4, 256>("imad-sub+vimin3", p, bytes, sms, 8);
	run<3, 5, 4, 256>("imad-sub+vimin3", p, bytes, sms, 8);
	run<4, 3, 4, 256>("sub+min tree", p, bytes, sms, 8);
	run<5, 1, 4, 256>("poly", p, bytes, sms, 8);
	run<5, 2, 4, 256>("poly", p, bytes, sms, 8);
	run<5, 3, 4, 256>("poly", p, bytes, sms, 8);
	run<5, 3, 4, 256>("poly", p, bytes, sms, 4);
	run<5, 3, 8, 256>("poly", p, bytes, sms, 4);
	run<5, 3, 4, 128>("poly", p, bytes, sms, 8);
	run<5, 4, 4, 256>("poly", p, bytes, sms, 8);
	run<5, 5, 4, 256>("poly", p, bytes, sms, 8);
	run<5, 5, 4, 256>("poly", p, bytes, sms, 4);
	run<6, 3, 4, 256>("poly12+cmp4", p, bytes, sms, 8);
	run<6, 3, 4, 256>("poly12+cmp4", p, bytes, sms, 4);
	run<6, 5, 4, 256>("poly12+cmp4", p, bytes, sms, 8);
	run<7, 3, 4, 256>("poly8+cmp8", p, bytes, sms, 8);
	run<7, 5, 4, 256>("poly8+cmp8", p, bytes, sms, 8);
	run<8, 1, 4, 256>("poly*256", p, bytes, sms, 8);
	run<8, 3, 4, 256>("poly*256", p, bytes, sms, 8);
	run<4, 1, 4, 256>("sub+min tree", p, bytes, sms, 8);
	run<4, 5, 4, 256>("sub+min tree", p, bytes, sms, 8);
	run<4, 3, 4, 256>("sub+min tree", p, bytes, sms, 4);
	run<0, 3, 2, 256>("viaddmnmx", p, bytes, sms, 8);
	run<0, 3, 8, 256>("viaddmnmx", p, bytes, sms, 4);
	run<0, 3, 4, 128>("viaddmnmx", p, bytes, sms, 16);
	run<3, 3, 8, 256>("imad-sub+vimin3", p, bytes, sms, 4);
	run<3, 3, 2, 256>("imad-sub+vimin3", p, bytes, sms, 8);
	return 0;
}
