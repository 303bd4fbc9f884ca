/* agrep_b200/csrc/refine_kernel.cuh -- stage 1.5's kernel and its launch templates, included by the translation units
 * that instantiate it (refine_u32a.cu, refine_u32b.cu, refine_u64.cu, refine_costs.cu: split so that they build in parallel) */
#ifndef AGB_REFINE_KERNEL_CUH
#define AGB_REFINE_KERNEL_CUH
#include "automaton.cuh"

#define REFINE_RING1 544          /* flagged chunks: < 32 left over + 512 new per refill (16 bitmap words) */
#define REFINE_RING2 64           /* chunks with further hit windows */
#define REFINE_RING3 128          /* pattern starts that passed the count: < 32 left over + up to 3 x 32 from one batch of ring 2 */
#define REFINE_MAXG  8
#define REFINE_PAD   32           /* words behind the last strip: the count step may read a few words past a lane's strip */

/* the hit windows of a chunk: bit s of the result = some anchor starts at byte s.  Stage 1's polynomial over the
 * 16 windows (IMADs on the FMA pipe); f == 0 is folded into a bit per window without a compare: min(f, 1) shifted
 * into the mask by a multiply-add.  x[0..4]: the chunk and the word that follows it, case-folded like stage 1 does. */
struct AnchorTable { int8_t idx[32]; uint32_t val[16], mask[16]; int8_t off[16]; int n; };
/* mixed plans (four-byte and three-byte anchors; rare): every window against every anchor under that anchor's mask, from
 * the table in shared memory */
__device__ __forceinline__ uint32_t hit_windows_tab(const uint32_t (&x)[5], const AnchorTable &A)
{
	uint32_t hits = 0;
#pragma unroll
	for (int w = 0; w < 4; w++) {
		const uint32_t wv[4] = { x[w], __funnelshift_r(x[w], x[w + 1], 8), __funnelshift_r(x[w], x[w + 1], 16), __funnelshift_r(x[w], x[w + 1], 24) };
		for (int a = 0; a < A.n; a++) {
			const uint32_t V = A.val[a], M = A.mask[a];
#pragma unroll
			for (int j = 0; j < 4; j++) if ((wv[j] & M) == V) hits |= 1u << (4 * w + j);
		}
	}
	return hits;
}

template <int NA, bool SCALED>
__device__ __forceinline__ uint32_t hit_windows_poly(const uint32_t (&x)[5], const RefineParams &P)
{
	uint32_t wv[16];
#pragma unroll
	for (int w = 0; w < 4; w++) {
		wv[4 * w] = x[w]; wv[4 * w + 1] = __funnelshift_r(x[w], x[w + 1], 8);
		wv[4 * w + 2] = __funnelshift_r(x[w], x[w + 1], 16); wv[4 * w + 3] = __funnelshift_r(x[w], x[w + 1], 24);
	}
	uint32_t nz = 0;                                        /* bit s: window s is NOT a hit */
#pragma unroll
	for (int s = 15; s >= 0; s--) {
		uint32_t r = wv[s] * P.one + P.coef[NA - 1];
#pragma unroll
		for (int i = NA - 2; i >= 0; i--) r = r * wv[s] + P.coef[i];
		if (SCALED) r *= P.scale;
		nz = nz * 2u + min(r, 1u);
	}
	return ~nz & 0xFFFFu;
}
/* the same by comparing (anchors that stage 1's polynomial guard rejects) */
__device__ __forceinline__ uint32_t hit_windows_cmp(const uint32_t (&x)[5], const RefineParams &P)
{
	uint32_t hits = 0;
#pragma unroll
	for (int w = 0; w < 4; w++) {
		const uint32_t wv[4] = { x[w], __funnelshift_r(x[w], x[w + 1], 8), __funnelshift_r(x[w], x[w + 1], 16), __funnelshift_r(x[w], x[w + 1], 24) };
		for (int a = 0; a < P.na; a++) {
			const uint32_t A = P.anchor[a];
#pragma unroll
			for (int j = 0; j < 4; j++) if ((wv[j] & P.amask) == A) hits |= 1u << (4 * w + j);
		}
	}
	return hits;
}
template <bool SCALED>
__device__ __forceinline__ uint32_t hit_windows_na(const uint32_t (&x)[5], const RefineParams &P)
{
	switch (P.na) {
	case 1: return hit_windows_poly<1, SCALED>(x, P);  case 2: return hit_windows_poly<2, SCALED>(x, P);
	case 3: return hit_windows_poly<3, SCALED>(x, P);  case 4: return hit_windows_poly<4, SCALED>(x, P);
	case 5: return hit_windows_poly<5, SCALED>(x, P);  case 6: return hit_windows_poly<6, SCALED>(x, P);
	case 7: return hit_windows_poly<7, SCALED>(x, P);  case 8: return hit_windows_poly<8, SCALED>(x, P);
	default: return hit_windows_poly<9, SCALED>(x, P);
	}
}
__device__ __forceinline__ uint32_t hit_windows(const uint32_t (&x)[5], const RefineParams &P)
{
	if (!P.poly) return hit_windows_cmp(x, P);
	return P.scale != 1 ? hit_windows_na<true>(x, P) : hit_windows_na<false>(x, P);
}

/* the pattern start a hit window stands for: code = 32 + s - off of the anchor that starts at byte s of the chunk
 * (p0 = 16 * chunk + code - 32).  cw: the chunk's words in the lane's strip.  Which anchor it is: a multiplicative hash
 * of the window's bytes picks a slot (the host found a multiplier that keeps the anchors apart); the four-byte reading
 * of the window is tried first, then (mixed plans) the three-byte one. */
__device__ __forceinline__ uint32_t start_code(const uint32_t *cw, const int s, const RefineParams &P, const AnchorTable &A)
{
	const uint32_t lo = cw[s >> 2] | P.fold, hi = cw[(s >> 2) + 1] | P.fold;
	const uint32_t v = __funnelshift_r(lo, hi, (s & 3) * 8);
	int off = 0;
	{
		const uint32_t v4 = v & P.amask;
		const int i = A.idx[(v4 * P.hmul) >> 27];
		if (i && A.val[i - 1] == (v & A.mask[i - 1])) off = A.off[i - 1];
		else if (P.n3) {
			const uint32_t v3 = v & 0x00FFFFFFu;
			const int i3 = A.idx[(v3 * P.hmul) >> 27];
			if (i3 && A.val[i3 - 1] == (v & A.mask[i3 - 1])) off = A.off[i3 - 1];
		}
	}
	return (uint32_t)(32 + s - off);
}

/* T1, the band count: the literal pattern positions no byte of whose band matches, for the pattern start whose window
 * [p0 - k, p0 + pat_len + k) begins at byte `so` of the lane's strip.  One diagonal per iteration, the window moving
 * down one byte each time, so every compare is word against word at a fixed register.  Text bytes are cut to 7 bits
 * (and case-folded when the pattern asks for it): x + 0x7f sets bit 7 of a byte iff it differs, three operations per
 * word and diagonal; a cut byte can only match more often, which is the safe side. */
template <int NW, int NWT, int ND>
__device__ __forceinline__ bool band_count_passes(const RefineParams &P, const uint32_t *strip, const int so)
{
	uint32_t W[NWT + 1];
	{
		const uint32_t *src = strip + (so >> 2);
		const uint32_t sh = ((uint32_t)so & 3u) * 8u;
		uint32_t Lw[NWT + 1];
#pragma unroll
		for (int i = 0; i <= NWT; i++) Lw[i] = src[i];
#pragma unroll
		for (int i = 0; i < NWT; i++) W[i] = (__funnelshift_r(Lw[i], Lw[i + 1], sh) & 0x7F7F7F7Fu) | P.t1_fold;
		W[NWT] = 0;
	}
	uint32_t acc[NW];
#pragma unroll
	for (int w = 0; w < NW; w++) acc[w] = 0x80808080u;
	const int nd = ND ? ND : 2 * P.k + 1;                     /* ND: known at compile time for unit costs (k = rows - 1) */
#pragma unroll (ND ? ND : 1)
	for (int d = 0; d < nd; d++) {
#pragma unroll
		for (int w = 0; w < NW; w++) acc[w] &= (W[w] ^ P.t1_pat[w]) + 0x7F7F7F7Fu;
#pragma unroll
		for (int i = 0; i < NWT; i++) W[i] = __funnelshift_r(W[i], W[i + 1], 8);
	}
	int miss = 0;
#pragma unroll
	for (int w = 0; w < NW; w++) miss += __popc(acc[w] & P.t1_care[w]);
	return miss <= P.k;
}

/* the recurrence over one window: rows started at Init[0]; the end bits of the last row are sticky (Init1 holds
 * them, maskgen.c:232), so looking at it after the walk is enough.  Called by all lanes together; the bytes come
 * straight from the text (cache hits: the batch that found the start has just read them). */
template <typename T, int NR, bool COSTS>
__device__ __forceinline__ bool window_passes(const uint8_t *bytes, const bool run, const int wlen, const T init0,
                                              const T *mask, const DevConsts<T> &C)
{
	T S[NR];
#pragma unroll
	for (int r = 0; r < NR; r++) S[r] = init0;
	int q = 0;
	for (; q + 4 <= wlen; q += 4) {
		int c[4];
#pragma unroll
		for (int i = 0; i < 4; i++) c[i] = run ? (int)__ldg(bytes + q + i) : 0;
		T m[4];
#pragma unroll
		for (int i = 0; i < 4; i++) m[i] = mask[c[i]];
#pragma unroll
		for (int i = 0; i < 4; i++) rows_step<T, NR, COSTS>(S, m[i], C);
	}
	for (; q < wlen; q++) {
		const int c = run ? (int)__ldg(bytes + q) : 0;
		rows_step<T, NR, COSTS>(S, mask[c], C);
	}
	return run && (S[NR - 1] & C.endpos) != 0;
}

/* append the flagged chunks of the next 16 bitmap words to ring 1.  A warp loads 32 words at a time (one per lane, one
 * group ahead) and zeroes the same words of the survivor bitmap (every word of it is written here before any bit of it
 * is set below); the words go into the ring in two halves, so that it needs 31 + 512 entries (shared memory per warp
 * is what limits the warps in flight, and this stage lives on them: most of its time is spent waiting for text). */
struct Refill { uint32_t word, next_word; uint32_t half; };
__device__ __forceinline__ void refine_refill(const RefineParams &P, Refill &R, uint32_t *ring, uint32_t &count, uint32_t lane,
                                              uint64_t &g, uint64_t g_begin, uint64_t g_end)
{
	if (R.half == 0) {
		const uint64_t w = g * 32 + lane;
		R.word = R.next_word;
		if (w < P.n_words) P.out[w] = 0u;
		R.next_word = (g + 1 < g_end && w + 32 < P.n_words) ? P.bitmap[w + 32] : 0u;
	}
	const uint32_t word = ((lane >> 4) == R.half) ? R.word : 0u;
	uint32_t c = __popc(word), pre = c;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) { uint32_t v = __shfl_up_sync(0xffffffffu, pre, o); if (lane >= (uint32_t)o) pre += v; }
	const uint32_t total = __shfl_sync(0xffffffffu, pre, 31);
	pre += count - c;
	const uint32_t rel0 = (uint32_t)(g - g_begin) * 1024u + lane * 32u;
	for (uint32_t b = word; b; b &= b - 1) ring[pre++] = rel0 + (uint32_t)(__ffs(b) - 1);
	count += total;
	if (R.half) g++;
	R.half ^= 1u;
	__syncwarp();
}

/* six CTAs per SM (80 registers): at eight (64) the headline instantiation spilled 60 bytes, and on H100 it ran in 3.87 ms
 * instead of 4.80 ms at 32 GiB -- fewer warps in flight, but no local-memory traffic in the judging loop */
template <typename T, int NR, bool COSTS, int NW>
__global__ void __launch_bounds__(REFINE_THREADS, 6)
k_refine(const RefineParams P)
{
	constexpr int NGC = NW <= 4 ? 4 : REFINE_MAXG;          /* groups of text a lane keeps in flight */
	constexpr int NWT = NW + (2 * (NR - 1) + 3) / 4;        /* words of the window [p0 - k, p0 + 4 NW + k), k <= NR - 1 */
	extern __shared__ __align__(16) uint32_t s_strip[];     /* REFINE_THREADS x (ng * 4 + 1) words + REFINE_PAD */
	__shared__ RecShared<T, NR> SH;
	__shared__ uint32_t s_ring1[REFINE_THREADS / 32][REFINE_RING1];
	__shared__ uint32_t s_ring2[REFINE_THREADS / 32][REFINE_RING2];
	__shared__ uint32_t s_ring3[REFINE_THREADS / 32][REFINE_RING3];
	__shared__ AnchorTable s_offs;
	if (threadIdx.x == 0) {
		/* (static indexes: a kernel parameter indexed by a run-time value is copied to local memory as a whole, and every
		 * later P.x would be a local load) */
#pragma unroll
		for (int i = 0; i < 32; i++) s_offs.idx[i] = (int8_t)(P.hidx64[i >> 3] >> (8 * (i & 7)));
#pragma unroll
		s_offs.n = P.na + P.n3;
#pragma unroll
		for (int i = 0; i < 16; i++) { s_offs.val[i] = P.hval[i]; s_offs.mask[i] = P.hmask[i]; s_offs.off[i] = (int8_t)(P.hoffs64[i >> 3] >> (8 * (i & 7))); }
	}
	DevConsts<T> C;
	shared_init<T, NR>(SH, C, P.desc, REFINE_THREADS);
	const T init0 = mirror<T>((T)P.desc->init0);
	const int wlen = P.pat_len + 2 * P.k;
	const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5, lt_mask = (1u << lane) - 1u;
	uint32_t *ring1 = s_ring1[wib], *ring2 = s_ring2[wib], *ring3 = s_ring3[wib];
	const int stride_w = P.ng * 4 + 1;                      /* odd number of words: lanes hit different banks */
	uint32_t *strip = s_strip + threadIdx.x * stride_w;
	const uint32_t *cw = strip + P.gb * 4;                  /* the chunk itself */
	const int so0 = P.gb * 16 - 32 - P.k;                   /* window offset in the strip = so0 + start code */

	/* this warp's groups of 32 bitmap words: [g_begin, g_end) */
	const uint64_t warp = ((uint64_t)blockIdx.x * REFINE_THREADS + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * REFINE_THREADS) >> 5;
	const uint64_t n_groups = (P.n_words + 31) / 32, per = (n_groups + nwarps - 1) / nwarps;
	const uint64_t g_begin = warp * per < n_groups ? warp * per : n_groups, g_end = (g_begin + per < n_groups) ? g_begin + per : n_groups;
	const uint64_t chunk0 = g_begin * 1024;                 /* ring entries are chunk numbers relative to this */
	/* chunks whose windows touch the virtual '\n', the appended delimiter or the end of the buffer are not judged but kept:
	 * as bounds on the relative chunk number */
	uint32_t rel_lo, rel_hi;
	{
		const int64_t lo_chunk = ((int64_t)P.lo_off + 15) / 16;                                     /* first chunk with base - lo_off >= 0 */
		int64_t hi_chunk = ((int64_t)P.n - P.hi_off - 16) / 16;                                     /* last chunk with base + hi_off + 16 <= n */
		if ((int64_t)P.n - P.hi_off - 16 < 0) hi_chunk = -1;
		if (hi_chunk > (int64_t)P.n_chunks - 3) hi_chunk = (int64_t)P.n_chunks - 3;
		const int64_t a = lo_chunk - (int64_t)chunk0, b = hi_chunk - (int64_t)chunk0;
		rel_lo = a < 0 ? 0u : (a > 0x7fffffff ? 0x7fffffffu : (uint32_t)a);
		rel_hi = b < 0 ? 0u : (b > 0x7fffffff ? 0x7fffffffu : (uint32_t)b);
		if (b < 0) rel_lo = 0x7fffffffu;                    /* nothing can be judged */
	}
	const uint4 *text4 = reinterpret_cast<const uint4 *>(P.text) + chunk0;
	uint32_t kept = 0;                                      /* survivor bits this lane set */
	auto keep_chunk = [&](uint32_t rel) {
		const uint64_t chunk = chunk0 + rel;
		const uint32_t bit = 1u << (chunk & 31);
		const uint32_t old = atomicOr(&P.out[chunk >> 5], bit);
		kept += (old & bit) ? 0u : 1u;
	};

	uint32_t n1 = 0, n2 = 0, n3 = 0;                        /* warp-uniform ring fills */
	uint64_t g = g_begin;
	Refill RF; RF.word = 0; RF.half = 0;
	RF.next_word = (g < g_end && g * 32 + lane < P.n_words) ? P.bitmap[g * 32 + lane] : 0u;     /* one group ahead */
	auto fill1 = [&]() { while (n1 < 32 && g < g_end) refine_refill(P, RF, ring1, n1, lane, g, g_begin, g_end); };
	/* the batch in flight: popped, its text on the way into registers */
	uint32_t nrel = 0; bool nrun = false, nedge = false; uint4 nx[NGC];
	auto pop_load = [&](uint32_t rel, bool active) {
		nrel = rel;
		nedge = active && (rel < rel_lo || rel > rel_hi);
		nrun = active && !nedge;
		if (nrun) {
			const uint4 *src = text4 + ((int64_t)rel - P.gb);
#pragma unroll
			for (int gi = 0; gi < NGC; gi++) if (gi < P.ng) nx[gi] = __ldg(src + gi);
		}
	};
	auto to_strip = [&]() {
#pragma unroll
		for (int gi = 0; gi < NGC; gi++) if (gi < P.ng) {
			strip[gi * 4 + 0] = nx[gi].x; strip[gi * 4 + 1] = nx[gi].y; strip[gi * 4 + 2] = nx[gi].z; strip[gi * 4 + 3] = nx[gi].w;
		}
	};
	/* count step for one start code of the chunk in the strip; passes go to ring 3 (called by all lanes) */
	auto count_push = [&](uint32_t rel, uint32_t code, bool run) {
		const bool pass = run && (!P.t1 || band_count_passes<NW, NWT, COSTS ? 0 : 2 * (NR - 1) + 1>(P, strip, so0 + (int)code));
		const uint32_t pm = __ballot_sync(0xffffffffu, pass);
		if (pass) ring3[n3 + __popc(pm & lt_mask)] = (rel << 6) | code;
		n3 += __popc(pm);
	};
	auto walk_batch = [&]() {
		const uint32_t m = n3 < 32 ? n3 : 32;
		const bool run = lane < m;
		const uint32_t e = run ? ring3[n3 - m + lane] : 0u;
		n3 -= m;
		const uint8_t *wbytes = P.text + ((int64_t)(chunk0 + (e >> 6)) * 16 + (int64_t)(e & 63u) - 32 - P.k);
		if (window_passes<T, NR, COSTS>(run ? wbytes : P.text, run, wlen, init0, SH.mask, C)) keep_chunk(e >> 6);
		__syncwarp();
	};
	/* chunks with more than one hit window: the rest of their windows, one lane per chunk, usually the same start again
	 * ("beca" and "use " of one "because ") */
	auto more_batch = [&]() {
		const uint32_t m = n2 < 32 ? n2 : 32;
		const bool run = lane < m;
		const uint32_t e = run ? ring2[n2 - m + lane] : 0u;
		n2 -= m;
		const uint32_t rel = e >> 6, first = e & 63u;
		if (run) {
			const uint4 *src = text4 + ((int64_t)rel - P.gb);
#pragma unroll
			for (int gi = 0; gi < NGC; gi++) if (gi < P.ng) {
				const uint4 v = __ldg(src + gi);
				strip[gi * 4 + 0] = v.x; strip[gi * 4 + 1] = v.y; strip[gi * 4 + 2] = v.z; strip[gi * 4 + 3] = v.w;
			}
		}
		uint32_t hits = 0;
		if (run) {
			const uint32_t x[5] = { cw[0] | P.fold, cw[1] | P.fold, cw[2] | P.fold, cw[3] | P.fold, cw[4] | P.fold };
			hits = P.n3 ? hit_windows_tab(x, s_offs) : hit_windows(x, P);
			hits &= hits - 1;                                 /* the first one has been judged */
		}
		uint32_t seen1 = first, seen2 = first;
		for (int it = 0; it < 3; it++) {                      /* up to three further windows; a chunk with more is kept as it is */
			if (!__ballot_sync(0xffffffffu, hits != 0)) break;
			uint32_t code = first; bool fresh = false;
			if (hits) {
				code = start_code(cw, __ffs(hits) - 1, P, s_offs);
				hits &= hits - 1;
				fresh = code != first && code != seen1 && code != seen2;
				seen2 = seen1; seen1 = code;
			}
			count_push(rel, code, fresh);
		}
		if (hits) keep_chunk(rel);
		__syncwarp();
	};
	auto pop1 = [&]() {
		const uint32_t m = n1 < 32 ? n1 : 32;
		const bool active = lane < m;
		pop_load(active ? ring1[n1 - m + lane] : 0u, active);
		n1 -= m;
	};

	bool have = false;
	for (;;) {
		if (n3 >= 32) { walk_batch(); continue; }
		if (n2 >= 32) { more_batch(); continue; }
		if (!have) {
			fill1();
			if (n1 == 0) break;                               /* range done (what is left in rings 2 and 3 is drained below) */
			pop1(); have = true;
			continue;
		}
		/* ---- the batch in nx[]: into the strips; the next one starts loading while this one is judged ---- */
		const uint32_t crel = nrel; const bool crun = nrun, cedge = nedge;
		if (crun) to_strip();
		fill1();
		have = n1 != 0;                                       /* fewer than 32 only when the range is exhausted */
		if (have) pop1();
		if (cedge) keep_chunk(crel);
		uint32_t hits = 0, code = 0;
		if (crun) {
			const uint32_t x[5] = { cw[0] | P.fold, cw[1] | P.fold, cw[2] | P.fold, cw[3] | P.fold, cw[4] | P.fold };
			hits = P.n3 ? hit_windows_tab(x, s_offs) : hit_windows(x, P);
			if (hits) code = start_code(cw, __ffs(hits) - 1, P, s_offs);
		}
		count_push(crel, code, hits != 0);
		{   /* further hit windows wait in ring 2 -- unless there is just one and it is the same start again ("beca" and
			 * "use " of one "because "), the usual case */
			uint32_t rest = hits & (hits - 1);
			if (rest && !(rest & (rest - 1)) && start_code(cw, __ffs(rest) - 1, P, s_offs) == code) rest = 0;
			const bool more = rest != 0;
			const uint32_t mm = __ballot_sync(0xffffffffu, more);
			if (more) ring2[n2 + __popc(mm & lt_mask)] = (crel << 6) | code;
			n2 += __popc(mm);
		}
		__syncwarp();
	}
	while (n2 || n3) { if (n3 >= 32 || !n2) walk_batch(); else more_batch(); }
	const uint32_t total = __reduce_add_sync(0xffffffffu, kept);
	if (lane == 0) P.warp_counts[warp] = total;
}

/* one wave: as many CTAs as the device holds at once (each warp's range is fixed up front, so a second, partial wave
 * would leave most SMs idle for its whole length), never more than there are groups of bitmap words */
template <typename T, int NR, bool COSTS, int NW>
static void launch_refine_nw(const RefineParams &P, unsigned &grid, cudaStream_t st)
{
	const size_t smem = ((size_t)REFINE_THREADS * (P.ng * 4 + 1) + REFINE_PAD) * sizeof(uint32_t);
	int per_sm = 0;
	if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_refine<T, NR, COSTS, NW>, REFINE_THREADS, smem) != cudaSuccess || per_sm < 1) per_sm = 4;
	grid = std::min<unsigned>(grid, (unsigned)per_sm * (unsigned)P.sm_count);
	if (!grid) grid = 1;
	k_refine<T, NR, COSTS, NW><<<grid, REFINE_THREADS, smem, st>>>(P);
}
/* the count step keeps the pattern words (and up to 4 more of the window) in registers: kernels for 2, 3, 4, 6, 8
 * pattern words with 32-bit rows (M <= 31: at most 29 pattern bytes), 8, 12, 16 with 64-bit rows; cost patterns
 * (asearch1, rare) take the widest */
template <typename T, int NR, bool COSTS>
static void launch_refine_one(const RefineParams &P, unsigned &grid, cudaStream_t st)
{
	const int pw = (P.pat_len + 3) / 4;
	if (COSTS) { if (sizeof(T) == 4) launch_refine_nw<T, NR, COSTS, 8>(P, grid, st); else launch_refine_nw<T, NR, COSTS, 16>(P, grid, st); return; }
	if (sizeof(T) == 4) {
		if (pw <= 2) launch_refine_nw<T, NR, COSTS, 2>(P, grid, st);
		else if (pw == 3) launch_refine_nw<T, NR, COSTS, 3>(P, grid, st);
		else if (pw == 4) launch_refine_nw<T, NR, COSTS, 4>(P, grid, st);
		else if (pw <= 6) launch_refine_nw<T, NR, COSTS, 6>(P, grid, st);
		else launch_refine_nw<T, NR, COSTS, 8>(P, grid, st);
	} else {
		if (pw <= 8) launch_refine_nw<T, NR, COSTS, 8>(P, grid, st);
		else if (pw <= 12) launch_refine_nw<T, NR, COSTS, 12>(P, grid, st);
		else launch_refine_nw<T, NR, COSTS, 16>(P, grid, st);
	}
}

#endif
