/* agrep_b200/csrc/automaton.cuh -- the device pieces stages 1.5 and 2 share */
#ifndef AGB_AUTOMATON_CUH
#define AGB_AUTOMATON_CUH
#include "scan_internal.cuh"
#include <type_traits>

/* ================================================================================================
 * shared device pieces of stages 1.5 and 2: the recurrence, the match test, the text reader
 * ============================================================================================== */
/* 32-bit rows run on the MIRRORED automaton: every word that holds pattern positions -- character masks, Init0/1,
 * NO_ERR_MASK, endposition, D_endpos, the reset and start rows -- is bit-reversed (__brev) when it is loaded, which
 * turns the recurrence's `>> 1` into `<< 1` and changes nothing else (the kernels only ever AND/OR/compare these
 * words).  A left shift by one is a multiply by two, and IMAD runs on the FMA pipe, which these kernels leave idle,
 * instead of the ALU pipe that bounds them: 5 ALU + 2 FMA operations per row and byte instead of 7 ALU.
 * 64-bit rows (M > 31) stay as the reference has them. */
template <typename T> __device__ __forceinline__ T mirror(T x) { return x; }
template <> __device__ __forceinline__ uint32_t mirror<uint32_t>(uint32_t x) { return __brev(x); }
template <typename T> __device__ __forceinline__ T shift1(T x) { return x >> 1; }
template <> __device__ __forceinline__ uint32_t shift1<uint32_t>(uint32_t x)
{
	uint32_t r;
	asm("mad.lo.u32 %0, %1, 2, 0;" : "=r"(r) : "r"(x));
	return r;
}

/* a 320-bit row (agb_wide: a simple literal of more than 63 positions, k = 0..8), word 0 = bits 0..63.  The kernels only
 * AND/OR/complement/compare rows and shift them right by one, so this is all a row needs. */
struct Wide {
	uint64_t w[AGB_WIDE_WORDS];
	Wide() = default;
	__device__ __forceinline__ Wide(int z) { w[0] = (uint64_t)(uint32_t)z; _Pragma("unroll") for (int i = 1; i < AGB_WIDE_WORDS; i++) w[i] = 0; }
	__device__ __forceinline__ static Wide load(const uint64_t (&x)[AGB_WIDE_WORDS]) { Wide r; _Pragma("unroll") for (int i = 0; i < AGB_WIDE_WORDS; i++) r.w[i] = x[i]; return r; }
	__device__ __forceinline__ explicit operator bool() const { uint64_t o = 0; _Pragma("unroll") for (int i = 0; i < AGB_WIDE_WORDS; i++) o |= w[i]; return o != 0; }
#define WIDE_OP(op) \
	__device__ __forceinline__ friend Wide operator op(const Wide &a, const Wide &b) { Wide r; _Pragma("unroll") for (int i = 0; i < AGB_WIDE_WORDS; i++) r.w[i] = a.w[i] op b.w[i]; return r; } \
	__device__ __forceinline__ Wide &operator op##=(const Wide &b) { _Pragma("unroll") for (int i = 0; i < AGB_WIDE_WORDS; i++) w[i] op##= b.w[i]; return *this; }
	WIDE_OP(&) WIDE_OP(|)
#undef WIDE_OP
	__device__ __forceinline__ Wide operator~() const { Wide r; _Pragma("unroll") for (int i = 0; i < AGB_WIDE_WORDS; i++) r.w[i] = ~w[i]; return r; }
	__device__ __forceinline__ friend bool operator==(const Wide &a, const Wide &b) { uint64_t o = 0; _Pragma("unroll") for (int i = 0; i < AGB_WIDE_WORDS; i++) o |= a.w[i] ^ b.w[i]; return o == 0; }
	__device__ __forceinline__ friend bool operator!=(const Wide &a, const Wide &b) { return !(a == b); }
};
template <> __device__ __forceinline__ Wide shift1<Wide>(Wide x)
{
	Wide r;
#pragma unroll
	for (int i = 0; i < AGB_WIDE_WORDS - 1; i++) r.w[i] = (x.w[i] >> 1) | (x.w[i + 1] << 63);
	r.w[AGB_WIDE_WORDS - 1] = x.w[AGB_WIDE_WORDS - 1] >> 1;
	return r;
}

template <typename T> struct DevConsts {
	T init1, noerr, endpos, dendpos;
	int L, k, and_mode, inverse, kind, ci, cs, cd;
};

template <typename T, int NR> struct RecShared {
	T mask[257];                 /* mask[256] = 0: "a byte outside the text" */
	T reset[NR], start[NR];
	uint8_t delim[2 * AGB_MAXDELIM + 2];     /* lower case where both cases end a record (dfold) */
	uint8_t dfold[2 * AGB_MAXDELIM + 2];
	unsigned long long hist[AGB_MAXERR + 1];
	int start_closes;
};

/* wide: the words come from the agb_wide table in device memory (RecParams.rx_tab), the rest from the descriptor */
template <typename T, int NR>
__device__ __forceinline__ void shared_init(RecShared<T, NR> &S, DevConsts<T> &C, const agb_desc *D, int nthreads, const void *wide = nullptr)
{
	if constexpr (std::is_same<T, Wide>::value) {
		const agb_wide *X = static_cast<const agb_wide *>(wide);
		for (int i = threadIdx.x; i < 256; i += nthreads) S.mask[i] = Wide::load(X->mask[i]);
		if (threadIdx.x == 0) { S.reset[0] = Wide::load(X->reset); S.start[0] = Wide::load(X->start); }
		if (threadIdx.x >= 1 && threadIdx.x < NR) { S.reset[threadIdx.x] = Wide::load(X->reset_up[threadIdx.x - 1]); S.start[threadIdx.x] = Wide::load(X->start_up[threadIdx.x - 1]); }
		C.init1 = Wide::load(X->init1); C.noerr = Wide::load(X->noerr); C.endpos = Wide::load(X->endpos); C.dendpos = Wide::load(X->dendpos);
	} else {
		for (int i = threadIdx.x; i < 256; i += nthreads) S.mask[i] = mirror<T>((T)D->mask[i]);
		if (threadIdx.x < NR) { S.reset[threadIdx.x] = mirror<T>((T)D->reset[threadIdx.x]); S.start[threadIdx.x] = mirror<T>((T)D->start[threadIdx.x]); }
		C.init1 = mirror<T>((T)D->init1); C.noerr = mirror<T>((T)D->noerr); C.endpos = mirror<T>((T)D->endpos); C.dendpos = mirror<T>((T)D->dendpos);
	}
	if (threadIdx.x == 0) { S.mask[256] = 0; S.start_closes = D->start_closes; }
	if (threadIdx.x < 2 * AGB_MAXDELIM + 2) { S.dfold[threadIdx.x] = D->delim_fold[threadIdx.x]; S.delim[threadIdx.x] = D->delim[threadIdx.x] | D->delim_fold[threadIdx.x]; }
	if (threadIdx.x <= AGB_MAXERR) S.hist[threadIdx.x] = 0;
	C.L = D->L; C.k = D->k; C.and_mode = D->and_mode; C.inverse = D->inverse; C.kind = D->delim_kind;
	C.ci = D->cost_i; C.cs = D->cost_s; C.cd = D->cost_d;
	__syncthreads();
}

/* text reader with a one-group (16 byte) register cache; positions are file offsets.
 * -1 is the virtual '\n' (bitap.c:140), n..n+L-1 the delimiter appended at EOF (bitap.c:161-165). */
struct Reader {
	const uint8_t *text; uint64_t n; const uint8_t *delim; int L;
	uint4 v; int64_t grp;
	__device__ __forceinline__ void init(const uint8_t *t, uint64_t n_, const uint8_t *d, int L_) { text = t; n = n_; delim = d; L = L_; grp = -1; v = make_uint4(0, 0, 0, 0); }
	__device__ __forceinline__ int get(int64_t p)
	{
		if (p < 0) return p == -1 ? '\n' : 256;
		if ((uint64_t)p >= n) { int64_t o = p - (int64_t)n; return o < L ? delim[o] : 256; }
		int64_t g = p >> 4;
		if (g != grp) { v = __ldg(reinterpret_cast<const uint4 *>(text) + g); grp = g; }
		uint32_t sel = (uint32_t)(p >> 2) & 3u;
		uint32_t w = sel == 0 ? v.x : (sel == 1 ? v.y : (sel == 2 ? v.z : v.w));
		return (int)((w >> (((uint32_t)p & 3u) * 8u)) & 0xFFu);
	}
};

/* the same reader in front of a stretch of the text that the thread has staged in shared memory: [lo, lo + len) comes
 * from there (one LDS), everything else from the slow path above */
struct WindowReader {
	Reader R; const uint8_t *sm; int64_t lo; uint32_t len;
	__device__ __forceinline__ void init(const uint8_t *t, uint64_t n_, const uint8_t *d, int L_) { R.init(t, n_, d, L_); sm = nullptr; lo = 0; len = 0; }
	__device__ __forceinline__ int get(int64_t p)
	{
		const uint64_t o = (uint64_t)(p - lo);
		if (o < (uint64_t)len) return sm[o];
		return R.get(p);
	}
};

/* does the delimiter occur with its last byte at q (file offset)? */
template <typename RD>
__device__ __forceinline__ bool delim_occurs(RD &R, int64_t q, const uint8_t *delim, const uint8_t *dfold, int L)
{
	for (int t = 0; t < L; t++) if ((R.get(q - t) | dfold[L - 1 - t]) != delim[L - 1 - t]) return false;
	return true;
}

/* kind 2 -- a delimiter that overlaps itself and is not a run ("aba", "=-="): the automaton takes occurrences from the
 * left and drops those that share a byte with one it took (after a close the state keeps no delimiter position:
 * asearch.c:55-57, 175-186).  Occurrences that share bytes form a chain, and what is taken in a chain depends only on
 * where the chain starts: walk back to its first occurrence, then forward. */
template <typename RD>
__device__ __noinline__ int64_t delim_chain_first(RD &R, int64_t q, const uint8_t *delim, const uint8_t *dfold, int L)
{
	int64_t e = q;
	for (;;) {
		int64_t found = e;
		for (int64_t c = e - L + 1; c < e; c++) if (delim_occurs(R, c, delim, dfold, L)) { found = c; break; }
		if (found == e) return e;
		e = found;
	}
}
template <typename RD>
__device__ __noinline__ bool delim_chain_takes(RD &R, int64_t q, const uint8_t *delim, const uint8_t *dfold, int L)
{
	int64_t last = delim_chain_first(R, q, delim, dfold, L);
	for (int64_t e = last + 1; e <= q; e++) if (e - L + 1 > last && delim_occurs(R, e, delim, dfold, L)) last = e;
	return last == q;
}

/* is q (file offset, < n) the last byte of a delimiter that closes a record?  kind 0: every occurrence
 * does (no self overlap); kind 1 (c^L, e.g. $$): greedy, non-overlapping from the start of the run of c,
 * the virtual '\n' counting as part of the run (asearch.c:55-57 D_Mask + the reset at :181); kind 2: above. */
template <typename RD>
__device__ __forceinline__ bool delim_ends_at(RD &R, int64_t q, const uint8_t *delim, const uint8_t *dfold, int L, int kind)
{
	if (L == 1) return (R.get(q) | dfold[0]) == delim[0];
	if (kind == 0) return delim_occurs(R, q, delim, dfold, L);
	if (kind == 2) return delim_occurs(R, q, delim, dfold, L) && delim_chain_takes(R, q, delim, dfold, L);
	const int c = delim[0], f = dfold[0];
	if ((R.get(q) | f) != c) return false;
	int64_t len = 1, p = q - 1;
	while (p >= -1 && (R.get(p) | f) == c) { len++; p--; }
	return (len % L) == 0;
}

/* delim_kind 3 (-p, L >= 2): the delimiter's state s (positions 1..s taken since the last close) on byte c, which takes
 * position s + 1 or not; the L-th closes the record and starts over (delim_state.cu).  true: c closes a record */
__device__ __forceinline__ bool dstate_step(int &s, int c, const uint8_t *delim, const uint8_t *dfold, int L)
{
	if ((c | dfold[s]) != delim[s]) return false;
	if (++s < L) return false;
	s = 0;
	return true;
}

/* one text byte through all rows: asearch.c:96-115 (unit costs), asearch1.c:88-97 (COSTS), bitap.c:175-176 (NR = 1) */
template <typename T, int NR, bool COSTS>
__device__ __forceinline__ void rows_step(T (&S)[NR], T cm, const DevConsts<T> &C)
{
	if (!COSTS) {
		T prevB = S[0];
		T prevA = (shift1<T>(prevB) & cm) | (C.init1 & prevB);
#pragma unroll
		for (int r = 1; r < NR; r++) {
			T b = S[r];
			T a = (shift1<T>(b) & cm) | (C.init1 & b) | prevB | (shift1<T>(prevA | prevB) & C.noerr);
			S[r - 1] = prevA; prevA = a; prevB = b;
		}
		S[NR - 1] = prevA;
	} else {
		T A[NR];
		A[0] = (shift1<T>(S[0]) & cm) | (C.init1 & S[0]);
#pragma unroll
		for (int r = 1; r < NR; r++) {
			T bi = (r - C.ci >= 0) ? S[r - C.ci] : (T)0, ad = (r - C.cd >= 0) ? A[r - C.cd] : (T)0, bs = (r - C.cs >= 0) ? S[r - C.cs] : (T)0;
			A[r] = (shift1<T>(S[r]) & cm) | bi | (shift1<T>(ad | bs) & C.noerr) | (C.init1 & S[r]);
		}
#pragma unroll
		for (int r = 0; r < NR; r++) S[r] = A[r];
	}
}

template <typename T>
__device__ __forceinline__ bool match_cond(T r, const DevConsts<T> &C)
{
	/* bitap.c:182, asearch.c:128 -- C precedence: (AND && all) || ((!AND && any) ^ INVERSE) */
	if (C.and_mode) return ((r & C.endpos) == C.endpos) || (C.inverse != 0);
	return ((r & C.endpos) != 0) != (C.inverse != 0);
}

#endif
