/* agrep_b200/csrc/delim_state.cu -- where the records of a -p pattern with a delimiter of two or more bytes begin
 * (delim_kind 3, DESIGN.md 3.3.1).
 *
 * -p makes every position of the automaton sticky (Init1 = ~0, bitap.c:123, asearch.c:49), the delimiter's too, and
 * those positions are fed by the always-on bits alone.  So row 0's delimiter state is a function of the text: state s
 * (positions 1..s taken since the last close), byte c takes position s + 1 or not, the L-th closes the record and starts
 * over (the & D_Mask reset, bitap.c:223-225).  Where a record begins can then depend on any stretch of text before it,
 * which no local search by the delimiter's bytes can see; this pass gives every 128-byte slice of [0, n + L) the state
 * it is entered in, and the consumers (the dense tile form, the ordinals) walk their slices from there.
 *
 * A slice's transition function maps the L states to L states.  It is computed for all of them at once: one word whose
 * byte s holds the set of start states that are in state s now; per text byte a table lookup gives the bytes (positions)
 * that accept it, the sets in those bytes move one byte up -- the L-th byte back to byte 0 -- the others stay.  States
 * need not converge (-d aa keeps two start states apart for ever), so the whole function is kept: 4 bits per state.
 *   k_dstate_tiles (count form)  the function of every 32 KiB tile (a block scan of its 256 slice functions)
 *   k_dstate_scan                one block: the tile functions composed in order from the state after the virtual
 *                                '\n' -> the state every tile is entered in
 *   k_dstate_tiles (apply form)  the same slice functions again, each slice's entry state from its tile's
 * The text is read twice; the result is one byte per 128 bytes of text.  In a set of files every file starts over from
 * the virtual '\n' (its tiles are those of the ordinals, SetFile.ord_tile0). */
#include "scan_internal.cuh"

#define DS_THREADS 256
#define DS_PER     128                                  /* = DENSE_PER = ORD_PER: a consumer thread's slice */
#define DS_TILE    (DS_THREADS * DS_PER)
#define DS_STRIDE  (DS_PER + 16)                        /* slices in shared memory 144 bytes apart: 16-byte reads without conflicts */
static_assert(DS_TILE == ORD_TILE && DS_TILE == DENSE_TILE && DS_PER == DENSE_PER, "a slice of this pass is a slice of its consumers");

#define DS_IDENTITY 0x76543210u                         /* function: 4 bits per state, state s -> nibble s */

__device__ __forceinline__ uint32_t ds_apply(uint32_t f, uint32_t s) { return (f >> (4 * s)) & 15u; }
/* f, then g */
__device__ __forceinline__ uint32_t ds_compose(uint32_t f, uint32_t g)
{
	uint32_t r = 0;
#pragma unroll
	for (uint32_t s = 0; s < 8; s++) r |= ds_apply(g, ds_apply(f, s)) << (4 * s);
	return r;
}
__device__ __forceinline__ uint32_t ds_const(uint32_t s) { return s * 0x11111111u; }

struct DsParams {
	const uint8_t *text; uint64_t n;                   /* whole text (SET: the set's buffer; each tile finds its file) */
	uint8_t delim[AGB_MAXDELIM], dfold[AGB_MAXDELIM];  /* delim: folded (lower case where dfold is 0x20), appended at EOF */
	int L, seed;                                       /* seed: the state after the virtual '\n' */
	uint64_t n_tiles;
	uint32_t *func;                                    /* per tile: its transition function */
	uint8_t *entry;                                    /* per tile: the state it is entered in */
	uint8_t *state;                                    /* per slice (256 per tile): the state it is entered in */
	const SetFile *set_files; const SetTile *set_tiles; /* SET: tile b is tile set_tiles[b].tile of [0, n + L) of its file */
};

/* one slice's function: SWAR over the start states, T = uint32_t for L <= 4, uint64_t for L <= 8 */
template <typename T>
__device__ __forceinline__ uint32_t ds_slice_func(const uint8_t *sl, int len, const T *tab, int L)
{
	const T lowL = (L * 8 >= (int)(8 * sizeof(T))) ? ~(T)0 : (((T)1 << (8 * L)) - 1);
	const int back = 8 * (L - 1);
	T x = 0;
	for (int s = 0; s < L; s++) x |= (T)1 << (9 * s);           /* byte s = {s} */
	for (int v = 0; v < DS_PER / 16 && 16 * v < len; v++) {
		const uint4 q = *reinterpret_cast<const uint4 *>(sl + 16 * v);
		const uint32_t w[4] = { q.x, q.y, q.z, q.w };
		const int m = len - 16 * v;
#pragma unroll
		for (int b = 0; b < 16; b++) {
			const T t = b < m ? tab[(w[b >> 2] >> (8 * (b & 3))) & 0xFFu] : (T)0;     /* (past the end: no position takes it) */
			const T adv = x & t;
			x = (x & ~t) | (((adv << 8) | (adv >> back)) & lowL);
		}
	}
	uint32_t f = DS_IDENTITY;
	for (int s = 0; s < L; s++) {
		const uint64_t at = (uint64_t)(x >> s) & 0x0101010101010101ull;      /* one byte holds start state s */
		const uint32_t to = (uint32_t)(__ffsll((long long)at) - 1) >> 3;
		f = (f & ~(15u << (4 * s))) | (to << (4 * s));
	}
	return f;
}

/* APPLY = false: tile functions into P.func; true: slice entry states into P.state from P.entry */
template <bool APPLY, bool SET, typename T>
__global__ void __launch_bounds__(DS_THREADS) k_dstate_tiles(const DsParams P)
{
	extern __shared__ __align__(16) uint8_t s_sl[];                    /* DS_THREADS slices, DS_STRIDE apart */
	__shared__ T s_tab[256];
	__shared__ uint32_t s_f[DS_THREADS];
	const uint32_t tid = threadIdx.x;
	const uint8_t *text = P.text; uint64_t n = P.n, tile = blockIdx.x; uint32_t file = 0;
	if constexpr (SET) set_enter(P.set_files, P.set_tiles, text, n, tile, file);
	{   /* byte c -> the delimiter positions that take it (byte s of the entry: position s + 1) */
		T t = 0;
		for (int s = 0; s < P.L; s++) if (((int)tid | P.dfold[s]) == P.delim[s]) t |= (T)0xFF << (8 * s);
		s_tab[tid] = t;
	}
	const int64_t tile0 = (int64_t)tile * DS_TILE, limit = (int64_t)n + P.L;
	/* the tile into shared memory, 16 bytes per load; past the text the appended delimiter, then nothing */
	for (int g = tid; g < DS_TILE / 16; g += DS_THREADS) {
		const int64_t p = tile0 + 16 * (int64_t)g;
		uint8_t *dst = s_sl + (g / (DS_PER / 16)) * DS_STRIDE + (g % (DS_PER / 16)) * 16;
		if (p + 16 <= (int64_t)n) *reinterpret_cast<uint4 *>(dst) = __ldg(reinterpret_cast<const uint4 *>(text + p));
		else if (p < limit)
			for (int b = 0; b < 16; b++) dst[b] = p + b < (int64_t)n ? text[p + b] : (p + b < limit ? P.delim[p + b - (int64_t)n] : 0);
	}
	__syncthreads();
	const int64_t s0 = tile0 + (int64_t)tid * DS_PER;
	const int len = s0 >= limit ? 0 : (limit - s0 < DS_PER ? (int)(limit - s0) : DS_PER);
	/* inclusive scan of the slice functions in order (Hillis-Steele: 8 steps of a cheap composition) */
	uint32_t f = ds_slice_func<T>(s_sl + tid * DS_STRIDE, len, s_tab, P.L);
	s_f[tid] = f;
	__syncthreads();
	for (uint32_t off = 1; off < DS_THREADS; off <<= 1) {
		const uint32_t before = tid >= off ? s_f[tid - off] : DS_IDENTITY;
		__syncthreads();
		f = ds_compose(before, f);
		s_f[tid] = f;
		__syncthreads();
	}
	const uint64_t gtile = SET ? (uint64_t)P.set_files[file].ord_tile0 + tile : tile;
	if (!APPLY) { if (tid == DS_THREADS - 1) P.func[gtile] = f; }
	else {
		const uint32_t e = P.entry[gtile];
		P.state[gtile * DS_THREADS + tid] = (uint8_t)(tid ? ds_apply(s_f[tid - 1], e) : e);
	}
}

/* the tile functions composed in order, one block, 4096 tiles per round with the state carried between rounds.  A tile
 * that starts a file is entered in the seed state; as a term of the composition it is then the constant f(seed) */
__global__ void __launch_bounds__(1024) k_dstate_scan(const DsParams P)
{
	__shared__ uint32_t s_w[32];
	__shared__ uint32_t s_carry;
	const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	if (tid == 0) s_carry = (uint32_t)P.seed;
	__syncthreads();
	for (uint64_t base = 0; base < P.n_tiles; base += 4096) {
		uint32_t f[4], agg = DS_IDENTITY; bool first[4];
#pragma unroll
		for (int j = 0; j < 4; j++) {
			const uint64_t i = base + (uint64_t)tid * 4 + j;
			f[j] = i < P.n_tiles ? P.func[i] : DS_IDENTITY;
			first[j] = i < P.n_tiles && (P.set_tiles ? P.set_tiles[i].tile == 0 : i == 0);
			agg = ds_compose(agg, first[j] ? ds_const(ds_apply(f[j], (uint32_t)P.seed)) : f[j]);
		}
		uint32_t inc = agg;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= (uint32_t)o) inc = ds_compose(t, inc); }
		const uint32_t exc_lane = __shfl_up_sync(0xffffffffu, inc, 1);
		if (lane == 31) s_w[wid] = inc;
		__syncthreads();
		if (wid == 0) {
			const uint32_t w = s_w[lane];
			uint32_t winc = w;
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= (uint32_t)o) winc = ds_compose(t, winc); }
			const uint32_t wexc = __shfl_up_sync(0xffffffffu, winc, 1);
			__syncwarp();
			s_w[lane] = lane ? wexc : DS_IDENTITY;               /* exclusive prefix of the warp aggregates */
		}
		__syncthreads();
		const uint32_t before = ds_compose(s_w[wid], lane ? exc_lane : DS_IDENTITY);
		uint32_t s = ds_apply(before, s_carry);
#pragma unroll
		for (int j = 0; j < 4; j++) {
			const uint64_t i = base + (uint64_t)tid * 4 + j;
			if (first[j]) s = (uint32_t)P.seed;
			if (i < P.n_tiles) P.entry[i] = (uint8_t)s;
			s = ds_apply(f[j], s);
		}
		__syncthreads();                                         /* every thread has read s_carry and s_w */
		if (tid == 1023) s_carry = s;
		__syncthreads();
	}
}

/* the entry states of the slices of [0, n + L) (SET: of every file's ordinals tiles) into W.dstate */
int dstate_launch(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n, int seed, cudaStream_t st,
                  const SetFile *set_files, const SetTile *set_tiles, uint64_t set_n_tiles)
{
	if (d.delim_kind != 3 || d.L < 2 || d.L > AGB_MAXDELIM) { snprintf(g_err, sizeof g_err, "internal: delimiter state pass for delim_kind %d, L = %d", d.delim_kind, d.L); return AGB_ERR_ARG; }
	const bool set = set_tiles != nullptr;
	const uint64_t tiles = set ? set_n_tiles : (n + (uint64_t)d.L + DS_TILE - 1) / DS_TILE;
	if (tiles > W.ds_tiles) {
		cudaFree(W.ds_func); cudaFree(W.ds_entry); cudaFree(W.dstate);
		W.ds_func = nullptr; W.ds_entry = nullptr; W.dstate = nullptr; W.ds_tiles = 0;
		CUDA_TRY(cudaMalloc(&W.ds_func, tiles * sizeof(uint32_t)));
		CUDA_TRY(cudaMalloc(&W.ds_entry, tiles));
		CUDA_TRY(cudaMalloc(&W.dstate, tiles * DS_THREADS));
		W.ds_tiles = tiles;
	}
	DsParams P; memset(&P, 0, sizeof P);
	P.text = (const uint8_t *)d_text; P.n = n; P.L = d.L; P.n_tiles = tiles;
	for (int i = 0; i < d.L; i++) { P.dfold[i] = d.delim_fold[i]; P.delim[i] = d.delim[i] | d.delim_fold[i]; }
	/* the virtual '\n' in front of the text: state 1 when the delimiter begins with a newline (L >= 2: it cannot close) */
	P.seed = seed >= 0 ? seed : (('\n' | P.dfold[0]) == P.delim[0] ? 1 : 0);
	P.func = W.ds_func; P.entry = W.ds_entry; P.state = W.dstate; P.set_files = set_files; P.set_tiles = set_tiles;
	if (!tiles) return AGB_OK;
	const size_t smem = DS_THREADS * DS_STRIDE;
	const bool w8 = d.L > 4;
#define DS_LAUNCH(APPLY) do { \
		if (set) { if (w8) k_dstate_tiles<APPLY, true, uint64_t><<<(unsigned)tiles, DS_THREADS, smem, st>>>(P); else k_dstate_tiles<APPLY, true, uint32_t><<<(unsigned)tiles, DS_THREADS, smem, st>>>(P); } \
		else { if (w8) k_dstate_tiles<APPLY, false, uint64_t><<<(unsigned)tiles, DS_THREADS, smem, st>>>(P); else k_dstate_tiles<APPLY, false, uint32_t><<<(unsigned)tiles, DS_THREADS, smem, st>>>(P); } \
		g_launches++; } while (0)
	DS_LAUNCH(false);
	k_dstate_scan<<<1, 1024, 0, st>>>(P); g_launches++;
	DS_LAUNCH(true);
#undef DS_LAUNCH
	CUDA_TRY(cudaGetLastError());
	return AGB_OK;
}
