/* agrep_b200/csrc/regex.cu -- stage 2 for regular expressions (AGB_ENGINE_REGEX): the recurrence of re()
 * (agrep.c:1267-1917) over every byte, in the dense tile form (DESIGN.md 3.6).
 *
 *   A0 = (Next(B0) & Mask[c]) | (Init1 & B0)
 *   Aj = (Next(Bj) & Mask[c]) | (Init1 & Bj) | ((B(j-1) | Next(B(j-1) | A(j-1))) & NO_ERR_MASK)
 *
 * At a newline the line matches when T = (Next(Bk) & Mask['\n']) | (Init1 & Bk), widened by T |= Next(T) under TAIL,
 * holds bit 0 (the trailing position), XOR -v; then every row restarts from the constant post-newline rows (reset[]).
 * Next(S) -- the union of the follow sets of the positions in S, compute_next()'s table taken to 8-bit slices -- is
 * sizeof(T) shared-memory loads: Next(S) = T0[S & 0xff] | T1[(S >> 8) & 0xff] | ...  (4 KiB of tables for <= 31
 * positions, 16 KiB for 63), with no data-dependent loop.
 *
 * '*' gives the state an unbounded memory within a line, so the slices form's warm-up does not apply; the tile form
 * does: one CTA per 32 KiB tile staged in shared memory (+2 KiB behind it), thread t owns the lines that open in its
 * 128-byte slice (the newline in front of them lies there) and walks them to their closing newline -- from shared
 * memory while the bytes are staged, from global memory after that, so a line of any length is finished by the
 * thread that owns it (serially: one thread per over-long line).  Count pass -> per-tile counts -> scan -> emit pass, as
 * k_records_dense; the emit launch recounts its tile before it writes, so a list walks every byte three times.
 *
 * LEVELS (AGB_WANT_LEVELS): a line's level is the smallest row that passes the match test at its newline (records.cu's
 * rule, -v included).  Row j depends on rows <= j only, so one pass at k yields every line's smallest level <= k.  The
 * rows are nested (the reset rows are, and each step keeps it), so the test is monotone in the row: the last row (row 0
 * under -v) is tested first and the other rows only behind a pass.  The extra work is per matching line; the count
 * launch keeps a per-CTA histogram in shared memory and adds it to totals[2 + level] once. */
#include "automaton.cuh"

#define RX_THREADS 256
#define RX_TAIL    2048
#define RX_PER     (RX_TILE / RX_THREADS)          /* 128 bytes per thread */
static_assert(RX_TILE == DENSE_TILE, "the tile counts of the workspace are sized for DENSE_TILE");

template <typename T>
__device__ __forceinline__ T rx_next(const T *tab, T s)
{
	T r = tab[s & 0xFFu];
#pragma unroll
	for (int i = 1; i < (int)sizeof(T); i++) r |= tab[i * 256 + (uint32_t)((s >> (8 * i)) & 0xFFu)];
	return r;
}

/* one byte other than '\n' through all rows (agrep.c:1586-1607) */
template <typename T, int NR>
__device__ __forceinline__ void rx_step(T (&S)[NR], T cm, const T *tab, T init1, T noerr)
{
	T prevB = S[0];
	T prevA = (rx_next<T>(tab, prevB) & cm) | (init1 & prevB);
#pragma unroll
	for (int r = 1; r < NR; r++) {
		const T b = S[r];
		const T a = (rx_next<T>(tab, b) & cm) | (init1 & b) | ((prevB | rx_next<T>(tab, prevA | prevB)) & noerr);
		S[r - 1] = prevA; prevA = a; prevB = b;
	}
	S[NR - 1] = prevA;
}

/* the newline test of agrep.c:1614-1658 on one row */
template <typename T>
__device__ __forceinline__ bool rx_line_matches(T s, const T *tab, T mask_nl, T init1, bool tail, bool inverse)
{
	T t = (rx_next<T>(tab, s) & mask_nl) | (init1 & s);
	if (tail) t |= rx_next<T>(tab, t);
	return ((t & (T)1) != 0) != inverse;
}

template <typename T, int NR, bool LEVELS, bool SET = false>
__global__ void __launch_bounds__(RX_THREADS)
k_regex(const RecParams P0)
{
	/* SET: this block's tile of a file of the set, the file's text as the whole text */
	RecParams Ps; uint64_t tile = 0; uint32_t file = 0;
	if constexpr (SET) { Ps = P0; set_enter(P0.set_files, P0.set_tiles, Ps.text, Ps.n, tile, file); Ps.n_chunks = (Ps.n + 15) / 16; }
	const RecParams &P = SET ? Ps : P0;
	extern __shared__ __align__(16) uint8_t s_raw[];
	T *s_tab = reinterpret_cast<T *>(s_raw);                               /* sizeof(T) slices of 256 */
	T *s_mask = s_tab + sizeof(T) * 256;                                   /* 256 */
	uint8_t *s_text = reinterpret_cast<uint8_t *>(s_mask + 256);           /* RX_TILE + RX_TAIL */
	__shared__ uint32_t s_scan[RX_THREADS];
	__shared__ uint32_t s_hist[NR];                                        /* LEVELS: owned matching lines by level */
	const uint32_t tid = threadIdx.x;
	const agb_desc *D = P.desc;
	const T *g_tab = reinterpret_cast<const T *>(P.rx_tab);
	for (uint32_t i = tid; i < sizeof(T) * 256; i += RX_THREADS) s_tab[i] = g_tab[i];
	for (uint32_t i = tid; i < 256; i += RX_THREADS) s_mask[i] = (T)D->mask[i];
	const int64_t n = (int64_t)P.n, tile0 = (int64_t)(SET ? (unsigned)tile : blockIdx.x) * RX_TILE;
	const uint64_t readable = P.n_chunks * 16;
	const uint64_t avail = (readable - (uint64_t)tile0) & ~15ull;
	const uint32_t loaded = (uint32_t)(avail < (uint64_t)(RX_TILE + RX_TAIL) ? avail : (uint64_t)(RX_TILE + RX_TAIL));
	for (uint32_t g = tid; g < loaded / 16; g += RX_THREADS)
		reinterpret_cast<uint4 *>(s_text)[g] = __ldg(reinterpret_cast<const uint4 *>(P.text + tile0) + g);
	const T init1 = (T)D->init1, noerr = (T)D->noerr;
	const bool inverse = D->inverse != 0, tail = P.rx_tail != 0;
	T RS[NR];
#pragma unroll
	for (int r = 0; r < NR; r++) RS[r] = (T)D->reset[r];
	if (LEVELS && tid < NR) s_hist[tid] = 0;
	__syncthreads();
	const T mask_nl = s_mask['\n'];
	const uint32_t in_smem = (uint32_t)((int64_t)loaded < n - tile0 ? (int64_t)loaded : n - tile0);
	const uint32_t tile_len = (uint32_t)((int64_t)RX_TILE < n - tile0 ? (int64_t)RX_TILE : n - tile0);

	/* the newlines in my slice (bit j: at byte RX_PER t + j), each opening a line that is mine */
	uint64_t bits[RX_PER / 64];
#pragma unroll
	for (int w = 0; w < RX_PER / 64; w++) bits[w] = 0;
#pragma unroll
	for (int v = 0; v < RX_PER / 16; v++) {
		const uint4 x = *reinterpret_cast<const uint4 *>(s_text + tid * RX_PER + v * 16);
		const uint32_t xs[4] = { x.x, x.y, x.z, x.w };
		uint32_t m16 = 0;
#pragma unroll
		for (int w = 0; w < 4; w++) {
			const uint32_t t = xs[w] ^ 0x0A0A0A0Au;
			const uint32_t z = ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t | 0x7F7F7F7Fu);    /* 0x80 where the byte is '\n' */
			m16 |= ((((z >> 7) * 0x00204081u) >> 21) & 0xFu) << (4 * w);
		}
		bits[v >> 2] |= (uint64_t)m16 << (16 * (v & 3));
	}
	{   /* only newlines inside the text */
		const int64_t last_q = (int64_t)tile_len - 1 - (int64_t)tid * RX_PER;
#pragma unroll
		for (int w = 0; w < RX_PER / 64; w++) {
			const int64_t hi = last_q - 64 * w;
			if (hi < 0) bits[w] = 0; else if (hi < 63) bits[w] &= (2ull << hi) - 1;
		}
	}
	/* the first line of the text opens at the virtual '\n' in front of it: thread 0 of tile 0 */
	const bool first = (tile0 == 0 && tid == 0);
	uint32_t owned = first ? 1u : 0u;
#pragma unroll
	for (int w = 0; w < RX_PER / 64; w++) owned += __popcll(bits[w]);

	uint32_t my_count = 0;
	uint64_t out_pos = 0;
	for (int pass = 0; pass < (P.emit ? 2 : 1); pass++) {
		uint32_t cnt = 0, left = owned;
		if (left) {
			int64_t p;                                              /* file offset of the next byte */
			if (first) p = 0;
			else p = tile0 + tid * RX_PER + 1 + (bits[0] ? __ffsll((long long)bits[0]) - 1 : 64 + __ffsll((long long)bits[1]) - 1);
			int64_t begin = p - 1;                                  /* the newline that opened the line (-1: the virtual one) */
			T S[NR];
#pragma unroll
			for (int r = 0; r < NR; r++) S[r] = RS[r];
			for (;; p++) {
				const int64_t rel = p - tile0;
				int c;
				if (rel < (int64_t)in_smem) c = s_text[rel];
				else c = p < n ? (int)__ldg(P.text + p) : '\n';     /* the newline appended at EOF closes the last line */
				if (c != '\n') { rx_step<T, NR>(S, s_mask[c], s_tab, init1, noerr); continue; }
				/* the empty line behind a final newline is no line (agrep.c:3811, as the other engines); ownership is
				 * decided whatever the line's match, so that an owned line cut off by the end of a shard's halo is always
				 * reported (rec_owned raises totals[11]) */
				const bool counts = begin + 1 < n && rec_owned(P, begin, 1, p);
				/* agrep.c:1614-1658: the match test on the last row (LEVELS: the smallest row that passes), then the next line */
				int level = -1;
				bool cond;
				if constexpr (LEVELS) {
					/* S[r] is a subset of S[r + 1] and the test is monotone in S, so without -v a line that fails the last
					 * row fails them all, and with -v a row passes only if row 0 does: one test for most lines, as without
					 * levels (a lane at its newline holds up its warp), the search only behind a pass */
					if (rx_line_matches<T>(inverse ? S[0] : S[NR - 1], s_tab, mask_nl, init1, tail, inverse)) {
						level = inverse ? 0 : NR - 1;
						if (!inverse) {
#pragma unroll
							for (int r = 0; r < NR - 1; r++)
								if (level == NR - 1 && rx_line_matches<T>(S[r], s_tab, mask_nl, init1, tail, false)) level = r;
						}
					}
					cond = level >= 0;
					if (cond && counts && !P.emit) atomicAdd(&s_hist[level], 1u);
				} else cond = rx_line_matches<T>(S[NR - 1], s_tab, mask_nl, init1, tail, inverse);
				if (cond && counts) {
					if (pass == 1) {
						const uint64_t at = out_pos + cnt;
						if (at < P.capacity) {
							agb_record rec; rec.begin = begin; rec.end = p; rec.ordinal = 0; rec.level = LEVELS ? level : D->k; rec.pad = (int32_t)file;
							P.records[at] = rec;
						}
					}
					cnt++;
				}
				if (--left == 0 || p >= n) break;
#pragma unroll
				for (int r = 0; r < NR; r++) S[r] = RS[r];
				begin = p;
			}
		}
		if (pass == 0) {
			my_count = cnt;
			s_scan[tid] = cnt;
			__syncthreads();
			for (int off = 1; off < RX_THREADS; off <<= 1) {
				const uint32_t v = (tid >= (unsigned)off) ? s_scan[tid - off] : 0;
				__syncthreads();
				s_scan[tid] += v;
				__syncthreads();
			}
			if (!P.emit) {
				if (tid == RX_THREADS - 1) {
					P.tile_counts[blockIdx.x] = s_scan[RX_THREADS - 1];
					if (s_scan[RX_THREADS - 1]) atomicAdd(&P.totals[0], (unsigned long long)s_scan[RX_THREADS - 1]);
					if (SET && s_scan[RX_THREADS - 1]) atomicAdd(&P.set_stats[SET_STATS * file], (unsigned long long)s_scan[RX_THREADS - 1]);
					atomicAdd(&P.totals[1], (unsigned long long)((tile_len + 15) / 16));
				}
				if (LEVELS && tid < NR && s_hist[tid]) atomicAdd(&P.totals[2 + tid], (unsigned long long)s_hist[tid]);
				if (SET && LEVELS && tid < NR && s_hist[tid]) atomicAdd(&P.set_stats[SET_STATS * file + 1 + tid], (unsigned long long)s_hist[tid]);
			} else out_pos = P.tile_offsets[blockIdx.x] + (s_scan[tid] - my_count);
		}
	}
}

template <typename T> static constexpr size_t rx_smem() { return sizeof(T) * 256 * sizeof(T) + 256 * sizeof(T) + RX_TILE + RX_TAIL; }

template <typename T, int NR, bool LEVELS, bool SET>
static void launch_regex_one(const RecParams &P, unsigned grid, cudaStream_t st)
{
	static bool configured[64] = {false};
	int dev = 0; cudaGetDevice(&dev);
	if (!configured[dev & 63]) {
		cudaFuncSetAttribute(k_regex<T, NR, LEVELS, SET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rx_smem<T>());
		configured[dev & 63] = true;
	}
	k_regex<T, NR, LEVELS, SET><<<grid, RX_THREADS, rx_smem<T>(), st>>>(P);
}

template <typename T, bool LEVELS, bool SET>
static int launch_regex_t(int nrows, const RecParams &P, unsigned grid, cudaStream_t st)
{
	return launch_rows<5>(nrows, [&](auto R) { launch_regex_one<T, decltype(R)::value, LEVELS, SET>(P, grid, st); });
}

/* 32-bit words hold positions 0..31 (M <= 31), 64-bit words the rest */
bool regex_narrow(const agb_desc &d) { return d.M <= 31; }

template <bool SET>
static int launch_regex_any(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st)
{
	if (!P.rx_tab) return -1;
	if (P.levels)
		return regex_narrow(d) ? launch_regex_t<uint32_t, true, SET>(d.nrows, P, grid, st) : launch_regex_t<uint64_t, true, SET>(d.nrows, P, grid, st);
	return regex_narrow(d) ? launch_regex_t<uint32_t, false, SET>(d.nrows, P, grid, st) : launch_regex_t<uint64_t, false, SET>(d.nrows, P, grid, st);
}
int launch_regex(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st) { return launch_regex_any<false>(d, P, grid, st); }
int launch_regex_set(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st) { return launch_regex_any<true>(d, P, grid, st); }

/* the byte-sliced Next tables of a regular expression, in the word width the kernel uses: slice s, byte value v ->
 * the union of follow[p] over the positions p whose bit (M - p) is bit i of v at 8 s + i */
size_t regex_tables(const agb_desc &d, const agb_regex &rx, uint64_t *out)
{
	const int M = d.M, W = regex_narrow(d) ? 4 : 8;
	uint64_t fb[64];
	for (int bit = 0; bit < 64; bit++) fb[bit] = bit <= M ? rx.follow[M - bit] : 0;
	uint32_t *o32 = reinterpret_cast<uint32_t *>(out);
	for (int s = 0; s < W; s++)
		for (int v = 0; v < 256; v++) {
			uint64_t r = 0;
			for (int i = 0; i < 8; i++) if (v >> i & 1) r |= fb[8 * s + i];
			if (W == 4) o32[s * 256 + v] = (uint32_t)r; else out[s * 256 + v] = r;
		}
	return (size_t)W * 256 * (size_t)W;
}
