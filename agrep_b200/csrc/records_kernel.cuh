/* agrep_b200/csrc/records_kernel.cuh -- stage 2, the forms that start from record boundaries: dense tile form
 * (k_records_dense), list form (k_records_list) (DESIGN.md 3.3).  Instantiated by records.cu (32- and 64-bit rows) and
 * records_wide.cu (320-bit rows) */
#ifndef AGB_RECORDS_KERNEL_CUH
#define AGB_RECORDS_KERNEL_CUH
#include "automaton.cuh"
#include "tma.cuh"

/* ================================================================================================
 * stage 2: records
 * ============================================================================================== */

/* The records candidate chunk c owns: a record [s-1, close) belongs to the FIRST flagged chunk that meets it, so
 *   (a) the record that contains byte 16c is ours iff its re-fed byte s-1 lies after prev, the flagged chunk before c
 *       (search backwards, stop at a delimiter end -> ours, or at prev -> theirs);
 *   (b) every record whose re-fed byte lies inside the chunk is ours.
 * Returns the number of reported records; writes them at out_pos.. when write is set. */
template <typename T, int NR, bool COSTS, typename RD>
__device__ __forceinline__ uint32_t chunk_records(const RecParams &P, const DevConsts<T> &C, RecShared<T, NR> &SH, RD &R,
                                                 const int64_t c, const bool write, const uint64_t out_pos, const bool hist,
                                                 agb_record *first_out, const int64_t prev)
{
	const int L = C.L;
	const int64_t n = (int64_t)P.n, lo = c * 16, hi = lo + 15;
	uint32_t cnt = 0;
	int64_t s = -2;                /* record start to run from; -2: none */
	bool found = false;
	if (c == 0) { s = 0; found = true; }
	for (int64_t cc = c - 1; !found; cc--) {
		if (cc < 0) { s = 0; found = true; break; }
		if (cc == prev) break;     /* an earlier flagged chunk meets that record: not ours */
		for (int64_t q = cc * 16 + 15; q >= cc * 16; q--)
			if (delim_ends_at(R, q, SH.delim, SH.dfold, L, C.kind)) { s = q + 1; found = true; break; }
	}
	if (!found) {
		for (int64_t q = lo; q <= hi && q < n; q++)
			if (delim_ends_at(R, q, SH.delim, SH.dfold, L, C.kind)) { s = q + 1; break; }
	}
	/* run records while their re-fed byte (s-1) is at or before the end of this chunk */
	while (s >= 0 && s - 1 <= hi && s <= n) {
		T S[NR];
		int64_t begin;
		if (s == 0) {
#pragma unroll
			for (int r = 0; r < NR; r++) S[r] = SH.start[r];
			begin = SH.start_closes ? -(int64_t)L : 0;
		} else {
#pragma unroll
			for (int r = 0; r < NR; r++) S[r] = SH.reset[r];
			begin = s - L;
		}
		int64_t p = s, close_at = -1;
		const int64_t limit = n + L;
		for (; p < limit; p++) {
			rows_step<T, NR, COSTS>(S, SH.mask[R.get(p)], C);
			if (S[0] & C.dendpos) { close_at = p; break; }
		}
		if (close_at < 0) break;                                      /* never closed: dropped, as the reference does */
		const int64_t end = close_at + 1 - L;
		const bool counts = (begin + 1 < n) && (begin + 1 <= end) && rec_owned(P, begin, L, close_at);       /* bitap.c:213 + agrep.c:3811 */
		int level = C.k;
		bool cond;
		if (P.levels) {
			level = -1;
#pragma unroll
			for (int r = 0; r < NR; r++) if (level < 0 && match_cond<T>(S[r], C)) level = r;
			cond = level >= 0;
			if (cond && counts && hist) atomicAdd(&SH.hist[level], 1ull);
			if (cond && P.want_level >= 0 && level > P.want_level) cond = false;
		} else cond = match_cond<T>(S[NR - 1], C);
		if (cond && counts) {
			if (write) {
				const uint64_t at = out_pos + cnt;
				if (at < P.capacity) {
					agb_record rec; rec.begin = begin; rec.end = end; rec.ordinal = 0; rec.level = level; rec.pad = 0;
					P.records[at] = rec;
				}
			}
			if (first_out && cnt == 0) { first_out->begin = begin; first_out->end = end; first_out->ordinal = 0; first_out->level = level; first_out->pad = 0; }
			cnt++;
		}
		s = close_at + 1;
	}
	return cnt;
}

/* delim_kind 3: the closes in a slice of DENSE_PER staged bytes (len of them in the text), walked from the delimiter's state
 * at its start (bit j: at byte j).  Not inlined: the other delimiters' dense kernels keep their registers */
static_assert(DENSE_PER == 128, "two words of close bits per slice");
static __device__ __noinline__ ulonglong2 dstate_slice_closes(const uint8_t *sl, int64_t len, int ds, const uint8_t *delim, const uint8_t *dfold, int L)
{
	ulonglong2 w = make_ulonglong2(0, 0);
	for (uint32_t v = 0; v < DENSE_PER / 16 && (int64_t)(16 * v) < len; v++) {
		const uint4 x = *reinterpret_cast<const uint4 *>(sl + v * 16);
		const uint32_t xs[4] = { x.x, x.y, x.z, x.w };
#pragma unroll
		for (uint32_t b = 0; b < 16; b++) {
			const uint32_t j = 16 * v + b;
			if ((int64_t)j < len && dstate_step(ds, (int)((xs[b >> 2] >> (8 * (b & 3))) & 0xFFu), delim, dfold, L)) {
				if (j < 64) w.x |= 1ull << j; else w.y |= 1ull << (j - 64);
			}
		}
	}
	return w;
}

/* dense tile form: the automaton over EVERYTHING (no anchor plan: classes, -v, -p, '#', short patterns ...).
 * One CTA per 32 KiB tile, brought into shared memory (+2 KiB that follow it) by one bulk-async copy.  Thread t
 * owns the records whose opening delimiter ends inside its 128-byte slice: it starts at the first of them in the
 * constant post-delimiter state and simply keeps walking -- a record that closes at a delimiter inside the slice
 * hands over to the next one at the following byte -- until the last of its records has closed (on average half a
 * record past the slice; the neighbour skips that head).  So every lane walks about the same number of bytes in
 * lockstep, bytes and the Mask[] table come from shared memory (global memory only for a record that outruns the
 * staged bytes), and nothing is carried between threads or tiles.  Same loop as asearch.c:94-199. */

template <typename T, int NR, bool COSTS, bool SET = false>
__global__ void __launch_bounds__(DENSE_THREADS)
k_records_dense(const RecParams P0)
{
	/* SET: this block's tile of a file of the set, the file's text as the whole text */
	RecParams Ps; uint64_t tile = blockIdx.x; uint32_t file = 0;
	if constexpr (SET) { Ps = P0; set_enter(P0.set_files, P0.set_tiles, Ps.text, Ps.n, tile, file); Ps.n_chunks = (Ps.n + 15) / 16; }
	const RecParams &P = SET ? Ps : P0;
	extern __shared__ __align__(128) uint8_t s_text[];                 /* DENSE_TILE + DENSE_TAIL */
	__shared__ RecShared<T, NR> SH;
	__shared__ uint64_t s_bar;
	__shared__ uint32_t s_scan[DENSE_THREADS];
	const uint32_t tid = threadIdx.x;
	const int64_t n = (int64_t)P.n, tile0 = (int64_t)tile * DENSE_TILE;
	const uint64_t readable = P.n_chunks * 16;
	const uint64_t avail = (readable - (uint64_t)tile0) & ~15ull;
	const uint32_t loaded = (uint32_t)(avail < (uint64_t)(DENSE_TILE + DENSE_TAIL) ? avail : (uint64_t)(DENSE_TILE + DENSE_TAIL));
	if (tid == 0) {
		mbar_init(&s_bar, 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		mbar_expect_tx(&s_bar, loaded);
		bulk_g2s(s_text, P.text + tile0, loaded, &s_bar);
	}
	DevConsts<T> C;
	shared_init<T, NR>(SH, C, P.desc, DENSE_THREADS, P.rx_tab);                 /* ends with __syncthreads(): the barrier init is visible */
	mbar_wait(&s_bar, 0);
	const int L = C.L;
	/* bytes [tile0, tile0 + in_smem) come from shared memory: staged AND inside the text */
	const uint32_t in_smem = (uint32_t)((int64_t)loaded < n - tile0 ? (int64_t)loaded : n - tile0);
	const uint32_t tile_len = (uint32_t)((int64_t)DENSE_TILE < n - tile0 ? (int64_t)DENSE_TILE : n - tile0);
	Reader R; R.init(P.text, P.n, SH.delim, L);

	/* ---- which delimiters end in my slice (bit j: at byte 128 t + j)?  The record that follows each is mine. ---- */
	uint64_t bits[DENSE_PER / 64];
#pragma unroll
	for (int w = 0; w < DENSE_PER / 64; w++) bits[w] = 0;
	if (L == 1) {
		/* 16 bytes at a time: exact per-byte equality by SWAR, 4 flags gathered by one multiply */
		const uint32_t d4 = SH.delim[0] * 0x01010101u, f4 = SH.dfold[0] * 0x01010101u;
#pragma unroll
		for (int v = 0; v < DENSE_PER / 16; v++) {
			const uint4 x = *reinterpret_cast<const uint4 *>(s_text + tid * DENSE_PER + v * 16);
			const uint32_t xs[4] = { x.x, x.y, x.z, x.w };
			uint32_t m16 = 0;
#pragma unroll
			for (int w = 0; w < 4; w++) {
				const uint32_t t = (xs[w] | f4) ^ d4;
				const uint32_t z = ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t | 0x7F7F7F7Fu);    /* 0x80 where the byte equals the delimiter */
				m16 |= ((((z >> 7) * 0x00204081u) >> 21) & 0xFu) << (4 * w);
			}
			bits[v >> 2] |= (uint64_t)m16 << (16 * (v & 3));
		}
	} else if (C.kind == 3) {
		/* -p: one walk over the slice from the state the delimiter pass found at its start */
		const uint64_t slice = SET ? ((uint64_t)P0.set_files[file].ord_tile0 + tile) * DENSE_THREADS + tid : (uint64_t)tile0 / DENSE_PER + tid;
		const ulonglong2 w = dstate_slice_closes(s_text + tid * DENSE_PER, n - (tile0 + (int64_t)tid * DENSE_PER), P.dstate[slice], SH.delim, SH.dfold, L);
		bits[0] = w.x; bits[1] = w.y;
	} else {
		for (uint32_t j = 0; j < DENSE_PER; j++) {
			const int64_t q = tile0 + (int64_t)tid * DENSE_PER + j;
			if (q < n && delim_ends_at(R, q, SH.delim, SH.dfold, L, C.kind)) bits[j >> 6] |= 1ull << (j & 63);
		}
	}
	{   /* only delimiters inside the text (q < n) */
		const int64_t last_q = (int64_t)tile_len - 1 - (int64_t)tid * DENSE_PER;
#pragma unroll
		for (int w = 0; w < DENSE_PER / 64; w++) {
			const int64_t hi = last_q - 64 * w;
			if (hi < 0) bits[w] = 0; else if (hi < 63) bits[w] &= (2ull << hi) - 1;
		}
	}
	/* the very first record of the text has no delimiter in front of it: thread 0 of tile 0.  (delim_kind 3 in a window after
	 * the first: the start rows do not hold the delimiter's state there, and that record belongs to the window before) */
	const bool first = (tile0 == 0 && tid == 0) && (C.kind != 3 || P.own_lo == INT64_MIN);
	uint32_t owned = first ? 1u : 0u;
#pragma unroll
	for (int w = 0; w < DENSE_PER / 64; w++) owned += __popcll(bits[w]);

	const int64_t limit = n + L;
	/* rows after a delimiter, kept in registers: a close is a handful of moves, not shared-memory traffic */
	T RS[NR];
#pragma unroll
	for (int r = 0; r < NR; r++) RS[r] = SH.reset[r];
	/* away from the end of the text every record counts unless it is empty (bitap.c:213, agrep.c:3811) */
	const bool easy = tile0 + (int64_t)DENSE_TILE + DENSE_TAIL + L + 2 < n;
	const bool sharded = P.own_lo > INT64_MIN / 2 || P.own_hi < INT64_MAX / 2;
	uint32_t my_count = 0;
	uint64_t out_pos = 0;
	for (int pass = 0; pass < (P.emit ? 2 : 1); pass++) {
		uint32_t cnt = 0, left = owned;
		if (left) {
			uint32_t rel;                                               /* position relative to tile0 while inside the staged bytes */
			if (first) rel = 0;
			else rel = tid * DENSE_PER + 1 + (bits[0] ? __ffsll((long long)bits[0]) - 1 : 64 + __ffsll((long long)bits[1]) - 1);
			T S[NR];
			int64_t begin;
			if (tile0 == 0 && rel == 0) {
#pragma unroll
				for (int r = 0; r < NR; r++) S[r] = SH.start[r];
				begin = SH.start_closes ? -(int64_t)L : 0;
			} else {
#pragma unroll
				for (int r = 0; r < NR; r++) S[r] = RS[r];
				begin = tile0 + rel - L;
			}
			uint32_t begin_rel = (uint32_t)(begin - tile0);              /* begin - tile0 (mod 2^32; -1 for the virtual newline) */
			/* ---- fast part: text bytes from shared memory, 32-bit bookkeeping.  The plain counting pass (no -B levels,
			 * no list) gets its own loop so that a close is a dozen instructions ---- */
			if (!P.levels && !P.emit) {
				for (; rel < in_smem; rel++) {
					rows_step<T, NR, COSTS>(S, SH.mask[s_text[rel]], C);
					if (S[0] & C.dendpos) {
						const uint32_t end_rel = rel + 1 - L;
						bool counts = (int32_t)(end_rel - begin_rel) >= 1;
						if (!easy) counts = counts && (tile0 + (int64_t)(int32_t)begin_rel + 1 < n);
						if (sharded) counts = counts && rec_owned(P, tile0 + (int64_t)(int32_t)begin_rel, L, tile0 + rel);
						cnt += (match_cond<T>(S[NR - 1], C) && counts) ? 1u : 0u;
						if (--left == 0) break;
#pragma unroll
						for (int r = 0; r < NR; r++) S[r] = RS[r];
						begin_rel = end_rel;
					}
				}
			} else
			for (; rel < in_smem; rel++) {
				rows_step<T, NR, COSTS>(S, SH.mask[s_text[rel]], C);
				if (S[0] & C.dendpos) {
					const uint32_t end_rel = rel + 1 - L;
					bool counts = (int32_t)(end_rel - begin_rel) >= 1;  /* begin + 1 <= end (agrep.c:3811) */
					if (!easy) counts = counts && (tile0 + (int64_t)(int32_t)begin_rel + 1 < n);
					if (sharded) counts = counts && rec_owned(P, tile0 + (int64_t)(int32_t)begin_rel, L, tile0 + rel);
					int level = C.k;
					bool cond;
					if (P.levels) {
						level = -1;
#pragma unroll
						for (int r = 0; r < NR; r++) if (level < 0 && match_cond<T>(S[r], C)) level = r;
						cond = level >= 0;
						if (cond && counts && pass == 0 && !P.emit) atomicAdd(&SH.hist[level], 1ull);
						if (cond && P.want_level >= 0 && level > P.want_level) cond = false;
					} else cond = match_cond<T>(S[NR - 1], C);
					if (cond && counts) {
						if (pass == 1) {
							const uint64_t at = out_pos + cnt;
							if (at < P.capacity) {
								agb_record rec; rec.begin = tile0 + (int64_t)(int32_t)begin_rel; rec.end = tile0 + end_rel;
								rec.ordinal = 0; rec.level = level; rec.pad = (int32_t)file;
								P.records[at] = rec;
							}
						}
						cnt++;
					}
					if (--left == 0) break;                               /* the record that starts at the next byte is somebody else's */
#pragma unroll
					for (int r = 0; r < NR; r++) S[r] = RS[r];
					begin_rel = end_rel;
				}
			}
			/* ---- slow part: the record outruns the staged bytes or the text ends (appended delimiter) ---- */
			if (left) {
				begin = tile0 + (int64_t)(int32_t)begin_rel;
				for (int64_t p = tile0 + rel; p < limit; p++) {
					rows_step<T, NR, COSTS>(S, SH.mask[R.get(p)], C);
					if (S[0] & C.dendpos) {
						const int64_t end = p + 1 - L;
						const bool counts = (begin + 1 < n) && (begin + 1 <= end) && rec_owned(P, begin, L, p);
						int level = C.k;
						bool cond;
						if (P.levels) {
							level = -1;
#pragma unroll
							for (int r = 0; r < NR; r++) if (level < 0 && match_cond<T>(S[r], C)) level = r;
							cond = level >= 0;
							if (cond && counts && pass == 0 && !P.emit) atomicAdd(&SH.hist[level], 1ull);
							if (cond && P.want_level >= 0 && level > P.want_level) cond = false;
						} else cond = match_cond<T>(S[NR - 1], C);
						if (cond && counts) {
							if (pass == 1) {
								const uint64_t at = out_pos + cnt;
								if (at < P.capacity) {
									agb_record rec; rec.begin = begin; rec.end = end; rec.ordinal = 0; rec.level = level; rec.pad = (int32_t)file;
									P.records[at] = rec;
								}
							}
							cnt++;
						}
						if (--left == 0) break;
#pragma unroll
						for (int r = 0; r < NR; r++) S[r] = RS[r];
						begin = end;
					}
				}
			}
		}
		if (pass == 0) {
			my_count = cnt;
			s_scan[tid] = cnt;
			__syncthreads();
			for (int off = 1; off < DENSE_THREADS; off <<= 1) {
				uint32_t v = (tid >= (unsigned)off) ? s_scan[tid - off] : 0;
				__syncthreads();
				s_scan[tid] += v;
				__syncthreads();
			}
			if (!P.emit) {
				if (tid == DENSE_THREADS - 1) {
					P.tile_counts[blockIdx.x] = s_scan[DENSE_THREADS - 1];
					if (s_scan[DENSE_THREADS - 1]) atomicAdd(&P.totals[0], (unsigned long long)s_scan[DENSE_THREADS - 1]);
					if (SET && s_scan[DENSE_THREADS - 1]) atomicAdd(&P.set_stats[SET_STATS * file], (unsigned long long)s_scan[DENSE_THREADS - 1]);
					atomicAdd(&P.totals[1], (unsigned long long)((tile_len + 15) / 16));
				}
				__syncthreads();
				if (P.levels && tid <= AGB_MAXERR && SH.hist[tid]) atomicAdd(&P.totals[2 + tid], SH.hist[tid]);
				if (SET && P.levels && tid <= AGB_MAXERR && SH.hist[tid]) atomicAdd(&P.set_stats[SET_STATS * file + 1 + tid], SH.hist[tid]);
			} else out_pos = P.tile_offsets[blockIdx.x] + (s_scan[tid] - my_count);
		}
	}
}

/* list form: one thread per surviving chunk of the ordered candidate list (all lanes busy however sparse the
 * survivors are).  Count launch: per-candidate counts; emit launch: writes at the scanned offsets.  The list length
 * is read from the device (totals[12]); the grid strides over it.
 * A candidate's record lies around its chunk: the thread loads LIST_GB groups before it and LIST_GA after it in one go
 * (independent 16-byte loads: one memory round trip instead of one per group met) into its strip of shared memory and
 * reads from there; a record that leaves the strip continues on the slow path.  The record belongs to the first flagged
 * chunk that meets it: with the list in hand that is "the backward search for the record start stops at the candidate
 * before this one". */
#define LIST_GB 5
#define LIST_GA 7
#define LIST_NG (LIST_GB + 1 + LIST_GA)
#define LIST_STRIDE (LIST_NG * 4 + 1)                   /* words; odd: the lanes of a warp hit different banks */
#define LIST_SMEM (REC_THREADS * LIST_STRIDE * 4)
/* 320-bit rows: 2 blocks per SM, so that the rows of k = 1..8 stay in registers (at 6 they go to local memory) */
template <typename T> constexpr int list_min_blocks() { return std::is_same<T, Wide>::value ? 2 : 6; }
template <typename T, int NR, bool COSTS>
__global__ void __launch_bounds__(REC_THREADS, list_min_blocks<T>())
k_records_list(const RecParams P)
{
	extern __shared__ __align__(16) uint32_t s_win[];
	__shared__ RecShared<T, NR> SH;
	DevConsts<T> C;
	shared_init<T, NR>(SH, C, P.desc, REC_THREADS, P.rx_tab);
	unsigned long long ncand = P.totals[12];
	if (ncand > P.cand_cap) ncand = P.cand_cap;
	uint32_t *strip = s_win + threadIdx.x * LIST_STRIDE;
	const int64_t n_groups = (int64_t)P.n_chunks;          /* 16-byte groups that may be read */
	uint32_t cnt = 0;
	for (uint64_t i = (uint64_t)blockIdx.x * REC_THREADS + threadIdx.x; i < ncand; i += (uint64_t)gridDim.x * REC_THREADS) {
		if (P.emit) {
			/* emit launch: 0 records -> nothing; exactly 1 -> the count launch kept it; more (rare) -> walk again */
			const uint32_t c0 = P.tile_counts[i];
			if (c0 == 1) { const uint64_t at = P.tile_offsets[i]; if (at < P.capacity) P.records[at] = P.cand_first[i]; }
			if (c0 <= 1) continue;
		}
		const int64_t c = (int64_t)P.cand[i], prev = i ? (int64_t)P.cand[i - 1] : -1;
		WindowReader R; R.init(P.text, P.n, SH.delim, C.L);
		{
			int64_t g0 = c - LIST_GB, g1 = c + 1 + LIST_GA;
			if (g0 < 0) g0 = 0;
			if (g1 > n_groups) g1 = n_groups;
			/* two batches of independent loads (13 groups in one go would hold 52 registers across the whole kernel) */
#pragma unroll
			for (int half = 0; half < 2; half++) {
				constexpr int H = (LIST_NG + 1) / 2;
				uint4 v[H];
#pragma unroll
				for (int gi = 0; gi < H; gi++) { const int g = half * H + gi; if (g < LIST_NG && g0 + g < g1) v[gi] = __ldg(reinterpret_cast<const uint4 *>(P.text) + g0 + g); }
#pragma unroll
				for (int gi = 0; gi < H; gi++) { const int g = half * H + gi; if (g < LIST_NG && g0 + g < g1) { strip[g * 4] = v[gi].x; strip[g * 4 + 1] = v[gi].y; strip[g * 4 + 2] = v[gi].z; strip[g * 4 + 3] = v[gi].w; } }
			}
			int64_t hi = g1 * 16;
			if (hi > (int64_t)P.n) hi = (int64_t)P.n;          /* only bytes of the text (the slow path knows the virtual and appended ones) */
			R.sm = reinterpret_cast<const uint8_t *>(strip); R.lo = g0 * 16; R.len = (uint32_t)(hi - g0 * 16);
		}
		if (P.emit) chunk_records<T, NR, COSTS>(P, C, SH, R, c, true, P.tile_offsets[i], false, nullptr, prev);
		else {
			const uint32_t c1 = chunk_records<T, NR, COSTS>(P, C, SH, R, c, false, 0, true, P.cand_first ? &P.cand_first[i] : nullptr, prev);
			P.tile_counts[i] = c1;
			cnt += c1;
		}
	}
	if (!P.emit) {
		uint32_t sum = __reduce_add_sync(0xffffffffu, cnt);
		if ((threadIdx.x & 31) == 0 && sum) atomicAdd(&P.totals[0], (unsigned long long)sum);
		__syncthreads();
		if (P.levels && threadIdx.x <= AGB_MAXERR && SH.hist[threadIdx.x]) atomicAdd(&P.totals[2 + threadIdx.x], SH.hist[threadIdx.x]);
	}
}

template <typename T, int NR, bool COSTS, bool SET>
static void launch_dense_one(const RecParams &P, unsigned grid, cudaStream_t st)
{
	static bool configured[64] = {false};
	int dev = 0; cudaGetDevice(&dev);
	if (!configured[dev & 63]) {
		cudaFuncSetAttribute(k_records_dense<T, NR, COSTS, SET>, cudaFuncAttributeMaxDynamicSharedMemorySize, DENSE_SMEM);
		configured[dev & 63] = true;
	}
	k_records_dense<T, NR, COSTS, SET><<<grid, DENSE_THREADS, DENSE_SMEM, st>>>(P);
}

/* the launchers at a row count known at run time (1..9; -1 for any other) */
template <typename T, bool COSTS, bool SET>
static int launch_dense_t(int nrows, const RecParams &P, unsigned grid, cudaStream_t st)
{
	return launch_rows<9>(nrows, [&](auto R) { launch_dense_one<T, decltype(R)::value, COSTS, SET>(P, grid, st); });
}

template <typename T, bool COSTS>
static int launch_records_list_t(int nrows, const RecParams &P, unsigned grid, cudaStream_t st)
{
	return launch_rows<9>(nrows, [&](auto R) { k_records_list<T, decltype(R)::value, COSTS><<<grid, REC_THREADS, LIST_SMEM, st>>>(P); });
}

#endif
