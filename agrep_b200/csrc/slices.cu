/* agrep_b200/csrc/slices.cu -- stage 2, slices form: the automaton over every byte in lockstep (DESIGN.md 3.3) */
#include "automaton.cuh"

/* slices form: the automaton over EVERYTHING in lockstep.  The dense tile form above gives every thread whole
 * records, so a warp waits for its longest lane (16 of 32 lanes busy on text lines).  Here every thread walks a
 * fixed slice of SL_PER bytes, whatever the records do:
 *   - the state of the automaton at a slice start depends only on the last M + rows bytes (a state bit moves on or
 *     costs an error every byte) unless the pattern has positions that hold for ever ('#', -p): the thread starts
 *     `warm` bytes early from the post-delimiter rows, throws the results of that stretch away and clears the
 *     sticky end bits -- from there on its rows are exactly the reference's;
 *   - what a record has matched so far lives in the sticky end bits (Init1 keeps them, maskgen.c:232), so for a
 *     record that spans slices the verdict is the OR of the end bits the slices saw: each thread publishes the
 *     end bits left after its last close, and a thread whose first close ends a record it did not see open ORs
 *     the tails of the threads before it back to the one that saw the opening delimiter;
 *   - the record that opens in the tile and closes after it is finished by the tile's last thread, which simply
 *     keeps walking (global memory); the next tile ignores that close.  Nothing is carried between tiles.
 * Text is staged in shared memory in strips of SL_PER + 4 bytes per thread (an odd number of words), so the 32
 * lanes of a warp, which all read the same offset of their strips, hit 32 different banks.
 * Not for: patterns with '#' or -p (unbounded memory), run delimiters ($$: the pairing depends on the start of
 * the run): those keep the dense tile form. */

#define SL_BATCH 8
template <typename T, int NR, bool COSTS>
__global__ void __launch_bounds__(SL_THREADS)
k_records_slices(const RecParams P)
{
	extern __shared__ __align__(16) uint8_t s_text[];       /* strip 0: the apron; strip t + 1: thread t's slice */
	__shared__ RecShared<T, NR> SH;
	__shared__ T s_tail[NR][SL_THREADS];                     /* end bits seen since the thread's last close (or its slice start) */
	__shared__ long long s_last[SL_THREADS];                 /* where the thread's last close ended = the begin of the open record */
	__shared__ uint8_t s_has[SL_THREADS];                    /* the thread knows where its open record begins */
	__shared__ uint32_t s_scan[SL_THREADS];
	const uint32_t tid = threadIdx.x;
	const int64_t n = (int64_t)P.n, tile0 = (int64_t)blockIdx.x * SL_TILE, tile_end = tile0 + SL_TILE;
	const int64_t readable = (int64_t)(P.n_chunks * 16);
	DevConsts<T> C;
	shared_init<T, NR>(SH, C, P.desc, SL_THREADS);
	const int L = C.L, warm = P.warm;
	const int64_t limit = n + L;
	/* ---- stage [tile0 - SL_APRON, tile_end): coalesced 16-byte loads, stored into the padded strips ---- */
	/* (eight loads in flight per thread before the first store: the loop is latency-bound otherwise) */
	for (uint32_t u0 = tid; u0 < (SL_APRON + SL_TILE) / 16; u0 += SL_BATCH * SL_THREADS) {
		uint4 v[SL_BATCH]; bool ok[SL_BATCH];
#pragma unroll
		for (int b = 0; b < SL_BATCH; b++) {
			const uint32_t u = u0 + b * SL_THREADS;
			const int64_t g = tile0 - SL_APRON + (int64_t)u * 16;
			ok[b] = u < (SL_APRON + SL_TILE) / 16 && g >= 0 && g < readable;
			if (ok[b]) v[b] = __ldg(reinterpret_cast<const uint4 *>(P.text + g));
		}
#pragma unroll
		for (int b = 0; b < SL_BATCH; b++) if (ok[b]) {
			const uint32_t x = (u0 + b * SL_THREADS) * 16 + (SL_PER - SL_APRON);      /* byte number counted from the start of strip 0 */
			uint32_t *dst = reinterpret_cast<uint32_t *>(s_text + (x / SL_PER) * SL_STRIDE + (x & (SL_PER - 1)));
			dst[0] = v[b].x; dst[1] = v[b].y; dst[2] = v[b].z; dst[3] = v[b].w;
		}
	}
	__syncthreads();
	if (tid < (uint32_t)L) {                                 /* the delimiter appended at EOF (bitap.c:161-165) */
		const int64_t g = n + tid;
		if (g >= tile0 - SL_APRON && g < tile_end) {
			const uint32_t x = (uint32_t)(g - tile0 + SL_PER);
			s_text[(x / SL_PER) * SL_STRIDE + (x & (SL_PER - 1))] = SH.delim[tid];
		}
	}
	__syncthreads();

	const int64_t a = tile0 + (int64_t)tid * SL_PER;         /* my slice: [a, a + SL_PER) */
	const uint8_t *mine = s_text + (tid + 1) * SL_STRIDE, *before = s_text + tid * SL_STRIDE + SL_PER;
	const bool text_start = (tile0 == 0 && tid == 0);
	const bool active = a < limit;
	const uint32_t steps = !active ? 0u : (uint32_t)((limit - a) < (int64_t)SL_PER ? (limit - a) : (int64_t)SL_PER);
	const bool overrun = active && tid == SL_THREADS - 1 && tile_end < limit;    /* finish the record that is open at the end of the tile */
	/* (a shard's tiles count the plain way only where every record that opens in them is the shard's own) */
	const bool easy = tile0 > 0 && tile_end + L + 2 < n && tile0 >= P.own_lo && tile_end <= P.own_hi;
	T RS[NR];
#pragma unroll
	for (int r = 0; r < NR; r++) RS[r] = SH.reset[r];
	Reader R; R.init(P.text, P.n, SH.delim, L);

	/* what the first walk leaves behind */
	bool has_first = false, first_ok = false; int first_level = 0;
	int64_t first_end = 0, first_begin = 0;
	T first_bits[NR];
#pragma unroll
	for (int r = 0; r < NR; r++) first_bits[r] = 0;
	uint32_t my_count = 0;
	uint64_t out_pos = 0;

	for (int pass = 0; pass < (P.emit ? 2 : 1); pass++) {
		const bool writing = pass == 1, tally = (pass == 0 && !P.emit);
		uint32_t cnt = 0;
		T S[NR];
		int64_t begin = 0; bool have_begin = false;
		if (active) {
			if (text_start) {
#pragma unroll
				for (int r = 0; r < NR; r++) S[r] = SH.start[r];
				begin = SH.start_closes ? -(int64_t)L : 0; have_begin = true;
			} else {
#pragma unroll
				for (int r = 0; r < NR; r++) S[r] = RS[r];
				/* four bytes per shared-memory word, their four Mask[] words fetched together: the loads of a group do
				 * not wait for the rows of the group before */
				for (int j = -warm; j < 0; j += 4) {
					const uint32_t w = *reinterpret_cast<const uint32_t *>(before + j);
					T m[4];
#pragma unroll
					for (int i = 0; i < 4; i++) m[i] = SH.mask[(w >> (8 * i)) & 0xFFu];
#pragma unroll
					for (int i = 0; i < 4; i++) {
						rows_step<T, NR, COSTS>(S, m[i], C);
						const bool cl = (S[0] & C.dendpos) != 0;             /* selects, not a branch: see below */
#pragma unroll
						for (int r = 0; r < NR; r++) S[r] = cl ? RS[r] : S[r];
					}
				}
#pragma unroll
				for (int r = 0; r < NR; r++) S[r] &= ~C.endpos;      /* whatever matched before the slice is somebody else's business */
			}
		}
		/* one close: the record [begin, end) is complete */
#define SL_CLOSE(endv) do { \
			const int64_t end_ = (endv); \
			if (!have_begin) { \
				if (pass == 0) { has_first = true; first_end = end_; _Pragma("unroll") for (int r = 0; r < NR; r++) first_bits[r] = S[r] & C.endpos; } \
			} else { \
				const bool counts = (begin + 1 < n) && (begin + 1 <= end_) && rec_owned(P, begin, L, end_ + L - 1); \
				int level = C.k; bool cond; \
				if (P.levels) { \
					level = -1; \
					_Pragma("unroll") for (int r = 0; r < NR; r++) if (level < 0 && match_cond<T>(S[r], C)) level = r; \
					cond = level >= 0; \
					if (cond && counts && tally) atomicAdd(&SH.hist[level], 1ull); \
					if (cond && P.want_level >= 0 && level > P.want_level) cond = false; \
				} else cond = match_cond<T>(S[NR - 1], C); \
				if (cond && counts) { \
					if (writing) { \
						const uint64_t at = out_pos + cnt; \
						if (at < P.capacity) { agb_record rec; rec.begin = begin; rec.end = end_; rec.ordinal = 0; rec.level = level; rec.pad = 0; P.records[at] = rec; } \
					} \
					cnt++; \
				} \
			} \
			begin = end_; have_begin = true; \
			_Pragma("unroll") for (int r = 0; r < NR; r++) S[r] = RS[r]; \
		} while (0)

		if (easy && !P.levels && !C.and_mode) {
			/* Plain counting away from both ends of the text: every record counts (agrep.c:3811 only bites at the ends).
			 * No branch on a close: one would be taken by one or two lanes in almost every other step of a warp (a line
			 * ends every ~60 bytes) and the divergence costs far more than it skips.  The loop only resets the rows with
			 * selects and shifts two flags per step into a pair of 32-bit histories -- "a record closed here", "and an
			 * end bit was up" (bitap.c:182 without -v; `;` patterns take
			 * the general loop) -- which are counted and located with popc/clz/ffs once per 32 bytes. */
			int first_j = -1, last_j = -1; bool first_found = false;
			const bool inv = C.inverse != 0;
			uint32_t w = *reinterpret_cast<const uint32_t *>(mine);
			for (uint32_t jb = 0; jb < SL_PER; jb += 32) {              /* easy: the whole slice is text */
				uint32_t cw = 0, fw = 0;                                   /* step jb + s  <->  bit 31 - s */
#pragma unroll (NR <= 3 ? 8 : 1)                                    /* many rows: the body is long enough, keep it in the instruction cache */
				for (int g = 0; g < 8; g++) {
					const uint32_t wn = *reinterpret_cast<const uint32_t *>(mine + jb + 4 * g + 4);   /* (the last one reads the strip's padding) */
					T m[4];
#pragma unroll
					for (int i = 0; i < 4; i++) m[i] = SH.mask[(w >> (8 * i)) & 0xFFu];
#pragma unroll
					for (int i = 0; i < 4; i++) {
						rows_step<T, NR, COSTS>(S, m[i], C);
						const bool cl = (S[0] & C.dendpos) != 0;
						cw = cw * 2u + (cl ? 1u : 0u);
						fw = fw * 2u + ((S[NR - 1] & C.endpos) ? 1u : 0u);         /* sticky: only looked at where cw has a bit */
#pragma unroll
						for (int r = 0; r < NR; r++) S[r] = cl ? RS[r] : S[r];
					}
					w = wn;
				}
				if (cw) {
					uint32_t hits = cw & (inv ? ~fw : fw);
					if (last_j < 0) {                                        /* the slice's first close: that record opened before my slice */
						const int sft = __clz(cw);
						first_j = (int)jb + sft; first_found = ((fw >> (31 - sft)) & 1u) != 0;
						hits &= ~(0x80000000u >> sft);
					}
					if (writing) {
						/* the emit pass walks the closes of this word in order: every hit is a record [previous close, this close) */
						int64_t bg = last_j >= 0 ? a + last_j + 1 - L : 0;       /* (the first close of the slice is never a hit here) */
						for (uint32_t c = cw; c; ) {
							const int sft = __clz(c); const uint32_t bit = 0x80000000u >> sft;
							const int64_t en = a + (int64_t)jb + sft + 1 - L;
							if (hits & bit) {
								const uint64_t at = out_pos + cnt;
								if (at < P.capacity) { agb_record rec; rec.begin = bg; rec.end = en; rec.ordinal = 0; rec.level = C.k; rec.pad = 0; P.records[at] = rec; }
								cnt++;
							}
							bg = en; c &= ~bit;
						}
					} else cnt += __popc(hits);
					last_j = (int)jb + 32 - __ffs(cw);
				}
			}
			const T fb = first_found ? C.endpos : (T)0;
			if (first_j >= 0 && pass == 0) { has_first = true; first_end = a + first_j + 1 - L; first_bits[NR - 1] = fb; }
			if (last_j >= 0) { begin = a + last_j + 1 - L; have_begin = true; }
		} else {
			uint32_t w = *reinterpret_cast<const uint32_t *>(mine);
			for (uint32_t j = 0; j < steps; j += 4) {
				const uint32_t wn = *reinterpret_cast<const uint32_t *>(mine + j + 4);
				T m[4];
#pragma unroll
				for (int i = 0; i < 4; i++) m[i] = SH.mask[(w >> (8 * i)) & 0xFFu];
#pragma unroll
				for (int i = 0; i < 4; i++) if (j + i < steps) {
					rows_step<T, NR, COSTS>(S, m[i], C);
					if (S[0] & C.dendpos) SL_CLOSE(a + (int64_t)(j + i) + 1 - L);
				}
				w = wn;
			}
		}
		if (overrun) {
			for (int64_t p = tile_end; p < limit; p++) {
				rows_step<T, NR, COSTS>(S, SH.mask[R.get(p)], C);
				if (S[0] & C.dendpos) { SL_CLOSE(p + 1 - L); break; }
			}
		}
#undef SL_CLOSE
		if (pass == 0) {
			/* ---- the records that span slices ---- */
#pragma unroll
			for (int r = 0; r < NR; r++) s_tail[r][tid] = active ? (T)(S[r] & C.endpos) : (T)0;
			s_last[tid] = begin; s_has[tid] = have_begin ? 1 : 0;
			__syncthreads();
			if (has_first) {
				bool found = false;
				for (int t = (int)tid - 1; t >= 0; t--) {
#pragma unroll
					for (int r = 0; r < NR; r++) first_bits[r] |= s_tail[r][t];
					if (s_has[t]) { first_begin = s_last[t]; found = true; break; }
				}
				if (found) {                                         /* else: it opened in an earlier tile, whose last thread reports it */
					const bool counts = (first_begin + 1 < n) && (first_begin + 1 <= first_end) && rec_owned(P, first_begin, L, first_end + L - 1);
					int level = C.k; bool cond;
					if (P.levels) {
						level = -1;
#pragma unroll
						for (int r = 0; r < NR; r++) if (level < 0 && match_cond<T>(first_bits[r], C)) level = r;
						cond = level >= 0;
						if (cond && counts && tally) atomicAdd(&SH.hist[level], 1ull);
						if (cond && P.want_level >= 0 && level > P.want_level) cond = false;
					} else cond = match_cond<T>(first_bits[NR - 1], C);
					first_ok = cond && counts; first_level = level;
				}
			}
			my_count = cnt + (first_ok ? 1u : 0u);
			{   /* inclusive scan of the counts: shuffles inside a warp, the warp totals through shared memory */
				uint32_t inc = my_count;
#pragma unroll
				for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if ((tid & 31) >= (uint32_t)o) inc += v; }
				if ((tid & 31) == 31) s_scan[tid >> 5] = inc;
				__syncthreads();
				uint32_t base = 0;
#pragma unroll
				for (int w = 0; w < SL_THREADS / 32; w++) if ((uint32_t)w < (tid >> 5)) base += s_scan[w];
				__syncthreads();
				s_scan[tid] = base + inc;
				__syncthreads();
			}
			if (!P.emit) {
				if (tid == SL_THREADS - 1) {
					P.tile_counts[blockIdx.x] = s_scan[SL_THREADS - 1];
					if (s_scan[SL_THREADS - 1]) atomicAdd(&P.totals[0], (unsigned long long)s_scan[SL_THREADS - 1]);
					const int64_t tile_len = (n - tile0) < (int64_t)SL_TILE ? (n - tile0) : (int64_t)SL_TILE;
					atomicAdd(&P.totals[1], (unsigned long long)((tile_len + 15) / 16));
				}
				__syncthreads();
				if (P.levels && tid <= AGB_MAXERR && SH.hist[tid]) atomicAdd(&P.totals[2 + tid], SH.hist[tid]);
			} else {
				out_pos = P.tile_offsets[blockIdx.x] + (s_scan[tid] - my_count);
				if (first_ok) {                                      /* the spanning record comes before the thread's own */
					if (out_pos < P.capacity) { agb_record rec; rec.begin = first_begin; rec.end = first_end; rec.ordinal = 0; rec.level = first_level; rec.pad = 0; P.records[out_pos] = rec; }
					out_pos++;
				}
			}
		}
	}
}

template <typename T, int NR, bool COSTS>
static void launch_slices_one(const RecParams &P, unsigned grid, cudaStream_t st)
{
	static bool configured[64] = {false};
	int dev = 0; cudaGetDevice(&dev);
	if (!configured[dev & 63]) {
		cudaFuncSetAttribute(k_records_slices<T, NR, COSTS>, cudaFuncAttributeMaxDynamicSharedMemorySize, SL_SMEM);
		configured[dev & 63] = true;
	}
	k_records_slices<T, NR, COSTS><<<grid, SL_THREADS, SL_SMEM, st>>>(P);
}
template <typename T, bool COSTS>
static int launch_slices_t(int nrows, const RecParams &P, unsigned grid, cudaStream_t st)
{
	return launch_rows<9>(nrows, [&](auto R) { launch_slices_one<T, decltype(R)::value, COSTS>(P, grid, st); });
}
int launch_slices(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st)
{
	const bool costs = d.engine == AGB_ENGINE_ASEARCH1, narrow = d.M <= 31;
	if (costs) return narrow ? launch_slices_t<uint32_t, true>(d.nrows, P, grid, st) : launch_slices_t<uint64_t, true>(d.nrows, P, grid, st);
	return narrow ? launch_slices_t<uint32_t, false>(d.nrows, P, grid, st) : launch_slices_t<uint64_t, false>(d.nrows, P, grid, st);
}
/* the slices form needs a bounded memory: no position that holds for ever ('#': wildmask; -p: Init1 = ~0) and a
 * delimiter whose occurrences do not depend on where a run of it started; and rows of at most 64 bits */
bool slices_usable(const agb_desc &d)
{
	return !d.wide && d.wildmask == 0 && d.init1 != ~0ull && (d.L == 1 || d.delim_kind == 0) && d.M + d.nrows + 2 <= SL_APRON;
}

