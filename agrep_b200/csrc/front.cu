/* agrep_b200/csrc/front.cu -- stage 1: the anchor front-end, the HBM-bound kernel (DESIGN.md 3.1) */
#include "scan_internal.cuh"
#include "tma.cuh"

/* ================================================================================================
 * stage 1: anchor front-end
 * ============================================================================================== */

/* The 4 windows that start in word `lo` (bytes 0..3; `hi` = the following word) against the NA anchors.
 * Result: acc stays non-zero unless some window equals some anchor.
 *
 * POLY: f(w) = prod_i (w - A_i) mod 2^32, evaluated by Horner -- NA IMADs on the FMA pipe per window and
 * half a VIMNMX3 on the ALU pipe, instead of NA compare-class ALU ops.  w == A_i  =>  f(w) == 0 exactly
 * (ring identity), so the filter never loses a match; f(w) == 0 without an equal factor needs the 2-adic
 * valuations of the NA differences to add up to 32, which front_launch() rules out up front (it falls back
 * to the compare form when anchors share low-order bytes).  Anchors shorter than 4 bytes: f is scaled by
 * 256^(4-len), which zeroes exactly when the low len bytes agree.
 * !POLY: unsigned min of the differences (VIADDMNMX), one ALU op per window and anchor. */
template <int NA, bool MASKED, bool POLY, int N3>
__device__ __forceinline__ uint32_t windows_test(uint32_t lo, uint32_t hi, const FrontParams &P, uint32_t acc)
{
	uint32_t w[4] = { lo, __funnelshift_r(lo, hi, 8), __funnelshift_r(lo, hi, 16), __funnelshift_r(lo, hi, 24) };
	if (POLY && N3 > 0) {
		/* mixed plan: NA anchors of four bytes and N3 of three (a piece of the pattern that is only three bytes long, or
		 * whose rare gram is).  Two polynomials -- one product would cut every anchor to its low three bytes -- the second
		 * scaled by 256 so that it vanishes exactly when the low three bytes agree; one VIMNMX3 per window takes both. */
#pragma unroll
		for (int t = 0; t < 4; t++) {
			uint32_t r = (NA >= 2) ? __viaddmin_u32(w[t], P.coef[NA - 1], 0xFFFFFFFFu) : w[t] * P.one + P.coef[NA - 1];
#pragma unroll
			for (int i = NA - 2; i >= 0; i--) r = r * w[t] + P.coef[i];
			if (MASKED) r *= P.scale;                            /* (two groups of three-byte anchors: both scaled) */
			uint32_t q;
			if (N3 == 1) q = w[t] * P.s256 + P.coef3[0];             /* 256 (w - B): coef3[0] = -256 B; s256: a run-time 256, so that this stays an IMAD (FMA pipe) and does not become a shift-add on the ALU pipe, which the min and funnel shifts already fill */
			else {
				q = w[t] * P.one + P.coef3[N3 - 1];
#pragma unroll
				for (int i = N3 - 2; i >= 0; i--) q = q * w[t] + P.coef3[i];
				q *= P.s256;
			}
			acc = __vimin3_u32(acc, r, q);
		}
		return acc;
	}
	if (POLY) {
		uint32_t f[4];
#pragma unroll
		for (int t = 0; t < 4; t++) {
			/* Horner.  IMAD (FMA pipe, 64 lanes/clk/SM) and the ALU pipe (64 lanes/clk/SM) both count: with three
			 * or more anchors the first step, w + c, goes to the ALU pipe as VIADDMNMX (min(w + c, ~0)), which
			 * leaves NA-1 IMADs per window; `one` is a runtime 1 that keeps the step an IMAD otherwise */
			uint32_t r = (NA >= 3) ? __viaddmin_u32(w[t], P.coef[NA - 1], 0xFFFFFFFFu) : w[t] * P.one + P.coef[NA - 1];
#pragma unroll
			for (int i = NA - 2; i >= 0; i--) r = r * w[t] + P.coef[i];
			f[t] = MASKED ? r * P.scale : r;
		}
		acc = __vimin3_u32(acc, f[0], f[1]);
		acc = __vimin3_u32(acc, f[2], f[3]);
	} else {
		if (MASKED) { w[0] &= P.amask; w[1] &= P.amask; w[2] &= P.amask; w[3] &= P.amask; }
#pragma unroll
		for (int a = 0; a < NA; a++) {
			uint32_t A = P.anchor[a];
			acc = __vimin3_u32(acc, w[0] - A, w[1] - A);
			acc = __vimin3_u32(acc, w[2] - A, w[3] - A);
		}
	}
	return acc;
}

/* -n: the delimiter bytes of chunk idx of the stage (SWAR: 0x80 where a byte equals the delimiter); summed over a warp
 * they make one 512-byte block of the ordinals pass (aux.cu), which then need not read the text again */
template <bool FULL>
__device__ __forceinline__ uint32_t chunk_delims(const FrontParams &P, const uint4 v, uint32_t idx, uint32_t rem)
{
	const uint32_t xs[4] = { v.x, v.y, v.z, v.w };
	uint32_t cn = 0;
#pragma unroll
	for (int w = 0; w < 4; w++) {
		const uint32_t t = (xs[w] | P.dfold4) ^ P.delim4;
		uint32_t z = ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t | 0x7F7F7F7Fu);
		if (!FULL) {                                     /* only bytes of the text */
			/* rem chunks are left from the start of the stage, the last one padded: bytes of this word inside the text */
			const int64_t valid = ((int64_t)rem - (int64_t)idx) * 16 - (int64_t)(P.n_chunks * 16 - P.n) - 4 * w;
			if (valid <= 0) z = 0; else if (valid < 4) z &= (1u << (8 * (uint32_t)valid)) - 1u;
		}
		cn += __popc(z);
	}
	return cn;
}

/* the FRONT_CH chunks a thread takes from one stage; FULL = no chunk of the stage is near the end of the text */
template <int NA, bool MASKED, bool FOLD, bool POLY, bool FULL, bool COUNT, int N3>
__device__ __forceinline__ void front_chunks(const FrontParams &P, const uint8_t *st, uint32_t tid, uint32_t lane, uint32_t rem, uint32_t *bm, uint16_t *nlb)
{
#pragma unroll
	for (int c = 0; c < FRONT_CH; c++) {
		const uint32_t idx = c * FRONT_THREADS + tid;
		uint4 v = *reinterpret_cast<const uint4 *>(st + idx * 16);
		/* the first word of the next chunk (a 4-way bank conflict; the alternative is a SHFL + a predicated LDS for
		 * the warp's last lane, which costs more issue slots) */
		uint32_t x4 = *reinterpret_cast<const uint32_t *>(st + idx * 16 + 16);
		if (COUNT) {
			const uint32_t blk = __reduce_add_sync(0xffffffffu, chunk_delims<FULL>(P, v, idx, rem));
			if (lane == 0 && (FULL || idx < rem)) nlb[c * (FRONT_THREADS / 32)] = (uint16_t)blk;
		}
		if (FOLD) { v.x |= P.fold; v.y |= P.fold; v.z |= P.fold; v.w |= P.fold; x4 |= P.fold; }
		uint32_t acc = 0xffffffffu;
		acc = windows_test<NA, MASKED, POLY, N3>(v.x, v.y, P, acc);
		acc = windows_test<NA, MASKED, POLY, N3>(v.y, v.z, P, acc);
		acc = windows_test<NA, MASKED, POLY, N3>(v.z, v.w, P, acc);
		acc = windows_test<NA, MASKED, POLY, N3>(v.w, x4, P, acc);
		if (FULL) {
			const uint32_t word = __ballot_sync(0xffffffffu, acc == 0);
			if (lane == 0) bm[c * (FRONT_THREADS / 32)] = word;
		} else {
			/* the last chunks are always passed on: a match may run into the delimiter appended at EOF
			 * (bitap.c:161-165), and their look-ahead bytes may not exist */
			const bool flag = (idx < rem) && (acc == 0 || idx + 2 >= rem);
			const uint32_t word = __ballot_sync(0xffffffffu, flag);
			if (lane == 0 && idx < rem) bm[c * (FRONT_THREADS / 32)] = word;
		}
	}
}

/* ---- the pair plan (DESIGN.md 3.1): k + 2 distinct pieces of len bytes; k errors leave two of them verbatim, and the
 * second of those starts at most (o_last - o_first) + k <= 16 bytes after the first (the planner checks the bound), so
 * it starts in the first one's chunk or in the chunk after it.  A chunk is flagged when some piece starts in it and
 * some other piece starts in it or in its successor. */

/* an IMAD the compiler may not split into a shared multiply and ALU adds (w * scale is the same for every piece) */
__device__ __forceinline__ uint32_t imad(uint32_t a, uint32_t b, uint32_t c)
{
	uint32_t r; asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r;
}

/* bit i = piece i starts in the chunk x[0..3] (x[4]: the word after it).  w * scale + coef[i] = (w - B_i) * 256^(4-len)
 * vanishes exactly when the low len bytes of window w are piece i: one IMAD per window and piece, half a VIMNMX3 to fold
 * it; the running minimum starts at 1, so it ends as 0 (present) or 1 */
template <int NP>
__device__ __forceinline__ uint32_t piece_bits(const uint32_t (&x)[5], const FrontParams &P)
{
	uint32_t acc[NP];
#pragma unroll
	for (int i = 0; i < NP; i++) acc[i] = 1u;
#pragma unroll
	for (int w = 0; w < 4; w++) {
		const uint32_t wv[4] = { x[w], __funnelshift_r(x[w], x[w + 1], 8), __funnelshift_r(x[w], x[w + 1], 16), __funnelshift_r(x[w], x[w + 1], 24) };
#pragma unroll
		for (int i = 0; i < NP; i++) {
			acc[i] = __vimin3_u32(acc[i], imad(wv[0], P.scale, P.coef[i]), imad(wv[1], P.scale, P.coef[i]));
			acc[i] = __vimin3_u32(acc[i], imad(wv[2], P.scale, P.coef[i]), imad(wv[3], P.scale, P.coef[i]));
		}
	}
	uint32_t absent = 0;
#pragma unroll
	for (int i = 0; i < NP; i++) absent |= acc[i] << i;
	return absent ^ ((1u << NP) - 1u);
}

/* A warp takes FRONT_CH consecutive groups of 32 chunks (bitmap words wid * FRONT_CH + c of the stage), so the successor of
 * a lane's chunk is the next lane's, or lane 0's of the next group: one SHFL.  The warp's very last chunk (1 in 128) has its
 * successor in another warp; it is flagged when it holds any piece, which keeps the filter exact. */
template <int NP, bool FOLD, bool FULL, bool COUNT>
__device__ __forceinline__ void pair_chunks(const FrontParams &P, const uint8_t *st, uint32_t wid, uint32_t lane, uint32_t rem, uint32_t *bm, uint16_t *nlb)
{
	uint32_t pres[FRONT_CH];
#pragma unroll
	for (int c = 0; c < FRONT_CH; c++) {
		const uint32_t idx = (wid * FRONT_CH + c) * 32 + lane;
		const uint4 v = *reinterpret_cast<const uint4 *>(st + idx * 16);
		const uint32_t x4 = *reinterpret_cast<const uint32_t *>(st + idx * 16 + 16);
		if (COUNT) {
			const uint32_t blk = __reduce_add_sync(0xffffffffu, chunk_delims<FULL>(P, v, idx, rem));
			if (lane == 0 && (FULL || idx < rem)) nlb[c] = (uint16_t)blk;
		}
		const uint32_t f = FOLD ? P.fold : 0u;
		const uint32_t x[5] = { v.x | f, v.y | f, v.z | f, v.w | f, x4 | f };
		pres[c] = piece_bits<NP>(x, P);
	}
#pragma unroll
	for (int c = 0; c < FRONT_CH; c++) {
		const uint32_t idx = (wid * FRONT_CH + c) * 32 + lane;
		const uint32_t give = (lane == 0 && c + 1 < FRONT_CH) ? pres[c + 1] : pres[c];
		uint32_t next = __shfl_sync(0xffffffffu, give, (lane + 1) & 31);
		if (c + 1 == FRONT_CH && lane == 31) next = ~0u;
		const bool pair = pres[c] != 0 && __popc(pres[c] | next) >= 2;
		if (FULL) {
			const uint32_t word = __ballot_sync(0xffffffffu, pair);
			if (lane == 0) bm[c] = word;
		} else {
			/* the last two chunks of the text are always passed on, as in front_chunks */
			const uint32_t word = __ballot_sync(0xffffffffu, (idx < rem) && (pair || idx + 2 >= rem));
			if (lane == 0 && idx < rem) bm[c] = word;
		}
	}
}

/* Persistent CTAs.  Thread 0 keeps FRONT_NST bulk copies of 16 KiB (+16 B) in flight into a shared-memory
 * ring, each completing on its own mbarrier; all 256 threads take 4 chunks per stage from shared memory
 * (LDS.128, conflict-free: a warp reads 512 consecutive bytes), test the 16 windows of each chunk and ballot
 * the 32 verdicts of a warp into one bitmap word.  Every text byte crosses HBM->SM once.  NP > 0: the pair plan's test
 * (pair_chunks) over NP pieces instead of the anchor test. */
template <int NA, bool MASKED, bool FOLD, bool POLY, bool COUNT, int N3, int NP = 0>
__global__ void __launch_bounds__(FRONT_THREADS, FRONT_CTAS_PER_SM)
k_front(const FrontParams P)
{
	extern __shared__ __align__(128) uint8_t s_ring[];
	__shared__ uint64_t s_bar[FRONT_NST];
	const uint32_t tid = threadIdx.x, lane = tid & 31;
	if (tid == 0) {
		for (int i = 0; i < FRONT_NST; i++) mbar_init(&s_bar[i], 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	auto issue = [&](uint64_t it) {
		const uint64_t sg = P.stage_begin + blockIdx.x + it * gridDim.x;
		if (sg >= P.stage_end) return;
		const uint32_t slot = (uint32_t)(it % FRONT_NST);
		const uint64_t off = sg * FRONT_STAGE_BYTES, avail = P.readable - off;
		const uint32_t bytes = (uint32_t)(avail < FRONT_SLOT_BYTES ? (avail & ~15ull) : FRONT_SLOT_BYTES);
		mbar_expect_tx(&s_bar[slot], bytes);
		bulk_g2s(s_ring + slot * FRONT_SLOT_BYTES, P.text + off, bytes, &s_bar[slot]);
	};
	if (tid == 0) for (int i = 0; i < FRONT_NST; i++) issue(i);
	const uint32_t warp_in_cta = tid >> 5;
	for (uint32_t it = 0;; it++) {
		const uint64_t sg = P.stage_begin + blockIdx.x + (uint64_t)it * gridDim.x;
		if (sg >= P.stage_end) break;
		const uint32_t slot = it % FRONT_NST;
		mbar_wait(&s_bar[slot], (it / FRONT_NST) & 1u);
		const uint8_t *st = s_ring + slot * FRONT_SLOT_BYTES;
		/* per-stage scalars, so that the per-chunk bookkeeping below is 32-bit */
		const uint64_t left = P.n_chunks - sg * FRONT_STAGE_CHUNKS;                    /* chunks from the start of this stage to EOF */
		const uint32_t rem = left > 0xFFFF0000ull ? 0xFFFF0000u : (uint32_t)left;
		uint32_t *bm = P.bitmap + sg * FRONT_WORDS_PER_STAGE + warp_in_cta;
		/* full = every chunk of the stage exists and none is among the last two of the text: no per-chunk EOF logic */
		const bool full = left >= FRONT_STAGE_CHUNKS + 2;
		if constexpr (NP > 0) {
			/* a warp's FRONT_CH words are consecutive here */
			uint32_t *bmp = P.bitmap + sg * FRONT_WORDS_PER_STAGE + warp_in_cta * FRONT_CH;
			uint16_t *nlp = COUNT ? P.nl_blocks + sg * FRONT_WORDS_PER_STAGE + warp_in_cta * FRONT_CH : nullptr;
			if (full) pair_chunks<NP, FOLD, true, COUNT>(P, st, warp_in_cta, lane, rem, bmp, nlp);
			else pair_chunks<NP, FOLD, false, COUNT>(P, st, warp_in_cta, lane, rem, bmp, nlp);
		} else {
			uint16_t *nlb = COUNT ? P.nl_blocks + sg * FRONT_WORDS_PER_STAGE + warp_in_cta : nullptr;
			if (full) front_chunks<NA, MASKED, FOLD, POLY, true, COUNT, N3>(P, st, tid, lane, rem, bm, nlb);
			else front_chunks<NA, MASKED, FOLD, POLY, false, COUNT, N3>(P, st, tid, lane, rem, bm, nlb);
		}
		__syncthreads();                       /* everyone is done reading this slot */
		if (tid == 0) issue((uint64_t)it + FRONT_NST);   /* refill it with the stage FRONT_NST iterations ahead */
	}
}

template <int NA, bool MASKED, bool FOLD, bool POLY, bool COUNT, int N3, int NP = 0>
static void launch_front_cnt(const FrontParams &P, unsigned grid, cudaStream_t st)
{
	static bool configured[64] = {false};
	int dev = 0; cudaGetDevice(&dev);
	if (!configured[dev & 63]) {
		cudaFuncSetAttribute(k_front<NA, MASKED, FOLD, POLY, COUNT, N3, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, FRONT_SMEM);
		configured[dev & 63] = true;
	}
	k_front<NA, MASKED, FOLD, POLY, COUNT, N3, NP><<<grid, FRONT_THREADS, FRONT_SMEM, st>>>(P);
}
/* the pair plan over NP pieces */
template <int NP>
static void launch_front_pairs(const FrontParams &P, bool fold, unsigned grid, cudaStream_t st)
{
	if (P.nl_blocks) { if (fold) launch_front_cnt<0, false, true, true, true, 0, NP>(P, grid, st); else launch_front_cnt<0, false, false, true, true, 0, NP>(P, grid, st); }
	else             { if (fold) launch_front_cnt<0, false, true, true, false, 0, NP>(P, grid, st); else launch_front_cnt<0, false, false, true, false, 0, NP>(P, grid, st); }
}
template <int NA, bool MASKED, bool FOLD, bool POLY, int N3>
static void launch_front_one(const FrontParams &P, unsigned grid, cudaStream_t st)
{
	if (P.nl_blocks) launch_front_cnt<NA, MASKED, FOLD, POLY, true, N3>(P, grid, st);
	else launch_front_cnt<NA, MASKED, FOLD, POLY, false, N3>(P, grid, st);
}
template <int NA, bool POLY>
static void launch_front_na(const FrontParams &P, bool masked, bool fold, unsigned grid, cudaStream_t st)
{
	if (masked) { if (fold) launch_front_one<NA, true, true, POLY, 0>(P, grid, st); else launch_front_one<NA, true, false, POLY, 0>(P, grid, st); }
	else        { if (fold) launch_front_one<NA, false, true, POLY, 0>(P, grid, st); else launch_front_one<NA, false, false, POLY, 0>(P, grid, st); }
}
/* mixed plans: four-byte anchors by the polynomial + one or two three-byte anchors */
template <int NA>
static void launch_front_mixed(const FrontParams &P, bool fold, unsigned grid, cudaStream_t st)
{
	if (P.n3 == 1) { if (fold) launch_front_one<NA, false, true, true, 1>(P, grid, st); else launch_front_one<NA, false, false, true, 1>(P, grid, st); }
	else           { if (fold) launch_front_one<NA, false, true, true, 2>(P, grid, st); else launch_front_one<NA, false, false, true, 2>(P, grid, st); }
}
/* three-byte anchors whose one polynomial fails the false-positive guard (two of them share their first byte, "aus" and
 * "ach"), split into two groups that pass it: both polynomials scaled by 256 */
template <int NA>
static void launch_front_split3(const FrontParams &P, bool fold, unsigned grid, cudaStream_t st)
{
	if (P.n3 == 1) { if (fold) launch_front_one<NA, true, true, true, 1>(P, grid, st); else launch_front_one<NA, true, false, true, 1>(P, grid, st); }
	else           { if (fold) launch_front_one<NA, true, true, true, 2>(P, grid, st); else launch_front_one<NA, true, false, true, 2>(P, grid, st); }
}

/* ================================================================================================
 * exact literal no longer than its anchor, count only (`agrep -c the`): no automaton at all.
 *
 * Every occurrence of the literal IS an anchor hit, so the number of matching records is the number of records that
 * hold a hit: hits and delimiters are both properties of the bytes, and "the record of this hit already had one" is
 * "no delimiter since the hit before".  One pass, the same persistent TMA ring as k_front; per 16-byte chunk the
 * anchor test (one window per byte) and "is there a delimiter byte in here" (SWAR); the 32 chunks of a warp are stitched
 * with ballots -- a hit starts a new record if a delimiter lies between it and the hit before -- and only chunks that
 * hold both a hit and a delimiter look at byte positions.  A warp writes one summary word per 512 bytes where stage 1
 * writes its bitmap word: records with a hit not counting the first hit's, and whether a delimiter lies before the
 * first hit / after the last / anywhere; the summaries form a monoid under concatenation (k_exact_reduce).
 * sgrep.c:731-795 (bm(): count the record, jump to its end), bitap.c:177-229 with a literal and no errors.
 * ============================================================================================== */
#define EX_HAS   (1u << 16)
#define EX_LEAD  (1u << 17)
#define EX_TRAIL (1u << 18)
#define EX_ANY   (1u << 19)

/* exact per-byte equality: 0x80 in every byte of x that equals the byte replicated in c4 */
__device__ __forceinline__ uint32_t eq_bytes(uint32_t x, uint32_t c4)
{
	const uint32_t t = x ^ c4;
	return ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t | 0x7F7F7F7Fu);
}

template <bool MASKED, bool FOLD, bool FULL>
__device__ __forceinline__ void exact_chunks(const FrontParams &P, const uint8_t *st, uint32_t tid, uint32_t lane, uint32_t rem, uint32_t *bmw, uint64_t stage_byte0)
{
	const uint32_t lt = (1u << lane) - 1u;
	static_assert(FRONT_CH % 2 == 0, "a lane takes two adjacent chunks");
#pragma unroll 1
	for (int c = 0; c < FRONT_CH / 2; c++) {
		/* a lane takes 32 consecutive bytes (two chunks), a warp 1 KiB = two summary words: the stitching below is paid once
		 * per 32 bytes */
		const uint32_t idx = 2 * (c * FRONT_THREADS + tid);
		const uint4 v0 = *reinterpret_cast<const uint4 *>(st + idx * 16);
		const uint4 v1 = *reinterpret_cast<const uint4 *>(st + idx * 16 + 16);
		const uint32_t x8 = *reinterpret_cast<const uint32_t *>(st + idx * 16 + 32);
		const uint32_t raw[9] = { v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, x8 };
		/* one bit per byte position, no branches: hm = windows that equal the literal, nm = delimiter bytes.  Both tests are
		 * "a scaled difference is zero" (IMAD), turned into a bit by min(.,1) and shifted in by a multiply-add: 4 FMA-pipe and
		 * 2.75 ALU-pipe instructions per window.  Windows run backwards so that byte 0 ends up in bit 0. */
		uint32_t ah = 0, ad = 0;
#pragma unroll
		for (int w = 7; w >= 0; w--) {
			const uint32_t wv[4] = { raw[w], __funnelshift_r(raw[w], raw[w + 1], 8), __funnelshift_r(raw[w], raw[w + 1], 16), __funnelshift_r(raw[w], raw[w + 1], 24) };
#pragma unroll
			for (int j = 3; j >= 0; j--) {
				const uint32_t dh = (FOLD ? (wv[j] | P.fold) : wv[j]) * P.scale - P.coef[0];   /* zero iff the low alen bytes are the literal */
				const uint32_t dd = wv[j] * P.coef3[2] - P.coef3[1];                            /* zero iff the low byte is the delimiter */
				ah = ah * P.coef3[0] + __vimin3_u32(dh, 1u, 1u);
				ad = ad * P.coef3[0] + __vimin3_u32(dd, 1u, 1u);
			}
		}
		uint32_t hm = ~ah, nm = ~ad;
		if (!FULL) {
			const int64_t nb = (int64_t)P.n - ((int64_t)stage_byte0 + (int64_t)idx * 16);   /* bytes of the text in these 32 */
			if (nb < 32 + 4) {
				const int64_t nh = nb - (int64_t)P.alen + 1;                                /* windows that lie inside the text */
				nm &= nb >= 32 ? 0xFFFFFFFFu : (nb <= 0 ? 0u : ((1u << nb) - 1u));
				hm &= nh >= 32 ? 0xFFFFFFFFu : (nh <= 0 ? 0u : ((1u << nh) - 1u));
			}
		}
		/* a hit counts if it is the first since the last delimiter.  Across lanes by ballots: has a hit been seen since the
		 * last delimiter before these bytes (within the warp's 1 KiB)? */
		const uint32_t Hb = __ballot_sync(0xffffffffu, hm != 0), Db = __ballot_sync(0xffffffffu, nm != 0);
		const uint32_t Tb = __ballot_sync(0xffffffffu, nm != 0 && hm > nm);      /* a hit after the lane's last delimiter */
		const uint32_t pd = Db & lt;
		uint32_t seen;
		if (pd) { const int p = 31 - __clz(pd); seen = ((Tb >> p) & 1u) | ((Hb & lt & ~((2u << p) - 1u)) ? 1u : 0u); }
		else seen = (Hb & lt) ? 1u : 0u;
		/* inside the lane by one subtraction: a borrow started at every record start (the bit after a delimiter; bit 0 unless
		 * a hit has been seen) runs up to the first hit or delimiter of that record and clears it (or leaves at the top) */
		const uint32_t ev = hm | nm;
		const uint32_t first = ev & ~(ev - ((nm << 1) | (seen ^ 1u))) & hm;
		const uint32_t Fs = __reduce_add_sync(0xffffffffu, (uint32_t)__popc(first));
		const uint32_t Lb = __ballot_sync(0xffffffffu, hm != 0 && (nm & ((hm & (0u - hm)) - 1u)) != 0);   /* a delimiter before the lane's first hit */
		const uint32_t Gb = __ballot_sync(0xffffffffu, hm != 0 && nm > hm);                                /* ... after its last hit */
		if (lane == 0) {
			uint32_t sum = 0;
			if (Hb) {
				const int fi = __ffs(Hb) - 1, la = 31 - __clz(Hb);
				sum = (Fs - 1u) | EX_HAS;
				if (((Lb >> fi) & 1u) || (Db & ((1u << fi) - 1u))) sum |= EX_LEAD;
				if (((Gb >> la) & 1u) || (la < 31 && (Db >> (la + 1)))) sum |= EX_TRAIL;
			}
			if (Db) sum |= EX_ANY;
			/* the summary of the 1 KiB in its first word, the identity in the second */
			const uint32_t word = idx / 32;
			if (FULL || idx < rem) bmw[word] = sum;
			if (FULL || idx + 32 < rem) bmw[word + 1] = 0;
		}
	}
}

template <bool MASKED, bool FOLD>
__global__ void __launch_bounds__(FRONT_THREADS, FRONT_CTAS_PER_SM)
k_front_exact(const FrontParams P)
{
	extern __shared__ __align__(128) uint8_t s_ring[];
	__shared__ uint64_t s_bar[FRONT_NST];
	const uint32_t tid = threadIdx.x, lane = tid & 31;
	if (tid == 0) {
		for (int i = 0; i < FRONT_NST; i++) mbar_init(&s_bar[i], 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	auto issue = [&](uint64_t it) {
		const uint64_t sg = P.stage_begin + blockIdx.x + it * gridDim.x;
		if (sg >= P.stage_end) return;
		const uint32_t slot = (uint32_t)(it % FRONT_NST);
		const uint64_t off = sg * FRONT_STAGE_BYTES, avail = P.readable - off;
		const uint32_t bytes = (uint32_t)(avail < FRONT_SLOT_BYTES ? (avail & ~15ull) : FRONT_SLOT_BYTES);
		mbar_expect_tx(&s_bar[slot], bytes);
		bulk_g2s(s_ring + slot * FRONT_SLOT_BYTES, P.text + off, bytes, &s_bar[slot]);
	};
	if (tid == 0) for (int i = 0; i < FRONT_NST; i++) issue(i);
	for (uint32_t it = 0;; it++) {
		const uint64_t sg = P.stage_begin + blockIdx.x + (uint64_t)it * gridDim.x;
		if (sg >= P.stage_end) break;
		const uint32_t slot = it % FRONT_NST;
		mbar_wait(&s_bar[slot], (it / FRONT_NST) & 1u);
		const uint8_t *st = s_ring + slot * FRONT_SLOT_BYTES;
		const uint64_t left = P.n_chunks - sg * FRONT_STAGE_CHUNKS;
		const uint32_t rem = left > 0xFFFF0000ull ? 0xFFFF0000u : (uint32_t)left;
		uint32_t *bmw = P.bitmap + sg * FRONT_WORDS_PER_STAGE;
		const bool full = left >= FRONT_STAGE_CHUNKS + 2;
		if (full) exact_chunks<MASKED, FOLD, true>(P, st, tid, lane, rem, bmw, sg * FRONT_STAGE_BYTES);
		else exact_chunks<MASKED, FOLD, false>(P, st, tid, lane, rem, bmw, sg * FRONT_STAGE_BYTES);
		__syncthreads();
		if (tid == 0) issue((uint64_t)it + FRONT_NST);
	}
}

/* the summaries of consecutive 512-byte stretches, combined in order: {records with a hit beyond the first hit's, a hit at
 * all, a delimiter before the first hit, after the last hit, anywhere} */
struct ExSum { unsigned long long cnt; uint32_t fl; };
__device__ __forceinline__ ExSum ex_combine(const ExSum a, const ExSum b)
{
	ExSum r;
	if (!(b.fl & EX_HAS)) { r = a; if (b.fl & EX_ANY) r.fl |= EX_ANY | ((a.fl & EX_HAS) ? EX_TRAIL : 0u); return r; }
	if (!(a.fl & EX_HAS)) { r = b; if (a.fl & EX_ANY) r.fl |= EX_ANY | EX_LEAD; return r; }
	r.cnt = a.cnt + b.cnt + (((a.fl & EX_TRAIL) || (b.fl & EX_LEAD)) ? 1ull : 0ull);
	r.fl = EX_HAS | (a.fl & EX_LEAD) | (b.fl & EX_TRAIL) | ((a.fl | b.fl) & EX_ANY);
	return r;
}
#define EXR_THREADS 256
#define EXR_PER     16
/* level 0: block b combines summaries [b * 4096, (b + 1) * 4096) into part[b]; level 1 (final): one block combines part[] and
 * writes the number of matching records */
__global__ void __launch_bounds__(EXR_THREADS) k_exact_reduce(const uint32_t *sums, uint64_t n, ExSum *part_in, ExSum *part_out, unsigned long long *total)
{
	__shared__ ExSum s_w[EXR_THREADS / 32];
	const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	ExSum acc; acc.cnt = 0; acc.fl = 0;
	const uint64_t i0 = ((uint64_t)blockIdx.x * EXR_THREADS + tid) * EXR_PER;
	for (int j = 0; j < EXR_PER; j++) {
		const uint64_t i = i0 + j;
		if (i >= n) break;
		ExSum e;
		if (part_in) e = part_in[i]; else { const uint32_t w = sums[i]; e.cnt = w & 0xFFFFu; e.fl = w & 0xFFFF0000u; }
		acc = ex_combine(acc, e);
	}
	for (int o = 1; o < 32; o <<= 1) {
		ExSum b; b.cnt = __shfl_down_sync(0xffffffffu, acc.cnt, o); b.fl = __shfl_down_sync(0xffffffffu, acc.fl, o);
		if (lane + o < 32 && (lane % (2 * o)) == 0) acc = ex_combine(acc, b);
	}
	if (lane == 0) s_w[wid] = acc;
	__syncthreads();
	if (tid == 0) {
		ExSum t = s_w[0];
		for (int w = 1; w < EXR_THREADS / 32; w++) t = ex_combine(t, s_w[w]);
		if (part_out) part_out[blockIdx.x] = t;
		if (total) *total = t.cnt + ((t.fl & EX_HAS) ? 1ull : 0ull);
	}
}

bool exact_count_usable(const agb_desc &d)
{
	if (!front_usable(d) || d.wide || d.k != 0 || d.n_anchors != 1 || d.n_anchors3 || d.pat_len != d.anchor_len || d.inverse || d.L != 1 || d.and_mode) return false;
	if (d.engine != AGB_ENGINE_BITAP && d.engine != AGB_ENGINE_SGREP_BM) return false;
	if (d.wildmask || d.init1 == ~0ull || d.delim_fold[0]) return false;
	for (int t = 0; t < d.anchor_len; t++) {
		const int c = (int)(d.anchor[0] >> (8 * t) & 0xFF);
		if (c == d.delim[0]) return false;
		/* the anchor test is exact for this byte: no fold, or a letter whose two cases are what the pattern accepts */
		const uint64_t bit = 1ull << (d.M - (d.L + 2 + t));
		int cnt = 0; for (int b = 0; b < 256; b++) if (d.mask[b] & bit) cnt++;
		const bool alpha = (c | 32) >= 'a' && (c | 32) <= 'z';
		if (d.anchor_fold) { if (!(alpha && cnt == 2 && (d.mask[c | 32] & bit) && (d.mask[(c | 32) - 32] & bit))) return false; }
		else if (!(cnt == 1 && (d.mask[c] & bit))) return false;
	}
	return true;
}

/* count of the records that hold the literal: the exact pass + the ordered reduction of its summaries into totals[0] */
int exact_count_launch(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n, cudaStream_t st)
{
	const uint64_t n_chunks = (n + 15) / 16, n_words = (n_chunks + 31) / 32;
	if (!n_words) return AGB_OK;
	FrontParams F; memset(&F, 0, sizeof F);
	F.text = (const uint8_t *)d_text; F.bitmap = W.bitmap; F.n = n; F.n_chunks = n_chunks;
	F.readable = n_chunks * 16;
	F.stage_begin = 0; F.stage_end = (n_words + FRONT_WORDS_PER_STAGE - 1) / FRONT_WORDS_PER_STAGE;
	F.fold = d.anchor_fold; F.amask = d.anchor_mask; F.anchor[0] = d.anchor[0]; F.alen = d.anchor_len;
	F.delim4 = d.delim[0] * 0x01010101u;
	/* the scaled differences of exact_chunks (run-time values keep the multiplies on the FMA pipe) */
	F.scale = 1u << (8 * (4 - d.anchor_len)); F.coef[0] = d.anchor[0] * F.scale;
	F.coef3[0] = 2u; F.coef3[1] = (uint32_t)d.delim[0] << 24; F.coef3[2] = 1u << 24;
	const unsigned grid = (unsigned)std::min<uint64_t>(F.stage_end, (uint64_t)W.sm_count * FRONT_CTAS_PER_SM);
	const bool masked = d.anchor_mask != 0xFFFFFFFFu, fold = d.anchor_fold != 0;
	static bool configured[64][4] = {{false}};
	int dev = 0; cudaGetDevice(&dev);
#define EX_LAUNCH(M_, F_) do { if (!configured[dev & 63][(M_) * 2 + (F_)]) { cudaFuncSetAttribute(k_front_exact<M_, F_>, cudaFuncAttributeMaxDynamicSharedMemorySize, FRONT_SMEM); configured[dev & 63][(M_) * 2 + (F_)] = true; } \
	k_front_exact<M_, F_><<<grid, FRONT_THREADS, FRONT_SMEM, st>>>(F); } while (0)
	if (masked) { if (fold) EX_LAUNCH(true, true); else EX_LAUNCH(true, false); }
	else { if (fold) EX_LAUNCH(false, true); else EX_LAUNCH(false, false); }
#undef EX_LAUNCH
	g_launches++;
	CUDA_TRY(cudaGetLastError());
	/* ordered reduction: 4096 summaries per block, then one block over the block results (W.tile_offsets as scratch: 16 B each) */
	const uint64_t per_block = (uint64_t)EXR_THREADS * EXR_PER, nb = (n_words + per_block - 1) / per_block;
	if ((nb + nb / per_block + 16) * sizeof(ExSum) > W.tiles * sizeof(uint64_t)) { snprintf(g_err, sizeof g_err, "internal: scratch too small for the exact count"); return AGB_ERR_NOMEM; }
	ExSum *part = reinterpret_cast<ExSum *>(W.tile_offsets);
	if (nb == 1) { k_exact_reduce<<<1, EXR_THREADS, 0, st>>>(W.bitmap, n_words, nullptr, nullptr, W.totals); g_launches++; }
	else {
		k_exact_reduce<<<(unsigned)nb, EXR_THREADS, 0, st>>>(W.bitmap, n_words, nullptr, part, nullptr); g_launches++;
		uint64_t m = nb; ExSum *in = part, *outp = part + nb;
		while (m > 1) {
			const uint64_t mb = (m + per_block - 1) / per_block;
			k_exact_reduce<<<(unsigned)mb, EXR_THREADS, 0, st>>>(nullptr, m, in, mb == 1 ? nullptr : outp, mb == 1 ? W.totals : nullptr); g_launches++;
			in = outp; outp += mb; m = mb;
		}
	}
	CUDA_TRY(cudaGetLastError());
	return AGB_OK;
}

/* coefficients of prod_i (x - a_i) mod 2^32 and the false-positive guard of the polynomial form:
 * a zero product without a zero factor needs sum_i v2(w - a_i) >= bits; with t = the largest v2(a_i - a_j)
 * at most one factor can exceed t, so w must agree with an anchor in its low bits - (na-1)*t bits.  We ask
 * for at least 20 agreeing bits (a 2.5-byte accidental match) or use the compare form instead. */
bool poly_setup(const uint32_t *a, int na, int bits, uint32_t *coef)
{
	uint32_t c[AGB_MAXANCHOR + 1]; int deg = 0, t = 0;
	memset(c, 0, sizeof c); c[0] = 1;
	for (int i = 0; i < na; i++) {
		uint32_t m = 0u - a[i];
		for (int j = deg + 1; j >= 1; j--) c[j] = c[j - 1] + c[j] * m;
		c[0] = c[0] * m; deg++;
		for (int j = 0; j < i; j++) { uint32_t dd = a[i] - a[j]; int v = dd ? __builtin_ctz(dd) : 32; if (v > t) t = v; }
	}
	for (int i = 0; i < na; i++) coef[i] = c[i];
	return bits - (na - 1) * t >= 20;
}

bool front_usable(const agb_desc &d)
{
	if (d.plan != AGB_PLAN_ANCHORS || d.n_anchors < 1 || d.n_anchors > 9) return false;
	return d.n_anchors3 == 0 || (d.n_anchors3 <= 2 && d.anchor_len == 4 && d.n_anchors <= 7);
}

/* stage 1 over bitmap words [word_begin, word_end) of a text of n bytes; word_begin must be a multiple of 32
 * (a stage is 32 words).  slack16: 16 more bytes after the last chunk are readable (true for our own buffers). */
int front_launch(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n,
                        uint64_t word_begin, uint64_t word_end, bool slack16, cudaStream_t st, bool count_delims)
{
	const uint64_t n_chunks = (n + 15) / 16, n_words = (n_chunks + 31) / 32;
	if (word_end > n_words) word_end = n_words;
	if (word_begin >= word_end) return AGB_OK;
	FrontParams F; memset(&F, 0, sizeof F);
	F.text = (const uint8_t *)d_text; F.bitmap = W.bitmap; F.n = n; F.n_chunks = n_chunks;
	F.readable = n_chunks * 16 + (slack16 ? 16 : 0);
	F.stage_begin = word_begin / FRONT_WORDS_PER_STAGE;
	F.stage_end = (word_end + FRONT_WORDS_PER_STAGE - 1) / FRONT_WORDS_PER_STAGE;
	F.fold = d.anchor_fold; F.amask = d.anchor_mask;
	F.nl_blocks = count_delims ? W.ord_blocks : nullptr; F.dfold4 = d.delim_fold[0] * 0x01010101u; F.delim4 = (d.delim[0] | d.delim_fold[0]) * 0x01010101u;
	const uint64_t stages = F.stage_end - F.stage_begin;
	unsigned grid = (unsigned)std::min<uint64_t>(stages, (uint64_t)W.sm_count * FRONT_CTAS_PER_SM);
	if (!grid) grid = 1;
	bool masked = d.anchor_mask != 0xFFFFFFFFu, fold = d.anchor_fold != 0;
	/* identical anchors (e.g. from "abababab") are tested once */
	int na = 0;
	for (int i = 0; i < d.n_anchors; i++) {
		bool dup = false;
		for (int j = 0; j < na; j++) if (F.anchor[j] == d.anchor[i]) dup = true;
		if (!dup) F.anchor[na++] = d.anchor[i];
	}
	F.one = 1; F.scale = 1; F.s256 = 256;
	for (int i = d.anchor_len; i < 4; i++) F.scale <<= 8;
	if (d.pair_plan) {
		/* the planner made the pieces distinct and at most four (k <= 2) */
		if (na != d.n_anchors || na < 2 || na > 4 || d.anchor_len < 3) { snprintf(g_err, sizeof g_err, "internal: pair plan with %d pieces", d.n_anchors); return AGB_ERR_ARG; }
		for (int i = 0; i < na; i++) F.coef[i] = 0u - F.anchor[i] * F.scale;
		switch (na) {
		case 2: launch_front_pairs<2>(F, fold, grid, st); break;
		case 3: launch_front_pairs<3>(F, fold, grid, st); break;
		default: launch_front_pairs<4>(F, fold, grid, st); break;
		}
		g_launches++;
		CUDA_TRY(cudaGetLastError());
		return AGB_OK;
	}
	bool poly = poly_setup(F.anchor, na, 8 * d.anchor_len, F.coef);
	if (d.n_anchors3 > 0) {
		/* mixed plan: the second polynomial over the three-byte anchors; if either guard fails the three-byte anchors join
		 * the compare form as four-byte... no such form: fall back to flagging on the four-byte group alone is NOT allowed
		 * (it would lose matches), so the compare form below gets the 3-byte anchors through their own mask */
		int n3 = 0; uint32_t a3[4];
		for (int i = 0; i < d.n_anchors3; i++) {
			bool dup = false;
			for (int j = 0; j < n3; j++) if (a3[j] == d.anchor3[i]) dup = true;
			if (!dup) a3[n3++] = d.anchor3[i];
		}
		uint32_t c3[AGB_MAXANCHOR];
		const bool poly3 = poly_setup(a3, n3, 24, c3);
		if (!(poly && poly3)) { snprintf(g_err, sizeof g_err, "internal: mixed anchor plan without a polynomial form"); return AGB_ERR_ARG; }
		F.n3 = n3;
		for (int i = 0; i < n3; i++) F.coef3[i] = c3[i];
		if (n3 == 1) F.coef3[0] = 0u - 256u * a3[0];
		switch (na) {
		case 1: launch_front_mixed<1>(F, fold, grid, st); break;  case 2: launch_front_mixed<2>(F, fold, grid, st); break;
		case 3: launch_front_mixed<3>(F, fold, grid, st); break;  case 4: launch_front_mixed<4>(F, fold, grid, st); break;
		case 5: launch_front_mixed<5>(F, fold, grid, st); break;  case 6: launch_front_mixed<6>(F, fold, grid, st); break;
		case 7: launch_front_mixed<7>(F, fold, grid, st); break;
		default: return AGB_ERR_ARG;
		}
		g_launches++;
		CUDA_TRY(cudaGetLastError());
		return AGB_OK;
	}
	if (!poly && d.anchor_len == 3 && na >= 2 && na <= 5) {
		/* split: anchors into group A while its guard holds, the rest (at most two) into group B */
		uint32_t ga[AGB_MAXANCHOR], gb[4], ca[AGB_MAXANCHOR], cb[AGB_MAXANCHOR]; int nga = 0, ngb = 0; bool ok = true;
		for (int i = 0; i < na && ok; i++) {
			ga[nga] = F.anchor[i];
			if (poly_setup(ga, nga + 1, 24, ca)) { nga++; continue; }
			if (ngb >= 2) { ok = false; break; }
			gb[ngb] = F.anchor[i];
			if (!poly_setup(gb, ngb + 1, 24, cb)) ok = false; else ngb++;
		}
		if (ok && ngb >= 1 && nga >= 1) {
			poly_setup(ga, nga, 24, ca); poly_setup(gb, ngb, 24, cb);
			for (int i = 0; i < nga; i++) F.coef[i] = ca[i];
			F.n3 = ngb;
			for (int i = 0; i < ngb; i++) F.coef3[i] = cb[i];
			if (ngb == 1) F.coef3[0] = 0u - 256u * gb[0];
			switch (nga) {
			case 1: launch_front_split3<1>(F, fold, grid, st); break;  case 2: launch_front_split3<2>(F, fold, grid, st); break;
			case 3: launch_front_split3<3>(F, fold, grid, st); break;  default: launch_front_split3<4>(F, fold, grid, st); break;
			}
			g_launches++;
			CUDA_TRY(cudaGetLastError());
			return AGB_OK;
		}
	}
#define FRONT_CASE(N) case N: if (poly) launch_front_na<N, true>(F, masked, fold, grid, st); else launch_front_na<N, false>(F, masked, fold, grid, st); break;
	switch (na) {
	FRONT_CASE(1) FRONT_CASE(2) FRONT_CASE(3) FRONT_CASE(4) FRONT_CASE(5) FRONT_CASE(6) FRONT_CASE(7) FRONT_CASE(8) FRONT_CASE(9)
	default: return AGB_ERR_ARG;
	}
#undef FRONT_CASE
	g_launches++;
	CUDA_TRY(cudaGetLastError());
	return AGB_OK;
}

