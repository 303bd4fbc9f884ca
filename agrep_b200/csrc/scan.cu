/* agrep_b200/csrc/scan.cu -- the host side of libagrepb200's scan path and its C ABI (include/agrep_b200.h).
 *
 * What the reference does in bitap()/asearch()/asearch0()/asearch1()/sgrep()+bm() (one byte at a time, one file
 * block at a time, bitap.c:169-284, asearch.c:94-306, :620-774, asearch1.c:86-235, sgrep.c:694-1016) is done in
 * device stages over text that is resident in HBM (DESIGN.md 3):
 *
 *   stage 1    k_front (front.cu)    which 16-byte chunks can matter: one of the pattern's k+1 disjoint literal
 *              anchors starts there (pigeonhole, pattern.c:plan_anchors); one bit per chunk.  HBM-bound.
 *   stage 1.5  k_refine (refine.cu)  the same recurrence over just the window around an anchor hit; chunks whose
 *              hits cannot belong to a match lose their bit.
 *   stage 2    records (records.cu, slices.cu, regex.cu)  exact: the recurrence from the record start in the constant
 *              post-delimiter state until the closing delimiter, the reference's match test and bookkeeping,
 *              ordered (lasti, print_end) lists by count pass -> scan -> emit pass.  The list form for the flagged
 *              chunks while they are sparse; the slices or dense tile form when every byte has to be walked; k_regex
 *              for regular expressions.
 *   ordinals   (aux.cu)  the j that -n prints, from delimiter counts.
 *
 * This file: the per-device workspace, which form runs when (records_launch), the streaming host entry points
 * (the fill_buf replacement) and the exported functions.  There is no CPU path anywhere in the library.
 */
#include "scan_internal.cuh"
#include "corpus.h"
#include <unistd.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

/* ------------------------------------------------------------------------------------------------ */
thread_local char g_err[512];
std::atomic<uint64_t> g_launches{0};

extern "C" const char *agb_last_error(void) { return g_err; }
extern "C" const char *agb_version(void) { return "agrep-b200 0.1 (sm_90a)"; }
extern "C" uint64_t agb_kernel_launches(void) { return g_launches.load(); }
static void host_release(int dev);
/* frees the per-device scratch of this process (bitmaps, candidate lists, pinned rings, streams, events); the next
 * scan allocates again */
extern "C" void agb_shutdown(void)
{
	int cur = 0; cudaGetDevice(&cur);
	for (int dev = 0; dev < 64; dev++) {
		host_release(dev);
		std::lock_guard<std::mutex> lk(g_ws_mu[dev]);
		Workspace &W = g_ws[dev];
		if (!W.totals && !W.bitmap) continue;
		if (cudaSetDevice(dev) != cudaSuccess) { cudaGetLastError(); continue; }
		cudaDeviceSynchronize();
		cudaFree(W.bitmap); cudaFree(W.bitmap2); cudaFree(W.range_counts); cudaFree(W.range_offsets);
		cudaFree(W.tile_counts); cudaFree(W.tile_offsets); cudaFree(W.cand); cudaFree(W.cand_counts); cudaFree(W.cand_offsets);
		cudaFree(W.cand_first); cudaFree(W.scan_sums); cudaFree(W.scan_offs); cudaFree(W.ord_blocks); cudaFree(W.totals);
		cudaFreeHost(W.h_totals); cudaFree(W.d_desc); cudaFree(W.d_gram); cudaFreeHost(W.h_gram);
		cudaFree(W.d_regex); cudaFree(W.ds_func); cudaFree(W.ds_entry); cudaFree(W.dstate);
		if (W.e0) cudaEventDestroy(W.e0); if (W.e1) cudaEventDestroy(W.e1); if (W.e2) cudaEventDestroy(W.e2);
		W = Workspace();
	}
	cudaSetDevice(cur);
}
extern "C" int agb_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) return 0; return n; }
extern "C" int agb_set_device(int dev) { CUDA_TRY(cudaSetDevice(dev)); return AGB_OK; }

/* ================================================================================================
 * host side of the scan
 * ============================================================================================== */

Workspace g_ws[64];
std::mutex g_ws_mu[64];          /* one scan at a time per DEVICE (its workspace is shared scratch); different devices run side by side */

static int ws_prepare(Workspace &W, uint64_t n)
{
	if (!W.totals) {
		CUDA_TRY(cudaMalloc(&W.totals, 24 * sizeof(unsigned long long)));
		CUDA_TRY(cudaMallocHost(&W.h_totals, 24 * sizeof(unsigned long long)));
		CUDA_TRY(cudaMalloc(&W.d_desc, sizeof(agb_desc)));
		CUDA_TRY(cudaMalloc(&W.range_counts, REFINE_MAX_RANGES * sizeof(uint32_t)));
		CUDA_TRY(cudaMalloc(&W.range_offsets, REFINE_MAX_RANGES * sizeof(uint64_t)));
		CUDA_TRY(cudaEventCreate(&W.e0)); CUDA_TRY(cudaEventCreate(&W.e1)); CUDA_TRY(cudaEventCreate(&W.e2));
		int dev = 0; CUDA_TRY(cudaGetDevice(&dev));
		CUDA_TRY(cudaDeviceGetAttribute(&W.sm_count, cudaDevAttrMultiProcessorCount, dev));
	}
	uint64_t n_chunks = (n + 15) / 16, n_words = (n_chunks + 31) / 32, tiles = (n + std::min<uint64_t>(DENSE_TILE, SL_TILE) - 1) / std::min<uint64_t>(DENSE_TILE, SL_TILE) + 1;
	size_t bb = (size_t)(n_words + FRONT_WORDS_PER_STAGE) * 4;
	if (bb > W.bitmap_bytes) {
		if (W.bitmap) cudaFree(W.bitmap);
		if (W.bitmap2) cudaFree(W.bitmap2);
		W.bitmap = nullptr; W.bitmap2 = nullptr; W.bitmap_bytes = 0;
		CUDA_TRY(cudaMalloc(&W.bitmap, bb));
		CUDA_TRY(cudaMalloc(&W.bitmap2, bb)); W.bitmap_bytes = bb;
	}
	if (tiles + 1 > W.tiles) {
		if (W.tile_counts) cudaFree(W.tile_counts);
		if (W.tile_offsets) cudaFree(W.tile_offsets);
		W.tile_counts = nullptr; W.tile_offsets = nullptr; W.tiles = 0;
		CUDA_TRY(cudaMalloc(&W.tile_counts, (tiles + 1) * sizeof(uint32_t)));
		CUDA_TRY(cudaMalloc(&W.tile_offsets, (tiles + 1) * sizeof(uint64_t)));
		W.tiles = tiles + 1;
	}
	return AGB_OK;
}

/* the candidate list of the list form is sized by what stage 1.5 actually left (known on the host by then) */
static int ws_cand_reserve(Workspace &W, size_t want_cand)
{
	want_cand = std::max<size_t>(want_cand, (size_t)1 << 20);
	if (want_cand > W.cand_cap) {
		want_cand += want_cand / 4;
		if (W.cand) cudaFree(W.cand);
		if (W.cand_counts) cudaFree(W.cand_counts);
		if (W.cand_offsets) cudaFree(W.cand_offsets);
		if (W.cand_first) cudaFree(W.cand_first);
		if (W.scan_sums) cudaFree(W.scan_sums);
		if (W.scan_offs) cudaFree(W.scan_offs);
		W.cand = nullptr; W.cand_counts = nullptr; W.cand_offsets = nullptr; W.cand_first = nullptr; W.cand_cap = 0;
		W.scan_sums = nullptr; W.scan_offs = nullptr; W.scan_cap = 0;
		CUDA_TRY(cudaMalloc(&W.cand_first, want_cand * sizeof(agb_record)));
		W.scan_cap = want_cand / SCAN_BLOCK + 2;
		CUDA_TRY(cudaMalloc(&W.scan_sums, W.scan_cap * sizeof(uint32_t)));
		CUDA_TRY(cudaMalloc(&W.scan_offs, W.scan_cap * sizeof(uint64_t)));
		CUDA_TRY(cudaMalloc(&W.cand, want_cand * sizeof(uint64_t)));
		CUDA_TRY(cudaMalloc(&W.cand_counts, want_cand * sizeof(uint32_t)));
		CUDA_TRY(cudaMalloc(&W.cand_offsets, want_cand * sizeof(uint64_t)));
		W.cand_cap = want_cand;
	}
	return AGB_OK;
}

static int ws_upload_desc(Workspace &W, const agb_desc &d, cudaStream_t st)
{
	if (!W.desc_valid || memcmp(&W.h_desc_copy, &d, sizeof d) != 0) {
		CUDA_TRY(cudaMemcpyAsync(W.d_desc, &d, sizeof d, cudaMemcpyHostToDevice, st));
		CUDA_TRY(cudaStreamSynchronize(st));     /* &d may be on the caller's stack */
		W.h_desc_copy = d; W.desc_valid = true;
	}
	return AGB_OK;
}

/* what the descriptor cannot hold, to the device, where the record stage reads it from RecParams.rx_tab: the Next tables
 * of AGB_ENGINE_REGEX (regex.cu), or the words of 320-bit rows (agb_desc.wide, records_wide.cu).  px: the pattern that
 * holds them (NULL: a descriptor that needs neither) */
static_assert(sizeof(agb_wide) <= sizeof(Workspace::h_regex), "the wide words travel in the regex table buffer");
static int tables_prepare(Workspace &W, const agb_desc &d, const agb_pattern *px, cudaStream_t st)
{
	if (d.engine != AGB_ENGINE_REGEX && !d.wide) return AGB_OK;
	const agb_regex *rx = agb_pattern_regex(px);
	const agb_wide *wide = agb_pattern_wide(px);
	if (d.wide ? !wide : !rx) {
		snprintf(g_err, sizeof g_err, d.wide ? "a literal of 320-bit rows needs its words (agb_compile)" : "a regular expression needs its follow sets (agb_pattern_from_regex)");
		return AGB_ERR_ARG;
	}
	if (!W.d_regex) CUDA_TRY(cudaMalloc(&W.d_regex, sizeof W.h_regex));
	uint64_t tab[8 * 256];
	size_t bytes;
	if (d.wide) { memcpy(tab, wide, sizeof *wide); bytes = sizeof *wide; }
	else bytes = regex_tables(d, *rx, tab);
	if (bytes != W.regex_bytes || memcmp(tab, W.h_regex, bytes) != 0) {
		CUDA_TRY(cudaMemcpyAsync(W.d_regex, tab, bytes, cudaMemcpyHostToDevice, st));
		CUDA_TRY(cudaStreamSynchronize(st));     /* tab is on this stack */
		memcpy(W.h_regex, tab, bytes); W.regex_bytes = bytes;
	}
	if (rx) W.regex_tail = rx->tail;
	return AGB_OK;
}

/* the ordered candidate list -> records: count launch (per-candidate counts, the first record of each kept), scan,
 * emit launch.  The list length lives on the device (totals[12]); every grid here is sized by the list's capacity. */
static int list_stage(const agb_desc &d, Workspace &W, RecParams &P, bool want_list, cudaStream_t st)
{
	P.cand = W.cand; P.cand_cap = W.cand_cap; P.tile_counts = W.cand_counts; P.tile_offsets = W.cand_offsets;
	P.cand_first = want_list ? W.cand_first : nullptr;
	const unsigned grid = (unsigned)std::min<uint64_t>((W.cand_cap + REC_THREADS - 1) / REC_THREADS, (uint64_t)W.sm_count * 16);
	if (launch_records_list(d, P, grid, st)) return AGB_ERR_ARG;
	CUDA_TRY(cudaGetLastError());
	if (want_list) {
		const unsigned nb = (unsigned)((W.cand_cap + SCAN_BLOCK - 1) / SCAN_BLOCK);
		k_scan_partial<<<nb, 1024, 0, st>>>(W.cand_counts, W.cand_cap, W.scan_sums, W.totals + 12);
		k_scan_tiles<<<1, 1024, 0, st>>>(W.scan_sums, W.scan_offs, nb, nullptr);
		k_scan_apply<<<nb, 1024, 0, st>>>(W.cand_counts, W.cand_cap, W.scan_offs, W.cand_offsets, W.totals + 12);
		g_launches += 3;
		P.emit = 1;
		if (launch_records_list(d, P, grid, st)) return AGB_ERR_ARG;
		CUDA_TRY(cudaGetLastError());
	}
	return AGB_OK;
}

/* a tile form (launch_slices, launch_dense, launch_regex and their SET forms) -> records: count launch (per-tile counts),
 * scan, emit launch, one block per tile */
typedef int (*TileLaunch)(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st);
static int tile_stage(TileLaunch launch, const agb_desc &d, RecParams &P, Workspace &W, unsigned grid, bool want_list, cudaStream_t st)
{
	P.tile_counts = W.tile_counts; P.tile_offsets = W.tile_offsets;
	if (launch(d, P, grid, st)) return AGB_ERR_ARG;
	CUDA_TRY(cudaGetLastError());
	if (want_list) {
		k_scan_tiles<<<1, 1024, 0, st>>>(W.tile_counts, W.tile_offsets, grid, nullptr); g_launches++;
		P.emit = 1;
		if (launch(d, P, grid, st)) return AGB_ERR_ARG;
		CUDA_TRY(cudaGetLastError());
	}
	return AGB_OK;
}

/* what feeds the record stage */
enum RecInput {
	REC_EVERY_BYTE,              /* no bitmap: every byte is walked */
	REC_FRONT,                   /* stage 1's bitmap (W.bitmap), for the patterns stage 1.5 cannot thin (refine_launch) */
	REC_SURVIVORS,               /* stage 1.5's survivors (W.bitmap2), their per-range counts in W.range_counts */
};

/* stage 2 over the whole text.  Regular expressions: k_regex over every byte.  Otherwise, by input:
 *   REC_SURVIVORS   compacted into the ordered candidate list, then the list form.  The list is sized without asking the
 *                   device how many survivors there are (W.cand_hint, or a fraction of the chunks); the caller,
 *                   stages_after_front, reads totals[12] back and, if it exceeds W.cand_cap, calls this again -- with the
 *                   list sized from that count, or with REC_EVERY_BYTE when the survivors are dense.
 *   REC_FRONT       the flagged chunks are counted and the count read back: the list form while list_form_pays, else
 *                   every byte.
 *   REC_EVERY_BYTE  the slices form, or the dense tile form for the patterns slices_usable turns away. */
static int records_launch(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n, RecInput in, int want,
                          int want_level, agb_record *d_records, uint64_t capacity, cudaStream_t st, const ShardInfo *sh)
{
	const uint64_t n_chunks = (n + 15) / 16;
	RecParams P; memset(&P, 0, sizeof P);
	P.text = (const uint8_t *)d_text; P.n = n; P.n_chunks = n_chunks; P.desc = W.d_desc;
	P.records = d_records; P.capacity = capacity;
	P.totals = W.totals; P.emit = 0; P.levels = (want & AGB_WANT_LEVELS) ? 1 : 0; P.want_level = want_level;
	P.own_lo = sh ? sh->own_lo : INT64_MIN; P.own_hi = sh ? sh->own_hi : INT64_MAX; P.shard_last = sh ? sh->last : 1;
	P.rx_tab = W.d_regex; P.rx_tail = W.regex_tail; P.dstate = W.dstate;
	if (!n) return AGB_OK;
	const bool want_list = (want & AGB_WANT_RECORDS) && capacity;
	/* (delim_kind 3 has no anchor plan: only the dense tile form reads the delimiter pass, the other forms find record
	 * starts by the delimiter's bytes) */
	if (d.delim_kind == 3 && (in != REC_EVERY_BYTE || slices_usable(d))) { snprintf(g_err, sizeof g_err, "internal: delim_kind 3 outside the dense tile form"); return AGB_ERR_ARG; }
	if (d.engine == AGB_ENGINE_REGEX)
		return tile_stage(launch_regex, d, P, W, (unsigned)((n + RX_TILE - 1) / RX_TILE), want_list, st);
	if (in == REC_SURVIVORS) {
		int rc = ws_cand_reserve(W, std::max<size_t>(W.cand_hint + W.cand_hint / 4, (size_t)(n_chunks / 512) + 65536)); if (rc) return rc;
		const unsigned ranges = W.refine_ctas * (REFINE_THREADS / 32);
		k_scan_tiles<<<1, 1024, 0, st>>>(W.range_counts, W.range_offsets, ranges, W.totals + 12); g_launches++;
		rc = compact_ranges_launch(W, n, st); if (rc) return rc;
		return list_stage(d, W, P, want_list, st);
	}
	if (in == REC_FRONT) {
		const uint64_t n_words = (n_chunks + 31) / 32, blocks = (n_words + COMPACT_THREADS * COMPACT_WPT - 1) / (COMPACT_THREADS * COMPACT_WPT);
		k_compact_count<<<(unsigned)blocks, COMPACT_THREADS, 0, st>>>(W.bitmap, n_words, W.tile_counts, W.totals); g_launches++;
		k_scan_tiles<<<1, 1024, 0, st>>>(W.tile_counts, W.tile_offsets, blocks, W.totals + 12); g_launches++;
		CUDA_TRY(cudaMemcpyAsync(W.h_totals + 12, W.totals + 12, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
		CUDA_TRY(cudaStreamSynchronize(st));
		const unsigned long long ncand = W.h_totals[12];
		if (list_form_pays(ncand, n_chunks)) {
			int rc = ws_cand_reserve(W, (size_t)ncand); if (rc) return rc;
			if (ncand == 0) return AGB_OK;
			k_compact_write<<<(unsigned)blocks, COMPACT_THREADS, 0, st>>>(W.bitmap, n_words, W.tile_offsets, W.cand, W.cand_cap); g_launches++;
			return list_stage(d, W, P, want_list, st);
		}
		CUDA_TRY(cudaMemsetAsync(W.totals + 1, 0, sizeof(unsigned long long), st));   /* the tile form counts totals[1] afresh */
	}
	const bool slices = slices_usable(d);
	P.warm = (d.M + d.nrows + 2 + 3) & ~3;
	return tile_stage(slices ? launch_slices : launch_dense, d, P, W,
	                  (unsigned)(slices ? (n + SL_TILE - 1) / SL_TILE : (n + DENSE_TILE - 1) / DENSE_TILE), want_list, st);
}

/* an exact pattern that is no longer than its anchor ('the'): every chunk stage 1 flags holds a real occurrence, so
 * stage 1.5 has nothing to remove -- if such flags are dense (front_is_dense), the record stage walks every byte
 * anyway and stages 1.5 and the compaction are skipped.  For every other pattern only stage 1.5 can tell (a k = 4
 * pattern of common words flags 8 % of the chunks and keeps none), so the decision waits for the list length. */
static bool refine_cannot_thin(const agb_desc &d) { return d.k == 0 && d.n_anchors == 1 && d.pat_len <= d.anchor_len; }

static int fetch_result(Workspace &W, int want, uint64_t capacity, bool refined, cudaStream_t st, agb_result *res)
{
	CUDA_TRY(cudaMemcpyAsync(W.h_totals, W.totals, 24 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));   /* [16..18]: shard_aux_enqueue */
	CUDA_TRY(cudaStreamSynchronize(st));
	res->n_matched = W.h_totals[0];
	res->n_flagged = refined ? W.h_totals[12] : W.h_totals[1];
	for (int i = 0; i <= AGB_MAXERR; i++) res->level_hist[i] = W.h_totals[2 + i];
	res->n_records = (want & AGB_WANT_RECORDS) ? std::min<uint64_t>(res->n_matched, capacity) : 0;
	res->truncated = ((want & AGB_WANT_RECORDS) && res->n_matched > capacity) ? 1 : 0;
	res->n_closes = (want & AGB_WANT_ORDINALS) ? W.h_totals[13] + (uint64_t)W.ord_virt : 0;
	return AGB_OK;
}

/* the block counters stage 1 fills when it counts delimiters: allocated, and zeroed behind the last bitmap word
 * (the tile sums read whole tiles; the block of the delimiter appended at EOF may lie there) */
static int ordinals_prepare_blocks(const agb_desc &d, Workspace &W, uint64_t n, cudaStream_t st)
{
	int rc = ordinals_reserve(d, W, n); if (rc) return rc;
	const uint64_t n_words = ((n + 15) / 16 + 31) / 32;
	if (W.ord_blocks_cap > n_words) CUDA_TRY(cudaMemsetAsync(W.ord_blocks + n_words, 0, (W.ord_blocks_cap - n_words) * sizeof(uint16_t), st));
	return AGB_OK;
}

/* ------------------------------------------------------------------------------------------------
 * the anchor planner.  Any k+1 disjoint literal grams of the pattern make a valid pigeonhole filter; which ones
 * decides how many chunks stage 1 flags -- 4.5 % of the benchmark text for beca|use |each, 2.4 % for beca|se e|ach --
 * and stage 1.5 pays per flagged chunk.  The static plan (pattern.c) takes the first k+1 runs; here, for texts large
 * enough to care, the candidate grams (every literal 4-gram and 3-gram of the pattern) are counted on a 4 MiB sample
 * of the text and the cheapest set is chosen by a small dynamic program: four-byte grams, plus up to two three-byte
 * grams (which cost stage 1 one more operation per window: they only pay when they save enough flags).  The same sample
 * also runs the pair plan's rule (k + 2 pieces, a chunk flagged only where two of them meet, DESIGN.md 3.1), which is
 * taken when it flags clearly fewer chunks than the k+1 plan -- 1.5 % instead of 4.5 % for because each.
 * Works from the Mask[] words alone, so the drop-in layer's descriptors are re-planned too.
 * ---------------------------------------------------------------------------------------------- */
#define PLAN_MIN_BYTES   (256ull << 20)
#define PLAN_SAMPLE_BLK  64               /* stretches */
#define PLAN_BLK_CHUNKS  4096             /* of 64 KiB */
#define PAIR_REACH       16               /* the pair rule sees a second piece up to the end of the next chunk */

/* The pair plan's pieces: k + 2 disjoint literal grams of one length, four bytes if the pattern has room, else three,
 * pairwise distinct.  k errors damage at most k of them, so two occur verbatim in a match, and the later of those two
 * starts at most (o_last - o_first) + k bytes after the earlier: with that within PAIR_REACH, the chunk where the
 * earlier one starts also sees the later one start in it or in the next chunk.  Taken from the left, the first set that
 * fits.  Returns the number of pieces (0: none). */
static int pair_pieces(const int *lit, int pat_len, int k, uint32_t fold, uint32_t *val, int *off, int *len_out)
{
	const int np = k + 2;
	if (k < 0 || np > 4) return 0;
	for (int len = 4; len >= 3; len--)
		for (int s0 = 0; s0 + np * len <= pat_len; s0++) {
			int got = 0;
			for (int p = s0; p + len <= pat_len && got < np; ) {
				bool ok = true; uint32_t v = 0;
				for (int t = 0; t < len; t++) { if (lit[p + t] < 0) ok = false; else v |= (uint32_t)(lit[p + t] | (fold & 0x20)) << (8 * t); }
				if (!ok) { p++; continue; }
				val[got] = v; off[got] = p; got++; p += len;
			}
			if (got < np || off[0] != s0 || off[np - 1] - off[0] + k > PAIR_REACH) continue;
			bool distinct = true;
			for (int a = 0; a < np; a++) for (int b = 0; b < a; b++) if (val[a] == val[b]) distinct = false;
			if (!distinct) continue;
			*len_out = len;
			return np;
		}
	return 0;
}

static int adaptive_plan(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n, bool count_delims, cudaStream_t st, agb_desc *out)
{
	*out = d;
	if (!d.adaptive || !front_usable(d) || !d.refine || d.n_anchors3 || n < PLAN_MIN_BYTES || d.pat_len < 4 || d.pat_len > 60) return AGB_OK;
	const int need = d.k + 1;
	if (need > 9) return AGB_OK;
	const char *pp = getenv("AGB_PLAN_PAIRS");          /* unset: the pair plan when the sample favours it; 0: never; 1: whenever it exists */
	const int pairs_env = (pp && *pp) ? atoi(pp) : -1;
	/* what a three-byte group costs, in units of flag rate (the dynamic program below): part of the key, so that a
	 * change of AGB_PLAN_MIXED between two scans of one text plans afresh */
	const char *mp = getenv("AGB_PLAN_MIXED");           /* (tests force mixed plans with AGB_PLAN_MIXED=0) */
	const double MIXED = mp ? atof(mp) : 0.03;
	uint64_t key = 1469598103934665603ull;
	{
		const unsigned char *b = (const unsigned char *)&d;
		for (size_t i = 0; i < sizeof d; i++) { key ^= b[i]; key *= 1099511628211ull; }
		key ^= (uint64_t)(uintptr_t)d_text; key *= 1099511628211ull; key ^= n; key *= 1099511628211ull;
		key ^= (uint64_t)(pairs_env + 2) * 2 + (count_delims ? 1 : 0); key *= 1099511628211ull;
		uint64_t mbits; memcpy(&mbits, &MIXED, sizeof mbits);
		key ^= mbits; key *= 1099511628211ull;
	}
	if (W.plan_valid && W.plan_key == key) {
		*out = W.plan_desc;
		if (getenv("AGB_DEBUG_PLAN") && out->pair_plan) {            /* a scan that reuses the plan says so too */
			fprintf(stderr, "agb plan: cached -> pair plan chosen:");
			for (int i = 0; i < out->n_anchors; i++) fprintf(stderr, " [%.*s]@%d", out->anchor_len, (const char *)&out->anchor[i], out->anchor_off[i]);
			fprintf(stderr, "\n");
		}
		return AGB_OK;
	}
	/* literal bytes of the pattern proper, from the masks */
	int lit[64]; bool pair_any = false;
	for (int j = 0; j < d.pat_len; j++) {
		const uint64_t bit = 1ull << (d.M - (d.L + 2 + j));
		int cnt = 0, c0 = -1, c1 = -1;
		for (int c = 0; c < 256; c++) if (d.mask[c] & bit) { if (cnt == 0) c0 = c; else if (cnt == 1) c1 = c; cnt++; }
		lit[j] = -1;
		if (cnt == 1 && c0 != '\n' && c0 < 0x80) lit[j] = c0;
		else if (cnt == 2 && (c0 ^ c1) == 0x20 && c1 < 0x80) { lit[j] = c0 | 0x20; pair_any = true; }
	}
	const uint32_t fold = pair_any ? 0x20202020u : 0u;
	/* candidate grams */
	struct Gram { int s, len; uint32_t v, m; double cost; };
	Gram g[128]; int ng = 0;
	for (int len = 4; len >= 3; len--)
		for (int s = 0; s + len <= d.pat_len && ng < 120; s++) {
			bool ok = true; uint32_t v = 0;
			for (int t = 0; t < len; t++) { if (lit[s + t] < 0) ok = false; else v |= (uint32_t)(lit[s + t] | (fold & 0x20)) << (8 * t); }
			if (!ok) continue;
			g[ng].s = s; g[ng].len = len; g[ng].v = v; g[ng].m = len == 4 ? 0xFFFFFFFFu : 0x00FFFFFFu; g[ng].cost = 0; ng++;
		}
	/* the pair plan's pieces are sampled along with the grams (behind them) */
	uint32_t pv[4]; int poff[4], plen = 0;
	const int n_pair = pairs_env != 0 ? pair_pieces(lit, d.pat_len, d.k, fold, pv, poff, &plen) : 0;
	if (ng < need && !n_pair) return AGB_OK;
	if (!W.d_gram) { CUDA_TRY(cudaMalloc(&W.d_gram, 3 * 128 * sizeof(uint32_t))); CUDA_TRY(cudaMallocHost(&W.h_gram, 3 * 128 * sizeof(uint32_t))); }
	for (int i = 0; i < 128; i++) {
		const bool gi = i < ng, pi = i >= ng && i < ng + n_pair;
		W.h_gram[i] = gi ? g[i].v : pi ? pv[i - ng] : 0;
		W.h_gram[128 + i] = gi ? g[i].m : pi ? (plen == 4 ? 0xFFFFFFFFu : 0x00FFFFFFu) : 0;
		W.h_gram[256 + i] = 0;
	}
	CUDA_TRY(cudaMemcpyAsync(W.d_gram, W.h_gram, 3 * 128 * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	const uint64_t n_chunks = (n + 15) / 16;
	const uint64_t threads = (uint64_t)PLAN_SAMPLE_BLK * PLAN_BLK_CHUNKS;
	k_gram_sample<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>((const uint8_t *)d_text, n_chunks, PLAN_SAMPLE_BLK, PLAN_BLK_CHUNKS,
	                                                                 ng + n_pair, W.d_gram, W.d_gram + 128, fold, W.d_gram + 256, ng, n_pair);
	g_launches++;
	CUDA_TRY(cudaGetLastError());
	CUDA_TRY(cudaMemcpyAsync(W.h_gram + 256, W.d_gram + 256, 128 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	CUDA_TRY(cudaStreamSynchronize(st));
	for (int i = 0; i < ng; i++) g[i].cost = (double)W.h_gram[256 + i] / (double)threads;
	const double pair_rate = (double)W.h_gram[256 + 127] / (double)threads;
	/* dynamic program over the pattern positions: f[p][j][t] = least total rate of j disjoint grams inside [0, p), t of them
	 * three bytes long */
	/* what a three-byte group costs, in units of flag rate: on the benchmark pattern (beca|se e|ach flags 2.4 % of the
	 * chunks instead of 4.5 %) stage 1 pays for a second polynomial and one VIMNMX3 per window instead of half of one,
	 * and stage 1.5 does not get cheaper in proportion -- a mixed plan only pays when the four-byte grams of a piece
	 * are really common (MIXED, above) */
	const double INF = 1e30;
	static double f[66][10][3]; static int from[66][10][3];   /* gram taken to get here, -1: position skipped */
	for (int p = 0; p <= d.pat_len; p++) for (int j = 0; j <= need; j++) for (int t = 0; t < 3; t++) { f[p][j][t] = INF; from[p][j][t] = -2; }
	f[0][0][0] = 0;
	for (int p = 0; p < d.pat_len; p++)
		for (int j = 0; j <= need; j++) for (int t = 0; t < 3; t++) {
			if (f[p][j][t] >= INF) continue;
			if (f[p][j][t] < f[p + 1][j][t]) { f[p + 1][j][t] = f[p][j][t]; from[p + 1][j][t] = -1; }
			if (j == need) continue;
			for (int i = 0; i < ng; i++) if (g[i].s == p) {
				const int t2 = t + (g[i].len == 3), p2 = p + g[i].len;
				if (t2 > 2) continue;
				if (f[p][j][t] + g[i].cost < f[p2][j + 1][t2]) { f[p2][j + 1][t2] = f[p][j][t] + g[i].cost; from[p2][j + 1][t2] = i; }
			}
		}
	int best_t = -1; double best = INF;
	for (int t = 0; t < 3; t++) {
		if (need - t < 1 || need - t > (t ? 7 : 9)) continue;
		const double c = f[d.pat_len][need][t] + (t ? MIXED : 0);
		if (c < best) { best = c; best_t = t; }
	}
	double cur = 0;                                     /* the static plan's rate, from the same sample where it can be read off */
	for (int a = 0; a < d.n_anchors; a++) { double r = 1.0; for (int i = 0; i < ng; i++) if (g[i].len == d.anchor_len && g[i].s == d.anchor_off[a]) r = g[i].cost; cur += r; }
	/* the k+1 plan: the static one unless the sample says a set of grams flags clearly fewer chunks */
	agb_desc plan = d;
	double rate = cur;
	if (best_t >= 0 && best < 0.85 * cur) {
		agb_desc nd = d;
		nd.n_anchors = 0; nd.n_anchors3 = 0; nd.anchor_len = 4; nd.anchor_mask = 0xFFFFFFFFu; nd.anchor_fold = fold;
		{
			int p = d.pat_len, j = need, t = best_t;
			while (p > 0 && j >= 0) {
				const int fr = from[p][j][t];
				if (fr == -1) { p--; continue; }
				if (fr < 0) break;
				if (g[fr].len == 4) { nd.anchor[nd.n_anchors] = g[fr].v; nd.anchor_off[nd.n_anchors] = g[fr].s; nd.n_anchors++; }
				else { nd.anchor3[nd.n_anchors3] = g[fr].v; nd.anchor3_off[nd.n_anchors3] = g[fr].s; nd.n_anchors3++; }
				p -= g[fr].len; j--; t -= (g[fr].len == 3);
			}
		}
		/* the kernels want their polynomials: both groups must pass the false-positive guard, and the anchors must be
		 * pairwise distinct (stage 1.5 tells them apart by their bytes) */
		bool ok = nd.n_anchors + nd.n_anchors3 == need && nd.n_anchors >= 1;
		uint32_t tmp[AGB_MAXANCHOR];
		if (ok) ok = poly_setup(nd.anchor, nd.n_anchors, 32, tmp);
		if (ok && nd.n_anchors3) ok = poly_setup(nd.anchor3, nd.n_anchors3, 24, tmp);
		for (int a = 0; a < nd.n_anchors && ok; a++) {
			for (int b = 0; b < a; b++) if (nd.anchor[a] == nd.anchor[b]) ok = false;
			for (int b = 0; b < nd.n_anchors3; b++) if ((nd.anchor[a] & 0x00FFFFFFu) == nd.anchor3[b]) ok = false;
		}
		for (int a = 0; a < nd.n_anchors3 && ok; a++) for (int b = 0; b < a; b++) if (nd.anchor3[a] == nd.anchor3[b]) ok = false;
		if (ok) { plan = nd; rate = best; }
		if (getenv("AGB_DEBUG_PLAN")) {
			fprintf(stderr, "agb plan: static rate %.4f -> %s rate %.4f:", cur, ok ? "chosen" : "rejected", best);
			for (int a = 0; a < nd.n_anchors; a++) fprintf(stderr, " [%.4s]@%d", (const char *)&nd.anchor[a], nd.anchor_off[a]);
			for (int a = 0; a < nd.n_anchors3; a++) fprintf(stderr, " [%.3s]@%d", (const char *)&nd.anchor3[a], nd.anchor3_off[a]);
			fprintf(stderr, "\n");
		}
	}
	/* the pair plan, by the same margin against the k+1 plan's rate (a sum over its grams: an upper bound).  Not when
	 * stage 1 also counts the delimiters (-n): its 24 more ALU operations per chunk on top of the pair test make stage 1
	 * cost about what stage 1.5 saves (on H100 the -n headline took 17.75 ms against 17.70 ms) */
	if (n_pair) {
		const bool take = pairs_env == 1 || (!count_delims && pair_rate < 0.85 * rate);
		if (take) {
			agb_desc pd = d;
			pd.pair_plan = 1; pd.n_anchors = n_pair; pd.n_anchors3 = 0; pd.anchor_len = plen;
			pd.anchor_mask = plen == 4 ? 0xFFFFFFFFu : 0x00FFFFFFu; pd.anchor_fold = fold;
			for (int i = 0; i < n_pair; i++) { pd.anchor[i] = pv[i]; pd.anchor_off[i] = poff[i]; }
			plan = pd;
		}
		if (getenv("AGB_DEBUG_PLAN")) {
			fprintf(stderr, "agb plan: k+1 rate %.4f, pair rate %.4f -> pair plan %s:", rate, pair_rate, take ? "chosen" : "not chosen");
			for (int i = 0; i < n_pair; i++) fprintf(stderr, " [%.*s]@%d", plen, (const char *)&pv[i], poff[i]);
			fprintf(stderr, "\n");
		}
	}
	W.plan_key = key; W.plan_valid = true; W.plan_desc = plan;
	*out = plan;
	return AGB_OK;
}

/* everything after stage 1, on one stream: stage 1.5, the record stage, the ordinals, the result read-back (the one
 * host synchronisation of a scan).  The candidate list of the list form is sized without asking the device how many
 * survivors there are; should it turn out too small (totals[12] > capacity, seen in the read-back) the record stage
 * and the ordinals are run again, the list with the right size -- or in its every-byte form when the survivors are
 * dense.  Stage 1's outputs (the bitmap, the delimiter counts per block) are reused as they are, so no pass after
 * stage 1 may change them. */
/* shard.cu: the delimiter counts of the halos and the run check of the left halo, into totals[16..18] (read back with the rest) */
int shard_aux_enqueue(const agb_desc &d, Workspace &W, const uint8_t *text, uint64_t n, const ShardInfo *sh, bool ordinals, cudaStream_t st);

static int stages_after_front(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n, bool use_front, bool count_in_front,
                              int want, int want_level, agb_record *d_records, uint64_t capacity, cudaStream_t st, agb_result *res,
                              const ShardInfo *sh = nullptr)
{
	int rc;
	const uint64_t n_chunks = (n + 15) / 16;
	if (d.delim_kind == 3) { rc = dstate_launch(d, W, d_text, n, sh ? sh->dseed : -1, st); if (rc) return rc; }
	RecInput in = use_front ? REC_FRONT : REC_EVERY_BYTE;
	if (in == REC_FRONT && refine_cannot_thin(d)) { bool dense = false; rc = front_is_dense(W, n, st, &dense); if (rc) return rc; if (dense) in = REC_EVERY_BYTE; }
	if (in == REC_FRONT) { bool refined = false; rc = refine_launch(d, W, d_text, n, st, &refined); if (rc) return rc; if (refined) in = REC_SURVIVORS; }
	for (int attempt = 0; ; attempt++) {
		rc = records_launch(d, W, d_text, n, in, want, want_level, d_records, capacity, st, sh); if (rc) return rc;
		if (want & AGB_WANT_ORDINALS) { rc = ordinals_launch(d, W, d_text, n, (want & AGB_WANT_RECORDS) ? d_records : nullptr, capacity, st, count_in_front); if (rc) return rc; }
		CUDA_TRY(cudaEventRecord(W.e2, st));
		if (sh) { rc = shard_aux_enqueue(d, W, (const uint8_t *)d_text, n, sh, (want & AGB_WANT_ORDINALS) != 0, st); if (rc) return rc; }
		rc = fetch_result(W, want, capacity, in == REC_SURVIVORS, st, res); if (rc) return rc;
		if (in != REC_SURVIVORS) break;
		const uint64_t ncand = W.h_totals[12];
		W.cand_hint = (size_t)ncand;
		if (ncand <= W.cand_cap || attempt) break;
		/* the list was too small: again, with the size known now (sparse) or over every byte (dense) */
		if (!list_form_pays(ncand, n_chunks)) in = REC_EVERY_BYTE;
		CUDA_TRY(cudaMemsetAsync(W.totals, 0, 12 * sizeof(unsigned long long), st));
	}
	return AGB_OK;
}

/* -v, count only: can the answer be had as (records) - (matching records)?  Newline records, one part, no wildcards, an
 * anchor plan that stage 1.5 can verify (pattern.c keeps the anchors of a -v pattern in the descriptor) */
static bool complement_usable(const agb_desc &d)
{
	if (!d.inverse || d.plan != AGB_PLAN_ALL || d.n_anchors < 1 || d.n_anchors > 9 || d.n_anchors3 || !d.refine) return false;
	if (d.L != 1 || d.delim[0] != '\n' || d.user_delim || d.delim_fold[0] || d.and_mode || d.wildmask || d.init1 == ~0ull) return false;
	return true;
}

int scan_device_impl(const agb_desc &d_in, const void *d_text, uint64_t n, int want, int want_level,
                     agb_record *d_records, uint64_t capacity, cudaStream_t st, agb_result *res, const ShardInfo *sh,
                     const agb_pattern *px)
{
	if (!res) return AGB_ERR_ARG;
	memset(res, 0, sizeof *res);
	if (((uintptr_t)d_text & 15) != 0) { snprintf(g_err, sizeof g_err, "text pointer must be 16-byte aligned"); return AGB_ERR_ARG; }
	if ((want & AGB_WANT_RECORDS) && capacity && !d_records) return AGB_ERR_ARG;
	int dev = 0; CUDA_TRY(cudaGetDevice(&dev));
	if (dev < 0 || dev >= 64) return AGB_ERR_ARG;
	if (want == AGB_WANT_COUNT && !sh && n >= (1u << 20) && complement_usable(d_in)) {
		/* `agrep -c -v pattern`, newline records: every record either matches or does not (the same test at the same close,
		 * bitap.c:182 with INVERSE flipped), so the count of the non-matching ones is the number of records minus the count of
		 * the matching ones -- and those the anchors find.  Records: one per newline of the text, one more for an unterminated
		 * last line (the delimiter appended at EOF closes it; after a final newline it would close the phantom record that
		 * agrep.c:3811 drops).  The newlines are counted by the same pass (j at EOF = newlines + appended + virtual). */
		agb_desc pos = d_in; pos.inverse = 0; pos.plan = AGB_PLAN_ANCHORS;
		agb_result r;
		int rc = scan_device_impl(pos, d_text, n, AGB_WANT_COUNT | AGB_WANT_ORDINALS, -1, nullptr, 0, st, &r, nullptr, px); if (rc) return rc;
		unsigned char last = 0;
		CUDA_TRY(cudaMemcpyAsync(&last, (const uint8_t *)d_text + n - 1, 1, cudaMemcpyDeviceToHost, st));
		CUDA_TRY(cudaStreamSynchronize(st));
		const uint64_t records = r.n_closes - 2 + (last != '\n' ? 1 : 0);
		if (r.n_closes < 2 || r.n_matched > records) { snprintf(g_err, sizeof g_err, "internal: complement count out of range"); return AGB_ERR_CUDA; }
		*res = r;
		res->n_matched = records - r.n_matched; res->n_closes = 0; res->n_records = 0;
		return AGB_OK;
	}
	std::lock_guard<std::mutex> lk(g_ws_mu[dev]);
	Workspace &W = g_ws[dev];
	int rc = ws_prepare(W, n); if (rc) return rc;
	agb_desc planned;
	rc = adaptive_plan(d_in, W, d_text, n, (want & AGB_WANT_ORDINALS) && d_in.L == 1, st, &planned); if (rc) return rc;
	const agb_desc &d = planned;
	if (want == AGB_WANT_COUNT && !sh && n >= (1u << 20) && exact_count_usable(d)) {
		/* `agrep -c the`: an exact literal no longer than its anchor needs no automaton (front.cu, exact_count_launch) */
		CUDA_TRY(cudaMemsetAsync(W.totals, 0, 16 * sizeof(unsigned long long), st));
		CUDA_TRY(cudaEventRecord(W.e0, st));
		rc = exact_count_launch(d, W, d_text, n, st); if (rc) return rc;
		CUDA_TRY(cudaEventRecord(W.e1, st));
		CUDA_TRY(cudaEventRecord(W.e2, st));
		rc = fetch_result(W, want, capacity, false, st, res); if (rc) return rc;
		res->n_flagged = 0;
		CUDA_TRY(cudaEventElapsedTime(&res->ms_front, W.e0, W.e1));
		res->ms_records = 0;
		return AGB_OK;
	}
	rc = ws_upload_desc(W, d, st); if (rc) return rc;
	rc = tables_prepare(W, d, px, st); if (rc) return rc;
	CUDA_TRY(cudaMemsetAsync(W.totals, 0, 16 * sizeof(unsigned long long), st));
	CUDA_TRY(cudaEventRecord(W.e0, st));
	bool use_front = front_usable(d) && n > 0;
	/* -n with a 1-byte delimiter: stage 1 reads every byte anyway and counts the delimiters of each 512-byte block */
	const bool count_in_front = use_front && (want & AGB_WANT_ORDINALS) && d.L == 1;
	if (count_in_front) { rc = ordinals_prepare_blocks(d, W, n, st); if (rc) return rc; }
	if (use_front) { rc = front_launch(d, W, d_text, n, 0, ~0ull, false, st, count_in_front); if (rc) return rc; }
	CUDA_TRY(cudaEventRecord(W.e1, st));
	rc = stages_after_front(d, W, d_text, n, use_front, count_in_front, want, want_level, d_records, capacity, st, res, sh); if (rc) return rc;
	/* (sh: a record that ran past the right halo raised totals[11]; shard_scan_geom reads it) */
	CUDA_TRY(cudaEventElapsedTime(&res->ms_front, W.e0, W.e1));
	CUDA_TRY(cudaEventElapsedTime(&res->ms_records, W.e1, W.e2));
	return AGB_OK;
}

extern "C" int agb_scan_device(const agb_pattern *p, const void *d_text, uint64_t n, int want,
                               agb_record *d_records, uint64_t capacity, void *stream, agb_result *res)
{
	if (!p) return AGB_ERR_ARG;
	return scan_device_impl(p->d, d_text, n, want, -1, d_records, capacity, (cudaStream_t)stream, res, nullptr, p);
}

/* Host text -> HBM -> scan: the replacement of the fill_buf()/read(2) loop (bitap.c:143,450-477).  The text is moved in
 * 64 MiB slices on a copy stream -- straight from the caller's memory when it is page-locked; through a pinned ring filled
 * by 4 host threads when it is pageable; pread(2) by 4 threads into the ring from a regular file -- while stage 1 runs on
 * the slice that arrived before (its last chunk looks 4 bytes into the next one), so the scan hides behind PCIe; stages 1.5
 * and 2 run once over the whole bitmap.  The whole-text, windowed and resident-text uploads share this one loop (upload),
 * one pinned ring and one pair of streams per device (HostPath). */
/* AGB_ODIRECT=1: read regular files past the page cache (a second descriptor on the same file, through /proc/self/fd);
 * -1 when not asked for, when the text does not start on a block boundary, or when the file system refuses */
static int open_direct(int fd, off_t fd_off)
{
	const char *e = getenv("AGB_ODIRECT");
	if (!e || !*e || *e == '0' || (fd_off & 4095)) return -1;
	char path[64]; snprintf(path, sizeof path, "/proc/self/fd/%d", fd);
	return open(path, O_RDONLY | O_DIRECT);
}

/* the n bytes of text a host path moves: host memory, or a regular file from fd_off on (fd_source) */
struct SliceSource {
	const uint8_t *mem = nullptr;  /* host memory source, or NULL */
	bool pinned = false;           /* mem is page-locked: copy from it directly */
	int fd = -1;                   /* file descriptor source when mem == NULL (a regular file) */
	off_t fd_off = 0;              /* where the text starts in it (-1: lseek failed, and n is 0) */
	int dfd = -1;                  /* the same file opened with O_DIRECT, or -1; closed for good when a read through it fails */
	uint64_t n = 0;
	/* a set of texts (agb_scan_set): text i is bytes [part_at[i], part_at[i] + part_n[i]) of the source, zeros in between */
	const void *const *parts = nullptr; const uint64_t *part_at = nullptr, *part_n = nullptr; uint32_t n_parts = 0;
	SliceSource(const void *h_text = nullptr, uint64_t len = 0) : mem((const uint8_t *)h_text), n(len)
	{
		cudaPointerAttributes attr; memset(&attr, 0, sizeof attr);
		pinned = len && cudaPointerGetAttributes(&attr, h_text) == cudaSuccess && attr.type == cudaMemoryTypeHost;
		cudaGetLastError();
	}
	SliceSource(const SliceSource &) = delete;
	SliceSource &operator=(const SliceSource &) = delete;
	~SliceSource() { if (dfd >= 0) close(dfd); }
};

/* a regular file from the descriptor's offset to its end (false: not a regular file) */
static bool fd_source(int fd, SliceSource &src)
{
	struct stat sb;
	if (fstat(fd, &sb) != 0 || !S_ISREG(sb.st_mode)) return false;
	src.fd = fd; src.fd_off = lseek(fd, 0, SEEK_CUR);
	src.n = (src.fd_off >= 0 && sb.st_size > src.fd_off) ? (uint64_t)(sb.st_size - src.fd_off) : 0;
	src.dfd = open_direct(fd, src.fd_off);
	return true;
}

/* bytes [off, off + len) of a set's source (SliceSource.parts) into dst */
static void gather_slice(const SliceSource &src, uint64_t off, uint8_t *dst, size_t len)
{
	const uint64_t end = off + len;
	uint64_t p = off;
	uint32_t i = (uint32_t)(std::upper_bound(src.part_at, src.part_at + src.n_parts, off) - src.part_at);
	for (i = i ? i - 1 : 0; p < end && i < src.n_parts; i++) {
		const uint64_t a = src.part_at[i], b = a + src.part_n[i];
		if (p < a) { const uint64_t z = std::min(a, end) - p; memset(dst + (p - off), 0, z); p += z; }
		if (p < end && p < b) { const uint64_t c = std::min(b, end) - p; memcpy(dst + (p - off), (const uint8_t *)src.parts[i] + (p - a), c); p += c; }
	}
	if (p < end) memset(dst + (p - off), 0, end - p);
}

/* bytes [off, off + len) of a pageable or file source into the ring buffer dst: 4 host threads memcpy or pread(2) a quarter
 * each (one thread's memcpy, or read(2) from the page cache, is a third of what PCIe takes; under 1 MiB of memory one thread
 * does).  Through the O_DIRECT descriptor whole 4 KiB blocks are asked for (the ring's buffers are page aligned and a multiple
 * of 4 KiB long; the file's last block comes back short); when that fails, the caller's own descriptor is used for good. */
static bool fill_slice(SliceSource &src, uint64_t off, uint8_t *dst, size_t len)
{
	if (src.mem && len < (1u << 20)) { memcpy(dst, src.mem + off, len); return true; }
	if (src.parts && len < (1u << 20)) { gather_slice(src, off, dst, len); return true; }
	for (;;) {
		const bool direct = !src.mem && src.dfd >= 0;
		const int fd = direct ? src.dfd : src.fd, T = 4;
		const size_t part = ((len + T - 1) / T + 4095) & ~(size_t)4095;
		std::thread th[T]; int used = 0; std::atomic<int> bad{0};
		for (int t = 0; t < T; t++) {
			const size_t a = (size_t)t * part; if (a >= len) break;
			const size_t l = std::min(part, len - a);
			const uint8_t *mem = src.mem ? src.mem + off + a : nullptr;
			const off_t at = src.fd_off + (off_t)(off + a);
			th[used++] = std::thread([=, &src, &bad] {
				if (src.parts) { gather_slice(src, off + a, dst + a, l); return; }
				if (mem) { memcpy(dst + a, mem, l); return; }
				for (size_t got = 0; got < l; ) {
					const size_t ask = direct ? ((l - got + 4095) & ~(size_t)4095) : l - got;
					ssize_t r = pread(fd, dst + a + got, ask, at + (off_t)got);
					if (r <= 0 || (direct && (size_t)r < l - got && ((size_t)r & 4095))) { bad = 1; return; }
					got += std::min((size_t)r, l - got);
				}
			});
		}
		for (int t = 0; t < used; t++) th[t].join();
		if (!bad || !direct) return !bad;
		close(src.dfd); src.dfd = -1;
	}
}

/* Per device, kept until agb_shutdown(): the copy and compute streams, the pinned ring and its events, the whole text of
 * agb_scan_host / agb_scan_fd and the device list behind records delivered to host memory.  A call holds g_host_mu[dev]
 * throughout.  Lock order: g_host_mu[dev] first, then g_ws_mu[dev] (in scan_device_impl and its kin), never the reverse. */
struct HostPath {
	cudaStream_t s_copy = nullptr, s_comp = nullptr;
	cudaEvent_t ev[STAGE_BUFS] = {nullptr, nullptr, nullptr};
	uint8_t *ring[STAGE_BUFS] = {nullptr, nullptr, nullptr};
	uint8_t *text = nullptr; size_t text_cap = 0;          /* (capacities in bytes) */
	agb_record *rec = nullptr; size_t rec_cap = 0;
	uint8_t *set_meta = nullptr; size_t set_meta_cap = 0;  /* agb_scan_set: its file and tile tables, the per-file counters */
};
static HostPath g_host[64];
static std::mutex g_host_mu[64];

/* the streams and events; the ring only when the source goes through it */
static int host_ensure(HostPath &H, const SliceSource &src)
{
	if (!H.s_copy) CUDA_TRY(cudaStreamCreateWithFlags(&H.s_copy, cudaStreamNonBlocking));
	if (!H.s_comp) CUDA_TRY(cudaStreamCreateWithFlags(&H.s_comp, cudaStreamNonBlocking));
	for (int i = 0; i < STAGE_BUFS; i++) if (!H.ev[i]) CUDA_TRY(cudaEventCreateWithFlags(&H.ev[i], cudaEventDisableTiming));
	if (src.n && !src.pinned) for (int i = 0; i < STAGE_BUFS; i++) if (!H.ring[i]) CUDA_TRY(cudaMallocHost(&H.ring[i], H2D_SLICE));
	return AGB_OK;
}

static void host_release(int dev)
{
	std::lock_guard<std::mutex> lk(g_host_mu[dev]);
	HostPath &H = g_host[dev];
	if (!H.s_copy && !H.text && !H.rec && !H.set_meta) return;              /* (the events and the ring are made after s_copy) */
	if (cudaSetDevice(dev) != cudaSuccess) { cudaGetLastError(); return; }
	cudaDeviceSynchronize();
	for (int i = 0; i < STAGE_BUFS; i++) { if (H.ev[i]) cudaEventDestroy(H.ev[i]); cudaFreeHost(H.ring[i]); }
	if (H.s_copy) cudaStreamDestroy(H.s_copy); if (H.s_comp) cudaStreamDestroy(H.s_comp);
	cudaFree(H.text); cudaFree(H.rec); cudaFree(H.set_meta);
	H = HostPath();
}

/* *p grown to `bytes` of device memory (what it held is not kept); a failed allocation leaves it NULL, the error cleared */
template <class T> static cudaError_t dev_reserve(T **p, size_t *cap, size_t bytes)
{
	if (bytes <= *cap) return cudaSuccess;
	cudaFree(*p); *p = nullptr; *cap = 0;
	const cudaError_t e = cudaMalloc(p, bytes);
	if (e != cudaSuccess) { *p = nullptr; cudaGetLastError(); return e; }
	*cap = bytes;
	return cudaSuccess;
}

/* bytes [lo, hi) of the source to dst on s_copy in H2D_SLICE pieces, straight from page-locked memory or through the ring,
 * after `slack` zero bytes at dst + (hi - lo) (stage 1 reads 16 bytes past its last chunk): every slice's event comes after
 * the zeroing.  after(i, ev) runs once slice i's copy is enqueued and ev recorded behind it.  Does not wait for the copies,
 * except on an error: then s_copy is drained first, so that no copy out of the ring or into dst is left in flight. */
static int upload(HostPath &H, SliceSource &src, uint64_t lo, uint64_t hi, uint8_t *dst, uint64_t slack,
                  const std::function<int(uint64_t, cudaEvent_t)> &after = nullptr)
{
	struct Drain { cudaStream_t s; bool on = true; ~Drain() { if (on) cudaStreamSynchronize(s); } } drain{H.s_copy};
	CUDA_TRY(cudaMemsetAsync(dst + (hi - lo), 0, slack, H.s_copy));
	for (uint64_t i = 0, off = lo; off < hi; i++, off += H2D_SLICE) {
		const uint64_t len = std::min<uint64_t>(H2D_SLICE, hi - off);
		const int sb = (int)(i % STAGE_BUFS);
		if (src.pinned) CUDA_TRY(cudaMemcpyAsync(dst + (off - lo), src.mem + off, len, cudaMemcpyHostToDevice, H.s_copy));
		else {
			CUDA_TRY(cudaEventSynchronize(H.ev[sb]));     /* that ring buffer has been consumed (by this call or an earlier one) */
			if (!fill_slice(src, off, H.ring[sb], (size_t)len)) {
				snprintf(g_err, sizeof g_err, "pread(2) failed or hit the end of the file in [%llu, %llu)", (unsigned long long)off, (unsigned long long)(off + len));
				return AGB_ERR_ARG;
			}
			CUDA_TRY(cudaMemcpyAsync(dst + (off - lo), H.ring[sb], len, cudaMemcpyHostToDevice, H.s_copy));
		}
		CUDA_TRY(cudaEventRecord(H.ev[sb], H.s_copy));
		if (after) { int rc = after(i, H.ev[sb]); if (rc) return rc; }
	}
	drain.on = false;
	return AGB_OK;
}

/* AGB_MAX_TEXT_BYTES: the most bytes of text the library keeps on the device (0 or unset: no cap) */
static uint64_t max_text_bytes(void)
{
	const char *e = getenv("AGB_MAX_TEXT_BYTES");
	return (e && *e) ? strtoull(e, nullptr, 10) : 0;
}

/* scan_stream_impl: the whole text does not fit on the device (cudaErrorMemoryAllocation, or more than AGB_MAX_TEXT_BYTES);
 * the caller scans it in windows instead */
#define SCAN_NEEDS_WINDOWS 1

static int scan_stream_impl(const agb_desc &d, const agb_pattern *px, SliceSource &src, int want,
                            agb_record *records, uint64_t capacity, agb_result *res)
{
	memset(res, 0, sizeof *res);
	int dev = 0; CUDA_TRY(cudaGetDevice(&dev));
	if (dev < 0 || dev >= 64) return AGB_ERR_ARG;
	std::lock_guard<std::mutex> hlk(g_host_mu[dev]);
	std::lock_guard<std::mutex> lk(g_ws_mu[dev]);
	HostPath &H = g_host[dev];
	Workspace &W = g_ws[dev];
	const uint64_t n = src.n;
	const size_t need = (size_t)((n + 15) / 16 * 16 + 4096);
	const uint64_t cap_bytes = max_text_bytes();
	if (cap_bytes && need > cap_bytes) {
		cudaFree(H.text); H.text = nullptr; H.text_cap = 0;       /* the cap holds between scans too */
		return SCAN_NEEDS_WINDOWS;
	}
	const cudaError_t e = dev_reserve(&H.text, &H.text_cap, need);
	if (e == cudaErrorMemoryAllocation) return SCAN_NEEDS_WINDOWS;
	CUDA_TRY(e);
	int rc = ws_prepare(W, n); if (rc) return rc;
	rc = host_ensure(H, src); if (rc) return rc;
	CUDA_TRY(dev_reserve(&H.rec, &H.rec_cap, (want & AGB_WANT_RECORDS) ? capacity * sizeof(agb_record) : 0));
	rc = ws_upload_desc(W, d, H.s_comp); if (rc) return rc;
	rc = tables_prepare(W, d, px, H.s_comp); if (rc) return rc;
	const bool use_front = front_usable(d) && n > 0;
	const bool count_in_front = use_front && (want & AGB_WANT_ORDINALS) && d.L == 1;
	if (count_in_front) { rc = ordinals_prepare_blocks(d, W, n, H.s_comp); if (rc) return rc; }
	const uint64_t words_per_slice = H2D_SLICE / 512, n_slices = (n + H2D_SLICE - 1) / H2D_SLICE;
	CUDA_TRY(cudaMemsetAsync(W.totals, 0, 16 * sizeof(unsigned long long), H.s_comp));
	CUDA_TRY(cudaEventRecord(W.e0, H.s_comp));
	rc = upload(H, src, 0, n, H.text, need - n, [&](uint64_t i, cudaEvent_t ev) -> int {
		CUDA_TRY(cudaStreamWaitEvent(H.s_comp, ev, 0));
		/* stage 1 on the previous slice: its last chunk looks 4 bytes into this one, which is now on its way */
		return use_front && i ? front_launch(d, W, H.text, n, (i - 1) * words_per_slice, i * words_per_slice, true, H.s_comp, count_in_front) : AGB_OK;
	});
	if (rc) return rc;
	if (use_front) { rc = front_launch(d, W, H.text, n, (n_slices - 1) * words_per_slice, ~0ull, true, H.s_comp, count_in_front); if (rc) return rc; }
	CUDA_TRY(cudaEventRecord(W.e1, H.s_comp));
	rc = stages_after_front(d, W, H.text, n, use_front, count_in_front, want, -1, H.rec, capacity, H.s_comp, res); if (rc) return rc;
	if (res->n_records) {
		CUDA_TRY(cudaMemcpyAsync(records, H.rec, res->n_records * sizeof(agb_record), cudaMemcpyDeviceToHost, H.s_comp));
		CUDA_TRY(cudaStreamSynchronize(H.s_comp));
	}
	CUDA_TRY(cudaStreamSynchronize(H.s_copy));
	CUDA_TRY(cudaEventElapsedTime(&res->ms_front, W.e0, W.e1));
	CUDA_TRY(cudaEventElapsedTime(&res->ms_records, W.e1, W.e2));
	return AGB_OK;
}

/* ------------------------------------------------------------------------------------------------
 * texts larger than the device's memory: the text in windows (DESIGN 3.4).  Window i owns the bytes [a_i, a_i + w) and is
 * scanned as a shard of the whole text (shard.cu): from hl bytes before it to hr bytes behind it, the cut rule deciding
 * which records are its own.  Two device buffers: while window i is scanned on the compute stream, a host thread moves
 * window i + 1 (halos included: the bytes it shares with window i are uploaded again) through the pinned ring on the copy
 * stream.  A window whose last record runs past hr, or whose left halo starts inside a run of the delimiter, is scanned
 * again with that halo doubled -- in a buffer of its own -- until it is long enough or the range reaches the text's end.
 * Counts and histograms are summed; each window's records are made global on the device and appended to the caller's
 * list until it is full; the ordinals follow the gather's arithmetic (agb_shard_part).
 * ---------------------------------------------------------------------------------------------- */
/* device memory of one windowed scan */
struct WinBuffers {
	uint8_t *buf[2] = {nullptr, nullptr}, *big = nullptr; size_t big_cap = 0;
	agb_record *rec = nullptr; size_t rec_cap = 0;          /* (capacities in bytes) */
	~WinBuffers() { cudaFree(buf[0]); cudaFree(buf[1]); cudaFree(big); cudaFree(rec); }
};

#define WIN_SLACK 4096            /* zeroed bytes behind a window's scanned range, as behind a whole text */

/* window i with halos of (at most) hl and hr bytes */
struct WinGeom { uint64_t a, n_local, hl, hr, lo, hi; bool first, open_end, reaches_end; };
static WinGeom win_geom(uint64_t n, uint64_t w, uint64_t i, uint64_t hl, uint64_t hr)
{
	WinGeom g;
	const uint64_t m = n ? (n + w - 1) / w : 1;
	g.a = i * w; g.n_local = std::min<uint64_t>(w, n - g.a);
	g.hl = i ? std::min<uint64_t>(hl, g.a) : 0;                       /* a, w and hl are multiples of 512: so is the clamp */
	g.hr = std::min<uint64_t>(hr, n - g.a - g.n_local);
	g.lo = g.a - g.hl; g.hi = g.a + g.n_local + g.hr;
	g.first = i == 0; g.open_end = i + 1 == m; g.reaches_end = g.hi >= n;
	return g;
}

static int scan_windowed(const agb_desc &d, const agb_pattern *px, SliceSource &src, uint64_t w, int want,
                         agb_record *records, uint64_t capacity, agb_result *res)
{
	memset(res, 0, sizeof *res);
	int dev = 0; CUDA_TRY(cudaGetDevice(&dev));
	if (dev < 0 || dev >= 64) return AGB_ERR_ARG;
	std::lock_guard<std::mutex> lk(g_host_mu[dev]);
	HostPath &H = g_host[dev];
	int rc = host_ensure(H, src); if (rc) return rc;
	const uint64_t n = src.n;
	const bool want_list = (want & AGB_WANT_RECORDS) && capacity, ord = (want & AGB_WANT_ORDINALS) != 0;
	WinBuffers B;
	const size_t buf_bytes = std::min<uint64_t>(n, w + AGB_HALO_LEFT + AGB_HALO_RIGHT) + WIN_SLACK;
	for (int b = 0; b < 2; b++) CUDA_TRY(cudaMalloc(&B.buf[b], buf_bytes));
	/* most windows own far fewer records than bytes; one that owns more is scanned again with a longer list */
	if (want_list) CUDA_TRY(dev_reserve(&B.rec, &B.rec_cap, std::min<uint64_t>(capacity, w / 256 + 4096) * sizeof(agb_record)));
	const uint64_t m = n ? (n + w - 1) / w : 1;
	rc = upload(H, src, 0, win_geom(n, w, 0, AGB_HALO_LEFT, AGB_HALO_RIGHT).hi, B.buf[0], WIN_SLACK); if (rc) return rc;
	CUDA_TRY(cudaStreamSynchronize(H.s_copy));
	uint64_t copied = 0; long long origin = 0, closes_before = 0;
	int dseed = -1, next_dseed = -1;                         /* delim_kind 3: the delimiter's state in front of a window's scan */
	for (uint64_t i = 0; i < m; i++) {
		/* the next window on its way while this one is scanned (the thread has the pinned ring and src.dfd to itself until joined) */
		int up_rc = AGB_OK; char up_err[sizeof g_err] = "";
		std::thread up;
		struct Joiner { std::thread &t; ~Joiner() { if (t.joinable()) t.join(); } } joiner{up};   /* every way out of this iteration */
		if (i + 1 < m) {
			const WinGeom gn = win_geom(n, w, i + 1, AGB_HALO_LEFT, AGB_HALO_RIGHT);
			uint8_t *dst = B.buf[(i + 1) & 1];
			up = std::thread([&, gn, dst] {
				up_rc = cudaSetDevice(dev) == cudaSuccess ? upload(H, src, gn.lo, gn.hi, dst, WIN_SLACK) : AGB_ERR_CUDA;
				if (up_rc) memcpy(up_err, g_err, sizeof up_err);     /* (g_err is per thread) */
			});
		}
		auto join_up = [&]() -> int {           /* the next window's bytes on the device, the ring free */
			if (up.joinable()) up.join();
			if (up_rc) { memcpy(g_err, up_err, sizeof up_err); return up_rc; }
			CUDA_TRY(cudaStreamSynchronize(H.s_copy));
			return AGB_OK;
		};
		uint64_t hl = AGB_HALO_LEFT, hr = AGB_HALO_RIGHT;
		const uint8_t *base = B.buf[i & 1];
		WinGeom g; agb_result lres; agb_shard_part part;
		/* delim_kind 3: the next window's scan starts where this one determines the delimiter's state (its lo lies inside this
		 * window's range; a kind-3 left halo is never too short) */
		const int64_t next_lo = i + 1 < m ? (int64_t)win_geom(n, w, i + 1, AGB_HALO_LEFT, AGB_HALO_RIGHT).lo : -1;
		for (;;) {
			g = win_geom(n, w, i, hl, hr);
			const uint64_t room = want_list ? std::min<uint64_t>(capacity - copied, B.rec_cap / sizeof(agb_record)) : 0;
			rc = shard_window_scan(d, px, base + g.hl, g.n_local, g.hl, g.hr, g.first, g.open_end, g.reaches_end, want,
			                       B.rec, room, H.s_comp, &lres, &part, dseed, next_lo >= 0 ? next_lo - (int64_t)g.lo : -1, &next_dseed);
			if (rc < 0) return rc;
			int short_halos = rc;
			if (g.lo == 0) short_halos &= ~HALO_SHORT_LEFT;      /* the scan starts where the text does: a run there really begins there */
			if (!short_halos) {
				if (!(want_list && lres.n_matched > room && room < capacity - copied)) break;
				/* more records than the list had room for, and the caller's list has more: again with room for all of them */
				CUDA_TRY(dev_reserve(&B.rec, &B.rec_cap, std::min<uint64_t>(capacity - copied, lres.n_matched) * sizeof(agb_record)));
				continue;
			}
			if (short_halos & HALO_SHORT_LEFT) hl *= 2;
			if (short_halos & HALO_SHORT_RIGHT) hr *= 2;
			g = win_geom(n, w, i, hl, hr);
			rc = join_up(); if (rc) return rc;                      /* the ring is needed here */
			const size_t need = g.hi - g.lo + WIN_SLACK;
			const cudaError_t e = dev_reserve(&B.big, &B.big_cap, need);
			if (e != cudaSuccess) {
				snprintf(g_err, sizeof g_err, "a record that begins in bytes [%llu, %llu) of the text does not fit in device memory with its halos (%llu bytes: %s)",
				         (unsigned long long)g.a, (unsigned long long)(g.a + g.n_local), (unsigned long long)need, cudaGetErrorString(e));
				return e == cudaErrorMemoryAllocation ? AGB_ERR_NOMEM : AGB_ERR_CUDA;
			}
			rc = upload(H, src, g.lo, g.hi, B.big, WIN_SLACK); if (rc) return rc;
			CUDA_TRY(cudaStreamSynchronize(H.s_copy));
			base = B.big;
		}
		res->n_matched += lres.n_matched; res->n_flagged += lres.n_flagged;
		for (int l = 0; l <= AGB_MAXERR; l++) res->level_hist[l] += lres.level_hist[l];
		res->ms_front += lres.ms_front; res->ms_records += lres.ms_records;
		if (ord && i == 0) { origin = part.ord_origin; res->n_closes += (uint64_t)part.virt; }
		if (lres.n_records) {
			/* offsets: local to the scanned range, which starts at g.lo = g.a + part.byte_base; ordinals as the gather makes them */
			rc = shard_window_rebase(B.rec, lres.n_records, (long long)g.a + part.byte_base, origin + closes_before - part.ord_fix, ord, H.s_comp);
			if (rc) return rc;
			CUDA_TRY(cudaMemcpyAsync(records + copied, B.rec, lres.n_records * sizeof(agb_record), cudaMemcpyDeviceToHost, H.s_comp));
			CUDA_TRY(cudaStreamSynchronize(H.s_comp));
			copied += lres.n_records;
		}
		if (ord) { closes_before += (long long)part.closes; res->n_closes += part.closes; }
		dseed = next_dseed;
		rc = join_up(); if (rc) return rc;
	}
	res->n_records = copied;
	res->truncated = ((want & AGB_WANT_RECORDS) && res->n_matched > capacity) ? 1 : 0;
	return AGB_OK;
}

/* the window of a text that does not fit: two windows and their halos in what AGB_MAX_TEXT_BYTES allows, and in three
 * quarters of the device's free memory less 512 MiB (the rest: the workspace of a window -- bitmaps, ordinal blocks and
 * candidate list, about 4 % of it -- and its record list) */
static uint64_t fallback_window(void)
{
	uint64_t budget = max_text_bytes();
	size_t fr = 0, tot = 0;
	if (cudaMemGetInfo(&fr, &tot) == cudaSuccess) {
		const uint64_t usable = fr > (512ull << 20) ? (fr - (512ull << 20)) / 4 * 3 : 0;
		if (!budget || usable < budget) budget = usable;
	} else cudaGetLastError();
	const uint64_t per = AGB_HALO_LEFT + AGB_HALO_RIGHT + WIN_SLACK;
	return budget / 2 >= per + 4096 ? (budget / 2 - per) & ~(uint64_t)511 : 4096;
}

/* window_bytes == 0: the whole text on the device when it fits, windows when it does not */
static int scan_host_any(const agb_pattern *p, const void *h_text, uint64_t n, uint64_t window_bytes, int want,
                         agb_record *records, uint64_t capacity, agb_result *res)
{
	if (!p || !res || (!h_text && n)) return AGB_ERR_ARG;
	if ((want & AGB_WANT_RECORDS) && capacity && !records) return AGB_ERR_ARG;
	SliceSource src(h_text, n);
	if (window_bytes) return scan_windowed(p->d, p, src, window_bytes, want, records, capacity, res);
	int rc = scan_stream_impl(p->d, p, src, want, records, capacity, res);
	if (rc == SCAN_NEEDS_WINDOWS) rc = scan_windowed(p->d, p, src, fallback_window(), want, records, capacity, res);
	return rc;
}

static int scan_fd_any(const agb_pattern *p, int fd, uint64_t window_bytes, int want, agb_record *records, uint64_t capacity, agb_result *res)
{
	if (!p || !res) return AGB_ERR_ARG;
	if ((want & AGB_WANT_RECORDS) && capacity && !records) return AGB_ERR_ARG;
	SliceSource src;
	if (fd_source(fd, src)) {
		/* regular file: the size is known, read(2) goes straight into the pinned ring, slice by slice */
		int rc = window_bytes ? scan_windowed(p->d, p, src, window_bytes, want, records, capacity, res)
		                      : scan_stream_impl(p->d, p, src, want, records, capacity, res);
		if (rc == SCAN_NEEDS_WINDOWS) rc = scan_windowed(p->d, p, src, fallback_window(), want, records, capacity, res);
		if (src.fd_off >= 0) lseek(fd, src.fd_off + (off_t)src.n, SEEK_SET);        /* as read(2) would have left it */
		return rc;
	}
	/* pipes, ttys: fill_buf() semantics -- read until EOF into a growing buffer, then as host memory */
	size_t cap = 1 << 20, len = 0; uint8_t *buf = (uint8_t *)malloc(cap);
	if (!buf) return AGB_ERR_NOMEM;
	for (;;) {
		if (len == cap) { cap *= 2; uint8_t *nb = (uint8_t *)realloc(buf, cap); if (!nb) { free(buf); return AGB_ERR_NOMEM; } buf = nb; }
		ssize_t r = read(fd, buf + len, cap - len);
		if (r < 0) { free(buf); snprintf(g_err, sizeof g_err, "read failed"); return AGB_ERR_ARG; }
		if (r == 0) break;
		len += (size_t)r;
	}
	int rc = scan_host_any(p, buf, len, window_bytes, want, records, capacity, res);
	free(buf);
	return rc;
}

extern "C" int agb_scan_host(const agb_pattern *p, const void *h_text, uint64_t n, int want,
                             agb_record *records, uint64_t capacity, agb_result *res)
{
	return scan_host_any(p, h_text, n, 0, want, records, capacity, res);
}

extern "C" int agb_scan_fd(const agb_pattern *p, int fd, int want, agb_record *records, uint64_t capacity, agb_result *res)
{
	return scan_fd_any(p, fd, 0, want, records, capacity, res);
}

static bool window_ok(uint64_t w)
{
	if (w >= 4096 && w % 512 == 0) return true;
	snprintf(g_err, sizeof g_err, "window_bytes (%llu) must be a multiple of 512 and at least 4096", (unsigned long long)w);
	return false;
}

extern "C" int agb_scan_host_windowed(const agb_pattern *p, const void *h_text, uint64_t n, uint64_t window_bytes, int want,
                                      agb_record *records, uint64_t capacity, agb_result *res)
{
	if (!window_ok(window_bytes)) return AGB_ERR_ARG;
	return scan_host_any(p, h_text, n, window_bytes, want, records, capacity, res);
}

extern "C" int agb_scan_fd_windowed(const agb_pattern *p, int fd, uint64_t window_bytes, int want,
                                    agb_record *records, uint64_t capacity, agb_result *res)
{
	if (!window_ok(window_bytes)) return AGB_ERR_ARG;
	return scan_fd_any(p, fd, window_bytes, want, records, capacity, res);
}

/* ------------------------------------------------------------------------------------------------
 * a set of files in one pass (DESIGN 3.4.1).  `agrep pattern *.c` scans many small files; one agb_scan_host per file pays
 * the fixed cost of a scan (copies, about ten launches, a synchronising read-back) per file.  Here the files go through the
 * pinned ring into one device buffer, each at a 16-byte boundary, and one launch sequence scans them all: the record stage's
 * tile form (k_records_dense, k_regex) and the ordinals in their SET form, one block per 32 KiB tile of a file, each block
 * taking its file's bounds as the text's.  A file's records come out in one ordered list, file after file, offsets and
 * ordinals relative to the file, the file's index in agb_record.pad; per-file counts are added up by the blocks.  Stages 1
 * and 1.5 do not run: the tile form walks every byte, which on small files costs less than the launches and the read-back
 * that the filters would add per file.
 * ---------------------------------------------------------------------------------------------- */
extern "C" int agb_scan_set(const agb_pattern *p, const void *const *h_texts, const uint64_t *sizes, uint32_t n_files, int want,
                            agb_record *records, uint64_t capacity, agb_result *per_file, agb_result *total)
{
	if (!p || !total) return AGB_ERR_ARG;
	memset(total, 0, sizeof *total);
	if (!n_files) {
		if (h_texts || sizes || per_file) { snprintf(g_err, sizeof g_err, "agb_scan_set: no files, but file arrays were given"); return AGB_ERR_ARG; }
		return AGB_OK;
	}
	if (!h_texts || !sizes || !per_file) { snprintf(g_err, sizeof g_err, "agb_scan_set: h_texts, sizes and per_file are needed"); return AGB_ERR_ARG; }
	const bool want_list = (want & AGB_WANT_RECORDS) && capacity, ord = (want & AGB_WANT_ORDINALS) != 0;
	if (want_list && !records) { snprintf(g_err, sizeof g_err, "agb_scan_set: a capacity without a record list"); return AGB_ERR_ARG; }
	for (uint32_t i = 0; i < n_files; i++)
		if (!h_texts[i] && sizes[i]) { snprintf(g_err, sizeof g_err, "agb_scan_set: file %u has no text but %llu bytes", i, (unsigned long long)sizes[i]); return AGB_ERR_ARG; }
	const agb_desc &d = p->d;
	/* the layout: file i at at[i]; its record tiles (of the kernel that runs) and its ordinals tiles (of [0, n + L)) */
	const uint64_t rec_tile = d.engine == AGB_ENGINE_REGEX ? RX_TILE : DENSE_TILE;
	std::vector<uint64_t> at(n_files);
	std::vector<SetFile> files(n_files);
	std::vector<SetTile> rtiles, otiles;
	uint64_t bytes = 0;
	for (uint32_t i = 0; i < n_files; i++) {
		const uint64_t n = sizes[i];
		at[i] = bytes;
		files[i].off = bytes; files[i].n = n; files[i].ord_tile0 = (uint32_t)otiles.size();
		/* bitap.c:151-156, as ordinals_launch */
		files[i].j0 = (d.user_delim && d.engine != AGB_ENGINE_ASEARCH0 && n >= (uint64_t)d.L && memcmp(h_texts[i], d.delim, (size_t)d.L) == 0) ? -1 : 0;
		for (uint64_t t = 0; t * rec_tile < n; t++) rtiles.push_back(SetTile{i, (uint32_t)t});
		for (uint64_t t = 0; t * ORD_TILE < n + (uint64_t)d.L; t++) otiles.push_back(SetTile{i, (uint32_t)t});
		bytes += (n + 15) & ~15ull;
	}
	int dev = 0; CUDA_TRY(cudaGetDevice(&dev));
	if (dev < 0 || dev >= 64) return AGB_ERR_ARG;
	std::lock_guard<std::mutex> hlk(g_host_mu[dev]);
	std::lock_guard<std::mutex> lk(g_ws_mu[dev]);
	HostPath &H = g_host[dev];
	Workspace &W = g_ws[dev];
	const size_t need = (size_t)bytes + 4096;
	const uint64_t cap_bytes = max_text_bytes();
	const cudaError_t e = (cap_bytes && need > cap_bytes) ? cudaErrorMemoryAllocation : dev_reserve(&H.text, &H.text_cap, need);
	if (e == cudaErrorMemoryAllocation) {
		snprintf(g_err, sizeof g_err, "a set of %u files (%llu bytes on the device) does not fit in device memory; scan it in smaller sets",
		         n_files, (unsigned long long)need);
		return AGB_ERR_NOMEM;
	}
	CUDA_TRY(e);
	/* no record is shorter than a byte but the empty ones, at most one per byte and file: the list never needs more */
	const uint64_t list_cap = want_list ? std::min<uint64_t>(capacity, bytes + 2ull * n_files) : 0;
	static_assert(RX_TILE == DENSE_TILE && ORD_TILE == DENSE_TILE, "ws_prepare sizes the tile counts for DENSE_TILE");
	int rc = ws_prepare(W, (uint64_t)std::max(rtiles.size(), otiles.size()) * DENSE_TILE); if (rc) return rc;
	SliceSource src;
	src.parts = h_texts; src.part_at = at.data(); src.part_n = sizes; src.n_parts = n_files; src.n = bytes;
	rc = host_ensure(H, src); if (rc) return rc;
	CUDA_TRY(dev_reserve(&H.rec, &H.rec_cap, list_cap * sizeof(agb_record)));
	const size_t fb = files.size() * sizeof(SetFile), rb = rtiles.size() * sizeof(SetTile), ob = otiles.size() * sizeof(SetTile);
	const size_t sb = (size_t)n_files * SET_STATS * sizeof(unsigned long long);
	const size_t o_r = (fb + 15) & ~(size_t)15, o_o = o_r + ((rb + 15) & ~(size_t)15), o_s = o_o + ((ob + 15) & ~(size_t)15);
	CUDA_TRY(dev_reserve(&H.set_meta, &H.set_meta_cap, o_s + sb));
	SetFile *d_files = reinterpret_cast<SetFile *>(H.set_meta);
	SetTile *d_rtiles = reinterpret_cast<SetTile *>(H.set_meta + o_r), *d_otiles = reinterpret_cast<SetTile *>(H.set_meta + o_o);
	unsigned long long *d_stats = reinterpret_cast<unsigned long long *>(H.set_meta + o_s);
	CUDA_TRY(cudaMemcpyAsync(d_files, files.data(), fb, cudaMemcpyHostToDevice, H.s_comp));
	if (rb) CUDA_TRY(cudaMemcpyAsync(d_rtiles, rtiles.data(), rb, cudaMemcpyHostToDevice, H.s_comp));
	CUDA_TRY(cudaMemcpyAsync(d_otiles, otiles.data(), ob, cudaMemcpyHostToDevice, H.s_comp));
	CUDA_TRY(cudaMemsetAsync(d_stats, 0, sb, H.s_comp));
	rc = ws_upload_desc(W, d, H.s_comp); if (rc) return rc;
	rc = tables_prepare(W, d, p, H.s_comp); if (rc) return rc;
	CUDA_TRY(cudaMemsetAsync(W.totals, 0, 16 * sizeof(unsigned long long), H.s_comp));
	rc = upload(H, src, 0, bytes, H.text, need - bytes, [&](uint64_t, cudaEvent_t ev) -> int {
		CUDA_TRY(cudaStreamWaitEvent(H.s_comp, ev, 0));
		return AGB_OK;
	});
	if (rc) return rc;
	if (!bytes) CUDA_TRY(cudaStreamSynchronize(H.s_copy));     /* (the slack's zeroing: no slice event follows it) */
	CUDA_TRY(cudaEventRecord(W.e1, H.s_comp));
	RecParams P; memset(&P, 0, sizeof P);
	P.text = H.text; P.n = bytes; P.desc = W.d_desc; P.records = H.rec; P.capacity = list_cap; P.totals = W.totals;
	P.levels = (want & AGB_WANT_LEVELS) ? 1 : 0; P.want_level = -1;
	P.own_lo = INT64_MIN; P.own_hi = INT64_MAX; P.shard_last = 1;
	P.rx_tab = W.d_regex; P.rx_tail = W.regex_tail;
	P.set_files = d_files; P.set_tiles = d_rtiles; P.set_stats = d_stats;
	/* -p with a delimiter of two or more bytes: the delimiter's state over the ordinals tiles, every file from its own start */
	if (d.delim_kind == 3) { rc = dstate_launch(d, W, H.text, bytes, -1, H.s_comp, d_files, d_otiles, otiles.size()); if (rc) return rc; }
	P.dstate = W.dstate;
	if (!rtiles.empty()) {
		rc = tile_stage(d.engine == AGB_ENGINE_REGEX ? launch_regex_set : launch_dense_set, d, P, W, (unsigned)rtiles.size(), want_list, H.s_comp);
		if (rc) return rc;
	}
	if (ord) { rc = ordinals_set_launch(d, W, H.text, d_files, d_otiles, otiles.size(), d_stats, want_list ? H.rec : nullptr, list_cap, H.s_comp); if (rc) return rc; }
	CUDA_TRY(cudaEventRecord(W.e2, H.s_comp));
	std::vector<unsigned long long> stats((size_t)n_files * SET_STATS);
	CUDA_TRY(cudaMemcpyAsync(stats.data(), d_stats, sb, cudaMemcpyDeviceToHost, H.s_comp));
	CUDA_TRY(cudaStreamSynchronize(H.s_comp));
	const uint64_t virt = (d.L == 1 && d.delim[0] == '\n') ? 1 : 0;   /* the virtual '\n' closes a record of its own (ordinals_launch) */
	for (uint32_t i = 0; i < n_files; i++) {
		agb_result &r = per_file[i];
		const unsigned long long *st = &stats[(size_t)i * SET_STATS];
		memset(&r, 0, sizeof r);
		r.n_matched = st[0];
		for (int l = 0; l <= AGB_MAXERR; l++) r.level_hist[l] = st[1 + l];
		r.n_closes = ord ? st[10] + virt : 0;
		if (want & AGB_WANT_RECORDS) {
			const uint64_t room = capacity > total->n_matched ? capacity - total->n_matched : 0;
			r.n_records = std::min<uint64_t>(r.n_matched, room);
			r.truncated = r.n_matched > room ? 1 : 0;
		}
		total->n_matched += r.n_matched;
		for (int l = 0; l <= AGB_MAXERR; l++) total->level_hist[l] += r.level_hist[l];
		total->n_closes += r.n_closes;
	}
	if (want & AGB_WANT_RECORDS) {
		total->n_records = std::min<uint64_t>(total->n_matched, capacity);
		total->truncated = total->n_matched > capacity ? 1 : 0;
	}
	if (total->n_records) {
		CUDA_TRY(cudaMemcpyAsync(records, H.rec, total->n_records * sizeof(agb_record), cudaMemcpyDeviceToHost, H.s_comp));
		CUDA_TRY(cudaStreamSynchronize(H.s_comp));
	}
	CUDA_TRY(cudaStreamSynchronize(H.s_copy));
	CUDA_TRY(cudaEventElapsedTime(&total->ms_records, W.e1, W.e2));
	return AGB_OK;
}

/* ---- a text kept in HBM across scans (the drop-in layer's exec() scans the same file K + 2 times under -B,
 * agrep.c:3582-3728: one upload instead of K + 2) ---- */
struct agb_text { uint8_t *d; uint64_t n; int dev; };

static int text_upload(SliceSource &src, agb_text **out)
{
	int dev = 0; CUDA_TRY(cudaGetDevice(&dev));
	if (dev < 0 || dev >= 64) return AGB_ERR_ARG;
	const uint64_t n = src.n;
	const size_t need = (size_t)((n + 15) / 16 * 16 + 4096);
	const uint64_t cap_bytes = max_text_bytes();
	if (cap_bytes && need > cap_bytes) {
		snprintf(g_err, sizeof g_err, "a text of %llu bytes does not fit in AGB_MAX_TEXT_BYTES=%llu; agb_scan_host and agb_scan_fd scan it in windows",
		         (unsigned long long)n, (unsigned long long)cap_bytes);
		return AGB_ERR_NOMEM;
	}
	std::unique_ptr<agb_text, decltype(&agb_text_free)> t(new agb_text{nullptr, n, dev}, agb_text_free);   /* freed on every error exit */
	if (cudaMalloc(&t->d, need) != cudaSuccess) { t->d = nullptr; snprintf(g_err, sizeof g_err, "cudaMalloc of %zu bytes for the text failed", need); cudaGetLastError(); return AGB_ERR_NOMEM; }
	std::lock_guard<std::mutex> lk(g_host_mu[dev]);
	HostPath &H = g_host[dev];
	int rc = host_ensure(H, src); if (rc) return rc;
	rc = upload(H, src, 0, n, t->d, need - n); if (rc) return rc;
	CUDA_TRY(cudaStreamSynchronize(H.s_copy));
	*out = t.release();
	return AGB_OK;
}

extern "C" int agb_text_from_host(const void *h_text, uint64_t n, agb_text **out)
{
	if (!out || (!h_text && n)) return AGB_ERR_ARG;
	SliceSource src(h_text, n);
	return text_upload(src, out);
}

extern "C" int agb_text_from_fd(int fd, agb_text **out)
{
	if (!out) return AGB_ERR_ARG;
	SliceSource src;
	if (!fd_source(fd, src)) { snprintf(g_err, sizeof g_err, "agb_text_from_fd needs a regular file"); return AGB_ERR_ARG; }
	int rc = text_upload(src, out);
	/* as read(2) would have left it; untouched when the text was not taken, so that the caller can read it another way */
	if (src.fd_off >= 0) lseek(fd, src.fd_off + (rc == AGB_OK ? (off_t)src.n : 0), SEEK_SET);
	return rc;
}

extern "C" void agb_text_free(agb_text *t) { if (t) { cudaFree(t->d); delete t; } }
extern "C" uint64_t agb_text_size(const agb_text *t) { return t ? t->n : 0; }
extern "C" const void *agb_text_device(const agb_text *t) { return t ? t->d : nullptr; }

/* device scan of a resident text with the record list delivered to host memory */
extern "C" int agb_scan_text(const agb_pattern *p, const agb_text *t, int want, agb_record *records, uint64_t capacity, agb_result *res)
{
	if (!p || !t || !res) return AGB_ERR_ARG;
	if ((want & AGB_WANT_RECORDS) && capacity && !records) return AGB_ERR_ARG;
	CUDA_TRY(cudaSetDevice(t->dev));
	std::lock_guard<std::mutex> lk(g_host_mu[t->dev]);
	HostPath &H = g_host[t->dev];
	CUDA_TRY(dev_reserve(&H.rec, &H.rec_cap, (want & AGB_WANT_RECORDS) ? capacity * sizeof(agb_record) : 0));
	int rc = scan_device_impl(p->d, t->d, t->n, want, -1, H.rec, capacity, nullptr, res, nullptr, p); if (rc) return rc;
	if (res->n_records) CUDA_TRY(cudaMemcpy(records, H.rec, res->n_records * sizeof(agb_record), cudaMemcpyDeviceToHost));
	return AGB_OK;
}

/* keep the records of one level (stable, in place: the output index never overtakes the input index) */
__global__ void __launch_bounds__(1024) k_filter_level(agb_record *recs, uint64_t n, int level, unsigned long long *n_out)
{
	__shared__ unsigned long long s_warp[32];
	__shared__ unsigned long long s_base;
	const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	if (tid == 0) s_base = 0;
	__syncthreads();
	for (uint64_t t0 = 0; t0 < n; t0 += 1024) {
		const uint64_t i = t0 + tid;
		agb_record r; r.level = -1;
		if (i < n) r = recs[i];
		const bool keep = i < n && r.level == level;
		const uint32_t m = __ballot_sync(0xffffffffu, keep);
		if (lane == 0) s_warp[wid] = __popc(m);
		__syncthreads();                                    /* every read of this tile is done */
		unsigned long long before = s_base;
		for (uint32_t w = 0; w < wid; w++) before += s_warp[w];
		if (keep) recs[before + __popc(m & ((1u << lane) - 1u))] = r;
		__syncthreads();
		if (tid == 0) { unsigned long long t = 0; for (int w = 0; w < 32; w++) t += s_warp[w]; s_base += t; }
		__syncthreads();
	}
	if (tid == 0) *n_out = s_base;
}

/* agrep.c:3582-3728: when the exact pass finds nothing, -B looks for the smallest D in 1..min(M-1,8) with a match,
 * rescanning every file once per D, and then once more at that D to print.  The rows are nested (A_j contains A_{j-1},
 * asearch.c:98-114), so ONE pass at a level k yields every record's smallest level <= k: the histogram tells the best
 * level, the list -- filtered to that level on the device -- is what the printing pass would print.  The pass runs at
 * k = 2 first (the anchor filter is still selective there; it also answers the exact question), then 4, then 8: one
 * pass for every best level up to 2, at most three.
 * best_k: smallest level with a match (-1: none up to min(M-1, 8)); res->n_matched: records at that level (what
 * the reference reports as "N words match within K errors"); d_records/capacity: their ordered list (level filled). */
extern "C" int agb_bestmatch_device(const char *pattern, const agb_options *opt, const void *d_text, uint64_t n,
                                    void *stream, agb_record *d_records, uint64_t capacity, int *best_k, agb_result *res,
                                    char *err, size_t errlen)
{
	if (!pattern || !opt || !best_k || !res) return AGB_ERR_ARG;
	if (capacity && !d_records) return AGB_ERR_ARG;
	agb_options o = *opt; agb_desc d; int m = (int)strlen(pattern);
	cudaStream_t st = (cudaStream_t)stream;
	o.bestmatch = 1;
	*best_k = -1;
	/* D < M of the exact pattern (agrep.c:3594); M there counts the delimiter and separator too */
	o.k = 0;
	int rc = agbi_build(pattern, &o, &d, err, errlen); if (rc) return rc;
	int kmax = d.M - 1; if (kmax > AGB_MAXERR) kmax = AGB_MAXERR; if (kmax > m - 1) kmax = m - 1;
	const int want = AGB_WANT_LEVELS | (capacity ? AGB_WANT_RECORDS : AGB_WANT_COUNT);
	int stages[3] = { 2, 4, 8 }, prev = -1;
	for (int si = 0; si < 3; si++) {
		int k = stages[si] < kmax ? stages[si] : kmax;
		if (k <= prev) break;
		o.k = k;
		rc = agbi_build(pattern, &o, &d, err, errlen); if (rc) return rc;
		rc = scan_device_impl(d, d_text, n, want, -1, d_records, capacity, st, res);
		if (rc) return rc;
		int best = -1;
		for (int l = prev + 1; l <= k; l++) if (res->level_hist[l]) { best = l; break; }    /* levels <= prev were already known to be empty */
		prev = k;
		if (best < 0) continue;
		*best_k = best;
		const uint64_t n_best = res->level_hist[best];
		if (capacity) {
			if (res->truncated) {
				/* the list of all levels up to k did not fit: once more, at the best level only */
				o.k = best;
				rc = agbi_build(pattern, &o, &d, err, errlen); if (rc) return rc;
				agb_result r2;
				rc = scan_device_impl(d, d_text, n, want, best, d_records, capacity, st, &r2); if (rc) return rc;
				res->n_records = r2.n_records; res->truncated = r2.truncated;
			} else if (best < k && res->n_records) {
				int dev = 0; CUDA_TRY(cudaGetDevice(&dev));
				std::lock_guard<std::mutex> lk(g_ws_mu[dev]);
				Workspace &W = g_ws[dev];
				k_filter_level<<<1, 1024, 0, st>>>(d_records, res->n_records, best, W.totals + 15); g_launches++;
				CUDA_TRY(cudaGetLastError());
				CUDA_TRY(cudaStreamSynchronize(st));
				res->n_records = std::min<uint64_t>(n_best, capacity);
			}
		}
		res->n_matched = n_best;
		return AGB_OK;
	}
	res->n_matched = 0; res->n_records = 0;
	return AGB_OK;
}
