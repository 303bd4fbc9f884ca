/* agrep_b200/csrc/scan_internal.cuh -- what the translation units of libagrepb200's device side share: launch
 * geometry, kernel parameter blocks, the per-device workspace and the host functions that cross files.
 *   front.cu    stage 1   k_front            (anchor filter, HBM-bound)
 *   refine.cu   stage 1.5 k_refine           (local verification of anchor hits)
 *   records.cu  stage 2   k_records_dense, k_records_list (records_kernel.cuh; records_wide.cu: 320-bit rows)
 *   slices.cu   stage 2   k_records_slices   (the automaton over every byte, in lockstep)
 *   regex.cu    stage 2   k_regex            (regular expressions: re()'s recurrence over every byte, tile form)
 *   aux.cu      bitmap compaction, scans, density sample, ordinals, synthetic corpus
 *   scan.cu     workspace, orchestration, the C ABI (include/agrep_b200.h)
 * automaton.cuh holds the device pieces stages 1.5 and 2 share (the recurrence, the match test, the text reader). */
#ifndef AGB_SCAN_INTERNAL_CUH
#define AGB_SCAN_INTERNAL_CUH
#include "agrep_b200.h"
#include "pattern_internal.h"
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <atomic>
#include <algorithm>
#include <type_traits>

extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

#define CUDA_TRY(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
	snprintf(g_err, sizeof g_err, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
	return AGB_ERR_CUDA; } } while (0)

/* ---- stage 1 ---- */
#define FRONT_THREADS 256
#define FRONT_CH      4                                   /* 16-byte chunks per thread and stage              */
#define FRONT_STAGE_CHUNKS (FRONT_THREADS * FRONT_CH)     /* 1024 chunks = 16 KiB = 32 bitmap words per stage */
#define FRONT_STAGE_BYTES  (FRONT_STAGE_CHUNKS * 16)
#define FRONT_SLOT_BYTES   (FRONT_STAGE_BYTES + 16)       /* + the 16 bytes that follow: the last chunk's windows look 3 bytes ahead */
#define FRONT_NST     2                                   /* stages in flight per CTA (32 KiB); 6 CTAs = 48 warps per SM */
/* tools/front_bench.cu on an H100 (16 GiB, 400 W power limit): this shape within the run-to-run spread (about 5 %) of the
 * best ring shapes tried, 4 stages x 3 CTAs and 3 x 4 -- stage 1 is DRAM-bound there, so the ring shape matters little */
#define FRONT_CTAS_PER_SM 6
#define FRONT_WORDS_PER_STAGE (FRONT_STAGE_CHUNKS / 32)

struct FrontParams {
	const uint8_t *text;         /* 16-byte aligned */
	uint32_t    *bitmap;         /* one word per 32 chunks */
	uint64_t     n;              /* bytes */
	uint64_t     n_chunks;       /* ceil(n/16) */
	uint64_t     readable;       /* bytes that may be read from text: 16 * n_chunks (+16 when the caller's slack allows) */
	uint64_t     stage_begin, stage_end;   /* this launch covers stages [stage_begin, stage_end) of 1024 chunks each */
	uint32_t     fold, amask;
	uint32_t     one, scale;     /* 1 (kept opaque so the first Horner step stays an IMAD) and 256^(4-anchor_len) */
	uint32_t     anchor[AGB_MAXANCHOR];
	uint32_t     coef[AGB_MAXANCHOR];   /* prod_i (x - anchor[i]) mod 2^32, low order first, leading 1 implied */
	int          n3;             /* mixed plan: three-byte anchors, their polynomial (scaled by 256 in the kernel) */
	uint32_t     s256;
	int          alen;           /* exact count: bytes of the literal */
	uint32_t     coef3[4];
	uint16_t    *nl_blocks;      /* COUNT: delimiter bytes per 512-byte block = per bitmap word (the ordinals' first pass, fused) */
	uint32_t     delim4, dfold4; /* the 1-byte delimiter, four times (lower case if both cases end a record: dfold4 = 0x20202020) */
};
#define FRONT_SMEM (FRONT_NST * FRONT_SLOT_BYTES)

/* ---- stage 1.5 ---- */
#define REFINE_THREADS 128
struct RefineParams {
	const uint8_t *text; const uint32_t *bitmap; uint32_t *out; uint32_t *warp_counts;
	uint64_t n, n_chunks, n_words;
	const agb_desc *desc;
	uint32_t fold, amask; int na, k, pat_len;
	int gb, ng;                  /* groups staged before the chunk, groups staged in total */
	int lo_off, hi_off;          /* the windows of a chunk at byte `base` lie inside [base - lo_off, base + hi_off) */
	uint32_t anchor[AGB_MAXANCHOR]; int32_t off[AGB_MAXANCHOR];
	uint32_t coef[AGB_MAXANCHOR]; uint32_t one, scale; int poly;   /* stage 1's polynomial, to spot the candidate windows cheaply */
	int t1, t1_words;            /* the band count: usable; words of the window [p0 - k, p0 + pat_len + k) */
	uint32_t t1_fold, t1_pat[16], t1_care[16];   /* literal pattern bytes (little endian words), 0x80 per literal position */
	uint32_t hmul; uint64_t hidx64[4];           /* anchor bytes -> anchor: slot (bytes * hmul) >> 27 holds its index + 1 (32 bytes, packed:
	                                                byte arrays in a kernel parameter get the whole struct copied to local memory) */
	uint32_t hval[16], hmask[16]; uint64_t hoffs64[2];   /* the anchors of both groups: bytes, mask (4 or 3 bytes), off (16 bytes, packed) */
	int n3; uint32_t coef3[4];                   /* mixed plan: the three-byte group's polynomial */
	int sm_count;
};

/* ---- stage 2 ---- */
#define REC_THREADS 128          /* list form: threads per block, one candidate each */

struct RecParams {
	const uint8_t  *text;
	uint64_t n, n_chunks;
	const agb_desc *desc;        /* device copy */
	uint32_t *tile_counts;       /* dense: per block; list: per candidate */
	const uint64_t *tile_offsets;/* exclusive scan of tile_counts (emit pass) */
	agb_record *records; uint64_t capacity;
	unsigned long long *totals;  /* [0] matched, [1] flagged chunks, [2..10] level histogram, [12] candidates in the list */
	const uint64_t *cand; uint64_t cand_cap;   /* list form: ordered flagged chunk numbers, totals[12] of them */
	agb_record *cand_first;      /* list form: the first record each candidate reported in the count launch (most report 0 or 1) */
	int emit;                    /* 0: count pass, 1: emit pass */
	int levels;                  /* 1: best-match bookkeeping (smallest matching row) */
	int want_level;              /* levels: report records whose smallest level <= want_level (-1: all matching) */
	int warm;                    /* slices form: bytes of warm-up before a slice (>= positions + rows) */
	/* a shard of a larger text (agb_scan_sharded): the scanned bytes include a halo on either side, and a record belongs
	 * to the shard whose own range [own_lo, own_hi) holds the last byte of the delimiter that OPENED it (the re-fed byte,
	 * asearch.c:175-196); unsharded: everything.  shard_last = 0: the delimiter appended behind the text (bitap.c:161-165)
	 * is not the text's own end -- an owned record that only it closes has outrun the halo (totals[11] is raised) */
	int64_t own_lo, own_hi; int shard_last;
	/* regular expressions (regex.cu): the byte-sliced Next tables on the device, TAIL's epsilon move at '\n';
	 * 320-bit rows (agb_desc.wide): the agb_wide words on the device */
	const void *rx_tab; int rx_tail;
	/* a set of files (agb_scan_set, the kernels' SET form): block b scans tile set_tiles[b].tile of file set_tiles[b].file */
	const struct SetFile *set_files; const struct SetTile *set_tiles; unsigned long long *set_stats;
	/* delim_kind 3: the delimiter's state at the start of every 128-byte slice (delim_state.cu; a set: slice 256 t + i of its
	 * ordinals tile t, SetFile.ord_tile0) */
	const uint8_t *dstate;
};
/* agb_scan_set: file f is the text [off, off + n) of one device buffer (off a multiple of 16), scanned as if alone.  A tile of
 * the record stage (32 KiB) and of the ordinals (32 KiB of [0, n + L)) lies in one file, so a block of the SET form takes its
 * file's text bounds where a whole-text scan takes 0 and n, and nothing is carried across a file's edge.  Per file, the
 * blocks add into set_stats[SET_STATS f + ...]: [0] matching records, [1 + l] records of smallest level l, [10] record
 * closes (ordinals).  j0: -1 when the file starts with the user's delimiter (bitap.c:151-156). */
struct SetFile { uint64_t off, n; uint32_t ord_tile0; int32_t j0; };
struct SetTile { uint32_t file, tile; };
#define SET_STATS 16
/* dseed: delim_kind 3, the delimiter's state in front of the scanned bytes (-1: the text's own start, the virtual '\n') */
struct ShardInfo { int64_t own_lo, own_hi; int last; int dseed; };
#define DENSE_THREADS 256
#define DENSE_TILE    32768
#define RX_TILE       32768                               /* regex.cu: k_regex's tile */
#define DENSE_TAIL    2048
#define DENSE_PER     (DENSE_TILE / DENSE_THREADS)          /* 128 bytes per thread */
#define DENSE_SMEM (DENSE_TILE + DENSE_TAIL)
#define SL_THREADS 128
#define SL_PER     256
#define SL_TILE    (SL_THREADS * SL_PER)        /* 32 KiB: six CTAs per SM, so that the staging of one overlaps the walk of others */
#define SL_APRON   128                          /* bytes staged before the tile: the warm-up of thread 0 */
#define SL_STRIDE  (SL_PER + 4)
#define SL_SMEM    ((SL_THREADS + 1) * SL_STRIDE + 12)
#define COMPACT_THREADS 256
#define COMPACT_WPT 4            /* words per thread: a block covers 1024 words */
#define SCAN_BLOCK 16384
/* the record stage's list form pays while at most 5 % of the chunks are flagged: one thread per candidate (20 B of
 * scratch each) against a tile form's walk over every byte ('the' flags 11 % of the chunks, 'government' 1.1 %) */
static inline bool list_form_pays(uint64_t flagged, uint64_t n_chunks) { return flagged <= n_chunks / 20 + 1024; }

/* ---- ordinals ---- */
#define ORD_THREADS 256
#define ORD_TILE    32768
#define ORD_PER     (ORD_TILE / ORD_THREADS)       /* 128 bytes per thread */
#define ORD_BLOCK   512

struct OrdParams {
	const uint8_t *text; uint64_t n;
	uint16_t *blocks; uint32_t *tiles; const uint64_t *tile_off;
	agb_record *records; const unsigned long long *totals; uint64_t capacity;
	uint8_t delim[AGB_MAXDELIM + 2], dfold[AGB_MAXDELIM + 2]; int L, kind;   /* delim: folded (lower case where dfold is 0x20) */
	long long j0;                /* 0, or -1 when the text starts with the user's delimiter (bitap.c:151-156) */
	const uint8_t *dstate;       /* delim_kind 3: as RecParams.dstate */
};

/* does the record opened by the delimiter that starts at `begin` belong to this scan (see RecParams.own_lo)?
 * close_pos: the last byte of the delimiter that closes it */
__device__ __forceinline__ bool rec_owned(const RecParams &P, int64_t begin, int L, int64_t close_pos)
{
	const int64_t oe = begin + L - 1;
	if (oe < P.own_lo || oe >= P.own_hi) return false;
	if (!P.shard_last && close_pos >= (int64_t)P.n) P.totals[11] = 1ull;
	return true;
}

/* a record-stage launcher at a row count known at run time: launch(std::integral_constant<int, nrows>()) for
 * 1 <= nrows <= N, counted in g_launches; -1 for any other row count */
template <int N, typename F>
static int launch_rows(int nrows, const F &launch)
{
	if (nrows == N) { launch(std::integral_constant<int, N>()); g_launches++; return 0; }
	if constexpr (N > 1) return launch_rows<N - 1>(nrows, launch);
	return -1;
}

/* ---- host ---- */
#define H2D_SLICE   (64ull << 20)      /* bytes per H2D slice of agb_scan_host; a multiple of the 16 KiB stage */
#define STAGE_BUFS  3
struct Workspace {               /* grow-only device scratch, one per device */
	uint32_t *bitmap = nullptr; size_t bitmap_bytes = 0;
	uint32_t *bitmap2 = nullptr;                                    /* stage 1.5: the survivors (same size as bitmap) */
	uint32_t *range_counts = nullptr; uint64_t *range_offsets = nullptr;   /* per warp range of stage 1.5: survivor counts, their scan */
	unsigned refine_ctas = 0;                                       /* grid of the last stage 1.5 launch */
	/* anchor planner: the sample counts of the candidate grams; the plan chosen for the last (descriptor, text) */
	uint32_t *d_gram = nullptr; unsigned int *h_gram = nullptr;     /* device: 128 grams + 128 masks + 128 counts; pinned: the same */
	uint64_t plan_key = 0; bool plan_valid = false; agb_desc plan_desc;
	size_t cand_hint = 0;                                          /* candidates the last scans needed (sizes the list without a host round trip) */
	uint32_t *tile_counts = nullptr; uint64_t *tile_offsets = nullptr; size_t tiles = 0;
	uint64_t *cand = nullptr; uint32_t *cand_counts = nullptr; uint64_t *cand_offsets = nullptr; agb_record *cand_first = nullptr; size_t cand_cap = 0;
	uint32_t *scan_sums = nullptr; uint64_t *scan_offs = nullptr; size_t scan_cap = 0;
	uint16_t *ord_blocks = nullptr; size_t ord_blocks_cap = 0;     /* delimiter ends per 512-byte block (AGB_WANT_ORDINALS) */
	long long ord_j0 = 0;                                          /* -1 when the text starts with the user's delimiter (bitap.c:151-156) */
	int ord_virt = 0;                                              /* 1: the virtual '\n' closes a record of its own (1-byte '\n' delimiter) */
	unsigned long long *totals = nullptr;          /* 16 counters */
	unsigned long long *h_totals = nullptr;        /* pinned */
	agb_desc *d_desc = nullptr; agb_desc h_desc_copy; bool desc_valid = false;
	cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr;
	int sm_count = 0;
	/* the Next tables of the last regular expression scanned (regex.cu), and their host copy */
	uint64_t *d_regex = nullptr; uint64_t h_regex[8 * 256]; size_t regex_bytes = 0; int regex_tail = 0;
	/* delim_kind 3 (delim_state.cu): per 32 KiB tile its transition function and entry state, per 128-byte slice its entry state */
	uint32_t *ds_func = nullptr; uint8_t *ds_entry = nullptr, *dstate = nullptr; size_t ds_tiles = 0;
};

/* scan.cu */
#include <mutex>
extern Workspace g_ws[64];
extern std::mutex g_ws_mu[64];   /* one scan at a time per device (the workspaces are shared scratch) */
int  scan_device_impl(const agb_desc &d, const void *d_text, uint64_t n, int want, int want_level,
                      agb_record *d_records, uint64_t capacity, cudaStream_t st, agb_result *res, const ShardInfo *sh = nullptr,
                      const agb_pattern *px = nullptr);
/* px (here and below): the pattern that holds what its descriptor cannot -- a regular expression's follow sets, the words
 * of 320-bit rows; NULL for a descriptor that needs neither */
/* shard.cu: one window of the windowed scan -- the shard scan, with a halo that is too short reported as a positive code
 * (a set of HALO_SHORT_*) instead of an error; and the window's records made global on the device.  delim_kind 3: dseed is
 * the delimiter's state in front of the scanned range, *state_out gets its state at offset state_at of that range */
enum { HALO_SHORT_RIGHT = 1, HALO_SHORT_LEFT = 2 };
int  shard_window_scan(const agb_desc &d, const agb_pattern *px, const void *d_win, uint64_t n_local, uint64_t halo_left, uint64_t halo_right,
                       bool first, bool open_end, bool reaches_end, int want, agb_record *d_records, uint64_t capacity,
                       cudaStream_t st, agb_result *lres, agb_shard_part *part,
                       int dseed = -1, int64_t state_at = -1, int *state_out = nullptr);
int  shard_window_rebase(agb_record *d_records, uint64_t n, long long byte_add, long long ord_add, bool ordinals, cudaStream_t st);
/* front.cu */
bool front_usable(const agb_desc &d);
bool exact_count_usable(const agb_desc &d);
int  exact_count_launch(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n, cudaStream_t st);
bool poly_setup(const uint32_t *a, int na, int bits, uint32_t *coef);
int  front_launch(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n, uint64_t word_begin, uint64_t word_end, bool slack16, cudaStream_t st, bool count_delims = false);
/* refine.cu */
int  refine_launch(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n, cudaStream_t st, bool *ran);
unsigned refine_grid(const Workspace &W, uint64_t n);
int  compact_ranges_launch(Workspace &W, uint64_t n, cudaStream_t st);
#define REFINE_MAX_RANGES 16384  /* >= warps of the largest stage 1.5 grid */
/* records.cu, slices.cu: one launch of the given form (count pass or emit pass, RecParams.emit) */
int  launch_dense(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st);
/* the SET form of the dense tile kernel and of k_regex: one block per entry of P.set_tiles */
int  launch_dense_set(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st);
int  launch_regex_set(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st);
int  launch_records_list(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st);
/* records_wide.cu: the same forms for 320-bit rows (agb_desc.wide: the words in RecParams.rx_tab), which the launchers
 * above hand over to */
int  launch_dense_wide(int nrows, const RecParams &P, unsigned grid, cudaStream_t st, bool set);
int  launch_records_list_wide(int nrows, const RecParams &P, unsigned grid, cudaStream_t st);
int  launch_slices(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st);
bool slices_usable(const agb_desc &d);
/* regex.cu: stage 2 of AGB_ENGINE_REGEX (RecParams.rx_tab set), and its tables (returns the bytes written: 32- or 64-bit words) */
int  launch_regex(const agb_desc &d, const RecParams &P, unsigned grid, cudaStream_t st);
size_t regex_tables(const agb_desc &d, const agb_regex &rx, uint64_t *out);
/* delim_state.cu: the delimiter's state at every slice of [0, n + L) into W.dstate (delim_kind 3); seed: the state in front
 * of the text (-1: after the virtual '\n'); a set: the slices of its ordinals tiles, each file from the virtual '\n' */
int  dstate_launch(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n, int seed, cudaStream_t st,
                   const struct SetFile *set_files = nullptr, const struct SetTile *set_tiles = nullptr, uint64_t set_n_tiles = 0);
/* aux.cu */
__global__ void k_gram_sample(const uint8_t *text, uint64_t n_chunks, uint32_t nblk, uint32_t blk_chunks,
                              int ngram, const uint32_t *gram, const uint32_t *gmask, uint32_t fold, unsigned int *counts,
                              int pair_first, int n_pair);
__global__ void k_compact_count(const uint32_t *bitmap, uint64_t n_words, uint32_t *block_counts, unsigned long long *totals);
__global__ void k_compact_write(const uint32_t *bitmap, uint64_t n_words, const uint64_t *block_offsets, uint64_t *cand, uint64_t cand_cap);
__global__ void k_scan_tiles(const uint32_t *counts, uint64_t *offsets, uint64_t n_tiles, unsigned long long *total);
__global__ void k_scan_partial(const uint32_t *counts, uint64_t n, uint32_t *block_sums, const unsigned long long *n_dev);
__global__ void k_scan_apply(const uint32_t *counts, uint64_t n, const uint64_t *block_offsets, uint64_t *offsets, const unsigned long long *n_dev);
int  front_is_dense(Workspace &W, uint64_t n, cudaStream_t st, bool *dense);
int  ordinals_launch(const agb_desc &d, Workspace &W, const void *d_text, uint64_t n, agb_record *d_records, uint64_t capacity, cudaStream_t st, bool blocks_counted = false);
int  ordinals_reserve(const agb_desc &d, Workspace &W, uint64_t n);
/* the ordinals of a set: delimiter ends per file into set_stats, every record's j counted from its own file's start */
int  ordinals_set_launch(const agb_desc &d, Workspace &W, const void *d_text, const SetFile *d_files, const SetTile *d_ord_tiles,
                         uint64_t ord_tiles, unsigned long long *d_stats, agb_record *d_records, uint64_t capacity, cudaStream_t st);
/* a block of a SET kernel: its tile's file, and the text bounds of that file */
__device__ __forceinline__ void set_enter(const SetFile *files, const SetTile *tiles, const uint8_t *&text, uint64_t &n,
                                          uint64_t &tile, uint32_t &file)
{
	const SetTile t = tiles[blockIdx.x];
	const SetFile f = files[t.file];
	text += f.off; n = f.n; tile = t.tile; file = t.file;
}
#endif
