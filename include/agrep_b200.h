/* include/agrep_b200.h -- C ABI of libagrepb200.so: the H100 scan engine behind agrep's scan path.
 *
 * Plain C, pointers and sizes only.  Two layers:
 *
 *  (1) The reentrant engine ABI (agb_*): an explicit scan descriptor (the words the reference keeps in
 *      globals: Mask[], Init[0], Init1, NO_ERR_MASK, endposition, D_endpos -- agrep.c:135-140 -- plus the
 *      flags the scan loops read) and a scan call over a device or host text span that returns the
 *      number of matching records and, on request, the ordered list of matching records in the exact
 *      (lasti, print_end, j) terms the reference hands to output() (bitap.c:212-214, asearch.c:162-168).
 *
 *  (2) The drop-in layer (libagrepb200_dropin.so, declared in agrep_b200_dropin.h): bitap(), asearch(),
 *      asearch0(), asearch1(), sgrep(), fill_buf(), alloc_buf(), free_buf() with the reference's own
 *      signatures, reading the reference's globals, so the reference's exec() links against it unchanged.
 *
 * There is no CPU fallback: every agb_scan_* call runs the sm_90a kernels and fails with
 * AGB_ERR_CUDA when no device is usable.
 */
#ifndef AGREP_B200_H
#define AGREP_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AGB_MAXERR    8     /* MaxError, reference agrep.h:45 */
#define AGB_MAXDELIM  8     /* MAXDELIM, reference agrep.h:35 */
#define AGB_MAXANCHOR 24

enum {
	AGB_OK = 0,
	AGB_ERR_PATTERN = -1,   /* pattern rejected; message in the err buffer (the reference prints it and returns -1) */
	AGB_ERR_CUDA = -2,      /* CUDA runtime error / no device; message via agb_last_error() */
	AGB_ERR_ARG = -3,
	AGB_ERR_NOMEM = -4
};

/* The subset of agrep's command line that reaches the scan path (reference agrep.c:2121-2739). */
typedef struct agb_options {
	int32_t k;            /* -#  number of errors D (0..8)                                   */
	int32_t nocase;       /* -i  NOUPPER                                                     */
	int32_t wordbound;    /* -w  WORDBOUND                                                   */
	int32_t wholeline;    /* -x  WHOLELINE                                                   */
	int32_t inverse;      /* -v  INVERSE                                                     */
	int32_t linenum;      /* -n  LINENUM: forces the bitap family (checksg.c:132)            */
	int32_t ins_free;     /* -p  I = 0                                                       */
	int32_t cost_i, cost_s, cost_d;   /* -I# -S# -D# ; 0 = not given                         */
	int32_t bestmatch;    /* -B  BESTMATCH: forces the bitap family (checksg.c:127)          */
	int32_t regex;        /* 1: accept regular expressions (an unescaped '|' or '*', preproce.c:139-142) as
	                         AGB_ENGINE_REGEX; 0: refuse them                                 */
	const char *delim;    /* -d  argument as typed, NULL = newline records                   */
	int32_t wide_approx;  /* 1: accept a simple literal of 64 to AGB_WIDE_MAXPOS positions at k = 1..8 (what the
	                         reference's sgrep() takes, up to 255 characters) in 320-bit rows; 0: refuse it     */
	int32_t sticky_delim; /* 1: accept -p (Init1 = ~0) with a delimiter of 2..AGB_MAXDELIM bytes, whose positions are then
	                         sticky too, so that records close at the delimiter as a subsequence (delim_kind 3);
	                         0: refuse it                                                                       */
} agb_options;

/* engines = which reference function the descriptor stands for */
enum { AGB_ENGINE_BITAP = 0,    /* bitap.c:169-284   exact shift-and                          */
       AGB_ENGINE_ASEARCH = 1,  /* asearch.c:94-306  k = 1..4                                 */
       AGB_ENGINE_ASEARCH0 = 2, /* asearch.c:620-774 k = 5..8                                 */
       AGB_ENGINE_ASEARCH1 = 3, /* asearch1.c:86-235 non-unit costs                           */
       AGB_ENGINE_SGREP_BM = 4, /* sgrep.c:262 + bm() sgrep.c:694: simple literal, k = 0      */
       AGB_ENGINE_REGEX = 5     /* re() agrep.c:1267-1917: regular expression, k = 0..4, lines */ };

/* front-end plan chosen by agb_compile for the device scan */
enum { AGB_PLAN_ALL = 0,        /* every 16-byte chunk goes to the record stage               */
       AGB_PLAN_ANCHORS = 1     /* pigeonhole pre-filter on k+1 disjoint literal anchors      */ };

/* The scan descriptor.  64-bit words, LSB aligned: pattern position p (1-based, delimiter first)
 * lives at bit M-p, bits >= M are the always-on feed (reference maskgen.c:218-234 with WORD=64). */
typedef struct agb_desc {
	uint64_t mask[256];       /* Mask[c]; for AGB_ENGINE_BITAP with -i the LUT[] of bitap.c:171 is pre-folded */
	uint64_t init0, init1, noerr, endpos, dendpos, dmask, wildmask;
	uint64_t reset[2 * AGB_MAXERR + 1]; /* rows right after a record closes (asearch.c:175-186), a constant */
	uint64_t start[2 * AGB_MAXERR + 1]; /* rows after the virtual leading '\n' when it does NOT close a record */
	int32_t  start_closes;    /* 1: the virtual '\n' closes a (never reported) record, scan starts from reset[] */
	int32_t  M, L;            /* positions; delimiter length                                  */
	uint8_t  delim[2 * AGB_MAXDELIM + 2];
	int32_t  delim_kind;      /* 0: border-free (every occurrence closes a record); 1: c^L run rule; 2: a self-overlapping
	                             delimiter (taken from the left); 3: -p with L >= 2, the delimiter's positions sticky: the
	                             closes come from a scan of the delimiter's state over the text (DESIGN 3.3.1) */
	int32_t  k;               /* error rows                                                   */
	int32_t  nrows;           /* k+1, or 2k+1 for ASEARCH1 (rows k..2k live)                  */
	int32_t  cost_i, cost_s, cost_d;
	int32_t  engine, and_mode, inverse, user_delim, outtail;
	/* plan */
	int32_t  plan;
	int32_t  n_anchors, anchor_len;           /* anchor_len in 2..4 bytes                    */
	uint32_t anchor[AGB_MAXANCHOR];           /* little-endian packed anchor bytes           */
	uint32_t anchor_fold;                     /* OR-mask applied to text and anchors (0x20 per letter byte under -i / bm) */
	uint32_t anchor_mask;                     /* 0xFFFFFFFF, 0x00FFFFFF or 0x0000FFFF        */
	/* local verification of anchor hits (stage 1.5): anchor i starts anchor_off[i] positions after the
	 * separator slot; the pattern proper has pat_len positions; refine = 1 when a hit can be checked on the
	 * window [p - off - k, p + pat_len - off + k) alone (single pattern, no '#', no -v/-p) */
	int32_t  refine, pat_len;
	int32_t  anchor_off[AGB_MAXANCHOR];
	/* mixed plan: besides the n_anchors anchors of anchor_len = 4 bytes, n_anchors3 pieces of the pattern stand with a
	 * three-byte gram (the piece is only three bytes long, or that is its rare gram); n_anchors + n_anchors3 = k + 1 */
	int32_t  n_anchors3;
	uint32_t anchor3[4];                      /* low three bytes, folded like anchor[] */
	int32_t  anchor3_off[4];
	int32_t  adaptive;                        /* 1: the device scan may re-plan the anchors from a sample of the text */
	/* 0x20 for the delimiter positions that accept both cases of a letter (-i lower-cases the whole internal pattern, the
	 * delimiter included, maskgen.c:52-58, 259-266), else 0: away from the automaton a delimiter byte c is recognised by
	 * (c | delim_fold[p]) == (delim[p] | delim_fold[p]); filled by agb_compile / agb_pattern_from_desc from mask[] */
	uint8_t  delim_fold[2 * AGB_MAXDELIM + 2];
	/* 1: the anchors are the k + 2 equal-length pieces of the pair plan -- stage 1 flags a chunk only where one piece starts
	 * and another one starts in it or in the chunk after it (set by the device scan's planner only; 0 from every caller) */
	uint8_t  pair_plan;
	/* 1: the automaton's rows are 320 bits wide and its words are in agb_pattern_wide(), not here (set by agb_compile only;
	 * 0 from every caller) */
	uint8_t  wide;
	/* 1: the caller accepts delim_kind 3 (-p with a delimiter of two or more bytes): set by agb_compile when
	 * agb_options.sticky_delim is on and the pattern needs it, by the caller of agb_pattern_from_desc; 0 refuses such
	 * a descriptor */
	uint8_t  sticky_delim;
} agb_desc;

typedef struct agb_pattern agb_pattern;       /* opaque: agb_desc + bookkeeping              */

/* What a regular expression adds to the descriptor (AGB_ENGINE_REGEX): the Glushkov automaton's follow sets.
 * Positions are numbered as in the descriptor: position p at bit M-p; position 0 is the start state at bit M, which every
 * state holds.  Next(S) = the union of follow[p] over the positions p of S (compute_next, agrep.c:396-457), so
 * follow[0] is the start feed.  The descriptor of a regex pattern holds mask[] (Mask[], '.' matching '\n' too,
 * maskgen.c:243), init0 (Init[0], with the HEAD position), init1 (Init0 | 1), noerr (NO_ERR_MASK), endpos = 1 (the
 * trailing position of the ".( ... )." wrapper, preproce.c:231-236, 334-339), L = 1 with delim '\n' and k <= 4;
 * reset[] = start[] = the rows after a newline.  Records are always lines. */
#define AGB_REGEX_MAXPOS 63
typedef struct agb_regex {
	uint64_t follow[AGB_REGEX_MAXPOS + 1];    /* follow[p], p = 0..M                                */
	int32_t  head, tail;                      /* HEAD / TAIL of preprocess(); tail: the epsilon move at '\n' (agrep.c:1332) */
	int32_t  pad[2];
} agb_regex;

/* What a simple literal of more than 63 positions adds to the descriptor (sgrep()'s bm() and monkey() at k = 0, up to 255
 * characters as the reference accepts them, agrep.c:3057; at k = 1..8 with agb_options.wide_approx, the automaton the
 * engines AGB_ENGINE_ASEARCH/ASEARCH0 run for shorter simple literals): the words of 320-bit rows.  Word 0 holds bits
 * 0..63 of a row; position p is bit M-p, the always-on feed is bit M, as in the descriptor.  Masks that the descriptor
 * fills "everywhere but" (init0's feed, noerr, dmask) are filled up to the end of the last word that holds bit M, and the
 * words above it are zero, so a pattern of at most 63 positions has exactly its 64-bit words in word 0.  The descriptor of
 * such a pattern has wide = 1, its k, nrows = k + 1, its real M and everything that is not a word (L, delim, delim_fold,
 * delim_kind, engine, plan, anchors, pat_len, start_closes, inverse, user_delim, outtail); its 64-bit word fields (mask,
 * init0 ... wildmask, reset, start) are zero.  Row 0 of the post-delimiter and start rows is in reset/start, rows 1..k in
 * reset_up[0..k-1]/start_up[0..k-1] (appended, so that the layout of the k = 0 fields stays put). */
#define AGB_WIDE_WORDS  5
#define AGB_WIDE_MAXPOS (64 * AGB_WIDE_WORDS - 1)
typedef struct agb_wide {
	uint64_t mask[256][AGB_WIDE_WORDS];
	uint64_t init0[AGB_WIDE_WORDS], init1[AGB_WIDE_WORDS], noerr[AGB_WIDE_WORDS], endpos[AGB_WIDE_WORDS];
	uint64_t dendpos[AGB_WIDE_WORDS], dmask[AGB_WIDE_WORDS], reset[AGB_WIDE_WORDS], start[AGB_WIDE_WORDS];
	uint64_t reset_up[AGB_MAXERR][AGB_WIDE_WORDS], start_up[AGB_MAXERR][AGB_WIDE_WORDS];
} agb_wide;

/* one matching record, in the reference's own terms (file offsets, not buffer indexes):
 *   begin   = offset of lasti: first byte of the delimiter that closed the previous record; -1 for the
 *             virtual '\n' in front of the text (bitap.c:140), 0 when a user delimiter has not been seen yet
 *   end     = offset of print_end + 1 = first byte of the delimiter that closes this record
 *   ordinal = j at output() time; -n prints j-1 (agrep.c:3878); filled on the device when the scan is asked for
 *             AGB_WANT_ORDINALS (one more pass over the text that counts delimiters), else 0;
 *             agb_fill_ordinals() computes the same on a host copy of the text
 *   level   = smallest matching error level in best-match and AGB_WANT_LEVELS scans (a regular expression's levels
 *             come from an AGB_WANT_LEVELS scan), else k                                                   */
typedef struct agb_record {
	int64_t begin;
	int64_t end;
	int64_t ordinal;
	int32_t level;
	int32_t pad;              /* agb_scan_set: the index of the record's file; 0 from every other scan */
} agb_record;

enum { AGB_WANT_COUNT = 0, AGB_WANT_RECORDS = 1, AGB_WANT_ORDINALS = 2, AGB_WANT_LEVELS = 4 };

typedef struct agb_result {
	uint64_t n_matched;       /* num_of_matched for this text                                 */
	uint64_t n_records;       /* entries written to records (<= capacity; see truncated)      */
	uint64_t n_flagged;       /* 16-byte chunks the front-end passed to the record stage      */
	uint64_t level_hist[AGB_MAXERR + 1];      /* AGB_WANT_LEVELS: records by smallest level   */
	float    ms_front, ms_records;            /* device time of the two stages (CUDA events)  */
	uint64_t n_closes;        /* AGB_WANT_ORDINALS: record closes in the whole text, the virtual '\n' included (j at EOF):
	                             what a following shard adds to its ordinals (SURVEY 8e)      */
	uint32_t truncated;       /* 1: AGB_WANT_RECORDS and n_matched > capacity -- the list holds only the first `capacity`
	                             records (n_records of them); count again with a list of n_matched entries */
	uint32_t pad;
} agb_result;

/* ---- pattern front-end (host; mirrors checksg.c + preproce.c + maskgen.c) ---- */
int  agb_compile(const char *pattern, const agb_options *opt, agb_pattern **out, char *err, size_t errlen);
void agb_pattern_free(agb_pattern *p);
const agb_desc *agb_pattern_desc(const agb_pattern *p);
/* wrap words produced elsewhere (the drop-in layer passes the reference's globals); the plan fields are honoured
 * when plan == AGB_PLAN_ANCHORS, else every chunk goes to the record stage */
int  agb_pattern_from_desc(const agb_desc *d, agb_pattern **out, char *err, size_t errlen);
/* regular expressions: the follow sets of a pattern of AGB_ENGINE_REGEX (NULL for every other engine), and a pattern
 * from words produced elsewhere (d->engine must be AGB_ENGINE_REGEX; reset[] and start[] are derived here) */
const agb_regex *agb_pattern_regex(const agb_pattern *p);
int  agb_pattern_from_regex(const agb_desc *d, const agb_regex *rx, agb_pattern **out, char *err, size_t errlen);
/* the 320-bit words of a simple literal of more than 63 positions (NULL for every other pattern).  agb_pattern_from_desc
 * refuses such descriptors: the drop-in's sgrep() compiles from the pattern text.  With AGB_FORCE_WIDE=1 in the
 * environment agb_compile gives every AGB_ENGINE_SGREP_BM pattern this form, and with agb_options.wide_approx every simple
 * literal at k >= 1 (tests compare the two forms with it). */
const agb_wide *agb_pattern_wide(const agb_pattern *p);

/* ---- device scan ----
 * d_text: device pointer, 16-byte aligned, readable up to the next 16-byte boundary after n.
 * d_records: device buffer for agb_record[capacity] (may be NULL with AGB_WANT_COUNT).
 * stream: cudaStream_t as void* (NULL = default stream).  The call is synchronous w.r.t. the host
 * only for the 64-byte result read-back. */
int  agb_scan_device(const agb_pattern *p, const void *d_text, uint64_t n, int want,
                     agb_record *d_records, uint64_t capacity, void *stream, agb_result *res);

/* host text: staged through pinned buffers in slices cut at record boundaries, H2D overlapped with the
 * scan (the fill_buf replacement, bitap.c:450-477).  records: host array.
 * A text that does not fit on the device -- its buffer fails with cudaErrorMemoryAllocation, or it is larger than the
 * environment's AGB_MAX_TEXT_BYTES -- is scanned in windows, as by agb_scan_host_windowed, with the same result.  The
 * window then is the largest multiple of 512 such that two windows and their halos fit in AGB_MAX_TEXT_BYTES and in three
 * quarters of the device's free memory less 512 MiB (DESIGN 3.4). */
int  agb_scan_host(const agb_pattern *p, const void *h_text, uint64_t n, int want,
                   agb_record *records, uint64_t capacity, agb_result *res);

/* file descriptor: read(2) loop into the pinned ring, as agb_scan_host (windows included).  Starts at the current offset
 * and leaves it at EOF; regular files are pread(2) by four threads (AGB_ODIRECT=1: past the page cache), pipes are read
 * into a host buffer first */
int  agb_scan_fd(const agb_pattern *p, int fd, int want, agb_record *records, uint64_t capacity, agb_result *res);

/* as agb_scan_host / agb_scan_fd, but at most window_bytes of text (plus halos) is in device memory at a time; the
 * result -- n_matched, level_hist, n_closes, the ordered list with global offsets and ordinals, truncated -- is what
 * the whole-text scan returns.  window_bytes: a multiple of 512, >= 4096.  Each window is scanned as a shard of the
 * whole text (the cut rule of agb_scan_shard_local) while the next one is uploaded; a halo that turns out too short (a
 * record running past the right one, a run of the delimiter longer than the left one) is doubled and the window scanned
 * again, so only a record that does not fit in device memory with its halos is an error (AGB_ERR_NOMEM, naming where
 * it begins).  n_flagged, ms_front and ms_records are sums over the windows. */
int  agb_scan_host_windowed(const agb_pattern *p, const void *h_text, uint64_t n, uint64_t window_bytes, int want,
                            agb_record *records, uint64_t capacity, agb_result *res);
int  agb_scan_fd_windowed(const agb_pattern *p, int fd, uint64_t window_bytes, int want,
                          agb_record *records, uint64_t capacity, agb_result *res);

/* ---- a set of files in one device pass (`agrep pattern *.c`) ----
 * File i is the text h_texts[i][0..sizes[i]) (host memory; NULL only with size 0), framed as a whole text is: the virtual
 * '\n' in front of it, its delimiter appended behind it, j's start-with-delimiter rule, the phantom record at its end
 * dropped.  per_file[i] (n_files entries) holds what agb_scan_host on file i alone returns -- n_matched, level_hist,
 * n_closes -- with n_records / truncated as for a list of the room left behind the files before it; n_flagged and the
 * times are 0.  total: the sums, n_records / truncated of the whole list.
 * records: ONE ordered list, file 0's records, then file 1's, ...; cut after the first `capacity` records of the set.
 * Each record's begin, end and ordinal are relative to its own file, and its `pad` field holds the file's index.
 * The files go to the device together (each at a 16-byte boundary) and are scanned by one sequence of launches whatever
 * their number.  A set that does not fit in device memory (or in AGB_MAX_TEXT_BYTES) is refused with AGB_ERR_NOMEM:
 * batching is the caller's job.  n_files == 0 is valid only with NULL arrays. */
int  agb_scan_set(const agb_pattern *p, const void *const *h_texts, const uint64_t *sizes, uint32_t n_files, int want,
                  agb_record *records, uint64_t capacity, agb_result *per_file, agb_result *total);

/* ---- a text kept in HBM across scans ----
 * exec() scans the same file up to K + 2 times under -B (agrep.c:3582-3728); the drop-in layer uploads it once.
 * agb_text_from_fd: regular files, from the current offset to EOF, read(2) straight into the pinned ring; the offset is
 * left at EOF, or where it was when the call fails.  A text larger than AGB_MAX_TEXT_BYTES (environment) is refused with
 * AGB_ERR_NOMEM: scan it with agb_scan_host / agb_scan_fd, which use windows. */
typedef struct agb_text agb_text;
int  agb_text_from_host(const void *h_text, uint64_t n, agb_text **out);
int  agb_text_from_fd(int fd, agb_text **out);
void agb_text_free(agb_text *t);
uint64_t agb_text_size(const agb_text *t);
const void *agb_text_device(const agb_text *t);
/* as agb_scan_device over the resident text, the record list delivered to HOST memory */
int  agb_scan_text(const agb_pattern *p, const agb_text *t, int want, agb_record *records, uint64_t capacity, agb_result *res);

/* ---- one text over several GPUs: one process per GPU, the text sharded by byte range, NCCL only to gather ----
 * Records are independent once their boundaries are known (the automaton is reset at every delimiter, asearch.c:175-196),
 * so a rank scans its shard on its own.  The cut rule (SURVEY 8e) runs on the device: a record belongs to the shard that
 * holds the last byte of the delimiter that opened it; the shard's scan starts AGB_HALO_LEFT bytes before the shard (so
 * that a delimiter, or a run of "$$", that straddles the cut is parsed as in the whole text) and runs into the next
 * shard's first AGB_HALO_RIGHT bytes to finish the record in progress.  agb_shard_halo() fetches both halos from the
 * neighbours (ncclSend/ncclRecv of 64.5 KiB); the caller's buffer has room for them in front of and behind the shard.
 *
 *   buffer layout on every rank:   [ AGB_HALO_LEFT | shard: n_local bytes | AGB_HALO_RIGHT + 16 ]
 *                                                   ^ d_shard, 16-byte aligned; n_local a multiple of 512 on every rank but the last
 *
 * agb_scan_sharded: every rank ends up with the same result -- counts summed over the ranks, offsets and ordinals of the
 * whole text, the ordered list of ALL ranks' records in d_records (ncclAllGather of a 128-byte header per rank, then of the
 * lists padded to the longest).  global_offset: where this shard starts in the whole text. */
#define AGB_HALO_LEFT  512
#define AGB_HALO_RIGHT 65536
typedef struct agb_comm agb_comm;
int  agb_comm_unique_id(void *id128);                        /* rank 0: ncclGetUniqueId (128 bytes), to be handed to every rank */
int  agb_comm_init(agb_comm **out, int world, int rank, const void *id128);   /* on the current device */
void agb_comm_free(agb_comm *c);
int  agb_comm_world(const agb_comm *c);
int  agb_comm_rank(const agb_comm *c);
int  agb_shard_halo(agb_comm *c, void *d_shard, uint64_t n_local, void *stream);
int  agb_scan_sharded(const agb_pattern *p, agb_comm *c, const void *d_shard, uint64_t n_local, uint64_t global_offset,
                      int want, agb_record *d_records, uint64_t capacity, void *stream, agb_result *res);
/* the local half of agb_scan_sharded, for callers that move the lists themselves (and for one process that walks the
 * shards of a text one after the other): scans [d_shard - halo_left, d_shard + n_local + halo_right) and keeps the
 * records the cut rule gives to this shard.  first: nothing precedes the shard; open_end: the shard owns everything up
 * to the end of what is scanned; reaches_end: the scanned bytes end where the whole text ends.  Offsets and ordinals
 * in d_records are local to the scanned range; part says how to make them global:
 *   begin/end += byte_base + (offset of the shard in the whole text);
 *   ordinal   += ord_origin of the first shard + the closes of all shards before this one - ord_fix. */
typedef struct agb_shard_part { uint64_t closes; int64_t ord_fix, ord_origin, byte_base; int32_t virt, pad; } agb_shard_part;
/* The sharded scans refuse a pattern of delim_kind 3 with AGB_ERR_PATTERN: a rank would need the delimiter's state at
 * the start of its shard, which the halos cannot give. */
int  agb_scan_shard_local(const agb_pattern *p, const void *d_shard, uint64_t n_local, uint64_t halo_left, uint64_t halo_right,
                          int first, int open_end, int reaches_end, int want, agb_record *d_records, uint64_t capacity,
                          void *stream, agb_result *res, agb_shard_part *part);
/* the -B sweep over the sharded text: the level histograms are summed over the ranks (they ride in the header), every rank
 * keeps the records of the best level of the WHOLE text, then the gather */
int  agb_bestmatch_sharded(const char *pattern, const agb_options *opt, agb_comm *c, const void *d_shard, uint64_t n_local,
                           uint64_t global_offset, agb_record *d_records, uint64_t capacity, void *stream,
                           int *best_k, agb_result *res, char *err, size_t errlen);

/* j of every record in `records` (ordered, as returned by a scan of h_text[0..n)): the number of record closes
 * up to and including its own (bitap.c:178), with the file-starts-with-the-delimiter correction of bitap.c:151-156.
 * A host walk over the delimiters, only needed for -n. */
void agb_fill_ordinals(const agb_pattern *p, const void *h_text, uint64_t n, agb_record *records, uint64_t n_records);

/* the -B sweep of agrep.c:3582-3728 in one pass for every best level up to 2 (at most three: k = 2, 4, 8; a regular
 * expression is refused with AGB_ERR_PATTERN and a message -- its levels come from an AGB_WANT_LEVELS scan, which the
 * command line runs at k = 2 and then 4): best_k =
 * smallest level 0..min(M-1,8) at which a record matches (-1: none), res->n_matched = the records at that level (the
 * reference's "N words match within K errors"), d_records[0..res->n_records) = their ordered list (what the final
 * printing pass, agrep.c:3673-3726, prints); capacity 0: count only */
int  agb_bestmatch_device(const char *pattern, const agb_options *opt, const void *d_text, uint64_t n,
                          void *stream, agb_record *d_records, uint64_t capacity, int *best_k, agb_result *res,
                          char *err, size_t errlen);

/* ---- synthetic corpus (bench / tests): deterministic, identical on host and device ---- */
typedef struct agb_corpus_spec {
	uint64_t seed;
	uint64_t n_bytes;          /* multiple of 4096                                            */
	uint64_t first_page;       /* page index of byte 0 (sharding)                             */
	int32_t  paragraphs;       /* 1: blank line every 3..8 lines                              */
	int32_t  needle_every;     /* a planted line every this many pages (0 = none)             */
	char     needle[64];       /* the pattern to plant, edited 0..needle_maxedits times       */
	int32_t  needle_maxedits;
	int32_t  pad;
} agb_corpus_spec;
int  agb_corpus_fill_device(const agb_corpus_spec *s, void *d_text, void *stream);
int  agb_corpus_fill_host(const agb_corpus_spec *s, void *h_text);

/* ---- misc ---- */
const char *agb_last_error(void);
int  agb_device_count(void);
int  agb_set_device(int dev);
const char *agb_version(void);
void agb_shutdown(void);              /* frees the library's per-device scratch (scans of different devices run side by side; one at a time per device) */
uint64_t agb_kernel_launches(void);   /* kernels this process launched through the library so far */

#ifdef __cplusplus
}
#endif
#endif
