/* agrep_b200/csrc/dropin.c -- the drop-in layer: the reference's own entry points over the H100 engine.
 *
 * Exports, with the reference's exact (K&R) signatures:
 *     bitap()    bitap.c:78      asearch()  asearch.c:32     asearch0() asearch.c:574
 *     asearch1() asearch1.c:28   sgrep()    sgrep.c:262
 *     fill_buf() bitap.c:450     alloc_buf() bitap.c:484     free_buf() bitap.c:496
 * and reads/writes the reference's globals exactly where those functions do (agrep.c:113-140), so the
 * reference's exec() (agrep.c:3332) and everything above it link against libagrepb200_dropin.so instead of
 * bitap.o asearch.o asearch1.o sgrep.o with no source change (INTEGRATION.md shows the link line).
 *
 * What happens per call: the globals maskgen() left behind become an agb_desc; the text goes to HBM and through
 * the CUDA stages; the ordered record list that comes back is replayed through the reference's own output()
 * (agrep.c:3805), which keeps every formatting switch (-n -b -h -l -c -s ...) byte-identical.  Regular
 * expressions that the reference gives to re() (at most SHORTREG positions, bitap.c:105-106) run on the engine as
 * well -- the descriptor and follow sets from Mask[], NO_ERR_MASK, HEAD/TAIL and table[][] -- and are replayed
 * through the reference's r_output() (agrep.c:1919); longer ones keep going to the reference's re1() (agrep.c:468).
 *
 * How the text gets there (the fill_buf() loop of bitap.c:143,450-477 replaced):
 *   - a regular file is never slurped: it is read(2) straight into the engine's pinned ring and on to the device
 *     (agb_text_from_fd / agb_scan_fd); offsets are 64-bit all the way, the reference's `int` only appears at the
 *     output() call, which gets a small buffer holding just that record (pread) and indexes relative to it;
 *   - the device copy is kept for the next call on the same file (same device, inode, size and mtime): exec() scans
 *     every file K + 2 times under -B (agrep.c:3582-3728), which then costs one upload, not K + 2;
 *   - under -B the counting passes D = 1, 2, ... are answered from ONE device pass that takes every record's
 *     smallest level (the rows are nested, asearch.c:98-114), and the final printing pass from the list that pass left;
 *     for a re() pattern the counting passes come from levels passes at k = 2 and 4 (regex_bestmatch_count);
 *   - pipes, and memory mode (fd == -1, agrep.c:3282), go through a host buffer.
 */
#define _GNU_SOURCE
#include "agrep_b200.h"
#include "agrep_b200_dropin.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <errno.h>
#include <unistd.h>
#include <sys/stat.h>
#include <sys/types.h>

#define AGREP_ERROR 123        /* agrep.h:173 */
#define SHORTREG 15            /* agrep.h:36  */

/* ---- the reference's globals (defined in agrep.c) ---- */
extern unsigned Mask[], Init1, NO_ERR_MASK, Init[], endposition, D_endpos, wildmask;
extern int AND, INVERSE, DELIMITER, D_length, I, S, DD, JUMP, REGEX, COUNT, FILENAMEONLY, SILENT;
extern int LIMITOUTPUT, LIMITPERFILE, NEW_FILE, POST_FILTER, num_of_matched, prev_num_of_matched;
extern int CurrentByteOffset, TRUNCATE, NOUPPER, WORDBOUND, WHOLELINE, LINENUM, OUTTAIL, BESTMATCH;
extern int FNAME, BYTECOUNT, PRINTOFFSET, PRINTRECORD;
extern unsigned char LUT[256];
extern char CurrentFileName[], D_pattern[], Progname[];
extern int agrep_inlen, agrep_outlen, agrep_outpointer;
extern unsigned char *agrep_inbuffer, *agrep_outbuffer;
extern FILE *agrep_finalfp;
extern int glimpse_clientdied;
extern int output();           /* agrep.c:3805 */
extern int r_output();         /* agrep.c:1919 */
extern int re1();              /* agrep.c:468 */
extern int HEAD, TAIL;         /* preproce.c:231-236, 334-339 */
extern int table[32][32];      /* follow sets of the regex positions, follow.c:210-255 (agrep.c:219, WORD = 32) */

/* ---- fill_buf / alloc_buf / free_buf: same contracts (other reference files, e.g. newmgrep.c and file_out(),
 * keep calling them) ---- */
int fill_buf(int fd, unsigned char *buf, int record_size)
{
	int num_read = 1, total_read = 0;
	if (fd < 0) return 0;                                   /* bitap.c:466 */
	while (total_read < record_size && num_read > 0) {      /* bitap.c:459-463 */
		if (glimpse_clientdied) return 0;
		num_read = (int)read(fd, buf + total_read, (size_t)(record_size - total_read));
		if (num_read > 0) total_read += num_read;
	}
	if (glimpse_clientdied) return 0;
	return total_read;
}
void alloc_buf(int fd, unsigned char **buf, int size) { if (fd != -1) *buf = (unsigned char *)malloc((size_t)size); }
void free_buf(int fd, char *buf) { if (fd != -1) free(buf); }

static int fail(const char *what)
{
	fprintf(stderr, "%s: %s: %s\n", Progname, what, agb_last_error());
	errno = AGREP_ERROR;
	return -1;
}

/* ================================================================================================
 * where the text of a call comes from
 * ============================================================================================== */
typedef struct {
	int kind;                    /* 0: resident device text of a regular file (records are pread from fd); 1: host buffer */
	int fd;
	agb_text *text;              /* kind 0 (owned by the cache below) */
	unsigned char *host;         /* kind 1: host[0..n) */
	int host_owned;
	unsigned long long n;
} source;

/* the device copies of the files scanned last: exec() comes back to the same file for every level of a -B sweep */
#define NCACHE 4
typedef struct {
	int used; dev_t dev; ino_t ino; off_t size; struct timespec mtim; unsigned long stamp;
	agb_text *text;
	/* what one -B pass learned about this file (valid for bm_sig): records per smallest level, the best level's list */
	int bm_valid; unsigned long long bm_sig; unsigned long long bm_hist[AGB_MAXERR + 1]; int bm_best, bm_kdone;
	agb_record *bm_recs; unsigned long long bm_nrecs;
} cache_entry;
static cache_entry g_cache[NCACHE];
static unsigned long g_stamp;

static void cache_drop(cache_entry *e)
{
	if (e->text) agb_text_free(e->text);
	free(e->bm_recs);
	memset(e, 0, sizeof *e);
}

static cache_entry *cache_get(int fd)
{
	struct stat sb; int i; cache_entry *victim = &g_cache[0];
	if (fstat(fd, &sb) != 0 || !S_ISREG(sb.st_mode) || lseek(fd, 0, SEEK_CUR) != 0) return NULL;
	for (i = 0; i < NCACHE; i++) {
		cache_entry *e = &g_cache[i];
		if (e->used && e->dev == sb.st_dev && e->ino == sb.st_ino && e->size == sb.st_size &&
		    e->mtim.tv_sec == sb.st_mtim.tv_sec && e->mtim.tv_nsec == sb.st_mtim.tv_nsec) { e->stamp = ++g_stamp; return e; }
	}
	for (i = 0; i < NCACHE; i++) { if (!g_cache[i].used) { victim = &g_cache[i]; break; } if (g_cache[i].stamp < victim->stamp) victim = &g_cache[i]; }
	cache_drop(victim);
	if (agb_text_from_fd(fd, &victim->text) != AGB_OK) return NULL;
	victim->used = 1; victim->dev = sb.st_dev; victim->ino = sb.st_ino; victim->size = sb.st_size; victim->mtim = sb.st_mtim; victim->stamp = ++g_stamp;
	return victim;
}

/* pipes and memory mode: everything into one host buffer (memory mode, agrep.c:3282: the caller's leading '\n' is the
 * virtual one of bitap.c:140) */
static int slurp(int fd, source *s)
{
	size_t cap = 1u << 22, n = 0; unsigned char *hb;
	if (fd == -1) {
		size_t len = agrep_inlen > 0 ? (size_t)agrep_inlen : 0, skip = (len && agrep_inbuffer[0] == '\n') ? 1 : 0;
		s->kind = 1; s->host = agrep_inbuffer + skip; s->host_owned = 0; s->n = len - skip; s->fd = -1;
		return 0;
	}
	hb = (unsigned char *)malloc(cap);
	if (!hb) return -1;
	for (;;) {
		ssize_t r;
		if (n == cap) { unsigned char *nb; cap *= 2; nb = (unsigned char *)realloc(hb, cap); if (!nb) { free(hb); return -1; } hb = nb; }
		r = read(fd, hb + n, cap - n);
		if (r <= 0) break;
		n += (size_t)r;
	}
	s->kind = 1; s->host = hb; s->host_owned = 1; s->n = n; s->fd = fd;
	return 0;
}

static cache_entry *source_open(int fd, source *s)
{
	cache_entry *e = fd >= 0 ? cache_get(fd) : NULL;
	memset(s, 0, sizeof *s);
	if (e) { s->kind = 0; s->fd = fd; s->text = e->text; s->n = agb_text_size(e->text); return e; }
	if (slurp(fd, s)) { s->kind = -1; }
	return NULL;
}
static void source_close(source *s) { if (s->kind == 1 && s->host_owned) free(s->host); }

static int source_scan(const agb_pattern *p, const source *s, int want, agb_record *recs, unsigned long long cap, agb_result *res)
{
	if (s->kind == 0) return agb_scan_text(p, s->text, want, recs, cap, res);
	return agb_scan_host(p, s->host, s->n, want, recs, cap, res);
}

/* a scan that wants the record list: the list is sized from a guess and, when the scan reports more matching records
 * than fit (agb_result.truncated), once more with exactly n_matched entries -- an empty record is a record too, so no
 * bound short of one entry per text byte is safe up front (the reference prints blank lines under -v) */
static int scan_records(const agb_pattern *p, const source *s, int want, agb_record **recs, agb_result *res)
{
	unsigned long long cap = s->n / 64 + 65536; int rc;
	for (;;) {
		agb_record *r = (agb_record *)realloc(*recs, (size_t)cap * sizeof **recs);
		if (!r) return AGB_ERR_NOMEM;
		*recs = r;
		rc = source_scan(p, s, want | AGB_WANT_RECORDS, r, cap, res);
		if (rc || !res->truncated) return rc;
		cap = res->n_matched;
	}
}

/* the bytes output() may look at for one record, in a buffer of their own: [begin, end + L) of the text -- index 0 =
 * file offset `begin` (the virtual '\n' of bitap.c:140 for begin = -1), the delimiter appended behind the text
 * (bitap.c:161-165) where the file has ended.  Returns the buffer (grown as needed) or NULL. */
static unsigned char *record_bytes(const source *s, const agb_record *r, const unsigned char *dpat, int L,
                                   unsigned char **buf, size_t *bufcap)
{
	const long long b = r->begin, e = r->end + L;              /* [b, e) */
	const size_t len = (size_t)(e - b);
	long long q = b; size_t at = 0;
	if (len + 8 > *bufcap) { unsigned char *nb = (unsigned char *)realloc(*buf, len + 4096); if (!nb) return NULL; *buf = nb; *bufcap = len + 4096; }
	if (q < 0) { (*buf)[at++] = '\n'; q = 0; }
	if (q < (long long)s->n && q < e) {
		const size_t want = (size_t)((e < (long long)s->n ? e : (long long)s->n) - q);
		if (s->kind == 1) memcpy(*buf + at, s->host + q, want);
		else {
			size_t got = 0;
			while (got < want) {
				ssize_t rd = pread(s->fd, *buf + at + got, want - got, (off_t)(q + (long long)got));
				if (rd <= 0) return NULL;
				got += (size_t)rd;
			}
		}
		at += want; q += (long long)want;
	}
	while (q < e) { (*buf)[at++] = dpat[q - (long long)s->n < L ? q - (long long)s->n : L - 1]; q++; }
	(*buf)[at] = 0;
	return *buf;
}

/* The anchor plan (stage 1 / 1.5 of the device scan) from the reference's INTERNAL pattern string, i.e. what
 * preprocess() hands to maskgen() and bitap() (preproce.c:221-341; symbols agrep.h:69-87): positions are counted
 * exactly as maskgen() counts them, literal runs are cut into k+1 disjoint anchors of 4 (3, 2) bytes.  Only for a
 * single pattern part without '#', not under -v or -p -- otherwise every chunk goes to the record stage. */
enum { S_HYPHEN = 129, S_NOCARE = 130, S_NNLINE = 131, S_WORDB = 133, S_LPAREN = 134, S_RPAREN = 135, S_LRANGE = 136,
       S_RRANGE = 137, S_LANGLE = 138, S_RANGLE = 139, S_NOT = 140, S_WILD = 141, S_ORSYM = 142, S_ORPAT = 143,
       S_ANDPAT = 144, S_STAR = 145 };

static void plan_from_internal(const unsigned char *P, int L, int D, agb_desc *d)
{
	int lit[80], n = 0, i, seps = 0, A, plen = (int)strlen((const char *)P);
	d->plan = AGB_PLAN_ALL; d->n_anchors = 0; d->refine = 0; d->n_anchors3 = 0; d->adaptive = 1;
	if (INVERSE || I == 0 || wildmask) return;
	for (i = 0; i < plen && n < 70; i++) {
		int c = P[i];
		if (c == S_LANGLE || c == S_RANGLE || c == S_LPAREN || c == S_RPAREN || c == S_STAR || c == S_ORSYM) continue;
		if (c == S_WILD) return;
		if (c == S_ORPAT || c == S_ANDPAT) { if (++seps > 1) return; lit[++n] = -1; continue; }
		if (c == S_LRANGE) { while (i < plen && P[i] != S_RRANGE) i++; lit[++n] = -1; continue; }
		if (c == '\n' || c >= 128) { lit[++n] = -1; continue; }                 /* newline, WORDB, NNLINE, NOCARE: a position, not a literal */
		lit[++n] = NOUPPER && c >= 'A' && c <= 'Z' ? c + 32 : c;
		/* (bytes >= 128 were excluded above: under -i the exact engine folds them through LUT[], bitap.c:171) */
	}
	if (n != d->M) return;                                                          /* our count must agree with maskgen's */
	for (A = 4; A >= 2; A--) {
		int got = 0, run = 0, p;
		for (p = L + 2; p <= n && got < D + 1; p++) {
			if (lit[p] < 0) { run = 0; continue; }
			if (++run == A) {
				uint32_t v = 0; int t;
				for (t = 0; t < A; t++) v |= (uint32_t)lit[p - A + 1 + t] << (8 * t);
				d->anchor[got] = v; d->anchor_off[got] = p - A + 1 - (L + 2); got++; run = 0;
			}
		}
		if (got < D + 1) continue;
		d->plan = AGB_PLAN_ANCHORS; d->n_anchors = D + 1; d->anchor_len = A;
		d->anchor_mask = A == 4 ? 0xFFFFFFFFu : (A == 3 ? 0x00FFFFFFu : 0x0000FFFFu);
		d->anchor_fold = NOUPPER ? 0x20202020u : 0;
		for (p = 0; p < d->n_anchors; p++) d->anchor[p] = (d->anchor[p] | d->anchor_fold) & d->anchor_mask;
		d->pat_len = n - L - 1; d->refine = 1;
		return;
	}
}

/* the scan descriptor from the globals maskgen() left behind, for error level D and the given engine */
static int desc_from_globals(agb_desc *d, const unsigned char *dpat, int L, const unsigned char *Pattern, int M, int D, int engine)
{
	const uint64_t HI = 0xFFFFFFFF00000000ull; int c;
	memset(d, 0, sizeof *d);
	for (c = 0; c < 256; c++) d->mask[c] = Mask[engine == AGB_ENGINE_BITAP ? LUT[c] : c];   /* bitap.c:171 vs asearch.c:96 */
	d->init0 = HI | Init[0]; d->init1 = HI | Init1; d->noerr = HI | NO_ERR_MASK;
	d->endpos = endposition; d->dendpos = D_endpos; d->wildmask = wildmask;
	d->dmask = 0;
	for (c = 0; c < L; c++) d->dmask |= (uint64_t)D_endpos << c;             /* bitap.c:131-133 */
	d->dmask = ~d->dmask;
	d->M = M; d->L = L; memcpy(d->delim, dpat, (size_t)L);
	d->k = D; d->engine = engine; d->and_mode = AND; d->inverse = INVERSE; d->user_delim = DELIMITER; d->outtail = OUTTAIL;
	d->cost_i = I > D ? D + 1 : I; d->cost_s = S > D ? D + 1 : S; d->cost_d = DD > D ? D + 1 : DD;   /* asearch1.c:42-44 */
	if (d->cost_i < 1) d->cost_i = 1;
	if (Pattern) plan_from_internal(Pattern, L, D, d);
	d->sticky_delim = 1;                                                      /* -p (I = 0) with a delimiter of two or more bytes */
	return 0;
}

/* what identifies "the same query" for the -B memo of a file: the automaton words and the options that shape them */
static unsigned long long bm_signature(int M, int L)
{
	unsigned long long h = 1469598103934665603ull; int c;
#define MIX(x) do { h ^= (unsigned long long)(x); h *= 1099511628211ull; } while (0)
	for (c = 0; c < 256; c++) MIX(Mask[c]);
	MIX(Init[0]); MIX(Init1); MIX(NO_ERR_MASK); MIX(endposition); MIX(D_endpos); MIX(wildmask); MIX(M); MIX(L);
	MIX(AND); MIX(INVERSE); MIX(DELIMITER); MIX(I); MIX(S); MIX(DD);
#undef MIX
	return h;
}

/* -B, counting passes (agrep.c:3591-3630: COUNT on, D = 1, 2, ... until something matches): the number of records
 * that match within D errors, from ONE device pass per file at a level k >= D that takes every record's smallest level.
 * Passes run at k = 2, 4, 8 (capped by M - 1): the anchor filter is still selective at the small levels. */
static int bestmatch_count(cache_entry *e, const source *s, const unsigned char *dpat, int L, const unsigned char *Pattern,
                           int M, int D, unsigned long long *count)
{
	const unsigned long long sig = bm_signature(M, L);
	int l;
	if (!e->bm_valid || e->bm_sig != sig) { e->bm_valid = 1; e->bm_sig = sig; e->bm_kdone = 0; e->bm_best = -1; memset(e->bm_hist, 0, sizeof e->bm_hist); free(e->bm_recs); e->bm_recs = NULL; e->bm_nrecs = 0; }
	while (e->bm_kdone < D) {
		agb_desc d; agb_pattern *p = NULL; agb_result res; agb_record *recs = NULL; char err[256]; int rc, k;
		k = e->bm_kdone < 2 ? 2 : (e->bm_kdone < 4 ? 4 : AGB_MAXERR);
		if (k > M - 1) k = M - 1;
		if (k > AGB_MAXERR) k = AGB_MAXERR;
		if (k < D) k = D;
		desc_from_globals(&d, dpat, L, Pattern, M, k, k > 4 ? AGB_ENGINE_ASEARCH0 : AGB_ENGINE_ASEARCH);
		rc = agb_pattern_from_desc(&d, &p, err, sizeof err);
		if (rc) { fprintf(stderr, "%s: %s\n", Progname, err); errno = AGREP_ERROR; return -1; }
		rc = scan_records(p, s, AGB_WANT_LEVELS | (LINENUM ? AGB_WANT_ORDINALS : 0), &recs, &res);
		agb_pattern_free(p);
		if (rc) { free(recs); return fail("scan"); }
		for (l = e->bm_kdone + 1; l <= k; l++) e->bm_hist[l] = res.level_hist[l];
		if (e->bm_best < 0) for (l = 1; l <= k; l++) if (e->bm_hist[l]) { e->bm_best = l; break; }
		if (e->bm_best > 0 && !e->bm_recs) {
			/* keep the best level's records: the printing pass (agrep.c:3673-3726) asks for exactly these */
			unsigned long long i, m = 0;
			for (i = 0; i < res.n_records; i++) if (recs[i].level == e->bm_best) recs[m++] = recs[i];
			e->bm_recs = recs; e->bm_nrecs = m; recs = NULL;
		}
		free(recs);
		e->bm_kdone = k;
	}
	*count = 0;
	for (l = 0; l <= D && l <= AGB_MAXERR; l++) *count += e->bm_hist[l];
	return 0;
}

/* one record through the reference's own output() (bitap.c:212-214); returns -1 on its error, 1 when a limit says stop */
static int replay_record(const source *s, const agb_record *r, const unsigned char *dpat, int L, unsigned char **buf, size_t *bufcap)
{
	unsigned char *rb = record_bytes(s, r, dpat, L, buf, bufcap);
	if (!rb) { errno = AGREP_ERROR; return -1; }
	/* CurrentByteOffset as the loop leaves it at the output() call (bitap.c:172,179): bytes consumed minus the delimiter */
	CurrentByteOffset = (int)(r->end + 1);
	TRUNCATE = 0;
	/* output(buffer, lasti, print_end, j): index 0 of rb is the text's `begin`, which the reference's buffer holds at lasti */
	if (-1 == output(rb, 0, (int)(r->end - r->begin - 1), (int)r->ordinal)) return -1;
	if ((LIMITOUTPUT > 0 && LIMITOUTPUT <= num_of_matched) ||
	    (LIMITPERFILE > 0 && LIMITPERFILE <= num_of_matched - prev_num_of_matched)) return 1;     /* bitap.c:215-219 */
	return 0;
}

/* the common tail of bitap()/asearch*(): desc from the globals, scan, replay through output() */
static int scan_and_replay(char old_D_pat[], const unsigned char *Pattern, int fd, int M, int D, int engine)
{
	agb_desc d; agb_pattern *p = NULL; agb_result res; agb_record *recs = NULL, *list; source src; cache_entry *ce;
	unsigned char dpat[2 * AGB_MAXDELIM + 2], *rbuf = NULL; size_t rcap = 0; unsigned long long i, nlist; int L, c, rc, ret = 0;
	char err[256];

	L = (int)strlen(old_D_pat);
	if (L < 1 || L > AGB_MAXDELIM) { fprintf(stderr, "%s: delimiter pattern too long\n", Progname); errno = AGREP_ERROR; return -1; }
	for (c = 0; c < L; c++) {                               /* bitap.c:92-94 */
		if (old_D_pat[c] == '^' || old_D_pat[c] == '$') old_D_pat[c] = '\n';
		dpat[c] = (unsigned char)old_D_pat[c];
	}
	D_length = L;
	if (I == 0) Init1 = 037777777777u;                      /* bitap.c:123, asearch.c:49, asearch1.c:41 */

	ce = source_open(fd, &src);
	if (src.kind < 0) { fprintf(stderr, "%s: out of memory\n", Progname); errno = AGREP_ERROR; return -1; }

	if (BESTMATCH && COUNT && !FILENAMEONLY && D >= 1 && ce && engine != AGB_ENGINE_ASEARCH1 && !INVERSE) {
		/* a counting pass of the -B sweep: answered from the level histogram of this file */
		unsigned long long cnt = 0;
		if (bestmatch_count(ce, &src, dpat, L, Pattern, M, D, &cnt)) ret = -1;
		else num_of_matched += (int)cnt;
		source_close(&src);
		return ret;
	}

	desc_from_globals(&d, dpat, L, Pattern, M, D, engine);
	rc = agb_pattern_from_desc(&d, &p, err, sizeof err);
	if (rc) { source_close(&src); fprintf(stderr, "%s: %s\n", Progname, err); errno = AGREP_ERROR; return -1; }

	if (COUNT && !FILENAMEONLY && fd != -1) {               /* output() would only count (agrep.c:3812-3813) */
		rc = source_scan(p, &src, AGB_WANT_COUNT, NULL, 0, &res);
		if (rc) ret = fail("scan");
		else num_of_matched += (int)res.n_matched;
		goto done;
	}
	if (BESTMATCH && !COUNT && D >= 1 && ce && ce->bm_valid && ce->bm_sig == bm_signature(M, L) && ce->bm_best == D && ce->bm_recs && !INVERSE) {
		/* the printing pass of the -B sweep (agrep.c:3673-3726): the list the counting pass left */
		list = ce->bm_recs; nlist = ce->bm_nrecs;
	} else {
		rc = scan_records(p, &src, LINENUM ? AGB_WANT_ORDINALS : 0, &recs, &res);   /* j for output() (-n) on the device */
		if (rc) { ret = fail("scan"); goto done; }
		list = recs; nlist = res.n_records;
	}
	for (i = 0; i < nlist; i++) {
		if (fd == -1 && list[i].end >= (long long)src.n) continue;      /* memory mode appends no delimiter (bitap.c:310-314) */
		if (COUNT && !FILENAMEONLY) { num_of_matched++; continue; } /* (memory mode: the count leaves that last record out too) */
		if (FILENAMEONLY && (NEW_FILE || !POST_FILTER)) {       /* bitap.c:184-210 */
			num_of_matched++;
			if (agrep_finalfp != NULL) fprintf(agrep_finalfp, "%s\n", CurrentFileName);
			else {
				size_t fl = strlen(CurrentFileName);
				if (agrep_outpointer + (int)fl + 1 >= agrep_outlen) { ret = -1; break; }
				memcpy(agrep_outbuffer + agrep_outpointer, CurrentFileName, fl);
				agrep_outbuffer[agrep_outpointer + fl] = '\n';
				agrep_outpointer += (int)fl + 1;
			}
			NEW_FILE = 0;
			break;
		}
		rc = replay_record(&src, &list[i], dpat, L, &rbuf, &rcap);
		if (rc < 0) { ret = -1; break; }
		if (rc > 0) break;
	}
done:
	free(recs); free(rbuf); source_close(&src); agb_pattern_free(p);
	return ret;
}

/* re() (agrep.c:1267-1917) on the engine.  The words are the reference's: Mask[] and NO_ERR_MASK as maskgen() left them
 * (position p at bit M - p, as in agb_desc), Init[0] = Bit[base] | (HEAD ? Bit[base+1] : 0) (agrep.c:1285-1286), and the
 * follow sets read from table[][] the way compute_next() reads them (agrep.c:405-415): positions 1 .. M-1, at most ten
 * entries each -- the reference's cap is kept on purpose here, the goal being its own output (SURVEY 8c).  Each matching
 * line goes through the reference's r_output() in a buffer of its own: '\n', the line, its newline. */
static void regex_follow(int M, agb_regex *rx)
{
	int q, j;
	memset(rx, 0, sizeof *rx);
	rx->follow[0] = 1ull << (M - 1);                         /* compute_next's constant k >> 1: the start feed */
	for (q = 1; q < M; q++)
		for (j = 0; j < 10 && table[q][j] > 0; j++) rx->follow[q] |= 1ull << (M - table[q][j]);
	rx->head = HEAD; rx->tail = TAIL;
}

/* re()'s pattern at D errors from the globals; prints the error and returns -1 when the engine refuses it */
static int regex_pattern(int M, int D, agb_pattern **p)
{
	agb_desc d; agb_regex rx; char err[256]; int c;
	memset(&d, 0, sizeof d);
	for (c = 0; c < 256; c++) d.mask[c] = Mask[c];
	d.noerr = NO_ERR_MASK;
	d.init0 = (1ull << M) | (HEAD ? 1ull << (M - 1) : 0);
	d.init1 = d.init0 | 1;
	d.endpos = 1; d.dmask = ~0ull;
	d.M = M; d.L = 1; d.delim[0] = '\n'; d.k = D; d.engine = AGB_ENGINE_REGEX; d.inverse = INVERSE;
	d.cost_i = d.cost_s = d.cost_d = 1;
	regex_follow(M, &rx);
	if (agb_pattern_from_regex(&d, &rx, p, err, sizeof err)) { fprintf(stderr, "%s: %s\n", Progname, err); errno = AGREP_ERROR; return -1; }
	return 0;
}

/* the -B memo key of a re() query: the words and follow sets regex_pattern() reads (-v never reaches the memo) */
static unsigned long long bm_regex_signature(int M)
{
	unsigned long long h = 1469598103934665603ull; agb_regex rx; int c, q;
#define MIX(x) do { h ^= (unsigned long long)(x); h *= 1099511628211ull; } while (0)
	MIX(AGB_ENGINE_REGEX);
	for (c = 0; c < 256; c++) MIX(Mask[c]);
	MIX(NO_ERR_MASK); MIX(HEAD); MIX(TAIL); MIX(M);
	regex_follow(M, &rx);
	for (q = 0; q < M; q++) MIX(rx.follow[q]);
#undef MIX
	return h;
}

/* -B, the counting passes of a re() pattern (agrep.c:3591-3630, D = 1, 2, ... <= 4): the lines that match within D
 * errors, from the file's memo of smallest levels.  re()'s rows are nested, so a levels pass at k = 2 answers D <= 2 and
 * one at k = 4 the rest; each runs only when a D needs it. */
static int regex_bestmatch_count(cache_entry *e, const source *s, int M, int D, unsigned long long *count)
{
	const unsigned long long sig = bm_regex_signature(M);
	int l;
	if (!e->bm_valid || e->bm_sig != sig) { e->bm_valid = 1; e->bm_sig = sig; e->bm_kdone = -1; e->bm_best = -1; memset(e->bm_hist, 0, sizeof e->bm_hist); free(e->bm_recs); e->bm_recs = NULL; e->bm_nrecs = 0; }
	while (e->bm_kdone < D) {
		agb_pattern *p = NULL; agb_result res; int rc, k = e->bm_kdone < 2 ? 2 : 4;
		if (k < D) k = D;
		if (regex_pattern(M, k, &p)) return -1;
		rc = source_scan(p, s, AGB_WANT_LEVELS, NULL, 0, &res);
		agb_pattern_free(p);
		if (rc) return fail("scan");
		for (l = e->bm_kdone + 1; l <= k; l++) e->bm_hist[l] = res.level_hist[l];
		e->bm_kdone = k;
	}
	*count = 0;
	for (l = 0; l <= D; l++) *count += e->bm_hist[l];
	return 0;
}

static int regex_scan(int fd, int M, int D)
{
	agb_pattern *p = NULL; agb_result res; agb_record *recs = NULL; source src; cache_entry *ce;
	unsigned char *buf = NULL; size_t bufcap = 0; unsigned long long i; int rc, ret = 0;
	const unsigned char nl = '\n';
	if (regex_pattern(M, D, &p)) return -1;
	ce = source_open(fd, &src);
	if (src.kind < 0) { agb_pattern_free(p); fprintf(stderr, "%s: out of memory\n", Progname); errno = AGREP_ERROR; return -1; }
	if (BESTMATCH && COUNT && !FILENAMEONLY && D >= 1 && ce && !INVERSE) {
		/* a counting pass of the -B sweep: answered from the levels memo of this file */
		unsigned long long cnt = 0;
		if (regex_bestmatch_count(ce, &src, M, D, &cnt)) ret = -1;
		else num_of_matched += (int)cnt;
		goto done;
	}
	if (COUNT && !FILENAMEONLY && fd != -1) {               /* r_output() would only count (agrep.c:1926-1927) */
		rc = source_scan(p, &src, AGB_WANT_COUNT, NULL, 0, &res);
		if (rc) ret = fail("scan");
		else num_of_matched += (int)res.n_matched;
		goto done;
	}
	rc = scan_records(p, &src, AGB_WANT_ORDINALS, &recs, &res);
	if (rc) { ret = fail("scan"); goto done; }
	for (i = 0; i < res.n_records; i++) {
		const agb_record *r = &recs[i];
		if (fd == -1 && r->end >= (long long)src.n) continue;     /* memory mode appends no newline */
		if (FILENAMEONLY && (NEW_FILE || !POST_FILTER)) {           /* agrep.c:1334-1356 */
			num_of_matched++;
			if (agrep_finalfp != NULL) fprintf(agrep_finalfp, "%s\n", CurrentFileName);
			else {
				size_t fl = strlen(CurrentFileName);
				if (agrep_outpointer + (int)fl + 1 >= agrep_outlen) { ret = -1; break; }
				memcpy(agrep_outbuffer + agrep_outpointer, CurrentFileName, fl);
				agrep_outbuffer[agrep_outpointer + fl] = '\n';
				agrep_outpointer += (int)fl + 1;
			}
			NEW_FILE = 0;
			break;
		}
		{
			/* record_bytes() gives [begin, end + 1): the opening newline (virtual for the first line), the line, its newline */
			unsigned char *rb = record_bytes(&src, r, &nl, 1, &buf, &bufcap);
			const int at = (int)(r->end - r->begin);            /* index of the closing newline */
			if (!rb) { ret = -1; errno = AGREP_ERROR; break; }
			rb[0] = '\n';
			CurrentByteOffset = (int)r->end;                    /* where re() leaves it at the newline (agrep.c:1329-1331) */
			if (-1 == r_output(rb, at, at + 1, (int)r->ordinal)) { ret = -1; break; }
		}
		if ((LIMITOUTPUT > 0 && LIMITOUTPUT <= num_of_matched) ||
		    (LIMITPERFILE > 0 && LIMITPERFILE <= num_of_matched - prev_num_of_matched)) break;     /* agrep.c:1359-1363 */
	}
done:
	free(recs); free(buf); source_close(&src); agb_pattern_free(p);
	return ret;
}

int bitap(char old_D_pat[], char *Pattern, int fd, int M, int D)
{
	if (REGEX) {                                            /* bitap.c:96-111 */
		if (D > 4) { fprintf(stderr, "%s: the maximum number of erorrs allowed for full regular expressions is 4\n", Progname); errno = AGREP_ERROR; return -1; }
		D_length = (int)strlen(old_D_pat);
		/* re1() (16-30 positions) prints wrong line numbers and misses matches with errors (SURVEY 8c): the reference's
		 * own output for those is its re1()'s, so it keeps running it */
		return M <= SHORTREG ? regex_scan(fd, M, D) : re1(fd, M, D);
	}
	if (D > 0 && JUMP == 1) return scan_and_replay(old_D_pat, (const unsigned char *)Pattern, fd, M, D, AGB_ENGINE_ASEARCH1);   /* bitap.c:113-116 */
	if (D > 4) return scan_and_replay(old_D_pat, (const unsigned char *)Pattern, fd, M, D, AGB_ENGINE_ASEARCH0);               /* asearch.c:50-52 */
	if (D > 0) return scan_and_replay(old_D_pat, (const unsigned char *)Pattern, fd, M, D, AGB_ENGINE_ASEARCH);                /* bitap.c:118-121 */
	return scan_and_replay(old_D_pat, (const unsigned char *)Pattern, fd, M, D, AGB_ENGINE_BITAP);
}

/* M is not a parameter of these three in the reference; it is recovered from the always-on bits of Init[0] */
static int positions_from_init0(void)
{
	unsigned v = ~Init[0]; int M = 0;           /* bits >= M of Init[0] are ones (maskgen.c:224) */
	while (v) { M++; v >>= 1; }
	return M;
}
int asearch(unsigned char old_D_pat[], int text, unsigned D)
{ return scan_and_replay((char *)old_D_pat, NULL, text, positions_from_init0(), (int)D, D > 4 ? AGB_ENGINE_ASEARCH0 : AGB_ENGINE_ASEARCH); }
int asearch0(unsigned char old_D_pat[], int text, unsigned D)
{ return scan_and_replay((char *)old_D_pat, NULL, text, positions_from_init0(), (int)D, AGB_ENGINE_ASEARCH0); }
int asearch1(char old_D_pat[], int Text, unsigned D)
{ return scan_and_replay(old_D_pat, NULL, Text, positions_from_init0(), (int)D, AGB_ENGINE_ASEARCH1); }

/* sgrep(): simple patterns (checksg.c:138).  k = 0: bm() semantics (ASCII case folded literal, once per record,
 * -w by isalnum neighbours, sgrep.c:741-755), also under -d.  k > 0: the reference runs lossy filters here
 * (SURVEY 8c); we run the exact automaton.  Record printing follows bm()/s_output() (sgrep.c:812-933, 1274-1483). */
int sgrep(unsigned char *in_pat, int in_m, int fd, int D, int samepattern)
{
	agb_options o; agb_pattern *p = NULL; agb_result res; agb_record *recs = NULL; source src;
	char err[256], pat[1024], delim[64]; unsigned char *rbuf = NULL; size_t rcap = 0; unsigned long long i; int rc, ret = 0, L;
	unsigned char dpat[2 * AGB_MAXDELIM + 2];
	(void)samepattern;
	memset(&o, 0, sizeof o);
	if (in_m < 1 || in_m >= (int)sizeof pat) { errno = AGREP_ERROR; return -1; }
	memcpy(pat, in_pat, (size_t)in_m); pat[in_m] = 0;
	o.k = D; o.wordbound = WORDBOUND; o.wholeline = WHOLELINE; o.inverse = (INVERSE && !COUNT) ? 1 : 0; o.nocase = NOUPPER;
	o.wide_approx = 1;                                                         /* up to 255 characters at k > 0 too (sgrep.c:303) */
	if (DELIMITER) {
		/* D_pattern holds the delimiter bytes themselves here (agrep.c:3182-3185); re-escape for agb_compile */
		int q = 0, t;
		for (t = 0; t < D_length && q + 2 < (int)sizeof delim; t++) { delim[q++] = '\\'; delim[q++] = D_pattern[t]; }
		delim[q] = 0; o.delim = delim;
	}
	rc = agb_compile(pat, &o, &p, err, sizeof err);
	if (rc) { fprintf(stderr, "%s: %s\n", Progname, err); errno = AGREP_ERROR; return -1; }
	L = agb_pattern_desc(p)->L; memcpy(dpat, agb_pattern_desc(p)->delim, (size_t)L);
	source_open(fd, &src);
	if (src.kind < 0) { agb_pattern_free(p); errno = AGREP_ERROR; return -1; }
	if (COUNT || SILENT || (FILENAMEONLY && !INVERSE)) {
		/* bm() only counts matching records here, also under -v (sgrep.c:813-815, 968-971) */
		rc = source_scan(p, &src, AGB_WANT_COUNT, NULL, 0, &res);
		if (rc) ret = fail("scan");
		else if (FILENAMEONLY) {
			if (res.n_matched) {
				num_of_matched++;                                       /* bm() returns at the first hit (sgrep.c:813-814) */
				if (NEW_FILE || !POST_FILTER) {                         /* sgrep.c:443-463 */
					if (agrep_finalfp != NULL) fprintf(agrep_finalfp, "%s\n", CurrentFileName);
					NEW_FILE = 0;
				}
			}
		} else num_of_matched += (int)res.n_matched;
		goto done;
	}
	rc = scan_records(p, &src, 0, &recs, &res);
	if (rc) { ret = fail("scan"); goto done; }
	for (i = 0; i < res.n_records; i++) {
		/* bm() prints [curtextbegin, curtextend): the line and its trailing newline (sgrep.c:775-789, 916); with a user
		 * delimiter the record together with the delimiter in FRONT of it, or behind it under -t
		 * (backward_/forward_delimiter(), delim.c:52-117).  rb[x] = text[begin + x]. */
		const int tail = !DELIMITER || OUTTAIL;
		const agb_record *r = &recs[i];
		unsigned char *rb = record_bytes(&src, r, dpat, L, &rbuf, &rcap);
		/* the first record has no delimiter in front of it unless the text starts with one (begin = 0 either way) */
		const int no_lead = r->begin < 0 || (DELIMITER && r->begin == 0 && !(src.n >= (unsigned long long)L && memcmp(rb, dpat, (size_t)L) == 0));
		long long b, e;
		if (!rb) { ret = -1; errno = AGREP_ERROR; break; }
		b = no_lead ? (r->begin < 0 ? 1 : 0) : (tail ? L : 0);                  /* offsets into rb */
		e = (r->end - r->begin) + (tail ? L : 0);
		if (r->end + (tail ? L : 0) > (long long)src.n) e = (long long)src.n - r->begin;
		if (e < b) e = b;
		if (!INVERSE) num_of_matched++;
		if (agrep_finalfp != NULL) {
			if (FNAME && (NEW_FILE || !POST_FILTER)) { fprintf(agrep_finalfp, "%s: ", CurrentFileName); }
			if (BYTECOUNT) fprintf(agrep_finalfp, "%d= ", (int)r->end);
			if (PRINTRECORD) {
				fwrite(rb + b, 1, (size_t)(e - b), agrep_finalfp);
				if (!DELIMITER && r->begin + e == (long long)src.n && src.n && e > b && rb[e - 1] != dpat[L - 1]) fputc('\n', agrep_finalfp);   /* sgrep.c:786-789: newline records only */
			} else if (FNAME || BYTECOUNT) fputc('\n', agrep_finalfp);
		} else {
			if (agrep_outpointer + (int)(e - b) + 1 >= agrep_outlen) { ret = -1; break; }
			memcpy(agrep_outbuffer + agrep_outpointer, rb + b, (size_t)(e - b));
			agrep_outpointer += (int)(e - b);
		}
		if ((LIMITOUTPUT > 0 && LIMITOUTPUT <= num_of_matched) ||
		    (LIMITPERFILE > 0 && LIMITPERFILE <= num_of_matched - prev_num_of_matched)) break;
	}
	if (INVERSE) {
		/* bm() counts the MATCHING records even when it prints the others (sgrep.c:813); keep num_of_matched faithful */
		agb_options o2 = o; agb_pattern *p2 = NULL; agb_result r2;
		o2.inverse = 0;
		if (agb_compile(pat, &o2, &p2, err, sizeof err) == 0) {
			if (source_scan(p2, &src, AGB_WANT_COUNT, NULL, 0, &r2) == 0) num_of_matched += (int)r2.n_matched;
			agb_pattern_free(p2);
		}
	}
done:
	free(recs); free(rbuf); source_close(&src); agb_pattern_free(p);
	return ret;
}
