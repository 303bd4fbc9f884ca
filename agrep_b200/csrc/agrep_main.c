/* agrep_b200/csrc/agrep_main.c -- `agrep-b200`: a small stand-alone command line over libagrepb200.
 *
 * It covers the switches of agrep that reach the scan path (reference agrep.c:2121-2739) and prints what the
 * reference's exec()/output() print for them (agrep.c:3332-3752, 3805-3956): -# -c -i -w -x -v -n -p -I# -S# -D#
 * -d delim -B -y -l -h -s -b -t -V# -e pat, one or more files.  It is NOT the drop-in (that is the reference's
 * own main() linked against libagrepb200_dropin.so, INTEGRATION.md); it exists so the engine can be used
 * where the reference's sources are not around.  Regular expressions (an unescaped '|' or '*') run on the device as
 * re() would (DESIGN.md 3.6).  No -f/-m multi-pattern, no -r (out of scope, DESIGN.md 7).
 */
#include "agrep_b200.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ctype.h>
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>

static const char *prog = "agrep-b200";
static int COUNT, SILENT, FILENAMEONLY, NOFILENAME, LINENUM, BYTECOUNT, BESTMATCH, NOPROMPT, VERBOSE = 1, OUTTAIL;
static int FNAME, num_of_matched, FIRSTOUTPUT = 1, EATFIRST, QUIET_OPEN;

static void usage(void)
{
	fprintf(stderr, "usage: %s [-#cdehilnpstvwxyBDIS] [-d delim] [-e] pattern [files]\n", prog);
	exit(2);
}

/* an unescaped '|' or '*' (preproce.c:139-142) */
static int is_regex(const char *s)
{
	for (; *s; s++) {
		if (*s == '\\') { if (!*++s) break; }
		else if (*s == '|' || *s == '*') return 1;
	}
	return 0;
}

static void cannot_open(const char *path)
{
	if (!QUIET_OPEN) fprintf(stderr, "%s: can't open file for reading: %s\n", prog, path);
}

/* the file with the virtual newline in front and the delimiter behind; NULL with *unopened set when it cannot be opened
 * (the caller says so once the output of the files before it is out) */
static unsigned char *slurp(const char *path, size_t *n, int L, const unsigned char *dpat, int *unopened)
{
	int fd = path ? open(path, O_RDONLY) : 0; struct stat sb; size_t cap, len = 0; unsigned char *b;
	*unopened = fd < 0;
	if (fd < 0) return NULL;
	cap = (fstat(fd, &sb) == 0 && S_ISREG(sb.st_mode)) ? (size_t)sb.st_size + 1 : (1u << 20);
	b = (unsigned char *)malloc(cap + 64);
	if (!b) { if (path) close(fd); return NULL; }
	b[0] = '\n';                                                  /* the virtual newline (bitap.c:140) */
	for (;;) {
		ssize_t r;
		if (len + 1 >= cap) { cap *= 2; b = (unsigned char *)realloc(b, cap + 64); if (!b) return NULL; }
		r = read(fd, b + 1 + len, cap - len - 1);
		if (r <= 0) break;
		len += (size_t)r;
	}
	if (path) close(fd);
	memcpy(b + 1 + len, dpat, (size_t)L);                         /* bitap.c:161-165 */
	*n = len;
	return b;
}

/* output() of the reference, agrep.c:3805-3956, for the switches we carry */
static void print_record(const unsigned char *hb, const agb_desc *d, const agb_record *rec, const char *fname)
{
	long long i1 = rec->begin + 1, i2 = rec->end, j = rec->ordinal; int L = d->L;   /* buffer indexes (lasti, print_end) */
	if (d->engine == AGB_ENGINE_REGEX) {
		/* re() prints through r_output(), agrep.c:1919-: the prefixes, then the line with its newline (no output() quirks) */
		num_of_matched++;
		if (COUNT || SILENT) return;
		if (FNAME) printf("%s: ", fname);
		if (LINENUM) printf("%lld: ", j - 1);
		if (BYTECOUNT) printf("%lld= ", (long long)rec->end);
		fwrite(hb + rec->begin + 2, 1, (size_t)(rec->end - rec->begin), stdout);       /* hb[x + 1] is byte x of the text */
		return;
	}
	if (i1 > i2) return;                                                             /* agrep.c:3811 */
	num_of_matched++;
	if (COUNT || SILENT) return;
	if (OUTTAIL || (!d->user_delim && L == 1 && d->delim[0] == '\n')) { if (j > 1) i1 += L; i2 += L; }   /* agrep.c:3815-3818 */
	if (d->user_delim) j++;                                                          /* agrep.c:3819 */
	if (FIRSTOUTPUT) { if (hb[i1] == '\n') { i1++; EATFIRST = 1; } FIRSTOUTPUT = 0; }  /* agrep.c:3820-3826 */
	while (hb[i1] == '\n' && i1 <= i2) { fputc('\n', stdout); i1++; }                /* agrep.c:3832-3843 */
	if (FNAME) printf("%s: ", fname);
	if (LINENUM) printf("%lld: ", j - 1);
	if (BYTECOUNT) printf("%lld= ", (long long)rec->end);
	if (i1 <= i2) fwrite(hb + i1, 1, (size_t)(i2 - i1 + 1), stdout);
}

/* what exec() does with one file's scan result (agrep.c:3411-3576): the histogram of a levels pass, the count, the records,
 * the -c / -l lines */
static void finish_file(const agb_desc *d, const char *fname, const unsigned char *hb, const agb_result *res, const agb_record *recs,
                        int counting, unsigned long long *hist)
{
	const int before = num_of_matched, count_only = counting || COUNT || SILENT || FILENAMEONLY;
	size_t i;
	if (hist) { for (i = 0; i <= AGB_MAXERR; i++) hist[i] += res->level_hist[i]; }
	else if (FILENAMEONLY && !counting) num_of_matched += res->n_matched ? 1 : 0;   /* the scan stops at the first hit (bitap.c:184-210, sgrep.c:813-814) */
	else if (count_only) num_of_matched += (int)res->n_matched;
	else {
		for (i = 0; i < res->n_records; i++) print_record(hb, d, &recs[i], fname ? fname : "");
	}
	if (!counting) {
		if (COUNT && !FILENAMEONLY) { if (FNAME) printf("%s: %d\n", fname, num_of_matched - before); else printf("%d\n", num_of_matched - before); }   /* agrep.c:3501-3557 */
		if (FILENAMEONLY && num_of_matched > before) printf("%s\n", fname ? fname : "(standard input)");
	}
}

static int scan_want(int counting, const unsigned long long *hist)
{
	const int count_only = counting || COUNT || SILENT || FILENAMEONLY;
	/* output() needs j even without -n (agrep.c:3815) */
	return count_only ? (hist ? AGB_WANT_LEVELS : AGB_WANT_COUNT) : (AGB_WANT_RECORDS | AGB_WANT_ORDINALS);
}

static agb_record *grow_list(agb_record *recs, size_t cap)
{
	if (cap) { recs = (agb_record *)realloc(recs, cap * sizeof *recs); if (!recs) { fprintf(stderr, "%s: out of memory\n", prog); exit(255); } }
	return recs;
}

/* Files of up to SET_BYTES are gathered, in order, into sets of up to SET_BYTES and scanned by one agb_scan_set each: a small
 * file alone costs a whole scan's fixed cost (copies, launches, a read-back), in a set it costs its bytes.  A larger file, and
 * standard input, is scanned alone (agb_scan_host: stages 1 and 1.5 filter it, windows if it does not fit). */
#define SET_BYTES (16u << 20)
struct pending { const char *fname; unsigned char *hb; size_t n; };

static void scan_set_of(const agb_pattern *p, struct pending *set, int nset, int counting, unsigned long long *hist)
{
	const agb_desc *d = agb_pattern_desc(p);
	static const void *texts[4096]; static uint64_t sizes[4096]; static agb_result per[4096]; agb_result total;
	agb_record *recs = NULL; size_t cap = 0, bytes = 0, at = 0; int i, rc;
	const int want = scan_want(counting, hist);
	for (i = 0; i < nset; i++) { texts[i] = set[i].hb + 1; sizes[i] = set[i].n; bytes += set[i].n; }
	/* the list is sized from a guess; a set that reports more matching records than fit is scanned again with exactly
	 * n_matched entries */
	cap = (want & AGB_WANT_RECORDS) ? bytes / 64 + 65536 : 0;
	for (;;) {
		recs = grow_list(recs, cap);
		rc = agb_scan_set(p, texts, sizes, (uint32_t)nset, want, recs, cap, per, &total);
		if (rc) { fprintf(stderr, "%s: scan failed: %s\n", prog, agb_last_error()); exit(255); }   /* no CPU fallback */
		if (!total.truncated) break;
		cap = (size_t)total.n_matched;
	}
	for (i = 0; i < nset; i++) {
		finish_file(d, set[i].fname, set[i].hb, &per[i], recs + at, counting, hist);
		at += per[i].n_records;
		free(set[i].hb);
	}
	free(recs);
}

/* one pass of exec() over the files (agrep.c:3411-3576); counting = the COUNT=ON passes of the -B sweep; hist (counting
 * only): a levels pass -- every file's histogram of smallest levels is added to hist[] */
static int scan_files(const agb_pattern *p, char **files, int nfiles, int counting, unsigned long long *hist)
{
	struct pending set[4096]; int nset = 0, fi; size_t set_bytes = 0;
	const agb_desc *d = agb_pattern_desc(p);
	for (fi = 0; fi < (nfiles ? nfiles : 1); fi++) {
		const char *fname = nfiles ? files[fi] : NULL;
		size_t n = 0, cap; int unopened; unsigned char *hb = slurp(fname, &n, d->L, d->delim, &unopened);
		agb_result res; agb_record *recs = NULL; int rc;
		if (!hb) {
			/* the files gathered before this one print first: messages and output keep the order of the files */
			if (unopened) { if (nset) { scan_set_of(p, set, nset, counting, hist); nset = 0; set_bytes = 0; } cannot_open(fname); }
			continue;
		}
		if (fname && n <= SET_BYTES) {
			if (nset == 4096 || set_bytes + n > SET_BYTES) { scan_set_of(p, set, nset, counting, hist); nset = 0; set_bytes = 0; }
			set[nset].fname = fname; set[nset].hb = hb; set[nset].n = n; nset++; set_bytes += n;
			continue;
		}
		if (nset) { scan_set_of(p, set, nset, counting, hist); nset = 0; set_bytes = 0; }
		cap = (scan_want(counting, hist) & AGB_WANT_RECORDS) ? n / 64 + 65536 : 0;
		for (;;) {
			recs = grow_list(recs, cap);
			rc = agb_scan_host(p, hb + 1, n, scan_want(counting, hist), recs, cap, &res);
			if (rc) { fprintf(stderr, "%s: scan failed: %s\n", prog, agb_last_error()); exit(255); }   /* no CPU fallback */
			if (!res.truncated) break;
			cap = (size_t)res.n_matched;
		}
		finish_file(d, fname, hb, &res, recs, counting, hist);
		free(recs); free(hb);
	}
	if (nset) scan_set_of(p, set, nset, counting, hist);
	return num_of_matched;
}

/* the counting passes of the -B sweep for a regular expression without -v.  The per-level sweep compiles and scans at
 * k = 1, 2, ... up to `lim` (k < M, k <= AGB_MAXERR), stops at the first k that fails to compile, and at 4, the most a
 * regular expression allows.  Here one count-only levels pass per file at k = min(2, top) gives every line's smallest
 * level (re()'s rows are nested, so row j decides whether a line matches within j errors); only when no line has a level
 * in 1..2 does a second pass at k = min(4, top) look at 3..4.  Returns the best level (-1: none) and sets num_of_matched to
 * the lines at that level; stderr gets what the per-level sweep printed. */
static int regex_best_level(const char *pattern, agb_options *o, char **files, int nfiles, int lim)
{
	unsigned long long hist[AGB_MAXERR + 1];
	char err[256]; int k, top = 0, failed = 0, best = -1, lo = 1, passes, fi, l;
	const int cap = lim < 4 ? lim : 4;
	for (k = 1; k <= cap; k++) {
		agb_pattern *pk; o->k = k;
		if (agb_compile(pattern, o, &pk, err, sizeof err)) { failed = 1; break; }
		agb_pattern_free(pk);
		top = k;
	}
	QUIET_OPEN = 1;
	while (best < 0 && lo <= top) {
		agb_pattern *pk;
		k = lo <= 2 && top > 2 ? 2 : top;
		o->k = k;
		if (agb_compile(pattern, o, &pk, err, sizeof err)) break;     /* compiled above */
		memset(hist, 0, sizeof hist);
		scan_files(pk, files, nfiles, 1, hist);
		agb_pattern_free(pk);
		for (l = lo; l <= k && best < 0; l++) if (hist[l]) best = l;
		lo = k + 1;
	}
	QUIET_OPEN = 0;
	/* the per-level sweep named every unreadable file once per pass: `best` passes, or one per level it tried */
	passes = best > 0 ? best : top;
	for (l = 0; l < passes; l++)
		for (fi = 0; fi < nfiles; fi++) {
			int fd = open(files[fi], O_RDONLY);
			if (fd < 0) cannot_open(files[fi]); else close(fd);
		}
	if (best < 0 && !failed && lim > 4) fprintf(stderr, "%s: no match within 4 errors, the most a regular expression allows\n", prog);
	num_of_matched = best > 0 ? (int)hist[best] : 0;
	return best;
}

int main(int argc, char **argv)
{
	agb_options o; agb_pattern *p = NULL; char err[256]; const char *pattern = NULL; int ai, nfiles, rc;
	memset(&o, 0, sizeof o);
	o.regex = 1;
	o.wide_approx = 1;                       /* long simple literals at k > 0, as the reference's sgrep() takes them */
	o.sticky_delim = 1;                      /* -p with a delimiter of two or more bytes, as the reference answers it */
	if (argc > 0 && argv[0]) { const char *s = strrchr(argv[0], '/'); prog = s ? s + 1 : argv[0]; }
	for (ai = 1; ai < argc && argv[ai][0] == '-' && argv[ai][1]; ai++) {
		const char *q = argv[ai] + 1; int stop = 0;
		for (; *q && !stop; q++) {
			switch (*q) {
			case 'c': COUNT = 1; break;            case 's': SILENT = 1; break;
			case 'l': FILENAMEONLY = 1; break;     case 'h': NOFILENAME = 1; break;
			case 'n': LINENUM = 1; o.linenum = 1; break;
			case 'b': BYTECOUNT = 1; break;        case 'i': o.nocase = 1; if (q[1] == '0') { o.nocase = 0; q++; } break;
			case 'w': o.wordbound = 1; break;      case 'x': o.wholeline = 1; break;
			case 'v': o.inverse = 1; break;        case 'p': o.ins_free = 1; break;
			case 'B': BESTMATCH = 1; o.bestmatch = 1; break;
			case 'y': NOPROMPT = 1; break;         case 't': OUTTAIL = 1; break;
			case 'I': o.cost_i = atoi(q + 1); stop = 1; break;
			case 'S': o.cost_s = atoi(q + 1); stop = 1; break;
			case 'D': o.cost_d = atoi(q + 1); stop = 1; break;
			case 'V': VERBOSE = isdigit((unsigned char)q[1]) ? atoi(q + 1) : 1; stop = 1; break;
			case 'd': if (q[1]) o.delim = q + 1; else if (ai + 1 < argc) o.delim = argv[++ai]; else usage(); stop = 1; break;
			case 'e': if (ai + 1 < argc) pattern = argv[++ai]; else usage(); stop = 1; break;
			default:
				if (isdigit((unsigned char)*q)) { o.k = atoi(q); if (o.k > AGB_MAXERR) { fprintf(stderr, "%s: the maximum number of errors is %d\n", prog, AGB_MAXERR); return 2; } stop = 1; }
				else { fprintf(stderr, "%s: illegal option  -%c\n", prog, *q); usage(); }
			}
		}
	}
	if (!pattern) { if (ai >= argc) usage(); pattern = argv[ai++]; }
	nfiles = argc - ai;
	if (BESTMATCH && (COUNT || FILENAMEONLY || o.k)) { BESTMATCH = 0; o.bestmatch = 0; fprintf(stderr, "%s: -B option ignored when -c, -l, -f, or -# is on\n", prog); }   /* compat.c:26-29 */
	if (COUNT && LINENUM) { LINENUM = 0; fprintf(stderr, "%s: -n option ignored with -c\n", prog); }   /* compat.c:30-33 (the engine choice stays) */
	FNAME = nfiles > 1 && !NOFILENAME;
	if (o.delim && strlen(o.delim) == 1 && (o.delim[0] == '\n' || o.delim[0] == '$' || o.delim[0] == '^')) OUTTAIL = 1;   /* agrep.c:2290 */
	if (is_regex(pattern) && (o.cost_i || o.cost_s || o.cost_d)) {
		fprintf(stderr, "%s: -D#, -I#, or -S# option is ignored for regular expression pattern\n", prog);   /* compat.c:75-79 */
		o.cost_i = o.cost_s = o.cost_d = 0;
	}
	rc = agb_compile(pattern, &o, &p, err, sizeof err);
	if (rc) {
		fprintf(stderr, "%s: %s\n", prog, err);
		/* bitap.c:96-104 refuses k > 4 at scan time, after main() has set up its output: the total is still printed */
		if (is_regex(pattern) && o.k > 4 && VERBOSE > 0 && o.k <= AGB_MAXERR) printf("Grand Total: 0 match(es) found.\n");
		return 255;
	}

	scan_files(p, argv + ai, nfiles, 0, NULL);
	if (BESTMATCH && num_of_matched == 0 && nfiles > 0) {
		/* agrep.c:3582-3728: nothing matched -> counting passes at D = 1, 2, ... < M, <= 8 until something matches,
		 * report, ask (unless -y), then one printing pass at that D.  A regular expression without -v takes its counting
		 * passes from levels scans (regex_best_level) */
		const int M = agb_pattern_desc(p)->M, regex = agb_pattern_desc(p)->engine == AGB_ENGINE_REGEX; int k, best = -1;
		if (regex && !o.inverse) best = regex_best_level(pattern, &o, argv + ai, nfiles, M - 1 < AGB_MAXERR ? M - 1 : AGB_MAXERR);
		else for (k = 1; k < M && k <= AGB_MAXERR && best < 0; k++) {
			/* a regular expression allows 4 errors at most: the reference's sweep goes on to k = 5 and fails there (SURVEY 8c) */
			if (regex && k > 4) { fprintf(stderr, "%s: no match within 4 errors, the most a regular expression allows\n", prog); break; }
			agb_pattern *pk; o.k = k;
			if (agb_compile(pattern, &o, &pk, err, sizeof err)) break;
			num_of_matched = 0;
			if (scan_files(pk, argv + ai, nfiles, 1, NULL) > 0) best = k;
			agb_pattern_free(pk);
		}
		if (best > 0) {
			int go = 1;
			if (num_of_matched == 1) fprintf(stderr, "%s: 1 word matches within ", prog); else fprintf(stderr, "%s: %d words match within ", prog, num_of_matched);
			if (best == 1) fprintf(stderr, "1 error"); else fprintf(stderr, "%d errors", best);
			if (NOPROMPT) fprintf(stderr, "\n");
			else {
				char c[8] = "y";
				fprintf(stderr, num_of_matched == 1 ? "; search for it? (y/n)" : "; search for them? (y/n)");
				if (!fgets(c, 4, stdin) || c[0] != 'y') go = 0;
			}
			if (go) {
				agb_pattern_free(p); p = NULL; o.k = best;
				if (agb_compile(pattern, &o, &p, err, sizeof err)) return 255;
				num_of_matched = 0;
				scan_files(p, argv + ai, nfiles, 0, NULL);
			}
		} else num_of_matched = 0;
	}
	if (EATFIRST) printf("\n");                                         /* agrep.c:3731-3741 */
	if (VERBOSE > 0) printf("Grand Total: %d match(es) found.\n", num_of_matched);   /* agrep.c:3229-3231 */
	if (p) agb_pattern_free(p);
	return num_of_matched;                                              /* main.c:96: exit status = number of matches */
}
