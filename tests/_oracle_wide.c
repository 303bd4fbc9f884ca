/* tests/_oracle_wide.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE: the checker's automaton in 320-bit rows.
 *
 * The checker (oracle/agrep_oracle.c) restates the reference with 64-bit words.  The device runs simple literals of more
 * than 63 positions (up to 255 characters, agb_wide) in rows of five 64-bit words; this file states the same automaton in
 * rows of ORC_WIDE_WORDS words, for patterns of up to 319 positions.  It includes the checker's source unchanged and reuses
 * its pattern preprocessing and record bookkeeping; only the word width differs.  The reference's own words stop at 32
 * positions, so nothing pins this path on it: the tests check it against the 64-bit checker on patterns of <= 63
 * positions, against an edit-distance restatement on longer ones, and against the lines the reference binary prints
 * (a subset: its sgrep() filters at k > 0 lose matches).
 *
 * Bit-parallel engines with unit costs only (exact bitap, asearch, asearch0): a simple literal needs linenum = 1 here, as
 * in orc_compile, and costs are refused.  o->width must be ORC_WIDE_BITS.  The 64-bit word fields of w->a stay zero;
 * everything else in it (M, L, dpat, engine, k, inverse, ...) is as orc_compile would set it.
 * Built by tests/_oracle_wide.py (cc -I oracle) into a temporary directory on first use. */
#include "agrep_oracle.c"

#define ORC_WIDE_WORDS 5
#define ORC_WIDE_BITS  (64 * ORC_WIDE_WORDS)
typedef struct {
	orc_automaton a;
	uint64_t mask[256][ORC_WIDE_WORDS];
	uint64_t init0[ORC_WIDE_WORDS], init1[ORC_WIDE_WORDS], noerr[ORC_WIDE_WORDS], endpos[ORC_WIDE_WORDS];
	uint64_t dendpos[ORC_WIDE_WORDS], dmask[ORC_WIDE_WORDS], wildmask[ORC_WIDE_WORDS];
} orc_wide;

int orc_compile_wide(const char *pattern, const orc_opts *o, orc_wide *w, char *err, size_t errlen);
/* orc_scan and orc_scan_levels of an orc_wide */
int64_t orc_scan_wide(const orc_wide *w, const unsigned char *text, uint64_t n, orc_record *recs, uint64_t cap);
int64_t orc_scan_levels_wide(const orc_wide *w, int kmax, const unsigned char *text, uint64_t n,
                             uint64_t histogram[ORC_MAXERR + 1], orc_record *recs, uint64_t cap, int want_level);

/* ---------------------------------------------------------------------------------------------
 * maskgen.c:26-269 and the loops of bitap.c / asearch.c, with rows of ORC_WIDE_WORDS words.  Position p (1-based)
 * lives at bit M-p; bits M..319 are the always-on feed.
 * ------------------------------------------------------------------------------------------- */
#define WW ORC_WIDE_WORDS
typedef struct { uint64_t w[WW]; } wrow;

static void wset(uint64_t *x, int bit) { x[bit >> 6] |= 1ull << (bit & 63); }
static wrow wload(const uint64_t *x) { wrow r; memcpy(r.w, x, sizeof r.w); return r; }
static wrow wshr1(wrow x) { wrow r; int i; for (i = 0; i < WW; i++) r.w[i] = (x.w[i] >> 1) | (i + 1 < WW ? x.w[i + 1] << 63 : 0); return r; }
static wrow wand(wrow x, wrow y) { int i; for (i = 0; i < WW; i++) x.w[i] &= y.w[i]; return x; }
static wrow wor(wrow x, wrow y) { int i; for (i = 0; i < WW; i++) x.w[i] |= y.w[i]; return x; }
static int wany(wrow x) { int i; uint64_t o = 0; for (i = 0; i < WW; i++) o |= x.w[i]; return o != 0; }
static int weq(wrow x, wrow y) { int i; for (i = 0; i < WW; i++) if (x.w[i] != y.w[i]) return 0; return 1; }

/* maskgen() of agrep_oracle.c with flags per position instead of 64-bit position sets */
static int maskgen_wide(unsigned char *P, int plen, int L, const orc_opts *o, orc_wide *w, char *err, size_t errlen)
{
	static struct { int compl_, wild, prot, sep; unsigned char cls[2 * 32 + 2]; int ncls; } pos[ORC_WIDE_BITS + 12];
	orc_automaton *a = &w->a;
	int i, j = 1, no_error = 0, even = 0, orflag = 0, M, k, c, p;
	memset(pos, 0, sizeof pos);
	a->and_mode = 0;
	if (o->nocase) for (i = 0; i < plen; i++) if (ascii_upper(P[i])) P[i] = (unsigned char)(P[i] + 32);
	for (i = 0; i < plen; i++) {
		unsigned char pp = P[i];
		if (pp == WILDCD) { if (j - 1 >= 1) pos[j - 1].wild = 1; }
		else if (pp == LANGLE) { no_error = 1; even++; }
		else if (pp == RANGLE) { no_error = 0; even--; if (even < 0) FAIL("unmatched '<', '>'"); }
		else if (pp == LRANGE) {
			int kk = 0;
			if (no_error) pos[j].prot = 1;
			i++;
			if (P[i] == NOTSYM) { pos[j].compl_ = 1; i++; }
			while (P[i] != RRANGE && i < plen) {
				if (P[i] == HYPHEN) { if (kk > 0) pos[j].cls[kk - 1] = P[i + 1]; i += 2; }
				else { if (kk + 2 > 64) FAIL("character class too long"); pos[j].cls[kk] = pos[j].cls[kk + 1] = P[i]; kk += 2; i++; }
			}
			if (i >= plen) FAIL("unmatched '[', ']'");
			pos[j].ncls = kk;
			j++;
		}
		else if (pp == RRANGE) FAIL("unmatched '[', ']'");
		else if (pp == ORPAT) {
			if (a->and_mode) FAIL("cannot handle OR (',') and AND (';') simultaneously");
			orflag = 1; pos[j].sep = 1; j++;
		}
		else if (pp == ANDPAT) {
			if (j > L + 1) a->and_mode = 1;
			if (orflag) FAIL("cannot handle AND (';') and OR (',') simultaneously");
			pos[j].sep = 1; j++;
		}
		else if (pp == '\n') { pos[j].prot = 1; pos[j].cls[0] = pos[j].cls[1] = '\n'; pos[j].ncls = 2; j++; }
		else if (pp == WORDB) {
			static const unsigned char wb[8] = { 1, 47, 58, 64, 91, 96, 123, 127 };
			pos[j].prot = 1; memcpy(pos[j].cls, wb, 8); pos[j].ncls = 8; j++;
		}
		else if (pp == NNLINE) {
			pos[j].prot = 1; pos[j].cls[0] = pos[j].cls[1] = '\n'; pos[j].cls[2] = pos[j].cls[3] = NNLINE; pos[j].ncls = 4; j++;
		}
		else if (pp != STAR && pp != ORSYM && pp != LPARENT && pp != RPARENT) {
			if (no_error) pos[j].prot = 1;
			pos[j].cls[0] = pos[j].cls[1] = pp; pos[j].ncls = 2; j++;
		}
		if (j > ORC_WIDE_BITS) FAIL("pattern too long (has > %d chars)", ORC_WIDE_BITS);
	}
	if (even != 0) FAIL("unmatched '<', '>'");
	M = j - 1;
	memset(w->init0, 0, sizeof w->init0); memset(w->wildmask, 0, sizeof w->wildmask); memset(w->endpos, 0, sizeof w->endpos);
	memset(w->dendpos, 0, sizeof w->dendpos); memset(w->mask, 0, sizeof w->mask);
	for (i = 0; i < WW; i++) { w->noerr[i] = ~0ull; w->dmask[i] = ~0ull; }
	for (i = M; i < ORC_WIDE_BITS; i++) wset(w->init0, i);                       /* Init[0] |= Bit[1..W-M] (:224) */
	wset(w->endpos, 0);                                                           /* endp = (sep << 1) + 1 (:231) */
	for (p = 1; p <= M; p++) {
		if (pos[p].sep) { wset(w->init0, M - p); wset(w->endpos, M - p + 1); }
		if (pos[p].wild) wset(w->wildmask, M - p);
		if (pos[p].prot) w->noerr[(M - p) >> 6] &= ~(1ull << ((M - p) & 63));
	}
	for (i = 0; i < WW; i++) w->init1[i] = w->init0[i] | w->wildmask[i] | w->endpos[i];   /* :232 */
	if (L >= 1 && L <= M && (w->endpos[(M - L) >> 6] >> ((M - L) & 63) & 1)) {   /* :233-234 */
		wset(w->dendpos, M - L); w->endpos[(M - L) >> 6] &= ~(1ull << ((M - L) & 63));
		for (p = 0; p < L; p++) w->dmask[(M - L + p) >> 6] &= ~(1ull << ((M - L + p) & 63));   /* bitap.c:131-133 */
	}
	for (c = 0; c < 256; c++) {
		for (k = 1; k <= M; k++) {
			int l, hit = 0;
			for (l = 0; l < pos[k].ncls; l += 2) {
				if (pos[k].cls[l] == NOCARE && c != '\n') { hit = 1; break; }
				if (c >= pos[k].cls[l] && c <= pos[k].cls[l + 1]) { hit = 1; break; }
			}
			if (pos[k].compl_) hit = !hit;
			if (hit) wset(w->mask[c], M - k);
		}
	}
	if (o->nocase) for (c = 'A'; c <= 'Z'; c++) memcpy(w->mask[c], w->mask[c + 32], sizeof w->mask[c]);
	a->M = M;
	return 0;
}

int orc_compile_wide(const char *pattern, const orc_opts *o, orc_wide *w, char *err, size_t errlen)
{
	unsigned char internal[1200], pat[600];
	char dpattern[64];
	orc_automaton *a = &w->a;
	int m, plen, notsgrep = 0, simple;
	memset(w, 0, sizeof *w);
	if (o->width != ORC_WIDE_BITS) FAIL("orc_compile_wide builds %d-bit rows (width = %d)", ORC_WIDE_BITS, ORC_WIDE_BITS);
	m = (int)strlen(pattern);
	if (m < 1) FAIL("pattern length too small");
	if (m >= 256) FAIL("pattern too long");                                /* agrep.c:3057 */
	if (m <= o->k) FAIL("size of pattern must be > #of errors %d", o->k);  /* checksg.c:34 */
	if (o->k < 0 || o->k > ORC_MAXERR) FAIL("the maximum number of errors is %d", ORC_MAXERR);
	if (o->wordbound && o->wholeline) FAIL("illegal option combination (-x and -w)");
	if (o->delim && o->wholeline) FAIL("-d and -x are not compatible");
	if (o->cost_i || o->cost_s || o->cost_d) FAIL("320-bit rows: unit costs only");
	memcpy(pat, pattern, (size_t)m + 1);
	a->k = o->k; a->inverse = o->inverse; a->ci = a->cs = a->cd = 1;
	a->user_delim = o->delim != NULL;
	if (o->delim) {
		size_t dl = strlen(o->delim);
		if (dl < 1 || dl > 16) FAIL("delimiter pattern too long");
		snprintf(dpattern, sizeof dpattern, "<%s>; ", o->delim);
		if (dl == 1 && (o->delim[0] == '\n' || o->delim[0] == '$' || o->delim[0] == '^')) a->outtail = 1;
	} else strcpy(dpattern, "\n; ");
	simple = simple_pattern(pat, m, o->k, &notsgrep);
	a->sgrep = simple && !o->bestmatch && !(o->nocase && o->k > 0) && !o->ins_free && !o->linenum
	           && !(o->wordbound && o->k > 0) && !(o->wholeline && o->k > 0) && !notsgrep;
	if (a->sgrep) FAIL("simple patterns go to sgrep() in the reference, which has no rows; force the automaton with linenum=1");
	if (preprocess(pat, o, dpattern, internal, &plen, a->dpat, &a->L, err, errlen)) return -1;
	if (maskgen_wide(internal, plen, a->L, o, w, err, errlen)) return -1;
	if (o->ins_free) memset(w->init1, 0xFF, sizeof w->init1);                   /* bitap.c:123 */
	if (o->k > 4) a->engine = 2;                                                /* asearch.c:50-52 */
	else if (o->k > 0) a->engine = 1;
	else { a->engine = 0; a->lut_fold = o->nocase; }
	return 0;
}

static int match_cond_wide(const orc_wide *w, wrow r)
{
	const wrow e = wload(w->endpos);
	if (w->a.and_mode) return weq(wand(r, e), e) || (w->a.inverse != 0);
	return wany(wand(r, e)) ^ (w->a.inverse != 0);
}

/* scan_exact() and scan_approx() of agrep_oracle.c on 320-bit rows */
static int64_t scan_wide(const orc_wide *w, int k, const unsigned char *text, uint64_t n,
                         orc_record *recs, uint64_t cap, uint64_t *hist, int want_level)
{
	const orc_automaton *a = &w->a;
	const wrow init0 = wload(w->init0), init1 = wload(w->init1), noerr = wload(w->noerr), dend = wload(w->dendpos), dmask = wload(w->dmask);
	recstate rs; wrow A[ORC_MAXERR + 1], B[ORC_MAXERR + 1]; uint64_t i, end = n + 1 + (uint64_t)a->L; int r;
	unsigned char lut[256]; int c;
	for (c = 0; c < 256; c++) lut[c] = (unsigned char)c;
	if (a->lut_fold) orc_lut_lower1(lut);                                       /* bitap.c:171 (exact engine only) */
	for (r = 0; r <= k; r++) A[r] = B[r] = init0;
	rec_init(&rs, a, text, n, recs, cap);
	for (i = 0; i < end; ) {
		const wrow cm = wload(w->mask[lut[ext_byte(a, text, n, i++)]]);
		int closed;
		A[0] = wor(wand(wshr1(B[0]), cm), wand(init1, B[0]));
		for (r = 1; r <= k; r++)
			A[r] = wor(wor(wor(wand(wshr1(B[r]), cm), wand(init1, B[r])), B[r - 1]), wand(wshr1(wor(A[r - 1], B[r - 1])), noerr));
		closed = wany(wand(A[0], dend));
		if (closed) {
			if (hist) {
				int lvl = -1;
				for (r = 0; r <= k; r++) if (match_cond_wide(w, A[r])) { lvl = r; break; }
				if (lvl >= 0) {
					if (rec_counts(&rs, i)) hist[lvl]++;
					rec_close(&rs, i, (want_level < 0) || (lvl <= want_level), lvl);
				} else rec_close(&rs, i, 0, -1);
			} else rec_close(&rs, i, match_cond_wide(w, A[k]), k);
			for (r = 0; r <= k; r++) B[r] = init0;                                  /* asearch.c:177-186, bitap.c:223-225 */
			A[0] = wand(wor(wand(wshr1(B[0]), cm), wand(B[0], init1)), dmask);
			for (r = 1; r <= k; r++)
				A[r] = wor(wor(wor(wand(wshr1(B[r]), cm), wand(init1, B[r])), B[r - 1]), wand(wshr1(wor(A[r - 1], B[r - 1])), noerr));
		}
		for (r = 0; r <= k; r++) B[r] = A[r];
	}
	return rs.matched;
}

int64_t orc_scan_wide(const orc_wide *w, const unsigned char *text, uint64_t n, orc_record *recs, uint64_t cap)
{
	if (w->a.engine > 2) return -1;
	return scan_wide(w, w->a.k, text, n, recs, cap, NULL, -1);
}

int64_t orc_scan_levels_wide(const orc_wide *w, int kmax, const unsigned char *text, uint64_t n,
                             uint64_t histogram[ORC_MAXERR + 1], orc_record *recs, uint64_t cap, int want_level)
{
	int r;
	if (w->a.engine > 2 || kmax < 0 || kmax > ORC_MAXERR) return -1;
	for (r = 0; r <= ORC_MAXERR; r++) histogram[r] = 0;
	return scan_wide(w, kmax, text, n, recs, cap, histogram, want_level);
}
