/* agrep_b200/csrc/pattern.c -- host-side pattern front-end of libagrepb200 (C, no CUDA).
 *
 * Turns (pattern, options) into the scan descriptor agb_desc the kernels consume.  It mirrors what the
 * reference does on the host before a scan -- checksg() (checksg.c:19-165: which engine), preprocess()
 * (preproce.c:137-341: delimiter + separator + -w/-x wrap + meta characters) and maskgen()
 * (maskgen.c:26-269: Mask[], Init[0], Init1, NO_ERR_MASK, endposition, D_endpos, wildmask) -- but is
 * organised as one pass over the user's pattern that emits automaton positions with 256-bit classes,
 * in 64-bit words (the reference stops at 32 positions, maskgen.c:201-208), or in the 320-bit words of agb_wide for a
 * simple literal of more than 63 positions: at k = 0 (sgrep()'s bm()/monkey(), which take up to 255 characters), and at
 * k = 1..8 when the caller asks for it (agb_options.wide_approx: the literals the reference hands to sgrep() at k > 0).
 *
 * It also derives what only the device path needs: the constant post-delimiter rows (asearch.c:175-186),
 * the delimiter kind, and the pigeonhole anchor plan for the front-end kernel.
 */
#include "agrep_b200.h"
#include "pattern_internal.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define WIDTH 64
#define FAIL(...) do { if (err && errlen) snprintf(err, errlen, __VA_ARGS__); return AGB_ERR_PATTERN; } while (0)

/* internal symbol codes of the reference (agrep.h:69-87); raw pattern bytes in this range are refused */
enum { S_HYPHEN = 129, S_NOCARE = 130, S_NNLINE = 131, S_WORDB = 133, S_LPAREN = 134, S_RPAREN = 135,
       S_LRANGE = 136, S_RRANGE = 137, S_LANGLE = 138, S_RANGLE = 139, S_NOT = 140, S_WILD = 141,
       S_ORSYM = 142, S_ORPAT = 143, S_ANDPAT = 144, S_STAR = 145 };

typedef struct {
	uint64_t cls[4];     /* 256-bit character class */
	int is_sep;          /* ORPAT / ANDPAT slot: empty class, always-on start bit (maskgen.c:136-163) */
	int prot;            /* NO_ERR_MASK position (maskgen.c:97,172,177,189,195) */
	int wild;            /* '#' after this position: sticky self loop (maskgen.c:72-79) */
	int lit;             /* single literal byte (anchor eligible), else -1 */
	int part;            /* index of the ','/';' sub-pattern this position belongs to */
} pos_t;

typedef struct {
	pos_t p[AGB_WIDE_MAXPOS + 4];
	int n;               /* positions so far (1-based: p[1..n]) */
	int wide_ok;         /* up to AGB_WIDE_MAXPOS positions (a simple literal that sgrep() takes), else up to WIDTH - 1 */
	int no_error, even;
	int or_seen, and_mode, nparts;
} build_t;

static void cls_set(pos_t *p, int c) { p->cls[c >> 6] |= 1ull << (c & 63); }
static int  cls_has(const pos_t *p, int c) { return (int)(p->cls[c >> 6] >> (c & 63) & 1); }
static void cls_range(pos_t *p, int lo, int hi)
{
	int c;
	if (lo == S_NOCARE) for (c = 0; c < 256; c++) if (c != '\n') cls_set(p, c);   /* maskgen.c:243-247 */
	for (c = lo; c <= hi && c < 256; c++) cls_set(p, c);                         /* maskgen.c:248-252 */
}
static int is_upper(int c) { return c >= 'A' && c <= 'Z'; }
static int is_alpha(int c) { return (c | 32) >= 'a' && (c | 32) <= 'z'; }
static int is_alnum(int c) { return is_alpha(c) || (c >= '0' && c <= '9'); }

static pos_t *new_pos(build_t *b)
{
	pos_t *p;
	if (b->n + 1 > (b->wide_ok ? AGB_WIDE_MAXPOS : WIDTH - 1)) return NULL;     /* M <= W-1: one always-on feed bit above the field */
	p = &b->p[++b->n];
	memset(p, 0, sizeof *p);
	p->lit = -1;
	p->part = b->nparts;
	return p;
}

/* one user-pattern character -> the reference's internal symbol (preproce.c:238-332) */
static int map_sym(const unsigned char *s, int *i, int n, int in_range, int *escaped)
{
	int c = s[*i];
	*escaped = 0;
	if (c == '\\') { (*i)++; *escaped = 1; return (*i < n) ? s[*i] : 0; }
	switch (c) {
	case '#': return S_WILD;   case '(': return S_LPAREN; case ')': return S_RPAREN;
	case '[': return S_LRANGE; case ']': return S_RRANGE; case '<': return S_LANGLE; case '>': return S_RANGLE;
	case '^': return (*i > 0 && s[*i - 1] == '[') ? S_NOT : '\n';
	case '$': return '\n';     case '.': return S_NOCARE; case '*': return S_STAR;   case '|': return S_ORSYM;
	case ',': return S_ORPAT;  case ';': return S_ANDPAT; case '-': return in_range ? S_HYPHEN : '-';
	default: return c;
	}
}

static int add_literal(build_t *b, int c, int nocase, char *err, size_t errlen)
{
	pos_t *p = new_pos(b);
	if (!p) FAIL("pattern too long (has > %d chars)", WIDTH);
	if (c == '\n') { p->prot = 1; cls_set(p, '\n'); return 0; }               /* maskgen.c:171-175 */
	if (b->no_error) p->prot = 1;                                              /* maskgen.c:195 */
	if (nocase && is_upper(c)) c += 32;                                        /* maskgen.c:52-59 */
	cls_set(p, c);
	if (nocase && is_alpha(c)) cls_set(p, c - 32);                             /* maskgen.c:259-266 */
	p->lit = c;
	return 0;
}

static int add_wordb(build_t *b, char *err, size_t errlen)
{
	pos_t *p = new_pos(b);
	if (!p) FAIL("pattern too long (has > %d chars)", WIDTH);
	p->prot = 1;                                                               /* maskgen.c:176-187 */
	cls_range(p, 1, 47); cls_range(p, 58, 64); cls_range(p, 91, 96); cls_range(p, 123, 127);
	return 0;
}

static int add_sep(build_t *b, int is_and, int L, char *err, size_t errlen)
{
	pos_t *p;
	if (is_and) {                                                              /* maskgen.c:150-163 */
		if (b->n + 1 > L + 1) b->and_mode = 1;
		if (b->or_seen) FAIL("illegal pattern: cannot handle AND (';') and OR (',') simultaneously");
	} else {                                                                   /* maskgen.c:136-149 */
		if (b->and_mode) FAIL("illegal pattern: cannot handle OR (',') and AND (';') simultaneously");
		b->or_seen = 1;
	}
	p = new_pos(b);
	if (!p) FAIL("pattern too long (has > %d chars)", WIDTH);
	p->is_sep = 1;
	b->nparts++;
	return 0;
}

/* one "[...]" class (maskgen.c:96-127); s[*i] is the '[', *i is left on the closing ']'.  regex: '.' inside the class
 * also matches '\n' (maskgen.c:243), and a range that parse_cset() refuses (parse.c:81-120) is an error */
static int add_class(build_t *b, const unsigned char *s, int *pi, int n, const agb_options *o, int regex, char *err, size_t errlen)
{
	pos_t *p = new_pos(b); int compl_ = 0, closed = 0, esc, i = *pi;
	uint64_t keep[4];
	if (!p) { if (regex) FAIL("regular expression too long"); FAIL("pattern too long (has > %d chars)", WIDTH); }
	if (b->no_error) p->prot = 1;
	i++;
	if (i < n && s[i] == '^') { compl_ = 1; i++; }
	{   /* maskgen.c:104-116 keeps the class as (low, high) pairs: a symbol opens the pair (c, c), "-x" replaces the high
	     * end of the last pair -- so a descending range like z-a matches nothing, not even z */
		int plo[2 * WIDTH], phi[2 * WIDTH], np = 0, q;
		for (; i < n; i++) {
			int cc = map_sym(s, &i, n, 1, &esc);
			if (!esc && cc == S_RRANGE) { closed = 1; break; }
			if (!esc && cc == S_HYPHEN) {                              /* class[k-1] = next symbol */
				int hi;
				if (regex && np == 0) FAIL("illegal regular expression");
				i++;
				if (i >= n) break;
				hi = map_sym(s, &i, n, 1, &esc);
				if (o->nocase && is_upper(hi)) hi += 32;
				if (regex && np > 0 && hi < plo[np - 1]) FAIL("illegal regular expression");
				if (np > 0) phi[np - 1] = hi;
				continue;
			}
			if (o->nocase && is_upper(cc)) cc += 32;                   /* Pattern[] is lower-cased as a whole */
			if (np < 2 * WIDTH) { plo[np] = phi[np] = cc; np++; }
		}
		if (regex && closed && np == 0) FAIL("illegal regular expression");
		for (q = 0; q < np; q++) {
			if (plo[q] == S_NOCARE) { cls_range(p, S_NOCARE, S_NOCARE); if (regex) cls_set(p, '\n'); }   /* maskgen.c:242-246 looks at the low end first: '.' = any */
			else if (plo[q] <= phi[q]) cls_range(p, plo[q], phi[q]);
		}
	}
	if (!closed) FAIL("unmatched '[', ']' (use \\[, \\] to search for [, ])");
	if (compl_) { p->cls[0] = ~p->cls[0]; p->cls[1] = ~p->cls[1]; p->cls[2] = ~p->cls[2]; p->cls[3] = ~p->cls[3]; }
	if (o->nocase) {                                                   /* maskgen.c:259-266: Mask[U] = Mask[u] */
		int u;
		memcpy(keep, p->cls, sizeof keep);
		for (u = 'A'; u <= 'Z'; u++) {
			p->cls[u >> 6] &= ~(1ull << (u & 63));
			if (keep[(u + 32) >> 6] >> ((u + 32) & 63) & 1) cls_set(p, u);
		}
	}
	*pi = i;
	return 0;
}

/* the user's pattern (after the delimiter part and the optional -w/-x opener) */
static int add_pattern(build_t *b, const unsigned char *s, int n, const agb_options *o, int L, char *err, size_t errlen)
{
	int i, esc;
	for (i = 0; i < n; i++) {
		if (s[i] == '\\') {                                                    /* preproce.c:139-142 */
			/* a lone backslash at the very end escapes whatever preprocess() appended behind the pattern (the string
			 * terminator, or the '<' of the -w/-x wrapper, preproce.c:148-175): not restated, refused */
			if (++i >= n) {
				if (o->wordbound || o->wholeline) FAIL("the pattern ends in a lone backslash");
				n--;                                                           /* it escapes the terminator: nothing (the reference's strlen() stops there) */
			}
		}
		else if (s[i] == '|' || s[i] == '*')
			FAIL("regular expressions (re()/re1(), agrep.c:468-1917) are outside the accelerated scan path");
	}
	for (i = 0; i < n; i++) {
		int c = map_sym(s, &i, n, 0, &esc);
		if (!esc && s[i] >= 129 && s[i] <= 145) FAIL("byte %d in the pattern collides with an internal symbol (agrep.h:69-87)", s[i]);
		if (esc) { if (add_literal(b, c, o->nocase, err, errlen)) return AGB_ERR_PATTERN; continue; }
		switch (c) {
		case S_WILD: if (b->n >= 1) b->p[b->n].wild = 1; break;
		case S_LANGLE: b->no_error = 1; b->even++; break;
		case S_RANGLE: b->no_error = 0; if (--b->even < 0) FAIL("unmatched '<', '>' (use \\<, \\> to search for <, >)"); break;
		case S_LPAREN: case S_RPAREN: break;                                   /* maskgen.c:194: no position */
		case S_RRANGE: FAIL("unmatched '[', ']' (use \\[, \\] to search for [, ])");
		case S_ORPAT: if (add_sep(b, 0, L, err, errlen)) return AGB_ERR_PATTERN; break;
		case S_ANDPAT: if (add_sep(b, 1, L, err, errlen)) return AGB_ERR_PATTERN; break;
		case S_NOCARE: {
			pos_t *p = new_pos(b);
			if (!p) FAIL("pattern too long (has > %d chars)", WIDTH);
			if (b->no_error) p->prot = 1;
			cls_range(p, S_NOCARE, S_NOCARE);
			break; }
		case S_LRANGE:
			if (add_class(b, s, &i, n, o, 0, err, errlen)) return AGB_ERR_PATTERN;
			break;
		default:
			if (add_literal(b, c, o->nocase, err, errlen)) return AGB_ERR_PATTERN;
		}
	}
	if (b->even != 0) FAIL("unmatched '<', '>' (use \\<, \\> to search for <, >)");
	return 0;
}

/* the -i table of bitap.c:171 as the reference leaves it: CP[ISO-8859-1].lower_1 (agrep.c:2769-2792,
 * codepage.c:399-533) with every byte that serves as a metasymbol put back to itself (agrep.c:2835-2848; in this
 * codepage that undoes the lower_1 entries of 0x83, 0x8f and 0x99), stated as identity + ASCII folding + the 29
 * high-half entries that remain */
void agbi_lut_lower1(unsigned char lut[256])
{
	static const unsigned char hi[] = {
		0x80,0x87, 0x8a,0x9a, 0x8c,0x9c, 0x8e,0x9e, 0x90,0x82, 0x92,0x91,
		0xc1,0xe1, 0xc3,0xe3, 0xc4,0xe4, 0xc5,0xe5, 0xc7,0xe7, 0xc8,0xe8, 0xc9,0xe9, 0xca,0xea, 0xcc,0xec,
		0xcd,0xed, 0xce,0xee, 0xcf,0xef, 0xd1,0xf1, 0xd2,0xf2, 0xd3,0xf3, 0xd4,0xf4, 0xd5,0xf5, 0xd6,0xf6,
		0xd8,0xf8, 0xda,0xfa, 0xdc,0xfc, 0xdd,0xfd, 0xde,0xfe };
	size_t i;
	for (i = 0; i < 256; i++) lut[i] = (unsigned char)(is_upper((int)i) ? i + 32 : i);
	for (i = 0; i + 1 < sizeof hi; i += 2) lut[hi[i]] = hi[i + 1];
}

/* one automaton step on all rows: asearch.c:96-115 (unit costs) / asearch1.c:88-97 (costs) / bitap.c:175-176 */
void agbi_step(const agb_desc *d, const uint64_t *B, uint64_t *A, uint64_t cm)
{
	int r, n = d->k;
	A[0] = ((B[0] >> 1) & cm) | (d->init1 & B[0]);
	if (d->engine == AGB_ENGINE_ASEARCH1) {
		int I = d->cost_i, S = d->cost_s, DD = d->cost_d;
		for (r = 1; r <= n; r++) {
			uint64_t bi = (r - I >= 0) ? B[r - I] : 0, ad = (r - DD >= 0) ? A[r - DD] : 0, bs = (r - S >= 0) ? B[r - S] : 0;
			A[r] = ((B[r] >> 1) & cm) | bi | (((ad | bs) >> 1) & d->noerr) | (d->init1 & B[r]);
		}
	} else {
		for (r = 1; r <= n; r++)
			A[r] = ((B[r] >> 1) & cm) | (d->init1 & B[r]) | B[r - 1] | (((A[r - 1] | B[r - 1]) >> 1) & d->noerr);
	}
}

static int has_border(const unsigned char *d, int L)
{
	int b;
	for (b = 1; b < L; b++) if (memcmp(d, d + L - b, (size_t)b) == 0) return 1;
	return 0;
}
/* the delimiter as the device compares it: letters that accept both cases in lower case */
static void folded_delim(const agb_desc *d, unsigned char *out) { int p; for (p = 0; p < d->L; p++) out[p] = (unsigned char)(d->delim[p] | d->delim_fold[p]); }

static int derive(agb_desc *d, agb_wide *w, char *err, size_t errlen);

/* a row of agb_wide: bit i in word i / 64 */
static void w_set(uint64_t *w, int bit) { w[bit >> 6] |= 1ull << (bit & 63); }
static int  w_has(const uint64_t *w, int bit) { return (int)(w[bit >> 6] >> (bit & 63) & 1); }
static void w_shr1(const uint64_t *x, uint64_t *r)
{
	int i;
	for (i = 0; i < AGB_WIDE_WORDS; i++) r[i] = (x[i] >> 1) | (i + 1 < AGB_WIDE_WORDS ? x[i + 1] << 63 : 0);
}

/* the words of finish() below in 320-bit rows, for a simple literal (no '#', no -p, no LUT, one separator).
 * The "everywhere but" masks fill the words up to the one that holds the feed bit M, so that M <= 63 gives the 64-bit
 * words in word 0 and zeros above */
static int finish_wide(const build_t *b, agb_desc *d, agb_wide *w, char *err, size_t errlen)
{
	const int M = b->n, L = d->L, top = M / 64 + 1;
	int p, c, i;
	memset(w, 0, sizeof *w);
	for (i = 0; i < top; i++) { w->noerr[i] = ~0ull; w->dmask[i] = ~0ull; }
	for (i = M; i < 64 * top; i++) w_set(w->init0, i);
	w_set(w->endpos, 0);                                                       /* endp = (sep << 1) + 1 */
	for (p = 1; p <= M; p++) {
		const pos_t *q = &b->p[p];
		if (q->is_sep) { w_set(w->init0, M - p); w_set(w->endpos, M - p + 1); }
		if (q->prot) w->noerr[(M - p) >> 6] &= ~(1ull << ((M - p) & 63));
		for (c = 0; c < 256; c++) if (cls_has(q, c)) w_set(w->mask[c], M - p);
	}
	for (i = 0; i < AGB_WIDE_WORDS; i++) w->init1[i] = w->init0[i] | w->endpos[i];
	if (w_has(w->endpos, M - L)) { w_set(w->dendpos, M - L); w->endpos[(M - L) >> 6] ^= 1ull << ((M - L) & 63); }
	for (p = 1; p <= L; p++) w->dmask[(M - p) >> 6] &= ~(1ull << ((M - p) & 63));
	d->M = M;
	d->and_mode = b->and_mode;
	d->wide = 1;                                                               /* (the 64-bit words stay zero) */
	return derive(d, w, err, errlen);
}

/* derive the words from the positions (maskgen.c:218-257 with WORD = 64, LSB aligned) and the device-only constants */
static int finish(build_t *b, agb_desc *d, const agb_options *o, const unsigned char *lut, char *err, size_t errlen)
{
	int M = b->n, p, c, L = d->L;
	uint64_t sep = 0, endp;
#define BITP(q) (1ull << (M - (q)))
	d->M = M;
	d->wildmask = 0; d->noerr = ~0ull; d->init0 = ~0ull << M;
	memset(d->mask, 0, sizeof d->mask);
	for (p = 1; p <= M; p++) {
		pos_t *q = &b->p[p];
		if (q->is_sep) sep |= BITP(p);
		if (q->wild) d->wildmask |= BITP(p);
		if (q->prot) d->noerr &= ~BITP(p);
		for (c = 0; c < 256; c++) if (cls_has(q, lut ? lut[c] : c)) d->mask[c] |= BITP(p);
	}
	d->init0 |= sep;
	endp = (sep << 1) + 1;
	d->init1 = d->init0 | d->wildmask | endp;
	d->dendpos = endp & BITP(L);
	d->endpos = endp ^ d->dendpos;
	d->dmask = 0;
	for (p = 1; p <= L; p++) d->dmask |= BITP(p);
	d->dmask = ~d->dmask;
	d->and_mode = b->and_mode;
	if (o->ins_free) d->init1 = ~0ull;                                         /* bitap.c:123, asearch.c:49 */
	return derive(d, NULL, err, errlen);
}

/* post-delimiter rows: asearch.c:175-186 / bitap.c:223-225 / asearch1.c:150-158.  Row 0 is masked with
 * D_Mask BEFORE the upper rows read it, exactly as the reference orders the statements. */
static void reset_rows(const agb_desc *d, uint64_t cm, uint64_t *A)
{
	uint64_t B[2 * AGB_MAXERR + 1]; int r;
	for (r = 0; r <= d->k; r++) B[r] = d->init0;
	A[0] = (((B[0] >> 1) & cm) | (d->init1 & B[0])) & d->dmask;
	if (d->engine == AGB_ENGINE_ASEARCH1) {
		int I = d->cost_i, S = d->cost_s, DD = d->cost_d;
		for (r = 1; r <= d->k; r++) {
			uint64_t bi = (r - I >= 0) ? B[r - I] : 0, ad = (r - DD >= 0) ? A[r - DD] : 0, bs = (r - S >= 0) ? B[r - S] : 0;
			A[r] = ((B[r] >> 1) & cm) | bi | (((ad | bs) >> 1) & d->noerr) | (d->init1 & B[r]);
		}
	} else {
		for (r = 1; r <= d->k; r++)
			A[r] = ((B[r] >> 1) & cm) | (d->init1 & B[r]) | B[r - 1] | (((A[r - 1] | B[r - 1]) >> 1) & d->noerr);
	}
}

/* does position p of the delimiter accept byte c? */
static int delim_accepts(const agb_desc *d, const agb_wide *w, int c, int p)
{
	return w ? w_has(w->mask[c], d->M - p) : (int)(d->mask[c] >> (d->M - p) & 1);
}

/* reset_rows() and agbi_step() in 320-bit rows, unit costs (a simple literal is never AGB_ENGINE_ASEARCH1): one step from
 * B[0..k] on the byte of mask cm; mask0: row 0 is masked with D_Mask before the upper rows read it */
typedef uint64_t wrow_t[AGB_WIDE_WORDS];
static void w_step(const agb_desc *d, const agb_wide *w, const wrow_t *B, wrow_t *A, const uint64_t *cm, int mask0)
{
	uint64_t s[AGB_WIDE_WORDS], t[AGB_WIDE_WORDS], u[AGB_WIDE_WORDS]; int r, i;
	w_shr1(B[0], s);
	for (i = 0; i < AGB_WIDE_WORDS; i++) A[0][i] = ((s[i] & cm[i]) | (w->init1[i] & B[0][i])) & (mask0 ? w->dmask[i] : ~0ull);
	for (r = 1; r <= d->k; r++) {
		w_shr1(B[r], s);
		for (i = 0; i < AGB_WIDE_WORDS; i++) u[i] = A[r - 1][i] | B[r - 1][i];
		w_shr1(u, t);
		for (i = 0; i < AGB_WIDE_WORDS; i++) A[r][i] = (s[i] & cm[i]) | (w->init1[i] & B[r][i]) | B[r - 1][i] | (t[i] & w->noerr[i]);
	}
}

/* everything the device path needs beyond the reference's words; w: the words are those of agb_wide */
int agbi_derive(agb_desc *d, char *err, size_t errlen) { return derive(d, NULL, err, errlen); }

static int derive(agb_desc *d, agb_wide *w, char *err, size_t errlen)
{
	int L = d->L, p, r;
	uint64_t B[2 * AGB_MAXERR + 1], A[2 * AGB_MAXERR + 1];
	if (L < 1 || L > AGB_MAXDELIM || d->M < L + 1 || d->M > (w ? AGB_WIDE_MAXPOS : WIDTH - 1)) FAIL("bad descriptor (M=%d, L=%d)", d->M, L);
	if (d->k < 0 || d->k > AGB_MAXERR) FAIL("bad descriptor (k=%d)", d->k);
	if (w ? !w_has(w->dendpos, d->M - L) : !d->dendpos) FAIL("internal: delimiter end bit missing");
	/* the device also recognises delimiters away from the automaton (record starts, ordinals), by their bytes: position p
	 * of the delimiter must accept delim[p-1] and nothing else (-i with letters in the delimiter makes it accept both cases) */
	/* -p (Init1 all ones, bitap.c:123) makes every position sticky, the delimiter's too: with a delimiter of two or more
	 * bytes "a ... b" then closes a record like "ab" does.  One byte is fine (its only position is D_endpos itself). */
	if (d->init1 == ~0ull && L > 1 && !d->sticky_delim)
		FAIL("-p with a delimiter of more than one byte is not supported (insertions inside the delimiter would be free too)");
	if (d->init1 != ~0ull || L == 1) d->sticky_delim = 0;
	memset(d->delim_fold, 0, sizeof d->delim_fold);
	for (p = 1; p <= L; p++) {
		int c, cnt = 0, lo = d->delim[p - 1] | 0x20;
		for (c = 0; c < 256; c++) if (delim_accepts(d, w, c, p)) cnt++;
		if (cnt == 1 && delim_accepts(d, w, d->delim[p - 1], p)) continue;
		/* -i with a letter in the delimiter: both cases end the record (maskgen.c:52-58, 259-266) */
		if (cnt == 2 && lo >= 'a' && lo <= 'z' && delim_accepts(d, w, lo, p) && delim_accepts(d, w, lo - 32, p)) { d->delim_fold[p - 1] = 0x20; continue; }
		FAIL("the delimiter matches more than its own bytes here: not supported by the device record search");
	}
	/* delimiter recognition away from the automaton (record-start search on the device) */
	unsigned char fd[2 * AGB_MAXDELIM + 2];
	folded_delim(d, fd);
	if (d->sticky_delim) {
		/* the delimiter's state is a function of the text alone (its positions are fed by the always-on bits only): the device
		 * scans it (delim_state.cu).  Free insertions leave no piece that a match must hold verbatim: no anchors */
		d->delim_kind = 3;
		d->plan = AGB_PLAN_ALL; d->n_anchors = 0; d->n_anchors3 = 0; d->refine = 0;
	}
	else if (L == 1 || !has_border(fd, L)) d->delim_kind = 0;
	else {
		for (p = 1; p < L; p++) if (fd[p] != fd[0]) break;
		d->delim_kind = p < L ? 2 : 1;          /* a run such as $$, or any other self-overlap ("aba"): automaton.cuh delim_ends_at */
	}
	d->nrows = d->k + 1;
	if (w) {
		/* rows 0..k: reset_rows() and the virtual '\n' below, in 320 bits.  Row 0 goes to reset/start, rows 1..k to
		 * reset_up/start_up */
		wrow_t WB[AGB_MAXERR + 1], RA[AGB_MAXERR + 1], SA[AGB_MAXERR + 1]; int i, hit = 0;
		for (r = 0; r <= d->k; r++) memcpy(WB[r], w->init0, sizeof WB[r]);
		w_step(d, w, (const wrow_t *)WB, RA, w->mask[d->delim[L - 1]], 1);
		w_step(d, w, (const wrow_t *)WB, SA, w->mask['\n'], 0);
		for (i = 0; i < AGB_WIDE_WORDS; i++) hit |= (SA[0][i] & w->dendpos[i]) != 0;
		d->start_closes = hit;
		if (hit) memcpy(SA, RA, sizeof SA);
		memcpy(w->reset, RA[0], sizeof w->reset); memcpy(w->start, SA[0], sizeof w->start);
		for (r = 1; r <= d->k; r++) { memcpy(w->reset_up[r - 1], RA[r], sizeof RA[r]); memcpy(w->start_up[r - 1], SA[r], sizeof SA[r]); }
		return 0;
	}
	reset_rows(d, d->mask[d->delim[L - 1]], d->reset);
	/* the virtual '\n' in front of the text (bitap.c:140,148-149) */
	for (r = 0; r <= d->k; r++) B[r] = d->init0;
	agbi_step(d, B, A, d->mask['\n']);
	if (A[0] & d->dendpos) { d->start_closes = 1; memcpy(d->start, d->reset, sizeof(uint64_t) * (size_t)(d->k + 1)); }
	else { d->start_closes = 0; memcpy(d->start, A, sizeof(uint64_t) * (size_t)(d->k + 1)); }
	return 0;
}

/* pigeonhole anchor plan: k errors can damage at most k of k+1 disjoint runs of consecutive literal
 * positions, so a matching record contains one run verbatim (the idea of sgrep.c:1053-1154, made exact). */
/* the bytes a position accepts, when they are at most two (a literal, or a class such as [ea]); 0: not usable in an anchor */
static int pos_values(const pos_t *q, int ascii_only, int literal_only, int *vals)
{
	int c, n = 0;
	if (q->is_sep || (literal_only && q->lit < 0)) return 0;
	if (q->lit >= 0) {
		/* ascii_only (-i): the exact engine folds bytes >= 0x80 through the ISO-8859-1 LUT (bitap.c:171), which the
		 * anchors' plain 0x20 fold cannot express -- such bytes never sit inside an anchor */
		if (q->lit == '\n' || (ascii_only && q->lit >= 0x80)) return 0;
		vals[0] = q->lit; return 1;
	}
	for (c = 0; c < 256; c++) if ((q->cls[c >> 6] >> (c & 63)) & 1) {
		/* (under -i the class holds both cases and the anchors are compared with 0x20 OR-ed in: one value per letter) */
		const int v = (ascii_only && is_alpha(c)) ? (c | 0x20) : c;
		if (c == '\n' || (ascii_only && c >= 0x80)) return 0;
		if (n && (vals[0] == v || (n == 2 && vals[1] == v))) continue;
		if (n == 2) return 0;
		vals[n++] = v;
	}
	return n;
}

#define PIECE_VARIANTS 4
typedef struct { int where, nvar; uint32_t v[PIECE_VARIANTS]; } piece_t;

/* disjoint runs of A consecutive positions that each accept one byte -- or two, as long as a run spells at most
 * PIECE_VARIANTS strings: "b[ea]c" is the two anchors "bec" and "bac" at the same place */
static int collect_runs(const build_t *b, int part, int A, int ascii_only, int literal_only, piece_t *out, int cap)
{
	int p, run = 0, n = 0;
	for (p = 1; p <= b->n; p++) {
		const pos_t *q = &b->p[p];
		int vals[2];
		if (q->part != part || !pos_values(q, ascii_only, literal_only, vals)) { run = 0; continue; }
		if (++run == A) {
			piece_t pc; int t, nv = 1, i;
			pc.where = p - A + 1; pc.v[0] = 0;
			for (t = 0; t < A && nv; t++) {
				int vv[2], m = pos_values(&b->p[p - A + 1 + t], ascii_only, literal_only, vv), old = nv;
				if (nv * m > PIECE_VARIANTS) { nv = 0; break; }
				for (i = 0; i < old; i++) {
					const uint32_t base = pc.v[i];
					pc.v[i] = base | (uint32_t)(vv[0] & 0xFF) << (8 * t);
					if (m == 2) pc.v[nv++] = base | (uint32_t)(vv[1] & 0xFF) << (8 * t);
				}
			}
			pc.nvar = nv;
			if (nv && n < cap) out[n++] = pc;
			run = 0;
		}
		if (q->wild) run = 0;     /* '#' behind q: free insertions there, a verbatim run cannot continue through it */
	}
	return n;
}

static void plan_anchors(const build_t *b, agb_desc *d, const agb_options *o, int fold_all)
{
	int A, p, part, step;
	d->plan = AGB_PLAN_ALL; d->n_anchors = 0; d->n_anchors3 = 0; d->adaptive = 1;
	/* -p makes insertions free: no piece need survive.  -v reports the NON-matching records: the anchors cannot point at
	 * them, so the plan stays AGB_PLAN_ALL -- but the pieces are worked out all the same (see the returns below): a count of
	 * non-matching records is the number of records minus the matching ones (scan.cu, the complement count) */
	if (o->ins_free) return;
	/* per anchor length: literal runs first, then runs that may hold two-valued classes (more anchors for the same pieces) */
	for (step = 0; step < 6; step++) {
		const int lit_only = !(step & 1);
		A = 4 - step / 2;
		uint32_t got[AGB_MAXANCHOR]; int pos[AGB_MAXANCHOR], ngot = 0, ok = 1, classes = 0;
		piece_t pcs[AGB_MAXANCHOR]; int i, v;
#define TAKE_PIECES(arr, cnt) do { \
			for (i = 0; i < (cnt) && ok; i++) for (v = 0; v < (arr)[i].nvar; v++) { \
				if (ngot >= AGB_MAXANCHOR) { ok = 0; break; } \
				got[ngot] = (arr)[i].v[v]; pos[ngot++] = (arr)[i].where; if ((arr)[i].nvar > 1) classes = 1; \
			} } while (0)
		if (b->or_seen) {                    /* a,b : any alternative may match -> k+1 runs from each */
			for (part = 1; part <= b->nparts && ok; part++) {
				int nt = collect_runs(b, part, A, o->nocase || fold_all, lit_only, pcs, AGB_MAXANCHOR);
				if (nt < d->k + 1) ok = 0; else TAKE_PIECES(pcs, d->k + 1);
			}
		} else {                             /* single pattern or a;b (all must match): the part richest in runs */
			int best = -1, bestpart = 0;
			for (part = 1; part <= b->nparts; part++) {
				int nt = collect_runs(b, part, A, o->nocase || fold_all, lit_only, pcs, AGB_MAXANCHOR);
				if (nt > best) { best = nt; bestpart = part; }
			}
			if (best < d->k + 1) ok = 0;
			else { collect_runs(b, bestpart, A, o->nocase || fold_all, lit_only, pcs, AGB_MAXANCHOR); TAKE_PIECES(pcs, d->k + 1); }
		}
#undef TAKE_PIECES
		if (!ok) continue;
		d->plan = AGB_PLAN_ANCHORS; d->anchor_len = A;
		d->anchor_mask = (A == 4) ? 0xFFFFFFFFu : (A == 3 ? 0x00FFFFFFu : 0x0000FFFFu);
		/* case folding: the SAME 0x20 is OR-ed into every byte of the text words and of the anchors (a window
		 * is cut from two words at any byte offset, so the fold must not depend on the byte lane).  Both
		 * sides are folded alike, so this only widens the filter ('@' and '`' fall together, etc.). */
		d->anchor_fold = 0;
		if (o->nocase || fold_all)
			for (p = 0; p < ngot; p++) {
				int t;
				for (t = 0; t < A; t++) if (is_alpha((int)(got[p] >> (8 * t) & 0xFF))) d->anchor_fold = 0x20202020u;
			}
		/* stage 1.5: a hit of anchor i at text offset t can only belong to a match inside
		 * [t - off_i - k, t + pat_len - off_i + k) when the pattern is a single part without '#' */
		d->pat_len = d->M - d->L - 1;
		d->n_anchors = 0;
		for (p = 0; p < ngot; p++) {
			const uint32_t val = (got[p] | d->anchor_fold) & d->anchor_mask; int dup = 0;
			for (i = 0; i < d->n_anchors; i++) if (d->anchor[i] == val && d->anchor_off[i] == pos[p] - (d->L + 2)) dup = 1;   /* [eE] under -i */
			if (dup) continue;
			d->anchor[d->n_anchors] = val; d->anchor_off[d->n_anchors++] = pos[p] - (d->L + 2);
		}
		/* (320-bit rows: no stage 1.5 -- the record stage judges the flagged chunks) */
		d->refine = (b->nparts == 1 && !b->and_mode && !b->or_seen && d->wildmask == 0 && !d->wide) ? 1 : 0;
		/* the planner in scan.cu re-derives plans from the literal positions alone: not for a plan that leans on classes */
		if (classes) d->adaptive = 0;
		if (d->inverse) d->plan = AGB_PLAN_ALL;       /* (the anchors stay in the descriptor for the complement count) */
		return;
	}
}

/* checksg.c:43-122 */
static int simple_pattern(const unsigned char *s, int m, int k, int *notsgrep)
{
	int i;
	*notsgrep = 0;
	for (i = 0; i < m; i++) {
		if (strchr(";,.*-[]()<>|#{}~", s[i])) return 0;
		if (s[i] == '^' || s[i] == '$') { *notsgrep = 1; return k > 0 ? 0 : 1; }
		if (s[i] == '\\') i++;
	}
	return 1;
}

static int parse_delim(const agb_options *o, build_t *b, agb_desc *d, char *err, size_t errlen)
{
	/* agrep.c:2272-2314 builds "<X>; "; preproce.c:181-210 walks it; bitap.c:92-94 maps ^,$ to '\n' */
	d->L = 0; d->user_delim = 0; d->outtail = 0;
	if (!o->delim) {
		pos_t *p = new_pos(b);
		p->prot = 1; cls_set(p, '\n');
		d->delim[d->L++] = '\n';
	} else {
		const unsigned char *s = (const unsigned char *)o->delim; size_t n = strlen(o->delim), i;
		if (n < 1) FAIL("the -d option must have a delimiter argument");
		if (n > 16) FAIL("delimiter pattern too long (has > %d chars)", 16);
		if (n == 1 && (s[0] == '\n' || s[0] == '$' || s[0] == '^')) d->outtail = 1;
		d->user_delim = 1;
		b->no_error = 1; b->even = 1;                  /* the '<' agrep.c:2287 puts in front */
		for (i = 0; i < n; i++) {
			int c = s[i]; pos_t *p;
			if (c == '\\') { if (++i >= n) break; c = s[i]; }
			else if (c == '<') { b->no_error = 1; b->even++; continue; }
			else if (c == '>') { b->no_error = 0; b->even--; continue; }
			else if (c == '^' || c == '$') c = '\n';
			if (c >= 129 && c <= 145) FAIL("byte %d in the delimiter collides with an internal symbol", c);
			if (d->L >= AGB_MAXDELIM) FAIL("delimiter pattern too long (has > %d chars)", AGB_MAXDELIM);
			p = new_pos(b);
			if (c == '\n' || b->no_error) p->prot = 1;
			cls_set(p, c);
			/* -i lower-cases the WHOLE internal pattern, the delimiter included, and copies every lower-case mask to its
			 * upper-case byte (maskgen.c:52-58, 259-266): 'x' and 'X' both end a record then.  Stated here as it is;
			 * agbi_derive() refuses it, because the device finds delimiters by their bytes. */
			if (o->nocase && is_alpha(c)) { cls_set(p, c | 32); cls_set(p, (c | 32) - 32); }
			d->delim[d->L++] = (unsigned char)c;
		}
		b->no_error = 0; b->even--;                    /* the closing '>' */
		if (b->even != 0) FAIL("unmatched '<', '>' in the delimiter");
		if (d->L < 1) FAIL("empty delimiter");
	}
	return 0;
}

/* ================================================================================================
 * regular expressions (REGEX): the syntax of parse.c:181-237, the positions of maskgen.c, the follow sets of
 * follow.c:210-255 as a Glushkov construction (first, last, nullable), in 64-bit words: up to 63 positions where the
 * reference stops at 30 (preproce.c:378).  The pattern is wrapped as ".( ... )." (preproce.c:231-236, 334-339):
 * position 1 is the leading '.', which the start state already holds (HEAD), position M the trailing one that the match
 * test reads (bit 0).  '?' is the optional operator parse.c:220 means it to be (the reference also counts it as a
 * literal position in maskgen(), so its bits no longer line up: SURVEY 8c).
 * ============================================================================================== */
typedef struct { uint64_t first, last; int nullable; } rx_frag;   /* sets of positions: bit p = position p */
typedef struct {
	build_t *b; const unsigned char *s; int i, n; const agb_options *o;
	uint64_t fol[WIDTH + 1];                                     /* bit q of fol[p]: position q may follow p */
	int and_seen;                                                /* a ';' was met (it never reaches parse(), preproce.c:308-311) */
	char *err; size_t errlen;
} rx_parser;

/* an unescaped '|' or '*' makes the pattern a regular expression (preproce.c:139-142) */
static int is_regex(const unsigned char *s, int m)
{
	int i;
	for (i = 0; i < m; i++) {
		if (s[i] == '\\') i++;
		else if (s[i] == '|' || s[i] == '*') return 1;
	}
	return 0;
}

static void rx_link(rx_parser *P, uint64_t from, uint64_t to)
{
	int p;
	for (p = 1; p < WIDTH; p++) if (from >> p & 1) P->fol[p] |= to;
}

static int rx_alt(rx_parser *P, rx_frag *out);

static int rx_atom(rx_parser *P, rx_frag *f)
{
	build_t *b = P->b; const unsigned char *s = P->s; const int n = P->n;
	char *err = P->err; size_t errlen = P->errlen;
	int c = s[P->i];
	pos_t *p;
	if (c == '(') {
		P->i++;
		if (rx_alt(P, f)) return AGB_ERR_PATTERN;
		if (P->i >= n || s[P->i] != ')') FAIL("illegal regular expression");
		P->i++;
		return 0;
	}
	if (c == '[') {
		if (add_class(b, s, &P->i, n, P->o, 1, err, errlen)) return AGB_ERR_PATTERN;
		P->i++;
	} else if (c == '\\') {
		if (P->i + 1 >= n) FAIL("illegal regular expression");
		P->i++;
		if (add_literal(b, s[P->i], P->o->nocase, err, errlen)) FAIL("regular expression too long");
		P->i++;
	} else if (c == '.' || c == '#') {                       /* '#' is ".*" under REGEX (preproce.c:247-253) */
		if (!(p = new_pos(b))) FAIL("regular expression too long");
		if (b->no_error) p->prot = 1;
		cls_range(p, S_NOCARE, S_NOCARE); cls_set(p, '\n');  /* NOCARE takes '\n' too under REGEX (maskgen.c:243) */
		P->i++;
	} else if (c == '^' || c == '$') {                       /* a newline position (preproce.c:281-290) */
		if (add_literal(b, '\n', 0, err, errlen)) FAIL("regular expression too long");
		P->i++;
	} else if (c == '*' || c == '?' || c == '|' || c == ')' || c == ']' || c == ',' || c == ';') {
		FAIL("illegal regular expression");                  /* RE_ERR (preproce.c:299-306), or parse() fails */
	} else {
		if (c >= 129 && c <= 145) FAIL("byte %d in the pattern collides with an internal symbol (agrep.h:69-87)", c);
		if (add_literal(b, c, P->o->nocase, err, errlen)) FAIL("regular expression too long");
		P->i++;
	}
	f->first = f->last = 1ull << b->n;
	f->nullable = 0;
	if (c == '#') { rx_link(P, f->last, f->first); f->nullable = 1; }
	return 0;
}

/* concatenation of starred / optional atoms; '<' '>' switch the error protection as elsewhere (maskgen.c:80-95) */
static int rx_cat(rx_parser *P, rx_frag *out)
{
	build_t *b = P->b; const unsigned char *s = P->s;
	char *err = P->err; size_t errlen = P->errlen;
	int any = 0;
	while (P->i < P->n && s[P->i] != '|' && s[P->i] != ')') {
		rx_frag f;
		if (s[P->i] == ';') { P->and_seen = 1; P->i++; continue; }
		if (s[P->i] == '<') { b->no_error = 1; b->even++; P->i++; continue; }
		if (s[P->i] == '>') { b->no_error = 0; if (--b->even < 0) FAIL("unmatched '<', '>' (use \\<, \\> to search for <, >)"); P->i++; continue; }
		if (rx_atom(P, &f)) return AGB_ERR_PATTERN;
		while (P->i < P->n && (s[P->i] == '*' || s[P->i] == '?')) {
			if (s[P->i] == '*') rx_link(P, f.last, f.first);
			f.nullable = 1;
			P->i++;
		}
		if (!any) *out = f;
		else {
			rx_link(P, out->last, f.first);
			out->first |= out->nullable ? f.first : 0;
			out->last = f.last | (f.nullable ? out->last : 0);
			out->nullable = out->nullable && f.nullable;
		}
		any = 1;
	}
	if (!any) FAIL("illegal regular expression");
	return 0;
}

static int rx_alt(rx_parser *P, rx_frag *out)
{
	if (rx_cat(P, out)) return AGB_ERR_PATTERN;
	while (P->i < P->n && P->s[P->i] == '|') {
		rx_frag f;
		P->i++;
		if (rx_cat(P, &f)) return AGB_ERR_PATTERN;
		out->first |= f.first; out->last |= f.last; out->nullable = out->nullable || f.nullable;
	}
	return 0;
}

uint64_t agbi_regex_next(const agb_regex *rx, int M, uint64_t S)
{
	uint64_t r = 0; int p;
	for (p = 0; p <= M; p++) if (S >> (M - p) & 1) r |= rx->follow[p];
	return r;
}

/* the rows right after a newline: Init[i] = Init[i-1] | Next(Init[i-1]) (agrep.c:1289), then the newline fed through
 * every row (agrep.c:1649-1658).  Every line starts from them, the first one too (the virtual '\n' in front of the text) */
static int rx_derive(agb_desc *d, const agb_regex *rx, char *err, size_t errlen)
{
	uint64_t B[AGB_MAXERR + 1], A[AGB_MAXERR + 1], m; int r, M = d->M;
	if (d->engine != AGB_ENGINE_REGEX) FAIL("bad descriptor (not a regular expression)");
	if (M < 2 || M > AGB_REGEX_MAXPOS) FAIL("regular expression too long");
	if (d->k < 0 || d->k > 4) FAIL("the maximum number of erorrs allowed for full regular expressions is 4");   /* bitap.c:96-104 */
	if (d->L != 1 || d->delim[0] != '\n') FAIL("-d or -w option is not supported for this pattern");
	m = d->mask['\n'];
	B[0] = d->init0;
	for (r = 1; r <= d->k; r++) B[r] = B[r - 1] | agbi_regex_next(rx, M, B[r - 1]);
	A[0] = (agbi_regex_next(rx, M, B[0]) & m) | (d->init1 & B[0]);
	for (r = 1; r <= d->k; r++)
		A[r] = (agbi_regex_next(rx, M, B[r]) & m) | (d->init1 & B[r]) | ((B[r - 1] | agbi_regex_next(rx, M, A[r - 1] | B[r - 1])) & d->noerr);
	memset(d->reset, 0, sizeof d->reset); memset(d->start, 0, sizeof d->start);
	memcpy(d->reset, A, sizeof(uint64_t) * (size_t)(d->k + 1));
	memcpy(d->start, A, sizeof(uint64_t) * (size_t)(d->k + 1));
	d->start_closes = 1;                         /* the virtual '\n' closes the (never reported) line in front of the text */
	d->nrows = d->k + 1;
	d->delim_kind = 0; memset(d->delim_fold, 0, sizeof d->delim_fold);
	d->plan = AGB_PLAN_ALL; d->n_anchors = 0; d->n_anchors3 = 0; d->adaptive = 0; d->refine = 0;
	return 0;
}

static int rx_build(const unsigned char *s, int m, const agb_options *o, agb_desc *d, agb_regex *rx, char *err, size_t errlen)
{
	rx_parser P; rx_frag u; build_t *b; pos_t *p; int M, q, c, rc = 0;
	/* preproce.c:347-364, 378; compat.c:75-79 (-I/-S/-D are ignored, the command line says so) */
	if (o->delim || o->wordbound) FAIL("-d or -w option is not supported for this pattern");
	if (o->wholeline) FAIL("-x is not supported for regular expressions");
	{   /* RE_ERR (preproce.c:299-311): any ',', or a second ';' */
		int i, ors = 0, ands = 0;
		for (i = 0; i < m; i++) {
			if (s[i] == '\\') i++;
			else if (s[i] == ',') ors++;
			else if (s[i] == ';') ands++;
		}
		if (ors || ands > 1) FAIL("illegal regular expression");
	}
	b = (build_t *)calloc(1, sizeof *b);
	if (!b) FAIL("out of memory");
	memset(&P, 0, sizeof P);
	P.b = b; P.s = s; P.i = 0; P.n = m; P.o = o; P.err = err; P.errlen = errlen;
	p = new_pos(b);                                          /* the leading '.' */
	cls_range(p, S_NOCARE, S_NOCARE); cls_set(p, '\n');
	rc = rx_alt(&P, &u);
	if (!rc && P.i < m) { rc = AGB_ERR_PATTERN; if (err && errlen) snprintf(err, errlen, "illegal regular expression"); }   /* an unmatched ')' */
	if (!rc && b->even != 0) { rc = AGB_ERR_PATTERN; if (err && errlen) snprintf(err, errlen, "unmatched '<', '>' (use \\<, \\> to search for <, >)"); }
	/* one ';' passes preprocess() and parse() and is refused by maskgen() (maskgen.c:150-163) */
	if (!rc && P.and_seen) { rc = AGB_ERR_PATTERN; if (err && errlen) snprintf(err, errlen, "illegal pattern: cannot handle AND (';') and OR (',')/regular-expressions simultaneously"); }
	if (!rc) {
		p = new_pos(b);                                      /* the trailing '.' */
		if (!p) { rc = AGB_ERR_PATTERN; if (err && errlen) snprintf(err, errlen, "regular expression too long"); }
		else { cls_range(p, S_NOCARE, S_NOCARE); cls_set(p, '\n'); }
	}
	if (rc) { free(b); return rc; }
	M = b->n;
	P.fol[0] = 1ull << 1;
	P.fol[1] |= u.first | (u.nullable ? 1ull << M : 0);
	rx_link(&P, u.last, 1ull << M);
	memset(rx, 0, sizeof *rx);
	rx->head = 1; rx->tail = 1;
	for (q = 0; q <= M; q++) {
		int t;
		for (t = 1; t <= M; t++) if (P.fol[q] >> t & 1) rx->follow[q] |= 1ull << (M - t);
	}
	/* the words (maskgen.c:218-257 under REGEX) */
	d->M = M; d->engine = AGB_ENGINE_REGEX; d->k = o->k; d->inverse = o->inverse != 0;
	d->cost_i = d->cost_s = d->cost_d = 1;
	d->L = 1; d->delim[0] = '\n'; d->user_delim = 0; d->outtail = 0; d->and_mode = 0;
	d->noerr = ~0ull; d->wildmask = 0; d->dmask = ~0ull; d->dendpos = 0; d->endpos = 1;
	memset(d->mask, 0, sizeof d->mask);
	for (q = 1; q <= M; q++) {
		const pos_t *pq = &b->p[q];
		if (pq->prot) d->noerr &= ~(1ull << (M - q));
		for (c = 0; c < 256; c++) if (cls_has(pq, c)) d->mask[c] |= 1ull << (M - q);
	}
	d->init0 = (1ull << M) | (rx->head ? 1ull << (M - 1) : 0);   /* Init[0] = Bit[base] | Bit[base+1] (agrep.c:1285-1286) */
	d->init1 = d->init0 | 1;
	free(b);
	return rx_derive(d, rx, err, errlen);
}

int agbi_build(const char *pattern, const agb_options *o, agb_desc *d, char *err, size_t errlen)
{
	return agbi_build_rx(pattern, o, d, NULL, NULL, err, errlen);
}

int agbi_build_rx(const char *pattern, const agb_options *o, agb_desc *d, agb_regex *rx, agb_wide *wide, char *err, size_t errlen)
{
	build_t *b; int m, rc, notsgrep = 0, simple, jump, sg; unsigned char lut[256];
	const unsigned char *s = (const unsigned char *)pattern;
	memset(d, 0, sizeof *d);
	if (!pattern || !o) FAIL("null argument");
	m = (int)strlen(pattern);
	if (m < 1) FAIL("pattern length %d too small", m);                         /* agrep.c:3052 */
	if (m >= 256) FAIL("pattern '%s' too long", pattern);                      /* agrep.c:3057 */
	if (o->k < 0 || o->k > AGB_MAXERR) FAIL("the maximum number of errors is %d", AGB_MAXERR);   /* agrep.c:2713 */
	if (m <= o->k) FAIL("size of pattern '%s' must be > #of errors %d", pattern, o->k);          /* checksg.c:34 */
	if (o->wordbound && o->wholeline) FAIL("illegal option combination (-x and -w)");            /* agrep.c:2194 */
	if (o->delim && o->wholeline) FAIL("-d and -x are not compatible");                          /* compat.c */
	if (o->regex && is_regex(s, m)) {
		/* the -B sweeps of this library (agb_bestmatch_*) rebuild the pattern at k = 2, 4, 8: not for re() */
		if (!rx) FAIL("-B (best match) is not supported for regular expressions by the device sweep; scan with k = 0..4");
		return rx_build(s, m, o, d, rx, err, errlen);
	}
	jump = (o->cost_i || o->cost_s || o->cost_d);
	if (jump && (o->cost_i < 0 || o->cost_s < 0 || o->cost_d < 0)) FAIL("the error cost cannot be 0");
	d->k = o->k; d->inverse = o->inverse != 0;
	d->cost_i = o->cost_i ? o->cost_i : 1; d->cost_s = o->cost_s ? o->cost_s : 1; d->cost_d = o->cost_d ? o->cost_d : 1;
	if (d->cost_i > d->k) d->cost_i = d->k + 1;                                /* asearch1.c:42-44 */
	if (d->cost_s > d->k) d->cost_s = d->k + 1;
	if (d->cost_d > d->k) d->cost_d = d->k + 1;

	/* engine choice: checksg.c:124-144 then bitap.c:96-121, asearch.c:50-52 */
	simple = simple_pattern(s, m, o->k, &notsgrep);
	sg = simple && !o->bestmatch && !(o->nocase && o->k > 0) && !jump && !o->ins_free && !o->linenum
	     && !(o->wordbound && o->k > 0) && !(o->wholeline && o->k > 0) && !notsgrep;
	if (sg && o->k == 0 && !o->wholeline) d->engine = AGB_ENGINE_SGREP_BM;   /* also under -d: checksg() does not look at the delimiter */
	else if (o->k > 0 && jump) d->engine = AGB_ENGINE_ASEARCH1;
	else if (o->k > 4) d->engine = AGB_ENGINE_ASEARCH0;
	else if (o->k > 0) d->engine = AGB_ENGINE_ASEARCH;     /* also simple k>0 literals: the reference's sgrep filters are lossy (SURVEY 8c) */
	else d->engine = AGB_ENGINE_BITAP;

	b = (build_t *)calloc(1, sizeof *b);
	if (!b) FAIL("out of memory");
	rc = parse_delim(o, b, d, err, errlen);
	if (!rc) rc = add_sep(b, 1, d->L, err, errlen);                            /* preproce.c:221: ANDPAT after the delimiter */
	b->and_mode = 0;
	if (!rc && d->engine == AGB_ENGINE_SGREP_BM) {
		/* sgrep.c:289-320 + bm() :741-755: literal compared under TR[] (ASCII case folded, unconditional,
		 * sgrep.c:226-236); -w = neither neighbour isalnum().  Stated as an exact automaton. */
		int i;
		b->wide_ok = wide != NULL;                                             /* (sgrep() takes up to 255 characters) */
		if (o->wordbound) { pos_t *p = new_pos(b); int c; if (p) { p->prot = 1; for (c = 0; c < 256; c++) if (!is_alnum(c)) cls_set(p, c); } else rc = AGB_ERR_PATTERN; }
		for (i = 0; i < m && !rc; i++) {
			int c = s[i]; pos_t *p;
			if (c == '\\') { if (++i >= m) break; c = s[i]; }
			p = new_pos(b);
			if (!p) { rc = AGB_ERR_PATTERN; if (err) snprintf(err, errlen, "pattern too long (has > %d chars)", WIDTH); break; }
			if (is_upper(c)) c += 32;
			cls_set(p, c); if (is_alpha(c)) cls_set(p, c - 32);
			p->lit = c;
			if (c == '\n') p->prot = 1;
		}
		if (!rc && o->wordbound) { pos_t *p = new_pos(b); int c; if (p) { p->prot = 1; for (c = 0; c < 256; c++) if (!is_alnum(c)) cls_set(p, c); } else rc = AGB_ERR_PATTERN; }
	} else if (!rc) {
		/* a simple literal at k > 0, which the reference hands to sgrep() too: as many positions when the caller asks for it */
		b->wide_ok = wide != NULL && sg && o->k > 0 && o->wide_approx;
		if (o->wholeline) {                                                    /* preproce.c:148-159, maskgen.c:188-193 */
			pos_t *p = new_pos(b); if (p) { p->prot = 1; cls_set(p, '\n'); cls_set(p, S_NNLINE); } else rc = AGB_ERR_PATTERN;
		} else if (o->wordbound) rc = add_wordb(b, err, errlen);               /* preproce.c:161-166 */
		if (!rc) rc = add_pattern(b, s, m, o, d->L, err, errlen);
		if (!rc && o->wholeline) { pos_t *p = new_pos(b); if (p) { p->prot = 1; cls_set(p, '\n'); } else rc = AGB_ERR_PATTERN; }
		else if (!rc && o->wordbound) rc = add_wordb(b, err, errlen);          /* preproce.c:169-173 */
	}
	if (rc) { if (err && errlen && !err[0]) snprintf(err, errlen, "pattern too long (has > %d chars)", WIDTH); free(b); return AGB_ERR_PATTERN; }
	d->sticky_delim = o->sticky_delim ? 1 : 0;                                  /* (derive() keeps it only where -p meets L >= 2) */
	if (d->engine == AGB_ENGINE_BITAP && o->nocase) { agbi_lut_lower1(lut); rc = finish(b, d, o, lut, err, errlen); }
	else if (b->wide_ok && (b->n > WIDTH - 1 || (getenv("AGB_FORCE_WIDE") && atoi(getenv("AGB_FORCE_WIDE")) == 1)))
		rc = finish_wide(b, d, wide, err, errlen);                             /* (AGB_FORCE_WIDE=1: every such literal, for tests) */
	else rc = finish(b, d, o, NULL, err, errlen);
	if (!rc) plan_anchors(b, d, o, d->engine == AGB_ENGINE_SGREP_BM);
	free(b);
	return rc;
}

/* ---- public wrappers ---- */
int agb_compile(const char *pattern, const agb_options *opt, agb_pattern **out, char *err, size_t errlen)
{
	agb_pattern *p; int rc;
	if (err && errlen) err[0] = 0;
	if (!out) return AGB_ERR_ARG;
	p = (agb_pattern *)calloc(1, sizeof *p);
	if (!p) return AGB_ERR_NOMEM;
	rc = agbi_build_rx(pattern, opt, &p->d, &p->rx, &p->wide, err, errlen);
	if (rc) { free(p); *out = NULL; return rc; }
	*out = p;
	return AGB_OK;
}

const agb_regex *agb_pattern_regex(const agb_pattern *p) { return (p && p->d.engine == AGB_ENGINE_REGEX) ? &p->rx : NULL; }
const agb_wide *agb_pattern_wide(const agb_pattern *p) { return (p && p->d.wide) ? &p->wide : NULL; }

int agb_pattern_from_regex(const agb_desc *d, const agb_regex *rx, agb_pattern **out, char *err, size_t errlen)
{
	agb_pattern *p; int rc, q;
	if (err && errlen) err[0] = 0;
	if (!d || !rx || !out) return AGB_ERR_ARG;
	p = (agb_pattern *)calloc(1, sizeof *p);
	if (!p) return AGB_ERR_NOMEM;
	p->d = *d; p->rx = *rx;
	p->d.wide = 0;
	/* nothing outside positions 0..M */
	if (p->d.M >= 1 && p->d.M <= AGB_REGEX_MAXPOS) {
		const uint64_t field = (p->d.M == 63) ? ~0ull : (2ull << p->d.M) - 1;
		for (q = 0; q <= AGB_REGEX_MAXPOS; q++) p->rx.follow[q] = q <= p->d.M ? p->rx.follow[q] & field : 0;
	}
	rc = rx_derive(&p->d, &p->rx, err, errlen);
	if (rc) { free(p); *out = NULL; return rc; }
	*out = p;
	return AGB_OK;
}

int agb_pattern_from_desc(const agb_desc *d, agb_pattern **out, char *err, size_t errlen)
{
	agb_pattern *p; int rc;
	if (err && errlen) err[0] = 0;
	if (!d || !out) return AGB_ERR_ARG;
	p = (agb_pattern *)calloc(1, sizeof *p);
	if (!p) return AGB_ERR_NOMEM;
	p->d = *d;
	/* the caller may bring its own anchor plan (the drop-in layer derives one from the reference's internal pattern) */
	if (p->d.plan != AGB_PLAN_ANCHORS || p->d.n_anchors < 1 || p->d.n_anchors > AGB_MAXANCHOR || p->d.anchor_len < 2 || p->d.anchor_len > 4) {
		p->d.plan = AGB_PLAN_ALL; p->d.n_anchors = 0; p->d.refine = 0;
	}
	if (p->d.n_anchors3 < 0 || p->d.n_anchors3 > 2 || p->d.plan != AGB_PLAN_ANCHORS) p->d.n_anchors3 = 0;
	p->d.pair_plan = 0;
	p->d.wide = 0;                 /* (the words must be in the descriptor: a descriptor of 320-bit rows is refused below) */
	rc = agbi_derive(&p->d, err, errlen);
	if (rc) { free(p); *out = NULL; return rc; }
	*out = p;
	return AGB_OK;
}

void agb_pattern_free(agb_pattern *p) { free(p); }
const agb_desc *agb_pattern_desc(const agb_pattern *p) { return p ? &p->d : NULL; }

/* j of the reference's loops (bitap.c:178, asearch.c:120): incremented at every record close, the virtual '\n'
 * included; pre-decremented when the text starts with the user's delimiter (bitap.c:151-156; asearch0() has no
 * such correction, asearch.c:609-612).  Same greedy delimiter rule as the device (scan.cu delim_ends_at), and for
 * delim_kind 3 the delimiter's state machine of delim_state.cu. */
void agb_fill_ordinals(const agb_pattern *p, const void *h_text, uint64_t n, agb_record *records, uint64_t n_records)
{
	const agb_desc *d = &p->d; const unsigned char *t = (const unsigned char *)h_text;
	const int L = d->L; uint64_t i = 0; long long j = 0, run = 0, q, taken = -(1ll << 60); unsigned char fd[2 * AGB_MAXDELIM + 2]; int z, head = 1;
	if (!n_records) return;
	folded_delim(d, fd);
#define DEQ(c, p) ((((c) | d->delim_fold[p]) & 0x1FF) == fd[p])
	(void)z; (void)head;
	/* (byte for byte against the delimiter as typed, also under -i: bitap.c:151-154 compares old_D_pat) */
	if (d->user_delim && d->engine != AGB_ENGINE_ASEARCH0 && n >= (uint64_t)L && memcmp(t, d->delim, (size_t)L) == 0) j = -1;
	/* position q = -1 is the virtual '\n'; positions n .. n+L-1 are the delimiter appended at EOF */
	for (q = -1; q < (long long)n + L && i < n_records; q++) {
		int c = q < 0 ? '\n' : (q < (long long)n ? t[q] : d->delim[q - (long long)n]), e;
		if (d->delim_kind == 3) {
			/* -p: position run + 1 of the delimiter takes c or not; the L-th closes and starts over (DESIGN 3.3.1) */
			if (DEQ(c, run) && ++run == L) run = 0, e = 1; else e = 0;
		}
		else if (L == 1) e = DEQ(c, 0);
		else if (d->delim_kind == 1) { run = DEQ(c, 0) ? run + 1 : 0; e = run > 0 && run % L == 0; }
		else if (d->delim_kind == 2) {
			/* occurrences are taken from the left; one that shares a byte with the one taken before it is dropped */
			int m = 1, u;
			for (u = 0; u < L && m; u++) {
				long long at = q - u; int cc = at < -1 ? 256 : (at < 0 ? '\n' : (at < (long long)n ? t[at] : d->delim[at - (long long)n]));
				if (!DEQ(cc, L - 1 - u)) m = 0;
			}
			e = m && q - L + 1 > taken;
			if (e) taken = q;
		}
		else {
			int m = 1, u;
			for (u = 0; u < L && m; u++) {
				long long at = q - u; int cc = at < -1 ? 256 : (at < 0 ? '\n' : (at < (long long)n ? t[at] : d->delim[at - (long long)n]));
				if (!DEQ(cc, L - 1 - u)) m = 0;
			}
			e = m;
		}
		if (!e) continue;
		j++;
		while (i < n_records && records[i].end + L - 1 == q) records[i++].ordinal = j;
	}
}
