"""The pair plan (DESIGN.md 3.1) modelled on the host, and the planted texts its tests scan.  Needs no device: the CPU
tests check the model against the checker, the GPU tests check the device against both.

  * positions() / pair_pieces(): scan.cu's pair_pieces() over the pattern's positions as adaptive_plan() reads them from
    the masks -- one byte, or None where a position is not one literal (`.`, the -w/-x wrapper positions);
  * flagged_chunks(): the chunk rule of stage 1 under the pair plan (front.cu pair_chunks);
  * CASES, sites(), record(), planted_text(): records planted so that the earlier of two surviving pieces starts `lead`
    bytes before a chunk, warp, stage, host-slice or window boundary, or in the last record of the text."""
from collections import namedtuple

MIB = 1 << 20
CHUNK = 16                 # one bitmap bit
REACH = 16                 # the pair rule sees a second piece up to the end of the next chunk
WARP = 2048                # a warp of the pair kernel takes 128 consecutive chunks: its last one has no successor in it
STAGE = 16384              # one k_front stage
SLICE = 64 * MIB           # the host ingest slice
WINDOW = 256 * MIB         # the planner's threshold, and the window of the windowed scans
N = 288 * MIB              # the texts: the planned window 0 and a 32 MiB tail under the threshold

WRAP_FILL, DOT_FILL, SUB, INS = b",", b"5", b"7", b"8"     # none is a piece byte, also under | 0x20
FILL = b"0123456789"


def positions(pattern, nocase=False, wrap=False):
    """the pattern's positions: its byte, None for `.`; wrap: the -w/-x wrapper positions at both ends.
    Returns (positions, fold): fold when some position stands for a case pair (then every piece is folded by | 0x20)."""
    if isinstance(pattern, str):
        pattern = pattern.encode("latin-1")
    lit = [None if c == ord(".") else c for c in pattern]
    fold = nocase and any(c is not None and chr(c).isalpha() for c in lit)
    return ([None] + lit + [None] if wrap else lit), fold


def pair_pieces(lit, k, fold=False):
    """scan.cu pair_pieces(): k + 2 pieces of 4 bytes if they fit, else 3, taken from the left over literal positions only
    (a window holding a None moves on by one), the first one at s0, pairwise distinct, (o_last - o_first) + k <= REACH.
    Returns [(bytes, offset)] or None."""
    np_ = k + 2
    if k < 0 or np_ > 4:
        return None
    f = 0x20 if fold else 0
    for ln in (4, 3):
        for s0 in range(0, len(lit) - np_ * ln + 1):
            got, p = [], s0
            while p + ln <= len(lit) and len(got) < np_:
                w = lit[p:p + ln]
                if any(c is None for c in w):
                    p += 1
                    continue
                got.append((bytes(c | f for c in w), p))
                p += ln
            if len(got) < np_ or got[0][1] != s0 or got[-1][1] - got[0][1] + k > REACH:
                continue
            if len({v for v, _ in got}) < np_:
                continue
            return got
    return None


_FOLD = bytes(c | 0x20 for c in range(256))


def piece_starts(text, pieces, fold=False, lo=0, hi=None, whole=False):
    """{chunk: bitmask of the pieces that start in it} for pieces starting in [lo, hi); whole: only pieces that end in
    their own chunk (a stage 1 that ignores the 4 bytes past the chunk)"""
    t = text.translate(_FOLD) if fold else text
    hi = len(t) if hi is None else hi
    pres = {}
    for i, (v, _) in enumerate(pieces):
        p = t.find(v, lo)
        while 0 <= p < hi:
            if not whole or p % CHUNK + len(v) <= CHUNK:
                pres[p // CHUNK] = pres.get(p // CHUNK, 0) | 1 << i
            p = t.find(v, p + 1)
    return pres


def flagged_chunks(text, pieces, fold=False, lo=0, hi=None, successor=True, whole=False):
    """the chunks c with lo <= 16c < hi that stage 1 flags under the pair plan: some piece starts in c and some other
    piece starts in c or (successor) in c + 1.  The last two chunks of the text, which stage 1 always passes on, are not
    added here."""
    hi = len(text) if hi is None else hi
    pres = piece_starts(text, pieces, fold, lo - lo % CHUNK, hi + CHUNK, whole)
    out = []
    for c in range((lo - lo % CHUNK) // CHUNK, (hi + CHUNK - 1) // CHUNK):
        here = pres.get(c, 0)
        both = here | (pres.get(c + 1, 0) if successor else 0)
        if here and bin(both).count("1") >= 2:
            out.append(c)
    return out


def chunk_flags(text, pieces, fold=False):
    """stage 1's verdict for every chunk of a whole text, the last two chunks passed on as always"""
    nch = (len(text) + CHUNK - 1) // CHUNK
    flags = [False] * nch
    for c in flagged_chunks(text, pieces, fold):
        flags[c] = True
    for c in range(max(0, nch - 2), nch):
        flags[c] = True
    return flags


# ---- the cases: a pattern, its switches (agrep_b200.Pattern keywords; the checker takes the same names) and what the
# model must compute for it.  span = (o_last - o_first) + k; the pair rule is sound up to REACH, the "bound" cases sit at it.
Case = namedtuple("Case", "name pattern kw wrap fold pieces span text")
CASES = [
    Case("bitap-k0", "governmental", dict(k=0, linenum=True), False, False, [(b"gove", 0), (b"rnme", 4)], 4, "lines"),
    Case("sgrep-k0", "governmental", dict(k=0), False, True, [(b"gove", 0), (b"rnme", 4)], 4, "lines"),
    Case("bound4-k0", "gove............ment", dict(k=0), False, False, [(b"gove", 0), (b"ment", 16)], 16, "lines"),
    Case("bound3-k0", "peo.............ple", dict(k=0), False, False, [(b"peo", 0), (b"ple", 16)], 16, "lines"),
    Case("nocase-k1", "people how too", dict(k=1, nocase=True), False, True,
         [(b"peop", 0), (b"le h", 4), (b"ow t", 8)], 9, "lines"),
    Case("word-k1", "state good", dict(k=1, wordbound=True), True, False, [(b"sta", 1), (b"te ", 4), (b"goo", 7)], 7, "lines"),
    Case("bound4-k1", "peop..le h.....ow t", dict(k=1), False, False, [(b"peop", 0), (b"le h", 6), (b"ow t", 15)], 16, "lines"),
    Case("bound3-k1", "sta.....te ....goo", dict(k=1), False, False, [(b"sta", 0), (b"te ", 8), (b"goo", 15)], 16, "lines"),
    Case("cost-k2", "governmental policy", dict(k=2, cost_s=2), False, False,
         [(b"gove", 0), (b"rnme", 4), (b"ntal", 8), (b" pol", 12)], 14, "lines"),
    Case("bound4-k2", "gove.nmen.al policy", dict(k=2), False, False,
         [(b"gove", 0), (b"nmen", 5), (b"al p", 10), (b"olic", 14)], 16, "lines"),
    Case("bound3-k2", "bec.aus.e e...ach", dict(k=2), False, False,
         [(b"bec", 0), (b"aus", 4), (b"e e", 8), (b"ach", 14)], 16, "lines"),
    Case("rows64-k2", "business give group toward young", dict(k=2), False, False,
         [(b"busi", 0), (b"ness", 4), (b" giv", 8), (b"e gr", 12)], 14, "lines"),
    Case("para-k2", "because each", dict(k=2, delim="$$"), False, False,
         [(b"bec", 0), (b"aus", 3), (b"e e", 6), (b"ach", 9)], 11, "paras"),
]
BY_NAME = {c.name: c for c in CASES}


def oracle_kw(case):
    """the case's switches for the checker (tests/_oracle.py): k > 0 simple literals run the automaton, as on the device
    (the reference's sgrep filters are lossy), so the checker is asked for it with linenum"""
    kw = {k: int(v) if isinstance(v, bool) else v for k, v in case.kw.items()}
    if case.kw["k"]:
        kw["linenum"] = 1
    return kw


def case_fold(case):
    return case.fold or positions(case.pattern, case.kw.get("nocase", False), case.wrap)[1]


def case_pieces(case):
    lit, _ = positions(case.pattern, False, case.wrap)
    return pair_pieces(lit, case.kw["k"], case_fold(case))


def shapes(case):
    """(a) k substitutions, first and last piece survive; (b) k insertions, one inside each middle piece: the first and
    last piece survive exactly span bytes apart; (c) k deletions; (d) two adjacent pieces survive.  k = 0: the pattern.
    Substitutions cost 2 under -S2, so there (a) is left out and (d) damages its pieces by deletions."""
    if case.kw["k"] == 0:
        return "a"
    return "bcd" if case.kw.get("cost_s", 1) > 1 else "abcd"


def content(case, shape, variant=0):
    """the planted bytes and the index in them at which the earlier surviving piece starts"""
    k = case.kw["k"]
    pieces = case_pieces(case)
    lit, _ = positions(case.pattern, False, case.wrap)
    cells = []
    for j, c in enumerate(lit):
        if c is not None:
            cells.append(bytes([c]))
        else:
            cells.append(WRAP_FILL if case.wrap and j in (0, len(lit) - 1) else DOT_FILL)
    if case.fold and variant % 2:                     # the other case on every other site (-i, the folded sgrep engine)
        cells = [c.swapcase() for c in cells]
    np_ = len(pieces)
    if shape == "d" and k:
        first = variant % (np_ - 1)
        keep = (first, first + 1)
    else:
        keep = (0, np_ - 1)
    edit = {"a": "sub", "b": "ins", "c": "del", "d": "del" if case.kw.get("cost_s", 1) > 1 else "sub"}[shape]
    damaged = [i for i in range(np_) if i not in keep][:k]
    for i in damaged:
        o = pieces[i][1]
        if edit == "sub":
            cells[o + 1] = SUB
        elif edit == "ins":
            cells[o + 1] = INS + cells[o + 1]
        else:
            cells[o + 1] = b""
    e = len(b"".join(cells[:pieces[keep[0]][1]]))
    return b"".join(cells), e


Site = namedtuple("Site", "case kind boundary lead shape variant at lo hi")


def _leads(case):
    ln = len(case_pieces(case)[0][0])
    return sorted({1, 2, ln - 1, ln, 5, 8})


# The boundaries a text has one of each: three host-slice edges, the window edge and the end of the text.  On the line
# text they go to the bound cases (shape (b) where k > 0, lead 1: the later piece on the last byte of the successor
# chunk); the paragraph text has them all for its one case, one shape each.
UNIQUE = {
    "lines": [("slice", SLICE, "bound4-k2", "b"), ("slice", 2 * SLICE, "bound3-k1", "b"), ("slice", 3 * SLICE, "bound3-k0", "a"),
              ("window", WINDOW, "bound3-k2", "b"), ("end", None, "bound4-k1", "b")],
    "paras": [("slice", SLICE, "para-k2", "a"), ("slice", 2 * SLICE, "para-k2", "c"), ("slice", 3 * SLICE, "para-k2", "d"),
              ("window", WINDOW, "para-k2", "b"), ("end", None, "para-k2", "b")],
}


def _place(case, kind, boundary, lead, shape, variant, n):
    body, e = content(case, shape, variant)
    delim = 2 if case.text == "paras" else 1
    if kind == "end":
        hi = n - 1
        end_at = hi - delim + 1 - CHUNK                   # content ends a chunk before the closing delimiter
        boundary = (end_at - len(body) + e - 2 * CHUNK) // CHUNK * CHUNK
    at = boundary - lead
    start = at - e
    lo = (start - 8) // CHUNK * CHUNK                     # the record's first byte: after its delimiter, on a chunk edge
    if kind != "end":
        hi = (start + len(body) + CHUNK + delim - 1 + CHUNK - 1) // CHUNK * CHUNK - 1
    return Site(case.name, kind, boundary, lead, shape, variant, at, lo, hi)


def sites(case, n=N):
    """every planted record of a case, in text order: each lead and shape before a chunk edge (not a warp's), a warp's
    last chunk (not a stage's) and a stage edge, one 128 KiB slot each; and the case's share of UNIQUE"""
    base = [c for c in CASES if c.text == case.text].index(case)
    out = []
    slot = 0
    for kind, off in (("chunk", 1040), ("warp", 3 * WARP), ("stage", 2 * STAGE)):
        for lead in _leads(case):
            for v, shape in enumerate(shapes(case)):
                s = MIB + (base * 96 + slot) * 128 * 1024
                slot += 1
                out.append(_place(case, kind, s + off, lead, shape, v + lead, n))
    for kind, b, name, shape in UNIQUE[case.text]:
        if name == case.name:
            out.append(_place(case, kind, b, 1, shape, CASES.index(case), n))
    out.sort(key=lambda s: s.at)
    return out


def record(case, site):
    """the bytes of text[lo - delim .. hi]: the delimiter before the record, digits, the planted bytes, digits, the
    closing delimiter.  Digits are never a piece byte, so the record holds no piece but the planted ones."""
    body, e = content(case, site.shape, site.variant)
    delim = b"\n\n" if case.text == "paras" else b"\n"
    start = site.at - e
    out = bytearray(FILL[j % 10] for j in range(site.lo, site.hi + 1 - len(delim)))
    out[start - site.lo:start - site.lo + len(body)] = body
    return delim + bytes(out) + delim


def all_sites(text_kind):
    return [s for c in CASES if c.text == text_kind for s in sites(c)]


def planted_text(text_kind, n=N):
    """the corpus (the library's generator, with matches of the headline pattern every 4 KiB) with every case's records
    of this text planted"""
    import agrep_b200 as ag
    buf = bytearray(ag.corpus_host(n, seed=41 if text_kind == "lines" else 43, paragraphs=text_kind == "paras",
                                   needle="because each", needle_every=4096, needle_maxedits=3))
    placed = []
    for c in CASES:
        if c.text != text_kind:
            continue
        for s in sites(c, n):
            r = record(c, s)
            a = s.lo - (len(r) - (s.hi + 1 - s.lo))
            buf[a:s.hi + 1] = r
            placed.append((a, s.hi))
    placed.sort()
    for (a0, b0), (a1, _) in zip(placed, placed[1:]):
        assert b0 + 64 < a1, (b0, a1)
    assert len(buf) == n
    return bytes(buf)
