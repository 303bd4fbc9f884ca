"""The pair plan's chunk rule, modelled on the CPU (tests/_plans.py; no device needed).

Stage 1 under the pair plan cuts the pattern into k + 2 disjoint, pairwise distinct literal pieces of one length and flags
a 16-byte chunk only where some piece starts in it and some *other* piece starts in it or in the next chunk (the last two
chunks of the text are always flagged).  k errors leave two pieces verbatim, and the later one starts at most
(o_last - o_first) + k bytes after the earlier one, so the rule cannot lose a match while that is at most 16.  Here:
  * on random texts and patterns with planted matches, every record the checker (tests/_oracle.py) reports holds a chunk
    the model flags;
  * the planner's choice of pieces (a model of scan.cu's pair_pieces, non-literal positions skipped) for every case the
    device tests run, and its distance bound: a match whose two surviving pieces are as far apart as the bound allows is
    still caught, one byte further it would not be, and with k >= len the rule still holds;
  * the records the device tests plant: each matches by the checker, each has exactly one flagged chunk (the one where
    its earlier surviving piece starts), and on the bound cases that chunk is flagged only through its successor chunk
    and the 4 bytes past the chunk -- so the device test would catch a stage 1 that ignores either."""
import random
import pytest
import _oracle, _corpus, _plans
from _plans import CHUNK, REACH, chunk_flags


def pieces_of(pattern, k, nocase=False, wrap=False):
    lit, fold = _plans.positions(pattern, nocase, wrap)
    return _plans.pair_pieces(lit, k, fold)


def covered(flags, begin, end):
    return any(flags[c] for c in range(max(0, begin // CHUNK), min(len(flags), (end + CHUNK - 1) // CHUNK)))


def random_case(rnd, k, alphabet="abcdefgh "):
    plen = rnd.randint(3 * (k + 2), 3 * (k + 2) + 4)
    pattern = "".join(rnd.choice("abcdefgh") for _ in range(plen))
    lines = []
    for _ in range(400):
        if rnd.random() < 0.3:
            line = _corpus.mutate(rnd, pattern, rnd.randint(0, k))
            line = "".join(rnd.choice(alphabet) for _ in range(rnd.randint(0, 20))) + line + \
                "".join(rnd.choice(alphabet) for _ in range(rnd.randint(0, 20)))
        else:
            line = "".join(rnd.choice(alphabet) for _ in range(rnd.randint(0, 60)))
        lines.append(line.replace("\n", ""))
    return pattern, ("\n".join(lines) + "\n").encode()


@pytest.mark.parametrize("k", [0, 1, 2])
@pytest.mark.parametrize("seed", range(6))
def test_every_match_has_a_flagged_chunk(k, seed):
    rnd = random.Random(1000 * k + seed)
    pattern, text = random_case(rnd, k)
    pieces = pieces_of(pattern, k)
    if pieces is None:
        pytest.skip("no pair plan for %r" % pattern)
    flags = chunk_flags(text, pieces)
    cnt, recs = _oracle.scan(_oracle.compile(pattern, k=k, linenum=1), text)
    assert cnt > 0
    for b, e, _ in recs:
        assert covered(flags, b, e), (pattern, k, b, e, text[b:e])
    # the point of the rule: it flags no chunk in which no piece starts
    t = text
    for c, f in enumerate(flags[:-2]):
        if f:
            assert any(t.find(v, c * CHUNK, c * CHUNK + CHUNK + len(v) - 1) >= 0 for v, _ in pieces)


def test_nocase_model():
    rnd = random.Random(7)
    pattern, text = random_case(rnd, 2)
    text = bytes(c - 32 if 97 <= c <= 122 and rnd.random() < 0.3 else c for c in text)
    pieces = pieces_of(pattern, 2, nocase=True)
    flags = chunk_flags(text, pieces, fold=True)
    cnt, recs = _oracle.scan(_oracle.compile(pattern, k=2, nocase=1, linenum=1), text)
    assert cnt > 0
    for b, e, _ in recs:
        assert covered(flags, b, e)


def test_headline_pieces():
    assert pieces_of("because each", 2) == [(b"bec", 0), (b"aus", 3), (b"e e", 6), (b"ach", 9)]
    # long enough for four-byte pieces
    assert pieces_of("governmental policy", 2) == [(b"gove", 0), (b"rnme", 4), (b"ntal", 8), (b" pol", 12)]
    # k > 2 has no pair plan (stage 1 would pay more than one IMAD per window for each extra piece)
    assert pieces_of("because each of them", 3) is None
    # pieces that repeat cannot be told apart
    assert pieces_of("abcabcabcabc", 2) is None


def test_pieces_skip_non_literal_positions():
    """a window that holds a `.` or a wrapper position moves the piece on by one byte; the first piece must sit at s0,
    so a pattern that starts with a non-literal position begins its pieces at the first literal one; the bound counts the
    skipped positions"""
    assert pieces_of("abcd.efgh", 0) == [(b"abcd", 0), (b"efgh", 5)]
    assert pieces_of("abc.defg", 0) == [(b"abc", 0), (b"def", 4)]           # no two four-byte pieces: three bytes
    assert pieces_of(".abcdefgh", 0) == [(b"abcd", 1), (b"efgh", 5)]
    assert pieces_of("ab.cdefghi", 0) == [(b"cde", 3), (b"fgh", 6)]         # "cdef" has no second four-byte piece
    assert pieces_of("state good", 1, wrap=True) == [(b"sta", 1), (b"te ", 4), (b"goo", 7)]
    # one position more between the pieces and the bound is exceeded: three-byte pieces one further on, or none
    assert pieces_of("gove............ment", 0) == [(b"gove", 0), (b"ment", 16)]
    assert pieces_of("gove.............ment", 0) == [(b"ove", 1), (b"men", 17)]
    assert pieces_of("peo..............ple", 0) is None
    # folded under -i, also where the pattern has capitals
    assert pieces_of("People How Too", 1, nocase=True) == [(b"peop", 0), (b"le h", 4), (b"ow t", 8)]


@pytest.mark.parametrize("case", _plans.CASES, ids=lambda c: c.name)
def test_model_gives_the_table_pieces(case):
    pieces = _plans.case_pieces(case)
    assert pieces == case.pieces
    assert len(pieces) == case.kw["k"] + 2 and len({len(v) for v, _ in pieces}) == 1
    assert pieces[-1][1] - pieces[0][1] + case.kw["k"] == case.span <= REACH


@pytest.mark.parametrize("case", _plans.CASES, ids=lambda c: c.name)
def test_model_positions_are_the_compiled_patterns(case):
    """the positions the model plans over are those adaptive_plan() reads from the compiled pattern's masks (one byte,
    a case pair, or neither), and the compiled pattern is one the planner re-plans: anchors, stage 1.5, adaptive"""
    import agrep_b200 as ag
    from agrep_b200 import _lib
    d = ag.Pattern(case.pattern, **case.kw).desc
    assert d.adaptive == 1 and d.plan == _lib.PLAN_ANCHORS and d.refine and d.n_anchors >= 1 and d.n_anchors3 == 0
    assert 4 <= d.pat_len <= 60 and not d.pair_plan
    got, pairs = [], False
    for j in range(d.pat_len):
        bit = 1 << (d.M - (d.L + 2 + j))
        cs = [c for c in range(256) if d.mask[c] & bit]
        if len(cs) == 1 and cs[0] != 10 and cs[0] < 0x80:
            got.append(cs[0])
        elif len(cs) == 2 and cs[0] ^ cs[1] == 0x20 and cs[1] < 0x80:
            got.append(cs[0] | 0x20)
            pairs = True
        else:
            got.append(None)
    fold = _plans.case_fold(case)
    assert pairs == fold
    lit, _ = _plans.positions(case.pattern, False, case.wrap)
    assert got == [None if c is None else c | (0x20 if fold and chr(c).isalpha() else 0) for c in lit]


def planted(first_at, gap, p, q, fill=b"x"):
    """a line in which piece p starts at byte first_at and piece q `gap` bytes after it"""
    line = bytearray(fill * (first_at + gap + len(q) + 8))
    line[first_at:first_at + len(p)] = p
    line[first_at + gap:first_at + gap + len(q)] = q
    return bytes(line)


@pytest.mark.parametrize("span,k", [(14, 2), (13, 3), (12, 4)])
def test_distance_bound_is_tight(span, k):
    """Two pieces at the bound: (gap between their starts) = span + k = REACH is caught when the first one starts at the
    last byte of a chunk; at REACH + 1 it would not be, which is why the planner refuses such plans."""
    p, q = b"QRS", b"UVW"
    pieces = [(p, 0), (q, span)]
    for gap, ok in ((span + k, True), (span + k + 1, False)):
        text = b"\n" * 32 + planted(15, gap, p, q) + b"\n" + b"z" * 64 + b"\n"
        at = 32 + 15
        flags = chunk_flags(text, pieces)
        assert flags[at // CHUNK] == ok
    assert (span + k <= REACH) and (span + k + 1 > REACH)


def test_swapped_pieces_with_k_at_least_len():
    """With k >= len the two pieces that stay verbatim may appear in the text in the other order.  The planner never
    builds such a plan (k <= 2 < 3 <= len), but the rule does not depend on it: pieces are paired by identity, not by
    pattern order, so the earlier one in the text still flags its chunk wherever the pair sits."""
    pieces = pieces_of("abcdefghijkl", 2)
    assert pieces == [(b"abc", 0), (b"def", 3), (b"ghi", 6), (b"jkl", 9)]
    for lead in range(0, 32):
        line = b"y" * lead + b"defabc" + b"y" * 20                     # "def" before "abc"
        flags = chunk_flags(b"\n" + line + b"\n" * 40, pieces)
        assert flags[(1 + lead) // CHUNK]


# ---- the planted records of the device tests (tests/test_gpu_plans_large.py) -----------------------------------------

def local(case, site):
    """the site's record at its offset modulo a chunk, as a small text: chunk 1 is the record's first chunk"""
    r = _plans.record(case, site)
    head = CHUNK - (len(r) - (site.hi + 1 - site.lo))
    text = b"9" * head + r + b"9" * (2 * CHUNK)
    return text, CHUNK - site.lo          # text index = offset + shift


@pytest.mark.parametrize("case", _plans.CASES, ids=lambda c: c.name)
def test_planted_records_match(case):
    """the checker finds every planted record of the case at its k, and nothing else in a text of only those records"""
    sites = _plans.sites(case)
    delim = b"\n\n" if case.text == "paras" else b"\n"
    recs = [_plans.record(case, s) for s in sites]
    assert all(r.startswith(delim) and r.endswith(delim) for r in recs)
    text = b"".join(r[len(delim):] for r in recs)
    cnt, got = _oracle.scan(_oracle.compile(case.pattern, **_plans.oracle_kw(case)), text)
    assert cnt == len(sites), (case.name, cnt, len(sites))


@pytest.mark.parametrize("case", _plans.CASES, ids=lambda c: c.name)
def test_planted_records_flag_one_chunk(case):
    """within each planted record the model flags exactly one chunk: the one where the earlier surviving piece starts,
    `lead` bytes before the site's boundary; shape (b) puts the later one exactly span bytes after it"""
    pieces, fold = _plans.case_pieces(case), _plans.case_fold(case)
    for s in _plans.sites(case):
        assert s.boundary - s.at == s.lead and s.boundary % CHUNK == 0
        text, shift = local(case, s)
        got = flagged_chunks_in(text, pieces, fold, s, shift)
        assert got == [(s.at + shift) // CHUNK], (case.name, s, got)
        starts = _plans.piece_starts(text, pieces, fold)
        assert bin(sum(1 << c for c in starts)).count("1") == len(starts)
        found = sorted((text.translate(_plans._FOLD) if fold else text).find(v) for v, _ in pieces)
        found = [p - shift for p in found if p >= 0]
        assert found[0] == s.at and len(found) >= 2, (case.name, s, found)
        if s.shape == "b" and case.kw["k"]:
            assert found[1] - found[0] == case.span


def flagged_chunks_in(text, pieces, fold, site, shift, **kw):
    return _plans.flagged_chunks(text, pieces, fold, site.lo - 2 + shift, site.hi + 1 + shift, **kw)


BOUND = [c for c in _plans.CASES if c.span == REACH]


@pytest.mark.parametrize("case", BOUND, ids=lambda c: c.name)
def test_bound_records_need_the_successor_and_the_bytes_past_the_chunk(case):
    """Tightness: on the bound cases a shape (b) record at lead 1 has its earlier piece on the last byte of a chunk and
    the later one on the last byte of the next.  The rule without the successor chunk flags no chunk of it, and neither
    does the rule that only sees pieces ending inside their chunk (the windows that read the 4 bytes past the chunk)."""
    pieces, fold = _plans.case_pieces(case), _plans.case_fold(case)
    tight = [s for s in _plans.sites(case) if s.lead == 1 and s.shape == ("b" if case.kw["k"] else "a")]
    assert len(tight) >= 3
    for s in tight:
        text, shift = local(case, s)
        assert flagged_chunks_in(text, pieces, fold, s, shift) == [(s.at + shift) // CHUNK]
        assert flagged_chunks_in(text, pieces, fold, s, shift, successor=False) == [], s
        assert flagged_chunks_in(text, pieces, fold, s, shift, whole=True) == [], s


def test_sites_cover_every_boundary():
    """each case has every lead and shape before a chunk edge, a warp's last chunk and a stage edge; the slice edges, the
    window edge and the end of the text are each taken by one case of each text"""
    for case in _plans.CASES:
        ss = _plans.sites(case)
        for kind, unit in (("chunk", CHUNK), ("warp", _plans.WARP), ("stage", _plans.STAGE)):
            mine = [s for s in ss if s.kind == kind]
            assert {(s.lead, s.shape) for s in mine} == {(l, sh) for l in _plans._leads(case) for sh in _plans.shapes(case)}
            assert all(s.boundary % unit == 0 for s in mine)
            if kind != "stage":
                assert not any(s.boundary % (unit * 8 if kind == "warp" else _plans.WARP) == 0 for s in mine)
    for kind in ("lines", "paras"):
        ss = _plans.all_sites(kind)
        assert sorted(s.boundary for s in ss if s.kind == "slice") == [_plans.SLICE, 2 * _plans.SLICE, 3 * _plans.SLICE]
        assert [s.boundary for s in ss if s.kind == "window"] == [_plans.WINDOW]
        assert [s.hi for s in ss if s.kind == "end"] == [_plans.N - 1]
