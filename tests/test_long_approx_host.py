"""Simple literals of more than 63 positions at k = 1..8 (agb_options.wide_approx: what the reference hands to sgrep()):
which patterns the front end accepts in 320-bit rows and which it refuses, the wide words against the 64-bit words of the
same literal, the anchor plan, and the checker's 320-bit rows -- against its 64-bit rows, against an edit-distance
restatement, and against the reference binary where it is built.  CPU only."""
import os, random, subprocess, tempfile
import pytest
import agrep_b200 as ag
import _oracle, _oracle_wide, _corpus
from golden.make_long_literal_golden import literal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "agrep")
LENGTHS = (62, 63, 64, 100, 200, 255)
KS = (1, 2, 4, 8)
DELIMS = ({}, dict(inverse=1), dict(delim=";"), dict(delim="@#"), dict(delim="$$"))


def wide_int(row):
    return sum(int(row[i]) << (64 * i) for i in range(ag._lib.WIDE_WORDS))


def approx_text(lit, k, sep=b"\n", final=True, nlines=240, seed=0, every=3):
    """seeded lines joined by sep; every third line has the literal planted inside it with 0..k+1 random edits"""
    rnd = random.Random(seed * 7919 + len(lit) * 31 + k)
    lines = _corpus.make_text(nlines, seed=seed + len(lit)).split(b"\n")[:nlines]
    text = lit.decode() if isinstance(lit, bytes) else lit
    for i in range(0, len(lines), every):
        v = _corpus.mutate(rnd, text, rnd.randint(0, k + 1)).encode()
        line = lines[i]
        at = rnd.randint(0, len(line))
        lines[i] = line[:at] + v + line[at:]
    return sep.join(lines) + (sep if final else b"")


def _error(pat, **kw):
    with pytest.raises(ag.AgrepError) as e:
        ag.Pattern(pat, **kw)
    return str(e.value)


# ---- what is accepted and what is refused -----------------------------------------------------------------------------
@pytest.mark.parametrize("m", LENGTHS)
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("kw", DELIMS, ids=["plain", "v", "d;", "d@#", "d$$"])
def test_accepted(m, k, kw, monkeypatch):
    monkeypatch.delenv("AGB_FORCE_WIDE", raising=False)
    lit = literal(m)
    p = ag.Pattern(lit, k=k, wide_approx=True, **kw)
    d = p.desc
    assert d.k == k and d.nrows == k + 1 and d.engine == (1 if k <= 4 else 2)
    assert d.M == len(kw.get("delim", "\n")) + 1 + m
    if d.M <= 63:
        assert d.wide == 0 and p.wide is None                # (62 characters on newline records: the 64-bit form)
        return
    assert d.wide == 1 and p.wide is not None
    assert not any(d.mask) and not any(d.reset) and not any(d.start)
    assert d.refine == 0 and d.n_anchors == k + 1 and d.anchor_len == 4
    assert d.plan == (ag.api.PLAN_ALL if kw.get("inverse") else ag.api.PLAN_ANCHORS)


@pytest.mark.parametrize("kw", [dict(nocase=1), dict(wordbound=1), dict(wholeline=1), dict(linenum=1), dict(bestmatch=1),
                                dict(ins_free=1), dict(cost_i=2), dict(wide_approx=0)],
                         ids=["i", "w", "x", "n", "B", "p", "I2", "flag-off"])
@pytest.mark.parametrize("k", [1, 8])
def test_refused_as_today(kw, k):
    lit = literal(100)
    kw = dict(dict(wide_approx=1), **kw)
    assert _error(lit, k=k, **kw) == "pattern too long (has > 64 chars)"
    # (and without the flag the same)
    kw["wide_approx"] = 0
    assert _error(lit, k=k, **kw) == "pattern too long (has > 64 chars)"


def test_refused_classes_length_and_errors():
    lit = literal(100)
    assert _error("[ab]" + lit, k=1, wide_approx=1) == "pattern too long (has > 64 chars)"
    assert _error(lit[:50] + "." + lit[51:], k=2, wide_approx=1) == "pattern too long (has > 64 chars)"
    assert _error("a" * 256, k=1, wide_approx=1) == "pattern '" + "a" * 256 + "' too long"
    assert _error("abc", k=3, wide_approx=1) == "size of pattern 'abc' must be > #of errors 3"
    assert ag.Pattern("a" * 255, k=8, wide_approx=1).desc.M == 257


# ---- the wide words against the 64-bit words --------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(1, 9))
def test_forced_wide_words_equal_the_64_bit_words(k, monkeypatch):
    rows = ("init0", "init1", "noerr", "endpos", "dendpos", "dmask")
    for lit in ("abcdefghij", "because each", "x" * 40, literal(59)):
        for kw in ({}, dict(inverse=1), dict(delim=";"), dict(delim="$$"), dict(delim="aba"), dict(delim="@#")):
            monkeypatch.delenv("AGB_FORCE_WIDE", raising=False)
            n = ag.Pattern(lit, k=k, wide_approx=True, **kw)
            assert n.wide is None and n.desc.wide == 0
            monkeypatch.setenv("AGB_FORCE_WIDE", "1")
            f = ag.Pattern(lit, k=k, wide_approx=True, **kw)
            dn, df, w = n.desc, f.desc, f.wide
            assert w is not None and df.wide == 1 and df.M == dn.M <= 63
            assert [wide_int(w.mask[c]) for c in range(256)] == list(dn.mask), (lit, kw)
            for r in rows:
                assert wide_int(getattr(w, r)) == getattr(dn, r), (lit, kw, r)
            assert wide_int(w.reset) == dn.reset[0] and wide_int(w.start) == dn.start[0], (lit, kw)
            for r in range(1, k + 1):
                assert wide_int(w.reset_up[r - 1]) == dn.reset[r] and wide_int(w.start_up[r - 1]) == dn.start[r], (lit, kw, r)
            for r in range(k + 1, 9):
                assert wide_int(w.reset_up[r - 1]) == 0 and wide_int(w.start_up[r - 1]) == 0
            for f_ in ("M", "L", "k", "nrows", "engine", "delim_kind", "start_closes", "inverse", "user_delim", "outtail", "plan",
                       "n_anchors", "anchor_len", "anchor_fold", "anchor_mask", "pat_len"):
                assert getattr(df, f_) == getattr(dn, f_), (lit, kw, f_)
            assert list(df.anchor) == list(dn.anchor) and list(df.anchor_off) == list(dn.anchor_off)
            assert list(df.delim_fold) == list(dn.delim_fold)
            assert df.refine == 0
    monkeypatch.setenv("AGB_FORCE_WIDE", "1")
    assert ag.Pattern("the", k=1).wide is None                    # without the flag: the 64-bit form
    assert ag.Pattern("the", k=1, wide_approx=True).wide is not None


@pytest.mark.parametrize("k", range(1, 9))
def test_k_plus_one_disjoint_anchors_for_every_length(k):
    for m in range(62, 256):
        lit = literal(m, seed=k).encode()
        d = ag.Pattern(lit, k=k, wide_approx=True).desc
        if d.M <= 63:
            continue
        assert d.plan == ag.api.PLAN_ANCHORS and d.n_anchors == k + 1 and d.anchor_len == 4 and d.refine == 0, (m, k)
        assert d.pat_len == m
        offs = [d.anchor_off[i] for i in range(d.n_anchors)]
        assert all(b - a >= 4 for a, b in zip(offs, offs[1:])), (m, k, offs)
        for i, off in enumerate(offs):
            assert 0 <= off and off + 4 <= m
            assert lit[off:off + 4] == d.anchor[i].to_bytes(4, "little"), (m, k, i)


# ---- the checker's 320-bit rows ---------------------------------------------------------------------------------------
# (separator in the text, checker keywords): '$' is '\n' in -d, so -d '$$' separates paragraphs
CHECK_DELIMS = (("\n", {}), (";", dict(delim=";")), ("\n\n", dict(delim="$$")), ("aba", dict(delim="aba")), ("@#", dict(delim="@#")))


@pytest.mark.parametrize("k", range(0, 9))
@pytest.mark.parametrize("sep,kw", CHECK_DELIMS, ids=["nl", ";", "$$", "aba", "@#"])
def test_wide_checker_equals_the_64_bit_checker(k, sep, kw):
    for lit in ("because each", literal(30 + k), literal(62 - len(kw.get("delim", "\n")))):     # (the last: 63 positions)
        if len(lit) <= k:
            continue
        for final in (True, False):
            data = approx_text(lit, k, sep.encode(), final, nlines=120, seed=k)
            for inv in (0, 1):
                o = dict(kw, k=k, linenum=1, inverse=inv)
                a, w = _oracle.compile(lit, **o), _oracle_wide.compile(lit, **o)
                assert w.a.M == a.M <= 63
                assert _oracle_wide.scan(w, data) == _oracle.scan(a, data), (lit, o, final)
            o = dict(kw, k=k, linenum=1)
            a, w = _oracle.compile(lit, **o), _oracle_wide.compile(lit, **o)
            for want in (-1, k // 2):
                assert _oracle_wide.scan_levels(w, k, data, want) == _oracle.scan_levels(a, k, data, want), (lit, o, final, want)


def _best_distance(pat, text):
    """the smallest edit distance between pat and any substring of text (Myers' bit-vector search, Python integers)"""
    m = len(pat)
    peq = {}
    for i, c in enumerate(pat):
        peq[c] = peq.get(c, 0) | (1 << i)
    full, high = (1 << m) - 1, 1 << (m - 1)
    pv, mv, score, best = full, 0, m, m
    for c in text:
        eq = peq.get(c, 0)
        xv = eq | mv
        xh = (((eq & pv) + pv) ^ pv) | eq
        ph = mv | (~(xh | pv) & full)
        mh = pv & xh
        if ph & high:
            score += 1
        elif mh & high:
            score -= 1
        ph = (ph << 1) & full
        mh = (mh << 1) & full
        pv = mh | (~(xv | ph) & full)
        mv = ph & xv
        best = min(best, score)
    return best


@pytest.mark.parametrize("m", [64, 80, 100, 160, 200, 255])
@pytest.mark.parametrize("k", KS)
def test_wide_checker_equals_edit_distance(m, k):
    lit = literal(m, seed=k).encode()
    for final in (True, False):
        data = approx_text(lit, k, b"\n", final, nlines=150, seed=m)
        w = _oracle_wide.compile(lit, k=k, linenum=1)
        cnt, recs = _oracle_wide.scan(w, data)
        want, begin = [], -1
        for line in data.split(b"\n")[:data.count(b"\n") + (0 if final else 1)]:
            end = begin + 1 + len(line)
            if line and _best_distance(lit, line) <= k:
                want.append((begin, end))
            begin = end
        assert [r[:2] for r in recs] == want, (m, k, final)
        assert cnt == len(want) and cnt > 10
        # the levels pass: each record's smallest level is its edit distance
        _, hist, lv = _oracle_wide.scan_levels(w, k, data)
        byrec = {(b, e): lvl for b, e, _, lvl in lv}
        assert sorted(byrec) == want
        for line_rec in want[:40]:
            b, e = line_rec
            assert byrec[line_rec] == _best_distance(lit, data[b + 1:e])


@pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref/agrep not built (no reference sources)")
@pytest.mark.parametrize("m", [40, 80, 160, 255])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_every_line_the_reference_prints_is_in_the_checker_list(m, k):
    """the reference's sgrep() filters lose matches at k > 0 (its k > 0 answer is a subset of the automaton's)"""
    lit = literal(m, seed=k).encode()
    data = approx_text(lit, k, b"\n", True, nlines=200, seed=m + 1)
    assert len(data) < 48 * 1024
    w = _oracle_wide.compile(lit, k=k, linenum=1)
    _, recs = _oracle_wide.scan(w, data)
    ours = [data[b + 1:e] for b, e, _ in recs]
    with tempfile.NamedTemporaryFile(suffix=".txt") as f:
        f.write(data)
        f.flush()
        out = subprocess.run([REF, "-V0", "-%d" % k, lit, f.name], capture_output=True, timeout=60).stdout
    printed = out.split(b"\n")[:-1]
    assert set(printed) <= set(ours), (m, k)
    assert len(ours) >= len(printed)
