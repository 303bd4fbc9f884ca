"""Simple literals of more than 63 positions (up to 255 characters, as sgrep()'s bm()/monkey() take them at k = 0): the
checker against the reference's answers, the 320-bit words of the front end against their closed form, the limits, and
the anchor plan.  CPU only."""
import os, json
import pytest
import agrep_b200 as ag
import _oracle
from golden import make_long_literal_golden as G

ANSWERS = json.load(open(G.GOLDEN))


def in_record(offset, rec, L):
    """the reference's -b offset (the end of the match) lies in the record: after the delimiter in front of it, at most
    at the first byte of the one that closes it"""
    return rec[0] + L <= offset <= rec[1] or (rec[0] < 0 and 0 <= offset <= rec[1])


@pytest.mark.parametrize("m,name,args,kw,final", G.CASES, ids=[G.key(c[0], c[1], c[4]) for c in G.CASES])
def test_checker_equals_the_reference(m, name, args, kw, final):
    data = G.case_text(m, kw, final)
    want = ANSWERS[G.key(m, name, final)]
    a = _oracle.compile(G.literal(m), **kw)
    assert a.engine == 4
    cnt, recs = _oracle.scan(a, data)
    L = len(kw.get("delim", "\n"))
    assert cnt == want["count"] and len(want["offsets"]) == cnt
    assert all(in_record(o, r, L) for o, r in zip(want["offsets"], recs)), (want["offsets"], recs)
    if os.path.exists(G.REF):                       # where the reference binary is built, ask it as well
        assert G.answer(m, args, kw, final) == want


def closed_form(lit, delim=b"\n", wordbound=False):
    """maskgen's closed form (position p at bit M-p, the feed above) in 320 bits, from the positions of an sgrep pattern:
    the delimiter, the separator, [-w neighbour], the literal ASCII case folded, [-w neighbour]"""
    def alnum(c):
        return chr(c).isascii() and chr(c).isalnum()
    nb = [c for c in range(256) if not alnum(c)]
    pos = [[c] for c in delim] + [None]
    lits = [[c, c ^ 32] if chr(c).isascii() and chr(c).isalpha() else [c] for c in lit]
    pos += ([nb] if wordbound else []) + lits + ([nb] if wordbound else [])
    M = len(pos)
    top = 64 * (M // 64 + 1)
    ones = (1 << top) - 1
    mask = [0] * 256
    for p, cls in enumerate(pos, 1):
        for c in cls or ():
            mask[c] |= 1 << (M - p)
    sep = 1 << (M - len(delim) - 1)
    init0 = (ones & ~((1 << M) - 1)) | sep
    endp = (sep << 1) | 1
    dend = endp & (1 << (M - len(delim)))
    prot = [p for p in range(1, M + 1) if p <= len(delim) or (wordbound and p in (len(delim) + 2, M)) or pos[p - 1] == [10]]
    noerr = ones & ~sum(1 << (M - p) for p in prot)
    dmask = ones & ~sum(1 << (M - p) for p in range(1, len(delim) + 1))
    return M, dict(mask=mask, init0=init0, init1=init0 | endp, noerr=noerr, endpos=endp ^ dend, dendpos=dend, dmask=dmask)


def wide_int(row):
    return sum(int(row[i]) << (64 * i) for i in range(ag._lib.WIDE_WORDS))


@pytest.mark.parametrize("m", [62, 64, 100, 255])
@pytest.mark.parametrize("kw", [{}, dict(nocase=1), dict(wordbound=1), dict(delim=";"), dict(delim="@#")])
def test_wide_words_are_the_closed_form(m, kw):
    lit = G.literal(m).encode()
    p = ag.Pattern(lit, **kw)
    d, w = p.desc, p.wide
    delim = kw.get("delim", "\n").encode()
    M, want = closed_form(lit, delim, wordbound=bool(kw.get("wordbound")))
    assert d.M == M and d.wide == 1 and d.k == 0 and d.nrows == 1 and d.engine == 4 and w is not None
    assert [wide_int(w.mask[c]) for c in range(256)] == want["mask"]
    for f in ("init0", "init1", "noerr", "endpos", "dendpos", "dmask"):
        assert wide_int(getattr(w, f)) == want[f], f
    # the descriptor holds no words of its own
    assert not any(d.mask) and d.init0 == d.init1 == d.noerr == d.endpos == d.dendpos == 0 and not any(d.reset) and not any(d.start)
    assert bytes(d.delim[:d.L]) == delim


def test_short_literals_keep_their_64_bit_form_and_the_forced_wide_form_equals_it(monkeypatch):
    rows = ("init0", "init1", "noerr", "endpos", "dendpos", "dmask", "reset", "start")
    for lit in ("a", "the", "because each", "x" * 40, G.literal(61)):
        for kw in ({}, dict(nocase=1), dict(wordbound=1), dict(inverse=1), dict(delim="$$"), dict(delim="aba")):
            monkeypatch.delenv("AGB_FORCE_WIDE", raising=False)
            n = ag.Pattern(lit, **kw)
            if n.desc.M > 63:                                    # (61 characters and -w or a 2-byte delimiter: 64 positions or more)
                assert n.wide is not None and n.desc.wide == 1
                continue
            assert n.wide is None and n.desc.wide == 0
            monkeypatch.setenv("AGB_FORCE_WIDE", "1")
            f = ag.Pattern(lit, **kw)
            dn, df, w = n.desc, f.desc, f.wide
            assert w is not None and df.wide == 1 and df.M == dn.M <= 63
            assert [wide_int(w.mask[c]) for c in range(256)] == list(dn.mask), (lit, kw)
            for r in rows:
                v = getattr(dn, r)
                assert wide_int(getattr(w, r)) == (v[0] if r in ("reset", "start") else v), (lit, kw, r)
            for f_ in ("M", "L", "delim_kind", "start_closes", "inverse", "user_delim", "outtail", "plan", "n_anchors", "anchor_len",
                       "anchor_fold", "anchor_mask", "pat_len", "engine"):
                assert getattr(df, f_) == getattr(dn, f_), (lit, kw, f_)
            assert list(df.anchor) == list(dn.anchor) and list(df.anchor_off) == list(dn.anchor_off) and list(df.delim_fold) == list(dn.delim_fold)
            assert df.refine == 0                                # no stage 1.5 for 320-bit rows
    monkeypatch.setenv("AGB_FORCE_WIDE", "1")
    assert ag.Pattern("the", k=1).wide is None and ag.Pattern("th.e").wide is None   # only the sgrep engine has the wide form


def test_limits():
    p = ag.Pattern("a" * 255)
    assert p.desc.M == 255 + 2 and p.wide is not None
    assert ag.Pattern("b" * 255, wordbound=1, delim="<12345678>").desc.M == 8 + 1 + 257
    with pytest.raises(ag.AgrepError, match="too long"):
        ag.Pattern("a" * 256)
    assert "pattern '" + "a" * 256 + "' too long" == _error("a" * 256)
    lit = G.literal(70)
    for kw in (dict(k=1), dict(linenum=1), dict(bestmatch=1), dict(ins_free=1), dict(cost_i=2, k=1), dict(wholeline=1)):
        assert _error(lit, **kw) == "pattern too long (has > 64 chars)", kw
    assert _error("[ab]" + lit) == "pattern too long (has > 64 chars)"
    # a descriptor of 320-bit rows holds no words: it cannot be wrapped
    d = p.desc
    h = ag._lib.C.c_void_p()
    err = ag._lib.C.create_string_buffer(256)
    assert ag._lib.lib().agb_pattern_from_desc(ag._lib.C.byref(d), ag._lib.C.byref(h), err, 256) != 0


def _error(pat, **kw):
    with pytest.raises(ag.AgrepError) as e:
        ag.Pattern(pat, **kw)
    return str(e.value)


@pytest.mark.parametrize("m", [62, 100, 255])
@pytest.mark.parametrize("kw", [{}, dict(wordbound=1), dict(delim="@#")])
def test_one_anchor_inside_the_literal(m, kw):
    lit = G.literal(m).encode()
    d = ag.Pattern(lit, **kw).desc
    assert d.plan == ag.api.PLAN_ANCHORS and d.n_anchors == 1 and d.n_anchors3 == 0 and d.refine == 0
    a = d.anchor[0].to_bytes(4, "little")[:d.anchor_len]
    start = d.anchor_off[0] - (1 if kw.get("wordbound") else 0)      # (the -w neighbour is the position in front of the literal)
    assert d.pat_len == len(lit) + (2 if kw.get("wordbound") else 0)
    assert bytes(c | 0x20 for c in lit[start:start + d.anchor_len]) == bytes(c | 0x20 for c in a)
