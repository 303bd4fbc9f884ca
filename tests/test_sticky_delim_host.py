"""-p with a record delimiter of two or more bytes (delim_kind 3), on the host: the checker against the reference's answers
(tests/golden/sticky_delim_answers.json), the refusal without agb_options.sticky_delim, the descriptor words, the host
ordinals, and the delimiter pass's slice functions (delim_state.cu) restated in Python against the byte-serial rule."""
import ctypes as C
import json, os, random
import pytest
import _oracle
import agrep_b200 as ag
from agrep_b200 import _lib
from golden.make_sticky_delim_golden import CASES, DELIMS, NOT_RESTATED, case_text, checker_kw, dbytes, key, reference_j

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sticky_delim_answers.json")))


def render(text, delim, recs, linenum):
    """what output() prints for these records under a user delimiter of two or more bytes (agrep.c:3805-3956): the buffer
    holds the virtual '\n', the text and the delimiter appended at EOF (bitap.c:140, 161-165)"""
    hb = b"\n" + text + dbytes(delim)
    out, first = bytearray(), True
    for b, e, j in recs:
        i1, i2 = b + 1, e
        if i1 > i2:
            continue
        if first:
            if hb[i1:i1 + 1] == b"\n":
                i1 += 1
            first = False
        while i1 <= i2 and hb[i1:i1 + 1] == b"\n":
            out += b"\n"
            i1 += 1
        if linenum:
            out += b"%d: " % j
        out += hb[i1:i2 + 1]
    return bytes(out)


def oracle_answer(dn, pn, tn):
    kw, pat = checker_kw(dn, pn)
    a = _oracle.compile(pat, **kw)
    data = case_text(dn, tn)
    cnt, recs = _oracle.scan(a, data)
    return data, a, cnt, reference_j(recs, kw, data)


@pytest.mark.parametrize("dn,pn,tn", CASES, ids=[key(*c) for c in CASES])
def test_the_checker_prints_what_the_reference_prints(dn, pn, tn):
    g = GOLDEN[key(dn, pn, tn)]
    if g["count"] is None:
        # -p -S#: the reference refuses it whatever the delimiter (-p makes the insertion cost 0); the checker and the engine
        # take it, as they did with newline records before -- not a matter of the delimiter, so not compared here
        assert "cost cannot be 0" in g["count_err"] and pn == "S2"
        return
    data, a, cnt, recs = oracle_answer(dn, pn, tn)
    assert cnt == g["count"]
    if (dn, pn, tn) in NOT_RESTATED:
        return
    delim = checker_kw(dn, pn)[0]["delim"]
    assert render(data, delim, recs, False) == g["plain"].encode("latin-1")
    assert render(data, delim, recs, True) == g["n"].encode("latin-1")


DELIM_ARGS = [d[1] for d in DELIMS]


@pytest.mark.parametrize("delim", DELIM_ARGS)
def test_refused_without_the_flag(delim):
    with pytest.raises(ag.AgrepError, match="-p with a delimiter"):
        ag.Pattern("because", ins_free=True, delim=delim)
    d = ag.Pattern("because", ins_free=True, delim=delim, sticky_delim=True).desc
    assert d.delim_kind == 3 and d.sticky_delim == 1 and d.plan == _lib.PLAN_ALL
    # agb_pattern_from_desc: the descriptor's own byte decides
    d.sticky_delim = 0
    h, err = C.c_void_p(), C.create_string_buffer(256)
    assert _lib.lib().agb_pattern_from_desc(C.byref(d), C.byref(h), err, 256) == -1
    assert b"-p with a delimiter" in err.value
    d.sticky_delim = 1
    assert _lib.lib().agb_pattern_from_desc(C.byref(d), C.byref(h), err, 256) == 0
    got = _lib.Desc.from_buffer_copy(_lib.lib().agb_pattern_desc(h).contents)
    assert got.delim_kind == 3
    _lib.lib().agb_pattern_free(h)


@pytest.mark.parametrize("kw", [dict(), dict(delim="ab"), dict(delim=";"), dict(delim="$$"), dict(delim="aba"), dict(ins_free=True),
                                dict(ins_free=True, delim=";"), dict(k=2, delim="e "), dict(nocase=True, delim="AB")])
def test_the_flag_changes_nothing_else(kw):
    """where -p does not meet a delimiter of two or more bytes, the flag leaves the descriptor as it was"""
    a, b = ag.Pattern("because", **kw).desc, ag.Pattern("because", sticky_delim=True, **kw).desc
    assert bytes(a) == bytes(b) and b.sticky_delim == 0


@pytest.mark.parametrize("pat,kw,msg", [("a|b", dict(regex=True, delim="ab", ins_free=True), "-d or -w option is not supported"),
                                        ("a;b,c", dict(delim="ab", ins_free=True), "cannot handle OR"),
                                        ("abc", dict(k=3, delim="ab", ins_free=True), "must be > #of errors"),
                                        ("because", dict(delim="abcdefghi", ins_free=True), "delimiter pattern too long")])
def test_other_refusals_keep_their_messages(pat, kw, msg):
    for flag in (False, True):
        with pytest.raises(ag.AgrepError, match=msg):
            ag.Pattern(pat, sticky_delim=flag, **kw)


@pytest.mark.parametrize("dn", [d[0] for d in DELIMS])
@pytest.mark.parametrize("pn", ["k0", "k2", "k6", "v", "w", "hash", "comma"])
def test_descriptor_words_equal_the_checker(dn, pn):
    kw, pat = checker_kw(dn, pn)
    a = _oracle.compile(pat, **kw)
    D = ag.Pattern(pat, sticky_delim=True, **kw).desc
    assert (D.M, D.L, D.k, D.and_mode, D.delim_kind) == (a.M, a.L, a.k, a.and_mode, 3)
    for f in ("init0", "init1", "noerr", "endpos", "dendpos", "dmask", "wildmask"):
        assert getattr(D, f) == getattr(a, f), f
    assert D.init1 == (1 << 64) - 1
    assert [D.mask[c] for c in range(256)] == [a.mask[c] for c in range(256)]


def fill_ordinals(p, data, recs):
    arr = (_lib.Record * max(1, len(recs)))()
    for i, (b, e, *_r) in enumerate(recs):
        arr[i].begin, arr[i].end = b, e
    buf = (C.c_char * max(1, len(data))).from_buffer_copy(data or b"\0")
    _lib.lib().agb_fill_ordinals(p._h, buf, len(data), arr, len(recs))
    return [arr[i].ordinal for i in range(len(recs))]


@pytest.mark.parametrize("dn", [d[0] for d in DELIMS])
@pytest.mark.parametrize("tn", ["base", "starts", "open", "never"])
def test_host_ordinals_equal_the_checker(dn, tn):
    for pn in ("k0", "v", "hash"):
        kw, pat = checker_kw(dn, pn)
        data, a, cnt, recs = oracle_answer(dn, pn, tn)
        p = ag.Pattern(pat, sticky_delim=True, **kw)
        assert fill_ordinals(p, data, recs) == [r[2] for r in recs], (dn, pn, tn)


# ---- the delimiter pass (delim_state.cu) restated: one word per slice, byte s = the start states in state s ----
def accept_table(d):
    return [sum(0xFF << (8 * s) for s in range(len(d)) if d[s] == c) for c in range(256)]


def slice_function(tab, L, data):
    low = (1 << (8 * L)) - 1
    x = sum(1 << (9 * s) for s in range(L))
    for c in data:
        t = tab[c]
        adv = x & t
        x = (x & ~t & low) | (((adv << 8) | (adv >> (8 * (L - 1)))) & low)
    return [next(b for b in range(L) if x >> (8 * b + s) & 1) for s in range(L)]


def serial(d, s, data):
    closes = 0
    for c in data:
        if c == d[s]:
            s += 1
            if s == len(d):
                s, closes = 0, closes + 1
    return s, closes


@pytest.mark.parametrize("L", range(2, 9))
def test_slice_functions_compose_to_the_serial_rule(L):
    rnd = random.Random(L)
    for trial in range(40):
        alphabet = bytes(rnd.sample(b"abcde", rnd.randint(1, 3)))
        d = bytes(rnd.choice(alphabet) for _ in range(L))
        data = bytes(rnd.choice(alphabet + b"xy") for _ in range(rnd.randint(0, 700)))
        tab = accept_table(d)
        slices = [data[i:i + 128] for i in range(0, len(data), 128)]
        funcs = [slice_function(tab, L, sl) for sl in slices]
        for s0 in range(L):
            s = s0
            for sl, f in zip(slices, funcs):
                assert f[s] == serial(d, s, sl)[0]
                s = f[s]
            assert s == serial(d, s0, data)[0]
