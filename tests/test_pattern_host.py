"""Host-side checks of the product's pattern front-end (agrep_b200/csrc/pattern.c) -- no GPU needed:
 * the descriptor words equal the reference's globals after maskgen() (golden dumps from the real reference);
 * they equal the oracle's independent restatement, also beyond 32 positions;
 * the C ABI library loads and exports every symbol include/agrep_b200.h declares."""
import ctypes, json, os, random, re
import pytest
import _oracle, _corpus
import agrep_b200 as ag
from agrep_b200 import _lib
from test_oracle_golden import G, _args_to_kw

LUT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "lut_lower1.json")))


def api_kw(okw):
    kw = {k: v for k, v in okw.items() if k != "width"}
    return kw


def test_library_exports_declared_symbols():
    L = _lib.lib()
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "include", "agrep_b200.h")).read()
    declared = set(re.findall(r"\b(agb_[a-z_0-9]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(L, name), name
    assert set(_lib.EXPORTS) <= declared
    assert b"sm_90a" in L.agb_version()


@pytest.mark.parametrize("name", sorted(G["dump"]))
def test_words_equal_reference_globals(name):
    d = G["dump"][name]
    kw = api_kw(_args_to_kw(d["ref_args"]))
    p = ag.Pattern(d["pattern"], **kw)
    D = p.desc
    m32 = 0xFFFFFFFF
    assert D.M == d["M"]
    assert D.init0 & m32 == d["Init0"]
    assert D.init1 & m32 == d["Init1"]
    assert D.noerr & m32 == d["NO_ERR_MASK"]
    assert D.endpos == d["endposition"]
    assert D.dendpos == d["D_endpos"]
    assert D.wildmask == d["wildmask"]
    assert D.and_mode == d["AND"]
    fold = D.engine == 0 and kw.get("nocase")           # bitap.c:171 applies LUT[] before Mask[]
    for c in range(256):
        src = LUT[c] if fold else c
        assert D.mask[c] == d["mask"].get(str(src), 0), c
    # upper halves: the always-on feed continues to bit 63
    assert D.init0 >> 32 == m32 and D.init1 >> 32 == m32 and D.noerr >> 32 == m32


PATTERNS = ["abc", "because each", "pat[a-t]ern", "<algo>rithm", "state;world", "state,world;", "a#t", "st.ing", "^the",
            "world$", "The World", "[^a-s]he ", "x[a\\-c]y", "x[\\]a]y", "a\\.b\\;c", "(ab)c", "[A-Z]x", "ab[.]c", "q<ab>#c",
            "people how too little state good very make world", "a,b,c", "[a-cx-z0-9]+", "one;two;three"]
OPTS = [dict(), dict(k=1), dict(k=2, nocase=1), dict(k=3, wordbound=1), dict(k=1, wholeline=1), dict(k=2, delim="$$"),
        dict(k=1, delim="the"), dict(k=2, ins_free=1), dict(k=3, cost_i=2, cost_d=3), dict(k=2, cost_s=2, inverse=1),
        dict(k=0, nocase=1), dict(k=0, delim="\\<x")]


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("oi", range(len(OPTS)))
def test_words_equal_oracle(pattern, oi):
    okw = dict(OPTS[oi], linenum=1)
    try:
        a = _oracle.compile(pattern, **okw)
    except _oracle.OracleError as e:
        with pytest.raises(ag.AgrepError):
            ag.Pattern(pattern, **okw)
        return
    D = ag.Pattern(pattern, **okw).desc
    assert (D.M, D.L, D.k, D.and_mode, D.engine) == (a.M, a.L, a.k, a.and_mode, a.engine)
    for f in ("init0", "init1", "noerr", "endpos", "dendpos", "dmask", "wildmask"):
        assert getattr(D, f) == getattr(a, f), f
    lut = LUT if (a.engine == 0 and okw.get("nocase")) else list(range(256))
    for c in range(256):
        assert D.mask[c] == a.mask[lut[c]], c
    assert bytes(D.delim[:D.L]) == bytes(a.dpat[:a.L])


def test_engine_selection_follows_checksg():
    E = lambda *a, **k: ag.Pattern(*a, **k).desc.engine
    assert E("the") == 4 and E("the", nocase=1) == 4 and E("the", wordbound=1) == 4      # sgrep/bm
    assert E("the", linenum=1) == 0 and E("th.e") == 0 and E("^the") == 0              # bitap exact
    assert E("the", bestmatch=1) == 0
    assert E("hello", k=1) == 1 and E("hello", k=4, nocase=1) == 1                      # asearch
    assert E("hello world", k=5) == 2 and E("hello world", k=8) == 2                    # asearch0
    assert E("hello", k=2, cost_s=2) == 3                                               # asearch1
    with pytest.raises(ag.AgrepError):
        ag.Pattern("ab", k=2)            # checksg.c:34
    with pytest.raises(ag.AgrepError):
        ag.Pattern("a*b")                # regular expressions are outside the path
    with pytest.raises(ag.AgrepError):
        ag.Pattern("a" * 63, k=1, linenum=1)   # 1 + 1 + 63 positions > 63
    assert ag.Pattern("a" * 61, k=1, linenum=1).desc.M == 63


def test_anchor_plan():
    d = ag.Pattern("because each", k=2).desc
    assert d.plan == ag.api.PLAN_ANCHORS and d.n_anchors == 3 and d.anchor_len == 4
    assert [d.anchor[i].to_bytes(4, "little") for i in range(3)] == [b"beca", b"use ", b"each"]
    d = ag.Pattern("because each", k=3).desc           # 4 runs of 3
    assert d.n_anchors == 4 and d.anchor_len == 3 and d.anchor_mask == 0xFFFFFF
    d = ag.Pattern("the").desc                          # bm: always case folded
    assert d.n_anchors == 1 and d.anchor_len == 3 and d.anchor_fold == 0x20202020 and d.anchor[0] == 0x656874
    assert ag.Pattern("because each", k=2, inverse=1).desc.plan == ag.api.PLAN_ALL
    assert ag.Pattern("government", k=2, ins_free=1).desc.plan == ag.api.PLAN_ALL
    assert ag.Pattern("a.b.c.d", k=1, linenum=1).desc.plan == ag.api.PLAN_ALL
    d = ag.Pattern("state,world", linenum=1).desc       # OR: one anchor per alternative
    assert d.n_anchors == 2
    d = ag.Pattern("Hello World", k=1, nocase=1).desc
    assert d.anchor_fold == 0x20202020 and all((d.anchor[i] & d.anchor_fold) == d.anchor_fold for i in range(d.n_anchors))


def test_anchor_plan_over_two_valued_classes():
    """a position that accepts two bytes may sit inside an anchor piece: every spelling of the piece is an anchor at the same
    place (pattern.c collect_runs); literal runs of the same length are preferred, and the text-sampling planner keeps away"""
    def anchors(d):
        return sorted((d.anchor[i].to_bytes(4, "little")[:d.anchor_len], d.anchor_off[i]) for i in range(d.n_anchors))
    d = ag.Pattern("b[ea]c.u[s-t]e", k=1, linenum=1).desc
    assert d.plan == ag.api.PLAN_ANCHORS and d.anchor_len == 3 and d.refine == 1 and d.adaptive == 0
    assert anchors(d) == [(b"bac", 0), (b"bec", 0), (b"use", 4), (b"ute", 4)]
    d = ag.Pattern("b[ea]cause", linenum=1).desc                      # the literal run "caus" does it alone
    assert anchors(d) == [(b"caus", 2)] and d.adaptive == 1
    d = ag.Pattern("ab[cd]efg[hi]jk", k=1, linenum=1).desc            # four-byte pieces with a class beat two-byte literal runs
    assert anchors(d) == [(b"abce", 0), (b"abde", 0), (b"fghj", 4), (b"fgij", 4)]
    d = ag.Pattern("[Tt]he [qQ]uick", k=1, nocase=1).desc            # under -i the two cases of a letter are one spelling
    assert anchors(d) == [(b"quic", 4), (b"the ", 0)]
    d = ag.Pattern("a[bcd]e[fgh]i[jkl]m", k=1, linenum=1).desc       # three-valued classes break the runs
    assert d.plan == ag.api.PLAN_ALL
    d = ag.Pattern("x[ab][cd][ef][gh]y", k=0, linenum=1).desc         # at most four spellings per piece
    assert d.plan == ag.api.PLAN_ANCHORS and d.n_anchors <= 4


def test_corpus_generator_properties():
    c = ag.corpus_host(64 * 4096, needle="because each", needle_every=4, needle_maxedits=3)
    assert len(c) == 64 * 4096 and c.count(b"\0") == 0 and max(c) < 128
    for pg in range(64):
        assert c[pg * 4096 + 4095] == 10
    assert c == ag.corpus_host(64 * 4096, needle="because each", needle_every=4, needle_maxedits=3)
    # shards are position independent
    assert c[16 * 4096:32 * 4096] == ag.corpus_host(16 * 4096, first_page=16, needle="because each", needle_every=4, needle_maxedits=3)
    assert c.count(b"because each") >= 4
    p = ag.corpus_host(16 * 4096, paragraphs=True)
    assert b"\n\n" in p


@pytest.mark.parametrize("pattern,kw,corpus_kw", [
    ("because each", dict(k=2, linenum=1), dict(nlines=2000, seed=31)),
    ("the", dict(k=0, linenum=1, wordbound=1), dict(nlines=800, seed=32, trailing_newline=False)),
    ("state", dict(k=1, linenum=1, delim="$$"), dict(nlines=1500, seed=33, paragraphs=True)),
    ("world", dict(k=1, linenum=1, delim="the"), dict(nlines=600, seed=34)),
    ("governmental", dict(k=5, linenum=1), dict(nlines=1500, seed=35)),
    ("state", dict(k=1, linenum=1, delim="aba"), "overlap"),            # a delimiter that overlaps itself: taken from the left
    ("e", dict(k=0, linenum=1, delim="e e"), "overlap"),
])
def test_fill_ordinals_reproduces_j(pattern, kw, corpus_kw):
    """agb_fill_ordinals() (host helper for -n) against the oracle's j, which is pinned to the reference's -n output"""
    data = _corpus.overlap_text(kw["delim"], 9) if corpus_kw == "overlap" else _corpus.make_text(**corpus_kw)
    a = _oracle.compile(pattern, **kw)
    cnt, recs = _oracle.scan(a, data)
    assert cnt > 0
    p = ag.Pattern(pattern, **kw)
    arr = (_lib.Record * cnt)()
    for i, (b, e, j) in enumerate(recs):
        arr[i].begin, arr[i].end = b, e
    _lib.lib().agb_fill_ordinals(p._h, data, len(data), arr, cnt)
    assert [arr[i].ordinal for i in range(cnt)] == [j for _, _, j in recs]


def test_random_patterns_product_front_end_equals_oracle_front_end():
    """differential fuzz of two independent restatements of checksg + preprocess + maskgen: the product's host front-end
    (agrep_b200/csrc/pattern.c) and the oracle's (oracle/agrep_oracle.c, pinned to the reference's dumps): same
    accept/reject decision, same automaton words, same masks, for random patterns over letters and metacharacters."""
    import random
    rnd = random.Random(2026)
    atoms = list("abcdeXYZ 09") + [".", "#", "[a-c]", "[^xy]", "<ab>", "\\.", "\\[", ",", ";", "^", "$", "[x\\-z]", "(", ")", "-", "~", "{", "]",
                                   "[z-a]", "[#-e]", "\\", "<", ">", "\xe9", "\xc9"]     # (no bare "[": "[-" and "-]" are undefined behaviour in maskgen.c:106-109)
    checked = rejected = 0
    for _ in range(600):
        pat = "".join(rnd.choice(atoms) for _ in range(rnd.randint(1, 12)))
        kw = dict(k=rnd.choice([0, 0, 1, 2, 3, 5]), linenum=1)
        if rnd.random() < 0.3: kw["nocase"] = 1
        if rnd.random() < 0.2: kw["wordbound"] = 1
        if rnd.random() < 0.1: kw["wholeline"] = 1
        if rnd.random() < 0.15: kw["delim"] = rnd.choice(["$$", "ab", "\\.", "X"])
        if rnd.random() < 0.1: kw["ins_free"] = 1
        # a lone backslash at the very end escapes what preprocess() appended: the terminator (ignored by both, like the
        # reference) or the '<' of the -w/-x wrapper (the oracle follows the reference's quirk, the product refuses)
        stripped = pat.replace("\\\\", "")
        if stripped.endswith("\\") and (kw.get("wordbound") or kw.get("wholeline")):
            with pytest.raises(ag.AgrepError):
                ag.Pattern(pat, **kw)
            rejected += 1
            continue
        try:
            a = _oracle.compile(pat, **kw)
        except _oracle.OracleError:
            with pytest.raises(ag.AgrepError):
                ag.Pattern(pat, **kw)
            rejected += 1
            continue
        if kw.get("nocase") and any(ch.isalpha() for ch in kw.get("delim", "")):
            # the reference folds the delimiter too (-i -d X splits at 'x' and 'X', maskgen.c:52-58, 259-266): the oracle
            # follows it; the product carries it as delim_fold (0x20 per delimiter letter) for the code that finds
            # delimiters by their bytes -- the descriptor words themselves are compared below like everyone else's
            assert a.mask[ord("x")] == a.mask[ord("X")] or "X" not in kw["delim"]
            if not kw.get("ins_free") or a.L == 1:
                Df = ag.Pattern(pat, **kw).desc
                assert [Df.delim_fold[i] for i in range(Df.L)] == [0x20 if chr(a.dpat[i]).isalpha() else 0 for i in range(a.L)], (pat, kw)
        if kw.get("ins_free") and a.L > 1:
            # -p makes the delimiter's positions sticky too ("a ... b" closes like "ab"): the oracle follows the reference,
            # the product refuses (found by the GPU scan fuzz: the device looks for delimiters by their bytes)
            with pytest.raises(ag.AgrepError, match="-p with a delimiter"):
                ag.Pattern(pat, **kw)
            rejected += 1
            continue
        D = ag.Pattern(pat, **kw).desc
        assert (D.M, D.L, D.k, D.and_mode, D.engine) == (a.M, a.L, a.k, a.and_mode, a.engine), (pat, kw)
        for f in ("init0", "init1", "noerr", "endpos", "dendpos", "dmask", "wildmask"):
            assert getattr(D, f) == getattr(a, f), (pat, kw, f)
        lut = LUT if (a.engine == 0 and kw.get("nocase")) else list(range(256))     # bitap.c:171: the exact engine folds through LUT[]
        assert [D.mask[c] for c in range(256)] == [a.mask[lut[c]] for c in range(256)], (pat, kw)
        assert bytes(D.delim[:D.L]) == bytes(a.dpat[:a.L])
        checked += 1
    assert checked > 150 and rejected > 20, (checked, rejected)
