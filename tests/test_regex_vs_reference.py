"""Pins the regular-expression checker (tests/_regex_oracle.py) against the unmodified reference agrep's re().  The
reference's answers -- counts and `-n` line numbers of the same seeded texts -- are stored in
tests/golden/regex_answers.json.gz, so the comparison runs on any checkout; tests/golden/make_regex_golden.py records
them again from a reference binary built by oracle/Makefile (same record-then-replace scheme as make_golden.py).

Pinned where re() is right (SURVEY 8c): <= 15 positions at k = 0..4 without '?' and without a position of more than ten
follow entries; past 15 positions (re1()) only the counts at k = 0.  One test per reference defect shows the difference."""
import gzip, hashlib, json, os, random, re, subprocess, tempfile
import pytest
import _corpus
import _regex_oracle as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "regex_answers.json.gz")
RECORD_WITH = os.environ.get("AGB_RECORD_REFERENCE")
ANSWERS = {} if RECORD_WITH else json.loads(gzip.decompress(open(GOLDEN, "rb").read()))
if RECORD_WITH:
    import atexit
    atexit.register(lambda: open(GOLDEN + ".new", "wb").write(gzip.compress(json.dumps(ANSWERS, sort_keys=True, separators=(",", ":")).encode(), 9, mtime=0)))


def _run(args, data):
    with tempfile.NamedTemporaryFile(suffix=".txt", delete=False) as f:
        f.write(data)
        path = f.name
    try:
        return subprocess.run([RECORD_WITH, "-V0"] + args + [path], capture_output=True, timeout=120)
    finally:
        os.unlink(path)


ASK = {
    "count": lambda p: int(p.stdout.strip() or b"0"),
    "ordinals": lambda p: [int(m.group(1)) for m in re.finditer(rb"^(\d+): ", p.stdout, re.M)],
    # the messages without the program name in front ("<path of the binary>: "), one per line
    "stderr": lambda p: [p.returncode, [ln.split(": ", 1)[1] if ln.startswith(RECORD_WITH + ": ") else ln
                                        for ln in p.stderr.decode("latin-1").splitlines()]],
}


def ref_answer(kind, args, data):
    h = hashlib.sha256(kind.encode())
    for a in args:
        h.update(b"\0" + (a if isinstance(a, bytes) else a.encode("latin-1")))
    h.update(b"\0\0" + data)
    key = h.hexdigest()[:24]
    if RECORD_WITH:
        ANSWERS[key] = ASK[kind](_run(args, data))
    assert key in ANSWERS, "no stored reference answer for %s %r (tests/golden/make_regex_golden.py)" % (kind, args)
    return ANSWERS[key]


# texts that end in a newline: re()'s file mode never reports an unterminated last line (r_output, agrep.c:1923)
TEXT = _corpus.make_text(1500, seed=12345)
SMALL = _corpus.make_text(300, seed=4242)
EDGE = b"colour\ncolor\n\nxyz\ncolouur colr\n^$\nthe colxur here\nfoo\n\n\nabc\n"


def oracle(pattern, data, k=0, nocase=False, inverse=False):
    return R.scan(R.compile(pattern, k=k, nocase=nocase, inverse=inverse), data)


def flags(k, nocase, inverse):
    return (["-%d" % k] if k else []) + (["-i"] if nocase else []) + (["-v"] if inverse else [])


def check(pattern, data, k=0, nocase=False, inverse=False):
    if k >= len(pattern):
        pytest.skip("the pattern must be longer than the number of errors (checksg.c:34)")
    cnt, recs = oracle(pattern, data, k, nocase, inverse)
    args = flags(k, nocase, inverse) + [pattern]
    assert cnt == ref_answer("count", ["-c"] + args, data), (pattern, k, nocase, inverse)
    assert [j - 1 for _, _, j in recs] == ref_answer("ordinals", ["-n"] + args, data), (pattern, k, nocase, inverse)


FIXED = [
    # every operator, nesting, '.', classes, ^ and $, '#'
    "c(o|x)lou*r", "(each|both) (st|wo)", "gov(ern)*ment", "th(e|a)*t", "((a|e)n)*d", "go*d",
    "wor.d|sta.e", "[a-d]e*t", "[^a-s]he*", "^the|day$", "^(an|the)* ", "s$|^t", "w#d", "a#t|zz", "(ma|pa)t*ern",
    "(x|y)*", "be(c|a)(a|u)*se", "\\.|e*s", "[abc]*x|never", "al(go|ri)*thm",
]


@pytest.mark.parametrize("k", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("pattern", FIXED)
def test_fixed(pattern, k):
    check(pattern, SMALL, k=k)


@pytest.mark.parametrize("pattern,k", [("c(o|x)lou*r", 0), ("c(o|x)lou*r", 2), ("^$|x*yz", 0), ("a*", 0), ("(f|x)o*", 1)])
def test_edges(pattern, k):
    check(pattern, EDGE, k=k)


@pytest.mark.parametrize("pattern,k", [("The|Government", 0), ("(Each|BOTH) wo*", 1), ("[A-G]over*n", 2)])
def test_nocase(pattern, k):
    check(pattern, TEXT, k=k, nocase=True)


@pytest.mark.parametrize("pattern,k", [("the|of", 0), ("(each|both) (st|wo)", 1), ("gov(ern)*ment", 3)])
def test_inverse(pattern, k):
    check(pattern, TEXT, k=k, inverse=True)


def random_regex(rnd, words):
    """a regex of corpus words: alternations, groups, stars and dots, at most 13 positions of its own"""
    def piece():
        w = rnd.choice(words)[:rnd.randint(2, 5)]
        r = rnd.random()
        if r < 0.25:
            i = rnd.randrange(len(w))
            return w[:i + 1] + "*" + w[i + 1:]
        if r < 0.4:
            i = rnd.randrange(len(w))
            return w[:i] + "." + w[i + 1:]
        if r < 0.5:
            return "(" + w + ")*"
        return w
    r = rnd.random()
    if r < 0.4:
        return "(" + piece() + "|" + piece() + ")" + rnd.choice(["", " ", "*", "e"]) + piece()
    if r < 0.7:
        return piece() + "|" + piece() + ("|" + piece() if rnd.random() < 0.3 else "")
    return piece() + "*" + piece()


def random_cases(n, seed=2024, maxpos=15):
    rnd = random.Random(seed)
    words = sorted({w for w in TEXT.decode().split() if w.isalpha() and len(w) >= 3})
    out = []
    while len(out) < n:
        p = random_regex(rnd, words)
        if not R.is_regex(p.encode()):
            continue
        a = R.compile(p)
        if a.M > maxpos or max(bin(f).count("1") for f in a.follow[1:]) > 10:
            continue
        out.append((p, rnd.randint(0, 4), rnd.random() < 0.15, rnd.random() < 0.1))
    return out


@pytest.mark.parametrize("pattern,k,nocase,inverse", random_cases(240))
def test_random_differential(pattern, k, nocase, inverse):
    check(pattern, SMALL, k=k, nocase=nocase, inverse=inverse)


@pytest.mark.parametrize("pattern", ["abcdefghijklmn(o|p)", "(because|each|state|world) ", "governmental|homogeneous"])
def test_re1_counts(pattern):
    """16..30 positions go to re1(): its counts are right here (its line numbers are not, defect 2; and at 29 positions
    '(because|each|state|world) (of|the)' finds nothing at all)"""
    assert R.compile(pattern).M > 15
    data = b"abcdefghijklmno\nx\nabcdefghijklmnp\nabcdefghijklmnq\n" + SMALL
    assert oracle(pattern, data)[0] == ref_answer("count", ["-c", pattern], data)


# ---- the reference's defects (SURVEY 8c): the checker (and the engine) differ on purpose ----
DEFECT_TEXT = b"xay\nxjy\nxky\nxly\nabcdefghijklmno\nq\nabcdefghijklmnop\nabcdefghijklmnox\ncolour\ncolor\nfoo\n"


def test_defect1_follow_cap():
    """compute_next keeps ten follow entries per position: the 11th and 12th alternatives are lost (the pattern has 16
    positions, so re1() also prints wrong line numbers for the two lines it finds)"""
    p = "x(a|b|c|d|e|f|g|h|i|j|k|l)y"
    ours = [j - 1 for _, _, j in oracle(p, DEFECT_TEXT)[1]]
    assert ours == [1, 2, 3, 4]
    assert ref_answer("count", ["-c", p], DEFECT_TEXT) == 2
    assert ref_answer("ordinals", ["-n", "x[a-l]y"], DEFECT_TEXT) == [1, 2, 3, 4]


def test_defect2_re1_line_numbers():
    p = "abcdefghijklmn(o|p)"
    ours = [j - 1 for _, _, j in oracle(p, DEFECT_TEXT)[1]]
    assert ours == [5, 7, 8]
    ref = ref_answer("ordinals", ["-n", p], DEFECT_TEXT)
    assert len(ref) == 3 and ref != ours


def test_defect3_re1_errors():
    p = "cdefghijklmn(o|p)x"
    assert [j - 1 for _, _, j in oracle(p, DEFECT_TEXT, k=1)[1]] == [5, 7, 8]
    assert 7 not in ref_answer("ordinals", ["-n", "-1", p], DEFECT_TEXT)
    assert 7 in ref_answer("ordinals", ["-n", "-1", "klmn(o|p)x"], DEFECT_TEXT)


def test_defect4_optional():
    """'?' is an operator to parse.c and a literal position to maskgen(): the reference matches nothing"""
    for p in ("colou?r|xyz", "(colou?r|xyz)"):
        assert [j - 1 for _, _, j in oracle(p, DEFECT_TEXT)[1]] == [9, 10]
        assert ref_answer("ordinals", ["-n", p], DEFECT_TEXT) == []
    assert ref_answer("ordinals", ["-n", "c(o|x)lou*r"], DEFECT_TEXT) == [9, 10]


def test_defect5_wholeline():
    """-x with a regex: the reference does not match 'foo' against fo*; the engine refuses -x with a regex"""
    assert ref_answer("ordinals", ["-n", "-x", "fo*"], DEFECT_TEXT) == []


REFUSALS = [  # (reference arguments, agb_compile keyword arguments)
    (["-d", "$$", "a|b"], dict(delim="$$")), (["-w", "a|b"], dict(wordbound=True)), (["a|b,c"], {}), (["a|b;c;d"], {}),
    (["a|b;c"], {}), (["b;c|zz"], {}), (["fo*;the"], {}), (["(ab|c"], {}), (["ab|c)"], {}), (["a||b"], {}), (["<ab|c"], {}),
    (["-5", "ab|cdef"], dict(k=5)), (["-8", "abcdefgh|ijk"], dict(k=8)),
]


@pytest.mark.parametrize("args,kw", REFUSALS)
def test_refusal_messages(args, kw):
    """the reference's refusals and agb_compile's: the same message (the command line prints it after its name)"""
    import agrep_b200 as ag
    rc, err = ref_answer("stderr", args, SMALL)
    assert rc == 255 and err, (args, rc, err)
    with pytest.raises(ag.AgrepError) as e:
        ag.Pattern(args[-1], regex=True, **kw)
    assert str(e.value) == err[0], (args, err)


def test_position_limit_difference():
    """32 positions: the reference refuses more than 30 (preproce.c:378); the engine takes up to 63 (DESIGN 3.6)"""
    import agrep_b200 as ag
    p = "(a|b)(c|d)(e|f)(g|h)(i|j)(k|l)(m|n)(o|p)(q|r)(s|t)(u|v)(w|x)(y|z)(a|b)(c|d)"
    assert ref_answer("stderr", [p], SMALL) == [255, ["regular expression too long"]]
    assert ag.Pattern(p, regex=True).desc.M == 32
