"""The regular-expression front-end of agb_compile (pattern.c) on the host: acceptance, refusals and their messages, and
the words and follow sets against the independent checker (tests/_regex_oracle.py)."""
import random
import pytest
import agrep_b200 as ag
from agrep_b200 import _lib
import _regex_oracle as R
import test_regex_vs_reference as T


def test_refused_without_regex_option():
    with pytest.raises(ag.AgrepError, match="regular expressions"):
        ag.Pattern("a*b")
    with pytest.raises(ag.AgrepError, match="regular expressions"):
        ag.Pattern("colo|colour")


def test_engine_value():
    p = ag.Pattern("c(o|x)lou*r", regex=True)
    assert p.desc.engine == _lib.ENGINE_REGEX == 5
    assert _lib.ENGINE_NAMES[5] == "regex"
    assert p.regex is not None and p.regex.head == 1 and p.regex.tail == 1
    # a pattern without '|' or '*' stays on its engine, '?' and '(' included
    assert ag.Pattern("colou?r", regex=True).desc.engine != 5
    assert ag.Pattern("colou?r", regex=True).regex is None


@pytest.mark.parametrize("kw,msg", [
    (dict(delim="$$"), "-d or -w option is not supported for this pattern"),
    (dict(wordbound=True), "-d or -w option is not supported for this pattern"),
    (dict(wholeline=True), "-x is not supported for regular expressions"),
    (dict(k=5), "the maximum number of erorrs allowed for full regular expressions is 4"),
    (dict(k=8), "the maximum number of erorrs allowed for full regular expressions is 4"),
])
def test_option_refusals(kw, msg):
    with pytest.raises(ag.AgrepError) as e:
        ag.Pattern("abcdefgh|ijk", regex=True, **kw)
    assert str(e.value) == msg


@pytest.mark.parametrize("pattern", ["a|b,c", "a|b;c;d", "(ab|c", "ab|c)", "a||b", "*ab|c", "(|a)*", "a|", "[z-a]*b", "[-a]*b",
                                     "ab*\\", "()*a"])
def test_illegal(pattern):
    with pytest.raises(ag.AgrepError) as e:
        ag.Pattern(pattern, regex=True)
    assert str(e.value) == "illegal regular expression"


@pytest.mark.parametrize("pattern", ["a|b;c", "b;c|zz", "fo*;the"])
def test_one_semicolon(pattern):
    """one ';' passes preprocess() and parse(); maskgen() refuses it (maskgen.c:150-163)"""
    with pytest.raises(ag.AgrepError) as e:
        ag.Pattern(pattern, regex=True)
    assert str(e.value) == "illegal pattern: cannot handle AND (';') and OR (',')/regular-expressions simultaneously"


def test_too_long():
    letters = "abcdefghijklmnopqrstuvwxyz" * 3
    assert ag.Pattern("(" + "|".join(letters[:61]) + ")*", regex=True).desc.M == 63     # 61 positions of its own + 2
    with pytest.raises(ag.AgrepError) as e:
        ag.Pattern("(" + "|".join(letters[:62]) + ")*", regex=True)
    assert str(e.value) == "regular expression too long"


def test_angle_unmatched():
    with pytest.raises(ag.AgrepError, match="unmatched '<', '>'"):
        ag.Pattern("<ab|c", regex=True)


def test_costs_ignored():
    """-I/-S/-D are ignored for a regular expression (compat.c:75-79): same words as without them"""
    a, b = ag.Pattern("ab*c|d", k=2, regex=True).desc, ag.Pattern("ab*c|d", k=2, cost_s=2, cost_i=3, regex=True).desc
    assert bytes(a) == bytes(b)


def test_bestmatch_refused():
    with pytest.raises(ag.AgrepError, match="-B"):
        ag.bestmatch_device("c(o|x)lou*r", 0, 0, regex=1)


def words_equal(pattern, k=0, nocase=False, inverse=False):
    p = ag.Pattern(pattern, k=k, nocase=nocase, inverse=inverse, regex=True)
    d, rx = p.desc, p.regex
    a = R.compile(pattern, k=k, nocase=nocase, inverse=inverse)
    M = a.M
    assert d.M == M, pattern
    assert [rx.follow[q] for q in range(M + 1)] == a.follow, pattern
    assert list(d.mask) == a.mask, pattern
    field = (1 << (M + 1)) - 1
    assert d.noerr & field == a.noerr & field, pattern
    assert (d.init0, d.init1, d.endpos, d.k, d.nrows, d.inverse) == (a.init0, a.init1, 1, k, k + 1, int(inverse))
    assert list(d.reset)[:k + 1] == list(a.reset) == list(d.start)[:k + 1], pattern
    assert (d.L, d.delim[0], d.start_closes, d.plan) == (1, 10, 1, _lib.PLAN_ALL)


@pytest.mark.parametrize("pattern", [p for p in T.FIXED if R.is_regex(p.encode())] + ["<ab>c*|d", "a<b|c>d*", "[.x]*y|z", "a.b*|$", "x?y*z", "(a|b)?(c|d)*e?"])
@pytest.mark.parametrize("k", [0, 2, 4])
def test_words_fixed(pattern, k):
    if k >= len(pattern):
        pytest.skip("pattern shorter than k")
    words_equal(pattern, k=k)


def test_words_random():
    """the words of 300 random regexes of corpus words, up to 63 positions, against the checker"""
    rnd = random.Random(77)
    words = sorted({w for w in T.TEXT.decode().split() if w.isalpha() and len(w) >= 3})
    done = 0
    while done < 300:
        p = "|".join(T.random_regex(rnd, words) for _ in range(rnd.randint(1, 4)))
        if rnd.random() < 0.2:
            p = "(" + p + ")?" + rnd.choice(words)[:3]
        try:
            a = R.compile(p)
        except R.RegexError:
            continue
        k = rnd.randint(0, 4)
        if k >= len(p):
            continue
        words_equal(p, k=k, nocase=rnd.random() < 0.3, inverse=rnd.random() < 0.2)
        done += 1
