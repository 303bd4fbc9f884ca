"""A set of files scanned in one device pass (agb_scan_set): every file's result, and its slice of the one record list,
equal agb_scan_host on that file alone, field by field; on small sets both equal the checker; the number of launches
does not grow with the number of files."""
import random, zlib
import pytest
import _oracle, _regex_oracle, _corpus
import agrep_b200 as ag
from agrep_b200 import _lib

pytestmark = pytest.mark.gpu

BODY = _corpus.make_text(6000, seed=4242, paragraphs=True)
SIZES = [0, 1, 15, 16, 17, 511, 512, 65535, 65536, 65537, 200 * 1024 + 3]

# (pattern, Pattern keywords): every engine -- bitap, asearch, asearch0, asearch1 costs, sgrep/bm, regex with levels --
# with -v, -n (ordinals), -w, -i, -x and user delimiters (a run, a word, an escaped byte)
CASES = [
    ("because", dict()),                                   # sgrep / bm
    ("because", dict(linenum=True)),                       # bitap
    ("because each", dict(k=2, linenum=True)),             # asearch
    ("government", dict(k=5)),                             # asearch0
    ("state good", dict(k=2, cost_i=2, cost_s=1, cost_d=3, linenum=True)),   # asearch1
    ("the", dict(inverse=True, linenum=True)),
    ("the", dict(inverse=True)),
    ("govern[a-m]ent", dict(k=1, wordbound=True, nocase=True, linenum=True)),
    ("state good", dict(ins_free=True, linenum=True)),                       # -p
    ("because", dict(k=1, linenum=True, delim="$$")),
    ("state good", dict(k=1, linenum=True, delim="the")),
    ("because", dict(k=2, inverse=True, linenum=True, delim="$$")),
    ("good", dict(k=0, linenum=True, delim="\\.")),
    ("state", dict(k=1, linenum=True, delim="aba")),                         # a delimiter that overlaps itself
    ("business give group toward young", dict(k=3, linenum=True)),          # 64-bit rows (M > 31)
    ("business give group toward young", dict(k=2, wordbound=True, linenum=True, delim="$$")),
    ("because|state", dict(regex=True, linenum=True)),
    ("gov(ern)*ment", dict(regex=True, k=1, inverse=True, linenum=True)),
    ("(business|give) group toward young people|state of the", dict(regex=True, k=2, linenum=True)),   # 64-bit regex words
]

# the cases the checker does not restate, and why (they are compared with agb_scan_host only); every other case must
# reach the checker
CHECKER_GAPS = {
    ("government", (("k", 5),)): "simple literals with k > 0: the checker forces the automaton only with linenum",
    ("the", (("inverse", True),)): "sgrep -v: the reference counts matching lines under -c, not restated",
}


def _key(pattern, kw):
    return (pattern, tuple(sorted(kw.items())))


def _file(rnd, size, delim):
    """a file of `size` bytes cut from the corpus, edges chosen at random: a leading delimiter, no trailing one, only
    delimiters, runs of the delimiter at both ends"""
    d = delim.replace("\\", "").encode() if delim else b"\n"
    kind = rnd.randrange(5)
    if kind == 0:
        body = (d * (size // len(d) + 1))[:size]
    else:
        st = rnd.randrange(max(1, len(BODY) - size))
        body = (BODY[st:st + size] * (size // max(1, len(BODY)) + 1))[:size]
        if kind == 1 and size >= 2 * len(d):
            head = d + d[1:] if len(d) > 1 else d      # ("ababa": occurrences that share a byte at the file's start)
            body = head + body[len(head):]
        elif kind == 2 and size >= 2 * len(d) + 2:
            body = d * 2 + body[2 * len(d):-2 * len(d)] + d * 2
        elif kind == 3 and size and body.endswith(b"\n"):
            body = body[:-1] + b"x"
    assert len(body) == size
    return body


def _fileset(rnd, delim, n):
    return [_file(rnd, rnd.choice(SIZES), delim) for _ in range(n)]


def _want(kw):
    return dict(ordinals=bool(kw.get("linenum")))


def _compare_alone(p, texts, kw, levels=False, capacity=None):
    """agb_scan_set against agb_scan_host per file; returns the set's per-file records"""
    total, per, recs = p.scan_set(texts, levels=levels, capacity=capacity, **_want(kw))
    assert len(per) == len(texts)
    at, used = 0, 0
    by_file = []
    for i, t in enumerate(texts):
        room = None if capacity is None else max(0, capacity - used)
        alone, arecs = p.scan_host(t, levels=levels, capacity=room, **_want(kw))
        r = per[i]
        assert r.n_matched == alone.n_matched, (i, len(t), r.n_matched, alone.n_matched)
        assert list(r.level_hist) == list(alone.level_hist), i
        assert r.n_closes == alone.n_closes, (i, r.n_closes, alone.n_closes)
        assert r.truncated == alone.truncated, i
        assert r.n_records == alone.n_records, i
        mine = recs[at:at + r.n_records]
        assert all(x[4] == i for x in mine), i
        assert [x[:4] for x in mine] == arecs, (i, len(t))
        by_file.append(mine)
        at += r.n_records
        used += r.n_matched
    assert at == len(recs) == total.n_records
    assert total.n_matched == sum(r.n_matched for r in per)
    return per, by_file


@pytest.mark.parametrize("pattern,kw", CASES)
def test_set_equals_each_file_alone(pattern, kw):
    rnd = random.Random(zlib.crc32(repr((pattern, sorted(kw.items()))).encode()))
    p = ag.Pattern(pattern, **kw)
    texts = _fileset(rnd, kw.get("delim"), 24)
    _compare_alone(p, texts, kw)
    if p.desc.engine == _lib.ENGINE_REGEX and not kw.get("inverse"):
        _compare_alone(p, texts, kw, levels=True)


@pytest.mark.parametrize("pattern,kw", CASES)
def test_small_sets_equal_the_checker(pattern, kw):
    rnd = random.Random(7)
    p = ag.Pattern(pattern, **kw)
    texts = [_file(rnd, s, kw.get("delim")) for s in (0, 1, 15, 16, 17, 511, 512, 3000)]
    per, by_file = _compare_alone(p, texts, kw)
    regex = p.desc.engine == _lib.ENGINE_REGEX
    gap = CHECKER_GAPS.get(_key(pattern, kw))
    if not regex:
        okw = {k: int(v) if not isinstance(v, str) else v for k, v in kw.items()}
        if gap:
            with pytest.raises(_oracle.OracleError):
                _oracle.compile(pattern, **okw)
            return
        a = _oracle.compile(pattern, **okw)
    else:
        a = _regex_oracle.compile(pattern, k=kw.get("k", 0), inverse=kw.get("inverse", False))
    for t, r, mine in zip(texts, per, by_file):
        cnt, orecs = (_regex_oracle if regex else _oracle).scan(a, t)
        assert r.n_matched == cnt
        assert [(b, e) for b, e, _, _, _ in mine] == [(b, e) for b, e, _ in orecs]
        if kw.get("linenum"):
            assert [o for _, _, o, _, _ in mine] == [o for _, _, o in orecs]


def test_levels_of_every_engine():
    rnd = random.Random(11)
    texts = _fileset(rnd, None, 16)
    for pattern, kw in (("because each", dict(k=3)), ("state good", dict(k=2, cost_i=2)), ("because|state", dict(regex=True, k=2)),
                        ("business give group toward young", dict(k=4)), ("(business|give) group toward young people|state of", dict(regex=True, k=3))):
        _compare_alone(ag.Pattern(pattern, **kw), texts, kw, levels=True)


def test_truncation_mid_file_and_at_a_file_end():
    rnd = random.Random(3)
    p = ag.Pattern("the", linenum=True)
    texts = [t for t in _fileset(rnd, None, 12) if t.count(b"the") > 2][:5]
    assert len(texts) >= 3
    per, _ = _compare_alone(p, texts, dict(linenum=True))
    counts = [r.n_matched for r in per]
    for cap in (1, counts[0] - 1, counts[0], counts[0] + counts[1], counts[0] + counts[1] + 1, sum(counts) - 1, sum(counts)):
        total, _, recs = p.scan_set(texts, capacity=cap, ordinals=True)
        assert total.truncated == (sum(counts) > cap) and len(recs) == min(cap, sum(counts))
        _compare_alone(p, texts, dict(linenum=True), capacity=cap)


def test_count_only_and_the_complement():
    rnd = random.Random(5)
    texts = _fileset(rnd, None, 30) + [BODY * 20]        # one file above the complement count pass's 1 MiB
    for pattern, kw in (("the", dict()), ("the", dict(inverse=True)), ("because each", dict(k=2))):
        p = ag.Pattern(pattern, **kw)
        total, per, recs = p.scan_set(texts, want_records=False)
        assert recs == []
        for t, r in zip(texts, per):
            alone, _ = p.scan_host(t, want_records=False)
            assert r.n_matched == alone.n_matched


def test_launches_do_not_grow_with_the_number_of_files():
    rnd = random.Random(9)
    p = ag.Pattern("because each", k=2, linenum=True)
    L = _lib.lib()
    many = [_file(rnd, rnd.choice([100, 4096, 9000]), None) for _ in range(1000)]
    p.scan_set(many[:2], ordinals=True)                   # the record list's size does not change the launches either
    grow = []
    for texts in (many[:2], many):
        before = L.agb_kernel_launches()
        p.scan_set(texts, ordinals=True)
        grow.append(L.agb_kernel_launches() - before)
    assert grow[0] == grow[1], grow


# ---- the command line: many small files go through agb_scan_set, one above its budget through agb_scan_host ----
CLI_CASES = [["-c", "the"], ["-l", "government"], ["-n", "because each"], ["-n", "-1", "because each"], ["-n", "-v", "-1", "the"],
             ["-c", "-n", "-v", "the"], ["-n", "-d", "$$", "-1", "because each"], ["-n", "-w", "-1", "matching"],
             ["-n", "-2", "c(o|x)lou*r"], ["-c", "-v", "the|of"], ["-n", "-1", "gov(ern)*ment"]]


@pytest.mark.parametrize("args", CLI_CASES)
def test_cli_over_many_files_equals_the_reference(args, tmp_path):
    import os, subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ref, mine = os.path.join(root, "oracle", "_ref", "agrep"), os.path.join(root, "agrep_b200", "agrep-b200")
    if not os.path.exists(ref):
        pytest.skip("oracle/_ref/agrep not built")
    rnd = random.Random(21)
    names = []
    for i in range(300):
        (tmp_path / ("f%03d.txt" % i)).write_bytes(_file(rnd, rnd.choice([0, 1, 17, 512, 3000, 9000]), "$$" if "$$" in args else None) + b"\n")
        names.append("f%03d.txt" % i)
    (tmp_path / "big.txt").write_bytes(BODY * 60)          # above the command line's set budget: scanned alone
    files = names[:150] + ["big.txt", "missing.txt"] + names[150:]
    outs = [subprocess.run([b] + args + files, capture_output=True, timeout=600, stdin=subprocess.DEVNULL, cwd=tmp_path) for b in (ref, mine)]
    assert outs[0].returncode == outs[1].returncode, args
    assert outs[0].stdout == outs[1].stdout, args
    assert b"missing.txt" in outs[0].stderr and b"missing.txt" in outs[1].stderr, args
