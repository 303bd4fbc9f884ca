"""Regular expressions on the device (regex.cu) against the checker (tests/_regex_oracle.py): bit-exact counts and ordered
(begin, end, ordinal) lists, every entry point, the shard-local walk, a 1 GiB corpus, and the stand-alone command line
against the reference's stdout."""
import ctypes as C
import hashlib, json, os, random, subprocess, tempfile
import pytest
import _corpus
import _regex_oracle as R
import agrep_b200 as ag
from agrep_b200 import _lib
import test_regex_vs_reference as T

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu(pattern, data, k=0, nocase=False, inverse=False):
    p = ag.Pattern(pattern, k=k, nocase=nocase, inverse=inverse, regex=True)
    res, recs = p.scan_host(data, capacity=len(data) + 2, ordinals=True)
    return res, [(b, e, j) for b, e, j, _ in recs]


def same(pattern, data, k=0, nocase=False, inverse=False):
    cnt, orecs = R.scan(R.compile(pattern, k=k, nocase=nocase, inverse=inverse), data)
    res, recs = gpu(pattern, data, k, nocase, inverse)
    assert res.n_matched == cnt, (pattern, k, nocase, inverse, res.n_matched, cnt)
    assert recs == orecs, (pattern, k, nocase, inverse)
    return cnt


@pytest.mark.parametrize("k", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("pattern", [p for p in T.FIXED if R.is_regex(p.encode())])
def test_fixed(pattern, k):
    if k >= len(pattern):
        pytest.skip("pattern shorter than k")
    same(pattern, T.TEXT, k=k)


@pytest.mark.parametrize("pattern,k,nocase,inverse", [("The|Government", 0, 1, 0), ("(Each|BOTH) wo*", 1, 1, 0), ("the|of", 0, 0, 1),
                                                        ("(because|each|state|world) (of|the)*", 0, 0, 0), ("x(a|b|c|d|e|f|g|h|i|j|k|l)y", 0, 0, 0),
                                                        ("colou?r|xyz", 0, 0, 0), ("(because|each) (state|world)", 4, 0, 1)])
def test_goldens(pattern, k, nocase, inverse):
    same(pattern, T.TEXT, k=k, nocase=nocase, inverse=inverse)
    same(pattern, T.DEFECT_TEXT, k=min(k, 1), nocase=nocase, inverse=inverse)


def differential_cases(n=320, seed=99):
    rnd = random.Random(seed)
    words = sorted({w for w in T.TEXT.decode().split() if w.isalpha() and len(w) >= 3})
    out = []
    while len(out) < n:
        p = "|".join(T.random_regex(rnd, words) for _ in range(rnd.choice([1, 1, 2, 3])))
        if rnd.random() < 0.15:
            p = "(" + p + ")?" + rnd.choice(words)[:3]
        if rnd.random() < 0.1:
            p = "^" + p
        try:
            R.compile(p)
        except R.RegexError:
            continue
        k = rnd.randint(0, 4)
        if k < len(p):
            out.append((p, k, rnd.random() < 0.2, rnd.random() < 0.15))
    return out


def test_random_differential():
    """320 random regexes of corpus words (up to 63 positions, both word widths) x k x -i/-v"""
    data = _corpus.make_text(800, seed=31) + b"no newline at the end"
    for p, k, nocase, inverse in differential_cases():
        same(p, data, k=k, nocase=nocase, inverse=inverse)


def edge_texts():
    rnd = random.Random(5)
    words = T.TEXT.decode().split()
    long_line = " ".join(rnd.choice(words) for _ in range(20000)).encode()[:100 * 1024]
    crossing = b"".join((" ".join(rnd.choice(words) for _ in range(rnd.randint(0, 700)))).encode() + b"\n" for _ in range(300))
    return {
        "empty": b"", "no_trailing_newline": b"colour\nthe colxur", "newline_first": b"\ncolour\n", "blank_lines": b"\n" * 100,
        "only_newline": b"\n", "long_line": b"colour\n" + long_line + b" colour\nxyz", "long_line_end": long_line,
        "tile_crossing": crossing, "tile_exact": (b"a" * 32767 + b"\n") * 3 + b"colour",
    }


@pytest.mark.parametrize("name", sorted(edge_texts()))
@pytest.mark.parametrize("pattern,k", [("c(o|x)lou*r", 0), ("c(o|x)lou*r", 2), ("^$|zzz*", 0), ("a*", 0), ("(th|wh)e*", 4)])
def test_edges(name, pattern, k):
    same(pattern, edge_texts()[name], k=k)


def test_entry_points_agree():
    import torch
    data = _corpus.make_text(3000, seed=8)
    L = _lib.lib()
    for pattern, k in (("(because|each) (state|world)", 0), ("gov(ern)*ment", 2), ("th(e|a)*t", 4)):
        p = ag.Pattern(pattern, k=k, regex=True)
        want = _lib.WANT_RECORDS | _lib.WANT_ORDINALS
        cap = 20000
        host_res, host = p.scan_host(data, capacity=cap, ordinals=True)
        t = torch.frombuffer(bytearray(data + b"\0" * 64), dtype=torch.uint8).cuda()
        rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
        res = _lib.Result()
        assert L.agb_scan_device(p._h, C.c_void_p(t.data_ptr()), len(data), want, C.c_void_p(rec.data_ptr()), cap, None, C.byref(res)) == 0
        dev = [tuple(r[:3]) for r in rec[:res.n_records].cpu().tolist()]
        with tempfile.TemporaryFile() as f:
            f.write(data); f.seek(0)
            recs = (_lib.Record * cap)(); rf = _lib.Result()
            assert L.agb_scan_fd(p._h, f.fileno(), want, recs, cap, C.byref(rf)) == 0
            fd = [(recs[i].begin, recs[i].end, recs[i].ordinal) for i in range(rf.n_records)]
        txt = C.c_void_p()
        assert L.agb_text_from_host(data, len(data), C.byref(txt)) == 0
        recs2 = (_lib.Record * cap)(); rt = _lib.Result()
        assert L.agb_scan_text(p._h, txt, want, recs2, cap, C.byref(rt)) == 0
        L.agb_text_free(txt)
        resident = [(recs2[i].begin, recs2[i].end, recs2[i].ordinal) for i in range(rt.n_records)]
        hostl = [(b, e, j) for b, e, j, _ in host]
        cnt, orecs = R.scan(R.compile(pattern, k=k), data)
        assert hostl == dev == fd == resident == orecs and cnt > 0
        assert host_res.n_matched == res.n_matched == rf.n_matched == rt.n_matched == cnt
        # count only, -c -v
        assert p.scan_host(data, want_records=False)[0].n_matched == cnt
        pv = ag.Pattern(pattern, k=k, inverse=True, regex=True)
        assert pv.scan_host(data, want_records=False)[0].n_matched == R.scan(R.compile(pattern, k=k, inverse=True), data)[0]


@pytest.mark.parametrize("world", [3, 7])
@pytest.mark.parametrize("pattern,k", [("(because|each) (state|world)", 0), ("gov(ern)*ment", 2), ("^$|the*y", 1)])
def test_shard_local(world, pattern, k):
    from test_gpu_shard import scan_in_shards, ragged_text
    data = ragged_text(5) + b"\n" + _corpus.make_text(1500, seed=9)
    cnt, recs = R.scan(R.compile(pattern, k=k), data)
    matched, got, n_closes = scan_in_shards(pattern, dict(k=k, regex=True), data, world)
    assert matched == cnt and cnt > 0
    assert got == recs


def test_1gib_corpus():
    """additivity over parts of a 1 GiB synthetic corpus, and 32 windows against the checker"""
    import torch
    n = 1 << 30
    t = torch.empty(n + 4096, dtype=torch.uint8, device="cuda")
    ag.corpus_device(t.data_ptr(), n, seed=4711)
    host = t[:n].cpu().numpy().tobytes()
    for pattern, k in (("(because|each) (state|world)", 0), ("(because|each) (state|world)", 2)):
        p = ag.Pattern(pattern, k=k, regex=True)
        whole = p.scan_device(t.data_ptr(), n).n_matched
        # parts scanned as texts of their own, cut behind the first newline after a page boundary (no line straddles two)
        parts, cuts = 0, [300 << 20, 301 << 20, 777 << 20]
        bounds = [0]
        for c in cuts:
            bounds.append(host.index(b"\n", c) + 1)
        bounds.append(n)
        for a, b in zip(bounds, bounds[1:]):
            sub = torch.zeros(b - a + 4096, dtype=torch.uint8, device="cuda")
            sub[:b - a] = t[a:b]
            parts += p.scan_device(sub.data_ptr(), b - a).n_matched
        assert parts == whole and whole > 0
        a_ = R.compile(pattern, k=k)
        rnd = random.Random(k)
        for _ in range(32):
            s = rnd.randrange(0, n - (1 << 16))
            s = host.index(b"\n", s) + 1
            e = host.index(b"\n", s + 60000) + 1
            win = host[s:e]
            res, _ = p.scan_host(win, want_records=False)
            assert res.n_matched == R.scan(a_, win, want_records=False)[0]


# ---- the stand-alone command line against the reference's stdout (tests/golden/regex_cli_stdout.json) ----
CLI_CASES = [
    ["-n", "-2", "c(o|x)lou*r"], ["-n", "c(o|x)lou*r"], ["-c", "(each|both) (st|wo)"], ["-n", "-1", "gov(ern)*ment"],
    ["-n", "-i", "The|GOVERNMENT"], ["-c", "-v", "the|of"], ["-n", "^the|day$"], ["-n", "-B", "c(o|x)lou*r"], ["-n", "-B", "-y", "co(x|z)lour*"],
    ["-n", "-4", "th(e|a)*t"], ["-d", "$$", "a|b"], ["-w", "a|b"], ["a|b,c"], ["-5", "abcdef|ghi"], ["-n", "-x", "fo*"],
]


def cli_files(d):
    with open(os.path.join(d, "t.txt"), "wb") as f:
        f.write(T.EDGE + _corpus.make_text(400, seed=3))


def run_cli(binary, args, d):
    p = subprocess.run([binary] + args + ["t.txt"], capture_output=True, timeout=300, stdin=subprocess.DEVNULL, cwd=d)
    return {"rc": p.returncode, "bytes": len(p.stdout), "sha256": hashlib.sha256(p.stdout).hexdigest()}


def test_cli_against_reference():
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "regex_cli_stdout.json")))
    binary = os.path.join(ROOT, "agrep_b200", "agrep-b200")
    with tempfile.TemporaryDirectory() as d:
        cli_files(d)
        for args in CLI_CASES:
            key = " ".join(args)
            if args[-1] == "fo*" and "-x" in args:
                # -x with a regex is refused (the reference quietly matches nothing, SURVEY 8c)
                assert run_cli(binary, args, d)["rc"] == 255
                continue
            got = run_cli(binary, args, d)
            assert got == golden[key], key


def test_cli_bestmatch_stops_at_four():
    """-B with a regex whose best level would be above 4: the sweep stops at 4 with a message (the reference crashes,
    SURVEY 8c)"""
    binary = os.path.join(ROOT, "agrep_b200", "agrep-b200")
    with tempfile.TemporaryDirectory() as d:
        cli_files(d)
        p = subprocess.run([binary, "-B", "-y", "-n", "qqqqqqqqq|zzzzzzzzz", "t.txt"], capture_output=True, timeout=300,
                           stdin=subprocess.DEVNULL, cwd=d)
    assert p.returncode == 0
    assert p.stdout == b"Grand Total: 0 match(es) found.\n"
    assert b"no match within 4 errors, the most a regular expression allows" in p.stderr


def test_shard_line_past_halo_is_reported():
    """a line of the first shard that runs past the right halo, and matches only behind it: the scan fails with
    AGB_ERR_ARG (the line cannot be finished) instead of leaving it out of the count"""
    import torch
    L = _lib.lib()
    head = _corpus.make_text(200, seed=2)
    long_line = b"x" * (200 * 1024) + b" colour"
    data = head + long_line + b"\n" + _corpus.make_text(2000, seed=3)
    per = (len(head) + 4096) // 512 * 512                      # the long line opens in shard 0 and crosses its end
    hr = _lib.HALO_RIGHT
    p = ag.Pattern("c(o|x)lou*r", regex=True)
    t = torch.frombuffer(bytearray(data[:per + hr] + b"\0" * 64), dtype=torch.uint8).cuda()
    cap = 100000
    rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
    res, part = _lib.Result(), _lib.ShardPart()
    rc = L.agb_scan_shard_local(p._h, C.c_void_p(t.data_ptr()), per, 0, hr, 1, 0, 0, _lib.WANT_RECORDS, C.c_void_p(rec.data_ptr()),
                                cap, None, C.byref(res), C.byref(part))
    assert rc == -3, (rc, res.n_matched)
    assert b"runs past its halo" in L.agb_last_error()


# ---- the drop-in: the reference program over libagrepb200_dropin.so, re() on the engine ----
DROPIN_CASES = [
    ["-n", "c(o|x)lou*r"], ["-n", "-2", "c(o|x)lou*r"], ["-c", "(each|both) (st|wo)"], ["-n", "-1", "gov(ern)*ment"],
    ["-n", "-i", "The|GOVERNMENT"], ["-n", "-v", "the|of"], ["-c", "-v", "the|of"], ["-n", "^the|day$"], ["-n", "-4", "th(e|a)*t"],
    ["-n", "-3", "(ma|pa)t*ern"], ["-l", "c(o|x)lou*r"], ["-n", "s$|^t"], ["-n", "abcdefghijklmn(o|p)"],
    ["-n", "-B", "-y", "co(x|z)lour*"], ["-n", "x(a|b|c|d|e|f|g|h|i|j|k|l)y"],
]


@pytest.mark.parametrize("args", DROPIN_CASES)
def test_dropin_stdout(args):
    ref, drop = os.path.join(ROOT, "oracle", "_ref", "agrep"), os.path.join(ROOT, "oracle", "_ref", "agrep_dropin")
    if not (os.path.exists(ref) and os.path.exists(drop)):
        pytest.skip("oracle/_ref binaries not built")
    with tempfile.TemporaryDirectory() as d:
        # small files that end in a newline: re()'s file-mode artefacts (SURVEY 8c) do not occur in them
        open(os.path.join(d, "t.txt"), "wb").write(T.EDGE + T.DEFECT_TEXT + _corpus.make_text(400, seed=3))
        open(os.path.join(d, "u.txt"), "wb").write(_corpus.make_text(300, seed=21))
        outs = [subprocess.run([b] + args + ["t.txt", "u.txt"], capture_output=True, timeout=300, stdin=subprocess.DEVNULL, cwd=d)
                for b in (ref, drop)]
    assert outs[0].returncode == outs[1].returncode, args
    assert outs[0].stdout == outs[1].stdout, args
    assert outs[0].stdout
