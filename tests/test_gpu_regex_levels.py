"""Levels scans of regular expressions (AGB_WANT_LEVELS on AGB_ENGINE_REGEX, regex.cu): every matching line's smallest
error level and the level histogram, against the checker (tests/_regex_oracle.py) run at each level; every entry point,
the shard-local walk, a 1 GiB corpus, and the -B sweeps of the stand-alone command line and of the drop-in against the
reference's output.

A line's expected level is the smallest k' in 0..K at which the checker reports it (under -v: the checker with
inverse=True).  A levels scan at K reports exactly the lines that have such a level; without -v these are the lines the
checker reports at K, because re()'s rows are nested (test_regex_levels_host.py checks that on the checker)."""
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


def checker_levels(pattern, data, K, nocase=False, inverse=False, counts=None):
    """the expected ordered (begin, end, ordinal, level) list and the checker's count at each k' in 0..K"""
    if counts is None:
        counts = [R.scan(R.compile(pattern, k=kk, nocase=nocase, inverse=inverse), data) for kk in range(K + 1)]
    first = {}
    for kk in range(K + 1):
        for r in counts[kk][1]:
            first.setdefault(r, kk)
    return sorted(r + (lv,) for r, lv in first.items()), [c for c, _ in counts[:K + 1]]


def gpu_levels(pattern, data, K, nocase=False, inverse=False):
    p = ag.Pattern(pattern, k=K, nocase=nocase, inverse=inverse, regex=True)
    res, recs = p.scan_host(data, capacity=len(data) + 2, ordinals=True, levels=True)
    return res, [tuple(r) for r in recs]


def same_levels(pattern, data, K, nocase=False, inverse=False, counts=None):
    want, cnt = checker_levels(pattern, data, K, nocase, inverse, counts)
    res, got = gpu_levels(pattern, data, K, nocase, inverse)
    key = (pattern, K, nocase, inverse)
    assert got == want, key
    assert res.n_matched == len(want), key
    hist = [0] * (_lib.AGB_MAXERR + 1)
    for r in want:
        hist[r[3]] += 1
    assert list(res.level_hist) == hist, key
    if not inverse:
        assert res.n_matched == cnt[K], key
        assert [res.level_hist[l] for l in range(K + 1)] == [cnt[l] - (cnt[l - 1] if l else 0) for l in range(K + 1)], key
    # count only: the same histogram
    rc, _ = ag.Pattern(pattern, k=K, nocase=nocase, inverse=inverse, regex=True).scan_host(data, want_records=False, levels=True)
    assert rc.n_matched == res.n_matched and list(rc.level_hist) == list(res.level_hist), key
    return want


@pytest.mark.parametrize("K", [2, 4])
@pytest.mark.parametrize("pattern", [p for p in T.FIXED if R.is_regex(p.encode())])
def test_fixed(pattern, K):
    if K >= len(pattern):
        pytest.skip("pattern shorter than k")
    same_levels(pattern, T.TEXT, K)


def test_random_differential():
    """the 320 random cases of test_gpu_regex (both word widths, -i, -v) at K = the case's k and at K = 4"""
    from test_gpu_regex import differential_cases
    data = _corpus.make_text(800, seed=31) + b"no newline at the end"
    for p, k, nocase, inverse in differential_cases():
        counts = [R.scan(R.compile(p, k=kk, nocase=nocase, inverse=inverse), data) for kk in range(5)]
        same_levels(p, data, k, nocase, inverse, counts)
        if k != 4 and len(p) > 4:
            same_levels(p, data, 4, nocase, inverse, counts)


@pytest.mark.parametrize("name", ["empty", "no_trailing_newline", "blank_lines", "long_line", "long_line_end", "tile_crossing", "tile_exact"])
@pytest.mark.parametrize("pattern,K", [("c(o|x)lou*r", 2), ("(th|wh)e*", 4), ("^$|zzz*", 1)])
def test_edges(name, pattern, K):
    from test_gpu_regex import edge_texts
    same_levels(pattern, edge_texts()[name], K)


def test_entry_points_agree():
    """host, device, file descriptor and resident text give the same levels; ordinals alongside"""
    import torch
    data = _corpus.make_text(3000, seed=8)
    L = _lib.lib()
    for pattern, K in (("(because|each) (state|world)", 2), ("gov(ern)*mentz", 4), ("th(e|a)*t", 4)):
        p = ag.Pattern(pattern, k=K, regex=True)
        want = _lib.WANT_RECORDS | _lib.WANT_ORDINALS | _lib.WANT_LEVELS
        cap = 40000
        host_res, host = p.scan_host(data, capacity=cap, ordinals=True, levels=True)
        t = torch.frombuffer(bytearray(data + b"\0" * 64), dtype=torch.uint8).cuda()
        rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
        res = _lib.Result()
        assert L.agb_scan_device(p._h, C.c_void_p(t.data_ptr()), len(data), want, C.c_void_p(rec.data_ptr()), cap, None, C.byref(res)) == 0
        dev = [tuple(r) for r in rec[:res.n_records].cpu().tolist()]           # level | pad << 32, pad = 0
        with tempfile.TemporaryFile() as f:
            f.write(data); f.seek(0)
            recs = (_lib.Record * cap)(); rf = _lib.Result()
            assert L.agb_scan_fd(p._h, f.fileno(), want, recs, cap, C.byref(rf)) == 0
            fd = [(recs[i].begin, recs[i].end, recs[i].ordinal, recs[i].level) for i in range(rf.n_records)]
        txt = C.c_void_p()
        assert L.agb_text_from_host(data, len(data), C.byref(txt)) == 0
        recs2 = (_lib.Record * cap)(); rt = _lib.Result()
        assert L.agb_scan_text(p._h, txt, want, recs2, cap, C.byref(rt)) == 0
        L.agb_text_free(txt)
        resident = [(recs2[i].begin, recs2[i].end, recs2[i].ordinal, recs2[i].level) for i in range(rt.n_records)]
        expect, cnt = checker_levels(pattern, data, K)
        assert host == dev == fd == resident == expect and cnt[K] > 0, pattern
        assert {l for *_, l in expect} != {K}, pattern                       # more than one level occurs
        hists = [list(r.level_hist) for r in (host_res, res, rf, rt)]
        assert hists[0] == hists[1] == hists[2] == hists[3], pattern
        # count only, every entry point: the same histogram as the list's
        c = _lib.Result()
        assert L.agb_scan_device(p._h, C.c_void_p(t.data_ptr()), len(data), _lib.WANT_LEVELS, None, 0, None, C.byref(c)) == 0
        assert list(c.level_hist) == hists[0] and c.n_matched == cnt[K]


def shard_levels(pattern, K, data, world):
    """the shard-local walk of test_gpu_shard.scan_in_shards with AGB_WANT_LEVELS: per-shard histograms and the stitched
    (begin, end, ordinal, level) list"""
    import torch
    L = _lib.lib()
    p = ag.Pattern(pattern, k=K, regex=True)
    n = len(data)
    per = max(512, (n // world) // 512 * 512)
    offs = [min(r * per, n) for r in range(world)] + [n]
    cap = n + 2
    out, hists, closes_before, origin, matched = [], [], 0, 0, 0
    for r in range(world):
        n_local = offs[r + 1] - offs[r]
        hl = _lib.HALO_LEFT if r > 0 else 0
        hr = min(_lib.HALO_RIGHT, n - offs[r + 1])
        ext = data[offs[r] - hl:offs[r + 1] + hr]
        t = torch.frombuffer(bytearray(ext + b"\0" * 64), dtype=torch.uint8).cuda()
        rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
        res, part = _lib.Result(), _lib.ShardPart()
        want = _lib.WANT_RECORDS | _lib.WANT_ORDINALS | _lib.WANT_LEVELS
        rc = L.agb_scan_shard_local(p._h, C.c_void_p(t.data_ptr() + hl), n_local, hl, hr, int(r == 0), int(r == world - 1),
                                    int(offs[r + 1] + hr >= n), want, C.c_void_p(rec.data_ptr()), cap, None, C.byref(res), C.byref(part))
        assert rc == 0, L.agb_last_error()
        if r == 0:
            origin = part.ord_origin
        base = offs[r] + part.byte_base
        for b, e, j, lv in rec[:res.n_records].cpu().tolist():
            out.append((b + base, e + base, j + origin + closes_before - part.ord_fix, lv))
        closes_before += part.closes
        matched += res.n_matched
        hists.append(list(res.level_hist))
    return matched, out, hists


@pytest.mark.parametrize("world", [3, 7])
@pytest.mark.parametrize("pattern,K", [("(because|each) (state|world)", 2), ("gov(ern)*mentz", 4), ("^$|the*y", 1)])
def test_shard_local(world, pattern, K):
    from test_gpu_shard import ragged_text
    data = ragged_text(5) + b"\n" + _corpus.make_text(1500, seed=9)
    expect, cnt = checker_levels(pattern, data, K)
    whole, _ = gpu_levels(pattern, data, K)
    matched, got, hists = shard_levels(pattern, K, data, world)
    assert matched == cnt[K] == len(expect) and cnt[K] > 0
    assert got == expect
    assert [sum(h[l] for h in hists) for l in range(_lib.AGB_MAXERR + 1)] == list(whole.level_hist)


def test_1gib_corpus():
    """one levels count at K = 4 over a 1 GiB synthetic corpus answers the plain counts at k = 0..4"""
    import torch
    n = 1 << 30
    t = torch.empty(n + 4096, dtype=torch.uint8, device="cuda")
    ag.corpus_device(t.data_ptr(), n, seed=4711)
    for pattern in ("(because|each) (state|world)", "gov(ern)*mentz"):
        lv = ag.Pattern(pattern, k=4, regex=True).scan_device(t.data_ptr(), n, levels=True)
        plain = [ag.Pattern(pattern, k=k, regex=True).scan_device(t.data_ptr(), n).n_matched for k in range(5)]
        assert [sum(lv.level_hist[:k + 1]) for k in range(5)] == plain, (pattern, list(lv.level_hist), plain)
        assert lv.n_matched == plain[4] and plain[4] > plain[0]


# ---- -B with a regular expression: the stand-alone command line against the reference's stdout
# (tests/golden/regex_levels_cli_stdout.json, recorded by tests/golden/make_regex_levels_golden.py) ----
# best levels 1, 2, 3 and 4 on t.txt; -n; two files whose best levels differ (u.txt's is the smaller one, so the sweep
# stops there -- the reference goes by the last file's count alone); no -y with stdin closed (the prompt reads EOF and
# nothing is printed); -B -v, whose sweep is the per-level one (a nullable pattern: every line matches, so the sweep ends
# at k = M - 1 without a match).  None has a best level above 4: the reference crashes there.
CLI_CASES = [
    (["-B", "-y", "co(x|z)lour*"], ["t.txt"]),
    (["-B", "-y", "stat(e|u)*xqw"], ["t.txt"]),
    (["-B", "-y", "stat(e|u)*xqwj"], ["t.txt"]),
    (["-B", "-y", "wor(l|d)*qzxjv"], ["t.txt"]),
    (["-n", "-B", "-y", "peo(p|l)*qjz"], ["t.txt"]),
    (["-B", "-y", "wor(l|d)*qzxj"], ["t.txt", "u.txt"]),
    (["-B", "stat(e|u)*xqw"], ["t.txt"]),
    (["-B", "-v", "-y", "(x|y)*"], ["t.txt"]),
]


def cli_key(args, files):
    return " ".join(args + files)


def cli_files(d):
    with open(os.path.join(d, "t.txt"), "wb") as f:
        f.write(T.EDGE + _corpus.make_text(400, seed=3))
    with open(os.path.join(d, "u.txt"), "wb") as f:
        f.write(_corpus.make_text(300, seed=21))


def run_cli(binary, args, files, d):
    p = subprocess.run([binary] + args + files, capture_output=True, timeout=300, stdin=subprocess.DEVNULL, cwd=d)
    return {"rc": p.returncode, "bytes": len(p.stdout), "sha256": hashlib.sha256(p.stdout).hexdigest()}


def test_cli_bestmatch_against_reference():
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "regex_levels_cli_stdout.json")))
    binary = os.path.join(ROOT, "agrep_b200", "agrep-b200")
    with tempfile.TemporaryDirectory() as d:
        cli_files(d)
        for args, files in CLI_CASES:
            assert run_cli(binary, args, files, d) == golden[cli_key(args, files)], cli_key(args, files)


def test_cli_bestmatch_stderr():
    """the count the sweep reports, and one 'can't open' line per pass the per-level sweep made: the first scan, the
    levels 1..3, and the printing pass"""
    binary = os.path.join(ROOT, "agrep_b200", "agrep-b200")
    with tempfile.TemporaryDirectory() as d:
        cli_files(d)
        p = subprocess.run([binary, "-B", "-y", "stat(e|u)*xqwj", "t.txt", "missing.txt"], capture_output=True, timeout=300,
                           stdin=subprocess.DEVNULL, cwd=d)
    want, _ = checker_levels("stat(e|u)*xqwj", T.EDGE + _corpus.make_text(400, seed=3), 4)
    n3 = sum(1 for r in want if r[3] == 3)
    assert n3 > 0 and not any(r[3] < 3 for r in want)
    assert p.returncode == n3
    missing = b"agrep-b200: can't open file for reading: missing.txt\n"
    assert p.stderr == missing * 4 + b"agrep-b200: %d words match within 3 errors\n" % n3 + missing


# ---- the drop-in: exec()'s -B counting passes of a re() pattern from the levels memo, against the reference ----
DROPIN_CASES = [
    (["-B", "-y", "stat(e|u)*xqw"], ["t.txt"]),
    (["-B", "-y", "stat(e|u)*xqwj"], ["t.txt"]),
    (["-B", "-y", "wor(l|d)*qzxjv"], ["t.txt"]),
    (["-n", "-B", "-y", "peo(p|l)*qjz"], ["t.txt"]),
    (["-B", "-y", "wor(l|d)*qzxj"], ["t.txt", "u.txt"]),
    (["-B", "-y", "sta(t|e)*qzjx"], ["t.txt", "u.txt"]),
]


@pytest.mark.parametrize("args,files", DROPIN_CASES)
def test_dropin_bestmatch(args, files):
    ref, drop = os.path.join(ROOT, "oracle", "_ref", "agrep"), os.path.join(ROOT, "oracle", "_ref", "agrep_dropin")
    if not (os.path.exists(ref) and os.path.exists(drop)):
        pytest.skip("oracle/_ref binaries not built")
    with tempfile.TemporaryDirectory() as d:
        cli_files(d)
        outs = [subprocess.run([b] + args + files, capture_output=True, timeout=300, stdin=subprocess.DEVNULL, cwd=d)
                for b in (ref, drop)]
    assert outs[0].returncode == outs[1].returncode, args
    assert outs[0].stdout == outs[1].stdout, args
    assert outs[0].stdout
