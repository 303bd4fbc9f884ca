"""-p with a record delimiter of two or more bytes (delim_kind 3) on the device: the delimiter pass (delim_state.cu) and the
dense tile form.  Counts, ordered records, ordinals and levels equal to the checker through every scan entry point --
host, fd, device, resident text, sets, windows small enough that their edges fall part way into a delimiter --; a record
that spans many tiles; 256 MiB against the checker; the sharded scans' refusal; and the stand-alone command line and the
drop-in print what the reference prints on the golden cases."""
import ctypes as C
import json, os, random, subprocess
import pytest
import _oracle, _corpus
import agrep_b200 as ag
from agrep_b200 import _lib
from golden.make_sticky_delim_golden import CASES, DELIMS, NOT_RESTATED, argv, case_text, checker_kw, dbytes, key, reference_j

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "agrep")
DROP = os.path.join(ROOT, "oracle", "_ref", "agrep_dropin")
CLI = os.path.join(ROOT, "agrep_b200", "agrep-b200")
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "sticky_delim_answers.json")))


def strewn(delim, nbytes, seed):
    """corpus text with the delimiter's bytes strewn about: records of every length, delimiters part way done everywhere"""
    db = dbytes(delim)
    rnd = random.Random(seed)
    t = bytearray(_corpus.make_text(nbytes // 60 + 1, seed=seed))[:nbytes]
    for _ in range(nbytes // 300):
        at = rnd.randrange(len(t))
        t[at:at + 1] = bytes([db[rnd.randrange(len(db))]])
    for _ in range(nbytes // 20000):
        at = rnd.randrange(len(t))
        t[at:at + len(db)] = db
    return bytes(t)


def checker(pat, kw, data):
    cnt, recs = _oracle.scan(_oracle.compile(pat, **kw), data)
    return cnt, reference_j(recs, kw, data)


def every_entry(p, data, tmp_path, windows=(4096, 8192)):
    """(count, ordered list with ordinals) through the host, windowed, fd, device and resident-text entries: all equal"""
    import torch
    res, recs = p.scan_host(data, ordinals=True)
    got = [(b, e, j) for b, e, j, _ in recs]
    assert p.scan_host(data, want_records=False)[0].n_matched == res.n_matched
    for window in windows:
        r2, rec2 = p.scan_host(data, ordinals=True, window=window)
        assert (r2.n_matched, r2.n_closes, [(b, e, j) for b, e, j, _ in rec2]) == (res.n_matched, res.n_closes, got), window
    f = tmp_path / "t.txt"
    f.write_bytes(data)
    with open(f, "rb") as fh:
        r3, rec3 = p.scan_fd(fh.fileno(), ordinals=True)
    assert (r3.n_matched, [(b, e, j) for b, e, j, _ in rec3]) == (res.n_matched, got)
    with open(f, "rb") as fh:
        r4, rec4 = p.scan_fd(fh.fileno(), ordinals=True, window=windows[0])
    assert (r4.n_matched, [(b, e, j) for b, e, j, _ in rec4]) == (res.n_matched, got)
    t = torch.frombuffer(bytearray(data + b"\0" * 64), dtype=torch.uint8).cuda()
    cap = res.n_matched + 16
    d_rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
    r5 = p.scan_device(t.data_ptr(), len(data), d_records=d_rec.data_ptr(), capacity=cap, ordinals=True)
    rows = d_rec[:r5.n_records].cpu().tolist()
    assert (r5.n_matched, [(b, e, j) for b, e, j, _ in rows]) == (res.n_matched, got)
    htxt = C.c_void_p()
    buf = (C.c_char * max(1, len(data))).from_buffer_copy(data or b"\0")
    assert _lib.lib().agb_text_from_host(buf, len(data), C.byref(htxt)) == 0
    try:
        arr, r6 = (_lib.Record * cap)(), _lib.Result()
        assert _lib.lib().agb_scan_text(p._h, htxt, _lib.WANT_RECORDS | _lib.WANT_ORDINALS, arr, cap, C.byref(r6)) == 0
        assert (r6.n_matched, [(arr[i].begin, arr[i].end, arr[i].ordinal) for i in range(r6.n_records)]) == (res.n_matched, got)
    finally:
        _lib.lib().agb_text_free(htxt)
    return res.n_matched, got


PATS = [("because", {}), ("because each", dict(k=2)), ("government policy", dict(k=6)), ("because", dict(inverse=1)),
        ("the", dict(wordbound=1)), ("wh#ld", {}), ("because,people", {})]


@pytest.mark.parametrize("dname,delim,_a,dkw", DELIMS, ids=[d[0] for d in DELIMS])
@pytest.mark.parametrize("pat,kw", PATS, ids=["k0", "k2", "k6", "v", "w", "hash", "comma"])
def test_parity_with_the_checker(dname, delim, _a, dkw, pat, kw, tmp_path):
    kw = dict(kw, ins_free=1, delim=delim, **dkw)
    data = strewn(delim, 150000, seed=len(delim) * 31 + len(pat))
    p = ag.Pattern(pat, sticky_delim=True, **kw)
    assert p.desc.delim_kind == 3
    cnt, recs = checker(pat, kw, data)
    n, got = every_entry(p, data, tmp_path)
    assert n == cnt and got == recs


@pytest.mark.parametrize("dn,pn,tn", [c for c in CASES if c[1] != "S2"], ids=[key(*c) for c in CASES if c[1] != "S2"])
def test_golden_texts(dn, pn, tn):
    kw, pat = checker_kw(dn, pn)
    data = case_text(dn, tn)
    p = ag.Pattern(pat, sticky_delim=True, **kw)
    res, recs = p.scan_host(data, ordinals=True)
    assert res.n_matched == GOLDEN[key(dn, pn, tn)]["count"]
    assert [(b, e, j) for b, e, j, _ in recs] == checker(pat, kw, data)[1]


@pytest.mark.parametrize("delim", ["ab", "e ", "aa", "the and "])
def test_levels(delim):
    data = strewn(delim, 120000, seed=9)
    kw = dict(ins_free=1, delim=delim)
    p = ag.Pattern("because each", k=4, sticky_delim=True, **kw)
    res, recs = p.scan_host(data, levels=True)
    cnt, hist, orecs = _oracle.scan_levels(_oracle.compile("because each", k=4, **kw), 4, data)
    assert list(res.level_hist)[:5] == hist[:5]
    assert [(b, e, l) for b, e, _, l in recs] == [(b, e, l) for b, e, _, l in orecs]


def test_a_set_of_files():
    texts = [b"", strewn("ab", 70000, 1), b"ab", b"xaxbyab", strewn("ab", 40000, 2)[:33333], strewn("ab", 5000, 3)]
    kw = dict(ins_free=1, delim="ab")
    p = ag.Pattern("because", sticky_delim=True, **kw)
    total, per, recs = p.scan_set(texts, ordinals=True)
    at = 0
    for i, t in enumerate(texts):
        cnt, orecs = checker("because", kw, t)
        assert per[i].n_matched == cnt, i
        assert [(b, e, j) for b, e, j, _l, f in recs[at:at + cnt]] == orecs and all(r[4] == i for r in recs[at:at + cnt]), i
        at += cnt
    assert total.n_matched == at


def test_one_record_over_many_tiles(tmp_path):
    """1 MiB of 'a' under -d ab: the delimiter is part way done from the first byte on and never completes in the text"""
    data = b"a" * (1 << 20)
    kw = dict(ins_free=1, delim="ab")
    for pat in ("aaaa", "xyz"):
        p = ag.Pattern(pat, sticky_delim=True, **kw)
        cnt, recs = checker(pat, kw, data)
        n, got = every_entry(p, data, tmp_path, windows=(65536,))
        assert n == cnt and got == recs
    data = b"a" * (1 << 20) + b"b" + b"a" * 5000 + b"b"
    p = ag.Pattern("aaaa", sticky_delim=True, **kw)
    assert every_entry(p, data, tmp_path, windows=(65536,))[1] == checker("aaaa", kw, data)[1]


def test_256_mib_against_the_checker():
    import torch
    n = 256 << 20
    t = torch.empty(n + 64, dtype=torch.uint8, device="cuda")
    ag.corpus_device(t.data_ptr(), n, seed=4242, needle="because each", needle_every=8, needle_maxedits=2)
    t[n:] = 0
    data = t[:n].cpu().numpy().tobytes()
    for pat, kw in (("because each", dict(k=2)), ("because", {})):
        kw = dict(kw, ins_free=1, delim="e ")
        p = ag.Pattern(pat, sticky_delim=True, **kw)
        a = _oracle.compile(pat, **kw)
        cap = 20000
        cnt, head = _oracle.scan(a, data, cap=cap)
        res = p.scan_device(t.data_ptr(), n)
        assert res.n_matched == cnt
        d_rec = torch.zeros((cnt + 16, 4), dtype=torch.int64, device="cuda")
        res = p.scan_device(t.data_ptr(), n, d_records=d_rec.data_ptr(), capacity=cnt + 16, ordinals=True)
        rows = d_rec[:min(cap, res.n_records)].cpu().tolist()
        assert res.n_matched == cnt and [tuple(r[:3]) for r in rows] == head


def test_bestmatch_device():
    """-B: the reference answers -B -p -d ab; the sweep's best level and its records equal the checker's levels scan"""
    import torch
    data = strewn("ab", 100000, 5)
    kw = dict(ins_free=1, delim="ab")
    t = torch.frombuffer(bytearray(data + b"\0" * 64), dtype=torch.uint8).cuda()
    for pat in ("bexause eaxh", "govxrnmxnt"):
        cnt, hist, orecs = _oracle.scan_levels(_oracle.compile(pat, k=8, **kw), 8, data)
        want = next((l for l in range(9) if hist[l]), -1)
        cap = len(orecs) + 16
        d_rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
        best, res = ag.bestmatch_device(pat, t.data_ptr(), len(data), d_records=d_rec.data_ptr(), capacity=cap, sticky_delim=1, **kw)
        assert best == want and res.n_matched == (hist[want] if want >= 0 else 0), pat
        rows = d_rec[:res.n_records].cpu().tolist()
        assert [(b, e) for b, e, _j, _l in rows] == [(b, e) for b, e, _j, l in orecs if l == want], pat


def test_sharded_scans_refuse():
    import torch
    p = ag.Pattern("because", ins_free=True, delim="ab", sticky_delim=True)
    t = torch.zeros(8192, dtype=torch.uint8, device="cuda")
    res, part = _lib.Result(), _lib.ShardPart()
    rc = _lib.lib().agb_scan_shard_local(p._h, C.c_void_p(t.data_ptr()), 4096, 0, 0, 1, 1, 1, _lib.WANT_COUNT, None, 0, None,
                                         C.byref(res), C.byref(part))
    assert rc == -1 and b"sharded" in _lib.lib().agb_last_error()


# ---- the stand-alone command line and the drop-in against the reference ----
def run(binary, args, cwd):
    p = subprocess.run([binary] + args, capture_output=True, timeout=120, stdin=subprocess.DEVNULL, cwd=cwd)
    return p.returncode, p.stdout, p.stderr


# (every delimiter; the texts and patterns that exercise the printing most: each case starts six processes)
CLI_CASES = [c for c in CASES if c[1] in ("k0", "k2", "v", "hash") and c[2] in ("base", "starts", "open") and c not in NOT_RESTATED]


@pytest.mark.parametrize("dn,pn,tn", CLI_CASES, ids=[key(*c) for c in CLI_CASES])
def test_cli_and_dropin_print_what_the_reference_prints(dn, pn, tn, tmp_path):
    (tmp_path / "t.txt").write_bytes(case_text(dn, tn))
    g = GOLDEN[key(dn, pn, tn)]
    for name, extra in (("count", ["-c"]), ("plain", []), ("n", ["-n"])):
        args = argv(dn, pn, extra) + ["t.txt"]
        want = (g[name + "_rc"], (("%d\n" % g["count"]) if name == "count" else g[name]).encode("latin-1"))
        if os.path.exists(DROP):
            rc, out, err = run(DROP, ["-V0"] + args, str(tmp_path))
            assert (rc, out) == want and err.replace(DROP.encode(), b"agrep") == g[name + "_err"].encode("latin-1"), args
        if os.path.exists(REF):
            r = run(REF, args, str(tmp_path))
            c = run(CLI, args, str(tmp_path))
            assert (c[0], c[1], c[2].replace(b"agrep-b200", b"agrep")) == (r[0], r[1], r[2].replace(REF.encode(), b"agrep")), args
