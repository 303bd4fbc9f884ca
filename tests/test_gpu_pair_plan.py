"""The pair plan on the device (stage 1 flags a chunk only where two different pieces of the pattern meet; DESIGN.md 3.1),
forced on and forced off with AGB_PLAN_PAIRS: both give the checker's counts, records, levels and ordinals.  The planner
only re-plans texts of 256 MiB and more that are scanned in device memory (scan_device, the shard-local scan, and each
window of 256 MiB or more of a windowed host scan; the whole-text host scan is not planned), so the texts here are that
large; planted matches with 0..k edits put their two surviving pieces across a chunk boundary, a warp's last chunk
(2 KiB), a 16 KiB stage boundary and the end of the text.  tests/test_gpu_plans_large.py covers the other pair plans."""
import ctypes as C
import os, random
import pytest
import _oracle
import agrep_b200 as ag
from agrep_b200 import _lib

pytestmark = pytest.mark.gpu
MIB = 1 << 20
PATTERN, K = "because each", 2
N = 288 * MIB


def plant(buf, at, line):
    """a record `line` whose bytes start at offset `at` (a newline before and after it)"""
    buf[at - 1] = 10
    buf[at:at + len(line)] = line
    buf[at + len(line)] = 10


def damaged(k, keep, nocase_rnd=None):
    """'because each' with k substitutions that leave only the pieces in `keep` (of bec|aus|e e|ach) verbatim"""
    s = bytearray(b"because each")
    for i in (0, 3, 6, 9):
        if i not in keep and k > 0:
            s[i + 1] = ord("#")
            k -= 1
    if nocase_rnd:
        s = bytearray(c ^ 0x20 if 97 <= c <= 122 and nocase_rnd.random() < 0.5 else c for c in s)
    return bytes(s)


@pytest.fixture(scope="module")
def text():
    buf = bytearray(ag.corpus_host(N, seed=31, needle=PATTERN, needle_every=512, needle_maxedits=3))
    rnd = random.Random(5)
    sites = []
    for base in (1 << 20, 64 << 20, 200 << 20):
        for boundary in (16, 2048, 16384):
            for lead in (1, 2, 3, 5, 8):                  # the first surviving piece starts `lead` bytes before the boundary
                sites.append(base + 65536 * len(sites) + 3 * boundary - lead)
    for i, at in enumerate(sites):
        keep = [(0, 3), (3, 6), (6, 9), (0, 9), (3, 9)][i % 5]
        line = damaged(K, keep, rnd if i % 7 == 0 else None)
        plant(buf, at - keep[0], line)
    plant(buf, N - 14, damaged(K, (3, 6)))               # the last record of the text
    return bytes(buf)


@pytest.fixture(scope="module")
def dev(text):
    import torch
    return torch.frombuffer(bytearray(text + b"\0" * 4096), dtype=torch.uint8).cuda()


@pytest.fixture
def pairs(monkeypatch):
    def set_(v):
        monkeypatch.setenv("AGB_PLAN_PAIRS", str(v))
    return set_


def device_scan(pat, t, n, levels=False):
    import torch
    cap = 1 << 20
    rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
    res = pat.scan_device(t.data_ptr(), n, d_records=rec.data_ptr(), capacity=cap, ordinals=True, levels=levels)
    assert not res.truncated
    return res, [tuple(r) for r in rec[:res.n_records].cpu().tolist()]


@pytest.mark.parametrize("nocase", [False, True])
def test_forced_on_and_off_match_the_checker(text, dev, pairs, capfd, nocase):
    a = _oracle.compile(PATTERN, k=K, nocase=int(nocase), linenum=1)
    cnt, hist, expect = _oracle.scan_levels(a, K, text, cap=1 << 20)
    assert cnt > 1000
    pat = ag.Pattern(PATTERN, k=K, nocase=nocase)
    got = {}
    for v in (0, 1):
        pairs(v)
        os.environ["AGB_DEBUG_PLAN"] = "1"
        try:
            res, recs = device_scan(pat, dev, N, levels=True)
        finally:
            del os.environ["AGB_DEBUG_PLAN"]
        err = capfd.readouterr().err
        assert ("pair plan chosen" in err) == (v == 1), err
        assert res.n_matched == cnt
        assert list(res.level_hist)[:K + 1] == hist[:K + 1]
        assert [(b, e, j, lv) for b, e, j, lv in recs] == expect
        got[v] = res
    assert got[1].n_flagged <= got[0].n_flagged


def test_count_and_host_entry_points(text, dev, pairs):
    """the count-only device scan and the windowed host scan (its first window, 256 MiB plus halos, is planned) under
    both settings; the whole-text host scan is not planned, so there both settings run the static plan"""
    pat = ag.Pattern(PATTERN, k=K)
    cnt, expect = _oracle.scan(_oracle.compile(PATTERN, k=K, linenum=1), text, cap=1 << 20)
    for v in (0, 1):
        pairs(v)
        assert pat.scan_device(dev.data_ptr(), N).n_matched == cnt
        res, recs = pat.scan_host(text, ordinals=True)
        assert res.n_matched == cnt and [r[:3] for r in recs] == expect
        res, recs = pat.scan_host(text, ordinals=True, window=256 * MIB)
        assert res.n_matched == cnt and [r[:3] for r in recs] == expect


def test_shard_local_whole_text(text, dev, pairs):
    import torch
    L = _lib.lib()
    p = ag.Pattern(PATTERN, k=K)
    cnt, expect = _oracle.scan(_oracle.compile(PATTERN, k=K, linenum=1), text, cap=1 << 20)
    for v in (0, 1):
        pairs(v)
        cap = 1 << 20
        rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
        res, part = _lib.Result(), _lib.ShardPart()
        rc = L.agb_scan_shard_local(p._h, C.c_void_p(dev.data_ptr()), N, 0, 0, 1, 1, 1, _lib.WANT_RECORDS | _lib.WANT_ORDINALS,
                                    C.c_void_p(rec.data_ptr()), cap, None, C.byref(res), C.byref(part))
        assert rc == 0, L.agb_last_error()
        assert res.n_matched == cnt
        got = [(b + part.byte_base, e + part.byte_base, j + part.ord_origin - part.ord_fix) for b, e, j, _ in rec[:res.n_records].cpu().tolist()]
        assert got == expect


def test_1gib_corpus_on_equals_off(pairs):
    import torch
    n = 1 << 30
    t = torch.empty(n + 4096, dtype=torch.uint8, device="cuda")
    t[n:].zero_()
    ag.corpus_device(t.data_ptr(), n, seed=0, needle=PATTERN, needle_every=4096, needle_maxedits=3)
    torch.cuda.synchronize()
    pat = ag.Pattern(PATTERN, k=K)
    out = {}
    for v in (0, 1):
        pairs(v)
        out[v] = device_scan(pat, t, n)
    assert out[0][0].n_matched == out[1][0].n_matched > 0
    assert out[0][1] == out[1][1]
    assert out[0][0].n_closes == out[1][0].n_closes
