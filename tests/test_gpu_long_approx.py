"""Simple literals of more than 63 positions at k = 1..8 on the device (agb_options.wide_approx): the record stage in 320-bit
rows at k + 1 rows (records_wide.cu).  Parity with the checker's 320-bit rows through every scan entry point, the levels
pass, both record forms, the wide form forced onto short literals against the 64-bit form bit for bit, and the drop-in and
the stand-alone command line against the checker and the reference."""
import os, random, subprocess
import pytest
import _oracle_wide, _corpus
import agrep_b200 as ag
from agrep_b200 import _lib
from golden.make_long_literal_golden import literal
from test_gpu_shard import scan_in_shards
from test_gpu_long_literal import every_entry, host_ordinals, summary, _forced, run, REF, DROP, CLI
from test_long_approx_host import approx_text

pytestmark = pytest.mark.gpu
BASE = _corpus.make_text(9000, seed=321)           # about 450 KB


def planted(m, k, sep=b"\n", final=False, seed=0):
    """the literal with 0..k+1 random edits (and once in upper case) across 32 KiB tile, 16 KiB stage, 512-byte word and
    16-byte chunk edges; at the very start of the text and at its end, unterminated unless final"""
    lit = literal(m, seed=k).encode()
    rnd = random.Random(1000 * m + 10 * k + seed)
    t = bytearray(BASE.replace(b"\n", sep))
    edges = [32768 * (1 + j) for j in range(8)] + [16384 * (17 + 2 * j) for j in range(4)] + [512 * (1061 + 2 * j) for j in range(4)]
    edges += [16 * (40001 + 3 * j) for j in range(4)]
    for i, edge in enumerate(edges):
        v = lit.upper() if i == 5 else _corpus.mutate(rnd, lit.decode(), i % (k + 2)).encode()
        at = edge - 1 - (1, m // 2, m - 1, 16)[i % 4]
        t[at:at + len(v) + 2] = b" " + v + b" "
    head = _corpus.mutate(rnd, lit.decode(), k).encode()
    tail = _corpus.mutate(rnd, lit.decode(), 1).encode()
    return lit, head + b" " + bytes(t) + b" " + tail + (sep if final else b"")


def checker(lit, data, k, kw):
    cnt, recs = _oracle_wide.scan(_oracle_wide.compile(lit, k=k, linenum=1, **kw), data)
    return cnt, [r[:2] for r in recs]


# (separator, Pattern keywords, final delimiter): each (m, k) runs two of them, so that every one meets every length and k
VARIANTS = [(b"\n", {}, True), (b"\n", {}, False), (b";", dict(delim=";"), True), (b";", dict(delim=";"), False),
            (b"@#", dict(delim="@#"), True), (b"@#", dict(delim="@#"), False), (b"\n\n", dict(delim="$$"), True)]       # ('$' is '\n' in -d)
CASES = [(m, k) + VARIANTS[v % len(VARIANTS)] + (v == i + j,)
         for i, m in enumerate((64, 100, 200, 255)) for j, k in enumerate((1, 2, 4, 8)) for v in (i + j, i + j + 3)]


@pytest.mark.parametrize("m,k,sep,kw,final,first", CASES,
                         ids=["m%d-k%d-%s-%s" % (c[0], c[1], c[2].decode().replace("\n", "nl"), "final" if c[4] else "open") for c in CASES])
def test_parity_with_the_checker(m, k, sep, kw, final, first, tmp_path):
    lit, data = planted(m, k, sep, final, seed=int(first))
    p = ag.Pattern(lit, k=k, wide_approx=True, **kw)
    assert p.desc.M > 63 and p.wide is not None and p.desc.nrows == k + 1
    cnt, recs = checker(lit, data, k, kw)
    assert cnt >= 8
    n, got = every_entry(p, data, tmp_path)
    assert n == cnt and [g[:2] for g in got] == recs
    assert [g[2] for g in got] == host_ordinals(p, data, got)
    if first:                                       # the one-GPU shard walk, once per (m, k)
        for world in (3, 7):
            matched, out, _ = scan_in_shards(lit, dict(kw, k=k, wide_approx=1), data, world)
            assert matched == cnt and out == got, world
    # -v: the complement, in the tile form
    pv = ag.Pattern(lit, k=k, wide_approx=True, inverse=True, **kw)
    cv, rv = _oracle_wide.scan(_oracle_wide.compile(lit, k=k, linenum=1, inverse=1, **kw), data)
    res, gv = pv.scan_host(data)
    assert res.n_matched == cv and [g[:2] for g in gv] == [r[:2] for r in rv]


@pytest.mark.parametrize("k", [4, 8])
@pytest.mark.parametrize("m", [64, 255])
def test_levels(m, k):
    lit, data = planted(m, k, final=True)
    p = ag.Pattern(lit, k=k, wide_approx=True)
    cnt, hist, recs = _oracle_wide.scan_levels(_oracle_wide.compile(lit, k=k, linenum=1), k, data)
    res, got = p.scan_host(data, levels=True)
    assert res.n_matched == cnt and list(res.level_hist) == hist
    assert [(b, e, lv) for b, e, _, lv in got] == [(b, e, lv) for b, e, _, lv in recs]
    assert len(set(lv for *_x, lv in recs)) > 2


def test_both_record_forms_run():
    """sparse flags go to the list form (few chunks handed over), dense ones and -v lists to the tile form (every chunk)"""
    import torch
    lit = literal(160, seed=2).encode()
    rnd = random.Random(4)
    sparse = bytearray(BASE.upper() * 6)             # (upper case: the literal's lower-case pieces occur only where planted)
    for at in range(1000, len(sparse) - 400, 20011):
        v = _corpus.mutate(rnd, lit.decode(), rnd.randint(0, 3)).encode()
        sparse[at:at + len(v)] = v
    sparse = bytes(sparse)
    n = len(sparse)
    p = ag.Pattern(lit, k=2, wide_approx=True)
    w = _oracle_wide.compile(lit, k=2, linenum=1)
    for data, is_sparse in ((sparse, True), ((lit[:40] + b"\n") * (n // 41), False)):
        chunks = (len(data) + 15) // 16
        before = _lib.lib().agb_kernel_launches()
        res, got = p.scan_host(data)
        cnt, recs = _oracle_wide.scan(w, data)
        assert res.n_matched == cnt and [g[:2] for g in got] == [r[:2] for r in recs]
        assert _lib.lib().agb_kernel_launches() > before
        assert (res.n_flagged < chunks // 20) if is_sparse else res.n_flagged == chunks, (is_sparse, res.n_flagged, chunks)
    pv = ag.Pattern(lit, k=2, wide_approx=True, inverse=True)
    wv = _oracle_wide.compile(lit, k=2, linenum=1, inverse=1)
    res, got = pv.scan_host(sparse)
    cnt, recs = _oracle_wide.scan(wv, sparse)
    assert res.n_matched == cnt and [g[:2] for g in got] == [r[:2] for r in recs] and res.n_flagged == (len(sparse) + 15) // 16
    # -c -v at a size where the 64-bit form takes the complement count
    big = sparse * 3
    t = torch.frombuffer(bytearray(big + b"\0" * 64), dtype=torch.uint8).cuda()
    assert pv.scan_device(t.data_ptr(), len(big)).n_matched == _oracle_wide.scan(wv, big, want_records=False)[0]


# ---- the wide form forced onto short literals: bit for bit the 64-bit form ----
SHORT = ["because each", "homogeneous approximate", "the", "x" * 40, literal(55)]


def _pair(monkeypatch, pat, kw):
    monkeypatch.delenv("AGB_FORCE_WIDE", raising=False)
    narrow = ag.Pattern(pat, wide_approx=True, **kw)
    monkeypatch.setenv("AGB_FORCE_WIDE", "1")
    wide = ag.Pattern(pat, wide_approx=True, **kw)
    monkeypatch.delenv("AGB_FORCE_WIDE")
    assert narrow.wide is None and wide.wide is not None and wide.desc.nrows == narrow.desc.nrows
    return narrow, wide


@pytest.mark.parametrize("k", range(1, 9))
def test_forced_wide_equals_the_64_bit_form(monkeypatch, k):
    import torch
    pat = SHORT[k % len(SHORT)]
    if len(pat) <= k:
        pat = SHORT[0]
    for kw in ({}, dict(inverse=1), dict(delim="$$"), dict(delim="aba"), dict(delim=";")):
        narrow, wide = _pair(monkeypatch, pat, dict(kw, k=k))
        data = _corpus.overlap_text("aba", 5) if kw.get("delim") == "aba" else _corpus.make_text(6000, seed=k, paragraphs=True)
        if kw.get("delim") == ";":                     # ("$$" is "\n\n": the paragraphs)
            data = data.replace(b"\n", b";")
        for opts in (dict(ordinals=True), dict(want_records=False), dict(levels=True), dict(window=4096, ordinals=True)):
            a, b = narrow.scan_host(data, **opts), wide.scan_host(data, **opts)
            assert summary(a[0]) == summary(b[0]) and a[1] == b[1] and list(a[0].level_hist) == list(b[0].level_hist), (kw, opts)
        big = data * ((2 << 20) // len(data)) + data[:1000]
        t = torch.frombuffer(bytearray(big + b"\0" * 64), dtype=torch.uint8).cuda()
        assert narrow.scan_device(t.data_ptr(), len(big)).n_matched == wide.scan_device(t.data_ptr(), len(big)).n_matched
        texts = [data, b"", data[:5000]]
        ta, tb = narrow.scan_set(texts, ordinals=True), wide.scan_set(texts, ordinals=True)
        assert summary(ta[0]) == summary(tb[0]) and ta[2] == tb[2] and [summary(r) for r in ta[1]] == [summary(r) for r in tb[1]]
        kk = dict(kw, k=k, wide_approx=1)
        assert scan_in_shards(pat, kk, data, 5) == _forced(monkeypatch, lambda: scan_in_shards(pat, kk, data, 5)), kw


def test_a_set_of_files():
    lit, data = planted(200, 3, final=True)
    p = ag.Pattern(lit, k=3, wide_approx=True)
    texts = [b"", BASE[:70000], data, data[:33333], data[-20000:]]
    total, per, recs = p.scan_set(texts, ordinals=True)
    at = 0
    for i, t in enumerate(texts):
        res, alone = p.scan_host(t, ordinals=True)
        cnt, want = checker(lit, t, 3, {})
        mine = [r[:3] for r in recs if r[4] == i]
        assert per[i].n_matched == res.n_matched == cnt and mine == [r[:3] for r in alone], i
        assert [r[:2] for r in mine] == want
        at += cnt
    assert total.n_matched == at and at > 8


# ---- the drop-in and the stand-alone command line ----
@pytest.fixture(scope="module")
def cli_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("agb_long_approx_")
    for m in (80, 160, 255):
        for k in (1, 3):
            lit = literal(m, seed=k)                # (under 48 KiB, with a final newline: SURVEY 8c(1), (2))
            (d / ("n%d_%d.txt" % (m, k))).write_bytes(approx_text(lit, k, nlines=200, seed=m + 1))
            (d / ("o%d_%d.txt" % (m, k))).write_bytes(approx_text(lit, k, nlines=150, seed=m + 2))
            (d / ("s%d_%d.txt" % (m, k))).write_bytes(approx_text(lit, k, b";", nlines=200, seed=m + 3))
    return str(d)


def _lines(out):
    """the printed records: stdout without the "Grand total: N match(es) found." summary of the reference's main() (whose
    exit code is the count)"""
    return [x for x in out.split(b"\n") if x and b"match(es) found" not in x]


@pytest.mark.parametrize("m", [80, 160, 255])
@pytest.mark.parametrize("k", [1, 3])
def test_dropin_and_cli(cli_files, m, k):
    lit = literal(m, seed=k)
    files = ["n%d_%d.txt" % (m, k), "o%d_%d.txt" % (m, k)]
    data = open(os.path.join(cli_files, files[0]), "rb").read()
    cnt, recs = checker(lit.encode(), data, k, {})
    assert cnt > 3
    have_dropin = os.path.exists(REF) and os.path.exists(DROP)
    for binary in [CLI] + ([DROP] if have_dropin else []):
        _, out, _ = run(binary, ["-%d" % k, "-c", lit, files[0]], cli_files)
        assert out.split(b"\n")[0] == b"%d" % cnt, binary
        _, out, _ = run(binary, ["-%d" % k, lit, files[0]], cli_files)
        assert _lines(out) == [data[b + 1:e] for b, e in recs], binary
    if not have_dropin:
        pytest.skip("oracle/_ref binaries not built")
    for args, fs in (([], files[:1]), (["-c"], files[:1]), (["-l"], files), (["-h"], files), (["-d", ";"], ["s%d_%d.txt" % (m, k)])):
        argv = ["-%d" % k] + args + [lit] + fs
        d = run(DROP, argv, cli_files)
        c = run(CLI, argv, cli_files)
        assert d[:2] == c[:2], argv
        if args in ([], ["-h"]):
            r = run(REF, ["-V0"] + argv, cli_files)
            assert set(_lines(r[1])) <= set(_lines(d[1])), argv          # (the reference's exit code is its count)
