"""Simple literals of more than 63 positions at k = 0 on the device: the record stage in 320-bit rows (records_wide.cu).
Parity with the checker through every scan entry point; the wide form forced onto short literals (AGB_FORCE_WIDE=1) equals
the 64-bit form bit for bit, also where the checker does not restate the semantics (-v lists, -c -v, $$, aba, sets); the
drop-in and the stand-alone command line print what the reference prints."""
import ctypes as C
import os, subprocess
import pytest
import _oracle, _corpus
import agrep_b200 as ag
from agrep_b200 import _lib
from golden.make_long_literal_golden import literal
from test_gpu_shard import scan_in_shards

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "agrep")
DROP = os.path.join(ROOT, "oracle", "_ref", "agrep_dropin")
CLI = os.path.join(ROOT, "agrep_b200", "agrep-b200")
BASE = _corpus.make_text(9000, seed=321)           # about 450 KB


def planted(m, sep=b"\n", final=False):
    """the literal planted exactly, in upper case, and with one byte changed at its start, middle or end, across 32 KiB tile,
    16 KiB stage, 512-byte word and 16-byte chunk boundaries; at the very start of the text and at its unterminated end"""
    lit = literal(m).encode()
    t = bytearray(BASE.replace(b"\n", sep))
    bad = [b"#" + lit[1:], lit[:m // 2] + b"#" + lit[m // 2 + 1:], lit[:-1] + b"#"]
    edges = [32768 * (1 + j) for j in range(8)] + [16384 * (17 + 2 * j) for j in range(4)] + [512 * (1061 + 2 * j) for j in range(4)]
    for i, edge in enumerate(edges):
        v = b" " + (lit, lit.upper(), bad[i % 3], lit)[i % 4] + b" "       # (spaces: words under -w)
        at = edge - 1 - (1, m // 2, m - 1, 16)[i % 4]
        t[at:at + len(v)] = v
    t[0:m + 1] = lit + b" "
    return lit, bytes(t) + b" " + lit + (sep if final else b"")


def checker(lit, data, kw):
    cnt, recs = _oracle.scan(_oracle.compile(lit, **kw), data)
    return cnt, [r[:2] for r in recs]


def host_ordinals(p, data, recs):
    """j of each record from the library's host walk (agb_fill_ordinals), against the device's ordinals pass"""
    arr = (_lib.Record * max(1, len(recs)))()
    for i, (b, e, *_r) in enumerate(recs):
        arr[i].begin, arr[i].end = b, e
    buf = (C.c_char * len(data)).from_buffer_copy(data)
    _lib.lib().agb_fill_ordinals(p._h, buf, len(data), arr, len(recs))
    return [arr[i].ordinal for i in range(len(recs))]


def every_entry(p, data, tmp_path):
    """(count, ordered list with ordinals) through the device, host, fd, resident-text and windowed entries: all equal"""
    import torch
    res, recs = p.scan_host(data, ordinals=True)
    got = [(b, e, j) for b, e, j, _ in recs]
    assert p.scan_host(data, want_records=False)[0].n_matched == res.n_matched
    for window in (4096, 65536):
        r2, rec2 = p.scan_host(data, ordinals=True, window=window)
        assert (r2.n_matched, [(b, e, j) for b, e, j, _ in rec2]) == (res.n_matched, got), window
    f = tmp_path / "t.txt"
    f.write_bytes(data)
    with open(f, "rb") as fh:
        r3, rec3 = p.scan_fd(fh.fileno(), ordinals=True)
    assert (r3.n_matched, [(b, e, j) for b, e, j, _ in rec3]) == (res.n_matched, got)
    with open(f, "rb") as fh:
        r4, rec4 = p.scan_fd(fh.fileno(), ordinals=True, window=4096)
    assert (r4.n_matched, [(b, e, j) for b, e, j, _ in rec4]) == (res.n_matched, got)
    t = torch.frombuffer(bytearray(data + b"\0" * 64), dtype=torch.uint8).cuda()
    cap = res.n_matched + 16
    d_rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
    r5 = p.scan_device(t.data_ptr(), len(data), d_records=d_rec.data_ptr(), capacity=cap, ordinals=True)
    rows = d_rec[:r5.n_records].cpu().tolist()
    assert (r5.n_matched, [(b, e, j) for b, e, j, _ in rows]) == (res.n_matched, got)
    assert p.scan_device(t.data_ptr(), len(data)).n_matched == res.n_matched
    htxt = C.c_void_p()
    buf = (C.c_char * len(data)).from_buffer_copy(data)
    assert _lib.lib().agb_text_from_host(buf, len(data), C.byref(htxt)) == 0
    try:
        arr, r6 = (_lib.Record * cap)(), _lib.Result()
        assert _lib.lib().agb_scan_text(p._h, htxt, _lib.WANT_RECORDS | _lib.WANT_ORDINALS, arr, cap, C.byref(r6)) == 0
        assert (r6.n_matched, [(arr[i].begin, arr[i].end, arr[i].ordinal) for i in range(r6.n_records)]) == (res.n_matched, got)
    finally:
        _lib.lib().agb_text_free(htxt)
    return res.n_matched, got


@pytest.mark.parametrize("m", [62, 63, 64, 100, 200, 255])
@pytest.mark.parametrize("kw,sep", [({}, b"\n"), (dict(wordbound=1), b"\n"), (dict(nocase=1), b"\n"), (dict(delim=";"), b";"),
                                    (dict(delim="@#"), b"@#")])
@pytest.mark.parametrize("final", [False, True])
def test_parity_with_the_checker(m, kw, sep, final, tmp_path):
    lit, data = planted(m, sep, final)
    p = ag.Pattern(lit, **kw)
    assert p.desc.M > 63 and p.wide is not None
    cnt, recs = checker(lit, data, kw)
    assert cnt >= 8
    n, got = every_entry(p, data, tmp_path)
    assert n == cnt and [g[:2] for g in got] == recs
    assert [g[2] for g in got] == host_ordinals(p, data, got)
    # the one-GPU shard walk: 512-byte cuts, several of them inside an occurrence
    for world in (3, 7):
        matched, out, _ = scan_in_shards(lit, kw, data, world)
        assert matched == cnt and out == got, world


def test_a_set_of_files():
    lit, data = planted(200)
    p = ag.Pattern(lit)
    texts = [b"", BASE[:70000], data, data[:33333], data[-20000:]]
    total, per, recs = p.scan_set(texts, ordinals=True)
    at = 0
    for i, t in enumerate(texts):
        res, alone = p.scan_host(t, ordinals=True)
        mine = [r[:3] for r in recs if r[4] == i]
        assert per[i].n_matched == res.n_matched and mine == [r[:3] for r in alone], i
        at += res.n_matched
    assert total.n_matched == at and at > 8


# ---- the wide form forced onto short literals: bit for bit the 64-bit form ----
SHORT = [("because each", {}), ("the", {}), ("homogeneous approximate matching", dict(wordbound=1)),
         ("government", dict(nocase=1)), ("the", dict(inverse=1)), ("and the", dict(delim="$$")),
         ("was", dict(delim="aba")), ("x" * 40, dict(delim=";")), ("because", dict(inverse=1, delim="$$"))]


def text_for(kw):
    if kw.get("delim") == "aba":
        return _corpus.overlap_text("aba", 5)
    if kw.get("delim") == ";":
        return BASE.replace(b"\n", b";") + b"x" * 40 + b";" + b"X" * 40
    return _corpus.make_text(9000, seed=5, paragraphs=True)


def both_forms(monkeypatch, pat, kw):
    monkeypatch.delenv("AGB_FORCE_WIDE", raising=False)
    narrow = ag.Pattern(pat, **kw)
    monkeypatch.setenv("AGB_FORCE_WIDE", "1")
    wide = ag.Pattern(pat, **kw)
    monkeypatch.delenv("AGB_FORCE_WIDE")
    assert narrow.wide is None and wide.wide is not None and wide.desc.M == narrow.desc.M
    return narrow, wide


def summary(res):
    return res.n_matched, res.n_records, res.n_closes, res.truncated


@pytest.mark.parametrize("pat,kw", SHORT)
def test_forced_wide_equals_the_64_bit_form(monkeypatch, pat, kw, tmp_path):
    import torch
    narrow, wide = both_forms(monkeypatch, pat, kw)
    data = text_for(kw)
    for opts in (dict(ordinals=True), dict(), dict(want_records=False), dict(window=4096, ordinals=True), dict(window=65536)):
        a, b = narrow.scan_host(data, **opts), wide.scan_host(data, **opts)
        assert summary(a[0]) == summary(b[0]) and a[1] == b[1], opts
    # the device entry at a size where -c -v takes the complement count, and a text with a planted record list
    big = data * ((2 << 20) // len(data)) + data[:1000]
    t = torch.frombuffer(bytearray(big + b"\0" * 64), dtype=torch.uint8).cuda()
    assert narrow.scan_device(t.data_ptr(), len(big)).n_matched == wide.scan_device(t.data_ptr(), len(big)).n_matched
    ta, tb = narrow.scan_set([data, b"", data[:5000]], ordinals=True), wide.scan_set([data, b"", data[:5000]], ordinals=True)
    assert summary(ta[0]) == summary(tb[0]) and ta[2] == tb[2] and [summary(r) for r in ta[1]] == [summary(r) for r in tb[1]]
    assert scan_in_shards(pat, kw, data, 5) == _forced(monkeypatch, lambda: scan_in_shards(pat, kw, data, 5))


def _forced(monkeypatch, fn):
    monkeypatch.setenv("AGB_FORCE_WIDE", "1")
    try:
        return fn()
    finally:
        monkeypatch.delenv("AGB_FORCE_WIDE")


# ---- the drop-in and the stand-alone command line against the reference ----
def run(binary, args, cwd):
    p = subprocess.run([binary] + args, capture_output=True, timeout=120, stdin=subprocess.DEVNULL, cwd=cwd)
    return p.returncode, p.stdout, p.stderr


@pytest.fixture(scope="module")
def cli_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("agb_long_")
    for m in (80, 160, 255):
        lit, data = planted(m)
        (d / ("n%d.txt" % m)).write_bytes(data[:40000] + b"\n" + lit.upper() + b" end\n")      # (under 48 KiB: -b is exact, SURVEY 8c(1))
        (d / ("o%d.txt" % m)).write_bytes(data[-30000:-m - 1] + b"xy " + lit + b" end\n")
        (d / ("s%d.txt" % m)).write_bytes(data[:40000].replace(b"\n", b";") + b";" + lit + b" end")
    return str(d)


# (not compared: -b and an unterminated last record, where monkey() -- every literal of more than 20 characters -- prints
# otherwise than the bm() output the drop-in restates; and -t in the stand-alone command line)
CLI_ARGS = [[], ["-c"], ["-l"], ["-i"], ["-w"], ["-h", "+2"], ["+2"], ["-d", ";", "+s"], ["-t", "-d", ";", "+s"]]


@pytest.mark.parametrize("m", [80, 160, 255])
@pytest.mark.parametrize("args", CLI_ARGS, ids=lambda a: " ".join(a) or "plain")
def test_dropin_and_cli_print_what_the_reference_prints(cli_files, m, args):
    if not (os.path.exists(REF) and os.path.exists(DROP)):
        pytest.skip("oracle/_ref binaries not built")
    opts = [a for a in args if not a.startswith("+")]
    files = ["s%d.txt" % m] if "+s" in args else (["n%d.txt" % m, "o%d.txt" % m] if "+2" in args else ["n%d.txt" % m])
    argv = opts + [literal(m)] + files
    r = run(REF, ["-V0"] + argv, cli_files)
    d = run(DROP, ["-V0"] + argv, cli_files)
    assert (d[0], d[1], d[2].replace(b"agrep_dropin", b"agrep")) == r, argv
    if os.path.exists(CLI) and "-t" not in args:
        r = run(REF, argv, cli_files)
        c = run(CLI, argv, cli_files)
        assert (c[0], c[1], c[2].replace(b"agrep-b200", b"agrep")) == r, argv
