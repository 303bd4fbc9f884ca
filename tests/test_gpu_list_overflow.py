"""The record stage's second attempt.  After stage 1.5 the list form sizes its candidate list from what earlier scans on the
device needed (Workspace.cand_hint), without asking the device; on a fresh workspace that is 1 Mi + 1/4 = 1 310 720
entries.  When the read-back shows more survivors than that, stages_after_front() runs the record stage and the
ordinals a second time: as a list of the right size when the survivors are at most 5 % of the chunks ("list again"),
over every byte otherwise ("dense").  Every entry point that scans a text goes through that loop.

Each case here starts from a fresh workspace (agb_shutdown), so its first scan ("cold") overflows the list, then scans
again ("warm", sized by the first scan's count, one attempt).  The cold scan must launch more kernels than the warm one,
the warm scan's survivor count proves the cold list was too small, and both must give the checker's answer: count, level
histogram, truncation, the ordered (begin, end, ordinal, level) list and the delimiter total.  The texts are corpus lines
with a phrase planted at 0..k+1 edits in most of them (some planted lines must not match), plus plants across 1 MiB and
64 MiB edges: a 64 MiB text dense enough for the every-byte form, a 768 MiB text whose survivors land inside the
list-again band (for the patterns whose survivors stay inside it), and the dense text behind 64 MiB of sparse text for the
windowed and the sharded scans, whose last window or shard alone overflows.  Each text also comes without its final
newline."""
import ctypes as C
import hashlib
import os
import random
import subprocess
from concurrent.futures import ThreadPoolExecutor
import numpy as np
import pytest
import _corpus, _oracle
import agrep_b200 as ag
from agrep_b200 import _lib, shard

MIB = 1 << 20
COLD_CAP = (1 << 20) + (1 << 18)          # ws_cand_reserve() on a fresh workspace: max(1 Mi, ...) plus a quarter
LONG = "homogeneous because each algorithm"   # 34 positions: 64-bit automaton rows
PATTERNS = {                                # name: (pattern, options, delimiter bytes)
    "nl-k1": ("because each", dict(k=1, linenum=1), b"\n"),
    "dd-k1": ("because each", dict(k=1, linenum=1, delim="$$"), b"\n\n"),   # L = 2: k_delim_count, not stage 1's counts
    "nocase-k1": ("Because Each", dict(k=1, linenum=1, nocase=1), b"\n"),
    "costs": ("because each", dict(k=2, linenum=1, cost_i=2, cost_s=1, cost_d=3), b"\n"),
    "rows64-k3": (LONG, dict(k=3, linenum=1), b"\n"),
}
WANTS = ("count", "records", "ordinals", "levels", "truncated")
REC_DT = np.dtype([("b", "<i8"), ("e", "<i8"), ("j", "<i8"), ("lev", "<i4"), ("pad", "<i4")])   # agb_record, orc_record
ORC_CAP = 4 << 20


# ---- texts ---------------------------------------------------------------------------------------------------------

def planted(rnd):
    """the long phrase with 0..4 edits, 0..2 of them inside "because each" (a k=1 pattern misses about one in twelve)"""
    b = rnd.choices((0, 1, 2), (0.8, 0.12, 0.08))[0]
    out = rnd.choices((0, 1, 2, 3), (0.45, 0.3, 0.15, 0.1))[0]
    a = rnd.randint(0, out)
    return (_corpus.mutate(rnd, "homogeneous ", a) + _corpus.mutate(rnd, "because each", b) +
            _corpus.mutate(rnd, " algorithm", out - a))


def build_text(n, p_plant, p_plain, seed):
    """n bytes of lines: a planted phrase (probability p_plant), a corpus line (p_plain) or an empty line (the rest, so
    that "$$" has paragraphs); then plants across every 1 MiB edge, 1..11 bytes of the needle before it; a final newline"""
    rnd = random.Random(seed)
    pool = [(planted(rnd) + "\n").encode() for _ in range(4096)]
    pool += [l + b"\n" for l in _corpus.make_text(4096, seed=seed).split(b"\n")[:4096]]
    pool.append(b"\n")
    avg = p_plant * np.mean([len(l) for l in pool[:4096]]) + p_plain * np.mean([len(l) for l in pool[4096:8192]]) + 1 - p_plant - p_plain
    rng = np.random.default_rng(seed)
    lines = int(n / avg * 1.05) + 1024
    cls = rng.choice(3, size=lines, p=(p_plant, p_plain, 1 - p_plant - p_plain))
    idx = np.where(cls == 2, 8192, cls * 4096 + rng.integers(0, 4096, size=lines))
    t = bytearray(b"".join(map(pool.__getitem__, idx.tolist())))
    assert len(t) >= n, len(t)
    del t[n:]
    for i, s in enumerate(range(MIB, n - 64, MIB)):
        at = s - 1 - i % 11
        t[at - 1:at + 13] = b"\nbecause each\n"
    t[-2:] = b"h\n"
    return t


@pytest.fixture(scope="module")
def texts():
    dense = build_text(64 * MIB, 0.85, 0.03, seed=101)
    out = {"dense": dense, "list": build_text(768 * MIB, 0.107, 0.76, seed=102),
           "split": build_text(64 * MIB, 0.02, 0.85, seed=103) + dense}
    for name in list(out):
        out[name + "-nonl"] = out[name][:-1]
    return {k: bytes(v) for k, v in out.items()}


@pytest.fixture(scope="module")
def devs(texts):
    import torch
    return {k: torch.frombuffer(bytearray(t + b"\0" * 4096), dtype=torch.uint8).cuda() for k, t in texts.items()}


# ---- the checker ---------------------------------------------------------------------------------------------------

def closes(text, delim):
    """shard.count_closes(text, delim) for "\\n" and "\\n\\n", at numpy speed (test_closes_is_count_closes)"""
    if delim == b"\n":
        return text.count(b"\n") + 2                         # the delimiter appended at EOF and the virtual '\n'
    assert delim == b"\n\n"
    nl = np.frombuffer(text + delim, dtype=np.uint8) == 10
    edges = np.flatnonzero(np.diff(np.concatenate(([0], nl.astype(np.int8), [0]))))
    runs = edges[1::2] - edges[0::2]
    if nl[0]:
        runs[0] += 1                                         # a run at the start pairs with the virtual '\n'
    return int((runs // 2).sum())


def test_closes_is_count_closes():
    rnd = random.Random(7)
    for _ in range(200):
        t = bytes(rnd.choice(b"ab\n") for _ in range(rnd.randint(0, 40)))
        for d in (b"\n", b"\n\n"):
            assert closes(t, d) == shard.count_closes(t, d), (t, d)


def oracle_kw(kw):
    return {k: (v if k == "delim" else int(v)) for k, v in kw.items()}


def oracle_answer(pattern, kw, text):
    """(count, level histogram or None, records as an (n, 4) array of begin, end, ordinal, level): levels where the
    checker has them (not for cost patterns)"""
    L = _oracle.lib()
    a = _oracle.compile(pattern, **oracle_kw(kw))
    recs = (_oracle.Record * ORC_CAP)()
    hist = (C.c_uint64 * 9)()
    cnt = L.orc_scan_levels(C.byref(a), kw["k"], text, len(text), hist, recs, ORC_CAP, -1)
    if cnt < 0:
        hist = None
        cnt = L.orc_scan(C.byref(a), text, len(text), recs, ORC_CAP)
    assert 0 <= cnt < ORC_CAP
    arr = np.frombuffer(recs, dtype=REC_DT, count=cnt)
    return cnt, (list(hist) if hist is not None else None), rows(arr)


def rows(arr):
    return np.stack([arr["b"], arr["e"], arr["j"], arr["lev"].astype(np.int64)], axis=1) if len(arr) else np.zeros((0, 4), np.int64)


LIST_PATTERNS = ("nl-k1", "dd-k1", "nocase-k1")   # costs and rows64-k3 keep 2.6-4.4 M survivors there: past the band
JOBS = [(p, "dense") for p in PATTERNS] + [(p, "list") for p in LIST_PATTERNS] + \
       [(p, t) for p in ("nl-k1", "dd-k1") for t in ("dense-nonl", "list-nonl", "split", "split-nonl")] + \
       [("-v", k, t) for k in (0, 1) for t in ("dense", "list")] + [("-B", "dense")]


@pytest.fixture(scope="module")
def answers(texts):
    """the checker's answers, once, in a thread pool (ctypes releases the GIL): (name, text) for PATTERNS, ("-v", k,
    text) for the -c -v counts, ("-B", text) for the levels of the -B sweep's first pass"""
    def one(job):
        if job[0] == "-v":          # (linenum=1: the automaton, as the device runs it; the checker does not restate sgrep's -v)
            return _oracle.scan(_oracle.compile("because each", k=job[1], inverse=1, linenum=1), texts[job[2]], want_records=False)[0]
        if job[0] == "-B":
            return oracle_answer("because each", dict(k=2, linenum=1), texts[job[1]])
        pattern, kw, _ = PATTERNS[job[0]]
        return oracle_answer(pattern, kw, texts[job[1]])
    with ThreadPoolExecutor(max_workers=max(1, min(len(JOBS), os.cpu_count() or 1))) as ex:
        return dict(zip(JOBS, ex.map(one, JOBS)))


# ---- scans ---------------------------------------------------------------------------------------------------------

def want_of(mode):
    return {"count": _lib.WANT_COUNT, "records": _lib.WANT_RECORDS, "ordinals": _lib.WANT_RECORDS | _lib.WANT_ORDINALS,
            "levels": _lib.WANT_RECORDS | _lib.WANT_ORDINALS | _lib.WANT_LEVELS,
            "truncated": _lib.WANT_RECORDS | _lib.WANT_ORDINALS}[mode]


def cold_then_warm(scan):
    """scan() on a fresh workspace, then again: [(kernel launches, result, records) cold, (...) warm]"""
    L = _lib.lib()
    L.agb_shutdown()
    out = []
    for _ in range(2):
        before = L.agb_kernel_launches()
        res, recs = scan()
        out.append((L.agb_kernel_launches() - before, res, recs))
    return out


def device_scan(pat, dev, n, want, cap):
    import torch
    rec = torch.zeros((max(cap, 1), 4), dtype=torch.int64, device="cuda")
    res = _lib.Result()
    rc = _lib.lib().agb_scan_device(pat._h, C.c_void_p(dev.data_ptr()), n, want, C.c_void_p(rec.data_ptr()), cap, None,
                                    C.byref(res))
    assert rc == 0, _lib.lib().agb_last_error()
    return res, rec[:res.n_records].cpu().numpy()


def host_call(fn, cap):
    """fn(records, result) is a host entry point's call"""
    recs = (_lib.Record * max(cap, 1))()
    res = _lib.Result()
    assert fn(recs, C.byref(res)) == 0, _lib.lib().agb_last_error()
    return res, rows(np.frombuffer(recs, dtype=REC_DT, count=res.n_records))


def cap_of(mode, cnt):
    return 0 if mode == "count" else (cnt // 2 if mode == "truncated" else cnt + 16)


def check(res, recs, answer, mode, delim, text):
    cnt, hist, expect = answer
    assert res.n_matched == cnt
    cap = cap_of(mode, cnt)
    assert res.truncated == (1 if mode == "truncated" else 0)
    assert res.n_records == min(cnt, cap)
    cols = {"count": 0, "records": 2, "ordinals": 3, "levels": 4, "truncated": 3}[mode]
    if cols:
        assert np.array_equal(recs[:, :cols], expect[:res.n_records, :cols])
    if mode == "levels":
        assert list(res.level_hist) == hist
    if mode in ("ordinals", "levels", "truncated"):
        assert res.n_closes == closes(text, delim)


def overflowed(runs, n, band):
    """the cold scan retried: more launches than the warm one, whose survivor count the cold list could not hold (and,
    for the list-again texts, at most 5 % of the chunks, so the retry was a list)"""
    (lc, rc_, _), (lw, rw, _) = runs
    print("cold %d launches, warm %d launches, survivors %d" % (lc, lw, rw.n_flagged))
    assert lc > lw, (lc, lw)
    assert rw.n_flagged > COLD_CAP, rw.n_flagged
    n_chunks = (n + 15) // 16
    if band == "list":
        assert rw.n_flagged <= n_chunks // 20 + 1024, "survivors %d: the text recipe misses the list-again band" % rw.n_flagged
    else:
        assert rw.n_flagged > n_chunks // 20 + 1024, rw.n_flagged


def band_of(text):
    return "list" if text.startswith("list") else "dense"


def same(runs, answer, mode, delim, text):
    for _, res, recs in runs:
        check(res, recs, answer, mode, delim, text)
    (_, r0, a0), (_, r1, a1) = runs
    assert (r0.n_matched, list(r0.level_hist), r0.n_closes, r0.n_records) == (r1.n_matched, list(r1.level_hist), r1.n_closes, r1.n_records)
    assert np.array_equal(a0, a1)


# ---- scan_device: every pattern, every output ---------------------------------------------------------------------

MATRIX = [(p, t, m) for t in ("dense", "list") for p in (PATTERNS if t == "dense" else LIST_PATTERNS) for m in WANTS
          if not (m == "levels" and p == "costs")] + \
         [(p, t, "ordinals") for p in ("nl-k1", "dd-k1") for t in ("dense-nonl", "list-nonl")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,text,mode", MATRIX)
def test_scan_device_overflow(name, text, mode, texts, devs, answers):
    pattern, kw, delim = PATTERNS[name]
    pat = ag.Pattern(pattern, **kw)
    answer = answers[(name, text)]
    n = len(texts[text])
    cap = cap_of(mode, answer[0])
    runs = cold_then_warm(lambda: device_scan(pat, devs[text], n, want_of(mode), cap))
    overflowed(runs, n, band_of(text))
    same(runs, answer, mode, delim, texts[text])


# ---- the host entry points -----------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("text", ["dense", "list", "dense-nonl", "list-nonl"])
@pytest.mark.parametrize("name", ["nl-k1", "dd-k1"])
def test_host_and_resident_text_overflow(name, text, texts, answers):
    """agb_scan_host (the whole text, stage 1 slice by slice) and agb_scan_text over a resident copy"""
    L = _lib.lib()
    pattern, kw, delim = PATTERNS[name]
    pat = ag.Pattern(pattern, **kw)
    data = texts[text]
    answer = answers[(name, text)]
    want, cap = want_of("levels"), answer[0] + 16
    runs = cold_then_warm(lambda: host_call(lambda r, s: L.agb_scan_host(pat._h, data, len(data), want, r, cap, s), cap))
    overflowed(runs, len(data), band_of(text))
    same(runs, answer, "levels", delim, data)

    L.agb_shutdown()
    t = C.c_void_p()
    assert L.agb_text_from_host(data, len(data), C.byref(t)) == 0, L.agb_last_error()
    try:
        runs = []
        for _ in range(2):
            before = L.agb_kernel_launches()
            res, recs = host_call(lambda r, s: L.agb_scan_text(pat._h, t, want, r, cap, s), cap)
            runs.append((L.agb_kernel_launches() - before, res, recs))
    finally:
        L.agb_text_free(t)
    overflowed(runs, len(data), band_of(text))
    same(runs, answer, "levels", delim, data)


@pytest.mark.gpu
@pytest.mark.parametrize("text", ["split", "split-nonl"])
@pytest.mark.parametrize("name", ["nl-k1", "dd-k1"])
def test_windowed_scan_last_window_overflows(name, text, texts, answers):
    """64 MiB windows over 64 MiB of sparse text and the dense text: the first window fits the list, the last overflows"""
    L = _lib.lib()
    pattern, kw, delim = PATTERNS[name]
    pat = ag.Pattern(pattern, **kw)
    data = texts[text]
    answer = answers[(name, text)]
    want, cap = want_of("levels"), answer[0] + 16
    runs = cold_then_warm(lambda: host_call(
        lambda r, s: L.agb_scan_host_windowed(pat._h, data, len(data), 64 * MIB, want, r, cap, s), cap))
    overflowed(runs, 64 * MIB, "dense")
    same(runs, answer, "levels", delim, data)


def shard_walk(pat, data, world, cap):
    """agb_scan_shard_local over each shard in turn, stitched as the gather does (tests/test_gpu_shard.py)"""
    import torch
    L = _lib.lib()
    n = len(data)
    per = (n // world) // 512 * 512
    offs = [r * per for r in range(world)] + [n]
    out, closes_before, origin, n_closes, matched, flagged = [], 0, 0, 0, 0, []
    for r in range(world):
        hl = _lib.HALO_LEFT if r > 0 else 0
        hr = min(_lib.HALO_RIGHT, n - offs[r + 1])
        t = torch.frombuffer(bytearray(data[offs[r] - hl:offs[r + 1] + hr] + b"\0" * 64), dtype=torch.uint8).cuda()
        rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
        res, part = _lib.Result(), _lib.ShardPart()
        rc = L.agb_scan_shard_local(pat._h, C.c_void_p(t.data_ptr() + hl), offs[r + 1] - offs[r], hl, hr, int(r == 0),
                                    int(r == world - 1), int(offs[r + 1] + hr >= n), _lib.WANT_RECORDS | _lib.WANT_ORDINALS,
                                    C.c_void_p(rec.data_ptr()), cap, None, C.byref(res), C.byref(part))
        assert rc == 0, L.agb_last_error()
        assert not res.truncated
        if r == 0:
            origin = part.ord_origin
            n_closes += part.virt
        got = rec[:res.n_records].cpu().numpy()[:, :3].copy()
        got[:, :2] += offs[r] + part.byte_base
        got[:, 2] += origin + closes_before - part.ord_fix
        out.append(got)
        closes_before += part.closes
        n_closes += part.closes
        matched += res.n_matched
        flagged.append(res.n_flagged)
    return matched, np.concatenate(out), n_closes, flagged


@pytest.mark.gpu
@pytest.mark.parametrize("text", ["split", "split-nonl"])
@pytest.mark.parametrize("name", ["nl-k1", "dd-k1"])
def test_shard_local_last_shard_overflows(name, text, texts, answers):
    """two shards of the split text, one after the other on one device: only the last one overflows"""
    L = _lib.lib()
    pattern, kw, delim = PATTERNS[name]
    pat = ag.Pattern(pattern, **kw)
    data = texts[text]
    cnt, _, expect = answers[(name, text)]
    runs, launches = [], []
    L.agb_shutdown()
    for _ in range(2):
        before = L.agb_kernel_launches()
        runs.append(shard_walk(pat, data, 2, cnt + 16))
        launches.append(L.agb_kernel_launches() - before)
    flagged = runs[1][3]
    print("launches %s, survivors per shard %s" % (launches, flagged))
    assert launches[0] > launches[1] and flagged[0] < COLD_CAP < flagged[1]
    for matched, got, n_closes, _ in runs:
        assert matched == cnt
        assert np.array_equal(got, expect[:, :3])
        assert n_closes == closes(data, delim)


@pytest.mark.gpu
def test_bestmatch_overflow(devs, answers):
    """-B: the sweep's first levels pass (k = 2) overflows; best level, its count and its records"""
    import torch
    cnt, hist, expect = answers[("-B", "dense")]
    best = next(l for l in range(3) if hist[l])
    want = expect[expect[:, 3] == best]
    n = devs["dense"].numel() - 4096
    cap = cnt + 16
    rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
    L = _lib.lib()
    L.agb_shutdown()
    launches = []
    for _ in range(2):
        before = L.agb_kernel_launches()
        b, res = ag.bestmatch_device("because each", devs["dense"].data_ptr(), n, d_records=rec.data_ptr(), capacity=cap, linenum=1)
        launches.append(L.agb_kernel_launches() - before)
        got = rec[:res.n_records].cpu().numpy()
        assert (b, res.n_matched, res.n_records) == (best, hist[best], len(want))
        assert np.array_equal(got[:, :2], want[:, :2]) and (got[:, 3] == best).all()
    assert launches[0] > launches[1], launches


# ---- -c -v ---------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("text", ["dense", "list"])
@pytest.mark.parametrize("k", [0, 1])
def test_complement_count_overflow(k, text, texts, devs, answers):
    """`agrep -c -v`: records minus matching records, the records counted by the positive scan's ordinals pass --
    through agb_scan_device and a resident text; the cold call is the one that retries"""
    L = _lib.lib()
    want = answers[("-v", k, text)]
    pat = ag.Pattern("because each", k=k, inverse=True, linenum=True)
    data = texts[text]
    counts, launches = [], []
    L.agb_shutdown()
    for _ in range(2):
        before = L.agb_kernel_launches()
        counts.append(pat.scan_device(devs[text].data_ptr(), len(data)).n_matched)
        launches.append(L.agb_kernel_launches() - before)
    L.agb_shutdown()
    t = C.c_void_p()
    assert L.agb_text_from_host(data, len(data), C.byref(t)) == 0, L.agb_last_error()
    try:
        for _ in range(2):
            before = L.agb_kernel_launches()
            res = _lib.Result()
            assert L.agb_scan_text(pat._h, t, _lib.WANT_COUNT, None, 0, C.byref(res)) == 0, L.agb_last_error()
            counts.append(res.n_matched)
            launches.append(L.agb_kernel_launches() - before)
    finally:
        L.agb_text_free(t)
    print("-c -v -%d %s: launches %s" % (k, text, launches))
    assert counts == [want] * 4
    assert launches[0] > launches[1] and launches[2] > launches[3], launches


# ---- the command lines ---------------------------------------------------------------------------------------------

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "agrep")
DROP = os.path.join(ROOT, "oracle", "_ref", "agrep_dropin")
CLI = os.path.join(ROOT, "agrep_b200", "agrep-b200")


@pytest.fixture(scope="module")
def dense_file(texts, tmp_path_factory):
    path = str(tmp_path_factory.mktemp("agb_overflow_") / "dense.txt")
    with open(path, "wb") as f:
        f.write(texts["dense"])
    yield path
    os.unlink(path)


def run(binary, args):
    p = subprocess.run([binary] + args, capture_output=True, timeout=600, stdin=subprocess.DEVNULL)
    return p.returncode, p.stdout


@pytest.mark.gpu
def test_command_line_line_numbers_are_the_references(dense_file):
    """`agrep-b200 -n -1 'because each'`: the process starts on a fresh workspace, so its one scan of the dense file
    overflows; its output, line numbers included, is the reference's (compared by hash: about 60 MB)"""
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref binaries not built")
    args = ["-V0", "-n", "-1", "because each", dense_file]
    rc_r, out_r = run(REF, args)
    rc_b, out_b = run(CLI, args)
    assert rc_b == rc_r
    assert len(out_r) > 1000 and hashlib.sha256(out_b).hexdigest() == hashlib.sha256(out_r).hexdigest(), (out_b[:200], out_r[:200])


@pytest.mark.gpu
@pytest.mark.parametrize("binary", [DROP, CLI], ids=["dropin", "cli"])
def test_command_line_complement_count(binary, dense_file, answers):
    """`-c -v -n -1 'because each'` over the dense file, in a fresh process (so its scan overflows): the checker's count,
    which the reference prints too.
    (-n is ignored under -c, but keeps the automaton: without it the reference counts through sgrep's lossy filters)"""
    if not os.path.exists(binary):
        pytest.skip("%s not built" % binary)
    args = ["-V0", "-c", "-v", "-n", "-1", "because each", dense_file]
    _, out = run(binary, args)
    assert out == b"%d\n" % answers[("-v", 1, "dense")]
    if os.path.exists(REF):
        assert run(REF, args)[1] == out
