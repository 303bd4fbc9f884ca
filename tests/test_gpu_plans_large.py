"""Stage 1's planned filters on the device, on texts of 256 MiB and more (the only texts adaptive_plan() re-plans), against
the checker.  Stage 1 is the one stage that can lose a match without anyone noticing: a chunk it does not flag is never
looked at again.  tests/_plans.py plants, for every case of its table (pair plans with 2, 3 and 4 pieces of 3 and 4
bytes, pieces spread apart by `.` and -w, bitap, sgrep, cost and 64-bit-row engines, -i, -n, a user delimiter), records
whose earlier surviving piece starts 1..8 bytes before a chunk edge, a warp's last chunk, a stage edge, a host slice,
the window edge and in the last record of the text -- on the bound cases with the later piece on the last byte of the
successor chunk.  Each case is scanned under the pair plan, the planner's k+1 plan and a forced mixed plan, each of
which must be seen to run (AGB_DEBUG_PLAN), and must give the checker's count, ordered records, ordinals and levels."""
import bisect
import ctypes as C
import os, re, subprocess
from concurrent.futures import ThreadPoolExecutor
import pytest
import _oracle, _plans
import agrep_b200 as ag
from agrep_b200 import _lib
from _plans import CASES, BY_NAME, MIB, N, WINDOW, REACH

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP = 1 << 20
LEVELS = ("rows64-k2", "nocase-k1")                  # their level histogram and levels are compared too
ENTRY = [c for c in CASES if c.span == REACH] + [BY_NAME["para-k2"]]
SETTINGS = (("pairs", {"AGB_PLAN_PAIRS": "1"}), ("k+1", {"AGB_PLAN_PAIRS": "0"}),
            ("mixed", {"AGB_PLAN_PAIRS": "0", "AGB_PLAN_MIXED": "0"}))
PIECE = re.compile(rb"\[(.*?)\]@(\d+)")


@pytest.fixture(scope="module")
def texts():
    return {kind: _plans.planted_text(kind) for kind in ("lines", "paras")}


@pytest.fixture(scope="module")
def devs(texts):
    import torch
    return {kind: torch.frombuffer(bytearray(t + b"\0" * 4096), dtype=torch.uint8).cuda() for kind, t in texts.items()}


@pytest.fixture(scope="module")
def answers(texts):
    """the checker's answer for each case, once: (count, level histogram or None, records); ctypes releases the GIL"""
    def one(case):
        a = _oracle.compile(case.pattern, **_plans.oracle_kw(case))
        if case.name in LEVELS:
            return _oracle.scan_levels(a, case.kw["k"], texts[case.text], cap=CAP)
        cnt, recs = _oracle.scan(a, texts[case.text], cap=CAP)
        return cnt, None, recs
    with ThreadPoolExecutor(max_workers=max(1, min(len(CASES), os.cpu_count() or 1))) as ex:
        return dict(zip((c.name for c in CASES), ex.map(one, CASES)))


@pytest.fixture
def env(monkeypatch):
    """set the planner's switches (only these), with AGB_DEBUG_PLAN on"""
    def set_(values):
        for v in ("AGB_PLAN_PAIRS", "AGB_PLAN_MIXED"):
            monkeypatch.delenv(v, raising=False)
        for k, v in values.items():
            monkeypatch.setenv(k, v)
        monkeypatch.setenv("AGB_DEBUG_PLAN", "1")
    return set_


def pair_lines(err):
    """the pieces of every 'pair plan chosen' line the planner printed, as [(bytes, offset)]"""
    if isinstance(err, str):
        err = err.encode("latin-1")
    return [[(m.group(1), int(m.group(2))) for m in PIECE.finditer(l.split(b"pair plan chosen:", 1)[1])]
            for l in err.splitlines() if b"pair plan chosen:" in l]


def three_byte_anchor(err):
    """did the planner choose a k+1 plan with a three-byte anchor?"""
    if isinstance(err, str):
        err = err.encode("latin-1")
    for l in err.splitlines():
        m = re.match(rb"agb plan: static rate \S+ -> chosen rate \S+:(.*)", l)
        if m and any(len(p.group(1)) == 3 for p in PIECE.finditer(m.group(1))):
            return True
    return False


def device_scan(pat, t, n, levels=False, ordinals=True):
    import torch
    rec = torch.zeros((CAP, 4), dtype=torch.int64, device="cuda")
    res = pat.scan_device(t.data_ptr(), n, d_records=rec.data_ptr(), capacity=CAP, ordinals=ordinals, levels=levels)
    assert not res.truncated
    return res, [tuple(r) for r in rec[:res.n_records].cpu().tolist()]


def missing_sites(case, recs):
    """the planted records of the case that no record of the list holds, named by their site"""
    begins = [r[0] for r in recs]
    out = []
    for s in _plans.sites(case):
        i = bisect.bisect_right(begins, s.at) - 1
        if i < 0 or not (recs[i][0] < s.at < recs[i][1]):
            out.append(s)
    return out


def same_answer(case, answer, res, recs, levels):
    cnt, hist, expect = answer
    lost = missing_sites(case, recs)
    assert not lost, "%s: planted records not reported: %s" % (case.name, lost[:8])
    assert res.n_matched == cnt
    # the reference never numbers sgrep's records (-n leaves sgrep for the automaton), and the checker's sgrep path counts
    # them from 1 where the automaton's j counts the virtual delimiter too: there the ordinal is not compared
    cols = 2 if ag.Pattern(case.pattern, **case.kw).desc.engine == 4 else 3         # 4: sgrep_bm (_lib.ENGINE_NAMES)
    assert [r[:cols] for r in recs] == [r[:cols] for r in expect]
    if levels:
        assert list(res.level_hist)[:case.kw["k"] + 1] == hist[:case.kw["k"] + 1]
        assert [r[3] for r in recs] == [r[3] for r in expect]


def test_the_checker_reports_every_planted_record(answers):
    for case in CASES:
        cnt, _, expect = answers[case.name]
        assert cnt < CAP
        assert not missing_sites(case, expect), case.name


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_every_plan_gives_the_checkers_answer(case, devs, answers, env, capfd):
    """the pair plan with the model's pieces, the planner's k+1 plan and a forced mixed plan: count, ordered records,
    ordinals (and levels for LEVELS); each plan seen to run"""
    pat = ag.Pattern(case.pattern, **case.kw)
    levels = case.name in LEVELS
    flagged = {}
    for name, values in SETTINGS:
        env(values)
        capfd.readouterr()
        res, recs = device_scan(pat, devs[case.text], N, levels=levels)
        err = capfd.readouterr().err
        chosen = pair_lines(err)
        if name == "pairs":
            assert chosen == [case.pieces], (case.name, err)
        else:
            assert chosen == [], (case.name, name, err)
        same_answer(case, answers[case.name], res, recs, levels)
        flagged[name] = res.n_flagged
    assert flagged["pairs"] > 0


def test_mixed_plans_run(devs, answers, env, capfd):
    """AGB_PLAN_MIXED=0 drops the three-byte grams' penalty: at least three cases then run a plan with a three-byte
    anchor (stage 1's second polynomial, launch_front_mixed) -- and still count what the checker counts"""
    mixed = []
    for case in CASES:
        env({"AGB_PLAN_PAIRS": "0", "AGB_PLAN_MIXED": "0"})
        capfd.readouterr()
        res = ag.Pattern(case.pattern, **case.kw).scan_device(devs[case.text].data_ptr(), N)
        err = capfd.readouterr().err
        assert res.n_matched == answers[case.name][0], case.name
        if three_byte_anchor(err):
            mixed.append(case.name)
    print("mixed plans with a three-byte anchor:", mixed)
    assert len(mixed) >= 3, mixed


@pytest.mark.parametrize("case", ENTRY, ids=lambda c: c.name)
def test_entry_points_under_the_pair_plan(case, texts, devs, answers, env, capfd):
    """scan_device (count only), agb_scan_shard_local over a world of one, agb_text_from_host + agb_scan_text and the
    windowed host scan (window 0, 256 MiB plus halos, is planned; the 32 MiB tail is under the threshold and keeps the
    static plan): the pair plan runs and the answer is the checker's.  The whole-text host scan (agb_scan_host without
    windows) does not plan at all; it keeps the static plan and still gives the checker's answer."""
    import torch
    L = _lib.lib()
    text, dev = texts[case.text], devs[case.text]
    cnt, _, expect = answers[case.name]
    expect3 = [r[:3] for r in expect]
    pat = ag.Pattern(case.pattern, **case.kw)
    env({"AGB_PLAN_PAIRS": "1"})

    capfd.readouterr()
    assert pat.scan_device(dev.data_ptr(), N).n_matched == cnt
    assert pair_lines(capfd.readouterr().err) == [case.pieces]

    rec = torch.zeros((CAP, 4), dtype=torch.int64, device="cuda")
    res, part = _lib.Result(), _lib.ShardPart()
    rc = L.agb_scan_shard_local(pat._h, C.c_void_p(dev.data_ptr()), N, 0, 0, 1, 1, 1, _lib.WANT_RECORDS | _lib.WANT_ORDINALS,
                                C.c_void_p(rec.data_ptr()), CAP, None, C.byref(res), C.byref(part))
    assert rc == 0, L.agb_last_error()
    assert pair_lines(capfd.readouterr().err) == [case.pieces]
    got = [(b + part.byte_base, e + part.byte_base, j + part.ord_origin - part.ord_fix)
           for b, e, j, _ in rec[:res.n_records].cpu().tolist()]
    assert res.n_matched == cnt and got == expect3

    t = C.c_void_p()
    assert L.agb_text_from_host(text, N, C.byref(t)) == 0
    try:
        recs, r2 = (_lib.Record * CAP)(), _lib.Result()
        assert L.agb_scan_text(pat._h, t, _lib.WANT_RECORDS | _lib.WANT_ORDINALS, recs, CAP, C.byref(r2)) == 0
    finally:
        L.agb_text_free(t)
    assert pair_lines(capfd.readouterr().err) == [case.pieces]
    assert r2.n_matched == cnt and [(recs[i].begin, recs[i].end, recs[i].ordinal) for i in range(r2.n_records)] == expect3

    res, recs = pat.scan_host(text, ordinals=True, window=WINDOW)
    err = capfd.readouterr().err
    assert pair_lines(err) == [case.pieces], err            # window 0 only: the tail window is not planned
    assert res.n_matched == cnt and [r[:3] for r in recs] == expect3

    res, recs = pat.scan_host(text, ordinals=True)
    err = capfd.readouterr().err
    assert "agb plan" not in err, err
    assert res.n_matched == cnt and [r[:3] for r in recs] == expect3


def test_bestmatch_under_the_pair_plan(devs, answers, env, capfd):
    """-B on a case whose best level is 2 (every planted record has two errors, nothing in the text fewer): the sweep's
    scans are planned, and it returns level 2 with the checker's records"""
    import torch
    case = BY_NAME["rows64-k2"]
    cnt, hist, expect = answers[case.name]
    assert hist[0] == hist[1] == 0 and hist[2] == cnt > 0
    env({"AGB_PLAN_PAIRS": "1"})
    capfd.readouterr()
    rec = torch.zeros((CAP, 4), dtype=torch.int64, device="cuda")
    best, res = ag.bestmatch_device(case.pattern, devs[case.text].data_ptr(), N, d_records=rec.data_ptr(), capacity=CAP)
    assert best == 2
    assert case.pieces in pair_lines(capfd.readouterr().err)
    assert res.n_matched == cnt
    assert [tuple(r[:2]) for r in rec[:res.n_records].cpu().tolist()] == [r[:2] for r in expect]


REF = os.path.join(ROOT, "oracle", "_ref", "agrep")
DROP = os.path.join(ROOT, "oracle", "_ref", "agrep_dropin")


@pytest.fixture(scope="module")
def lines_file(texts, tmp_path_factory):
    path = str(tmp_path_factory.mktemp("agb_plans_") / "lines.txt")
    with open(path, "wb") as f:
        f.write(texts["lines"])
    yield path
    os.unlink(path)


@pytest.mark.parametrize("args,name", [(["-2", "because each"], "para-k2"), (["-1", "-i", "-n", "people how too"], "nocase-k1")])
def test_dropin_under_the_pair_plan(lines_file, args, name):
    """the reference's own program over the drop-in layer prints what the unmodified reference prints for the 288 MiB
    text, with the pair plan forced on (the drop-in's descriptors are re-planned too: stderr shows the plan)"""
    if not (os.path.exists(REF) and os.path.exists(DROP)):
        pytest.skip("oracle/_ref binaries not built")
    r = subprocess.run([REF, "-V0"] + args + [lines_file], capture_output=True, timeout=900, stdin=subprocess.DEVNULL)
    e = dict(os.environ, AGB_PLAN_PAIRS="1", AGB_DEBUG_PLAN="1")
    d = subprocess.run([DROP, "-V0"] + args + [lines_file], capture_output=True, timeout=900, stdin=subprocess.DEVNULL, env=e)
    assert d.returncode == r.returncode, d.stderr[-500:]
    assert d.stdout == r.stdout and len(r.stdout) > 1000
    assert BY_NAME[name].pieces in pair_lines(d.stderr), d.stderr[-500:]
