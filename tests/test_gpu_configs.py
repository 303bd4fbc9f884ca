"""BASELINE.json configs[2] and configs[3] as parity cases (SURVEY 8d):
  configs[2]: 32-char pattern, -3 -w, paragraph records (-d '$$'): M = 37 > 32, the reference refuses it
              ("pattern too long", maskgen.c:201-208), so parity is against the widened oracle (validated on M<=31
              against the real reference in test_oracle_vs_reference.py); a 26-char variant the reference accepts is in the
              golden vectors (para_k3_26).
  configs[3]: -i -B best-match sweep with a 20-char mixed-case pattern (agrep.c:3582-3728)."""
import pytest
import _oracle
import agrep_b200 as ag

pytestmark = pytest.mark.gpu
PAGE = 4096
P32 = "business give group toward young"          # 32 chars, five adjacent vocabulary words
P20 = "Because Each Just Th"                      # 20 chars, mixed case


def test_config2_wide_pattern_paragraph_records():
    assert len(P32) == 32
    with pytest.raises(_oracle.OracleError):
        _oracle.compile(P32, width=32, k=3, linenum=1, wordbound=1, delim="$$")      # the reference's own limit
    n = 2048 * PAGE
    host = ag.corpus_host(n, paragraphs=True, needle=P32, needle_every=16, needle_maxedits=4)
    kw = dict(k=3, linenum=1, wordbound=1, delim="$$")
    a = _oracle.compile(P32, **kw)
    assert a.M == 37
    cnt, recs = _oracle.scan(a, host)
    p = ag.Pattern(P32, k=3, linenum=True, wordbound=True, delim="$$")
    d = p.desc
    assert d.M == 37 and d.plan == ag.api.PLAN_ANCHORS and d.n_anchors == 4
    res, got = p.scan_host(host)
    assert res.n_matched == cnt and cnt >= 60
    assert [(b, e) for b, e, _, _ in got] == [(b, e) for b, e, _ in recs]


def test_config3_bestmatch_sweep_case_insensitive():
    import torch
    n = 4096 * PAGE
    for maxedits, every in ((0, 64), (3, 64), (2, 1 << 20)):
        needle = "because each just th"
        host = ag.corpus_host(n, needle=needle, needle_every=every, needle_maxedits=maxedits)
        t = torch.frombuffer(bytearray(host + b"\0" * 64), dtype=torch.uint8).cuda()
        want = -1
        for k in range(0, 9):
            a = _oracle.compile(P20, k=k, linenum=1, nocase=1)
            cnt, _ = _oracle.scan(a, host, want_records=False)
            if cnt:
                want = (k, cnt)
                break
        best, res = ag.bestmatch_device(P20, t.data_ptr(), n, nocase=1)
        assert (best, res.n_matched) == want, (maxedits, every, best, res.n_matched, want)


def test_the_record_stage_gets_few_chunks_when_the_filters_can_thin():
    """which form runs is a performance decision, not a parity one -- so it gets its own check: n_flagged is the number
    of chunks handed to the record stage.  Patterns of common words flag several per cent of the chunks in stage 1;
    stage 1.5 must still run and leave almost nothing (a shortcut that sent the k=4 case to the every-byte form cost
    6x), while an exact short literal that is everywhere goes to the every-byte form directly.  A multi-part pattern has
    no stage 1.5: stage 1's flags go to the list form while they are few ('gove' of the;government flags 1.1 %) and to
    the every-byte form when they are not ('the' or 'gov' of the,government flags 12 %); both against the checker."""
    n = 16384 * PAGE                                  # 64 MiB
    host = ag.corpus_host(n, needle="because each", needle_every=4096, needle_maxedits=3)
    chunks = n // 16
    for pat, kw in (("because each just those", dict(k=4, nocase=True, linenum=True)), ("because each", dict(k=2)),
                    ("because each", dict(k=3)), ("government", dict())):
        res, _ = ag.Pattern(pat, **kw).scan_host(host, want_records=False)
        assert res.n_flagged < chunks // 20, (pat, kw, res.n_flagged, chunks)
    res, _ = ag.Pattern("the").scan_host(host, want_records=False)
    assert res.n_flagged == chunks
    for pat, sparse in (("the;government", True), ("the,government", False)):
        a = _oracle.compile(pat)
        cnt, _ = _oracle.scan(a, host, want_records=False)
        _, recs = _oracle.scan(a, host, cap=cnt)          # (the default room, a record per byte, is 1.6 GB here)
        res, got = ag.Pattern(pat).scan_host(host)
        assert res.n_matched == cnt and [(b, e) for b, e, _, _ in got] == [(b, e) for b, e, _ in recs], pat
        assert (0 < res.n_flagged < chunks // 20) if sparse else res.n_flagged == chunks, (pat, res.n_flagged, chunks)


def test_anchor_planner_plans_agree(monkeypatch):
    """the anchor planner (scan.cu: grams counted on a sample of the text, k+1 disjoint grams by dynamic program) only
    changes which chunks stage 1 flags, never the answer: the static plan (small texts), the planned one and a forced
    mixed plan (four-byte + three-byte anchors: two polynomials in stage 1, table compare in stage 1.5) return the same
    ordered list on a 320 MiB text, and a window of it equals the oracle's"""
    import torch
    n = 320 << 20
    t = torch.empty(n + 4096, dtype=torch.uint8, device="cuda")
    t[n:].zero_()
    ag.corpus_device(t.data_ptr(), n, needle="because each", needle_every=512, needle_maxedits=3)
    torch.cuda.synchronize()
    cap = 1 << 20
    lists = []
    pats = (("because each", dict(k=2, linenum=True)), ("because each just those", dict(k=3, nocase=True, linenum=True)),
            ("Government", dict(k=1, nocase=True, linenum=True)), ("national order", dict(k=3, linenum=True)))
    for env in (None, "0", "10"):
        if env is None:
            monkeypatch.delenv("AGB_PLAN_MIXED", raising=False)
        else:
            monkeypatch.setenv("AGB_PLAN_MIXED", env)
        for pat, kw in pats:
            rec = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
            # each setting scans the text shifted by one page more: three overlapping texts, compared below where they
            # overlap (the plan cache's key covers AGB_PLAN_MIXED, so the shift is not what makes each setting re-plan)
            off = {None: 0, "0": 4096, "10": 8192}[env]
            r = ag.Pattern(pat, **kw).scan_device(t.data_ptr() + off, n - 16384, d_records=rec.data_ptr(), capacity=cap)
            lists.append((env, pat, off, int(r.n_matched), (rec[:r.n_records, :2] + off).cpu()))
    import _oracle
    by_pat = {}
    for env, pat, off, cnt, l in lists:
        by_pat.setdefault(pat, []).append((env, off, cnt, l))
    for pat, runs in by_pat.items():
        # the three texts overlap in [8192, n - 16384): same records there
        def inside(l):
            m = (l[:, 0] >= 8192 + 4096) & (l[:, 1] < n - 16384 - 4096)
            return l[m]
        base = inside(runs[0][3])
        assert base.shape[0] > 10 or pat != "because each", pat
        for env, off, cnt, l in runs[1:]:
            assert inside(l).shape == base.shape and bool((inside(l) == base).all()), (pat, env)
    # a 4 MiB window (pages end in '\n', so it starts on a record) against the oracle
    w0, wn = 16 << 20, 4 << 20
    host = bytes(t[w0:w0 + wn].cpu().numpy())
    for pat, kw in pats:
        okw = {k: (1 if v is True else v) for k, v in kw.items()}
        cnt, orecs = _oracle.scan(_oracle.compile(pat, **okw), host)
        l = by_pat[pat][0][3]
        m = (l[:, 0] >= w0 - 1) & (l[:, 0] < w0 + wn - 1)
        assert [(int(b) - w0, int(e) - w0) for b, e in l[m].tolist()] == [(b, e) for b, e, _ in orecs], pat
