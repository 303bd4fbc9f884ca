"""Parity at BASELINE.json's full size (32 GiB on one H100) through size-independent properties -- the oracle
cannot scan 32 GiB in seconds, so we use what the domain offers:
  * additivity: the corpus is made of independent pages, so count(whole) == sum of count(shard) for any
    page-aligned sharding (a checksum of checksums), and the whole-corpus record list is the concatenation;
  * sampling: on 64 randomly chosen 1 MiB windows the device scan equals the oracle bit for bit (the window is
    regenerated on the host by the same generator);
  * monotonicity in k (the rows are nested, asearch.c:98-114) and determinism (two runs, identical lists);
  * completeness on planted needles: every planted line with e <= k substitutions is reported.
Size: AGB_FULLSIZE_GIB (default 32; the test skips if the device cannot hold it)."""
import os, random
import pytest
import _oracle
import agrep_b200 as ag

pytestmark = pytest.mark.gpu
GIB = float(os.environ.get("AGB_FULLSIZE_GIB", "32"))
PAGE = 4096
NEEDLE, EVERY, MAXE = "because each", 4096, 3


@pytest.fixture(scope="module")
def corpus():
    import torch
    n = int(GIB * (1 << 30)) // PAGE * PAGE
    free, _ = torch.cuda.mem_get_info()
    if free < n * 1.05 + (2 << 30):
        pytest.skip("device memory too small for %.0f GiB" % GIB)
    t = torch.empty(n + 4096, dtype=torch.uint8, device="cuda")
    t[n:].zero_()
    ag.corpus_device(t.data_ptr(), n, needle=NEEDLE, needle_every=EVERY, needle_maxedits=MAXE)
    torch.cuda.synchronize()
    return t, n


def scan(pat, t, off, n, cap=0):
    import torch
    if cap:
        recs = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
        res = pat.scan_device(t.data_ptr() + off, n, d_records=recs.data_ptr(), capacity=cap)
        return res, recs[:res.n_records, :2].cpu()
    return pat.scan_device(t.data_ptr() + off, n), None


def test_additivity_and_determinism(corpus):
    t, n = corpus
    pat = ag.Pattern(NEEDLE, k=2)
    cap = 1 << 22
    whole, recs = scan(pat, t, 0, n, cap)
    assert whole.n_matched <= cap
    again, recs2 = scan(pat, t, 0, n, cap)
    assert again.n_matched == whole.n_matched and bool((recs == recs2).all())
    assert bool((recs[1:, 0] > recs[:-1, 0]).all())              # ordered, no record twice
    parts, total, pieces = 8, 0, []
    per = n // (PAGE * parts) * PAGE
    for i in range(parts):
        length = per if i < parts - 1 else n - per * (parts - 1)
        r, rr = scan(pat, t, i * per, length, cap)
        total += r.n_matched
        rr = rr.clone(); rr += i * per
        pieces.append(rr)
    assert total == whole.n_matched
    import torch
    cat = torch.cat(pieces)
    # a shard's first record begins at its own virtual '\n' (-1): the same byte as the page-ending '\n' before it
    assert bool((cat == recs).all())


def test_monotone_in_k_and_planted_needles(corpus):
    t, n = corpus
    counts = []
    for k in range(0, 4):
        r, _ = scan(ag.Pattern(NEEDLE, k=k, linenum=True), t, 0, n)
        counts.append(r.n_matched)
    assert counts == sorted(counts)
    pages = n // PAGE
    planted = [sum(1 for p in range(0, pages, EVERY) if (p // EVERY) % (MAXE + 1) <= k) for k in range(4)]
    assert all(c >= p for c, p in zip(counts, planted)), (counts, planted)
    # each planted line is in the k=3 list: it starts its page
    pat = ag.Pattern(NEEDLE, k=3, linenum=True)
    for p in random.Random(5).sample(range(0, pages, EVERY), min(64, len(range(0, pages, EVERY)))):
        r, rr = scan(pat, t, p * PAGE, PAGE, 64)
        assert r.n_matched >= 1 and int(rr[0, 0]) == -1          # the page's first line


def test_sampled_windows_equal_oracle(corpus):
    t, n = corpus
    rnd = random.Random(11)
    win = 256 * PAGE            # 64 windows x 1 MiB x 4 patterns: the oracle reads 256 MiB, a few seconds
    pats = [("because each", dict(k=2, linenum=1)), ("the", dict()), ("Government", dict(k=1, nocase=1, linenum=1)),
            ("national order", dict(k=3, wordbound=1, linenum=1))]
    for _ in range(64):
        pg = rnd.randrange(0, n // PAGE - 256)
        host = ag.corpus_host(win, first_page=pg, needle=NEEDLE, needle_every=EVERY, needle_maxedits=MAXE)
        for p, kw in pats:
            a = _oracle.compile(p, **kw)
            cnt, orecs = _oracle.scan(a, host)
            r, rr = scan(ag.Pattern(p, **{k: bool(v) if k != "k" else v for k, v in kw.items()}), t, pg * PAGE, win, 1 << 18)
            assert r.n_matched == cnt, (p, pg)
            assert [(int(b), int(e)) for b, e in rr.tolist()] == [(b, e) for b, e, _ in orecs], (p, pg)


def test_every_byte_forms_and_ordinals_at_full_size(corpus):
    """the record stage that walks every byte (slices form: classes, -v, 'the') and the ordinals pass, at full size:
    count(whole) == sum of count(part) over page-aligned parts; record closes add up the same way (each part counts
    its own virtual '\\n' and the delimiter appended at its EOF, shard.ordinal_base); ordinals are the line numbers of
    the generator: a record's ordinal is 1 + (newlines at or before its closing newline)."""
    import torch
    from agrep_b200 import shard
    t, n = corpus
    parts = 4
    per = n // (PAGE * parts) * PAGE
    spans = [(i * per, per if i < parts - 1 else n - per * (parts - 1)) for i in range(parts)]
    for p, kw in (("t[hx]e", dict(k=0, linenum=True)), ("because each", dict(k=2, inverse=True, linenum=True)), ("the", dict())):
        pat = ag.Pattern(p, **kw)
        whole, _ = scan(pat, t, 0, n)
        assert whole.n_matched == sum(scan(pat, t, o, l)[0].n_matched for o, l in spans), p
    pat = ag.Pattern(NEEDLE, k=2, linenum=True)
    cap = 1 << 22
    recs = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
    whole = pat.scan_device(t.data_ptr(), n, d_records=recs.data_ptr(), capacity=cap, ordinals=True)
    ords = recs[:whole.n_records, 2].clone()
    ends = recs[:whole.n_records, 1].clone()
    assert bool((ords[1:] > ords[:-1]).all())
    closes, got = [], []
    for r, (o, l) in enumerate(spans):
        res = pat.scan_device(t.data_ptr() + o, l, d_records=recs.data_ptr(), capacity=cap, ordinals=True)
        got.append(recs[:res.n_records, 2].clone() + shard.ordinal_base(closes, r))
        closes.append(int(res.n_closes))
    assert bool((torch.cat(got) == ords).all())
    assert whole.n_closes == sum(closes) - 2 * (parts - 1)
    # against a direct count on a sample: newlines in [0, end] + the virtual one
    for i in random.Random(3).sample(range(int(whole.n_records)), 8):
        e = int(ends[i])
        if e > (1 << 31):
            continue
        assert int(ords[i]) == int((t[:e + 1] == 10).sum().item()) + 1
