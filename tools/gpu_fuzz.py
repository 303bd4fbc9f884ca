"""tools/gpu_fuzz.py [seed] -- development fuzz on an H100: random metacharacter patterns and options, the GPU path
(agb_scan_host, list + ordinals, and count only) against the oracle.  Found the -p + multi-byte delimiter case.
The committed, shorter version is tests/test_gpu_parity.py::test_random_metachar_differential."""
import random, sys, os
sys.path.insert(0, os.getcwd()); sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import _oracle, _corpus
import agrep_b200 as ag
base = _corpus.make_text(3000, seed=5)
words = [w for w in base.decode().split() if w.isalpha()]
rnd = random.Random(int(sys.argv[1]) if len(sys.argv) > 1 else 77)
def rand_pattern():
    w = (rnd.choice(words) + " " + rnd.choice(words))[:rnd.randint(3, 20)]
    out = []
    for ch in w:
        r = rnd.random()
        out.append("." if r < 0.08 else "[" + ch + "x]" if r < 0.12 else "[^q]" if r < 0.15 else "#" if r < 0.17 else ch.upper() if r < 0.19 else ch)
    p = "".join(out)
    r = rnd.random()
    return ("<" + p[:2] + ">" + p[2:] if r < 0.08 else p + "," + rnd.choice(words) if r < 0.14 else p + ";" + rnd.choice(words) if r < 0.20 else "^" + p if r < 0.24 else p + "$" if r < 0.28 else p)
bad = done = 0
for _ in range(700):
    n = rnd.randint(1000, 2900)
    data = ("\n".join(base.decode().split("\n")[:n]) + rnd.choice(["\n", "", "\n\n"])).encode()
    pat = rand_pattern()
    k = rnd.choice([0, 0, 1, 2, 3, 4, 6, 8])
    kw = dict(k=k)
    if rnd.random() < 0.8: kw["linenum"] = 1
    for p_, key in ((0.25, "nocase"), (0.15, "wordbound"), (0.1, "inverse"), (0.05, "ins_free"), (0.04, "wholeline")):
        if rnd.random() < p_: kw[key] = 1
    if rnd.random() < 0.15: kw["delim"] = rnd.choice(["$$", "e ", "ab", "\\."])
    if k and rnd.random() < 0.06: kw["cost_s"] = 2
    try:
        a = _oracle.compile(pat, **kw)
    except _oracle.OracleError:
        continue
    try:
        p = ag.Pattern(pat, **kw)
    except ag.AgrepError as e:
        if "delimiter matches more" in str(e): continue
        print("PRODUCT REJECTS", repr(pat), kw, e); bad += 1; continue
    cnt, recs = _oracle.scan(a, data)
    res, got = p.scan_host(data, ordinals=True)
    res2, _ = p.scan_host(data, want_records=False)
    done += 1
    keep = (lambda t: t[:3]) if a.engine != 4 else (lambda t: t[:2])      # sgrep/bm has no j (no -n on that path)
    if res.n_matched != cnt or res2.n_matched != cnt or [keep(t) for t in got] != [keep(t) for t in recs]:
        bad += 1
        print("DIFF", repr(pat), kw, "oracle", cnt, "gpu", res.n_matched, res2.n_matched, "first", recs[:2], got[:2])
print("done", done, "bad", bad)
