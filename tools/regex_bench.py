#!/usr/bin/env python3
"""Throughput of regular-expression scans (regex.cu) over a device-resident synthetic corpus: GB/s of text per scan at
k = 0, 2, 4, count only (-c) and with the ordered list of matching lines; with --levels also a count-only levels scan
(AGB_WANT_LEVELS: every line's smallest level, the -B counting pass).  Device time from CUDA events around whole
scans (warm-up first, median of --reps), the card's name, power limit and SM clock read in the same run.  Separate from
bench.py, which measures the flagship literal workload.

    python tools/regex_bench.py --gib 32 --reps 5 [--pattern '(because|each) (state|world)'] [--levels] [--out DIR]"""
import argparse, json, os, statistics, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pattern", default="(because|each) (state|world)")
    ap.add_argument("--ks", default="0,2,4")
    ap.add_argument("--levels", action="store_true", help="also time a count-only levels scan per k")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import agrep_b200 as ag
    n = int(a.gib * (1 << 30)) // 4096 * 4096
    t = torch.empty(n + 4096, dtype=torch.uint8, device="cuda")
    ag.corpus_device(t.data_ptr(), n, seed=12345)
    torch.cuda.synchronize()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    out = {"gpu": card[0] if card else "unknown", "bytes": n, "pattern": a.pattern, "rows": []}
    cap = 1 << 26
    recs = torch.empty((cap, 4), dtype=torch.int64, device="cuda")
    for k in [int(x) for x in a.ks.split(",")]:
        p = ag.Pattern(a.pattern, k=k, regex=True)
        for mode in ("count", "list") + (("levels",) if a.levels else ()):
            kw = dict(d_records=recs.data_ptr(), capacity=cap) if mode == "list" else dict(levels=True) if mode == "levels" else {}
            p.scan_device(t.data_ptr(), n, **kw)                      # warm-up
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.reps)]
            matched = None
            for e0, e1 in ev:
                e0.record()
                r = p.scan_device(t.data_ptr(), n, **kw)
                e1.record()
                matched = r.n_matched
            torch.cuda.synchronize()
            ms = statistics.median(e0.elapsed_time(e1) for e0, e1 in ev)
            row = {"k": k, "mode": mode, "ms": round(ms, 3), "GB/s": round(n / ms / 1e6, 2), "matched": int(matched)}
            if mode == "levels":
                row["level_hist"] = [int(x) for x in r.level_hist[:k + 1]]
            out["rows"].append(row)
            print(json.dumps(row), flush=True)
    clk = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out["clocks_after"] = clk
    print(json.dumps({"gpu": out["gpu"], "clocks_after": clk}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(out, open(os.path.join(a.out, "regex_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
