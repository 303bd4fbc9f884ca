#!/usr/bin/env python3
"""Cost of -p with a record delimiter of two or more bytes (delim_kind 3, delim_state.cu) over a device-resident synthetic
corpus: GB/s of `-p -d 'e '` against `-p` with newline records (the dense tile form both ways), count only and with the
ordered list, from CUDA events around whole scans (warm-up first, median of --reps); and the GB/s of the delimiter pass
alone, from the kernel times torch.profiler records for its three launches in one more count scan.  The card's name,
power limit and SM clock are read in the same run.  Separate from bench.py, which measures the flagship workload.

    python tools/sticky_delim_bench.py --gib 32 --reps 5 [--pattern 'because each' --k 2] [--out DIR]"""
import argparse, json, os, statistics, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pattern", default="because each")
    ap.add_argument("--k", type=int, default=2)
    ap.add_argument("--delim", default="e ")
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
    out = {"gpu": card[0] if card else "unknown", "bytes": n, "pattern": a.pattern, "k": a.k, "rows": []}
    cap = 1 << 26
    recs = torch.empty((cap, 4), dtype=torch.int64, device="cuda")
    forms = (("-p -d %r" % a.delim, dict(delim=a.delim)), ("-p (newline records)", {}))
    for name, dkw in forms:
        p = ag.Pattern(a.pattern, k=a.k, ins_free=True, sticky_delim=True, **dkw)
        for mode in ("count", "list"):
            kw = dict(d_records=recs.data_ptr(), capacity=cap) if mode == "list" else {}
            p.scan_device(t.data_ptr(), n, **kw)                      # warm-up
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.reps)]
            for e0, e1 in ev:
                e0.record()
                r = p.scan_device(t.data_ptr(), n, **kw)
                e1.record()
            torch.cuda.synchronize()
            ms = statistics.median(e0.elapsed_time(e1) for e0, e1 in ev)
            row = {"form": name, "mode": mode, "ms": round(ms, 3), "GB/s": round(n / ms / 1e6, 2), "matched": int(r.n_matched),
                   "truncated": int(r.truncated)}
            out["rows"].append(row)
            print(json.dumps(row), flush=True)
    # the delimiter pass alone: its kernels' device time inside one count scan
    from torch.profiler import profile, ProfilerActivity
    p = ag.Pattern(a.pattern, k=a.k, ins_free=True, sticky_delim=True, delim=a.delim)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        p.scan_device(t.data_ptr(), n)
        torch.cuda.synchronize()
    us = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "k_dstate" in e.name:
            us[e.name] = us.get(e.name, 0.0) + e.device_time_total
    total = sum(us.values()) / 1e3
    row = {"form": "delimiter pass alone", "ms": round(total, 3), "GB/s": round(n / total / 1e6, 2) if total else None,
           "ms_by_kernel": {k: round(v / 1e3, 3) for k, v in us.items()}}
    out["rows"].append(row)
    print(json.dumps(row), flush=True)
    clk = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out["clocks_after"] = clk
    print(json.dumps({"gpu": out["gpu"], "clocks_after": clk}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(out, open(os.path.join(a.out, "sticky_delim_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
