#!/usr/bin/env python3
"""tools/pair_plan_bench.py [--gib 32] [--steps 10] [--rounds 3] -- the headline step with the pair plan off and on.

bench.py's headline query (`agrep -2 'because each'` over the same device-resident synthetic corpus, the ordered list of
matching records returned), scanned with AGB_PLAN_PAIRS=0 and =1 alternately, `--rounds` times each: CUDA events around
`--steps` steps per round, then one torch.profiler pass per setting for the per-kernel times.  The planner's sampled flag
rates (k+1 plan and pair plan) are printed by AGB_DEBUG_PLAN on the first scan of each setting, and the card's name, power
limit and SM clock with the numbers.  Development tool; it writes nothing into the tree."""
import argparse, collections, os, sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import agrep_b200 as ag
from stage_split import PATTERN, K, PAGE, NEEDLE_EVERY, smi, ClockSampler


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=32.0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pair_plan_bench.py needs a CUDA device")
    n = int(args.gib * (1 << 30)) // PAGE * PAGE
    buf = torch.empty(n + 4096, dtype=torch.uint8, device="cuda")
    buf[n:].zero_()
    stream = torch.cuda.current_stream().cuda_stream
    ag.corpus_device(buf.data_ptr(), n, stream=stream, needle=PATTERN, needle_every=NEEDLE_EVERY, needle_maxedits=3)
    torch.cuda.synchronize()
    pat = ag.Pattern(PATTERN, k=K)
    cap = 1 << 22
    recs = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")

    def step():
        return pat.scan_device(buf.data_ptr(), n, stream=stream, d_records=recs.data_ptr(), capacity=cap)

    results = {0: [], 1: []}
    last = {}
    for v in (0, 1):                             # warm-up, and the planner's rates once per setting
        os.environ["AGB_PLAN_PAIRS"] = str(v)
        os.environ["AGB_DEBUG_PLAN"] = "1"
        print("AGB_PLAN_PAIRS=%d:" % v, flush=True)
        step()
        torch.cuda.synchronize()
        sys.stderr.flush()
        del os.environ["AGB_DEBUG_PLAN"]
        for _ in range(2):
            step()
    torch.cuda.synchronize()
    clk = ClockSampler()
    for _ in range(args.rounds):
        for v in (0, 1):
            os.environ["AGB_PLAN_PAIRS"] = str(v)
            step()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                r = step()
            e1.record()
            torch.cuda.synchronize()
            results[v].append(e0.elapsed_time(e1) / args.steps)
            last[v] = r
    mhz, samples, capped = clk.stop()
    print("card: %s | power limit, max SM clock: %s | SM clock during the timed steps: %s MHz (median of %d samples)%s"
          % (torch.cuda.get_device_name(), smi("power.limit,clocks.max.sm"), mhz, samples, ", sw_power_cap seen" if capped else ""))
    print("text %.2f GiB  pattern %r k=%d" % (n / (1 << 30), PATTERN, K))
    for v in (0, 1):
        r = last[v]
        print("AGB_PLAN_PAIRS=%d  matched %d  survivors of stage 1.5 %d  ms/step %s  ms_front %.3f  ms_records %.3f"
              % (v, r.n_matched, r.n_flagged, " ".join("%.3f" % x for x in results[v]), r.ms_front, r.ms_records))

    from torch.profiler import profile, ProfilerActivity
    for v in (0, 1):
        os.environ["AGB_PLAN_PAIRS"] = str(v)
        step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                step()
            torch.cuda.synchronize()
        per = collections.defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                per[ev.name.split("(")[0].split("<")[0].replace("void ", "").strip()] += ev.device_time_total / 1000.0 / 5
        print("AGB_PLAN_PAIRS=%d per kernel (ms/step, torch.profiler, 5 steps): %s  | all device activity %.3f"
              % (v, ", ".join("%s %.3f" % kv for kv in sorted(per.items(), key=lambda kv: -kv[1]) if kv[1] >= 0.01), sum(per.values())))


if __name__ == "__main__":
    main()
