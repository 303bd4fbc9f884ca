#!/usr/bin/env python3
"""tools/long_literal_bench.py [--gib 32] [--steps 5] [--rounds 3] [--every 64] [--k 0,1,2] -- simple literals of 80, 160
and 255 characters (320-bit rows, records_wide.cu) against one of 40 characters (64-bit rows), count and ordered list, at
each of the given numbers of errors (k > 0: Pattern(..., wide_approx=True)).

The synthetic corpus of bench.py, device-resident; each literal is planted, on a line of its own, into every `--every`-th
4 KiB page by a copy on the device (the corpus spec's needle holds at most 63 bytes).  Every query runs `--steps` steps
per round, the queries alternating, `--rounds` rounds; printed: the median ms per step over the rounds, each round's
number, the stage times of the last scan, and the card's name, power limit and SM clock read in the same run.
Development tool; it writes nothing into the tree."""
import argparse, os, statistics, sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
import agrep_b200 as ag
from golden.make_long_literal_golden import literal
from stage_split import PAGE, smi, ClockSampler

LENGTHS = (40, 80, 160, 255)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=32.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--every", type=int, default=64)
    ap.add_argument("--k", default="0", help="comma-separated numbers of errors, e.g. 1,2,4,8")
    args = ap.parse_args()
    ks = [int(x) for x in args.k.split(",")]
    if not torch.cuda.is_available():
        raise SystemExit("long_literal_bench.py needs a CUDA device")
    n = int(args.gib * (1 << 30)) // PAGE * PAGE
    buf = torch.empty(n + 4096, dtype=torch.uint8, device="cuda")
    buf[n:].zero_()
    stream = torch.cuda.current_stream().cuda_stream
    ag.corpus_device(buf.data_ptr(), n, stream=stream)
    pages = buf[:n].view(-1, PAGE)[::args.every]
    lits = {m: literal(m).encode() for m in LENGTHS}
    at = 64
    for m in LENGTHS:                            # "\n<literal>\n" at a fixed place of the page, one place per literal
        line = torch.frombuffer(bytearray(b"\n" + lits[m] + b"\n"), dtype=torch.uint8).cuda()
        pages[:, at:at + line.numel()] = line
        at += line.numel() + 64
    torch.cuda.synchronize()
    planted = pages.shape[0]
    cap = 2 * planted + 4096
    recs = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
    pats = {(m, k): ag.Pattern(lits[m], k=k, wide_approx=True) for m in LENGTHS for k in ks}
    assert all((pats[(m, k)].wide is not None) == (m > 61) for m in LENGTHS for k in ks)

    def step(m, k, listed):
        if listed:
            return pats[(m, k)].scan_device(buf.data_ptr(), n, stream=stream, d_records=recs.data_ptr(), capacity=cap)
        return pats[(m, k)].scan_device(buf.data_ptr(), n, stream=stream)

    queries = [(m, k, listed) for k in ks for m in LENGTHS for listed in (False, True)]
    for q in queries:                            # warm-up; every query finds each planted line once (k > 0: at least)
        r = step(*q)
        assert r.n_matched == planted if q[1] == 0 else planted <= r.n_matched <= cap, (q, r.n_matched, planted)
    torch.cuda.synchronize()
    times, last = {q: [] for q in queries}, {}
    clk = ClockSampler()
    for _ in range(args.rounds):
        for q in queries:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                last[q] = step(*q)
            e1.record()
            torch.cuda.synchronize()
            times[q].append(e0.elapsed_time(e1) / args.steps)
    mhz, samples, capped = clk.stop()
    print("card: %s | power limit, max SM clock: %s | SM clock during the timed steps: %s MHz (median of %d samples)%s"
          % (torch.cuda.get_device_name(), smi("power.limit,clocks.max.sm"), mhz, samples, ", sw_power_cap seen" if capped else ""))
    print("text %.2f GiB, each literal planted %d times (every %d pages)" % (n / (1 << 30), planted, args.every))
    for m, k, listed in queries:
        r = last[(m, k, listed)]
        print("%3d chars k=%d (%s rows) %-5s  median %.3f ms/step  rounds %s  matched %d  flagged chunks %d  ms_front %.3f  ms_records %.3f"
              % (m, k, "320-bit" if m > 61 else "64-bit", "list" if listed else "count", statistics.median(times[(m, k, listed)]),
                 " ".join("%.3f" % x for x in times[(m, k, listed)]), r.n_matched, r.n_flagged, r.ms_front, r.ms_records))


if __name__ == "__main__":
    main()
