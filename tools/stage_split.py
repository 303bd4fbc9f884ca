#!/usr/bin/env python3
"""tools/stage_split.py [--gib 32] [--steps 5] -- where the headline step's time goes, kernel by kernel.

Runs bench.py's headline query (`agrep -2 'because each'` over the same device-resident synthetic corpus, the ordered
list of matching records returned) a few times with CUDA events around the steps, then again under torch.profiler
with CUDA activities, and prints each kernel's mean device time per step.  The card's name, its power limit and the
SM clock (sampled by nvidia-smi while the timed steps run) are printed with the numbers: a time without them means
little.  Development tool; it writes nothing into the tree."""
import argparse, collections, os, subprocess, sys, threading, time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import agrep_b200 as ag

PATTERN, K, PAGE, NEEDLE_EVERY = "because each", 2, 4096, 4096     # as bench.py


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=" + query,
                               "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:                      # the numbers are still printed, marked as without their card state
        return "unavailable (%s)" % e


class ClockSampler:
    """nvidia-smi's SM clock every 100 ms while the timed steps run"""
    def __init__(self):
        self.proc = subprocess.Popen(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm,clocks_event_reasons.sw_power_cap",
                                      "--format=csv,noheader,nounits", "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        self.lines = []
        self.t = threading.Thread(target=lambda: [self.lines.append(ln) for ln in self.proc.stdout], daemon=True)
        self.t.start()

    def stop(self):
        self.proc.terminate()
        self.proc.wait(timeout=5)
        self.t.join(timeout=2)
        mhz = sorted(float(ln.split(",")[0]) for ln in self.lines if ln.split(",")[0].strip().isdigit())
        capped = any(ln.split(",")[-1].strip() == "Active" for ln in self.lines)
        return (mhz[len(mhz) // 2] if mhz else None), len(mhz), capped


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=32.0)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stage_split.py needs a CUDA device")
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

    for _ in range(3):
        r = step()
    torch.cuda.synchronize()
    clk = ClockSampler()
    time.sleep(0.3)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fronts, rests = [], []
    e0.record()
    for _ in range(args.steps):
        r = step()
        fronts.append(r.ms_front); rests.append(r.ms_records)
    e1.record()
    torch.cuda.synchronize()
    mhz, samples, capped = clk.stop()
    ms_step = e0.elapsed_time(e1) / args.steps

    print("card: %s | power limit, max SM clock: %s | SM clock during the timed steps: %s MHz (median of %d samples)%s"
          % (torch.cuda.get_device_name(), smi("power.limit,clocks.max.sm"), mhz, samples, ", sw_power_cap seen" if capped else ""))
    print("text %.2f GiB  pattern %r k=%d  matched %d  flagged (survivors) %d" % (n / (1 << 30), PATTERN, K, r.n_matched, r.n_flagged))
    print("step %.3f ms (CUDA events, %d steps)  ms_front %.3f  ms_records %.3f (means)" % (ms_step, args.steps, sum(fronts) / len(fronts), sum(rests) / len(rests)))

    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    per = collections.defaultdict(lambda: [0.0, 0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            name = ev.name.split("(")[0].split("<")[0].replace("void ", "").strip()
            per[name][0] += ev.device_time_total / 1000.0
            per[name][1] += 1
    total = sum(v[0] for v in per.values()) / args.steps
    print("%-26s %10s %8s %7s" % ("kernel / activity", "ms/step", "calls", "share"))
    for name, (ms, calls) in sorted(per.items(), key=lambda kv: -kv[1][0]):
        print("%-26s %10.3f %8.1f %6.1f%%" % (name[:26], ms / args.steps, calls / args.steps, 100 * ms / args.steps / total))
    print("%-26s %10.3f" % ("sum of device activity", total))


if __name__ == "__main__":
    main()
