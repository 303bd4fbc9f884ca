#!/usr/bin/env python3
"""tools/window_bench.py [--gib 16] [--reps 3] -- what scanning a host text in windows costs against the whole-text scan.

The headline query (`agrep -2 'because each'`, the ordered list of matching records with ordinals) over the synthetic
corpus, two ways in:
  - agb_scan_fd on a page-cached file (pread(2) by four threads into the pinned ring), whole text on the device, against
    agb_scan_fd_windowed with windows of 256 MiB, 1 GiB and 4 GiB;
  - agb_scan_host from page-locked host memory (straight DMA), the same way.
Each configuration runs --reps times, alternated with the others; the best wall time of each is reported as GB/s of
text.  Every run must return the same count and list as the first.  The card's name, its power limit and the SM clock
(sampled by nvidia-smi while the scans run) are printed with the numbers.  The file goes to /dev/shm when it has room
(else the temporary directory) and is removed at the end; nothing is written into the tree."""
import argparse, ctypes as C, hashlib, os, shutil, sys, tempfile, time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import torch
import agrep_b200 as ag
from agrep_b200 import _lib
from stage_split import smi, ClockSampler

PATTERN, K, PAGE, NEEDLE_EVERY = "because each", 2, 4096, 4096     # as bench.py
PIECE = 256 << 20
WINDOWS = [256 << 20, 1 << 30, 4 << 30]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=16.0)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("window_bench.py needs a CUDA device")
    n = int(args.gib * (1 << 30)) // PIECE * PIECE
    L = _lib.lib()
    base = "/dev/shm" if os.path.isdir("/dev/shm") and shutil.disk_usage("/dev/shm").free > n + (2 << 30) else tempfile.gettempdir()
    if shutil.disk_usage(base).free < n + (1 << 30):
        raise SystemExit("no room for a %.1f GiB file in %s" % (n / (1 << 30), base))
    path = os.path.join(base, "agb_window_bench_%d.txt" % os.getpid())
    host = torch.empty(n, dtype=torch.uint8, pin_memory=True)          # page-locked: agb_scan_host copies from it directly
    try:
        for i in range(n // PIECE):
            spec = ag.corpus_spec(PIECE, first_page=i * (PIECE // PAGE), needle=PATTERN, needle_every=NEEDLE_EVERY, needle_maxedits=3)
            assert L.agb_corpus_fill_host(C.byref(spec), C.c_void_p(host.data_ptr() + i * PIECE)) == 0
        with open(path, "wb") as f:
            f.write(memoryview(host.numpy()))
        with open(path, "rb") as f:                                     # into the page cache
            while f.read(PIECE):
                pass
        pat = ag.Pattern(PATTERN, k=K)
        cap = 1 << 22
        recs = (_lib.Record * cap)()
        want = _lib.WANT_RECORDS | _lib.WANT_ORDINALS

        def run(src, window):
            res = _lib.Result()
            t0 = time.perf_counter()
            if src == "fd":
                fd = os.open(path, os.O_RDONLY)
                try:
                    rc = (L.agb_scan_fd(pat._h, fd, want, recs, cap, C.byref(res)) if window is None else
                          L.agb_scan_fd_windowed(pat._h, fd, window, want, recs, cap, C.byref(res)))
                finally:
                    os.close(fd)
            else:
                ptr = C.c_void_p(host.data_ptr())
                rc = (L.agb_scan_host(pat._h, ptr, n, want, recs, cap, C.byref(res)) if window is None else
                      L.agb_scan_host_windowed(pat._h, ptr, n, window, want, recs, cap, C.byref(res)))
            dt = time.perf_counter() - t0                               # the calls return after their last synchronisation
            assert rc == 0, L.agb_last_error()
            digest = hashlib.sha256(C.string_at(C.addressof(recs), res.n_records * C.sizeof(_lib.Record))).hexdigest()
            return dt, (res.n_matched, res.n_closes, res.truncated, digest)

        configs = [(src, w) for src in ("fd", "host") for w in [None] + [w for w in WINDOWS if w < n]]
        for c in configs:                                               # warm-up: module load, pinned rings, planner
            run(*c)
        best, answer = {}, None
        clk = ClockSampler()
        time.sleep(0.3)
        for _ in range(args.reps):
            for c in configs:
                dt, a = run(*c)
                answer = answer or a
                assert a == answer, (c, a, answer)
                best[c] = min(best.get(c, 1e9), dt)
        mhz, samples, capped = clk.stop()
        print("card: %s | power limit, max SM clock: %s | SM clock during the timed scans: %s MHz (median of %d samples)%s"
              % (torch.cuda.get_device_name(), smi("power.limit,clocks.max.sm"), mhz, samples, ", sw_power_cap seen" if capped else ""))
        print("text %.1f GiB (%s), pattern %r k=%d, list + ordinals: %d records, best of %d" %
              (n / (1 << 30), "page-cached file in " + base, PATTERN, K, answer[0], args.reps))
        print("%-6s %-12s %9s %8s %10s" % ("source", "window", "s", "GB/s", "vs whole"))
        for src in ("fd", "host"):
            whole = best[(src, None)]
            for c in [c for c in configs if c[0] == src]:
                w = "whole text" if c[1] is None else "%d MiB" % (c[1] >> 20)
                print("%-6s %-12s %9.3f %8.2f %9.1f%%" % (src, w, best[c], n / best[c] / 1e9, 100.0 * whole / best[c]))
    finally:
        try:
            os.unlink(path)
        except OSError:
            pass


if __name__ == "__main__":
    main()
