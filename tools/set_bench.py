"""Files per second: the synthetic corpus cut into files, scanned one agb_scan_host per file and as sets (agb_scan_set), and
the command line over the same files on disk -- agrep-b200 (sets under its budget, one scan per larger file) against the
reference binary on one core, and against another agrep-b200 binary (--cli-before, e.g. one built from the parent commit).
Workloads on both sides of the command line's 16 MiB set budget: 10 000 x 4 KiB, 1 000 x 64 KiB, 100 x 1 MiB in sets,
4 x 32 MiB alone.  The library calls are made with their arrays built beforehand (no Python copies in the timed region);
next to the wall time of agb_scan_set, its device time from the stream's events (agb_result.ms_records).  Prints a
markdown table and one JSON line; needs a GPU.
usage: python tools/set_bench.py [--out DIR] [--cli-before PATH]"""
import argparse, ctypes as C, json, os, subprocess, sys, tempfile, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import agrep_b200 as ag
from agrep_b200 import _lib

WORKLOADS = [(10000, 4096), (1000, 65536), (100, 1 << 20), (4, 32 << 20)]
PATTERNS = [("because each", dict(k=2), ["-2", "-c", "because each"]), ("the", dict(), ["-c", "the"])]
CLI = os.path.join(ROOT, "agrep_b200", "agrep-b200")
REF = os.path.join(ROOT, "oracle", "_ref", "agrep")
HOST_FILES = 500


def best_of(f, reps=2):
    f()                                           # warm-up: modules, workspaces, page cache
    ts = []
    for _ in range(reps):
        t = time.perf_counter(); f(); ts.append(time.perf_counter() - t)
    return min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--cli-before", default=None, help="another agrep-b200 binary to time over the same files")
    a = ap.parse_args()
    L = _lib.lib()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    corpus = ag.corpus_host(128 << 20, needle="because each", needle_every=16, needle_maxedits=3)
    rows = []
    with tempfile.TemporaryDirectory() as d:
        for nf, size in WORKLOADS:
            texts = [bytes(memoryview(corpus)[(i * size) % (len(corpus) - size):][:size]) for i in range(nf)]
            wd = os.path.join(d, "%dx%d" % (nf, size)); os.mkdir(wd)
            names = []
            for i, t in enumerate(texts):
                names.append(os.path.join(wd, "f%05d.txt" % i))
                with open(names[-1], "wb") as f:
                    f.write(t)
            total = nf * size
            print("workload %d x %d" % (nf, size), flush=True)
            ptrs = (C.c_void_p * nf)(*[C.cast(C.c_char_p(t), C.c_void_p) for t in texts])
            sizes = (C.c_uint64 * nf)(*[len(t) for t in texts])
            per = (_lib.Result * nf)()
            sub = min(nf, HOST_FILES)                # the per-file path is timed on the first HOST_FILES files, scaled to all
            for pat, kw, args in PATTERNS:
                p = ag.Pattern(pat, **kw)
                res = _lib.Result()

                def one_by_one():
                    got = 0
                    for i in range(sub):
                        assert L.agb_scan_host(p._h, ptrs[i], sizes[i], _lib.WANT_COUNT, None, 0, C.byref(res)) == 0
                        got += res.n_matched
                    return got
                tot = _lib.Result()

                def as_set(n=nf):
                    assert L.agb_scan_set(p._h, ptrs, sizes, n, _lib.WANT_COUNT, None, 0, per, C.byref(tot)) == 0
                    return tot.n_matched
                assert one_by_one() == as_set(sub), (nf, size, pat)
                together = as_set()
                t_host = best_of(one_by_one, 1) * nf / sub
                ms_dev = []
                t_set = best_of(lambda: (as_set(), ms_dev.append(tot.ms_records)), 3)
                t_cli = best_of(lambda: subprocess.run([CLI, "-V0"] + args + names, capture_output=True), 1)
                t_before = best_of(lambda: subprocess.run([a.cli_before, "-V0"] + args + names, capture_output=True), 1) \
                    if a.cli_before else None
                t_ref = best_of(lambda: subprocess.run(["taskset", "-c", "0", REF, "-V0"] + args + names, capture_output=True), 1) \
                    if os.path.exists(REF) else None
                rows.append(dict(files=nf, file_bytes=size, pattern=" ".join(args), matched=int(together),
                                 per_file_host_s=t_host, set_s=t_set, set_device_ms=min(ms_dev), cli_s=t_cli, cli_before_s=t_before,
                                 ref_1core_s=t_ref, bytes=total))
                print(json.dumps(rows[-1]), flush=True)
    lines = ["measured on: %s (name, power limit, maximum SM clock)" % q, "",
             "| files | size | command | per-file agb_scan_host (first %d files, scaled) | agb_scan_set | its device time |"
             " agrep-b200 before | agrep-b200 | reference, 1 core |" % HOST_FILES,
             "|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        def cell(t):
            return "not measured" if t is None else "%.1f ms, %.0f files/s, %.2f GB/s" % (t * 1e3, r["files"] / t, r["bytes"] / t / 1e9)
        lines.append("| %d | %d KiB | `%s` | %s | %s | %.2f ms | %s | %s | %s |" % (
            r["files"], r["file_bytes"] >> 10, r["pattern"], cell(r["per_file_host_s"]), cell(r["set_s"]), r["set_device_ms"],
            cell(r["cli_before_s"]), cell(r["cli_s"]), cell(r["ref_1core_s"])))
    table = "\n".join(lines)
    print(table)
    print(json.dumps({"gpu": q, "rows": rows}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "set_bench.md"), "w") as f:
            f.write(table + "\n")


if __name__ == "__main__":
    main()
