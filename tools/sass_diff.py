#!/usr/bin/env python3
"""tools/sass_diff.py OLD.so NEW.so [--ptxas OLD_ptxas.log NEW_ptxas.log] -- which kernels two builds compile differently.

Dumps the SASS of both libraries (cuobjdump -sass), splits each dump at its `Function :` headers and compares the
kernels by name.  Addresses and encodings are dropped, and every constant-bank operand c[0x0][0x...] becomes one
placeholder, so a kernel whose parameter block only moved (a field added to or removed from RecParams) compares equal.
With --ptxas, the registers, stack frame and spills that ptxas reported for each kernel (agrep_b200/csrc/ptxas.log)
are compared too.  Prints the kernels found in one build only, the kernels that differ (demangled) and a count of the
identical ones; exits 1 when a kernel present in both builds differs.  Development tool; it needs no GPU."""
import argparse, collections, re, subprocess, sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def kernels(so):
    """kernel name -> its normalised instructions"""
    out = subprocess.run([CUOBJDUMP, "-sass", so], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            if name in funcs:
                sys.exit("%s: kernel %s appears twice" % (so, name))
            funcs[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s*(.*?)\s*;", line)     # /*0040*/ INSTRUCTION ; /* encoding */
        if m and name is not None:
            funcs[name].append(re.sub(r"c\[0x0\]\[0x[0-9a-f]+\]", "c[0x0][PARAM]", m.group(1)))
    return funcs


def ptxas_usage(log):
    """kernel name -> (registers, stack frame, spill stores, spill loads) as ptxas reported them"""
    use, name = {}, None
    for line in open(log):
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            use[name] = [None] + [int(x) for x in m.groups()]
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and name in use:
            use[name][0] = int(m.group(1))
            name = None
    return {k: tuple(v) for k, v in use.items()}


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return out if len(out) == len(names) else list(names)


def family(name):
    """the kernel's own name, the same for all its instantiations (k_records_list)"""
    m = re.match(r"_Z(\d+)", name)
    return name[m.end():m.end() + int(m.group(1))] if m else name


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--ptxas", nargs=2, metavar=("OLD_LOG", "NEW_LOG"))
    a = ap.parse_args()
    old, new = kernels(a.old), kernels(a.new)
    only_old, only_new = sorted(set(old) - set(new)), sorted(set(new) - set(old))
    both = sorted(set(old) & set(new))
    differ = [k for k in both if old[k] != new[k]]
    if a.ptxas:
        uo, un = ptxas_usage(a.ptxas[0]), ptxas_usage(a.ptxas[1])
        usage_differ = [k for k in both if uo.get(k) != un.get(k)]
    print("kernels: %d in %s, %d in %s" % (len(old), a.old, len(new), a.new))
    for title, names in (("only in the old build", only_old), ("only in the new build", only_new)):
        print("%s: %d  %s" % (title, len(names), dict(collections.Counter(family(k) for k in names))))
    print("in both, same code: %d" % (len(both) - len(differ)))
    print("in both, different code: %d  %s" % (len(differ), dict(collections.Counter(family(k) for k in differ))))
    for k, d in zip(differ, demangle(differ)):
        print("  %s  (%d -> %d instructions)" % (d, len(old[k]), len(new[k])))
    if a.ptxas:
        print("in both, different registers / stack / spills: %d" % len(usage_differ))
        for k, d in zip(usage_differ, demangle(usage_differ)):
            print("  %s  %s -> %s" % (d, uo.get(k), un.get(k)))
    return 1 if differ else 0


if __name__ == "__main__":
    sys.exit(main())
