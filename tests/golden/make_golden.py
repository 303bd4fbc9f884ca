#!/usr/bin/env python3
"""Generates tests/golden/* from the UNMODIFIED reference (oracle/_ref, built by oracle/Makefile from the reference
sources).  Run where oracle/_ref exists:  python tests/golden/make_golden.py
Inputs are the seeded corpora of tests/_corpus.py, so only the answers are committed."""
import json, os, re, subprocess, sys, tempfile
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _corpus
REF = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref")

CORPORA = {
    "nl": dict(nlines=4000, seed=12345),
    "nonl": dict(nlines=500, seed=7, trailing_newline=False),
    "para": dict(nlines=3000, seed=99, paragraphs=True),
}

# (name, corpus, pattern, reference args (without -V0/-c/-n), api kwargs for oracle/product)
SCAN_CASES = [
    ("exact_n", "nl", "against three", ["-n"], dict(k=0, linenum=1)),
    ("k1", "nl", "against three", ["-n", "-1"], dict(k=1, linenum=1)),
    ("k2", "nl", "because each", ["-n", "-2"], dict(k=2, linenum=1)),
    ("k2_nonl", "nonl", "also should", ["-n", "-2"], dict(k=2, linenum=1)),
    ("k3", "nl", "government", ["-n", "-3"], dict(k=3, linenum=1)),
    ("k4_i", "nl", "governmental", ["-n", "-4", "-i"], dict(k=4, linenum=1, nocase=1)),
    ("k5", "nl", "governmental", ["-n", "-5"], dict(k=5, linenum=1)),
    ("k8", "nl", "homogeneous approx", ["-n", "-8"], dict(k=8, linenum=1)),
    ("k1_w", "nl", "matching", ["-n", "-1", "-w"], dict(k=1, linenum=1, wordbound=1)),
    ("k0_w", "nl", "the", ["-n", "-w"], dict(k=0, linenum=1, wordbound=1)),
    ("k2_v", "nl", "the", ["-n", "-1", "-v"], dict(k=1, linenum=1, inverse=1)),
    ("class_k1", "nl", "pat[a-t]ern", ["-n", "-1"], dict(k=1, linenum=1)),
    ("dot", "nl", "st.ing", ["-n"], dict(k=0, linenum=1)),
    ("angle_k2", "nl", "<algo>rithm", ["-n", "-2"], dict(k=2, linenum=1)),
    ("bol", "nl", "^the", ["-n"], dict(k=0, linenum=1)),
    ("eol_k1", "nl", "world$", ["-n", "-1"], dict(k=1, linenum=1)),
    ("and", "nl", "state;world", ["-n"], dict(k=0, linenum=1)),
    ("negclass", "nl", "[^a-s]he ", ["-n"], dict(k=0, linenum=1)),
    ("cost_s1", "nl", "the other", ["-n", "-2", "-S1"], dict(k=2, linenum=1, cost_s=1)),
    ("cost_s2", "nl", "of the other", ["-n", "-3", "-S2"], dict(k=3, linenum=1, cost_s=2)),
    ("cost_i2d3", "nl", "of the other", ["-n", "-3", "-I2", "-D3"], dict(k=3, linenum=1, cost_i=2, cost_d=3)),
    ("insfree", "nl", "government", ["-n", "-2", "-p"], dict(k=2, linenum=1, ins_free=1)),
    ("wild", "nl", "a#t", ["-n"], dict(k=0, linenum=1)),
    ("i_k0", "nl", "Against Three", ["-n", "-i"], dict(k=0, linenum=1, nocase=1)),
    ("x_k0", "para", "", ["-n", "-x"], None),  # placeholder, removed below
    ("para_w_k0", "para", "world", ["-n", "-w", "-d", "$$"], dict(k=0, linenum=1, wordbound=1, delim="$$")),
    ("para_w_k2", "para", "because each", ["-n", "-w", "-d", "$$", "-2"], dict(k=2, linenum=1, wordbound=1, delim="$$")),
    ("para_k3_26", "para", "well eaxh into him here no", ["-n", "-w", "-d", "$$", "-3"],
     dict(k=3, linenum=1, wordbound=1, delim="$$")),
    ("delim_word", "nl", "world", ["-n", "-d", "the", "-1"], dict(k=1, linenum=1, delim="the")),
    # sgrep()/bm() path (config 1)
    ("bm_the", "nl", "the", [], dict()),
    ("bm_The", "nl", "The", [], dict()),
    ("bm_the_nonl", "nonl", "the", [], dict()),
    ("bm_w", "nl", "the", ["-w"], dict(wordbound=1)),
    ("bm_gov", "nl", "government", [], dict()),
    ("bm_none", "nl", "zzzz", [], dict()),
]
SCAN_CASES = [c for c in SCAN_CASES if c[4] is not None]

DUMP_CASES = [
    ("abc", ["-n", "-1"]), ("because each", ["-n", "-2"]), ("win", ["-n", "-w", "-d", "$$"]),
    ("pat[a-t]ern", ["-n", "-1"]), ("<algo>rithm", ["-n", "-2"]), ("state;world", ["-n"]),
    ("state,world", ["-n"]), ("a#t", ["-n"]), ("st.ing", ["-n"]), ("^the", ["-n"]), ("world$", ["-n", "-1"]),
    ("The World", ["-n", "-i"]), ("[^a-s]he ", ["-n"]), ("matching", ["-n", "-x"]), ("government", ["-n", "-2", "-p"]),
    ("between both life", ["-n", "-3", "-I2", "-D3"]), ("world", ["-n", "-d", "the", "-1"]),
    ("a\\.b\\;c", ["-n"]), ("x[a\\-c]y", ["-n"]), ("x[\\]a]y", ["-n"]),
]


def run(cmd):
    return subprocess.run(cmd, capture_output=True, timeout=300).stdout


def main():
    out = {"scan": {}, "dump": {}}
    files = {}
    for name, kw in CORPORA.items():
        f = tempfile.NamedTemporaryFile(suffix=".txt", delete=False)
        f.write(_corpus.make_text(**kw)); f.close()
        files[name] = f.name
    for name, corpus, pat, rargs, kw in SCAN_CASES:
        cnt = run([REF + "/agrep", "-V0", "-c"] + rargs + [pat, files[corpus]]).strip()
        rec = {"corpus": corpus, "pattern": pat, "ref_args": rargs, "api": kw, "count": int(cnt) if cnt else 0}
        if "-n" in rargs:
            o = run([REF + "/agrep", "-V0"] + rargs + [pat, files[corpus]])
            rec["ordinals"] = [int(m.group(1)) for m in re.finditer(rb"^(\d+): ", o, re.M)]
        out["scan"][name] = rec
    for pat, rargs in DUMP_CASES:
        o = run([REF + "/memagrep_cli", "-dump", files["nl"], "-V0", "-c"] + rargs + [pat]).decode("latin-1")
        d = {"pattern": pat, "ref_args": rargs, "mask": {}}
        for line in o.splitlines():
            if line.startswith("M="):
                d.update({k: int(v) for k, v in (kv.split("=") for kv in line.split())})
            elif line.startswith("Init0="):
                d.update({k: int(v, 16) for k, v in (kv.split("=") for kv in line.split())})
            elif line.startswith("Mask["):
                m = re.match(r"Mask\[(\d+)\]=([0-9a-f]+)", line)
                d["mask"][m.group(1)] = int(m.group(2), 16)
        out["dump"][pat + " " + " ".join(rargs)] = d
    for p in files.values():
        os.unlink(p)
    json.dump(out, open(os.path.join(HERE, "reference_vectors.json"), "w"), indent=1, sort_keys=True)
    # the -i translation table as the reference ends up with it: CP[ISO-8859-1].lower_1 (agrep.c:2769-2792), identity
    # again for every byte that serves as a metasymbol (agrep.c:2835-2848)
    import ctypes
    lib = ctypes.CDLL(REF + "/libagrepref.so")
    class E(ctypes.Structure):
        _fields_ = [("l1", ctypes.c_ubyte), ("l2", ctypes.c_ubyte), ("l3", ctypes.c_ubyte), ("m", ctypes.c_int)]
    CP = ((E * 257) * 3).in_dll(lib, "CP")
    json.dump([CP[2][i].l1 if CP[2][i].m == 0 else i for i in range(256)], open(os.path.join(HERE, "lut_lower1.json"), "w"))
    print("wrote", len(out["scan"]), "scan cases,", len(out["dump"]), "dumps")
    # the stand-alone command line's cases (tests/test_gpu_dropin.py): exit status and stdout digest, run in the files'
    # directory so that the file names printed do not depend on where it ran
    import hashlib
    import test_gpu_dropin as tg
    cli = {}
    with tempfile.TemporaryDirectory() as d:
        tg.make_files(d)
        for args, names in tg.CLI_CASES:
            p = subprocess.run([REF + "/agrep"] + args + names, capture_output=True, timeout=300, stdin=subprocess.DEVNULL, cwd=d)
            cli[" ".join(args + names)] = {"rc": p.returncode, "bytes": len(p.stdout), "sha256": hashlib.sha256(p.stdout).hexdigest()}
    json.dump(cli, open(os.path.join(HERE, "cli_stdout.json"), "w"), indent=1, sort_keys=True)
    # tests/test_oracle_vs_reference.py asks the reference binary itself and stores its answers (reference_answers.json.gz):
    # every test of the module must have run and passed before the new answers replace the committed ones
    answers = os.path.join(HERE, "reference_answers.json.gz")
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join(os.path.dirname(HERE), "test_oracle_vs_reference.py")],
                   env=dict(os.environ, AGB_RECORD_REFERENCE=REF + "/agrep"), check=True)
    os.replace(answers + ".new", answers)


if __name__ == "__main__":
    main()
