#!/usr/bin/env python3
"""Records tests/golden/sticky_delim_answers.json from the UNMODIFIED reference (oracle/_ref/agrep, built by oracle/Makefile
from the reference sources).  Run where oracle/_ref exists:  python tests/golden/make_sticky_delim_golden.py

-p with a record delimiter of two or more bytes: -p makes the delimiter's positions sticky too, so a record closes where
the delimiter's bytes have occurred in order since the last close ("a ... b" closes like "ab" under -d ab).  For every case
-- a delimiter, a pattern with its options, a text -- the file holds what `agrep -c`, `agrep` and `agrep -n` print, their
exit codes and what they print on stderr (-p with -S2 is refused: the insertion cost is 0 then).
CASES and case_text() are shared with the tests that hold the checker and the product to these answers."""
import json, os, random, subprocess, sys, tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "agrep")
GOLDEN = os.path.join(HERE, "sticky_delim_answers.json")
sys.path.insert(0, os.path.dirname(HERE))
import _corpus  # noqa: E402

# (name, -d argument, extra options, checker keywords): overlapping, self-overlapping, run, newline, 8-byte, case-folded
DELIMS = (("ab", "ab", [], {}), ("e_", "e ", [], {}), ("nl2", "$$", [], {}), ("aa", "aa", [], {}), ("aba", "aba", [], {}),
          ("eqd", "=-=", [], {}), ("eight", "the and ", [], {}), ("AB_i", "AB", ["-i"], dict(nocase=1)))
# (name, agrep options, pattern, checker keywords); -p is added to all of them
PATTERNS = (("k0", [], "because", {}), ("k2", ["-2"], "because each", dict(k=2)), ("k6", ["-6"], "government policy", dict(k=6)),
            ("S2", ["-1", "-S2"], "people", dict(k=1, cost_s=2)), ("v", ["-v"], "because", dict(inverse=1)),
            ("w", ["-w"], "the", dict(wordbound=1)), ("hash", [], "wh#ld", {}), ("comma", [], "because,people", {}))
TEXTS = ("base", "starts", "open", "never", "empty")
CASES = [(dn, pn, tn) for dn, *_ in DELIMS for pn, *_ in PATTERNS for tn in TEXTS]
# where the reference prints what the checker does not restate: under -v, after the last record of a text that begins with
# "$$", one more newline (the records, counts and ordinals agree)
NOT_RESTATED = {("nl2", "v", "starts")}


def dbytes(delim):
    """the delimiter's bytes as the records see them ('$' and '^' are newlines in -d)"""
    return delim.replace("$", "\n").replace("^", "\n").encode()


def case_text(dname, tname):
    """about 700 bytes of text with the delimiter's bytes strewn about (alone, in order with other bytes between them, and
    whole), in five forms: as is; starting with the delimiter; ending part way into it without a final newline; with its
    last byte taken out everywhere (it never completes); empty"""
    delim = dict((d[0], d[1]) for d in DELIMS)[dname]
    db = dbytes(delim)
    if tname == "empty":
        return b""
    rnd = random.Random(sum(db) * 7 + len(db))
    t = bytearray(_corpus.make_text(10, seed=40 + len(db)))
    for _ in range(24):
        at = rnd.randrange(len(t))
        t[at:at] = bytes([db[rnd.randrange(len(db))]])
    for _ in range(3):
        at = rnd.randrange(len(t))
        t[at:at] = db
    t = bytes(t)
    if tname == "starts":
        return db + t
    if tname == "open":
        return t.rstrip(b"\n") + db[:(len(db) + 1) // 2]
    if tname == "never":
        last = db[-1:]
        t = t.replace(last, b"").replace(last.upper(), b"").replace(last.lower(), b"")
        return t
    return t


def argv(dname, pname, extra):
    d = next(x for x in DELIMS if x[0] == dname)
    p = next(x for x in PATTERNS if x[0] == pname)
    return ["-p", "-d", d[1]] + d[2] + p[1] + extra + [p[2]]


def checker_kw(dname, pname):
    d = next(x for x in DELIMS if x[0] == dname)
    p = next(x for x in PATTERNS if x[0] == pname)
    kw = dict(ins_free=1, delim=d[1])
    kw.update(d[3]); kw.update(p[3])
    return kw, p[2]


def reference_j(recs, kw, data):
    """the checker's records with j as the reference prints it: asearch0() (k > 4) does not start j at -1 for a text that
    begins with the delimiter (asearch.c:609-612; bitap.c:151-156 and asearch() do), the checker always does"""
    db = dbytes(kw["delim"])
    fix = 1 if kw.get("k", 0) > 4 and data[:len(db)] == db else 0
    return [(b, e, j + fix) for b, e, j in recs]


def ask(args, data):
    with tempfile.NamedTemporaryFile(suffix=".txt", delete=False) as f:
        f.write(data)
        path = f.name
    try:
        return subprocess.run([REF, "-V0"] + args + [path], capture_output=True, timeout=120)
    finally:
        os.unlink(path)


def key(dname, pname, tname):
    return "%s %s %s" % (dname, pname, tname)


def main():
    out = {}
    for dn, pn, tn in CASES:
        data = case_text(dn, tn)
        r = {}
        for name, extra in (("count", ["-c"]), ("plain", []), ("n", ["-n"])):
            p = ask(argv(dn, pn, extra), data)
            r[name] = p.stdout.decode("latin-1")
            r[name + "_rc"] = p.returncode
            r[name + "_err"] = p.stderr.decode("latin-1").replace(REF, "agrep").replace(tempfile.gettempdir(), "")
        r["count"] = None if r["count_err"] else int(r["count"].split()[0])
        out[key(dn, pn, tn)] = r
    json.dump(out, open(GOLDEN, "w"), indent=0, sort_keys=True)


if __name__ == "__main__":
    main()
