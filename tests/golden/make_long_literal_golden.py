#!/usr/bin/env python3
"""Records tests/golden/long_literal_answers.json from the UNMODIFIED reference (oracle/_ref/agrep, built by oracle/Makefile
from the reference sources).  Run where oracle/_ref exists:  python tests/golden/make_long_literal_golden.py

Simple literals of 62..255 characters at k = 0, which the reference searches with sgrep()'s monkey() (sgrep.c:1540-1834).
For every case -- a literal, its options, a seeded text -- the file holds what `agrep -c` prints and the byte offsets that
`agrep -b` puts in front of each printed record (the offset of the match inside that record; a record list without -n).
tests/test_long_literal_host.py holds the checker to these answers; CASES and case_text() are shared with it."""
import json, os, re, subprocess, sys, tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "agrep")
GOLDEN = os.path.join(HERE, "long_literal_answers.json")
sys.path.insert(0, os.path.dirname(HERE))
import _corpus  # noqa: E402

LENGTHS = (62, 63, 64, 70, 100, 120, 180, 200, 255)
# (name, agrep arguments, checker / Pattern keywords)
OPTIONS = (("plain", [], {}), ("i", ["-i"], dict(nocase=1)), ("w", ["-w"], dict(wordbound=1)),
           ("d;", ["-d", ";"], dict(delim=";")), ("d@#", ["-d", "@#"], dict(delim="@#")))
CASES = [(m, name, args, kw, final) for m in LENGTHS for name, args, kw in OPTIONS for final in (True, False)]


def literal(m, seed=0):
    """m characters of vocabulary words (letters and spaces: a simple pattern), starting and ending with a letter"""
    import random
    rnd = random.Random(1000 * m + seed)
    s = ""
    while len(s) < m + 1:
        s += rnd.choice(_corpus.VOCAB) + " "
    s = s[:m]
    return s[:-1] + "x" if s.endswith(" ") else s


def case_text(m, kw, final):
    """a seeded text of about 30 KB (under the 48 KiB where -b's offsets are exact, SURVEY 8c(1)) with the literal planted:
    inside a line, in upper case (bm() folds ASCII case always), glued to a letter on the left (not a word under -w), with one
    byte changed at the start, the middle and the end (no match), twice in one record, and in the text's last record"""
    lit = literal(m).encode()
    base = _corpus.make_text(450, seed=77 + m)
    cut = [i for i in range(len(base)) if base[i:i + 1] == b"\n"]
    parts, last = [], 0
    plants = [b" xx " + lit + b" yy", b" " + lit.upper() + b" ", b" a" + lit + b" ",
              b" " + b"#" + lit[1:] + b" ", b" " + lit[:m // 2] + b"#" + lit[m // 2 + 1:] + b" ", b" " + lit[:-1] + b"# ",
              b" " + lit + b" and " + lit + b" "]
    for j, pl in enumerate(plants):
        at = cut[(j + 1) * len(cut) // (len(plants) + 2)]
        parts.append(base[last:at] + pl)
        last = at
    text = b"".join(parts) + base[last:].rstrip(b"\n") + b"\n" + lit
    if kw.get("wordbound"):
        text += b" end"        # (under -w bm() sees its sentinel copy of the pattern behind an unterminated text as a letter)
    if final:
        text += b"\n"
    d = kw.get("delim")
    return text.replace(b"\n", d.encode()) if d else text


def ask(args, data):
    with tempfile.NamedTemporaryFile(suffix=".txt", delete=False) as f:
        f.write(data)
        path = f.name
    try:
        return subprocess.run([REF, "-V0"] + args + [path], capture_output=True, timeout=120)
    finally:
        os.unlink(path)


def answer(m, args, kw, final):
    data = case_text(m, kw, final)
    c = ask(["-c"] + args + [literal(m)], data)
    b = ask(["-b"] + args + [literal(m)], data)
    assert not c.stderr and not b.stderr, (m, args, c.stderr, b.stderr)
    return {"count": int(c.stdout.split()[0]), "offsets": [int(x) for x in re.findall(rb"(\d+)= ", b.stdout)]}


def key(m, name, final):
    return "%d %s %s" % (m, name, "final" if final else "open")


def main():
    out = {key(m, name, final): answer(m, args, kw, final) for m, name, args, kw, final in CASES}
    json.dump(out, open(GOLDEN, "w"), indent=0, sort_keys=True)


if __name__ == "__main__":
    main()
