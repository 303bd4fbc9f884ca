"""What a levels scan of a regular expression rests on, checked on the host: the checker's (tests/_regex_oracle.py, pinned
to the reference's re()) matching lines at k = 0..4 are nested, so one pass at k gives every line's smallest level <= k;
and every -B case of the stand-alone command line in test_gpu_regex_levels.py has a recorded reference answer."""
import json, os, random
import _regex_oracle as R
import test_regex_vs_reference as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_checker_levels_nested():
    """200 random regexes of corpus words over T.TEXT: the lines found within k errors are among those found within k + 1"""
    rnd = random.Random(606)
    words = sorted({w for w in T.TEXT.decode().split() if w.isalpha() and len(w) >= 3})
    done = grew = 0
    while done < 200:
        p = T.random_regex(rnd, words)
        if not R.is_regex(p.encode()) or len(p) <= 4:
            continue
        nocase = rnd.random() < 0.2
        sets = [{r for r in R.scan(R.compile(p, k=k, nocase=nocase), T.TEXT)[1]} for k in range(5)]
        for k in range(4):
            assert sets[k] <= sets[k + 1], (p, nocase, k)
        grew += sets[4] != sets[0]
        done += 1
    assert grew > 100                                  # the errors do find more lines


def test_cli_cases_have_golden():
    import test_gpu_regex_levels as tl
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "regex_levels_cli_stdout.json")))
    keys = [tl.cli_key(a, f) for a, f in tl.CLI_CASES]
    assert sorted(keys) == sorted(golden)
    for key in keys:
        assert set(golden[key]) == {"rc", "bytes", "sha256"}, key
