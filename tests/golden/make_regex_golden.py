#!/usr/bin/env python3
"""Records tests/golden/regex_answers.json.gz from the UNMODIFIED reference (oracle/_ref/agrep, built by oracle/Makefile
from the reference sources).  Run where oracle/_ref exists:  python tests/golden/make_regex_golden.py
tests/test_regex_vs_reference.py asks the reference binary itself; every test of the module must have run and passed
before the new answers replace the committed ones (the scheme of make_golden.py).  Also records the stand-alone command
line's stdout digests (regex_cli_stdout.json).  The other golden files are not touched."""
import hashlib, json, os, subprocess, sys, tempfile
HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref")


def main():
    answers = os.path.join(HERE, "regex_answers.json.gz")
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join(os.path.dirname(HERE), "test_regex_vs_reference.py")],
                   env=dict(os.environ, AGB_RECORD_REFERENCE=REF + "/agrep"), check=True)
    os.replace(answers + ".new", answers)
    # the stand-alone command line's cases (tests/test_gpu_regex.py): exit status and stdout digest, run in the file's
    # directory so that the output does not depend on where it ran
    sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
    import test_gpu_regex as tg
    cli = {}
    with tempfile.TemporaryDirectory() as d:
        tg.cli_files(d)
        for args in tg.CLI_CASES:
            cli[" ".join(args)] = tg.run_cli(REF + "/agrep", args, d)
    json.dump(cli, open(os.path.join(HERE, "regex_cli_stdout.json"), "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
