#!/usr/bin/env python3
"""Records tests/golden/regex_levels_cli_stdout.json from the UNMODIFIED reference (oracle/_ref/agrep, built by
oracle/Makefile from the reference sources): exit status and stdout digest of every -B case of the stand-alone command
line in tests/test_gpu_regex_levels.py, run in the files' directory so that the output does not depend on where it ran.
Run where oracle/_ref exists:  python tests/golden/make_regex_levels_golden.py
The other golden files are not touched."""
import json, os, sys, tempfile
HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref")


def main():
    sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
    import test_gpu_regex_levels as tl
    cli = {}
    with tempfile.TemporaryDirectory() as d:
        tl.cli_files(d)
        for args, files in tl.CLI_CASES:
            cli[tl.cli_key(args, files)] = tl.run_cli(REF + "/agrep", args, files, d)
    json.dump(cli, open(os.path.join(HERE, "regex_levels_cli_stdout.json"), "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
