import os, sys, subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    # build the checker (oracle) and, when the reference sources are present, oracle/_ref
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "all"], check=True,
                   stdout=subprocess.DEVNULL)
