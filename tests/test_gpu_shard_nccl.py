"""agb_scan_sharded over NCCL with one process per GPU, records straddling the cuts, against the oracle on the whole text
(tests/shard_nccl_worker.py).  Needs as many GPUs as ranks and skips otherwise; with one GPU the cut rule is covered by
tests/test_gpu_shard.py and the communicator by its world-of-one case."""
import os, socket, subprocess, sys
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_scan_over_nccl(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                        "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "shard_nccl_worker.py")],
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "shard_nccl_worker ok" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
