"""Multi-GPU explicit subscriptions under pytest: launches tests/run_multigpu_subs.py with one rank per GPU (2, and 3 when the box has
them).  Skipped on boxes with fewer GPUs."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpus():
    import torch

    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_subscriptions_match_a_whole_world_engine(world):
    n = _gpus()
    if n < world:
        pytest.skip("needs %d GPUs, this box has %d" % (world, n))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(29680 + 13 * world), os.path.join(ROOT, "tests", "run_multigpu_subs.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    sys.stdout.write(out.stdout[-6000:])
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "multi-GPU subscriptions OK" in out.stdout
