"""Node-striped multi-GPU parity as pytest cases (skipped below 2 GPUs): torchrun starts one rank per GPU on
tests/mgpu_check.py, every rank compares its outcome with the CPU oracle (bindings, statuses, visit order, queue tables,
its own node rows) for allocate workloads, whole five-action cycles and topology gangs."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("world", [2, 4, 8])
def test_striped_gpus_match_the_oracle(world):
    if _n_gpus() < world:
        pytest.skip(f"needs {world} GPUs")
    env = dict(os.environ)
    port = 29500 + world * 7
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "mgpu_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    tail = (out.stdout + out.stderr)[-3000:]
    assert out.returncode == 0 and "MGPU PARITY PASS" in out.stdout, tail
