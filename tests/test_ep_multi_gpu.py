"""Expert-parallel MoE block on real peer memory: needs >= 2 GPUs (skipped otherwise)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world", [2, 4, 8])
def test_ep_block_on_peer_memory(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29500 + world
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "ep_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("EP block OK") == world, r.stdout[-3000:]
