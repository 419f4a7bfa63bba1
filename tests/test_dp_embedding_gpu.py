"""N-GPU data-parallel parity of the token-embedding steps (needs >= 2 visible GPUs; skipped on a 1-GPU
box): runs scripts/dp_embedding_parity.py under torchrun with 2 ranks (and 4 when 4 GPUs are visible),
once over the NVLink peer exchange and once over NCCL (LB_DP_NCCL=1). LoraEmbeddingStep (both modes,
eager and captured) and TextualInversionStep after 4 steps on N ranks must equal one process on the
concatenated batch, with the same slot list and bitwise identical replicas."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_GPUS = torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(N_GPUS < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_embedding_steps_on_n_ranks_equal_single_process(world, exchange):
    if world > N_GPUS:
        pytest.skip(f"needs {world} GPUs")
    env = dict(os.environ, LB_DP_NCCL="1" if exchange == "nccl" else "0")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29541 + world + (10 if exchange == "nccl" else 0)),
           os.path.join(ROOT, "scripts", "dp_embedding_parity.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    print(out.stdout)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "dp_embedding_parity OK" in out.stdout
    assert ("exchange=nvlink-peer" if exchange == "peer" else "exchange=nccl") in out.stdout
