"""GPU, >= 2 devices: a ray-sharded render over a background map (DESIGN §4.16) -- the fused peer-store gather and the NCCL all_gather --
equals the 1-GPU render of the whole batch with the same map, bit for bit on every rank, rays that miss the mesh included
(tools/peer_gather_check.py --background).  Skipped on a single-GPU box."""
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_sharded_render_over_a_background_map_equals_single_gpu_render():
    n = min(torch.cuda.device_count(), 8)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
                          "--master-port", "29613", str(ROOT / "tools" / "peer_gather_check.py"), "--background"], capture_output=True,
                         text=True, timeout=600, cwd=str(ROOT))
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert "peer_gather_check ok" in out.stdout and "over a background map" in out.stdout
