"""Multi-GPU parity (needs >= 2 GPUs on the box; skipped otherwise): the row-sharded local_laplacian must equal
the single-GPU filter bit for bit on every band."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpu():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("world,w,band_h", [(1, 1000, 640), (2, 1000, 640), (2, 333, 517)])  # (world 1: the sharded code path alone)
def test_sharded_local_laplacian_matches_single_gpu(world, w, band_h):
    if _ngpu() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
           "127.0.0.1", "--master-port", "29531", os.path.join(ROOT, "tools", "dist_check.py"), str(w), str(band_h)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=240)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "mismatches=0" in out.stdout


def test_input_halo_filters_sharded_match_single_gpu():
    """blur / nl_means / stencil_chain / bilateral_grid / camera_pipe row-sharded over 2 GPUs (NCCL row exchange +
    the ordinary filter on the extended band) equal the whole-frame call on one GPU (bit for bit for the integer
    pipelines, 1e-4 relative for the float ones)."""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29532", os.path.join(ROOT, "tools", "dist_rows_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=240)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "mismatches=0" in out.stdout
