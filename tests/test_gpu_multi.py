"""Multi-GPU result equality on real devices (VERDICT r01 weak #4): N NCCL ranks, each tracking its shard through the
C ABI, gathered poses == the single-GPU run of the whole job, bit for bit. Needs >= 2 GPUs;
skipped on a 1-GPU machine. The host-side sharding logic alone is covered on CPU by test_sharding_gloo.py."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("which", ["c2", "c3"])
def test_nccl_gathered_poses_equal_single_gpu_run(which):
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least 2 GPUs")
    world = 2
    port = 29600 + (os.getpid() % 300)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "multi", "nccl_pose_equality.py"), "5", which]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "bit-identical" in r.stdout
