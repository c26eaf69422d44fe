"""The view-sharded step with bilateral grids under NCCL on real GPUs (needs >= 2 devices; tests/dp_bilagrid_worker.py holds
the checks)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_view_sharded_bilagrid_step_under_nccl_two_ranks():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    env = dict(os.environ)
    env.pop("OMP_NUM_THREADS", None)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29548", os.path.join(ROOT, "tests", "dp_bilagrid_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "DP_BILAGRID_WORKER_OK" in r.stdout, r.stdout[-3000:] + "\n" + r.stderr[-6000:]
