"""Tensor parallelism over NCCL (needs >= 2 GPUs on the box; skipped otherwise)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("eager", ["1", "0"])
def test_tp2_engine_matches_oracle(eager):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    env = dict(os.environ, TP_EAGER=eager)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(29555 + int(eager)), os.path.join(ROOT, "tests", "tp_worker.py")]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "TP_RESULT" in r.stdout and '"ok": true' in r.stdout


def test_tp2_spawned_by_the_engine():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "tp_spawn_check.py")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "SPAWN_RESULT" in r.stdout and '"ok": true' in r.stdout


def test_tp2_on_one_gpu_over_gloo():
    """Runs on EVERY GPU box, including single-GPU ones: two tensor-parallel ranks time-slice GPU 0 and reduce through
    gloo (eager).  Covers the head / MLP-column / vocabulary sharding, the (score, token) key combine and the SPMD
    engine replicas end to end against the oracle.  The exchange kernel over real NVLink needs two GPUs (tests above and
    the parity leg of bench.py at N > 1); its data path and flag protocol run on one GPU in test_gpu_tp_exchange.py."""
    env = dict(os.environ, TP_EAGER="1", B200_TP_BACKEND="gloo", B200_TP_ONE_DEVICE="1", B200_TP_ALLREDUCE="nccl")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29557", os.path.join(ROOT, "tests", "tp_worker.py")]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "TP_RESULT" in r.stdout and '"ok": true' in r.stdout and '"backend": "gloo"' in r.stdout
