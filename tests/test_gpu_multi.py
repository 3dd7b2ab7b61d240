"""Multi-GPU data-parallel parity (needs >= 2 GPUs; skipped on single-GPU boxes)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world,precision", [(2, "fp32"), (2, "tf32x3"), (4, "tf32x3"), (8, "tf32x3"), (8, "fp32")])
def test_data_parallel_ranks_match_single_big_batch_oracle(world, precision):
    """N ranks (own shard, own uniforms, rank-order gradient sum over peer memory) == ONE oracle learner on the
    concatenated batches; at 4 / 8 ranks the in-kernel rank-order sum is a different code path than at 2."""
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    env = dict(os.environ, D4PG_PRECISION=precision)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % world, "--master-addr", "127.0.0.1",
           "--master-port", str(29517 + world), os.path.join(ROOT, "tests", "dp_worker.py")]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and "DP_OK" in r.stdout, r.stdout[-3000:]


@pytest.mark.parametrize("world", [2, 4, 8])
def test_data_parallel_device_sampling_replicas_stay_identical(world):
    """The benchmark's DP configuration (device sampling + prefetch + fused peer-memory gradient exchange, 3xTF32 wgmma)."""
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    env = dict(os.environ, D4PG_PRECISION="tf32x3", D4PG_DP_MODE="device")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % world, "--master-addr", "127.0.0.1",
           "--master-port", str(29537 + world), os.path.join(ROOT, "tests", "dp_worker.py")]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and "DP_OK" in r.stdout and "mode=device" in r.stdout, r.stdout[-3000:]


@pytest.mark.parametrize("world,mode", [(2, "mc2"), (8, "mc2"), (2, "pull"), (8, "pull")])
def test_data_parallel_exchange_modes(world, mode):
    """The non-default gradient exchange shapes against the same single-big-batch oracle: "mc2" = two-phase in-switch
    reduction (multimem.ld_reduce of 1/N + multimem.st broadcast; falls back to the peer-memory pull when the box has no
    NVLS multicast), "pull" = rank-order sum over IPC-mapped peer memory."""
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    for dp_mode in ("", "device"):
        env = dict(os.environ, D4PG_PRECISION="tf32x3", D4PG_COMM_MODE=mode, D4PG_DP_MODE=dp_mode)
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % world, "--master-addr", "127.0.0.1",
               "--master-port", str(29557 + world), os.path.join(ROOT, "tests", "dp_worker.py")]
        r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0 and "DP_OK" in r.stdout, r.stdout[-3000:]
