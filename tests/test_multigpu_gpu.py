"""GPU tier, needs >= 2 GPUs (skipped otherwise): SyncBatchNorm + DistributedDataParallel on real ranks, one process per
GPU over NCCL / NVLink, against the fp32 oracle on the concatenated batch (tests/_ddp_worker.py). Covers SURVEY.md §8
rows a14 (SyncBN statistics exchange forward and backward) and a15 (DDP gradient averaging) in both operand modes.
Run on a machine with two or more GPUs:  python -m pytest tests/test_multigpu_gpu.py -m gpu ."""
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(world, mode, extra_env=None):
    env = dict(os.environ)
    env.update(extra_env or {})
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
           os.path.join(ROOT, "tests", "_ddp_worker.py"), mode]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    sys.stdout.write(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "multi-rank parity [%s, world %d]: OK" % (mode, world) in r.stdout


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("mode", ["bf16x3", "bf16"])
def test_syncbn_ddp_two_ranks_vs_fp32_oracle(mode):
    _run(2, mode)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_syncbn_nccl_fallback_two_ranks_vs_fp32_oracle():
    """The NCCL all_gather / all_reduce exchange (used where NVLink peer memory is unavailable) gives the same parity."""
    _run(2, "bf16x3", {"SEMSEG_B200_SYNCBN": "nccl"})


@pytest.mark.skipif(torch.cuda.device_count() < 8, reason="needs 8 GPUs")
def test_syncbn_ddp_eight_ranks_vs_fp32_oracle():
    _run(8, "bf16x3")
