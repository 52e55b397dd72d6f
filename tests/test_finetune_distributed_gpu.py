"""NCCL parity of the OSCC fine-tuning step (tests/finetune_ddp_check.py under torch.distributed.run): the loss is
identical on all ranks and equal to the single-process full batch, DDP gradient x world equals the full-batch gradient.
World size 1 runs on any GPU box; world size 2 needs two GPUs."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(world, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "finetune_ddp_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_oscc_step_world1():
    out = _run(1, 29561)
    assert '"ok": true' in out, out[-2000:]


def test_oscc_step_two_rank_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = _run(2, 29562)
    assert '"ok": true' in out, out[-2000:]
