"""NCCL parity of the data-parallel step (tests/ddp_check.py under torch.distributed.run): the fused packed-gather step
and the reference trainer's literal call sequence agree with each other and with the single-process full-batch loss /
gradients.  World size 1 runs on any GPU box; world size 2 needs two GPUs."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(world, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "ddp_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_trainer_sequence_equals_fused_step_world1():
    out = _run(1, 29541)
    assert '"ok": true' in out, out[-2000:]


def test_two_rank_nccl_loss_and_gradients():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = _run(2, 29542)
    assert '"ok": true' in out, out[-2000:]
