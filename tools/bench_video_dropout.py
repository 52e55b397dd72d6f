"""Cost of the video tower's training dropouts: the cfg3 training step (32 clips of 16 frames, L = 16, EgoNCE, fused
AdamW, seeded synthetic inputs) with drop_rate = drop_path_rate = 0.1 against all rates 0, in both activation modes
(default and `set_grad_checkpointing`), on one GPU.

    python tools/bench_video_dropout.py [--batch 32] [--steps 8] [--warmup 3] [--rounds 2]

The four cases run alternately in one process, `--rounds` times.  Prints one JSON line per case: clips/s between CUDA
events after the warm-up steps, then the GEMM launches of one further step timed by CUDA events (ops.profile_gemm), with
the card name, power limit and median SM clock of the run.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (SM clock sampler of the headline benchmark)
from bench_finetune import card  # noqa: E402

FRAMES, TEXT_LEN = 16, 16


def set_rates(tower, drop, path):
    """The rates SpaceTimeTransformer(drop_rate=drop, drop_path_rate=path) would have, set on a built tower."""
    from egovlp_b200.model.video_transformer import DropPath
    tower.pos_drop.p = drop
    dpr = torch.linspace(0, path, len(tower.blocks))
    for blk, r in zip(tower.blocks, dpr):
        blk.timeattn.proj_drop.p = blk.attn.proj_drop.p = blk.mlp.drop.p = drop
        blk.drop_path = DropPath(r.item()) if r.item() > 0 else torch.nn.Identity()


def run_case(net, opt, data, B, rates, low, steps, warmup):
    from egovlp_b200 import ops
    from egovlp_b200.distributed import egoclip_step_loss
    from egovlp_b200.model.loss import EgoNCE
    set_rates(net.video_model, *rates)
    net.video_model.set_grad_checkpointing(low)
    loss_fn = EgoNCE()

    def step():
        opt.zero_grad(set_to_none=True)
        loss = egoclip_step_loss(net, loss_fn, data)
        loss.backward()
        opt.step()
        return loss

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    ms = e0.elapsed_time(e1)
    ops.profile_gemm(True)
    step()
    flops, gemm_ms, launches = ops.profile_gemm(False)
    return {"drop_rate": rates[0], "drop_path_rate": rates[1], "low_memory": low, "batch": B,
            "clips_per_s": B * steps / (ms / 1e3), "ms_per_step": ms / steps, "gemm_ms_per_step": gemm_ms,
            "gemm_launches": launches, "gemm_tflops": flops / (gemm_ms / 1e3) / 1e12, "loss": loss.item(),
            "steps": steps, "warmup": warmup, "sm_clock_mhz_median": clocks.get("sm_mhz")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    assert args.steps >= 8 and args.warmup >= 3, "time at least 8 steps after 3 warm-up steps"
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.model import FrozenInTime
    from egovlp_b200.optim import AdamW
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    device = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": FRAMES,
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=FRAMES), seed=0), strict=True)
    net.to(device)
    opt = AdamW(net.parameters(), lr=3e-5)
    B = args.batch
    txt = syn.synthetic_text(B, TEXT_LEN, seed=0)
    verb, noun = syn.synthetic_tags(B, seed=0)
    data = {"video": syn.synthetic_video(B, FRAMES, seed=0).to(device),
            "text": {k: v.to(device) for k, v in txt.items()}, "verb_vec": verb.to(device), "noun_vec": noun.to(device)}
    name, power = card()
    for _ in range(args.rounds):
        for low in (False, True):
            for rates in ((0.0, 0.0), (0.1, 0.1)):
                line = run_case(net, opt, data, B, rates, low, args.steps, args.warmup)
                line.update({"gpu": name, "power_limit": power})
                print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
