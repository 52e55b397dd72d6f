"""clips/s of the Ego4D OSCC / PNR fine-tuning step on one GPU (trainer/trainer_oscc.py:333-341,
trainer/trainer_pnr.py:341-351): zero_grad -> FrozenInTime(data, video_only=True) with the 2- / 16-wide head -> gather
(identity at world 1, local-slice backward) -> CrossEntropy (PNR: the trainer's mean(state) * CE expression) -> backward ->
fused AdamW, timed between CUDA events after the warm-up steps.

    python tools/bench_finetune.py --task oscc|pnr --batch N [--steps K] [--warmup W] [--dump-outputs DIR]

Prints ONE JSON line: clips/s, algorithmic FLOPs from the shapes (3 F_video - F_patch: the backward costs two forwards
except the patch embedding's input gradient, which the video does not need), the same step in eager PyTorch through the
oracle on the same GPU (fp32 and bf16 autocast), and the card name, power limit and median SM clock of this run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (FLOP model and SM clock sampler of the headline benchmark)

TASKS = {"oscc": 2, "pnr": 16}            # projection_dim of configs/ft/oscc.json, configs/ft/pnr.json
FRAMES = 16


def video_flops(B, T, C):
    """-> (F_video, F_patch) of one forward: the tower of bench.flops_per_clip with a C-wide head instead of 256."""
    _, video, _ = bench.flops_per_clip(T, 0)
    patch = 2 * T * 196 * 768 * 768
    return B * (video - 2 * 768 * 256 + 2 * 768 * C), B * patch


def inputs(task, B, device):
    from egovlp_b200 import synthetic as syn
    g = torch.Generator().manual_seed(5)
    video = syn.synthetic_video(B, FRAMES, seed=5).to(device)
    state = torch.randint(0, 2, (B,), generator=g).to(device)
    labels = torch.zeros(B, 16)
    labels[torch.arange(B), torch.randint(0, 16, (B,), generator=g)] = 1.0
    return video, state, labels.to(device)


def step_loss(task, scores, state, labels, crit):
    if task == "oscc":
        return crit(scores, state)
    return torch.mean(state.T * crit(scores.squeeze(dim=-1), torch.argmax(labels.long(), dim=1)))


def timed(step, steps, warmup, sampler=None):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    if sampler is not None:
        sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / steps, out


def ours(task, B, steps, warmup, device, sampler):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.distributed import AllGatherLocalGrad
    from egovlp_b200.model.loss import CrossEntropy
    from egovlp_b200.model.model import FrozenInTime
    from egovlp_b200.optim import AdamW
    C = TASKS[task]
    net = FrozenInTime(bench_video_params(), {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"},
                       projection_dim=C)
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=FRAMES, proj_dim=C), seed=0))
    net.to(device).train()
    opt = AdamW(net.parameters(), lr=3e-5)
    crit = CrossEntropy()
    video, state, labels = inputs(task, B, device)

    def step():
        opt.zero_grad(set_to_none=True)
        scores = AllGatherLocalGrad.apply(net({"video": video}, video_only=True))
        loss = step_loss(task, scores, AllGatherLocalGrad.apply(state), AllGatherLocalGrad.apply(labels), crit)
        loss.backward()
        opt.step()
        return scores.detach(), loss.detach()

    sec, (scores, loss) = timed(step, steps, warmup, sampler)
    return sec, scores, loss


def bench_video_params():
    return {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": FRAMES, "pretrained": True,
            "time_init": "zeros"}


def eager(task, B, device, autocast, steps=3, warmup=1):
    """The reference's algorithm (oracle port) in eager PyTorch on the same GPU, fp32 or bf16 autocast, with
    torch.optim.AdamW: seconds per step (None if it does not fit)."""
    from egovlp_b200 import synthetic as syn
    from oracle import finetune_port as fp, reference_port as rp
    C = TASKS[task]
    torch.backends.cuda.matmul.allow_tf32 = False
    p = {k: v.to(device).requires_grad_(k.startswith(("video_model.", "vid_proj.")))
         for k, v in syn.seeded_state_dict(syn.model_dims(num_frames=FRAMES, proj_dim=C), seed=0).items()}
    opt = torch.optim.AdamW([v for v in p.values() if v.requires_grad], lr=3e-5)
    video, state, labels = inputs(task, B, device)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            scores = rp.compute_video(video, p)
        scores = scores.float()
        loss = (fp.oscc_step_loss([scores], [state]) if task == "oscc"
                else fp.pnr_step_loss([scores], [labels], [state]))
        loss.backward()
        opt.step()
        return loss.detach()

    try:
        sec, _ = timed(step, steps, warmup)
    except torch.cuda.OutOfMemoryError:
        sec = None
    del p, opt
    torch.cuda.empty_cache()
    return sec


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().split(",")[:2]]
        return name, power
    except (OSError, ValueError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(), None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", choices=sorted(TASKS), default="oscc")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump-outputs", default=None)
    ap.add_argument("--no-eager", action="store_true", help="skip the eager PyTorch comparison")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_finetune.py measures the CUDA path: no CUDA device")
    warmup = max(3, args.warmup)
    device = torch.device("cuda", torch.cuda.current_device())
    sampler = bench.ClockSampler(device.index)          # started after the warm-up: clocks of the timed steps only
    t0 = time.time()
    sec, scores, loss = ours(args.task, args.batch, args.steps, warmup, device, sampler)
    clocks = sampler.stop()
    f_video, f_patch = video_flops(args.batch, FRAMES, TASKS[args.task])
    flops = 3 * f_video - f_patch
    line = {"task": args.task, "projection_dim": TASKS[args.task], "batch": args.batch, "frames": FRAMES,
            "steps": args.steps, "warmup": warmup, "clips_per_s": args.batch / sec, "step_ms": sec * 1e3,
            "flop_per_step": flops, "tflops": flops / sec / 1e12, "loss": loss.item()}
    if not args.no_eager:
        # at most 8 clips: the fp32 oracle keeps every activation of 16-frame clips and 32 of them do not fit in 80 GB
        eb = min(args.batch, 8)
        line["eager_pytorch_same_gpu"] = {"batch": eb}
        for mode, ac in (("fp32", False), ("bf16_autocast", True)):
            s = eager(args.task, eb, device, ac)
            line["eager_pytorch_same_gpu"][mode] = None if s is None else {"clips_per_s": eb / s, "step_ms": s * 1e3}
    name, power = card()
    line.update({"gpu": name, "power_limit": power, "sm_clock_mhz_median": clocks.get("sm_mhz"),
                 "sm_clock_max_mhz": clocks.get("sm_max_mhz"), "throttle_reasons": clocks.get("reasons"),
                 "wall_s": time.time() - t0})
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        torch.save({"scores": scores.cpu(), "loss": loss.cpu()},
                   os.path.join(args.dump_outputs, f"finetune_{args.task}_b{args.batch}.pt"))
    print(json.dumps(line))


if __name__ == "__main__":
    main()
