"""Spatial attention for large frames (space_attn_long_*, csrc/space_attention.cu): kernel times, and the 16-frame
training step at 224 to 384 px.

    python tools/bench_space_attn_long.py [--iters 30] [--steps 5] [--batch 8] [--json out.json]

Kernels: B = 8 clips x T = 16 frames x H = 12 heads (a training step's attention), N = 196 (the existing kernel,
divided_attn_* mode 1, which the tower runs there, and the new one on the same inputs), 256, 400, 576 and 1024 patches
per frame.  Forward and backward are timed separately with CUDA events over `--iters` launches after a warm-up.
TFLOP/s are algorithmic: 4 * 64 * (N + 1) FLOP per query row and head forward (two products over the N + 1 keys of its
group), 10 * 64 * (N + 1) backward (five), over the B * H * T * N patch queries; the share is of the 989 TFLOP/s dense
bf16 figure of the H100 SXM data sheet.

Step: FrozenInTime (TimeSformer-B, 16 frames, DistilBERT, 16-token captions) forward + EgoNCE + backward, `--batch`
clips, at 224, 256, 320 and 384 px; clips/s over `--steps` timed steps after two warm-up steps, then one more step
with the per-launch probes of ops.profile on: the attention kernels' time (time and space, forward and backward) over
the unprofiled step time is the attention's share.  The card name, power limit and SM clocks are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egovlp_b200 import ops  # noqa: E402

PEAK_BF16 = 989e12


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
        return r.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name()


def time_ms(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_case(N, iters, B=8, T=16, H=12, old=False):
    S, D = 1 + T * N, 64 * H
    g = torch.Generator(device="cuda").manual_seed(N)
    qkv = torch.randn(B * S, 3 * D, generator=g, device="cuda")
    qkv[:, :D] *= 0.125
    qkv = qkv.to(torch.bfloat16)
    dout = torch.randn(B * S, D, generator=g, device="cuda").to(torch.bfloat16)
    if old:
        fwd = lambda: ops.divided_attn_fwd(qkv, B, T, N, H, 1)                           # noqa: E731
        out, lse = fwd()
        bwd = lambda: ops.divided_attn_bwd(qkv, out, dout, lse, B, T, N, H, 1, 0.125)    # noqa: E731
    else:
        fwd = lambda: ops.space_attn_long_fwd(qkv, B, T, N, H)                           # noqa: E731
        out, lse = fwd()
        bwd = lambda: ops.space_attn_long_bwd(qkv, out, dout, lse, B, T, N, H, 0.125)    # noqa: E731
    tf, tb = time_ms(fwd, iters), time_ms(bwd, iters)
    rows = B * H * T * N
    ff, fb = 4 * 64 * (N + 1) * rows, 10 * 64 * (N + 1) * rows
    res = {"kernel": "divided_attn (existing)" if old else "space_attn_long", "B": B, "T": T, "N": N, "H": H,
           "fwd_ms": tf, "bwd_ms": tb, "fwd_tflops": ff / tf / 1e9, "bwd_tflops": fb / tb / 1e9}
    res["fwd_share"], res["bwd_share"] = res["fwd_tflops"] * 1e12 / PEAK_BF16, res["bwd_tflops"] * 1e12 / PEAK_BF16
    return res


def step_case(img, batch, steps, T=16, L=16):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.loss import EgoNCE
    from egovlp_b200.model.model import FrozenInTime
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": T,
                        "pretrained": True, "time_init": "zeros", "img_size": img},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(img=img, num_frames=T), seed=0), strict=True)
    net.cuda()
    data = {"video": syn.synthetic_video(batch, T, seed=1, img=img).cuda(),
            "text": {k: v.cuda() for k, v in syn.synthetic_text(batch, L, seed=1, ragged=True).items()}}
    verb, noun = [t.cuda() for t in syn.synthetic_tags(batch, seed=1)]
    loss_fn = EgoNCE()

    def step():
        net.zero_grad(set_to_none=True)
        t, v = net(data)
        loss_fn.fused(t, v, verb, noun).backward()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    step_ms = (time.perf_counter() - t0) * 1e3 / steps
    ops.profile(True)
    step()
    prof = ops.profile(False)
    attn_ms = sum(ms for k, (_, ms, _) in prof.items() if k.startswith("attn_"))
    gemm_flops, gemm_ms, _ = prof.get("gemm", (0.0, 0.0, 0))
    res = {"img": img, "T": T, "batch": batch, "N": (img // 16) ** 2, "step_ms": step_ms,
           "clips_per_s": batch * 1e3 / step_ms, "attn_ms_profiled": attn_ms, "attn_share": attn_ms / step_ms,
           "gemm_ms_profiled": gemm_ms, "gemm_tflops": gemm_flops / max(gemm_ms, 1e-9) / 1e9,
           "attn_kinds_ms": {k: round(ms, 3) for k, (_, ms, _) in prof.items() if k.startswith("attn_")},
           "max_mem_gb": torch.cuda.max_memory_allocated() / 1e9}
    del net, data
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--sizes", default="224,256,320,384")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    warnings.simplefilter("ignore")
    assert torch.cuda.is_available(), "this benchmark measures the GPU: no CUDA device found"
    res = {"card_before": card(), "kernels": [], "steps": []}
    print("card:", res["card_before"], flush=True)
    for N, old in ((196, True), (196, False), (256, False), (400, False), (576, False), (1024, False)):
        r = kernel_case(N, args.iters, old=old)
        res["kernels"].append(r)
        print(json.dumps(r), flush=True)
    for img in (int(s) for s in args.sizes.split(",")):
        r = step_case(img, args.batch, args.steps)
        res["steps"].append(r)
        print(json.dumps(r), flush=True)
    res["card_after"] = card()
    print("card:", res["card_after"], flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
