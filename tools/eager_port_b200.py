"""Same-box GPU baseline (SURVEY.md 8d): the oracle port -- the reference's algorithm restated op for op in eager
PyTorch (oracle/reference_port.py) -- timed on the GPU in fp32 (TF32 off / on) and under bf16 autocast, fwd + bwd +
torch AdamW, at the largest per-GPU batch the eager path's fp32 activations allow.  This is a measurement tool, not a
product path: it is the "what the reference's own code path costs on this GPU" denominator quoted in DESIGN.md.

    python tools/eager_port_b200.py [--frames 16] [--batch 8] [--steps 3]
"""
import argparse
import json
import os
import sys
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import reference_port as rp          # noqa: E402
from egovlp_b200 import synthetic as syn         # noqa: E402


def run(T, L, B, steps, mode):
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
    torch.backends.cudnn.allow_tf32 = mode == "tf32"
    dims = syn.model_dims(num_frames=max(T, 4))
    params = {k: v.to(dev).requires_grad_(True) for k, v in syn.seeded_state_dict(dims, seed=0).items()}
    opt = torch.optim.AdamW(list(params.values()), lr=3e-5, eps=1e-6, weight_decay=0.0)
    text = {k: v.to(dev) for k, v in syn.synthetic_text(B, L, seed=0).items()}
    data = {"video": syn.synthetic_video(B, T, seed=0).to(dev), "text": text}
    verb, noun = (x.to(dev) for x in syn.synthetic_tags(B, seed=0))

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=(mode == "bf16-autocast")):
            t, v = rp.frozen_in_time_forward(data, params)
        loss = rp.egonce_loss(rp.sim_matrix(t.float(), v.float()), rp.sim_matrix(verb, verb), rp.sim_matrix(noun, noun))
        loss.backward()
        opt.step()
        return loss

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return {"mode": mode, "batch": B, "frames": T, "text_len": L, "ms_per_step": ms, "clips_per_s": B / ms * 1e3,
            "loss": float(loss), "peak_mem_gb": torch.cuda.max_memory_allocated() / 2**30}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--text-len", type=int, default=16)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = []
    for mode in ("fp32", "tf32", "bf16-autocast"):
        torch.cuda.reset_peak_memory_stats()
        try:
            r = run(a.frames, a.text_len, a.batch, a.steps, mode)
        except torch.cuda.OutOfMemoryError as e:                       # report, do not hide
            r = {"mode": mode, "batch": a.batch, "error": "out of memory: " + str(e)[:120]}
            torch.cuda.empty_cache()
        print(json.dumps(r), flush=True)
        res.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"tool": "tools/eager_port_b200.py", "device": torch.cuda.get_device_name(0), "results": res}, f, indent=1)


if __name__ == "__main__":
    main()
