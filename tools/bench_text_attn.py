"""Kernel times of the tiled text attention (text_attn_long_*, csrc/text_attention.cu) at B = 32, H = 12.

    python tools/bench_text_attn.py [--iters 50] [--json out.json]

Cases: L = 128, 256, 512 with every key valid, and L = 512 ragged (one caption of 512, the others 2..32 tokens).
Forward and backward are timed separately with CUDA events over `--iters` launches after a warm-up.  TFLOP/s are
algorithmic, counted over the valid 64-key tiles the kernels visit (forward 2 products of 2*64 FLOP per
(query, key, head); backward 5, with the key pass visiting every query tile of a valid key tile), and the share is of
the card's dense bf16 peak (989 TFLOP/s for the H100 SXM data sheet).  At L = 128 the L <= 128 kernel (text_attn_*),
which the tower keeps using there, is timed on the same inputs for the record.  Dropout cost: p_att = 0.1 vs 0.
The card name, power limit and SM clocks are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egovlp_b200 import ops  # noqa: E402

PEAK_BF16 = 989e12
HBM = 3.35e12


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
        return r.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name()


def time_ms(fn, iters):
    for _ in range(5):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def flops(mask, L, H):
    """(forward, backward) FLOPs over the valid key tiles: per sample, queries L x valid tiles x 64 keys."""
    nt = (L + 63) // 64
    tiles = mask.view(mask.shape[0], -1)
    tiles = torch.nn.functional.pad(tiles, (0, nt * 64 - L)).view(mask.shape[0], nt, 64).any(-1).sum().item()
    per = L * 64 * 64 * 2 * H * tiles          # one product of (queries x 64 keys x 64 dims) per valid tile
    return 2 * per, 5 * per


def case(name, mask, L, H, iters, p=0.0, old=False):
    B = mask.shape[0]
    D = 64 * H
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = (torch.randn(B * L, 3 * D, generator=g, device="cuda") * 0.5).bfloat16()
    dout = torch.randn(B * L, D, generator=g, device="cuda").bfloat16()
    out, lse = torch.empty(B * L, D, device="cuda", dtype=torch.bfloat16), torch.empty(B, H, L, device="cuda")
    dq = torch.empty_like(qkv)
    if old:
        fwd = lambda: ops.text_attn_fwd(qkv, mask, out, B, L, H, p, 1, 1)
        bwd = lambda: ops.text_attn_bwd(qkv, mask, dout, dq, B, L, H, 0.125, p, 1, 1)
    else:
        fwd = lambda: ops.text_attn_long_fwd(qkv, mask, out, lse, B, L, H, p, 1, 1)
        fwd()
        bwd = lambda: ops.text_attn_long_bwd(qkv, mask, out, lse, dout, dq, B, L, H, 0.125, p, 1, 1)
    tf, tb = time_ms(fwd, iters), time_ms(bwd, iters)
    ff, fb = flops(mask, L, H)
    io = (B * L * 3 * D + B * L * D) * 2                        # qkv read + out written, bf16
    r = {"case": name, "kernel": "text_attn (L<=128)" if old else "text_attn_long", "B": B, "L": L, "H": H, "p": p,
         "fwd_ms": round(tf, 4), "bwd_ms": round(tb, 4),
         "fwd_tflops": round(ff / tf / 1e9, 1), "bwd_tflops": round(fb / tb / 1e9, 1),
         "fwd_share_bf16_peak": round(ff / tf / 1e9 / (PEAK_BF16 / 1e12), 3),
         "bwd_share_bf16_peak": round(fb / tb / 1e9 / (PEAK_BF16 / 1e12), 3),
         "fwd_share_hbm": round(io / (tf * 1e-3) / HBM, 3)}
    print(json.dumps(r))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_text_attn: needs a CUDA device")
    info = card()
    print("card:", info)
    B, H = 32, 12
    res = []
    for L in (128, 256, 512):
        full = torch.ones(B, L, dtype=torch.int64, device="cuda")
        res.append(case(f"full L={L}", full, L, H, a.iters))
        if L == 128:
            res.append(case(f"full L={L}", full, L, H, a.iters, old=True))
    g = torch.Generator().manual_seed(1)
    lens = torch.randint(2, 33, (B,), generator=g)
    lens[0] = 512
    ragged = (torch.arange(512)[None] < lens[:, None]).long().cuda()
    res.append(case("ragged L=512 (one 512, rest <= 32)", ragged, 512, H, a.iters))
    full = torch.ones(B, 512, dtype=torch.int64, device="cuda")
    res.append(case("full L=512 p_att=0.1", full, 512, H, a.iters, p=0.1))
    res.append(case("full L=128 p_att=0.1", torch.ones(B, 128, dtype=torch.int64, device="cuda"), 128, H, a.iters, p=0.1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": info, "results": res}, f, indent=1)


if __name__ == "__main__":
    main()
