"""Micro-benchmark of the wgmma GEMM on the shapes of the 16-frame step (B=64 -> M=200768 tokens)."""
import json
import sys
import os
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egovlp_b200 import ops

M = int(os.environ.get("M", 200768))
dev = "cuda"
peaks = json.load(open("MEASURED_PEAKS.json")) if os.path.exists("MEASURED_PEAKS.json") else {"bf16_tflops": 1590.0}


def t(fn, iters=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def rnd(*shape, dt=torch.bfloat16):
    return (torch.randn(*shape, device=dev) * 0.05).to(dt)


rows = []
for name, N, K in [("qkv", 2304, 768), ("proj", 768, 768), ("fc1", 3072, 768), ("fc2", 768, 3072)]:
    a, w = rnd(M, K), rnd(N, K)
    bias = rnd(N, dt=torch.float32)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    ms = t(lambda: ops.gemm(a, w, out, bias=bias))
    ref = t(lambda: torch.nn.functional.linear(a, w, bias.to(torch.bfloat16)))
    fl = 2.0 * M * N * K
    rows.append((f"fwd {name} bias", ms, fl / ms / 1e9, ref))
    if name == "fc1":
        u = torch.empty_like(out)
        ms = t(lambda: ops.gemm(a, w, out, bias=bias, act=1, out2=u))
        rows.append((f"fwd {name} bias+gelu+preact", ms, fl / ms / 1e9, ref))
    if name in ("proj", "fc2"):
        res = rnd(M, N, dt=torch.float32)
        o32 = torch.empty(M, N, device=dev, dtype=torch.float32)
        ms = t(lambda: ops.gemm(a, w, o32, bias=bias, residual=res))
        rows.append((f"fwd {name} bias+res->f32", ms, fl / ms / 1e9, ref))
    # dgrad: dx[M,K] = dy[M,N] @ W[N,K]
    dy = rnd(M, N)
    dx = torch.empty(M, K, device=dev, dtype=torch.float32 if name != "fc2" else torch.bfloat16)
    ms = t(lambda: ops.gemm(dy, w, dx, b_mn=True))
    ref = t(lambda: torch.matmul(dy, w))
    rows.append((f"dgrad {name}", ms, fl / ms / 1e9, ref))
    # wgrad: dW[N,K] += dy^T a
    dw = torch.zeros(N, K, device=dev, dtype=torch.float32)
    for split in (4, 8, 16):
        ms = t(lambda: ops.gemm(dy, a, dw, a_mn=True, b_mn=True, accumulate=True, split_k=split))
        rows.append((f"wgrad {name} split{split}", ms, fl / ms / 1e9, None))
    ref = t(lambda: torch.matmul(dy.t(), a))
    rows[-1] = rows[-1][:3] + (ref,)

print(f"M={M}  peak(burst)={peaks['bf16_tflops']} TF/s")
for name, ms, tf, ref in rows:
    extra = f"  cublas {ref:.3f} ms" if ref else ""
    print(f"{name:32s} {ms:8.3f} ms  {tf:8.1f} TF/s  {tf / peaks['bf16_tflops'] * 100:5.1f}%{extra}")
