"""Tiny driver for ncu: a few launches of the wgmma GEMM on the step's dominant shapes."""
import os
import sys
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egovlp_b200 import ops

M = int(os.environ.get("M", 200768))
which = os.environ.get("WHICH", "qkv")
N, K = {"qkv": (2304, 768), "fc1": (3072, 768), "fc2": (768, 3072), "proj": (768, 768)}[which]
a = (torch.randn(M, K, device="cuda") * 0.05).bfloat16()
w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
bias = torch.randn(N, device="cuda")
out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
res = torch.randn(M, N, device="cuda") if which in ("proj", "fc2") else None
o32 = torch.empty(M, N, device="cuda") if res is not None else None
for _ in range(3):
    if which == "fc1":
        ops.gemm(a, w, out, bias=bias, act=1, out2=torch.empty_like(out))
    elif res is not None:
        ops.gemm(a, w, o32, bias=bias, residual=res)
    else:
        ops.gemm(a, w, out, bias=bias)
torch.cuda.synchronize()
