"""The GEMM check of gemm_ref.py on the CPU: it accepts an fp32 emulation of the kernel's arithmetic (one rounding per
k16 step, the fp32 epilogue, the Abramowitz-Stegun GELU, round-to-nearest bf16) and rejects each of six subtle faults,
most of which the relative-L2 thresholds the GEMM tests used before accept."""
import functools

import pytest
import torch
from gemm_ref import bf16_interval, check, check_all, reference
from kernel_checks import BF16, F32, rel_l2

M, N = 200, 512                 # two 128-row m-blocks, the second ragged (last valid row 199); two 256-column tiles


def operands(K, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(BF16)
    b = (0.05 * torch.randn(N, K, generator=g)).to(BF16)
    bias = 0.1 * torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g)
    return a, b, bias, res


def accumulate(a, b):
    """fp32 accumulator rounded once per k16 step (each step's 16 products summed exactly)."""
    acc = torch.zeros(a.shape[0], b.shape[0], dtype=F32)
    for k in range(0, a.shape[1], 16):
        acc = (acc.double() + a[:, k:k + 16].double() @ b[:, k:k + 16].double().t()).float()
    return acc


def gelu_as(v, tanh=False):
    """GELU and GELU' in fp32: Phi through Abramowitz-Stegun 7.1.26 as the kernel does, or the tanh approximation."""
    if tanh:
        c = (2 / torch.pi) ** 0.5
        th = torch.tanh(c * (v + 0.044715 * v ** 3))
        return 0.5 * v * (1 + th), 0.5 * (1 + th) + 0.5 * v * (1 - th * th) * c * (1 + 3 * 0.044715 * v * v)
    t = 1 / (1 + 0.3275911 / 2 ** 0.5 * v.abs())
    poly = t * (0.254829592 + t * (-0.284496736 + t * (1.421413741 + t * (-1.453152027 + t * 1.061405429))))
    e = torch.exp(-0.5 * v * v)
    phi = 0.5 + 0.5 * torch.sign(v) * (1 - poly * e)
    return v * phi, phi + v * e * 0.3989422804014327


def to_bf16(x, truncate=False):
    if not truncate:
        return x.to(BF16)
    return (x.view(torch.int32) >> 16).to(torch.int16).view(BF16)


def emulate(a, b, bias, tanh=False, truncate=False, bias_mask=None):
    """act 3 (out = GELU(v), out2 = GELU'(v), bf16) of v = A B^T + bias."""
    bb = bias if bias_mask is None else bias * bias_mask
    v = (accumulate(a, b).double() + bb.double()).float()
    g, d = gelu_as(v, tanh)
    return {"out": to_bf16(g, truncate), "out2": to_bf16(d, truncate)}


@functools.lru_cache(maxsize=None)
def case(K):
    a, b, bias, res = operands(K)
    return (a, b, bias, res), emulate(a, b, bias), reference(a, b, bias=bias, act=3, out2=True)


@pytest.mark.parametrize("K", [768, 3072])
def test_the_check_accepts_the_kernels_arithmetic(K):
    (a, b, bias, res), got, want = case(K)
    check_all(f"emulated act 3 K={K}", got, want)
    # bias + fp32 residual -> fp32 (out_mode 1)
    out32 = ((accumulate(a, b).double() + bias.double()).float().double() + res.double()).float()
    check(f"emulated residual K={K}", out32, reference(a, b, bias=bias, residual=res)["out"])


def step_outside(out, want):
    """One element one bf16 step past the upper end of its interval."""
    _, hi = bf16_interval(*want)
    i = int(want[0].abs().argmax())
    bits = hi.flatten()[i:i + 1].view(torch.int16)
    nxt = (bits + 1 if hi.flatten()[i] > 0 else bits - 1).view(BF16)
    out = out.clone()
    out.view(-1)[i] = nxt[0]
    return out


def mutant(kind):
    (a, b, bias, _), good, want = case(768)
    got = {k: v.clone() for k, v in good.items()}
    if kind == "one step outside":
        got["out"] = step_outside(got["out"], want["out"])
    elif kind == "bias left out of one tile":
        mask = torch.ones(M, N)
        mask[:128, 256:] = 0
        v = (accumulate(a, b).double() + (bias * mask).double()).float()
        g, d = gelu_as(v)
        got = {"out": g.to(BF16), "out2": d.to(BF16)}
    elif kind == "ragged last row repeats the row above":
        for t in got.values():
            t[M - 1] = t[M - 2]
    elif kind == "tanh GELU":
        got = emulate(a, b, bias, tanh=True)
    elif kind == "truncating bf16 conversion":
        got = emulate(a, b, bias, truncate=True)
    elif kind == "8-column group from its neighbour":
        for t in got.values():
            t[:128, 264:272] = t[:128, 256:264]
    return got, want


MUTANTS = ["one step outside", "bias left out of one tile", "ragged last row repeats the row above", "tanh GELU",
           "truncating bf16 conversion", "8-column group from its neighbour"]


@pytest.mark.parametrize("kind", MUTANTS)
def test_the_check_rejects_a_subtle_fault(kind):
    got, want = mutant(kind)
    passes_rel_l2 = all(rel_l2(got[k], want[k][0]) < 4e-3 for k in got)
    print(f"[mutant] {kind}: {'accepted' if passes_rel_l2 else 'rejected'} by the rel-L2 < 4e-3 threshold")
    with pytest.raises(AssertionError):
        check_all(f"mutant: {kind}", got, want)
