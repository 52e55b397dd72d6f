"""The bound of tests/text_attention_ref.py for the short-caption attention (text_attn_kernel, csrc/text.cu), checked on
the CPU against an fp32 emulation of the kernel in its own operation order:
  * soundness: with __expf and 1 / x pushed to their worst-case ulps (alternating in sign), every output of every shape
    the GPU test runs stays within the bound;
  * sensitivity: each of seven subtle faults planted in the emulation misses the bound by 10x or more (run with -s for
    the table)."""
import numpy as np
import pytest
import torch
from philox_ref import multiplier, short_attn_keep
from text_attention_ref import case, short_reference, worst_ratios

F32, F64, BF16 = torch.float32, torch.float64, torch.bfloat16


def _ulp(x):
    """One fp32 ulp of each element of x (fp32, finite, non-zero)."""
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), (e - 24).int())


def _fma(a, b, c):
    """fl32(a b + c): the product of two fp32 values is exact in fp64."""
    return (a.double() * b.double() + c.double()).float()


def _butterfly(v):
    """warp_sum over the last dim (32 lanes): v += shfl_xor(v, o), o = 16 .. 1; every lane ends with the same value."""
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lane ^ o]
    return v[..., 0]


def emulate(qkv, dout, mask, B, L, H, q_scale, p=0.0, keep=None, worst=True, fault=None):
    """text_attn_fwd + text_attn_bwd in fp32, statement by statement; -> (out, dqkv) bf16.  worst: __expf and MUFU.RCP
    results moved by their largest error (2 + floor(1.173 |x|) ulp and 1 ulp), in alternating directions."""
    x = qkv.float().view(B, L, 3, H, 64).permute(2, 0, 3, 1, 4)
    q, k, v = x[0], x[1], x[2]
    do = dout.float().view(B, L, H, 64).permute(0, 2, 1, 3)
    valid = mask.bool().clone()
    if fault == "last key padded":
        for b in range(B):
            if int(valid[b].sum()) > 1:                 # a sample with one key would only turn NaN
                valid[b, int(valid[b].nonzero().max())] = False
    valid = valid.view(B, 1, 1, L)
    keep = torch.ones(B, H, L, L, dtype=torch.bool) if keep is None else keep.clone()
    if fault == "keep bit flipped":
        keep[0, 0, 5, 100] = ~keep[0, 0, 5, 100]
    sign = torch.where((torch.arange(L)[:, None] + torch.arange(L)[None]) % 2 == 0, 1.0, -1.0)     # [i, j]
    # scores, softmax
    s = torch.zeros(B, H, L, L)
    for d in range(64):
        s = _fma(q[..., :, None, d], k[..., None, :, d], s)
    s = s.masked_fill(~valid, float("-inf"))
    xa = s - s.amax(-1, keepdim=True)
    e = torch.exp(xa.double()).float()
    if worst:
        n = 2 + torch.floor(1.173 * xa.abs().double().nan_to_num(0.0)).float()
        e = torch.where(e > 0, e + sign * n * _ulp(e), e)
    ep = torch.nn.functional.pad(e, (0, 128 - L)).view(B, H, L, 4, 32)
    acc = torch.zeros(B, H, L, 32)
    for jj in range(4):
        acc = acc + ep[..., jj, :]
    ssum = _butterfly(acc)
    inv = (1.0 / ssum.double()).float()
    if worst:
        inv = inv + torch.where(torch.arange(L) % 2 == 0, 1.0, -1.0) * _ulp(inv)
    P = e * inv[..., None]
    p32 = np.float32(p)
    inv_keep = np.float32(1.0) / (np.float32(1.0) - p32) if p > 0 else np.float32(1.0)
    if worst and p > 0:
        inv_keep = np.nextafter(inv_keep, np.float32(2))
    dropf = torch.where(keep, torch.tensor(float(inv_keep)), torch.tensor(0.0))
    rn = (lambda t: t.to(BF16)) if fault != "bf16 truncation" else (lambda t: (t.view(torch.int32) & ~0xFFFF).view(F32).to(BF16))
    # forward
    pd = P * dropf
    o = torch.zeros(B, H, L, 64)
    for j in range(L):
        o = _fma(pd[..., :, j, None], v[..., None, j, :], o)
    # backward: dV
    pv = P * keep.float() if fault == "dv without 1/(1-p)" else pd
    a = torch.zeros(B, H, L, 64)
    for i in range(L):
        a = _fma(pv[..., i, :, None], do[..., None, i, :], a)
    dv = a
    # dp, delta, dS
    dp = torch.zeros(B, H, L, L)
    for d in range(64):
        dp = _fma(do[..., :, None, d], v[..., None, :, d], dp)
    raw = dp
    dp = dp * dropf
    src = raw if fault == "delta without keep" else dp
    Pp = torch.nn.functional.pad(P, (0, 128 - L)).view(B, H, L, 4, 32)
    sp = torch.nn.functional.pad(src, (0, 128 - L)).view(B, H, L, 4, 32)
    dl = torch.zeros(B, H, L, 32)
    for jj in range(4):
        dl = _fma(Pp[..., jj, :], sp[..., jj, :], dl)
    delta = _butterfly(dl)
    if fault == "dp keys j, j+32 swapped":
        dp = dp.clone()
        dp[4, 0, 7, [0, 32]] = dp[4, 0, 7, [32, 0]]       # sample 4 has 33 valid keys: lane 0's first two
    ds = P * (dp - delta[..., None])
    # dQ, dK
    a = torch.zeros(B, H, L, 64)
    for j in range(L):
        a = _fma(ds[..., :, j, None], k[..., None, j, :], a)
    qs = np.float32(0.125 if fault == "q_scale 0.125" else q_scale)
    dq = a * float(qs)
    a = torch.zeros(B, H, L, 64)
    for i in range(L):
        a = _fma(ds[..., i, :, None], q[..., None, i, :], a)
    dk = a
    rows = lambda t: rn(t.permute(0, 2, 1, 3).reshape(B * L, H * 64))
    return rows(o), torch.cat([rows(dq), rows(dk), rows(dv)], 1)


def _max_ratio(qkv, dout, mask, B, L, H, q_scale, p=0.0, seed=0, site=0, **kw):
    keep = short_attn_keep(p, seed, site, B, H, L)
    out, dqkv = emulate(qkv, dout, mask, B, L, H, q_scale, p, keep, **kw)
    want = short_reference(qkv, dout, mask, B, L, H, q_scale, multiplier(keep, p) if p > 0 else None)
    return worst_ratios(out, dqkv, want)


# the element-wise shapes of test_text_attention_gpu.py (H = 12 at two lengths: the emulation is slow on the CPU)
SHAPES = [(L, 1) for L in (1, 2, 31, 32, 33, 63, 64, 65, 96, 97, 127, 128)] + [(33, 12), (128, 12)]


@pytest.mark.parametrize("L,H", SHAPES)
def test_emulated_kernel_at_its_worst_stays_within_the_bound(L, H):
    for q_scale in (0.125, 0.1):
        qkv, dout, mask, B = case(L, H, q_scale, seed=L * 31 + H, device="cpu")
        r = _max_ratio(qkv, dout, mask, B, L, H, q_scale)
        print(f"[emulation] L={L} H={H} q_scale={q_scale}: " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()))
        assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize("L", [33, 64, 65, 128])
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_emulated_kernel_with_dropout_stays_within_the_bound(L, p):
    qkv, dout, mask, B = case(L, 2, 0.125, seed=L + 7, device="cpu")
    r = _max_ratio(qkv, dout, mask, B, L, 2, 0.125, p=p, seed=0x8000000000000123, site=5)
    print(f"[emulation] dropout p={p} L={L}: " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()))
    assert max(r.values()) <= 1.0, r


FAULTS = ["keep bit flipped", "dp keys j, j+32 swapped", "last key padded", "delta without keep",
          "dv without 1/(1-p)", "bf16 truncation", "q_scale 0.125"]


def test_planted_faults_miss_the_bound_by_10x():
    L, H, q_scale, p = 128, 2, 0.1, 0.1
    qkv, dout, mask, B = case(L, H, q_scale, seed=3, device="cpu")
    clean = _max_ratio(qkv, dout, mask, B, L, H, q_scale, p=p, seed=11, site=3, worst=False)
    assert max(clean.values()) <= 1.0, clean
    misses = {}
    for fault in FAULTS:
        r = _max_ratio(qkv, dout, mask, B, L, H, q_scale, p=p, seed=11, site=3, worst=False, fault=fault)
        misses[fault] = max(r.values())
        print(f"[fault] {fault:26s} misses the bound by {misses[fault]:.3g}x (" +
              ", ".join(f"{k} {v:.3g}" for k, v in r.items()) + ")")
    assert all(m >= 10 for m in misses.values()), misses
