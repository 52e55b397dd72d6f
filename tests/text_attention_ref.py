"""float64 reference of the text tower's key-padding-masked attention with a dropout multiplier (text_attn_* and
text_attn_long_*), the input cases of its tests, and the element-wise bound of the short-caption kernel
(text_attn_kernel, csrc/text.cu, L <= 128).  Used by test_text_attention_gpu.py and test_text_long_gpu.py;
test_text_attention_ref_host.py shows on the CPU that the bound holds for an fp32 emulation of the kernel with its
approximate exp and reciprocal pushed to their worst case, and that subtle faults miss it by 10x or more.

The short kernel computes in fp32 on the CUDA cores (text.cu is built with --use_fast_math: FTZ, __expf = FMUL + MUFU.EX2,
1 / x = MUFU.RCP) and rounds to bf16 only when it stores.  With u = 2^-24, per (b, h), P the exact softmax over the valid
keys, m the dropout multiplier (keep / (1 - p), 1 without dropout), first-order in u:
  scores      bf16 inputs widen exactly; s_ij is a 64-term FMA chain: 64 u T_ij, T_ij = sum_d |q_id k_jd|.
  exp         x = s_ij - max_k s_ik (one FADD: u |x|); __expf is within 2 + floor(1.173 |x|) ulp (CUDA Programming Guide),
              one ulp <= 2u relative: rho_ij = 64 u T_ij + 4 u + 3.346 u |x_ij|.  The error of the max cancels in the
              normalisation.
  normalise   per-lane sums of up to 4 keys, then a 5-level butterfly (8 u), 1 / sum by MUFU.RCP (1 ulp, 2 u), one FMUL:
              |dP_ij| <= P_ij (rho_ij + sum_k P_ik rho_ik + 11 u).
  dropout     the kernel's fp32 1 / (1 - p) is an FADD and a MUFU.RCP from the exact one (3 u), and P m is one FMUL:
              |dP'_ij| <= m_ij |dP_ij| + 4 u P_ij m_ij.
  out, dv     L-term FMA chains: out_id: sum_j |dP'_ij| |v_jd| + L u sum_j P'_ij |v_jd|; dv_jd the same over i with dO.
  dp, delta   dp_ij = m_ij (dO_i . v_j): 64 u sum_d |dO_id v_jd| m_ij + 4 u |dp_ij|;  delta_i = sum_j P_ij dp_ij through
              4 FMAs per lane and the butterfly: sum_j (|dP_ij| |dp_ij| + P_ij e(dp_ij)) + 9 u sum_j P_ij |dp_ij|.
  dS          P (dp - delta), an FADD and an FMUL: |dP_ij| |A_ij| + P_ij (e(dp_ij) + e(delta_i) + u |A_ij|) + u |dS_ij|.
  dq, dk      L-term FMA chains over dS; dq then one FMUL by the fp32 q_scale the kernel is given (the reference uses
              that value too): |qs| (sum_j e(dS_ij) |k_jd| + L u sum_j |dS_ij k_jd|) + u |dq_id|; dk the same over i
              with |q_id|.
A slack of SLACK = 1.25 covers the second-order terms and the fp64 magnitude sums standing in for the fp32 ones.  Each
bf16 output must lie in [rn(ref - e), rn(ref + e)] (tests/gemm_ref.py: exact, since rounding is monotone).  FTZ is not
modelled: every probability in the cases is far above 2^-126 (score spread about 18, and exact zeros for padded keys)."""
import numpy as np
import torch
from gemm_ref import bf16_ratio, check
from kernel_checks import BF16, F64

U = 2.0 ** -24
SLACK = 1.25
SENTINEL_ROWS = 3
SENTINEL = -3.0


def _heads(qkv, dout, B, L, H):
    x = qkv.to(F64).view(B, L, 3, H, 64).permute(2, 0, 3, 1, 4)
    return x[0], x[1], x[2], dout.to(F64).view(B, L, H, 64).permute(0, 2, 1, 3)


def reference(qkv, dout, mask, B, L, H, q_scale, mult=None):
    """float64 masked attention (dropout multipliers `mult` [B, H, L, L] on the probabilities) and the magnitude sums
    of the divided attention's bounds (DESIGN section 6; the long kernel's)."""
    q, k, v, do = _heads(qkv, dout, B, L, H)
    valid = mask.bool().view(B, 1, 1, L)
    s = (q @ k.transpose(-1, -2)).masked_fill(~valid, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    m = mult.to(qkv.device) if mult is not None else torch.ones((), dtype=F64, device=qkv.device)
    pd = p * m
    o = pd @ v
    pv = pd @ v.abs()
    dp = (do @ v.transpose(-1, -2)) * m
    delta = (do * o).sum(-1, keepdim=True)
    ds = p * (dp - delta)
    e = (do.abs() * (pv + 2 * o.abs())).sum(-1, keepdim=True)
    w = p * ((dp - delta).abs() + e)
    lse_t = (q.abs() @ k.abs().transpose(-1, -2)).masked_fill(~valid, 0.0).amax(-1)
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(B * L, H * 64)
    return {"out": rows(o), "out_t": rows(pv), "lse": lse, "lse_t": lse_t,
            "dq": rows(q_scale * (ds @ k)), "dq_t": rows(q_scale * (w @ k.abs())),
            "dk": rows(ds.transpose(-1, -2) @ q), "dk_t": rows(w.transpose(-1, -2) @ q.abs()),
            "dv": rows(pd.transpose(-1, -2) @ do), "dv_t": rows(pd.transpose(-1, -2) @ do.abs())}


def short_reference(qkv, dout, mask, B, L, H, q_scale, mult=None):
    """{name: (float64 value [B*L, H*64], bound)} for out, dq, dk, dv of text_attn_fwd / text_attn_bwd, with the
    bound of the module docstring."""
    q, k, v, do = _heads(qkv, dout, B, L, H)
    valid = mask.bool().view(B, 1, 1, L)
    s = (q @ k.transpose(-1, -2)).masked_fill(~valid, float("-inf"))
    p = torch.softmax(s, -1)
    x = (s - s.amax(-1, keepdim=True)).masked_fill(~valid, 0.0)
    rho = (64 * (q.abs() @ k.abs().transpose(-1, -2)) + 4 + 3.346 * x.abs()) * U
    dp0 = p * (rho + (p * rho).sum(-1, keepdim=True) + 11 * U)                  # the stored probabilities
    m = mult.to(qkv.device, F64) if mult is not None else torch.ones((), dtype=F64, device=qkv.device)
    pd, dpd = p * m, m * dp0 + 4 * U * p * m                                     # the dropped ones
    out = pd @ v
    e_out = dpd @ v.abs() + L * U * (pd @ v.abs())
    dv = pd.transpose(-1, -2) @ do
    e_dv = dpd.transpose(-1, -2) @ do.abs() + L * U * (pd.transpose(-1, -2) @ do.abs())
    g = do @ v.transpose(-1, -2)
    dpr = m * g
    e_dp = m * (64 * U * (do.abs() @ v.abs().transpose(-1, -2)) + 4 * U * g.abs())
    delta = (p * dpr).sum(-1, keepdim=True)
    e_delta = (dp0 * dpr.abs() + p * e_dp).sum(-1, keepdim=True) + 9 * U * (p * dpr.abs()).sum(-1, keepdim=True)
    a = dpr - delta
    ds = p * a
    e_ds = dp0 * a.abs() + p * (e_dp + e_delta + U * a.abs()) + U * ds.abs()
    qs = float(np.float32(q_scale))
    dq = qs * (ds @ k)
    e_dq = abs(qs) * (e_ds @ k.abs() + L * U * (ds.abs() @ k.abs())) + U * dq.abs()
    dk = ds.transpose(-1, -2) @ q
    e_dk = e_ds.transpose(-1, -2) @ q.abs() + L * U * (ds.abs().transpose(-1, -2) @ q.abs())
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(B * L, H * 64)
    return {name: (rows(val), SLACK * rows(err)) for name, val, err in
            (("out", out, e_out), ("dq", dq, e_dq), ("dk", dk, e_dk), ("dv", dv, e_dv))}


def split_dqkv(dqkv, H):
    D = 64 * H
    return {"dq": dqkv[:, :D], "dk": dqkv[:, D:2 * D], "dv": dqkv[:, 2 * D:]}


def worst_ratios(out, dqkv, want):
    """{name: worst error / bound over the elements} of out and the three parts of dqkv against short_reference."""
    got = dict(split_dqkv(dqkv, out.shape[1] // 64), out=out)
    res = {}
    for name, (ref, bound) in want.items():
        ratio, _ = bf16_ratio(got[name], ref, bound)
        res[name] = float("inf") if bool(ratio.isnan().any()) else ratio.max().item()
    return res


def check_short(tag, out, dqkv, mask, want):
    """Every element of out, dq, dk, dv in its interval (printing each worst fraction of the bound); dk and dv of
    padded keys exactly 0.  Returns {name: worst fraction}."""
    got = dict(split_dqkv(dqkv, out.shape[1] // 64), out=out)
    for name in ("out", "dq", "dk", "dv"):
        check(f"{name} {tag}", got[name], want[name])
    pad = mask.reshape(-1) == 0
    for name in ("dk", "dv"):
        assert bool((got[name][pad] == 0).all()), f"{tag}: {name} of padded keys not exactly 0"
    return worst_ratios(out, dqkv, want)


# ------------------------------------------------------------------------------------------------ cases
def make_inputs(B, L, H, seed, q_scale=0.125, device="cuda"):
    """qkv [B*L, 3*D] bf16 with q pre-scaled by q_scale (as the QKV GEMM's epilogue does; scores of standard deviation
    8 q_scale), dout [B*L, D] bf16."""
    g = torch.Generator(device=device).manual_seed(seed)
    D = 64 * H
    x = torch.randn(B * L, 3 * D, generator=g, device=device)
    x[:, :D] *= q_scale
    return x.to(BF16), torch.randn(B * L, D, generator=g, device=device).to(BF16)


def plant_maxima(qkv, mask, B, L, H, score=18.0):
    """Every third query row points at its sample's last valid key, `score` above the rest."""
    x = qkv.float().view(B, L, 3, H, 64)
    for b in range(B):
        last = int(mask[b].nonzero().max())
        kk = x[b, last, 1]                                         # [H, 64]
        x[b, ::3, 0] = (kk * (score / kk.pow(2).sum(-1, keepdim=True)))[None]
    return x.reshape(B * L, 3 * H * 64).to(BF16)


def short_masks(L, device="cuda"):
    """Key masks [B, L] for L <= 128: full; one key; prefixes on and around the 32-key boundaries (a lane's 2nd, 3rd and
    4th key); a holed, non-prefix pattern with a whole 32-key run missing; 5 keys.  Duplicates dropped."""
    j = torch.arange(L)
    rows = [torch.ones(L, dtype=torch.int64), (j == (L - 1) // 2).long()]
    for n in (31, 32, 33, 64, 65, 96, 97, L - 1):
        if 1 <= n < L:
            rows.append((j < n).long())
    holes = ((j % 7 != 3) & ~((j >= 32) & (j < 64))).long()
    holes[0] = 1
    rows += [holes, (j < 5).long()]
    uniq = []
    for r in rows:
        if not any(torch.equal(r, o) for o in uniq):
            uniq.append(r)
    return torch.stack(uniq).to(device)


def case(L, H, q_scale, seed, device="cuda"):
    """(qkv, dout, mask, B) of one element-wise case: short_masks(L), planted maxima."""
    mask = short_masks(L, device)
    B = mask.shape[0]
    qkv, dout = make_inputs(B, L, H, seed, q_scale, device)
    return plant_maxima(qkv, mask, B, L, H), dout, mask, B
