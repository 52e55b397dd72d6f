"""float64 reference of the bf16 GEMM (egovlp_gemm_bf16, csrc/gemm_wgmma.cu), the element-wise bound its arithmetic
allows, and the checks its tests share (test_kernels_gpu.py, test_gemm_staged_epilogue_gpu.py,
test_gemm_wgrad_epilogue_gpu.py, test_front_end_kernels_gpu.py, test_activation_memory_gpu.py,
test_video_dropout_gpu.py; test_gemm_ref_host.py shows on the CPU that the check accepts an fp32 emulation of the kernel
and rejects subtle faults).  Needs no GPU: every function works on the device its inputs are on.

The reference computes the epilogue of include/egovlp_b200.h in float64 from the same bf16 / fp32 values the kernel reads:
  p = A B^T,  v = p + bias,  v *= col_scale on columns n < col_scale_ncols,  out2 = v (act 0 / 1 with out2);
  act 1: gelu(v);  act 2: v gelu'(aux);  act 3: gelu(v), out2 = gelu'(v);  act 4: v aux;
  act 5: v gelu'(aux), out2 = gelu(aux);  dropout: the stored value (and act 5's out2) times the materialised multiplier;
  + residual[m] (row m % res_row_mod with a broadcast table);  out_mode 2: out = base + v;
  colsum += sum_m v (the fp32 values, before any bf16 rounding);  colsum_a += sum_k A[k, m].

Bound e of each element, u = 2^-24 (one fp32 ulp is at most 2u of the value), S = sum_k |a_k b_k| (products of bf16
values are exact in fp32):
  accumulation  the fp32 accumulator takes one k16 wgmma step at a time.  Allowing one fp32 ulp of the running sum per
                step, and one more per split-K partial, assumes nothing about rounding inside the tensor core:
                e = (ceil(K / 16) + split_k) 2u S.
  epilogue      each fp32 operation rounds once, within u of its result: the bias fma adds u (S + |bias|); col_scale
                scales e and adds u |v|; a product with aux or gelu'(aux) scales e by |factor| and adds u |product|; the
                residual add adds u (|v| + |r|); out_mode 2 adds split_k atomic adds, u (|base| + S) each.
  GELU          the kernels evaluate Phi through Abramowitz-Stegun 7.1.26 (|erf error| <= 1.5e-7) with approximate rcp /
                ex2, so GELU and GELU' are within g(x) = 2e-7 (1 + |x|) of the exact functions, plus the rounding of the
                result.  An input error e passes through |GELU'| <= 1.13 and |GELU''| <= 0.8:
                gelu(v): 1.13 e + g(v);  gelu'(v): 0.8 e + g(v);  v gelu'(z): |gelu'(z)| e + |v| g(z) (z = aux is exact);
                gelu(z): g(z).
  dropout       the kernel scales by its own fp32 multiplier (1 / (1 - p) times the drop-path factor: up to two roundings
                away from the materialised one) and rounds the product: |m| e + 3u |m value|.
  colsum        sum_m e_m plus the fp32 additions: a thread adds its two rows, three shuffle levels fold a warp's 16 rows,
                then ceil(M / 16) atomic adds land in any order: (ceil(M / 16) + 5) u (|colsum| + sum_m |v_m|).
  colsum_a      exact bf16 addends summed in fp32 in any order: (K + 5) u (|colsum_a| + sum_k |A[k, m]|).

fp32 outputs: |got - ref| <= e.  bf16 outputs: the kernel rounds an fp32 value within e of ref to nearest.  Rounding is
monotone (torch's fp64 -> fp32 -> bf16 as well), so rn(ref - e) <= got <= rn(ref + e) in bf16 order, exactly: a value one
bf16 step off, or a truncating conversion, falls outside the interval, where a tolerance of one ulp lets both through.
Each check prints its worst error as a fraction of its bound (run pytest with -s)."""
import math

import torch
from kernel_checks import BF16, F32, F64, _ordered_bf16, _worst

U = 2.0 ** -24


def gelu64(x):
    return x * 0.5 * (1 + torch.erf(x / 2 ** 0.5))


def dgelu64(x):
    return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5


def gelu_err(x):
    return 2e-7 * (1 + x.abs())


def reference(a, b, *, a_mn=False, b_mn=False, bias=None, col_scale=1.0, col_scale_ncols=0, act=0, aux=None,
              out2=False, residual=None, res_row_mod=0, mult=None, base=None, split_k=1, colsum=None, colsum_a=None,
              rows=None):
    """{output name: (fp64 value, bound)} of what ops.gemm(a, b, out, ...) computes with the same arguments.  `out2`:
    whether the call passes out2; `base`, `colsum`, `colsum_a`: the values out (accumulate=True) and the column-sum
    vectors hold before the call; `mult`: the fp32 [M, N] dropout multiplier; `rows`: only these rows of the output."""
    A = (a.t() if a_mn else a).double()
    Bt = (b if b_mn else b.t()).double()
    M, N = A.shape[0], Bt.shape[1]
    idx = torch.arange(M, device=A.device) if rows is None else rows

    def at_rows(t):
        return t.double() if rows is None else t[rows].double()

    p = A[idx] @ Bt
    S = A[idx].abs() @ Bt.abs()
    e = (math.ceil(A.shape[1] / 16) + split_k) * 2 * U * S
    v = p
    if bias is not None:
        v = p + bias.double()
        e = e + U * (S + bias.double().abs())
    if col_scale_ncols:
        scale = torch.ones(N, dtype=F64, device=A.device)
        scale[:col_scale_ncols] = torch.tensor(col_scale, dtype=F32).item()
        v = v * scale
        e = e * scale.abs() + U * v.abs()
    res = {}
    if out2 and act in (0, 1):
        res["out2"] = (v, e)
    if act in (1, 3):
        out = gelu64(v)
        if act == 3:
            d = dgelu64(v)
            res["out2"] = (d, 0.8 * e + gelu_err(v) + U * d.abs())
        e = 1.13 * e + gelu_err(v) + U * out.abs()
    elif act in (2, 5):
        z = at_rows(aux)
        d = dgelu64(z)
        out = v * d
        e = e * d.abs() + v.abs() * gelu_err(z) + U * out.abs()
        if act == 5:
            h = gelu64(z)
            res["out2"] = (h, gelu_err(z) + U * h.abs())
    elif act == 4:
        x = at_rows(aux)
        out = v * x
        e = e * x.abs() + U * out.abs()
    else:
        out = v
    if mult is not None:
        m = at_rows(mult)
        out = out * m
        e = e * m.abs() + 3 * U * out.abs()
        if act == 5:
            h, eh = res["out2"]
            res["out2"] = (h * m, eh * m.abs() + 3 * U * (h * m).abs())
    if residual is not None:
        r = residual.double()[idx % res_row_mod if res_row_mod else idx]
        e = e + U * (out.abs() + r.abs())
        out = out + r
    if colsum is not None:
        assert rows is None
        c0 = colsum.double()
        res["colsum"] = (c0 + out.sum(0), e.sum(0) + (math.ceil(M / 16) + 5) * U * (c0.abs() + out.abs().sum(0)))
    if base is not None:
        b0 = at_rows(base)
        e = e + split_k * U * (b0.abs() + S)
        out = b0 + out
    if colsum_a is not None:
        c0 = colsum_a.double()
        res["colsum_a"] = (c0 + A.sum(1), (A.shape[1] + 5) * U * (c0.abs() + A.abs().sum(1)))
    res["out"] = (out, e)
    return res


def _from_ordered(o):
    """Inverse of kernel_checks._ordered_bf16."""
    return torch.where(o < 0, -o - 32768, o).to(torch.int16).view(BF16)


def bf16_interval(ref, bound):
    """[rn(ref - e), rn(ref + e)]: the bf16 values an fp32 result within `bound` of `ref` can round to."""
    return (ref - bound).to(BF16), (ref + bound).to(BF16)


def bf16_ratio(got, ref, bound):
    """Per element of a bf16 `got`: the error it needs as a fraction of `bound` (<= 1 exactly inside [rn(ref - e),
    rn(ref + e)], > 1 outside, NaN where got is NaN), and the number of bf16 steps it lies outside that interval."""
    lo, hi = bf16_interval(ref, bound)
    g, lo_o, hi_o = _ordered_bf16(got), _ordered_bf16(lo), _ordered_bf16(hi)
    outside = (lo_o - g).clamp_min(0) + (g - hi_o).clamp_min(0)       # bf16 steps outside the interval
    # the error the result needs: 0 if it is ref rounded, else the distance from ref to the rounding boundary
    # between got and its neighbour towards ref; as a fraction of the bound, <= 1 exactly inside the interval
    r_o = _ordered_bf16(ref.to(BF16))
    nb = _from_ordered(g + torch.sign(r_o - g))
    need = torch.where(g == r_o, 0.0, ((got.double() + nb.double()) / 2 - ref).abs())
    ratio = need / bound.clamp_min(1e-300)
    ratio = torch.where(outside > 0, ratio.clamp_min(1 + 1e-9), ratio.clamp_max(1.0))
    return ratio.masked_fill(got.isnan(), float("nan")), outside


def check(name, got, want):
    """`got` (bf16 or fp32) against want = (fp64 value, bound), element by element, as the module docstring says."""
    ref, bound = want
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    if got.dtype == BF16:
        lo, hi = bf16_interval(ref, bound)
        ratio, outside = bf16_ratio(got, ref, bound)
        worst, at = _worst(name, ratio)
        assert not bool(outside.any()) and worst <= 1.0, (
            f"{name}: {int((outside > 0).sum())} elements outside their interval; at {at}: got {got[at].item()}, "
            f"interval [{lo[at].item()}, {hi[at].item()}], exact {ref[at].item()}, bound {bound[at].item():.3e}")
    else:
        assert got.dtype == F32, (name, got.dtype)
        err = (got.double() - ref).abs()
        worst, at = _worst(name, err / bound.clamp_min(1e-300))
        assert worst <= 1.0, (f"{name}: |got - ref| = {err[at].item():.3e} > {bound[at].item():.3e} at {at} "
                              f"(got {got[at].item()}, ref {ref[at].item()})")


def check_all(name, got, want):
    """Every output of one call: got = {name: tensor} with the keys of want = reference(...)."""
    assert set(got) == set(want), (name, sorted(got), sorted(want))
    for k in sorted(want):
        check(f"{name} {k}", got[k], want[k])


def assert_outside_untouched(name, buf, index, fill=float("nan")):
    """Every element of `buf` outside buf[index] still holds `fill` (NaN: is still NaN)."""
    outside = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    outside[index] = False
    rest = buf[outside]
    ok = rest.isnan() if math.isnan(fill) else rest == fill
    assert bool(ok.all()), f"{name}: {int((~ok).sum())} elements outside the view were written"


def gelu_tail_inputs(a, bias):
    """Inputs whose pre-activations reach GELU's tails and zero: rows of A scaled by 0, 4/15, ..., 4 (so that at the
    tests' operand scales, where the products' standard deviation is about 1, the largest reach about +-10, and rows
    of zeros give exact zeros where the bias is zero) and every 7th bias entry zero.  -> (a, bias)"""
    M = a.shape[0]
    f = 4.0 * (torch.arange(M, device=a.device) % 16).double() / 15
    a = (a.double() * f[:, None]).to(a.dtype)
    bias = bias.clone()
    bias[::7] = 0
    return a, bias


def spread(shape, seed, device="cuda"):
    """bf16 values uniform in [-10, 10] with exact zeros in every 9th column: an aux operand through GELU's tails."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.rand(shape, generator=g, device=device, dtype=F32) * 20 - 10
    x[..., ::9] = 0
    return x.to(BF16)


def forms_references(a, b, bias, res, aux):
    """(value, bound) of the twelve outputs of test_gemm_staged_epilogue_gpu.run_forms: bias -> bf16 with the column
    scale, GELU + GELU', x aux, bias + residual, GELU, first with K-major B (`b`, [N, K]), then the same forms with the
    MN-major B b^T (no bias and no column scale on its first output)."""
    N = b.shape[0]
    outs = []
    for bb, b_mn in ((b, False), (b.t(), True)):
        first = (reference(a, bb, b_mn=True) if b_mn else
                 reference(a, bb, bias=bias, col_scale=0.125, col_scale_ncols=min(N, 64)))
        act3 = reference(a, bb, b_mn=b_mn, bias=bias, act=3, out2=True)
        outs += [first["out"], act3["out"], act3["out2"],
                 reference(a, bb, b_mn=b_mn, aux=aux, act=4)["out"],
                 reference(a, bb, b_mn=b_mn, bias=bias, residual=res)["out"],
                 reference(a, bb, b_mn=b_mn, act=1)["out"]]
    return outs


def check_lowmem_pair(out, n2, w1, b1, dy, w2, z_in, rows):
    """The eight outputs of test_activation_memory_gpu.run_pair on the rows `rows`: fc1 in both training forms (act 1
    with out2, act 3 with out2) and the fc2 input gradient (act 5) with W2 as K-major (w2^T) and MN-major B."""
    fc1z = reference(n2, w1, bias=b1, act=1, out2=True, rows=rows)
    fc1d = reference(n2, w1, bias=b1, act=3, out2=True, rows=rows)
    check_all("fc1 act 1", {"out": out[0][rows], "out2": out[1][rows]}, fc1z)
    check_all("fc1 act 3", {"out": out[2][rows], "out2": out[7][rows]}, fc1d)
    for name, (du, hz), b_mn in (("fc2 act 5, K-major B", out[3:5], False), ("fc2 act 5, MN-major B", out[5:7], True)):
        want = reference(dy, w2 if b_mn else w2.t(), b_mn=b_mn, aux=z_in, act=5, out2=True, rows=rows)
        check_all(name, {"out": du[rows], "out2": hz[rows]}, want)
