"""LayerNorm (layernorm.cu) against float64, element by element, on both kernel paths.

Two kernel pairs implement it.  The pipelined bulk-copy kernels (`layernorm_{fwd,bwd}_pipe_kernel`) take calls with
D = NV * 128, at least 4096 contiguous rows and 16-byte aligned inputs; every other call runs the occupancy kernels.
A process reads EGOVLP_LN_PIPE once, so each case reaches its path through its inputs, and its id names the path:
"pipe" or "occ".  The reference (`ln_reference`) is computed in float64 from the same fp32 / bf16 values the kernels
read.  The backward is given the mean and rstd it reads (fp32) and uses them as they are:
  x^ = (x - mean) rstd,  dx = rstd (dy g - mean(dy g) - x^ mean(dy g x^)) + add1 + add2,
  d(gamma) = sum_rows dy x^,  d(beta) = sum_rows dy,  colsum_dx = sum_rows dx.
The host test pins it to torch.nn.functional.layer_norm and its autograd in float64.

The bounds follow from the kernels' arithmetic.  u = 2^-24 (fp32 unit roundoff), u16 = 2^-8 (bf16), S = 1.25 slack.
A row sum is taken by one warp: each lane adds its 4 NV values, then 5 shuffle levels, so every value passes through at
most k = 4 NV + 5 additions.  Per row, with mu, var (biased), rstd = 1 / sqrt(var + eps) exact, V = var + eps:
  mean   e_mu   = S u (k + 2) sum|x| / D                      fp32 row sum, times 1/D rounded, one product rounding;
  rstd   e_rstd = S rstd (((k + 4) u var + e_mu^2) / (2 V) + 4.5 u)
                                                             squares of x - mean (3u each) summed, fma with 1/D and eps,
                                                             the mean's error adds e_mu^2 to the variance; rsqrtf's
                                                             documented 2 ulp = 4u relative;
  y32    e_y    = S (|g| (rstd e_mu + |x - mu| e_rstd + 3 u |x^|) + u |y|)
                                                             the mean's error times rstd |g| dominates a row with a large
                                                             common offset or zero variance;
  y16    e_y + u16 (|y| + e_y)                              one bf16 rounding of the fp32 value.
Backward, with g = dy gamma, A1 = mean|g|, A2 = mean|g x^|, o = the normalisation's gradient before the addends:
  dx     e_dx   = S (u (rstd (4 |g| + (k + 6) A1 + (k + 9) |x^| A2) + |o|) + 2 u (|o| + |add1| + |add2|))
                                                             x^ recomputed (2u), both row means (sums of depth k), the
                                                             three-term combination, the two addends;
  dx16   e_dx + u16 (|dx| + e_dx);
  d(gamma), d(beta)  `assert_sum_bound` with rel = S u (n + 3) and S u n over |init| + sum|terms|, n = the additions a
                     column's sum passes through: rows per warp + the CTA's 4 warps + one atomic per CTA;
  colsum_dx          S u n (|init| + sum|dx|) + sum e_dx.
Each check prints its worst element as a fraction of its bound (run with -s).

Outputs land in NaN-filled buffers followed by sentinel rows (and, for the engine's strided dx, sentinel columns the
view does not own): every element must be written and no sentinel touched.  A row's forward outputs and its dx / dx16
do not depend on the path: the two kernels do the same per-row arithmetic, so 4095 rows (occupancy) and the same rows
inside 4096 + 7 (pipelined) must match bit for bit."""
import ctypes as C
import math

import pytest
import torch
from kernel_checks import (BF16, F32, F64, assert_bits_equal, assert_elementwise_bound, assert_sum_bound,
                           nan_filled)

U = 2.0 ** -24
U16 = 2.0 ** -8
SLACK = 1.25
EPS = 1e-6                   # the video tower's LayerNorm eps
EPS_F32 = float(torch.tensor(EPS, dtype=torch.float32))      # as the kernels receive it
PIPE_MIN_ROWS = 4096
SENTINEL_ROWS = 3
SENTINEL = -3.0
E4M3 = torch.float8_e4m3fn
DS = [4, 64, 100, 128, 516, 768, 1000, 1024]


# ---------------------------------------------------------------------------------------------------------- reference
def ln_reference(x, gamma, beta, eps, dy=None, mean=None, rstd=None, add1=None, add2=None):
    """float64 LayerNorm of x [rows, D]: mean, rstd, var, x^, y and sum|x| per row; with dy also the analytic backward
    (`dx`, its LN part `o`, `dgamma`, `dbeta`, `colsum`) and the magnitude sums of the bounds.  The backward uses `mean`
    / `rstd` if given (the values the kernel reads), else the exact ones."""
    x, g, b = x.to(F64), gamma.to(F64), beta.to(F64)
    D = x.shape[1]
    mu = x.mean(1)
    var = (x - mu[:, None]).pow(2).mean(1)
    rs = (var + eps).rsqrt()
    xh = (x - mu[:, None]) * rs[:, None]
    r = {"mean": mu, "var": var, "rstd": rs, "xhat": xh, "y": xh * g + b, "abs_sum": x.abs().sum(1)}
    if dy is None:
        return r
    mb = mu if mean is None else mean.to(F64)
    rb = rs if rstd is None else rstd.to(F64)
    xb = (x - mb[:, None]) * rb[:, None]
    dy = dy.to(F64)
    dg = dy * g
    o = rb[:, None] * (dg - dg.mean(1, keepdim=True) - xb * (dg * xb).mean(1, keepdim=True))
    a1 = add1.to(F64) if add1 is not None else torch.zeros_like(o)
    a2 = add2.to(F64) if add2 is not None else torch.zeros_like(o)
    dx = o + a1 + a2
    r.update(o=o, dx=dx, dgamma=(dy * xb).sum(0), dbeta=dy.sum(0), colsum=dx.sum(0), bxhat=xb, brstd=rb, g=dg,
             A1=dg.abs().sum(1) / D, A2=(dg * xb).abs().sum(1) / D, a1=a1, a2=a2,
             dgamma_t=(dy * xb).abs().sum(0), dbeta_t=dy.abs().sum(0), colsum_t=dx.abs().sum(0))
    return r


def lane_depth(D):
    return 4 * ((D + 127) // 128) + 5


def fwd_bounds(r, gamma, eps):
    """e_mu, e_rstd per row and e_y32, e_y16 per element, as in the module docstring."""
    D = r["xhat"].shape[1]
    k = lane_depth(D)
    e_mu = SLACK * U * (k + 2) * r["abs_sum"] / D
    V = r["var"] + eps
    rs = r["rstd"]
    e_rstd = SLACK * rs * (((k + 4) * U * r["var"] + e_mu ** 2) / (2 * V) + 4.5 * U)
    g = gamma.to(F64).abs()
    dev = r["xhat"].abs() / rs[:, None]                                     # |x - mu|
    e_y = SLACK * (g * (rs[:, None] * e_mu[:, None] + dev * e_rstd[:, None] + 3 * U * r["xhat"].abs()) + U * r["y"].abs())
    return e_mu, e_rstd, e_y, e_y + U16 * (r["y"].abs() + e_y)


def dx_bounds(r):
    D = r["o"].shape[1]
    k = lane_depth(D)
    e_o = U * (r["brstd"][:, None] * (4 * r["g"].abs() + (k + 6) * r["A1"][:, None]
                                      + (k + 9) * r["bxhat"].abs() * r["A2"][:, None]) + r["o"].abs())
    e_dx = SLACK * (e_o + 2 * U * (r["o"].abs() + r["a1"].abs() + r["a2"].abs()))
    return e_dx, e_dx + U16 * (r["dx"].abs() + e_dx)


def column_depth(rows, pipe, sms):
    """Additions a d(gamma) / d(beta) / colsum_dx column passes through (see launch_ln_bwd's grids)."""
    if pipe:
        tiles = -(-rows // 4)
        grid = min(tiles, 2 * sms)
        per_warp = -(-tiles // grid)
    else:
        grid = min(-(-rows // 4), 12 * sms)
        per_warp = -(-rows // (4 * grid))
    return per_warp + 4 + grid


# ---------------------------------------------------------------------------------------------------------- host test
@pytest.mark.parametrize("D", [4, 100, 768])
def test_host_reference_matches_torch_layer_norm_and_its_autograd(D):
    """ln_reference (forward and analytic backward, addends included) against torch.nn.functional.layer_norm and its
    autograd gradients, on the CPU, in float64."""
    gen = torch.Generator().manual_seed(D)
    rows = 9
    x = torch.randn(rows, D, generator=gen, dtype=F64) * 1.5 + 0.2
    x[1] = 300 + 0.3 * x[1]
    gamma = 1 + 0.5 * torch.randn(D, generator=gen, dtype=F64)
    beta = 0.3 * torch.randn(D, generator=gen, dtype=F64)
    dy, a1, a2 = (torch.randn(rows, D, generator=gen, dtype=F64) for _ in range(3))
    r = ln_reference(x, gamma, beta, EPS, dy=dy, add1=a1, add2=a2)
    xr, gr, br = (t.clone().requires_grad_(True) for t in (x, gamma, beta))
    y = torch.nn.functional.layer_norm(xr, (D,), gr, br, EPS)
    y.backward(dy)
    var, mean = torch.var_mean(x, 1, unbiased=False)
    tol = dict(rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(r["mean"], mean, **tol)
    torch.testing.assert_close(r["rstd"], (var + EPS).rsqrt(), **tol)
    torch.testing.assert_close(r["y"], y.detach(), **tol)
    torch.testing.assert_close(r["dx"], xr.grad + a1 + a2, **tol)
    torch.testing.assert_close(r["o"], xr.grad, **tol)
    torch.testing.assert_close(r["dgamma"], gr.grad, **tol)
    torch.testing.assert_close(r["dbeta"], br.grad, **tol)
    torch.testing.assert_close(r["colsum"], (xr.grad + a1 + a2).sum(0), **tol)


# ---------------------------------------------------------------------------------------------------------- GPU harness
@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def randn(shape, seed, scale=1.0):
    return torch.randn(shape, generator=gen(seed), device="cuda") * scale


def plant_hard_rows(x, eps=EPS):
    """Row 0 constant (var = 0: rstd = 1 / sqrt(eps)); row 1 with mean = 10^3 std; row 2 of values near sqrt(eps)."""
    rows, D = x.shape
    hard = [torch.full((D,), 0.37, device="cuda"), 300 + 0.3 * randn((D,), 7), math.sqrt(eps) * randn((D,), 8)]
    for i, h in enumerate(hard[:rows]):
        x[i] = h
    return x


def make_x(rows, D, seed, ld=None):
    """fp32 [rows, D] with the hard rows planted; a view of a [rows, ld] buffer if ld is given."""
    buf = randn((rows, ld or D), seed, 1.5) + 0.2
    x = buf[:, :D]
    plant_hard_rows(x)
    return x


def affine(D, seed):
    return 1 + 0.5 * randn((D,), seed), 0.3 * randn((D,), seed + 1)


def with_sentinels(rows, D, dtype):
    buf = nan_filled((rows + SENTINEL_ROWS,) + ((D,) if D else ()), dtype)
    buf[rows:] = SENTINEL
    return buf


def check_written(name, buf, rows):
    assert not buf[:rows].isnan().any(), f"{name}: {int(buf[:rows].isnan().sum())} elements left unwritten"
    assert bool((buf[rows:] == SENTINEL).all()), f"{name}: a row past the output was written"


def e4m3_buf(rows, D):
    """uint8 0x7F (e4m3 NaN) everywhere; rows past `rows` hold 0x55."""
    buf = torch.full((rows + SENTINEL_ROWS, D), 0x7F, dtype=torch.uint8, device="cuda")
    buf[rows:] = 0x55
    return buf


def run_fwd(ops, x, gamma, beta, outs, eps=EPS, add=None, e4m3=False):
    """Forward into NaN-filled buffers with sentinel rows; outs is a subset of {"y16", "y32", "stats"}.  Returns the
    outputs as [rows, ...] views."""
    rows, D = x.shape
    bufs = {"y16": with_sentinels(rows, D, BF16) if "y16" in outs else None,
            "y32": with_sentinels(rows, D, F32) if "y32" in outs else None,
            "mean": with_sentinels(rows, 0, F32) if "stats" in outs else None,
            "rstd": with_sentinels(rows, 0, F32) if "stats" in outs else None,
            "sum": with_sentinels(rows, D, F32) if add is not None else None}
    y8 = scale = None
    if e4m3:
        y8, scale = e4m3_buf(rows, D), with_sentinels(rows, 0, F32)
    v = {k: (b[:rows] if b is not None else None) for k, b in bufs.items()}
    ops.layernorm_fwd(x, gamma, beta, eps, add=add, sum_out=v["sum"], y16=v["y16"], y32=v["y32"], mean=v["mean"],
                      rstd=v["rstd"], y8=y8[:rows].view(E4M3) if e4m3 else None,
                      row_scale=scale[:rows] if e4m3 else None)
    torch.cuda.synchronize()
    for k, b in bufs.items():
        if b is not None:
            check_written(k, b, rows)
    if e4m3:
        check_written("row_scale", scale, rows)
        assert not bool(((y8[:rows] & 0x7F) == 0x7F).any()), "y8: elements left unwritten"
        assert bool((y8[rows:] == 0x55).all()), "y8: a row past the output was written"
        v["y8"], v["row_scale"] = y8[:rows], scale[:rows]
    return v


def check_fwd(tag, v, r, gamma, eps=EPS):
    e_mu, e_rstd, e_y32, e_y16 = fwd_bounds(r, gamma, eps)
    if v["mean"] is not None:
        assert_elementwise_bound(f"mean {tag}", v["mean"], r["mean"], e_mu)
        assert_elementwise_bound(f"rstd {tag}", v["rstd"], r["rstd"], e_rstd)
    if v["y32"] is not None:
        assert_elementwise_bound(f"y32 {tag}", v["y32"], r["y"], e_y32)
    if v["y16"] is not None:
        assert_elementwise_bound(f"y16 {tag}", v["y16"], r["y"], e_y16)


def pipe_eligible(rows, D):
    return D % 128 == 0 and rows >= PIPE_MIN_ROWS


OUT_SETS = [("y16",), ("y32",), ("y16", "stats"), ("y32", "stats"), ("y16", "y32", "stats")]
# (rows, D, path): every D on the occupancy kernels; the pipelined ones at each D = NV * 128, with the last tile partial
FWD_CASES = ([(300, D, "occ") for D in DS] + [(5, 768, "occ"), (4095, 1024, "occ")]
             + [(4097, 128, "pipe"), (4103, 768, "pipe"), (5000, 1024, "pipe"), (5003, 1024, "pipe")])


@pytest.mark.gpu
@pytest.mark.parametrize("rows,D,path", [pytest.param(*c, id=f"{c[2]}-rows{c[0]}-D{c[1]}") for c in FWD_CASES])
def test_forward_matches_fp64(ops, rows, D, path):
    assert path == ("pipe" if pipe_eligible(rows, D) else "occ")
    x = make_x(rows, D, seed=D + rows)
    gamma, beta = affine(D, 11)
    r = ln_reference(x, gamma, beta, EPS_F32)
    for outs in OUT_SETS:
        v = run_fwd(ops, x, gamma, beta, outs)
        check_fwd(f"{path} rows={rows} D={D} {'+'.join(outs)}", v, r, gamma, EPS_F32)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,D", [pytest.param(r, D, id=f"occ-rows{r}-D{D}") for r, D in
                                    [(300, D) for D in DS] + [(4103, 768)]])
def test_forward_fused_add_matches_fp64(ops, rows, D):
    """x + add written to sum_out (bit for bit as torch's fp32 add) and normalised, non-trivial gamma / beta; eps =
    1e-12, DistilBERT's.  `add` always takes the occupancy kernel, 4103 rows included."""
    eps = 1e-12
    x = make_x(rows, D, seed=3 * D + rows)
    a = randn((rows, D), 99, 0.5)
    a[:3] = 0                                       # x + a keeps the hard rows
    gamma, beta = affine(D, 13)
    s = x + a
    r = ln_reference(s, gamma, beta, float(torch.tensor(eps, dtype=F32)))
    v = run_fwd(ops, x, gamma, beta, ("y16", "y32", "stats"), eps=eps, add=a)
    assert_bits_equal(f"sum_out D={D}", v["sum"], s)
    check_fwd(f"occ add rows={rows} D={D}", v, r, gamma, float(torch.tensor(eps, dtype=F32)))


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,path", [pytest.param(16, 197, "occ", id="occ-strided-B16-S197-D768"),
                                      pytest.param(4100, 2, "occ", id="occ-strided-B4100-S2-D768")])
def test_engine_strided_cls_rows(ops, B, S, path):
    """The video tower's final norm as the engine calls it: the CLS rows in place (x.view(B, S D)[:, :D], row stride
    S D), forward, then the backward with dx written into dx.view(B, S D)[:, :D]; the other columns of dx hold sentinels
    that must survive.  Strided rows never take the pipelined kernels, even at 4100 rows."""
    D = 768
    xs = randn((B, S, D), 5, 1.5) + 0.2
    x = xs.view(B, S * D)[:, :D]
    plant_hard_rows(x)
    gamma, beta = affine(D, 17)
    v = run_fwd(ops, x, gamma, beta, ("y16", "y32", "stats"))
    r = ln_reference(x, gamma, beta, EPS_F32)
    check_fwd(f"strided B={B} S={S}", v, r, gamma, EPS_F32)
    dy = randn((B, D), 6)
    dxb = torch.full((B + SENTINEL_ROWS, S * D), SENTINEL, device="cuda")
    dxb[:B, :D] = float("nan")
    dg, db = randn((D,), 9), randn((D,), 10)
    dg0, db0 = dg.clone(), db.clone()
    ops.layernorm_bwd(dy, x, gamma, v["mean"], v["rstd"], dx=dxb[:B].view(B, S * D)[:, :D], dgamma=dg, dbeta=db)
    torch.cuda.synchronize()
    assert not dxb[:B, :D].isnan().any(), "dx: elements left unwritten"
    assert bool((dxb[:B, D:] == SENTINEL).all()) and bool((dxb[B:] == SENTINEL).all()), "dx: wrote outside the view"
    rb = ln_reference(x, gamma, beta, EPS_F32, dy=dy, mean=v["mean"], rstd=v["rstd"])
    e_dx, _ = dx_bounds(rb)
    assert_elementwise_bound(f"dx strided B={B} S={S}", dxb[:B, :D], rb["dx"], e_dx)
    n = column_depth(B, False, torch.cuda.get_device_properties(0).multi_processor_count)
    assert_sum_bound("dgamma strided", dg, dg0.double() + rb["dgamma"], dg0.double().abs() + rb["dgamma_t"],
                     rel=SLACK * U * (n + 3))
    assert_sum_bound("dbeta strided", db, db0.double() + rb["dbeta"], db0.double().abs() + rb["dbeta_t"],
                     rel=SLACK * U * n)


# ---------------------------------------------------------------------------------------------------------- backward
DTYPES = [(dy, a1, a2) for dy in (F32, BF16) for a1 in (None, F32, BF16) for a2 in (None, F32, BF16)]
BWD_CASES = ([(300, D, "occ") for D in DS] + [(4095, 1024, "occ")]
             + [(4097, 128, "pipe"), (4103, 768, "pipe"), (5000, 1024, "pipe"), (5003, 1024, "pipe")])


def bwd_inputs(rows, D, seed, dy_t, a1_t, a2_t):
    x = make_x(rows, D, seed)
    gamma, beta = affine(D, seed + 1)
    r0 = ln_reference(x, gamma, beta, EPS_F32)
    mean, rstd = r0["mean"].to(F32), r0["rstd"].to(F32)
    dy = randn((rows, D), seed + 2).to(dy_t)
    a1 = randn((rows, D), seed + 3, 0.5).to(a1_t) if a1_t is not None else None
    a2 = randn((rows, D), seed + 4, 2.0).to(a2_t) if a2_t is not None else None
    return x, gamma, beta, mean, rstd, dy, a1, a2


def run_bwd(ops, x, gamma, mean, rstd, dy, a1, a2, want_dx, want_dx16, grads, colsum):
    rows, D = x.shape
    dxb = with_sentinels(rows, D, F32) if want_dx else None
    dx16b = with_sentinels(rows, D, BF16) if want_dx16 else None
    acc = {k: torch.cat([randn((D,), 40 + i), torch.full((SENTINEL_ROWS,), SENTINEL, device="cuda")])
           for i, k in enumerate(("dgamma", "dbeta", "colsum"))}
    init = {k: t[:D].clone() for k, t in acc.items()}
    ops.layernorm_bwd(dy, x, gamma, mean, rstd, add1=a1, add2=a2,
                      dx=dxb[:rows] if want_dx else None, dx16=dx16b[:rows] if want_dx16 else None,
                      dgamma=acc["dgamma"][:D] if grads else None, dbeta=acc["dbeta"][:D] if grads else None,
                      colsum_dx=acc["colsum"][:D] if colsum else None)
    torch.cuda.synchronize()
    out = {}
    for name, b in (("dx", dxb), ("dx16", dx16b)):
        if b is not None:
            check_written(name, b, rows)
            out[name] = b[:rows]
    for k, t in acc.items():
        assert bool((t[D:] == SENTINEL).all()), f"{k}: wrote past D"
        if (k == "colsum" and colsum) or (k != "colsum" and grads):
            out[k] = t[:D]
        else:
            assert torch.equal(t[:D], init[k]), f"{k}: written though not requested"
    return out, init


@pytest.mark.gpu
@pytest.mark.parametrize("rows,D,path", [pytest.param(*c, id=f"{c[2]}-rows{c[0]}-D{c[1]}") for c in BWD_CASES])
def test_backward_matches_fp64(ops, sms, rows, D, path):
    """Every dtype combination (dy fp32 / bf16; add1, add2 each absent, fp32 or bf16), cycling through the outputs (dx,
    dx16, both) and the optional column sums, which accumulate onto non-zero vectors."""
    assert path == ("pipe" if pipe_eligible(rows, D) else "occ")
    n = column_depth(rows, path == "pipe", sms)
    for i, (dy_t, a1_t, a2_t) in enumerate(DTYPES):
        want_dx, want_dx16 = [(True, False), (False, True), (True, True)][i % 3]
        grads, colsum = i % 2 == 0, i % 4 < 2
        x, gamma, beta, mean, rstd, dy, a1, a2 = bwd_inputs(rows, D, 100 + i, dy_t, a1_t, a2_t)
        out, init = run_bwd(ops, x, gamma, mean, rstd, dy, a1, a2, want_dx, want_dx16, grads, colsum)
        r = ln_reference(x, gamma, beta, EPS_F32, dy=dy, mean=mean, rstd=rstd, add1=a1, add2=a2)
        e_dx, e_dx16 = dx_bounds(r)
        tag = (f"{path} rows={rows} D={D} dy={str(dy_t)[6:]} add1={str(a1_t)[6:] if a1_t else '-'} "
               f"add2={str(a2_t)[6:] if a2_t else '-'}")
        if want_dx:
            assert_elementwise_bound(f"dx {tag}", out["dx"], r["dx"], e_dx)
        if want_dx16:
            assert_elementwise_bound(f"dx16 {tag}", out["dx16"], r["dx"], e_dx16)
        if grads:
            assert_sum_bound(f"dgamma {tag}", out["dgamma"], init["dgamma"].double() + r["dgamma"],
                             init["dgamma"].double().abs() + r["dgamma_t"], rel=SLACK * U * (n + 3))
            assert_sum_bound(f"dbeta {tag}", out["dbeta"], init["dbeta"].double() + r["dbeta"],
                             init["dbeta"].double().abs() + r["dbeta_t"], rel=SLACK * U * n)
        if colsum:
            bound = SLACK * U * n * (init["colsum"].double().abs() + r["colsum_t"]) + e_dx.sum(0)
            assert_elementwise_bound(f"colsum_dx {tag}", out["colsum"], init["colsum"].double() + r["colsum"], bound)


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["occ-dy16-off8-rows4103-D768", "occ-add16-off8-rows4103-D768"])
def test_backward_bf16_operand_off_16_bytes_takes_the_occupancy_kernel(ops, sms, what):
    """A bf16 dy or addend whose base is 8 bytes off 16 cannot feed the bulk copies: the occupancy kernel runs, and
    matches fp64 as everywhere else."""
    rows, D = 4103, 768
    x, gamma, beta, mean, rstd, dy, a1, _ = bwd_inputs(rows, D, 7, BF16, BF16, None)
    pad = torch.empty(rows * D + 4, dtype=BF16, device="cuda")
    moved = pad[4:].view(rows, D)
    if what.startswith("occ-dy16"):
        moved.copy_(dy); dy = moved
    else:
        moved.copy_(a1); a1 = moved
    assert moved.data_ptr() % 16 == 8
    out, init = run_bwd(ops, x, gamma, mean, rstd, dy, a1, None, True, True, True, True)
    r = ln_reference(x, gamma, beta, EPS_F32, dy=dy, mean=mean, rstd=rstd, add1=a1)
    e_dx, e_dx16 = dx_bounds(r)
    assert_elementwise_bound(f"dx {what}", out["dx"], r["dx"], e_dx)
    assert_elementwise_bound(f"dx16 {what}", out["dx16"], r["dx"], e_dx16)
    n = column_depth(rows, False, sms)
    assert_sum_bound(f"dgamma {what}", out["dgamma"], init["dgamma"].double() + r["dgamma"],
                     init["dgamma"].double().abs() + r["dgamma_t"], rel=SLACK * U * (n + 3))


# ---------------------------------------------------------------------------------------------------------- row-count invariance
@pytest.mark.gpu
@pytest.mark.parametrize("D", [128, 768, 1024])
def test_pipelined_and_occupancy_kernels_agree_bit_for_bit(ops, D):
    """4096 + 7 rows (pipelined kernels), then the first 4095 of the same rows (occupancy kernels): y16, y32, mean and
    rstd of the plain forward, the same four plus y8 / row_scale of the e4m3 form (D > 256, a kernel instantiation of
    its own), dx and dx16 are bit-identical row for row."""
    R, r = PIPE_MIN_ROWS + 7, PIPE_MIN_ROWS - 1
    x = make_x(R, D, seed=D)
    gamma, beta = affine(D, 21)
    for e4m3 in (False, True) if D > 256 else (False,):
        form = "e4m3" if e4m3 else "plain"
        full = run_fwd(ops, x, gamma, beta, ("y16", "y32", "stats"), e4m3=e4m3)
        part = run_fwd(ops, x[:r], gamma, beta, ("y16", "y32", "stats"), e4m3=e4m3)
        for k in ["y16", "y32", "mean", "rstd"] + (["row_scale"] if e4m3 else []):
            assert_bits_equal(f"{k} {form} D={D} pipe vs occ", part[k], full[k][:r])
        if e4m3:
            assert torch.equal(part["y8"], full["y8"][:r]), f"y8 D={D}: pipe and occ differ"
            print(f"[bound] y8 D={D} pipe vs occ: bit-identical")
        else:
            plain = full
    dy = randn((R, D), 23)
    a1, a2 = randn((R, D), 24), randn((R, D), 25).to(BF16)
    mean, rstd = plain["mean"], plain["rstd"]
    fb, _ = run_bwd(ops, x, gamma, mean, rstd, dy, a1, a2, True, True, True, True)
    pb, _ = run_bwd(ops, x[:r], gamma, mean[:r], rstd[:r], dy[:r], a1[:r], a2[:r], True, True, True, True)
    for k in ("dx", "dx16"):
        assert_bits_equal(f"{k} D={D} pipe vs occ", pb[k], fb[k][:r])


# ---------------------------------------------------------------------------------------------------------- refusals
def _fwd_call(ops, x_ptr, ldx, g, y32, rows, D):
    """egovlp_layernorm_fwd with raw pointers (past ops.layernorm_fwd's own asserts); g serves as gamma and beta."""
    ops.call("egovlp_layernorm_fwd", C.c_void_p(x_ptr), C.c_longlong(ldx), C.c_void_p(0), C.c_void_p(0), ops._ptr(g),
             ops._ptr(g), C.c_void_p(0), ops._ptr(y32), C.c_void_p(0), C.c_void_p(0), rows, D, C.c_float(EPS),
             ops._stream())


def _bwd_call(ops, dy_ptr, dy16, x_ptr, ldx, g, dx, rows, D):
    """egovlp_layernorm_bwd with raw pointers; g serves as gamma, mean and rstd."""
    ops.call("egovlp_layernorm_bwd", C.c_void_p(dy_ptr), dy16, C.c_longlong(D), C.c_void_p(x_ptr), C.c_longlong(ldx),
             ops._ptr(g), ops._ptr(g), ops._ptr(g), C.c_void_p(0), 0, C.c_void_p(0), 0, ops._ptr(dx),
             C.c_longlong(D), C.c_void_p(0), C.c_void_p(0), C.c_void_p(0), C.c_void_p(0), rows, D, ops._stream())


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["D0", "D6", "D1028", "ldx770", "x-off4", "dy32-off4", "dy16-off4"])
def test_bad_arguments_are_refused_and_write_nothing(ops, case):
    """D = 0, D % 4 != 0, D > 1024, ldx % 4 != 0, and a base off the alignment of the kernels' vector accesses (16
    bytes for fp32, 8 for bf16) raise EgovlpError before any launch; rows = 0 is a no-op."""
    from egovlp_b200._lib import EgovlpError
    g = torch.ones(2048, device="cuda")
    rows = 8
    src = torch.ones(rows * 1100 + 8, device="cuda")
    out = nan_filled((rows * 1100 + 8,), F32)
    D = {"D0": 0, "D6": 6, "D1028": 1028}.get(case, 768)
    ldx = 770 if case == "ldx770" else max(D, 4)
    x_ptr = src.data_ptr() + (4 if case == "x-off4" else 0)
    if case.startswith("dy"):
        dy_ptr = src.data_ptr() + 4                      # fp32: 4 bytes off 16; bf16: 4 bytes off 8
        dy16 = int(case == "dy16-off4")
        with pytest.raises(EgovlpError, match="aligned"):
            _bwd_call(ops, dy_ptr, dy16, src.data_ptr(), D, g, out, rows, D)
    else:
        with pytest.raises(EgovlpError, match="aligned" if case == "x-off4" else "bad D"):
            _fwd_call(ops, x_ptr, ldx, g, out, rows, D)
        with pytest.raises(EgovlpError, match="aligned" if case == "x-off4" else "bad D"):
            _bwd_call(ops, src.data_ptr(), 0, x_ptr, ldx, g, out, rows, D)
    torch.cuda.synchronize()
    assert out.isnan().all()
    # rows = 0 with valid arguments: nothing launched, nothing written
    _fwd_call(ops, src.data_ptr(), 768, g, out, 0, 768)
    _bwd_call(ops, src.data_ptr(), 0, src.data_ptr(), 768, g, out, 0, 768)
    torch.cuda.synchronize()
    assert out.isnan().all()
