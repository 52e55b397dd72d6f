"""Per-kernel parity on the GPU: every CUDA op against a plain torch fp32 restatement of the same op
(called through the C-ABI via egovlp_b200.ops).  The divided attention is checked against the fp64 reference of
test_divided_attention_gpu.py (divided_attention_ref.py), element by element, and every GEMM output against the fp64
reference and bound of gemm_ref.py, element by element, beside the relative-L2 checks."""
import pytest
import torch
from divided_attention_ref import check_case
from gemm_ref import check, check_all, gelu_tail_inputs, reference, spread
from kernel_checks import nan_filled

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


@pytest.fixture(params=["pair", "single"])
def gemm_mode(request, monkeypatch):
    """Run every GEMM test on both tile schedulers: single CTAs (the default) and CTA pairs (a 2-CTA cluster, 256 x 256
    tile, B multicast; taken by K-major A with N % 256 == 0 under EGOVLP_GEMM_PAIR=1)."""
    monkeypatch.setenv("EGOVLP_GEMM_PAIR", "1" if request.param == "pair" else "0")
    return request.param


def rel_err(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30)).item()


def mk(shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def past_k(x, ld=64):
    """x as the first columns of a [rows, ld] buffer whose other columns hold 1e4: a read past K cannot hide."""
    buf = torch.full((x.shape[0], ld), 1e4, device="cuda", dtype=x.dtype)
    buf[:, :x.shape[1]] = x
    return buf[:, :x.shape[1]]


# K = 8 and 40: one partial k-block; K = 20: a view with row stride 64 (K itself is not a multiple of 8)
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 768), (300, 768, 768), (1570, 2304, 768),
                                   (130, 128, 64), (200, 64, 128), (1000, 3072, 768), (257, 768, 3072), (64, 32, 64),
                                   (300, 256, 8), (200, 384, 40), (130, 512, 20)])
def test_gemm_kmajor_bias(ops, M, N, K, gemm_mode):
    a, b = mk((M, K), 1), mk((N, K), 2, 0.05)
    if K % 8:
        a, b = past_k(a), past_k(b)
    bias = mk((N,), 3, dtype=torch.float32)
    want = reference(a, b, bias=bias)["out"]
    out = nan_filled((M, N), torch.bfloat16)
    ops.gemm(a, b, out, bias=bias)
    ref = a.float() @ b.float().t() + bias
    assert rel_err(out, ref) < 4e-3
    check(f"gemm bias bf16 {(M, N, K)} {gemm_mode}", out, want)
    out32 = nan_filled((M, N), torch.float32)
    ops.gemm(a, b, out32, bias=bias)
    assert rel_err(out32, ref) < 2e-5
    check(f"gemm bias fp32 {(M, N, K)} {gemm_mode}", out32, want)


@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (300, 768, 2304), (1000, 3072, 768), (200, 64, 128)])
def test_gemm_b_mn_major_dgrad(ops, M, N, K, gemm_mode):
    """dx = dy @ W with W stored [K, N] (n contiguous): the dgrad form."""
    a, w = mk((M, K), 4), mk((K, N), 5, 0.05)
    out = nan_filled((M, N), torch.float32)
    ops.gemm(a, w, out, b_mn=True)
    assert rel_err(out, a.float() @ w.float()) < 2e-5
    check(f"gemm dgrad fp32 {(M, N, K)} {gemm_mode}", out, reference(a, w, b_mn=True)["out"])


@pytest.mark.parametrize("Mtok,N,Kin,split", [(512, 256, 256, 1), (1000, 768, 768, 4), (3137, 2304, 768, 7),
                                              (777, 128, 64, 3)])
def test_gemm_both_mn_major_wgrad(ops, Mtok, N, Kin, split, gemm_mode):
    """dW[N,Kin] += dy^T x : contraction over tokens, both operands token-major; split-K atomics."""
    mt = (Mtok + 7) // 8 * 8
    dy, x = mk((mt, N), 6), mk((mt, Kin), 7)
    dy[Mtok:] = 0
    base = mk((N, Kin), 8, dtype=torch.float32)
    out = base.clone()
    ops.gemm(dy, x, out, a_mn=True, b_mn=True, accumulate=True, split_k=split)
    ref = base + dy.float().t() @ x.float()
    assert rel_err(out, ref) < 2e-5
    name = f"gemm wgrad {(Mtok, N, Kin, split)} {gemm_mode}"
    check(name, out, reference(dy, x, a_mn=True, b_mn=True, base=base, split_k=split)["out"])
    if Kin % 256 == 0:        # fused bias gradient: column sums of dy taken from the smem tiles of the same GEMM
        out2, db = base.clone(), torch.full((N,), 0.5, device="cuda")
        db0 = db.clone()
        ops.gemm(dy, x, out2, a_mn=True, b_mn=True, accumulate=True, split_k=split, colsum_a=db)
        assert rel_err(out2, ref) < 2e-5
        assert rel_err(db, 0.5 + dy.float().sum(0)) < 1e-5
        check_all(name + " + colsum_a", {"out": out2, "colsum_a": db},
                  reference(dy, x, a_mn=True, b_mn=True, base=base, split_k=split, colsum_a=db0))


@pytest.mark.parametrize("inputs", ["randn", "tails"])
def test_gemm_epilogues(ops, gemm_mode, inputs):
    """Every epilogue of the generic form and the forms beside it, each output element-wise against fp64.  "tails": rows
    of A scaled so that the pre-activations reach about +-10 with exact zeros among them, and an aux uniform in
    [-10, 10] with zeros, so that GELU and GELU' are checked where few elements of random inputs lie."""
    M, N, K = 515, 768, 256
    a, b = mk((M, K), 9), mk((N, K), 10, 0.06)
    bias = mk((N,), 11, dtype=torch.float32)
    res = mk((M, N), 12, dtype=torch.float32)
    aux = mk((M, N), 13)
    if inputs == "tails":
        a, bias = gelu_tail_inputs(a, bias)
        aux = spread((M, N), 13)
    name = f"gemm epilogue {inputs} {gemm_mode}"
    acc = a.float() @ b.float().t() + bias
    # bias + residual -> fp32
    out = nan_filled((M, N), torch.float32)
    ops.gemm(a, b, out, bias=bias, residual=res)
    assert rel_err(out, acc + res) < 2e-5
    check(f"{name} residual fp32", out, reference(a, b, bias=bias, residual=res)["out"])
    # bias + gelu, pre-activation saved
    h = nan_filled((M, N), torch.bfloat16)
    u = nan_filled((M, N), torch.bfloat16)
    ops.gemm(a, b, h, bias=bias, act=1, out2=u)
    assert rel_err(u, acc) < 4e-3
    assert rel_err(h, torch.nn.functional.gelu(acc)) < 4e-3
    check_all(f"{name} act 1", {"out": h, "out2": u}, reference(a, b, bias=bias, act=1, out2=True))
    # multiply by gelu'(aux)
    out = nan_filled((M, N), torch.float32)
    ops.gemm(a, b, out, aux=aux, act=2)
    x = aux.float().requires_grad_(True)
    torch.nn.functional.gelu(x).sum().backward()
    assert rel_err(out, (a.float() @ b.float().t()) * x.grad) < 1e-4
    check(f"{name} act 2 fp32", out, reference(a, b, aux=aux, act=2)["out"])
    # same, bf16 output + fused column sums (the fc1 bias gradient)
    out16 = nan_filled((M, N), torch.bfloat16)
    cs = torch.ones(N, device="cuda")
    ops.gemm(a, b, out16, aux=aux, act=2, colsum=cs)
    assert rel_err(out16, out) < 4e-3
    assert rel_err(cs, 1 + out.sum(0)) < 1e-4
    check_all(f"{name} act 2 bf16", {"out": out16, "colsum": cs},
              reference(a, b, aux=aux, act=2, colsum=torch.ones(N, device="cuda")))
    # the Mlp pair of the training step: act 3 = GELU with its derivative saved to out2, act 4 = multiply by aux
    h3, d3 = nan_filled((M, N), torch.bfloat16), nan_filled((M, N), torch.bfloat16)
    ops.gemm(a, b, h3, bias=bias, act=3, out2=d3)
    accg = acc.clone().requires_grad_(True)
    torch.nn.functional.gelu(accg).sum().backward()
    assert torch.equal(h3, h)
    assert rel_err(d3, accg.grad) < 4e-3
    check_all(f"{name} act 3", {"out": h3, "out2": d3}, reference(a, b, bias=bias, act=3, out2=True))
    out4 = nan_filled((M, N), torch.bfloat16)
    cs4 = torch.ones(N, device="cuda")
    ops.gemm(a, b, out4, aux=d3, act=4, colsum=cs4)
    ref4 = (a.float() @ b.float().t()) * d3.float()
    assert rel_err(out4, ref4) < 4e-3 and rel_err(cs4, 1 + ref4.sum(0)) < 1e-4
    check_all(f"{name} act 4", {"out": out4, "colsum": cs4},
              reference(a, b, aux=d3, act=4, colsum=torch.ones(N, device="cuda")))
    # q-scale on the first 256 columns
    out = nan_filled((M, N), torch.float32)
    ops.gemm(a, b, out, bias=bias, col_scale=0.125, col_scale_ncols=256)
    ref = acc.clone(); ref[:, :256] *= 0.125
    assert rel_err(out, ref) < 2e-5
    check(f"{name} column scale fp32", out, reference(a, b, bias=bias, col_scale=0.125, col_scale_ncols=256)["out"])


# the training step's shapes at M = 2 x 3137 and 6 x 3137 tokens (qkv, fc1, fc2 forward and fc1 dgrad), and a 128-column
# one: at least 3 tiles per CTA (per CTA pair when pairs run), so that the bias row, the epilogue buffers and the stage
# ring are reused across tiles with their phase bits flipping
STEP_SHAPES = [(6274, 2304, 768), (6274, 3072, 768), (18822, 768, 3072), (17000, 384, 256)]


@pytest.mark.parametrize("M,N,K", [(1570, 768, 256), (515, 3072, 768), (4099, 1024, 128)] + STEP_SHAPES)
def test_gemm_specialised_epilogues_match_the_generic_one(ops, monkeypatch, gemm_mode, M, N, K):
    """The K-major-A kernels carry compile-time specialised epilogues for the step's hot forms (bias -> bf16, GELU + GELU',
    x aux, bias + fp32 residual -> fp32); EGOVLP_GEMM_GENERIC_EPI=1 routes the same calls through the generic epilogue.
    Same arithmetic in the same order: the results must be bit-identical (ragged last m-block, several tiles per CTA),
    and every output is held element-wise to fp64."""
    if (M, N, K) in STEP_SHAPES:
        pair = gemm_mode == "pair" and N % 256 == 0
        tile_m, tile_n = (256, 256) if pair else (128, 256 if N % 256 == 0 else 128)
        sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
        tiles = -(-M // tile_m) * -(-N // tile_n)
        assert tiles >= 3 * (sms // 2 if pair else sms), (tiles, sms, pair)
    a, b = mk((M, K), 30), mk((N, K), 31, 0.06)
    wt = mk((K, N), 32, 0.06)                      # MN-major B (dgrad form)
    bias = mk((N,), 33, dtype=torch.float32)
    res = mk((M, N), 34, dtype=torch.float32)
    aux = mk((M, N), 35)
    bf, f32 = torch.bfloat16, torch.float32

    def run():
        outs = []
        o = nan_filled((M, N), bf)
        ops.gemm(a, b, o, bias=bias, col_scale=0.125, col_scale_ncols=256); outs.append(o)            # EPI_BF16
        o = nan_filled((M, N), bf)
        ops.gemm(a, wt, o, b_mn=True); outs.append(o)                                                  # EPI_BF16, dgrad
        h, d = nan_filled((M, N), bf), nan_filled((M, N), bf)
        ops.gemm(a, b, h, bias=bias, act=3, out2=d); outs += [h, d]                                     # EPI_ACT3
        o = nan_filled((M, N), bf)
        ops.gemm(a, wt, o, b_mn=True, aux=aux, act=4); outs.append(o)                                   # EPI_MUL_AUX
        o = nan_filled((M, N), f32)
        ops.gemm(a, b, o, bias=bias, residual=res); outs.append(o)                                      # EPI_RES_F32
        o = nan_filled((M, N), bf)
        ops.gemm(a, b, o, bias=bias, act=1); outs.append(o)                                             # EPI_ACT1
        torch.cuda.synchronize()
        return outs

    monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", "1")
    ref = run()
    monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", "0")
    got = run()
    for i, (r, g) in enumerate(zip(ref, got)):
        assert torch.equal(r, g), i
    acc = a.float() @ b.float().t() + bias
    assert rel_err(got[5], acc + res) < 2e-5
    assert rel_err(got[2], torch.nn.functional.gelu(acc)) < 4e-3
    assert torch.equal(got[6], got[2])             # inference-form GELU == the training form's first output
    assert rel_err(got[4], (a.float() @ wt.float()) * aux.float()) < 4e-3
    del acc, ref
    name = f"gemm {(M, N, K)} {gemm_mode}"
    check(f"{name} bf16 + column scale", got[0], reference(a, b, bias=bias, col_scale=0.125, col_scale_ncols=256)["out"])
    check(f"{name} bf16 dgrad", got[1], reference(a, wt, b_mn=True)["out"])
    check_all(f"{name} act 3", {"out": got[2], "out2": got[3]}, reference(a, b, bias=bias, act=3, out2=True))
    check(f"{name} x aux dgrad", got[4], reference(a, wt, b_mn=True, aux=aux, act=4)["out"])
    check(f"{name} residual fp32", got[5], reference(a, b, bias=bias, residual=res)["out"])
    check(f"{name} act 1", got[6], reference(a, b, bias=bias, act=1)["out"])


def test_gemm_strided_views(ops, gemm_mode):
    """Operands / outputs that are column slices of wider buffers (ld > width)."""
    M, N, K = 384, 256, 192
    abuf, bbuf = mk((M, 3 * K), 14), mk((N, 2 * K), 15, 0.05)
    obuf = torch.zeros(M, 2 * N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(abuf[:, K:2 * K], bbuf[:, K:], obuf[:, N:])
    assert rel_err(obuf[:, N:], abuf[:, K:2 * K].float() @ bbuf[:, K:].float().t()) < 4e-3
    assert torch.all(obuf[:, :N] == 0)
    check(f"gemm strided views {gemm_mode}", obuf[:, N:], reference(abuf[:, K:2 * K], bbuf[:, K:])["out"])


@pytest.mark.parametrize("rows,D", [(1000, 768), (37, 64), (785 * 2, 768), (5, 128), (4999, 768), (6001, 128),
                                    (3137 * 4, 768)])
def test_layernorm_fwd_bwd(ops, rows, D):
    """rows >= 4096 with D % 128 == 0 take the bulk-copy pipelined kernels (ragged last tile at 4999 / 6001 rows)."""
    x = mk((rows, D), 20, 2.0, torch.float32) + 0.3
    g, b = mk((D,), 21, dtype=torch.float32) * 0.1 + 1, mk((D,), 22, dtype=torch.float32) * 0.1
    y16 = torch.empty(rows, D, device="cuda", dtype=torch.bfloat16)
    y32 = torch.empty(rows, D, device="cuda", dtype=torch.float32)
    mean, rstd = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
    ops.layernorm_fwd(x, g, b, 1e-6, y16=y16, y32=y32, mean=mean, rstd=rstd)
    xr = x.clone().requires_grad_(True)
    gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(xr, (D,), gr, br, 1e-6)
    assert rel_err(y32, ref) < 1e-5 and rel_err(y16, ref) < 4e-3
    dy = mk((rows, D), 23, dtype=torch.float32)
    dy16 = dy.to(torch.bfloat16)
    a1, a2 = mk((rows, D), 24, dtype=torch.float32), mk((rows, D), 25, dtype=torch.float32)
    ref.backward(dy)
    dx = torch.empty_like(x)
    dx16 = torch.empty(rows, D, device="cuda", dtype=torch.bfloat16)
    dg, db = torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    ops.layernorm_bwd(dy, x, g, mean, rstd, add1=a1, add2=a2, dx=dx, dx16=dx16, dgamma=dg, dbeta=db)
    assert rel_err(dx, xr.grad + a1 + a2) < 1e-5
    assert rel_err(dx16, xr.grad + a1 + a2) < 4e-3
    assert rel_err(dg, gr.grad) < 1e-4 and rel_err(db, br.grad) < 1e-4
    # bf16 upstream gradient (what the dgrad GEMMs hand over)
    ref2 = torch.nn.functional.layer_norm(xr2 := x.clone().requires_grad_(True), (D,), g, b, 1e-6)
    ref2.backward(dy16.float())
    ops.layernorm_bwd(dy16, x, g, mean, rstd, dx=dx)
    assert rel_err(dx, xr2.grad) < 1e-5
    # bf16 residual-gradient addends (block-internal d space/time residual)
    a1h, a2h = a1.to(torch.bfloat16), a2.to(torch.bfloat16)
    ops.layernorm_bwd(dy16, x, g, mean, rstd, add1=a1h, add2=a2h, dx=dx, dx16=dx16)
    assert rel_err(dx, xr2.grad + a1h.float() + a2h.float()) < 1e-5
    cs = torch.ones(D, device="cuda")
    ops.layernorm_bwd(dy16, x, g, mean, rstd, add1=a1, add2=a2h, dx16=dx16, colsum_dx=cs)   # mixed dtypes, bf16-only output
    assert rel_err(dx16, xr2.grad + a1 + a2h.float()) < 4e-3
    assert rel_err(cs, 1 + (xr2.grad + a1 + a2h.float()).sum(0)) < 1e-4


def test_layernorm_fused_add(ops):
    rows, D = 300, 768
    x, a = mk((rows, D), 30, dtype=torch.float32), mk((rows, D), 31, dtype=torch.float32)
    g, b = torch.ones(D, device="cuda"), torch.zeros(D, device="cuda")
    s = torch.empty_like(x); y = torch.empty_like(x)
    ops.layernorm_fwd(x, g, b, 1e-12, add=a, sum_out=s, y32=y)
    assert torch.equal(s, x + a)
    assert rel_err(y, torch.nn.functional.layer_norm(x + a, (D,), g, b, 1e-12)) < 1e-5


def test_cast_and_colsum(ops):
    w = mk((1000, 771), 40, dtype=torch.float32)
    assert torch.equal(ops.cast_bf16(w), w.to(torch.bfloat16))
    for dt in (torch.float32, torch.bfloat16):
        dy = mk((3137, 768), 41, dtype=dt)
        out = torch.ones(768, device="cuda")
        ops.colsum_accum(dy, out)
        assert rel_err(out, 1 + dy.float().sum(0)) < 1e-5


@pytest.mark.parametrize("generic", [False, True, "tc", "w8"])
@pytest.mark.parametrize("B,T,N,H,mode", [(2, 4, 196, 2, 1), (2, 4, 196, 2, 0), (1, 16, 196, 1, 0), (1, 16, 196, 1, 1),
                                          (2, 3, 4, 2, 0), (2, 3, 4, 2, 1), (3, 8, 50, 1, 0), (2, 1, 30, 1, 0),
                                          (2, 5, 196, 1, 0), (2, 8, 196, 1, 0), (1, 8, 196, 2, 1), (2, 16, 100, 1, 0),
                                          (2, 4, 30, 1, 0), (2, 2, 20, 1, 1), (3, 16, 196, 8, 1), (2, 4, 150, 2, 1)])
def test_divided_attention_fwd_bwd(ops, B, T, N, H, mode, generic, monkeypatch):
    """Both implementations (specialised span kernels; generic group-id kernels), incl. partially filled time groups
    (N not a multiple of the patches per group), with q_scale = 0.125 as the engine passes it.  Every element of out,
    lse and dq | dk | dv is held to the bounds of test_divided_attention_gpu.py, outputs land in NaN-filled buffers
    with sentinel rows; the relative L2 bounds below are kept on top of those."""
    # False: default dispatch (mma.sync span kernels); True: generic group-id kernels; "tc": + the wgmma space-attention
    # forward (128 < N + 1 <= 208); "w8": the 8-warp time backward ("tc" on a time shape and "w8" on a space shape run
    # the default dispatch).  (3, 16, 196, 8, 1) has 384 groups; (2, 4, 150, 2, 1) has 151 keys: a partly filled last
    # key tile.
    path = {False: "default", True: "generic", "tc": "tc", "w8": "w8"}[generic]
    out, dqkv, r = check_case(ops, monkeypatch, B, T, N, H, mode, path, seed=50 + T + mode)
    S, D = 1 + T * N, 64 * H
    assert rel_err(out, r["out"]) < 6e-3
    for i, name in enumerate(("dq", "dk", "dv")):
        assert rel_err(dqkv[:, i * D:(i + 1) * D], r[name]) < 1.5e-2, name
    # CLS rows on their own (summed over every group)
    cls = torch.arange(B, device="cuda") * S
    assert rel_err(dqkv[cls], torch.cat([r["dq"], r["dk"], r["dv"]], 1)[cls]) < 1.5e-2
    assert rel_err(out[cls], r["out"][cls]) < 6e-3
