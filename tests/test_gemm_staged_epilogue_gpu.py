"""The specialised GEMM epilogues move their bytes by TMA (residual / aux subtiles in, outputs out through shared
memory).  These tests cover what that path has to get right beyond the step's shapes: ragged rows and columns
(zero-filled loads, clipped stores), 128-column tiles, outputs that are views of wider buffers, and calls whose
tensors TMA cannot address, which must take the generic epilogue and still compute the same values."""
import pytest
import torch
from gemm_ref import assert_outside_untouched, check, check_all, forms_references, reference
from kernel_checks import nan_filled

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


@pytest.fixture(params=["pair", "single"])
def gemm_mode(request, monkeypatch):
    monkeypatch.setenv("EGOVLP_GEMM_PAIR", "1" if request.param == "pair" else "0")
    return request.param


def mk(shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def rel_err(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def run_forms(ops, a, b, wt, bias, res, aux):
    """Every specialised epilogue form -- bias -> bf16 (BF16), GELU + GELU' (ACT3), x aux (MUL_AUX), bias + fp32
    residual (RES_F32), GELU (ACT1) -- first with K-major B (`b`, [N, K]), then with MN-major B (`wt`, [K, N]): ten
    calls, twelve outputs, in the order of gemm_ref.forms_references."""
    M, N = a.shape[0], b.shape[0]
    outs = []
    for bb, b_mn in ((b, False), (wt, True)):
        o = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
        if b_mn:
            ops.gemm(a, bb, o, b_mn=True); outs.append(o)
        else:
            ops.gemm(a, bb, o, bias=bias, col_scale=0.125, col_scale_ncols=min(N, 64)); outs.append(o)
        h, d = nan_filled((M, N), torch.bfloat16), nan_filled((M, N), torch.bfloat16)
        ops.gemm(a, bb, h, b_mn=b_mn, bias=bias, act=3, out2=d); outs += [h, d]
        o = nan_filled((M, N), torch.bfloat16)
        ops.gemm(a, bb, o, b_mn=b_mn, aux=aux, act=4); outs.append(o)
        o = nan_filled((M, N), torch.float32)
        ops.gemm(a, bb, o, b_mn=b_mn, bias=bias, residual=res); outs.append(o)
        o = nan_filled((M, N), torch.bfloat16)
        ops.gemm(a, bb, o, b_mn=b_mn, bias=None, act=1); outs.append(o)
    torch.cuda.synchronize()
    return outs


# M ragged for a warpgroup's or a whole CTA's rows; N = 384 runs 128-column tiles and N = 512 256-column ones (CTA pairs
# under the fixture); K = 72 and 200 end in a partial k-block that TMA zero-fills
@pytest.mark.parametrize("M,N,K", [(70, 256, 64), (333, 384, 192), (129, 96, 64), (517, 512, 128), (190, 256, 72),
                                   (301, 384, 200)])
def test_staged_epilogues_match_the_generic_one_on_ragged_shapes(ops, monkeypatch, gemm_mode, M, N, K):
    """All ten (form, B layout) pairs: bit for bit against the generic epilogue, within the GEMM tolerances of fp64
    (bf16 outputs rel-L2 4e-3, fp32 outputs 2e-5) and element-wise within gemm_ref's bound.  Rows past M,
    N % 128 != 0 (partial 64-column subtiles), no bias."""
    a, b = mk((M, K), 40), mk((N, K), 41, 0.06)
    wt = b.t().contiguous()
    bias, res, aux = mk((N,), 43, dtype=torch.float32), mk((M, N), 44, dtype=torch.float32), mk((M, N), 45)
    monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", "1")
    ref = run_forms(ops, a, b, wt, bias, res, aux)
    monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", "0")
    got = run_forms(ops, a, b, wt, bias, res, aux)
    assert len(got) == 12
    for i, (r, g, want) in enumerate(zip(ref, got, forms_references(a, b, bias, res, aux))):
        assert torch.equal(r, g), i
        tol = 2e-5 if g.dtype == torch.float32 else 4e-3
        assert rel_err(g, want[0]) < tol, (i, rel_err(g, want[0]))
        check(f"staged form {i} {(M, N, K)} {gemm_mode}", g, want)


@pytest.mark.parametrize("K", [2304, 3072])
@pytest.mark.parametrize("M", [117, 512])
def test_residual_f32_with_mn_major_b_at_text_backward_shapes(ops, monkeypatch, gemm_mode, M, K):
    """dx = dy @ W + fp32 residual with W stored [K, N]: the text tower's backward runs it twice per layer (the lin1
    input gradient plus the residual path, K = 3072, and the q|k|v input gradient plus the attention branch, K = 2304)."""
    N = 768
    a, w, res = mk((M, K), 70), mk((K, N), 71, 0.03), mk((M, N), 72, dtype=torch.float32)

    def run():
        o = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float32)
        ops.gemm(a, w, o, b_mn=True, residual=res)
        torch.cuda.synchronize()
        return o

    monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", "1")
    ref = run()
    monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", "0")
    got = run()
    assert torch.equal(ref, got)
    assert rel_err(got, a.double() @ w.double() + res.double()) < 2e-5
    check(f"residual fp32, MN-major B {(M, K)} {gemm_mode}", got, reference(a, w, b_mn=True, residual=res)["out"])


def test_staged_epilogue_writes_only_its_view(ops, gemm_mode):
    """Outputs and inputs that are column slices of wider buffers: the TMA stores touch exactly the view."""
    M, N, K = 300, 256, 128
    a, b = mk((M, K), 50), mk((N, K), 51, 0.06)
    bias = mk((N,), 52, dtype=torch.float32)
    rbuf = mk((M, 3 * N), 53, dtype=torch.float32)
    obuf = nan_filled((M, 3 * N), torch.float32)
    ops.gemm(a, b, obuf[:, N:2 * N], bias=bias, residual=rbuf[:, 2 * N:])
    acc = a.float() @ b.float().t() + bias
    assert rel_err(obuf[:, N:2 * N], acc + rbuf[:, 2 * N:]) < 2e-5
    assert_outside_untouched(f"residual fp32 view {gemm_mode}", obuf, (slice(None), slice(N, 2 * N)))
    check(f"residual fp32 view {gemm_mode}", obuf[:, N:2 * N], reference(a, b, bias=bias, residual=rbuf[:, 2 * N:])["out"])
    hbuf, dbuf = nan_filled((M, 2 * N), torch.bfloat16), nan_filled((M, 2 * N), torch.bfloat16)
    ops.gemm(a, b, hbuf[:, N:], bias=bias, act=3, out2=dbuf[:, :N])
    assert rel_err(hbuf[:, N:], torch.nn.functional.gelu(acc)) < 4e-3
    assert_outside_untouched(f"act 3 view {gemm_mode}", hbuf, (slice(None), slice(N, None)))
    assert_outside_untouched(f"act 3 out2 view {gemm_mode}", dbuf, (slice(None), slice(None, N)))
    check_all(f"act 3 views {gemm_mode}", {"out": hbuf[:, N:], "out2": dbuf[:, :N]},
              reference(a, b, bias=bias, act=3, out2=True))


def test_calls_tma_cannot_address_take_the_generic_epilogue(ops, monkeypatch, gemm_mode):
    """Base addresses 8 bytes off 16 or row strides not a multiple of 16 bytes (bf16 output, fp32 residual, bias, aux):
    the call is routed to the generic epilogue and computes the same values as the generic epilogue does by choice."""
    M, N, K = 260, 256, 128
    a, b, wt = mk((M, K), 60), mk((N, K), 61, 0.06), mk((K, N), 62, 0.06)
    # the generic epilogue reads bias / residual as float2 and aux as bf16x2: 8- and 4-byte alignment stay required
    bias_buf = mk((N + 2,), 63, dtype=torch.float32)
    bias = bias_buf[2:]                                         # 8 bytes off 16
    res_buf = mk((M, N + 2), 64, dtype=torch.float32)
    res = res_buf[:, :N]                                        # row stride (N + 2) * 4 bytes
    aux_buf = mk((M, N + 8), 65)
    aux = aux_buf[:, 4:4 + N]                                   # 8 bytes off 16

    def run():
        outs = []
        obuf = torch.zeros(M, N + 16, device="cuda", dtype=torch.bfloat16)
        ops.gemm(a, b, obuf[:, 4:4 + N], bias=bias); outs.append(obuf)            # output 8 bytes off 16
        o = nan_filled((M, N), torch.float32)
        ops.gemm(a, b, o, bias=bias_buf[:N].clone(), residual=res); outs.append(o)
        o = nan_filled((M, N), torch.bfloat16)
        ops.gemm(a, wt, o, b_mn=True, aux=aux, act=4); outs.append(o)
        torch.cuda.synchronize()
        return outs

    monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", "1")
    ref = run()
    monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", "0")
    got = run()
    for i, (r, g) in enumerate(zip(ref, got)):
        assert torch.equal(r, g), i
    acc = a.float() @ b.float().t()
    assert rel_err(got[0][:, 4:4 + N], acc + bias) < 4e-3
    assert torch.all(got[0][:, :4] == 0) and torch.all(got[0][:, 4 + N:] == 0)
    assert rel_err(got[1], acc + bias_buf[:N] + res) < 2e-5
    assert rel_err(got[2], (a.float() @ wt.float()) * aux.float()) < 4e-3
    name = f"TMA-unaddressable {gemm_mode}"
    check(f"{name} bf16 view", got[0][:, 4:4 + N], reference(a, b, bias=bias)["out"])
    check(f"{name} residual fp32", got[1], reference(a, b, bias=bias_buf[:N], residual=res)["out"])
    check(f"{name} x aux", got[2], reference(a, wt, b_mn=True, aux=aux, act=4)["out"])
