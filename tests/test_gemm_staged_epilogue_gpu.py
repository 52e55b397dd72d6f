"""The specialised GEMM epilogues move their bytes by TMA (residual / aux subtiles in, outputs out through shared
memory).  These tests cover what that path has to get right beyond the step's shapes: ragged rows and columns
(zero-filled loads, clipped stores), 128-column tiles, outputs that are views of wider buffers, and calls whose
tensors TMA cannot address, which must take the generic epilogue and still compute the same values."""
import pytest
import torch

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
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30)).item()


def run_forms(ops, a, b, wt, bias, res, aux):
    M, N = a.shape[0], b.shape[0]
    outs = []
    o = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, b, o, bias=bias, col_scale=0.125, col_scale_ncols=min(N, 64)); outs.append(o)
    o = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, wt, o, b_mn=True); outs.append(o)
    h, d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16), torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, b, h, bias=bias, act=3, out2=d); outs += [h, d]
    o = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, wt, o, b_mn=True, aux=aux, act=4); outs.append(o)
    o = torch.empty(M, N, device="cuda", dtype=torch.float32)
    ops.gemm(a, b, o, bias=bias, residual=res); outs.append(o)
    o = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, b, o, bias=None, act=1); outs.append(o)
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("M,N,K", [(70, 256, 64), (333, 384, 192), (129, 96, 64), (517, 512, 128)])
def test_staged_epilogues_match_the_generic_one_on_ragged_shapes(ops, monkeypatch, gemm_mode, M, N, K):
    """Rows past M (a warpgroup's or a whole CTA's rows), N % 128 != 0 (partial 64-column subtiles), no bias."""
    a, b, wt = mk((M, K), 40), mk((N, K), 41, 0.06), mk((K, N), 42, 0.06)
    bias, res, aux = mk((N,), 43, dtype=torch.float32), mk((M, N), 44, dtype=torch.float32), mk((M, N), 45)
    monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", "1")
    ref = run_forms(ops, a, b, wt, bias, res, aux)
    monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", "0")
    got = run_forms(ops, a, b, wt, bias, res, aux)
    for i, (r, g) in enumerate(zip(ref, got)):
        assert torch.equal(r, g), i
    assert rel_err(got[5], a.float() @ b.float().t() + bias + res) < 2e-5


def test_staged_epilogue_writes_only_its_view(ops, gemm_mode):
    """Outputs and inputs that are column slices of wider buffers: the TMA stores touch exactly the view."""
    M, N, K = 300, 256, 128
    a, b = mk((M, K), 50), mk((N, K), 51, 0.06)
    bias = mk((N,), 52, dtype=torch.float32)
    rbuf = mk((M, 3 * N), 53, dtype=torch.float32)
    obuf = torch.zeros(M, 3 * N, device="cuda", dtype=torch.float32)
    ops.gemm(a, b, obuf[:, N:2 * N], bias=bias, residual=rbuf[:, 2 * N:])
    acc = a.float() @ b.float().t() + bias
    assert rel_err(obuf[:, N:2 * N], acc + rbuf[:, 2 * N:]) < 2e-5
    assert torch.all(obuf[:, :N] == 0) and torch.all(obuf[:, 2 * N:] == 0)
    hbuf, dbuf = (torch.zeros(M, 2 * N, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    ops.gemm(a, b, hbuf[:, N:], bias=bias, act=3, out2=dbuf[:, :N])
    assert rel_err(hbuf[:, N:], torch.nn.functional.gelu(acc)) < 4e-3
    assert torch.all(hbuf[:, :N] == 0) and torch.all(dbuf[:, N:] == 0)


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
        o = torch.empty(M, N, device="cuda", dtype=torch.float32)
        ops.gemm(a, b, o, bias=bias_buf[:N].clone(), residual=res); outs.append(o)
        o = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
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
