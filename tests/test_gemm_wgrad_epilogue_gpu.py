"""The weight-gradient GEMM (MN-major dy and x, split-K) adds each unit's fp32 partial tile into dW through shared
memory with a TMA reduce (EPI_RED_F32).  These tests cover what that path has to get right: ragged n_out / n_in
(clipped reduces), 128-column tiles, token counts that are not whole k-blocks, accumulation onto a non-zero dW, the
fused bias gradient, dW views inside wider buffers, and dW tensors TMA cannot address, which take the generic epilogue."""
import pytest
import torch
from gemm_ref import check, check_all, reference

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


def mk(shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def rel_err(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def operands(tokens, n_out, n_in):
    return mk((tokens, n_out), 6), mk((tokens, n_in), 7)


# (tokens, n_out, n_in, split): the shapes of test_kernels_gpu's wgrad test, then ragged n_out (not a multiple of 128),
# n_in = 32 / 96 (128-column tiles, partly outside dW) and 768 / 3072, token counts that are not multiples of 64
SHAPES = [(512, 256, 256, 1), (1000, 768, 768, 4), (3144, 2304, 768, 7), (784, 128, 64, 3),
          (1000, 200, 32, 1), (1000, 200, 96, 3), (1096, 136, 768, 5), (2056, 768, 3072, 9), (520, 3072, 768, 2),
          (4104, 776, 256, 6)]


@pytest.mark.parametrize("tokens,n_out,n_in,split", SHAPES)
@pytest.mark.parametrize("base", ["zero", "nonzero"])
def test_wgrad_matches_fp64(ops, tokens, n_out, n_in, split, base):
    dy, x = operands(tokens, n_out, n_in)
    b0 = mk((n_out, n_in), 8, dtype=torch.float32) if base == "nonzero" else torch.zeros(n_out, n_in, device="cuda")
    ref = b0.double() + dy.double().t() @ x.double()
    dw = b0.clone()
    ops.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=split)
    assert rel_err(dw, ref) < 2e-5
    name = f"wgrad {(tokens, n_out, n_in, split)} {base}"
    check(name, dw, reference(dy, x, a_mn=True, b_mn=True, base=b0, split_k=split)["out"])
    if n_in % 256 == 0:       # the fused bias gradient (column sums of dy) beside the reduce epilogue
        dw2, db = b0.clone(), torch.full((n_out,), 0.5, device="cuda")
        ops.gemm(dy, x, dw2, a_mn=True, b_mn=True, accumulate=True, split_k=split, colsum_a=db)
        assert rel_err(dw2, ref) < 2e-5
        assert rel_err(db, 0.5 + dy.double().sum(0)) < 1e-5
        check_all(name + " + colsum_a", {"out": dw2, "colsum_a": db},
                  reference(dy, x, a_mn=True, b_mn=True, base=b0, split_k=split,
                            colsum_a=torch.full((n_out,), 0.5, device="cuda")))


@pytest.mark.parametrize("tokens,n_out,n_in", [(3144, 2304, 768), (1000, 200, 96), (784, 128, 64), (2056, 768, 3072)])
@pytest.mark.parametrize("base", ["zero", "nonzero"])
def test_wgrad_single_split_is_bitwise_the_generic_epilogue(ops, monkeypatch, tokens, n_out, n_in, base):
    """One split adds each dW element once, so the TMA reduce and the generic epilogue's red.add give the same bits."""
    dy, x = operands(tokens, n_out, n_in)
    b0 = mk((n_out, n_in), 9, dtype=torch.float32) if base == "nonzero" else torch.zeros(n_out, n_in, device="cuda")
    outs = []
    for generic in ("1", "0"):
        monkeypatch.setenv("EGOVLP_GEMM_GENERIC_EPI", generic)
        dw = b0.clone()
        ops.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=1)
        outs.append(dw)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    check(f"wgrad one split {(tokens, n_out, n_in)} {base}", outs[1],
          reference(dy, x, a_mn=True, b_mn=True, base=b0)["out"])


@pytest.mark.parametrize("n_out,n_in,split", [(200, 96, 3), (776, 256, 4), (136, 768, 2)])
def test_wgrad_into_a_view_leaves_the_rest_of_the_buffer(ops, n_out, n_in, split):
    """dW is a window of a NaN-filled buffer with a wider row stride: the reduces are clipped to n_out x n_in."""
    dy, x = operands(1000, n_out, n_in)
    buf = torch.full((n_out + 40, n_in + 72), float("nan"), device="cuda")
    dw = buf[24:24 + n_out, 32:32 + n_in]
    dw.zero_()
    ops.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=split)
    assert rel_err(dw, dy.double().t() @ x.double()) < 2e-5
    check(f"wgrad view {(n_out, n_in, split)}", dw,
          reference(dy, x, a_mn=True, b_mn=True, base=torch.zeros_like(dw), split_k=split)["out"])
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[24:24 + n_out, 32:32 + n_in] = False
    assert buf[outside].isnan().all()


@pytest.mark.parametrize("n_out,n_in,split", [(256, 256, 3), (200, 96, 2)])
def test_wgrad_dw_tma_cannot_address_takes_the_generic_epilogue(ops, n_out, n_in, split):
    """A dW base 8 bytes off a 16-byte boundary cannot be a TMA tensor: the call must still compute dW (generic path)."""
    dy, x = operands(1000, n_out, n_in)
    ld = n_in + 8
    flat = torch.zeros(n_out * ld + 8, device="cuda")
    dw = flat[2:2 + n_out * ld].view(n_out, ld)[:, :n_in]
    assert dw.data_ptr() % 16 == 8
    b0 = mk((n_out, n_in), 10, dtype=torch.float32)
    dw.copy_(b0)
    ops.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=split)
    assert rel_err(dw, b0.double() + dy.double().t() @ x.double()) < 2e-5
    check(f"wgrad TMA-unaddressable {(n_out, n_in, split)}", dw,
          reference(dy, x, a_mn=True, b_mn=True, base=b0, split_k=split)["out"])
