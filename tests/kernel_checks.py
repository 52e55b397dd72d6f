"""Check helpers shared by the per-kernel reference tests (test_front_end_kernels_gpu.py, test_divided_attention_gpu.py).

Each check compares a kernel's output with a float64 reference at the bound the kernel's arithmetic allows, and prints
its worst element or row as a fraction of that bound (run pytest with -s to see them)."""
import torch

F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64


def mk(shape, seed, scale=1.0, dtype=BF16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def nan_filled(shape, dtype):
    return torch.full(shape, float("nan"), device="cuda", dtype=dtype)


def rel_l2(got, ref):
    ref = ref.double()
    return ((got.double() - ref).norm() / ref.norm().clamp_min(1e-300)).item()


def _worst(name, ratio):
    """Largest error / bound ratio of `ratio` (NaN if any is NaN) and where it is; printed for the record."""
    flat = ratio.flatten()
    nan = flat.isnan()
    i = int(nan.nonzero()[0, 0]) if nan.any() else int(flat.argmax())
    worst = flat[i].item()
    at = tuple(int(j) for j in torch.unravel_index(torch.tensor(i), ratio.shape))
    print(f"[bound] {name}: worst {worst:.3g} of the bound at {at}")
    return worst, at


def assert_bits_equal(name, got, ref):
    """Same dtype, same bit patterns."""
    assert got.dtype == ref.dtype and got.shape == ref.shape, (name, got.dtype, ref.dtype, got.shape, ref.shape)
    as_int = {F32: torch.int32, BF16: torch.int16}[got.dtype]
    same = got.contiguous().view(as_int) == ref.contiguous().view(as_int)
    if not bool(same.all()):
        i = int((~same).flatten().nonzero()[0, 0])
        at = tuple(int(j) for j in torch.unravel_index(torch.tensor(i), got.shape))
        raise AssertionError(f"{name}: {int((~same).sum())} elements differ, first at {at}: got {got[at].item()!r}, "
                             f"want {ref[at].item()!r}")
    print(f"[bound] {name}: bit-identical")


def _ordered_bf16(x):
    """bf16 bit patterns as integers in value order (neighbouring values differ by 1; +0 and -0 both map to 0)."""
    b = x.contiguous().view(torch.int16).int()
    return torch.where(b < 0, -(b & 0x7FFF), b)


def assert_bf16_ulps(name, got16, ref64, ulps=1):
    """got16 (bf16) is at most `ulps` bf16 steps from the exact value ref64 rounded to bf16."""
    steps = (_ordered_bf16(got16) - _ordered_bf16(ref64.to(BF16))).abs().double()
    worst, at = _worst(name, steps / ulps)
    assert worst <= 1.0, f"{name}: {steps[at].item():.0f} bf16 ulps at {at}: got {got16[at].item()}, exact {ref64[at].item()}"


def assert_sum_bound(name, got, ref, abs_terms, rel=4e-5):
    """Element-wise |got - ref| <= rel * abs_terms + 1e-30, abs_terms = the same sum taken over the terms' magnitudes."""
    err = (got.double() - ref).abs()
    bound = rel * abs_terms + 1e-30
    worst, at = _worst(name, err / bound)
    assert worst <= 1.0, (f"{name}: |got - ref| = {err[at].item():.3e} > {bound[at].item():.3e} at {at} "
                          f"(got {got[at].item()}, ref {ref[at].item()}, sum|terms| {abs_terms[at].item()})")


def assert_elementwise_bound(name, got, ref, bound):
    """Element-wise |got - ref| <= bound (bound > 0 wherever ref or got can differ)."""
    err = (got.double() - ref).abs()
    worst, at = _worst(name, err / bound.clamp_min(1e-300))
    assert worst <= 1.0, (f"{name}: |got - ref| = {err[at].item():.3e} > {bound[at].item():.3e} at {at} "
                          f"(got {got[at].item()}, ref {ref[at].item()})")


def assert_rows_close(name, got, ref, rtol, atol=1e-3):
    """Per row of the last dim: ||got - ref|| <= rtol ||ref|| + atol rms(ref), rms over the whole tensor (the absolute
    part covers rows whose value cancels to ~0)."""
    got, ref = got.double(), ref.double()
    err = (got - ref).norm(dim=-1)
    bound = (rtol * ref.norm(dim=-1) + atol * ref.pow(2).mean().sqrt()).clamp_min(1e-300)
    worst, at = _worst(name, err / bound)
    assert worst <= 1.0, (f"{name}: row {at}: ||got - ref|| = {err[at].item():.3e} > {bound[at].item():.3e} "
                          f"(||ref|| = {ref[at].norm().item():.3e})")
