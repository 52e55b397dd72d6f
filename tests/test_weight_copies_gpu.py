"""The column sums (`colsum_accum`) and the bf16 copies of the fp32 master weights that the GEMMs read: `cast_bf16`,
`cast_multi` (layernorm.cu, optim.cu), the copies the fused AdamW writes in its own pass, and `Bf16Cache.refresh()`.

A stale or wrong bf16 copy trains the next step on the wrong weights, and a whole-model test sees that only as a
slightly different loss.  So every copy is compared with `master.to(torch.bfloat16)` bit for bit (round to nearest
even, the same as torch), NaN compared by NaN-ness only, with sentinels around every destination.

Bounds (u = 2^-24, S = 1.25 slack):
  colsum   |got - ref| <= S u n (|init| + sum_m |dy_mn|)     the terms are exact (fp32 or bf16 inputs); n = the additions
                                                             a column's sum passes through: rows per thread (step 8) +
                                                             the block's 8 row lanes + one atomic per row block;
  AdamW    the HF update in float64 from the fp32 state the kernel read and its fp32 hyper-parameters, with
           M = b1 |m| + (1 - b1) |g|, V = b2 v + (1 - b2) g^2:
           m  S 3u M;   v  S 4u V;
           p  S (u ss (3 M + 6 |m'|) / (sqrt(v') + eps) + u |p1| + 2u lr wd |p1| + u |p'|)
              (ss = the bias-corrected step size, p1 = p before the weight decay, primes = new values): the update's
              operands and its four roundings, then the decay's product and subtraction.
Each check prints its worst element as a fraction of its bound (run with -s)."""
import math

import pytest
import torch
from kernel_checks import BF16, F32, F64, assert_bits_equal, assert_elementwise_bound, assert_sum_bound

U = 2.0 ** -24
SLACK = 1.25
SENTINEL = -3.0

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


def randn(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda") * scale


def f32(v):
    return float(torch.tensor(v, dtype=F32))


# ---------------------------------------------------------------------------------------------------------- colsum_accum
def colsum_depth(M, N, vec, sms):
    """As egovlp_colsum_accum sizes its grid."""
    col_blocks = (N // vec + 31) // 32
    row_blocks = max(1, min((M + 63) // 64, (sms * 8 + col_blocks - 1) // col_blocks))
    rpb = (M + row_blocks - 1) // row_blocks
    row_blocks = (M + rpb - 1) // rpb
    return -(-rpb // 8) + 8 + row_blocks


@pytest.mark.parametrize("M", [1, 7, 64, 65, 100003])
@pytest.mark.parametrize("N", ["vec", 40, 776, 3072])
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
def test_colsum_accum_matches_fp64(ops, dtype, N, M):
    """Onto a non-zero `out` with sentinels after N; rows contiguous (ld = N) and a column slice of a wider buffer."""
    vec = 4 if dtype == F32 else 8
    N = vec if N == "vec" else N
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = colsum_depth(M, N, vec, sms)
    for ld in (N, N + 3 * vec):
        dy = randn((M, ld), M + N)
        dy = (dy if dtype == F32 else dy.to(dtype))[:, :N]
        buf = torch.cat([randn((N,), 3), torch.full((8,), SENTINEL, device="cuda")])
        init = buf[:N].clone()
        ops.colsum_accum(dy, buf[:N])
        torch.cuda.synchronize()
        assert bool((buf[N:] == SENTINEL).all()), "colsum: wrote past N"
        ref, mag = init.double(), init.double().abs()
        for r0 in range(0, M, 8192):                     # fp64 in row chunks: no full-size fp64 temporaries
            d = dy[r0:r0 + 8192].to(F64)
            ref, mag = ref + d.sum(0), mag + d.abs().sum(0)
        assert_sum_bound(f"colsum {str(dtype)[6:]} M={M} N={N} ld={ld}", buf[:N], ref, mag, rel=SLACK * U * n)
        del dy


@pytest.mark.parametrize("dtype,N,ld", [(F32, 6, 8), (F32, 8, 10), (BF16, 12, 16), (BF16, 16, 20)])
def test_colsum_refuses_widths_off_the_vector(ops, dtype, N, ld):
    from egovlp_b200._lib import EgovlpError
    dy = torch.ones(10, ld, device="cuda", dtype=dtype)[:, :N]
    out = torch.zeros(N, device="cuda")
    with pytest.raises(EgovlpError, match="multiples"):
        ops.colsum_accum(dy, out)
    torch.cuda.synchronize()
    assert bool((out == 0).all())


# ---------------------------------------------------------------------------------------------------------- casts
def special_values():
    """fp32 bit patterns where a cast goes wrong: signed zeros, infinities, NaNs, subnormals, exact round-to-nearest-even
    ties with an even and an odd kept part (both signs, normal and subnormal), their neighbours, and values at and
    past the largest bf16."""
    bits = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FA00001, 0xFFC12345,
            0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00008000, 0x00018000, 0x80008000, 0x80018000, 0x00010000,
            0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000, 0x3F807FFF, 0x3F808001, 0x3F817FFF, 0x3F818001,
            0x00800000, 0x00808000, 0x00818000, 0x7F7F0000, 0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0x7F7E8000,
            0xFF7F8000, 0xFF7FFFFF, 0x477FE000, 0x3DCCCCCD, 0x3EAAAAAB]
    t = torch.tensor([b - (1 << 32) if b >= 1 << 31 else b for b in bits], dtype=torch.int32)
    return t.view(F32).cuda()


def cast_input(n, seed):
    """n fp32 values: the special ones first, then random values over a wide range of exponents."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, generator=g, device="cuda") * torch.exp2(torch.randint(-140, 120, (n,), generator=g,
                                                                           device="cuda").float())
    sp = special_values()
    x[:min(n, sp.numel())] = sp[:n]
    return x


def assert_cast_exact(name, got, src):
    want = src.to(BF16)
    nan = src.isnan()
    assert torch.equal(got.isnan(), nan), f"{name}: NaN-ness differs"
    assert_bits_equal(name, torch.where(nan, torch.zeros_like(got), got), torch.where(nan, torch.zeros_like(want), want))


@pytest.mark.parametrize("n", [1, 3, 39, 4095, 4096, 4097, 1 << 20])
def test_cast_bf16_rounds_as_torch(ops, n):
    """Aligned views (vector path + tail), and views 4 / 12 bytes off 16 (source) or 2 bytes off 8 (destination), the
    scalar path that Bf16Cache.cat slices take."""
    for src_off, dst_off in ((0, 0), (1, 0), (0, 1), (3, 1)):
        srcbuf = torch.empty(n + 4, device="cuda")
        src = srcbuf[src_off:src_off + n]
        src.copy_(cast_input(n, n + src_off))
        buf = torch.full((n + 12,), SENTINEL, dtype=BF16, device="cuda")
        lead = 4 + dst_off
        ops.cast_bf16(src, buf[lead:lead + n])
        torch.cuda.synchronize()
        assert bool((buf[:lead] == SENTINEL).all()) and bool((buf[lead + n:] == SENTINEL).all()), \
            "cast_bf16: wrote outside its destination"
        assert_cast_exact(f"cast_bf16 n={n} src+{4 * src_off}B dst+{2 * dst_off}B", buf[lead:lead + n], src)


CAST_NUMELS = [1, 3, 4095, 4096, 4097, 3 * 4096 + 5]


def test_cast_multi_rounds_as_torch_on_every_path(ops):
    """One table: every numel aligned (vector path + tails), and each again from a source 4 bytes off 16 and into a
    destination 4 bytes off 8 (scalar path).  Every destination sits between sentinels."""
    pairs, checks = [], []
    for i, n in enumerate(CAST_NUMELS):
        for src_off, dst_off in ((0, 0), (1, 0), (0, 2), (3, 2)):              # elements: fp32 4 / 12 B, bf16 4 B
            srcbuf = torch.empty(n + 4, device="cuda")
            src = srcbuf[src_off:src_off + n]
            src.copy_(cast_input(n, 10 * i + src_off + dst_off))
            lead = 4 + dst_off
            dstbuf = torch.full((lead + n + 5,), SENTINEL, dtype=BF16, device="cuda")
            dst = dstbuf[lead:lead + n]
            assert src.data_ptr() % 16 == 4 * src_off and dst.data_ptr() % 8 == 2 * dst_off
            pairs.append((src, dst))
            checks.append((n, src_off, dst_off, src, dstbuf, lead))
    ops.cast_multi(*ops.build_cast_table(pairs))
    torch.cuda.synchronize()
    for n, so, do, src, dstbuf, lead in checks:
        assert bool((dstbuf[:lead] == SENTINEL).all()) and bool((dstbuf[lead + n:] == SENTINEL).all()), \
            f"cast_multi n={n}: wrote outside its destination"
        assert_cast_exact(f"cast_multi n={n} src+{4 * so}B dst+{2 * do}B", dstbuf[lead:lead + n], src)


# ---------------------------------------------------------------------------------------------------------- AdamW copies
SHAPES = {"n16": (16,), "n5": (5,), "n6": (2, 3), "n7": (7,), "n4101": (3, 1367)}


def adamw_reference(p, g, m, v, lr, b1, b2, eps, wd, ss):
    """One HF AdamW step in float64 from fp32 state and the fp32 hyper-parameters; returns (p, m, v) and their bounds."""
    p, g, m, v = (t.to(F64) for t in (p, g, m, v))
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    den = v1.sqrt() + eps
    p1 = p - ss * m1 / den
    p2 = p1 - lr * wd * p1
    M = b1 * m.abs() + (1 - b1) * g.abs()
    V = b2 * v + (1 - b2) * g * g
    e_p = SLACK * (U * ss * (3 * M + 6 * m1.abs()) / den + U * p1.abs() + 2 * U * lr * wd * p1.abs() + U * p2.abs())
    return (p2, e_p), (m1, SLACK * 3 * U * M), (v1, SLACK * 4 * U * V)


def test_fused_adamw_keeps_every_bf16_copy_exact(ops):
    """Parameters with Bf16Cache copies: numel % 4 in {0, 1, 2, 3}, 4101 elements (two chunks, a tail), and a
    Bf16Cache.cat group of three [3, 5] weights whose slices of one bf16 buffer start 30 and 60 bytes in (the kernel's
    scalar path); one parameter has no copy.  After each of three steps every copy equals p.to(bf16) bit for bit, and
    p, m, v are within the fp64 bound of the HF update.  A write through p.data after the last step, then refresh():
    the copies follow the new masters."""
    from egovlp_b200 import engine
    from egovlp_b200.optim import AdamW
    params = {k: torch.nn.Parameter(randn(s, i)) for i, (k, s) in enumerate(SHAPES.items())}
    cat = [torch.nn.Parameter(randn((3, 5), 20 + i)) for i in range(3)]
    plain = torch.nn.Parameter(randn((33,), 30))
    cache = engine.Bf16Cache()
    for p in params.values():
        cache.get(p)
    buf = cache.cat("qkv", cat)
    named = dict(params, **{f"cat{i}": p for i, p in enumerate(cat)})
    assert [engine.shadow_entry(p).t16.data_ptr() - buf.data_ptr() for p in cat] == [0, 30, 60]
    every = list(named.values()) + [plain]
    lr, b1, b2, eps, wd = 1e-2, 0.9, 0.999, 1e-6, 0.05
    opt = AdamW(every, lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    for step in range(1, 4):
        for i, p in enumerate(every):
            p.grad = randn(p.shape, 100 * step + i, 0.1 if i % 2 else 3.0)
        before = [(p.detach().clone(), torch.zeros_like(p) if step == 1 else opt.state[p]["exp_avg"].clone(),
                   torch.zeros_like(p) if step == 1 else opt.state[p]["exp_avg_sq"].clone()) for p in every]
        opt.step()
        torch.cuda.synchronize()
        ss = f32(lr * math.sqrt(1 - b2 ** step) / (1 - b1 ** step))
        for (name, p), (p0, m0, v0) in zip(list(named.items()) + [("plain", plain)], before):
            (pr, ep), (mr, em), (vr, ev) = adamw_reference(p0, p.grad, m0, v0, f32(lr), f32(b1), f32(b2), f32(eps),
                                                           f32(wd), ss)
            st = opt.state[p]
            assert_elementwise_bound(f"adamw p {name} step {step}", p.detach(), pr, ep)
            assert_elementwise_bound(f"adamw m {name} step {step}", st["exp_avg"], mr, em)
            assert_elementwise_bound(f"adamw v {name} step {step}", st["exp_avg_sq"], vr, ev)
        for name, p in named.items():
            assert_bits_equal(f"bf16 copy {name} after step {step}", engine.shadow_entry(p).t16, p.detach().to(BF16))
    for i, p in enumerate(named.values()):
        p.data.add_(randn(p.shape, 500 + i, 0.5))
    cache.refresh()
    torch.cuda.synchronize()
    for name, p in named.items():
        assert_bits_equal(f"bf16 copy {name} after p.data.add_ + refresh", engine.shadow_entry(p).t16,
                          p.detach().to(BF16))
    assert_bits_equal("Bf16Cache.cat buffer", buf, torch.cat([p.detach() for p in cat]).to(BF16))
