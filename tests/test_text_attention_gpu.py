"""The short-caption text attention (text_attn_fwd / text_attn_bwd, text_attn_kernel in csrc/text.cu; L <= 128, the
length every step of the flagship workload runs) against float64, element by element, at the bound derived in
tests/text_attention_ref.py:
  * L = 1 .. 128 around each 32-key boundary (a lane's 1st .. 4th key) x H = 1 and 12, q_scale 0.125 and 0.1, full,
    one-key, prefix, holed and 5-key masks, score maxima of spread 18 planted on the last valid key, and a batch of
    more than two waves of CTAs; outputs in NaN-filled buffers followed by sentinel rows;
  * attention dropout p = 0.1 and 0.5, with the multiplier from the host Philox of tests/philox_ref.py, and the keep
    bits read back through the forward bit for bit against it for every L <= 128;
  * bitwise reproducibility, batch-position independence, a sample without a valid key, and argument refusals.
Run with -s for the worst fraction of the bound of every output ([bound] lines)."""
import pytest
import torch
from kernel_checks import BF16, assert_bits_equal, nan_filled
from philox_ref import multiplier, short_attn_keep
from text_attention_ref import SENTINEL, SENTINEL_ROWS, case, check_short, make_inputs, short_reference

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


def _sentinel_buf(rows, cols):
    buf = nan_filled((rows + SENTINEL_ROWS, cols), BF16)
    buf[rows:] = SENTINEL
    return buf


def run(ops, qkv, dout, mask, B, L, H, q_scale, p=0.0, seed=0, site=0):
    """Forward and backward into NaN-filled buffers with sentinel rows; checks that every element was written and no
    sentinel changed; -> (out [B*L, D], dqkv [B*L, 3D])."""
    D, M = 64 * H, B * L
    out_buf, dq_buf = _sentinel_buf(M, D), _sentinel_buf(M, 3 * D)
    ops.text_attn_fwd(qkv, mask, out_buf, B, L, H, p, seed, site)
    ops.text_attn_bwd(qkv, mask, dout, dq_buf, B, L, H, q_scale, p, seed, site)
    torch.cuda.synchronize()
    for name, buf in (("out", out_buf), ("dqkv", dq_buf)):
        assert not buf[:M].isnan().any(), f"{name}: {int(buf[:M].isnan().sum())} elements left unwritten"
        assert bool((buf[M:] == SENTINEL).all()), f"{name}: a row past the output was written"
    return out_buf[:M], dq_buf[:M]


def check(tag, qkv, dout, mask, out, dqkv, B, L, H, q_scale, p=0.0, seed=0, site=0):
    """Every element within the bound; the dropout multiplier is the host's for samples 0 .. B - 1."""
    mult = multiplier(short_attn_keep(p, seed, site, B, H, L), p) if p > 0 else None
    return check_short(tag, out, dqkv, mask, short_reference(qkv, dout, mask, B, L, H, q_scale, mult))


LS = [1, 2, 31, 32, 33, 63, 64, 65, 96, 97, 127, 128]


@pytest.mark.parametrize("q_scale", [0.125, 0.1])
@pytest.mark.parametrize("H", [1, 12])
@pytest.mark.parametrize("L", LS)
def test_text_attention_vs_fp64(ops, L, H, q_scale):
    qkv, dout, mask, B = case(L, H, q_scale, seed=L * 31 + H)
    out, dqkv = run(ops, qkv, dout, mask, B, L, H, q_scale)
    check(f"L={L} H={H} q_scale={q_scale}", qkv, dout, mask, out, dqkv, B, L, H, q_scale)


@pytest.mark.parametrize("L", [16, 128])
def test_text_attention_more_than_two_waves_of_ctas(ops, L):
    """B = 32, H = 12: 384 CTAs, more than two per SM of a 132-SM H100; valid-key counts all, 1, on a 32-key boundary
    and random (the step's captions are 16 tokens)."""
    B, H, q_scale = 32, 12, 0.125
    lens = torch.randint(1, L + 1, (B,), generator=torch.Generator().manual_seed(L))
    lens[0], lens[1], lens[2] = L, 1, (L - 1) // 32 * 32 or L
    mask = (torch.arange(L)[None] < lens[:, None]).long().cuda()
    qkv, dout = make_inputs(B, L, H, seed=100 + L, q_scale=q_scale)
    out, dqkv = run(ops, qkv, dout, mask, B, L, H, q_scale)
    check(f"B={B} L={L} H={H}", qkv, dout, mask, out, dqkv, B, L, H, q_scale)


def test_text_attention_dropout_vs_fp64_with_the_host_mask(ops):
    """p = 0.1 and 0.5 at L = 33, 64, 65 and 128: keys 64 .. 127 are a lane's 3rd and 4th key (keep words 2 and 3,
    dp_local[2..3] in the backward).  Run to run bit-identical; a sample run alone is sample 0 of its own launch, so it
    is checked against the host mask of b = 0."""
    for p in (0.1, 0.5):
        for L in (33, 64, 65, 128):
            _dropout_case(ops, L, p)


def _dropout_case(ops, L, p):
    H, q_scale, seed, site = 2, 0.125, 0x8000_0000_DEAD_BEEF, 5
    qkv, dout, mask, B = case(L, H, q_scale, seed=L + 7)
    out, dqkv = run(ops, qkv, dout, mask, B, L, H, q_scale, p, seed, site)
    check(f"dropout p={p} L={L}", qkv, dout, mask, out, dqkv, B, L, H, q_scale, p, seed, site)
    again = run(ops, qkv, dout, mask, B, L, H, q_scale, p, seed, site)
    assert_bits_equal(f"out dropout run to run L={L}", out, again[0])
    assert_bits_equal(f"dqkv dropout run to run L={L}", dqkv, again[1])
    s = B - 1
    one = lambda t: t.view(B, L, -1)[s].contiguous()
    o1, d1 = run(ops, one(qkv), one(dout), mask[s:s + 1].contiguous(), 1, L, H, q_scale, p, seed, site)
    check(f"dropout p={p} L={L} sample {s} alone", one(qkv), one(dout), mask[s:s + 1], o1, d1, 1, L, H, q_scale, p,
          seed, site)


@pytest.mark.parametrize("L", [16, 65, 128])
def test_text_attention_bitwise_reproducible_and_batch_position_independent(ops, L):
    B, H, q_scale = 8, 12, 0.125
    lens = torch.tensor([L, 3, L - 1, min(L, 32), min(L, 33), 1, 7, L // 2]).clamp(1, L)
    mask = (torch.arange(L)[None] < lens[:, None]).long().cuda()
    qkv, dout = make_inputs(B, L, H, seed=L)
    a, b = run(ops, qkv, dout, mask, B, L, H, q_scale), run(ops, qkv, dout, mask, B, L, H, q_scale)
    for name, x, y in zip(("out", "dqkv"), a, b):
        assert_bits_equal(f"{name} run to run L={L}", x, y)
    for s in (0, 5, 7):
        one = run(ops, qkv.view(B, L, -1)[s].contiguous(), dout.view(B, L, -1)[s].contiguous(),
                  mask[s:s + 1].contiguous(), 1, L, H, q_scale)
        for name, x, y in zip(("out", "dqkv"), one, a):
            assert_bits_equal(f"{name} sample {s} alone L={L}", x, y.view(B, L, -1)[s])
    # p = 0 with any (seed, site) is the dropout-free call
    c = run(ops, qkv, dout, mask, B, L, H, q_scale, 0.0, 123456789, 9)
    for name, x, y in zip(("out", "dqkv"), a, c):
        assert_bits_equal(f"{name} p=0 L={L}", x, y)


def test_text_attention_sample_without_a_valid_key_is_nan_only_there(ops):
    """A mask with no valid key (a tokenizer always emits [CLS] and [SEP], so never in training): that sample's rows
    are NaN (0 / 0 in its softmax, as in a masked_fill(-inf) softmax), and every other sample is bit-identical to the
    batch without it."""
    B, L, H, q_scale = 3, 40, 2, 0.125
    D = 64 * H
    mask = torch.ones(B, L, dtype=torch.int64, device="cuda")
    mask[2, 30:] = 0
    mask[1] = 0
    qkv, dout = make_inputs(B, L, H, seed=9)
    out, dqkv = nan_filled((B * L, D), BF16), nan_filled((B * L, 3 * D), BF16)
    ops.text_attn_fwd(qkv, mask, out, B, L, H)
    ops.text_attn_bwd(qkv, mask, dout, dqkv, B, L, H, q_scale)
    torch.cuda.synchronize()
    rows = slice(L, 2 * L)
    assert bool(out[rows].isnan().all()) and bool(dqkv[rows].isnan().all())
    keep = torch.tensor([0, 2], device="cuda")
    sub = lambda t: t.view(B, L, -1)[keep].reshape(2 * L, -1)
    o2, d2 = run(ops, sub(qkv), sub(dout), mask[keep], 2, L, H, q_scale)
    assert_bits_equal("out beside an empty sample", sub(out), o2)
    assert_bits_equal("dqkv beside an empty sample", sub(dqkv), d2)


@pytest.mark.parametrize("L,p", [(0, 0.0), (129, 0.0), (64, -0.1), (64, 1.0)])
def test_text_attention_refuses_bad_arguments_and_writes_nothing(ops, L, p):
    from egovlp_b200._lib import EgovlpError
    B, H = 2, 2
    Ln = max(L, 1)
    qkv = torch.zeros(B * Ln, 3 * 64 * H, device="cuda", dtype=BF16)
    mask = torch.ones(B, Ln, dtype=torch.int64, device="cuda")
    out, dq = nan_filled((B * Ln, 64 * H), BF16), nan_filled((B * Ln, 3 * 64 * H), BF16)
    dout = torch.zeros(B * Ln, 64 * H, device="cuda", dtype=BF16)
    with pytest.raises(EgovlpError):
        ops.text_attn_fwd(qkv, mask, out, B, L, H, p)
    with pytest.raises(EgovlpError):
        ops.text_attn_bwd(qkv, mask, dout, dq, B, L, H, 0.125, p)
    torch.cuda.synchronize()
    assert bool(out.isnan().all()) and bool(dq.isnan().all())


# ------------------------------------------------------------------------------------------------ keep bits
def extract_keep(ops, B, L, H, p, seed, site):
    """The kernel's keep mask [B, H, L, L] read back through the forward: q = k = 0 makes the softmax uniform over the
    valid keys; a window of n <= 64 valid keys with v = one-hot of the key's offset makes output column d of row i
    equal keep(i, j0 + d) / (1 - p) / n.  Two windows cover L <= 128."""
    D = 64 * H
    qkv = torch.zeros(B * L, 3 * D, device="cuda", dtype=BF16)
    keep = torch.zeros(B, H, L, L, dtype=torch.bool)
    j = torch.arange(L, device="cuda")
    for j0 in range(0, L, 64):
        n = min(64, L - j0)
        v = qkv.view(B, L, 3, H, 64)[:, :, 2]
        v.zero_()
        v[:, j0:j0 + n] = torch.eye(64, device="cuda", dtype=BF16)[:n, None, :]
        mask = ((j >= j0) & (j < j0 + n)).long()[None].expand(B, L).contiguous()
        out = nan_filled((B * L, D), BF16)
        ops.text_attn_fwd(qkv, mask, out, B, L, H, p, seed, site)
        o = out.float().view(B, L, H, 64)[..., :n].permute(0, 2, 1, 3) * n     # kept -> 1 / (1 - p), dropped -> 0
        keep[..., j0:j0 + n] = (o > 0.5).cpu()
    return keep


def test_attention_keep_bits_are_the_documented_philox_stream_for_every_length(ops):
    """Every L = 1 .. 128 (B = 2, H = 3): the kernel's keep bits equal the host's bit for bit.  Then B = 8, H = 12,
    L = 128 (1.6M draws on distinct counters; the lengths above reuse counters): bit for bit again, the keep rate
    within 3 sigma of 1 - p, and the streams of the next site and the next seed agree with it as independent streams
    would."""
    p, seed, site = 0.1, 0x9234_5678_9ABC_DEF1, 3
    for L in range(1, 129):
        want = short_attn_keep(p, seed, site, 2, 3, L)
        got = extract_keep(ops, 2, L, 3, p, seed, site)
        assert torch.equal(got, want), f"L={L}: {int((got != want).sum())} of {want.numel()} keep bits differ"
    B, H, L = 8, 12, 128
    host = short_attn_keep(p, seed, site, B, H, L)
    got = extract_keep(ops, B, L, H, p, seed, site)
    assert torch.equal(got, host), f"{int((got != host).sum())} of {host.numel()} keep bits differ"
    n = host.numel()
    assert n > 1_000_000
    rate = host.double().mean().item()
    assert abs(rate - (1 - p)) < 3 * (p * (1 - p) / n) ** 0.5, rate
    want = (1 - p) ** 2 + p ** 2                                               # independent streams agree this often
    for other in (short_attn_keep(p, seed, site + 1, B, H, L), short_attn_keep(p, seed + 1, site, B, H, L)):
        agree = (other == host).double().mean().item()
        assert abs(agree - want) < 3 * (want * (1 - want) / n) ** 0.5 + 1e-4, agree
    blocks = host.view(-1, 4096).double().mean(1)                              # no structure along the index
    assert (blocks - (1 - p)).abs().max().item() < 0.03
