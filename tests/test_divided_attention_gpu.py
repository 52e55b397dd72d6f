"""The video tower's divided space-time attention (attention.cu, attention_wgmma.cu) against float64, element by
element, on every kernel path.

The reference (`reference`) is computed per attention group from the same bf16 values the kernels read: space, one
group per (b, h, frame) over its N patches; time, one per (b, h, patch) over its T frames; each group's keys are its
own rows plus the CLS key.  The CLS query is its own group over all S keys, with the CLS key counted once.  It gives
out, lse (natural log, q as stored: already scaled), the analytic backward, and the magnitude sums the bounds are
made of.  It never forms a dense S x S matrix, which at S = 3137, H = 12 would cost gigabytes per (b, h).  The host
tests pin it to oracle.reference_port.divided_attention_core and its autograd gradients.

The bounds follow from the kernels' arithmetic: scores accumulated in fp32 from exact bf16 products, P rounded to bf16
before each mma, dS rounded to bf16, every output rounded once to bf16.  With u = 2^-8 (bf16 unit roundoff):
  out   |got - ref| <= u (sum_j P_ij |v_jd| + 2 |ref|)     P rounded in the numerator (and in the normaliser, if a path
                                                          sums it from the rounded P), one final rounding;
  lse   |got - ref| <= 2e-5 max_j sum_d |q_id k_jd| + 1e-6 (1 + |ref|)
                                                          fp32 scores, exp2 / log approximations; a dropped key moves
                                                          lse by about P_j, far above this;
  dv    |got - ref| <= u (sum_i P_ij |dO_id| + |ref|);
  dq    |got - ref| <= u (q_scale sum_j P_ij (|dP_ij - delta_i| + E_i) |k_jd| + |ref|),
  dk    the same summed over queries i, with |q_id| in place of |k_jd|;
        E_i = sum_d |dO_id| (sum_j P_ij |v_jd| + 2 |O_id|): the kernels take delta from the bf16 `out`, whose error
        is bounded above, so u E_i bounds the error of delta.
The CLS rows' terms are summed over every group.  Every bound carries a fixed slack of SLACK for fp32 accumulation.
Each check prints its worst element as a fraction of its bound (run with -s).

Outputs are prefixes of NaN-filled buffers followed by sentinel rows: every element must be written, no sentinel
touched.  Forward outputs and the backward's patch rows are written without atomics, so they must be bit-identical
from run to run and independent of the other clips in the batch; only the CLS rows of the backward (fp32 atomics
across groups) are held to the bounds alone."""
import ctypes as C

import pytest
import torch
from divided_attention_ref import (Q_SCALE, check_against_reference, check_case, make_inputs, paths_for, plant_maxima,
                                   reference, run_attention, set_path)
from kernel_checks import BF16, F32, assert_bits_equal, nan_filled


# ---------------------------------------------------------------------------------------------------------- host tests
def dense_reference(qkv, dout, B, T, N, H, mode):
    """Dense masked S x S softmax (small shapes only): lse and the P-weighted magnitude sums."""
    S = 1 + T * N
    x = qkv.view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    q, k, v = x[0], x[1], x[2]
    do = dout.view(B, S, H, 64).permute(0, 2, 1, 3)
    tok = torch.arange(S)
    gid = torch.where(tok == 0, -1, ((tok - 1) // N) if mode == 1 else ((tok - 1) % N))
    allowed = (gid[:, None] == gid[None, :]) | (tok[None, :] == 0) | (tok[:, None] == 0)
    s = (q @ k.transpose(-1, -2)).masked_fill(~allowed, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    return lse, (p @ v.abs()), (p.transpose(-1, -2) @ do.abs())


@pytest.mark.parametrize("B,T,N,H,mode", [(2, 3, 5, 1, 1), (2, 4, 9, 2, 1), (2, 3, 5, 2, 0), (2, 16, 8, 1, 0),
                                          (2, 5, 7, 2, 0), (2, 1, 6, 1, 0), (3, 2, 1, 2, 1)])
def test_reference_matches_the_oracle_and_its_autograd(B, T, N, H, mode):
    """The per-group fp64 reference against oracle.reference_port.divided_attention_core (pinned to the unmodified
    reference by test_oracle_vs_live_reference.py) and its autograd gradients, on the CPU, in fp64.  (2, 16, 8): the
    kernels' time groups of 7 patches leave a second, partly filled group; the reference has no such groups."""
    from oracle import reference_port as rp
    S, D = 1 + T * N, 64 * H
    qkv, dout = make_inputs(B, T, N, H, seed=B * 100 + T * 10 + N + H + mode, device="cpu")
    qkv, dout = qkv.double(), dout.double()
    res = reference(qkv, dout, B, T, N, H, mode, Q_SCALE)
    xr = qkv.view(B, S, 3 * D).clone().requires_grad_(True)
    ref = rp.divided_attention_core(xr, H, T, N, "space" if mode else "time", scale_q=False)
    ref.backward(dout.view(B, S, D))
    g = xr.grad.reshape(B * S, 3 * D)
    torch.testing.assert_close(res["out"], ref.detach().reshape(B * S, D), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(res["dq"], Q_SCALE * g[:, :D], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(res["dk"], g[:, D:2 * D], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(res["dv"], g[:, 2 * D:], rtol=1e-12, atol=1e-12)
    lse, pv, pdo = dense_reference(qkv, dout, B, T, N, H, mode)
    torch.testing.assert_close(res["lse"], lse, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(res["out_t"], pv.permute(0, 2, 1, 3).reshape(B * S, D), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(res["dv_t"], pdo.permute(0, 2, 1, 3).reshape(B * S, D), rtol=1e-12, atol=1e-12)


def test_planted_maxima_dominate():
    """plant_maxima gives each aimed row one key whose score leads the rest by far more than the unit spread."""
    B, T, N, H, mode = 2, 16, 8, 1, 0
    qkv, dout = make_inputs(B, T, N, H, seed=5, device="cpu")
    qkv = plant_maxima(qkv, B, T, N, H, mode)
    lse, _, _ = dense_reference(qkv.double(), dout.double(), B, T, N, H, mode)
    S = 1 + T * N
    x = qkv.double().view(B, S, 3, H, 64)
    assert (x[:, 0, 0] * x[:, S - 1, 1]).sum(-1).min() > 15          # the CLS query at the last patch
    assert (x[:, 1, 0] * x[:, 0, 1]).sum(-1).min() > 15              # frame 0 of patch 0 at the CLS key
    assert (lse[:, :, 0] - 15).min() > 0


# ---------------------------------------------------------------------------------------------------------- GPU harness
@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


def cases(shapes, heads=(1, 12)):
    """(B, T, N, H, mode, path) for every head count and every path the geometry admits."""
    return [pytest.param(B, T, N, H, mode, path, id=f"{'space' if mode else 'time'}-B{B}-T{T}-N{N}-H{H}-{path}")
            for B, T, N, mode in shapes for H in heads for path in paths_for(T, N, mode)]


# space: N = 1; 15 and 16 (NP % 16 == 0: the CLS row alone in its tile); 100 and 127 (the 4-warp kernels loop over
# more row tiles than warps; 127 is their largest NPAD, 128); 128 (the smallest 7-warp and wgmma geometry), 196, 207
# (the largest wgmma); 208; 240 (NP % 16 == 0 on 7 warps); 255 (NPAD = 256, the largest).
SPACE = [(2, 2 + i % 2, n, 1) for i, n in enumerate([1, 15, 16, 100, 127, 128, 196, 207, 208, 240, 255])]
# time, fast path: one full group of 112 / T patches; one more patch, so the second group holds a single patch and three
# of its four CLS parts see no valid key; 196
TIME_FAST = [(2, t, n, 0) for t in (4, 8, 16) for n in (112 // t, 112 // t + 1, 196)]
# time, generic path: T = 1 (two groups of 112 and 1), T = 2 (56 + 1), T = 3 (42 + 8), T = 5 (25 + 5), T = 16 with
# N = 5 (a fast-path T with NP = 80), T = 32 (PG = 3: 3 + 3 + 3 + 1), T = 127 (PG = 1)
TIME_GENERIC = [(2, 1, 113, 0), (2, 2, 57, 0), (3, 3, 50, 0), (2, 5, 30, 0), (2, 16, 5, 0), (2, 32, 10, 0),
                (2, 127, 3, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,N,H,mode,path", cases(SPACE) + cases(TIME_FAST) + cases(TIME_GENERIC))
def test_divided_attention_matches_fp64(ops, monkeypatch, B, T, N, H, mode, path):
    check_case(ops, monkeypatch, B, T, N, H, mode, path, seed=1000 * T + N + 7 * H + mode)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,N,H,mode,path", cases([(2, 16, 196, 1), (2, 16, 196, 0)], heads=(12,)))
def test_training_step_geometry(ops, monkeypatch, B, T, N, H, mode, path):
    """The training step's own shape: 16 frames of 14 x 14 patches, 12 heads."""
    check_case(ops, monkeypatch, B, T, N, H, mode, path, seed=77 + mode)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,N,H,mode,path", cases([(2, 4, 29, 0), (2, 3, 100, 1)], heads=(2,)))
def test_q_scale_not_a_power_of_two(ops, monkeypatch, B, T, N, H, mode, path):
    """q_scale = 0.1: a scale applied to the wrong tensor or rows, or twice, cannot hide in exact power-of-two steps."""
    check_case(ops, monkeypatch, B, T, N, H, mode, path, seed=31 + mode, q_scale=0.1)


# sharp scores: the running-max rescale of the online softmax, and cls_merge_kernel's weights across groups whose
# maxima differ by ~18; (2, 16, 8) / (2, 5, 30) / (2, 1, 113) put the CLS query's maximum in a partly filled last group
@pytest.mark.gpu
@pytest.mark.parametrize("B,T,N,H,mode,path", cases([(2, 3, 100, 1), (2, 2, 196, 1), (2, 3, 255, 1), (2, 16, 8, 0),
                                                      (2, 4, 196, 0), (2, 5, 30, 0), (2, 1, 113, 0)], heads=(1, 12)))
def test_sharp_scores(ops, monkeypatch, B, T, N, H, mode, path):
    check_case(ops, monkeypatch, B, T, N, H, mode, path, seed=500 + T + N, sharp=True)


# ---------------------------------------------------------------------------------------------------------- determinism
DETERMINISM = [(2, 100, 1), (2, 196, 1), (3, 255, 1), (8, 15, 0), (16, 196, 0), (5, 30, 0), (32, 10, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("T,N,mode,path", [pytest.param(T, N, mode, p, id=f"{'space' if mode else 'time'}-T{T}-N{N}-{p}")
                                           for T, N, mode in DETERMINISM for p in paths_for(T, N, mode)])
def test_bit_identical_across_runs_and_batch_positions(ops, monkeypatch, T, N, mode, path):
    """One clip alone (B = 1) and as the middle clip of three different clips (B = 3), each run twice: the forward's
    out and lse (the CLS row included: its merge runs in a fixed order) and the backward's patch rows must match bit
    for bit.  The backward's CLS rows are sums of fp32 atomics across groups and are held to the bounds."""
    set_path(monkeypatch, path)
    H = 2
    S, D = 1 + T * N, 64 * H
    qkv3, dout3 = make_inputs(3, T, N, H, seed=900 + T + N)
    qkv1, dout1 = qkv3[S:2 * S].contiguous(), dout3[S:2 * S].contiguous()
    runs1 = [run_attention(ops, qkv1, dout1, 1, T, N, H, mode, Q_SCALE) for _ in range(2)]
    runs3 = [run_attention(ops, qkv3, dout3, 3, T, N, H, mode, Q_SCALE) for _ in range(2)]
    tag = f"{'space' if mode else 'time'} T={T} N={N} {path}"
    ref_out, ref_lse, ref_d = runs1[0]
    for what, (out, lse, dqkv) in (("B=1 rerun", runs1[1]), ("B=3", runs3[0]), ("B=3 rerun", runs3[1])):
        if what.startswith("B=3"):
            out, lse, dqkv = out[S:2 * S], lse[1:2], dqkv[S:2 * S]
        assert_bits_equal(f"out {tag} {what}", out, ref_out)
        assert_bits_equal(f"lse {tag} {what}", lse, ref_lse)
        assert_bits_equal(f"dqkv patch rows {tag} {what}", dqkv[1:], ref_d[1:])
    # the first run of each batch size, CLS rows included, against fp64
    check_against_reference(f"{tag} B=1", qkv1, dout1, *runs1[0], 1, T, N, H, mode, Q_SCALE)
    check_against_reference(f"{tag} B=3", qkv3, dout3, *runs3[0], 3, T, N, H, mode, Q_SCALE)


# ---------------------------------------------------------------------------------------------------------- refusals
@pytest.mark.gpu
@pytest.mark.parametrize("T,N,mode", [(2, 256, 1), (128, 1, 0)])
def test_unsupported_geometry_is_refused_and_writes_nothing(ops, T, N, mode):
    """Space N = 256 (NPAD = 272 > 256) and time T = 128 (127 // 128 = 0 patches per group): both C entry points return
    an error before any launch; ops.divided_attn_fwd refuses them by its own assert."""
    from egovlp_b200._lib import EgovlpError
    B, H = 2, 1
    S, D = 1 + T * N, 64 * H
    qkv = torch.zeros(B * S, 3 * D, dtype=BF16, device="cuda")
    dout = torch.zeros(B * S, D, dtype=BF16, device="cuda")
    out, lse, dqkv = nan_filled((B * S, D), BF16), nan_filled((B * H * S,), F32), nan_filled((B * S, 3 * D), BF16)
    ws = torch.zeros(4 * 66, dtype=F32, device="cuda")
    with pytest.raises(EgovlpError, match="unsupported geometry"):
        ops.call("egovlp_divided_attn_fwd", ops._ptr(qkv), ops._ptr(out), ops._ptr(lse), ops._ptr(ws), B, T, N, H, mode,
                 ops._stream())
    with pytest.raises(EgovlpError, match="unsupported geometry"):
        ops.call("egovlp_divided_attn_bwd", ops._ptr(qkv), ops._ptr(out), ops._ptr(dout), ops._ptr(lse), ops._ptr(dqkv),
                 ops._ptr(ws), B, T, N, H, mode, C.c_float(Q_SCALE), ops._stream())
    torch.cuda.synchronize()
    assert out.isnan().all() and lse.isnan().all() and dqkv.isnan().all() and bool((ws == 0).all())
    with pytest.raises(AssertionError, match="unsupported attention geometry"):
        ops.divided_attn_fwd(qkv, B, T, N, H, mode)
