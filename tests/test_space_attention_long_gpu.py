"""The video tower's spatial attention for large frames (space_attention.cu: egovlp_space_attn_long_*) against float64,
element by element, and the existing time attention at the same patch counts.

Harness and bounds are those of test_divided_attention_gpu.py (divided_attention_ref: the per-group fp64 reference,
u = 2^-8 with a slack of 1.25, NaN-filled outputs with sentinel rows): out, lse, dq, dk and dv, the CLS rows
included, every element within its bound.  The new kernels reduce the CLS rows' per-frame partials in frame order, with
no atomics, so every output -- the CLS rows of the backward too -- must be bit-identical from run to run and
independent of the other clips in the batch."""
import ctypes as C

import pytest
import torch
from divided_attention_ref import (Q_SCALE, SENTINEL, _with_sentinels, check_against_reference, check_case,
                                   make_inputs, paths_for, plant_maxima)
from kernel_checks import BF16, F32, assert_bits_equal, nan_filled

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


def run_long(ops, qkv, dout, B, T, N, H, q_scale):
    """Forward and backward through the C entry points into NaN-filled buffers with sentinel rows; returns
    (out [B*S, D], lse [B, H, S], dqkv [B*S, 3*D]) after checking that every element was written and no sentinel
    changed."""
    S, D = 1 + T * N, 64 * H
    M = B * S
    out_buf, lse_buf, dq_buf = _with_sentinels(M, D, BF16), _with_sentinels(B * H, S, F32), _with_sentinels(M, 3 * D, BF16)
    ws = nan_filled((ops.lib().egovlp_space_attn_long_workspace_floats(B, T, N, H),), F32)
    ops.call("egovlp_space_attn_long_fwd", ops._ptr(qkv), ops._ptr(out_buf), ops._ptr(lse_buf), ops._ptr(ws), B, T, N,
             H, ops._stream())
    out, lse = out_buf[:M], lse_buf[:B * H].view(B, H, S)
    ops.call("egovlp_space_attn_long_bwd", ops._ptr(qkv), ops._ptr(out), ops._ptr(dout), ops._ptr(lse),
             ops._ptr(dq_buf), ops._ptr(ws), B, T, N, H, C.c_float(q_scale), ops._stream())
    torch.cuda.synchronize()
    for name, buf, rows in (("out", out_buf, M), ("lse", lse_buf, B * H), ("dqkv", dq_buf, M)):
        assert not buf[:rows].isnan().any(), f"{name}: {int(buf[:rows].isnan().sum())} elements left unwritten"
        assert bool((buf[rows:] == SENTINEL).all()), f"{name}: a row past the output was written"
    return out, lse, dq_buf[:M]


def check_long(ops, B, T, N, H, seed, q_scale=Q_SCALE, sharp=False):
    qkv, dout = make_inputs(B, T, N, H, seed, q_scale)
    if sharp:
        qkv = plant_maxima(qkv, B, T, N, H, 1)
    out, lse, dqkv = run_long(ops, qkv, dout, B, T, N, H, q_scale)
    tag = f"space-long B={B} T={T} N={N} H={H} q_scale={q_scale}" + (" sharp" if sharp else "")
    return check_against_reference(tag, qkv, dout, out, lse, dqkv, B, T, N, H, 1, q_scale)


# N: 1; 64 and 255 (N + 1 = 65 / 256: one row into a new tile, a full last tile); 196 (the 224-px step); 256 and 257
# (the smallest frames the engine sends here); 319, 320 (256 x 320 px), 400, 511, 576 (384 px), 1023, 1024 (512 px).
# T in {1, 2, 16} and H in {1, 12} rotate over them; B = 1 where the fp64 reference would not fit twice.
CASES = [(2, 2, 1, 1), (2, 1, 64, 12), (2, 16, 196, 1), (2, 2, 255, 12), (2, 2, 256, 1), (2, 16, 256, 12),
         (2, 1, 257, 12), (2, 2, 319, 1), (2, 2, 320, 12), (2, 16, 400, 1), (2, 2, 511, 12), (2, 1, 576, 12),
         (2, 16, 576, 1), (1, 2, 1023, 12), (1, 16, 1023, 1), (1, 2, 1024, 12), (1, 16, 1024, 12)]


@pytest.mark.parametrize("B,T,N,H", CASES, ids=[f"B{b}-T{t}-N{n}-H{h}" for b, t, n, h in CASES])
def test_space_attn_long_matches_fp64(ops, B, T, N, H):
    check_long(ops, B, T, N, H, seed=3000 + 17 * T + N + H)


Q_CASES = [(2, 2, 256, 2), (2, 16, 320, 1), (1, 2, 1024, 12)]


@pytest.mark.parametrize("B,T,N,H", Q_CASES, ids=[f"B{b}-T{t}-N{n}-H{h}" for b, t, n, h in Q_CASES])
def test_space_attn_long_q_scale_not_a_power_of_two(ops, B, T, N, H):
    check_long(ops, B, T, N, H, seed=3100 + N, q_scale=0.1)


# planted maxima (divided_attention_ref.plant_maxima, space): every 5th patch query on the CLS key (the extra key ahead
# of the first tile), every 3rd other one on its frame's last key (the partial last tile when N + 1 is not a multiple
# of 64), and the CLS query on the last patch of the last frame -- the merge's weights then differ by about e^18.
SHARP = [(2, 2, 256, 1), (2, 16, 257, 12), (2, 3, 319, 12), (2, 2, 400, 1), (1, 16, 1023, 12), (1, 2, 1024, 1)]


@pytest.mark.parametrize("B,T,N,H", SHARP, ids=[f"B{b}-T{t}-N{n}-H{h}" for b, t, n, h in SHARP])
def test_space_attn_long_sharp_scores(ops, B, T, N, H):
    check_long(ops, B, T, N, H, seed=3200 + T + N, sharp=True)


@pytest.mark.parametrize("T,N", [(2, 196), (16, 196)])
def test_both_kernels_at_the_224px_geometry(ops, monkeypatch, T, N):
    """At N = 196 the existing kernel (the engine's choice there) and the new one both meet the fp64 bounds on the
    same inputs."""
    B, H = 2, 12
    check_case(ops, monkeypatch, B, T, N, H, 1, "default", seed=3300 + T)
    check_long(ops, B, T, N, H, seed=3300 + T)


@pytest.mark.parametrize("T,N", [(4, 256), (16, 400), (2, 1024)])
def test_bit_identical_across_runs_and_batch_positions(ops, T, N):
    """One clip alone (B = 1) and as the middle clip of three (B = 3), each run twice: out, lse and all of dqkv, the CLS
    rows included, bit for bit."""
    H = 2
    S = 1 + T * N
    qkv3, dout3 = make_inputs(3, T, N, H, seed=3400 + T + N)
    qkv1, dout1 = qkv3[S:2 * S].contiguous(), dout3[S:2 * S].contiguous()
    runs1 = [run_long(ops, qkv1, dout1, 1, T, N, H, Q_SCALE) for _ in range(2)]
    runs3 = [run_long(ops, qkv3, dout3, 3, T, N, H, Q_SCALE) for _ in range(2)]
    ref_out, ref_lse, ref_d = runs1[0]
    for what, (out, lse, dqkv) in (("B=1 rerun", runs1[1]), ("B=3", runs3[0]), ("B=3 rerun", runs3[1])):
        if what.startswith("B=3"):
            out, lse, dqkv = out[S:2 * S], lse[1:2], dqkv[S:2 * S]
        assert_bits_equal(f"out T={T} N={N} {what}", out, ref_out)
        assert_bits_equal(f"lse T={T} N={N} {what}", lse, ref_lse)
        assert_bits_equal(f"dqkv T={T} N={N} {what}", dqkv, ref_d)
    check_against_reference(f"T={T} N={N} B=3", qkv3, dout3, *runs3[0], 3, T, N, H, 1, Q_SCALE)


@pytest.mark.parametrize("B,T,N,H", [(2, 2, 1025, 1), (2, 2, 0, 1), (2, 0, 256, 1), (65536, 1, 256, 1),
                                     (2, 2, 256, 0)])
def test_unsupported_shapes_are_refused_and_write_nothing(ops, B, T, N, H):
    from egovlp_b200._lib import EgovlpError
    Bs, Ts, Ns, Hs = 2, 2, 16, 1                          # buffers of a small valid shape: nothing may be written
    S, D = 1 + Ts * Ns, 64 * Hs
    qkv = torch.zeros(Bs * S, 3 * D, dtype=BF16, device="cuda")
    dout = torch.zeros(Bs * S, D, dtype=BF16, device="cuda")
    out, lse, dqkv = nan_filled((Bs * S, D), BF16), nan_filled((Bs * Hs * S,), F32), nan_filled((Bs * S, 3 * D), BF16)
    ws = nan_filled((4096,), F32)
    with pytest.raises(EgovlpError, match="unsupported"):
        ops.call("egovlp_space_attn_long_fwd", ops._ptr(qkv), ops._ptr(out), ops._ptr(lse), ops._ptr(ws), B, T, N, H,
                 ops._stream())
    with pytest.raises(EgovlpError, match="unsupported"):
        ops.call("egovlp_space_attn_long_bwd", ops._ptr(qkv), ops._ptr(out), ops._ptr(dout), ops._ptr(lse),
                 ops._ptr(dqkv), ops._ptr(ws), B, T, N, H, C.c_float(Q_SCALE), ops._stream())
    torch.cuda.synchronize()
    assert out.isnan().all() and lse.isnan().all() and dqkv.isnan().all() and ws.isnan().all()


# ------------------------------------------------------------------------------------------------ time attention
# The time attention keeps its kernels at large frames (N only sets the number of groups): T = 4, 8, 16 on the fast
# path, T = 3 on the generic one, every path paths_for admits.
TIME = [(2, t, n, 0) for n in (256, 576, 1024) for t in (4, 8, 16, 3)]


@pytest.mark.parametrize("B,T,N,H,mode,path", [
    pytest.param(B, T, N, H, mode, path, id=f"time-B{B}-T{T}-N{N}-H{H}-{path}")
    for B, T, N, mode in TIME for H in (1, 12) if not (H == 12 and T == 16 and N == 1024)
    for path in paths_for(T, N, mode)])
def test_time_attention_at_large_frames(ops, monkeypatch, B, T, N, H, mode, path):
    check_case(ops, monkeypatch, B, T, N, H, mode, path, seed=3500 + 10 * T + N + H)
