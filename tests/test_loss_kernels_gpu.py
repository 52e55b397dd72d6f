"""The similarity and contrastive-loss kernels (csrc/loss.cu, csrc/loss_fused.cu) against float64, element by element.

loss_ref.py holds the reference, derives every bound from the kernels' arithmetic and builds the inputs; its host test
shows that deliberate faults miss those bounds by 10x or more.  Inputs come in two regimes: Gaussian embeddings (flat
softmaxes) and the training regime (diagonal cosines about 0.9, logits up to 18-20, duplicated clips, an all-zero row
and a row of norm 1e-9 below eps, EgoClip-sized tags with an all-zero noun row).

The fused kernels are called through their C entry points, on row-strided column views of one packed buffer with an
odd row stride (as the gathered step hands them), into NaN-filled outputs followed by sentinel rows: every element must
be written and no sentinel touched.  Only the column partials of the workspace are NaN-filled; its ticket word starts
at zero.  Each check prints its worst element as a fraction of its bound (run with -s)."""
import ctypes as C

import pytest
import torch
from kernel_checks import F32, F64, assert_bits_equal, assert_elementwise_bound, assert_sum_bound, nan_filled
from loss_ref import (EPS_F32, SLACK, U, egonce_reference, f32, fused_case, mask_from_sims_ref, maxmargin_case,
                      maxmargin_reference, nce_case, nce_reference, norm_rel, pack_bits, positives,
                      rownorm_bwd_reference, signed_sims, sgemm_reference, tags)

pytestmark = pytest.mark.gpu

SENT_ROWS = 3
SENTINEL = -3.0
GSCALE = 0.75
FUSED_G = [1, 2, 7, 31, 32, 33, 63, 64, 65, 255, 256, 257, 511, 512]
FUSED_C = [1, 31, 32, 33, 255, 256]
TAG_WIDTHS = [(118, 582), (1, 31), (32, 33), (33, 32), (31, 582)]
FUSED_CASES = [(G, FUSED_C[i % 6], i % 4, *TAG_WIDTHS[i % 5], regime)
               for i, G in enumerate(FUSED_G) for regime in ("train", "gauss")]


@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


def with_sentinels(rows, *cols, dtype=F32):
    buf = nan_filled((rows + SENT_ROWS, *cols), dtype)
    buf[rows:] = SENTINEL
    return buf


def check_written(name, buf, rows):
    torch.cuda.synchronize()
    assert not buf[:rows].isnan().any(), f"{name}: {int(buf[:rows].isnan().sum())} elements NaN (unwritten, or NaN data)"
    assert bool((buf[rows:] == SENTINEL).all()), f"{name}: a row past the output was written"
    return buf[:rows]


def packed_views(t, v, verb, noun):
    """Column views of ONE [G, W] buffer, W odd (a NaN pad column if needed): text | video | verb | noun."""
    parts = [t, v, verb, noun]
    W = sum(p.shape[1] for p in parts)
    buf = nan_filled((t.shape[0], W + (W % 2 == 0)), F32)
    views, c = [], 0
    for p in parts:
        buf[:, c:c + p.shape[1]] = p.cuda()
        views.append(buf[:, c:c + p.shape[1]])
        c += p.shape[1]
    return views


def widths(mode, nv, nn):
    return (nv + 31) // 32 if mode in (1, 3) else 0, (nn + 31) // 32 if mode in (1, 2) else 0


def fused_fwd(ops, views, mode, inv_temp):
    from egovlp_b200._lib import lib
    t, v, vb, nb = views
    G, Cc = t.shape
    nv, nn = vb.shape[1], nb.shape[1]
    Wv, Wn = widths(mode, nv, nn)
    na, nvid, stats, loss = (with_sentinels(n) for n in (G, G, 4 * G, 1))
    want_bits = torch.cat([pack_bits(vb)[:, :Wv], pack_bits(nb)[:, :Wn]], 1).cuda()
    bits = torch.full((G + SENT_ROWS, max(1, Wv + Wn)), -3, dtype=torch.int32, device="cuda")
    bits[:G, :Wv + Wn] = ~want_bits                       # every word must be overwritten
    ws = nan_filled((lib().egovlp_egonce_fused_workspace_floats(G),), F32)
    ws[-4:] = 0.0                                          # the ticket word
    ops.call("egovlp_egonce_fused_fwd", ops._ptr(t), C.c_longlong(t.stride(0)), ops._ptr(v), C.c_longlong(v.stride(0)),
             ops._ptr(vb), C.c_longlong(vb.stride(0)), nv, ops._ptr(nb), C.c_longlong(nb.stride(0)), nn, G, Cc,
             C.c_float(inv_temp), mode, C.c_float(EPS_F32), ops._ptr(na), ops._ptr(nvid), ops._ptr(bits),
             ops._ptr(stats), ops._ptr(ws), ops._ptr(loss), ops._stream())
    out = {k: check_written(k, b, n) for k, b, n in
           (("norm_text", na, G), ("norm_video", nvid, G), ("stats", stats, 4 * G), ("loss", loss, 1))}
    assert torch.equal(bits[:G, :Wv + Wn], want_bits), "tag_bits differ from the host packing"
    assert bool((bits[G:] == -3).all()), "tag_bits: a row past the output was written"
    assert ws[-4:].view(torch.int32)[0].item() == 0, "the ticket word was not reset"
    out["bits"] = bits[:G]
    return out


def fused_bwd(ops, views, fwd, mode, inv_temp, row0, n_local):
    t, v, vb, nb = views
    G, Cc = t.shape
    dt, dv = with_sentinels(n_local, Cc), with_sentinels(n_local, Cc)
    gscale = torch.tensor(GSCALE, dtype=F32, device="cuda")
    ops.call("egovlp_egonce_fused_bwd", ops._ptr(t), C.c_longlong(t.stride(0)), ops._ptr(v), C.c_longlong(v.stride(0)),
             ops._ptr(fwd["norm_text"]), ops._ptr(fwd["norm_video"]), ops._ptr(fwd["bits"]), vb.shape[1], nb.shape[1],
             ops._ptr(fwd["stats"]), G, Cc, C.c_float(inv_temp), mode, C.c_float(EPS_F32), ops._ptr(gscale), row0,
             n_local, ops._ptr(dt), ops._ptr(dv), ops._stream())
    return check_written("d_text", dt, n_local), check_written("d_video", dv, n_local)


def check_scalar(name, got, ref, bound):
    assert_elementwise_bound(name, got.reshape(1), ref.reshape(1), bound.reshape(1))


def check_fused(tag, r, fwd):
    check_scalar(f"loss {tag}", fwd["loss"], r["loss"], r["loss_err"])
    assert_elementwise_bound(f"stats {tag}", fwd["stats"], r["stats"], r["stats_err"])
    for k in ("norm_text", "norm_video"):
        assert_elementwise_bound(f"{k} {tag}", fwd[k], r[k], r[k + "_err"] + 1e-45)


def slices(G):
    s = [(0, G)]
    if G >= 16:
        s += [(0, 1), (5, 3), (G - 13, 13)]
    return s


@pytest.mark.parametrize("G,Cc,mode,nv,nn,regime", FUSED_CASES)
def test_fused_matches_fp64(ops, G, Cc, mode, nv, nn, regime):
    t, v, verb, noun, mask, temp = fused_case(G, Cc, mode, nv, nn, G + Cc, regime)
    it = f32(1 / temp)
    views = packed_views(t, v, verb, noun)
    fwd = fused_fwd(ops, views, mode, it)
    r = egonce_reference(t.cuda(), v.cuda(), mask.cuda(), it, "fused", gscale=GSCALE)
    tag = f"fused G={G} C={Cc} mode={mode} tags={nv}/{nn} {regime}"
    check_fused(tag, r, fwd)
    for row0, n in slices(G):
        dt, dv = fused_bwd(ops, views, fwd, mode, it, row0, n)
        sl = slice(row0, row0 + n)
        assert_elementwise_bound(f"d_text {tag} rows {row0}+{n}", dt, r["d_text"][sl], r["d_text_err"][sl])
        assert_elementwise_bound(f"d_video {tag} rows {row0}+{n}", dv, r["d_video"][sl], r["d_video_err"][sl])


@pytest.mark.parametrize("G,ranks", [(9, 3), (96, 8), (512, 8)])
def test_fused_reproducible_and_sliceable(ops, G, ranks):
    """Two runs agree bit for bit, and the per-rank backward slices concatenated equal one call over all rows."""
    t, v, verb, noun, mask, temp = fused_case(G, 256, 1, 118, 582, G, "train")
    it = f32(1 / temp)
    views = packed_views(t, v, verb, noun)
    runs = []
    for _ in range(2):
        fwd = fused_fwd(ops, views, 1, it)
        runs.append((fwd, *fused_bwd(ops, views, fwd, 1, it, 0, G)))
    for name, i in (("loss", 0), ("stats", 0), ("norm_text", 0)):
        assert_bits_equal(f"{name} G={G} run to run", runs[1][0][name], runs[0][0][name])
    assert_bits_equal(f"d_text G={G} run to run", runs[1][1], runs[0][1])
    assert_bits_equal(f"d_video G={G} run to run", runs[1][2], runs[0][2])
    B = G // ranks
    parts = [fused_bwd(ops, views, runs[0][0], 1, it, k * B, B) for k in range(ranks)]
    assert_bits_equal(f"d_text G={G} per-rank slices", torch.cat([p[0] for p in parts]), runs[0][1])
    assert_bits_equal(f"d_video G={G} per-rank slices", torch.cat([p[1] for p in parts]), runs[0][2])


@pytest.mark.parametrize("G", [1, 2, 7, 31])
def test_fused_bwd_small_g_after_nan_launches(ops, G):
    """Below G = 32 the backward's one column tile is partly empty.  Launched right after kernels that leave NaN in
    shared memory (the fused forward and backward on NaN inputs), it must not read the rows it did not load."""
    tn, vn, vb, nb = packed_views(*(torch.full((64, c), float("nan")) for c in (256, 256, 118, 582)))
    _poison_launches(ops, (tn, vn, vb, nb))
    t, v, verb, noun, mask, temp = fused_case(G, 256, 1, 118, 582, G, "train")
    it = f32(1 / temp)
    views = packed_views(t, v, verb, noun)
    fwd = fused_fwd(ops, views, 1, it)
    _poison_launches(ops, (tn, vn, vb, nb))
    r = egonce_reference(t.cuda(), v.cuda(), mask.cuda(), it, "fused", gscale=GSCALE)
    dt, dv = fused_bwd(ops, views, fwd, 1, it, 0, G)
    assert_elementwise_bound(f"d_text G={G} after NaN launches", dt, r["d_text"], r["d_text_err"])
    assert_elementwise_bound(f"d_video G={G} after NaN launches", dv, r["d_video"], r["d_video_err"])


def _poison_launches(ops, views):
    """The fused forward and backward at G = 64 on NaN inputs: NaN in every shared-memory row they use."""
    from egovlp_b200._lib import lib
    t, v, vb, nb = views
    G = t.shape[0]
    na, nvid, stats, loss = (torch.empty(n, device="cuda") for n in (G, G, 4 * G, 1))
    bits = torch.empty(G, 23, dtype=torch.int32, device="cuda")
    ws = nan_filled((lib().egovlp_egonce_fused_workspace_floats(G),), F32)
    ws[-4:] = 0.0
    ops.call("egovlp_egonce_fused_fwd", ops._ptr(t), C.c_longlong(t.stride(0)), ops._ptr(v), C.c_longlong(v.stride(0)),
             ops._ptr(vb), C.c_longlong(vb.stride(0)), 118, ops._ptr(nb), C.c_longlong(nb.stride(0)), 582, G, 256,
             C.c_float(20.0), 1, C.c_float(EPS_F32), ops._ptr(na), ops._ptr(nvid), ops._ptr(bits), ops._ptr(stats),
             ops._ptr(ws), ops._ptr(loss), ops._stream())
    fwd = {"norm_text": na, "norm_video": nvid, "bits": bits, "stats": stats}
    dt, dv = (torch.empty(G, 256, device="cuda") for _ in range(2))
    ops.call("egovlp_egonce_fused_bwd", ops._ptr(t), C.c_longlong(t.stride(0)), ops._ptr(v), C.c_longlong(v.stride(0)),
             ops._ptr(na), ops._ptr(nvid), ops._ptr(bits), 118, 582, ops._ptr(stats), G, 256, C.c_float(20.0), 1,
             C.c_float(EPS_F32), ops._ptr(None), 0, G, ops._ptr(dt), ops._ptr(dv), ops._stream())
    torch.cuda.synchronize()
    assert dt.isnan().all(), "the NaN launches were expected to produce NaN"


# ------------------------------------------------------------------------------------------------ staged path kernels
@pytest.mark.parametrize("G", [1, 33, 513, 1024])
def test_pack_and_positives_masks(ops, G):
    verb, noun = tags(G, 118, 582, G)
    for t in (verb, noun):
        W = (t.shape[1] + 31) // 32
        bits = torch.full((G + SENT_ROWS, W), -3, dtype=torch.int32, device="cuda")
        want = pack_bits(t).cuda()
        bits[:G] = ~want
        ops.call("egovlp_pack_multihot", ops._ptr(t.cuda()), ops._ptr(bits), G, t.shape[1], ops._stream())
        assert torch.equal(bits[:G], want) and bool((bits[G:] == -3).all()), f"pack_multihot G={G} n={t.shape[1]}"
    sv, sn = signed_sims(G, G)
    sv.diagonal()[::3] = 0.0
    for mode in range(4):
        m = ops.positives_mask_from_tags(verb.cuda(), noun.cuda(), mode)
        assert torch.equal(m.bool().cpu(), positives(verb, noun, mode)), f"mask_from_bits G={G} mode={mode}"
        got = ops.positives_mask_from_sims(sv.cuda() if mode else None, sn.cuda() if mode else None, G, mode,
                                           device="cuda")
        want = mask_from_sims_ref(sv, sn, mode, G)
        assert torch.equal(got.bool().cpu(), want), f"mask_from_sims G={G} mode={mode}"
    print(f"[bound] pack_multihot / mask_from_bits / mask_from_sims G={G}: exact")


@pytest.mark.parametrize("Cc", [1, 31, 32, 33, 256, 257, 768])
def test_rownorm_matches_fp64(ops, Cc):
    rows = 67
    g = torch.Generator().manual_seed(Cc)
    a = torch.randn(rows, Cc, generator=g)
    a[3] = 0.0
    a[5] *= 1e-9 / a[5].norm()
    a[7] *= 1e6 / a[7].norm()
    a = a.cuda()
    an_buf, n_buf = with_sentinels(rows, Cc), with_sentinels(rows)
    ops.call("egovlp_rownorm_fwd", ops._ptr(a), ops._ptr(an_buf), ops._ptr(n_buf), rows, Cc, C.c_float(EPS_F32),
             ops._stream())
    an, n = check_written("an", an_buf, rows), check_written("norm", n_buf, rows)
    n64 = a.double().norm(dim=1)
    an64 = a.double() / n64.clamp_min(EPS_F32)[:, None]
    nrel = norm_rel(Cc, False)
    assert_elementwise_bound(f"rownorm norm C={Cc}", n, n64, SLACK * nrel * n64 + 1e-45)
    assert_elementwise_bound(f"rownorm an C={Cc}", an, an64, SLACK * (nrel + 2 * U) * an64.abs() + 1e-45)
    dan = torch.randn(rows, Cc, generator=g).cuda()
    da_buf = with_sentinels(rows, Cc)
    ops.call("egovlp_rownorm_bwd", ops._ptr(dan), ops._ptr(an), ops._ptr(n), ops._ptr(da_buf), rows, Cc,
             C.c_float(EPS_F32), ops._stream())
    da = check_written("da", da_buf, rows)
    ref, err = rownorm_bwd_reference(dan, an, n, EPS_F32, Cc)
    assert_elementwise_bound(f"rownorm da C={Cc}", da, ref, err + 1e-45)


SGEMM_SHAPES = [(1, 1, 1), (31, 32, 33), (33, 31, 257), (257, 33, 32), (1024, 1, 33), (32, 1024, 31), (257, 257, 1024),
                (1, 257, 1024)]


@pytest.mark.parametrize("M,N,K", SGEMM_SHAPES)
@pytest.mark.parametrize("trans_a,trans_b", [(False, True), (False, False), (True, True), (True, False)])
def test_sgemm_matches_fp64(ops, M, N, K, trans_a, trans_b):
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, generator=g).cuda()
    b = torch.randn(N, K, generator=g).cuda()
    a_in = a.T.contiguous() if trans_a else a
    b_in = b if trans_b else b.T.contiguous()
    for alpha, beta in ((1.0, 0.0), (-1.5, 0.0), (0.75, 0.5)):
        buf = with_sentinels(M, N + 5)                  # ldc = N + 5 > N: the pad columns must stay NaN
        c0 = torch.randn(M, N, generator=g).cuda()
        if beta != 0.0:
            buf[:M, :N] = c0
        ops.sgemm(a_in, b_in, trans_a=trans_a, trans_b=trans_b, out=buf[:M, :N], alpha=alpha, beta=beta)
        torch.cuda.synchronize()
        assert buf[:M, N:].isnan().all() and bool((buf[M:] == SENTINEL).all()), "sgemm wrote outside C"
        got = buf[:M, :N]
        assert not got.isnan().any(), "sgemm read C with beta = 0, or left it unwritten"
        ref, mag = sgemm_reference(a, b, f32(alpha), f32(beta), c0)
        assert_sum_bound(f"sgemm {M}x{N}x{K} ta={trans_a} tb={trans_b} a={alpha} b={beta}", got, ref, mag,
                         rel=SLACK * (K + 3) * U)


@pytest.mark.parametrize("G", [1, 2, 33, 512, 513, 1024, 2048])
def test_nce_matches_fp64(ops, G):
    x, mask, temp = nce_case(G, G)
    it = f32(1 / temp)
    xc, mc = x.cuda(), mask.to(torch.uint8).cuda()
    stats_buf, loss_buf = with_sentinels(4 * G), with_sentinels(1)
    ops.call("egovlp_nce_fwd", ops._ptr(xc), ops._ptr(mc), G, C.c_float(it), ops._ptr(stats_buf), ops._ptr(loss_buf),
             ops._stream())
    stats, loss = check_written("stats", stats_buf, 4 * G), check_written("loss", loss_buf, 1)
    r = nce_reference(xc, mask.cuda(), it, GSCALE)
    assert_elementwise_bound(f"nce stats G={G}", stats, r["stats"], r["stats_err"])
    check_scalar(f"nce loss G={G}", loss, r["loss"], r["loss_err"])
    dx_buf = with_sentinels(G, G)
    gscale = torch.tensor(GSCALE, device="cuda")
    ops.call("egovlp_nce_bwd", ops._ptr(xc), ops._ptr(mc), ops._ptr(stats), G, C.c_float(it), ops._ptr(gscale),
             ops._ptr(dx_buf), ops._stream())
    dx = check_written("dx", dx_buf, G)
    assert_elementwise_bound(f"nce dx G={G}", dx, r["dx"], r["dx_err"])


@pytest.mark.parametrize("G,Cc,nv,nn", [(513, 256, 118, 582), (1024, 256, 118, 582), (2048, 256, 118, 582),
                                        (512, 257, 118, 582), (512, 256, 118, 2000)])
def test_staged_egonce_matches_fp64(ops, G, Cc, nv, nn):
    """EgoNCE.fused on the kernel-per-stage path: above 512 rows, at C > 256, and with a tag vocabulary whose bits do
    not fit in the fused kernel's shared memory."""
    from egovlp_b200.model.loss import EgoNCE
    assert not ops.egonce_fused_supported(G, Cc, nv, nn, 1)
    t, v, verb, noun, mask, temp = fused_case(G, Cc, 1, nv, nn, G, "train")
    tc, vc = t.cuda().requires_grad_(True), v.cuda().requires_grad_(True)
    loss = EgoNCE(temperature=temp).fused(tc, vc, verb.cuda(), noun.cuda())
    (loss * GSCALE).backward()
    r = egonce_reference(t.cuda(), v.cuda(), mask.cuda(), f32(1 / temp), "staged", gscale=GSCALE)
    tag = f"staged G={G} C={Cc} tags={nv}/{nn}"
    check_scalar(f"loss {tag}", loss.detach(), r["loss"], r["loss_err"])
    assert_elementwise_bound(f"d_text {tag}", tc.grad, r["d_text"], r["d_text_err"])
    assert_elementwise_bound(f"d_video {tag}", vc.grad, r["d_video"], r["d_video_err"])


@pytest.mark.parametrize("G", [2, 3, 33, 256, 257, 1024])
@pytest.mark.parametrize("fix_norm", [True, False])
@pytest.mark.parametrize("adaptive", [False, True])
def test_maxmargin_matches_fp64(ops, G, fix_norm, adaptive):
    x, w = maxmargin_case(G, G, adaptive)
    xc = x.cuda()
    wc = w.cuda() if w is not None else None
    r = maxmargin_reference(x.cuda(), 0.25, fix_norm, wc, GSCALE)
    loss = ops.maxmargin_fwd(xc, 0.25, fix_norm, wc)
    dx = ops.maxmargin_bwd(xc, 0.25, fix_norm, torch.tensor(GSCALE, device="cuda"), wc)
    tag = f"maxmargin G={G} fix_norm={fix_norm} adaptive={adaptive}"
    check_scalar(f"loss {tag}", loss, r["loss"], r["loss_err"])
    assert_elementwise_bound(f"dx {tag}", dx, r["dx"], r["dx_err"])
    assert bool((dx[r["active"] == 0] == 0).all()), "a gradient where no hinge is active (relu'(0) = 0)"
