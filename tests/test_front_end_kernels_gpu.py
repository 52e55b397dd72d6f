"""Per-kernel reference tests of the video patch-embedding front end (embed.cu) and the text tower's small kernels
(text.cu; its attention is checked in test_text_attention_gpu.py).  Whole-tower tests check these kernels only through twelve bf16 blocks, at tolerances sized for
that, where a bug in one kernel or one branch is diluted or never runs.

Each reference is the same operation written plainly in torch, computed in float64 on the GPU from the same bf16 / fp32
values the kernel reads.  The bound follows from what the kernel does:
  * gathers, casts and adds done in the order torch does them match bit for bit (`assert_bits_equal`);
  * fp32 arithmetic rounded once to bf16 is within one bf16 ulp per element (`assert_bf16_ulps`);
  * reductions stay within |got - ref| <= rel * sum|terms| element-wise (`assert_sum_bound`): the error of an fp32 sum
    scales with the magnitudes it adds, not with its (possibly cancelled) result, and one relative L2 over the whole
    tensor would let a single wrong element through;
  * GEMM outputs are also checked per row (`assert_rows_close`), so that one wrong row cannot hide among thousands of
    correct ones.
Each check prints its worst element or row as a fraction of its bound (run with -s to see them)."""
import pytest
import torch
from gemm_ref import check, reference
from kernel_checks import (BF16, F32, F64, assert_bf16_ulps, assert_bits_equal, assert_rows_close, assert_sum_bound, mk,
                           nan_filled, rel_l2)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


@pytest.fixture(params=["pair", "single"])
def gemm_mode(request, monkeypatch):
    monkeypatch.setenv("EGOVLP_GEMM_PAIR", "1" if request.param == "pair" else "0")
    return request.param


# ---------------------------------------------------------------------------------------------------------- A. video front end
def patches_of(video, P):
    """[B, T, C, H, W] -> [B * S, C * P * P]: patch rows b*S + 1 + t*N + n, column c*P*P + iy*P + ix, CLS rows zero."""
    B, T, C, H, W = video.shape
    gh, gw = H // P, W // P
    tok = video.reshape(B * T, C, gh, P, gw, P).permute(0, 2, 4, 1, 3, 5).reshape(B, T * gh * gw, C * P * P)
    return torch.cat([torch.zeros_like(tok[:, :1]), tok], dim=1).reshape(-1, C * P * P)


# the last shape has 8*16*196*3*16*4 = 4.8M work items, more than the 132 * 32 * 256 threads of the grid: the
# grid-stride loop runs more than once
@pytest.mark.parametrize("B,T,C,H,W,P", [(2, 4, 3, 224, 224, 16), (3, 1, 3, 32, 48, 16), (2, 3, 1, 24, 24, 12),
                                         (1, 2, 3, 16, 16, 4), (8, 16, 3, 224, 224, 16)])
def test_patch_im2col_is_an_exact_gather_and_cast(ops, B, T, C, H, W, P):
    video = mk((B, T, C, H, W), 1, dtype=F32)
    S, K = 1 + T * (H // P) * (W // P), C * P * P
    patches = nan_filled((B * S, K), BF16)
    ops.patch_im2col(video, patches, P)
    assert not patches.isnan().any(), "patch_im2col left elements unwritten"
    assert torch.all(patches.view(B, S, K)[:, 0] == 0)
    assert_bits_equal(f"patch_im2col {(B, T, C, H, W, P)}", patches, patches_of(video, P).to(BF16))


def test_patch_im2col_u8_normalises_every_byte_within_one_ulp(ops):
    B, T, H, W, P = 2, 3, 32, 48, 16
    g = torch.Generator(device="cuda").manual_seed(2)
    video = torch.randint(0, 256, (B, T, 3, H, W), generator=g, device="cuda", dtype=torch.uint8)
    video[1, 2, :, :16, :16] = torch.arange(256, device="cuda", dtype=torch.uint8).view(16, 16)   # every byte, every channel
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    S, K = 1 + T * (H // P) * (W // P), 3 * P * P
    patches = nan_filled((B * S, K), BF16)
    ops.patch_im2col_u8(video, patches, P, mean, std)
    assert not patches.isnan().any()
    assert torch.all(patches.view(B, S, K)[:, 0] == 0)
    # the kernel receives mean / std as fp32
    m = torch.tensor(mean, dtype=F32).to("cuda", F64).view(1, 1, 3, 1, 1)
    s = torch.tensor(std, dtype=F32).to("cuda", F64).view(1, 1, 3, 1, 1)
    assert_bf16_ulps("patch_im2col_u8", patches, patches_of((video.double() / 255 - m) / s, P))


def test_video_pos_table_is_exact(ops):
    T, N, D, F = 3, 10, 96, 16                   # temporal_embed has more rows (frames) than the clip uses
    cls, pos = mk((1, 1, D), 3, dtype=F32), mk((1, 1 + N, D), 4, dtype=F32)
    temporal, bias = mk((1, F, D), 5, dtype=F32), mk((D,), 6, dtype=F32)
    table = nan_filled((1 + T * N, D), F32)
    ops.video_pos_table(cls, pos, temporal, bias, table, T, N, D)
    ref = torch.empty_like(table)
    ref[0] = (cls[0, 0] + pos[0, 0]) - bias
    ref[1:] = (pos[0, 1:].unsqueeze(0) + temporal[0, :T].unsqueeze(1)).reshape(T * N, D)
    assert_bits_equal("video_pos_table", table, ref)


def embed_sums(dx, T, N):
    """(dcls, dpos, dtemporal[:T], dbias) of the embedding assembly for an upstream gradient dx [B, S, D]."""
    B, _, D = dx.shape
    cls = dx[:, 0].sum(0)
    tok = dx[:, 1:].reshape(B, T, N, D)
    return cls, torch.cat([cls[None], tok.sum((0, 1))]), tok.sum((0, 2)), tok.sum((0, 1, 2))


@pytest.mark.parametrize("B,T,N,D", [(32, 16, 196, 768), (2, 16, 4, 64), (3, 1, 1, 8), (1, 5, 7, 12)])
def test_video_embed_bwd_accumulates_within_the_reduction_bound(ops, B, T, N, D):
    """(2, 16, 4, 64) has T > N: the reduction grid is sized by max(N, T) * D."""
    F, S = T + 3, 1 + T * N
    dx = mk((B, S, D), 7, dtype=F32)
    bases = [mk(shape, 8 + i, dtype=F32) for i, shape in enumerate([(D,), (1 + N, D), (F, D), (D,)])]
    outs = [b.clone() for b in bases]                 # the outputs accumulate
    tmp = nan_filled((S * D,), F32)
    ops.video_embed_bwd(dx, tmp, *outs, B, T, N, D)
    ref, terms = embed_sums(dx.double(), T, N), embed_sums(dx.double().abs(), T, N)
    for name, got, base, r, t in zip(("dcls", "dpos", "dtemporal", "dbias"), outs, bases, ref, terms):
        rows = r.shape[0] if name == "dtemporal" else got.shape[0]
        base = base[:rows].double()
        assert_sum_bound(f"video_embed_bwd {name} {(B, T, N, D)}", got[:rows], base + r, base.abs() + t)
    assert_bits_equal("video_embed_bwd dtemporal rows >= T", outs[2][T:], bases[2][T:])


@pytest.mark.parametrize("B,S", [(3, 197), (2, 1 + 4 * 196)])
def test_patch_embed_gemm_adds_the_table_row_m_mod_s(ops, gemm_mode, B, S):
    """The conv-as-GEMM of the patch embedding: out = patches @ W^T + bias + table[m % S] (res_row_mod = S); B * S rows,
    so the last m-block is ragged."""
    D, K = 768, 768
    M = B * S
    a, w = mk((M, K), 20), mk((D, K), 21, 0.05)
    bias, table = mk((D,), 22, dtype=F32), mk((S, D), 23, dtype=F32)
    out = nan_filled((M, D), F32)
    ops.gemm(a, w, out, bias=bias, residual=table, res_row_mod=S)
    rows = torch.arange(M, device="cuda") % S
    ref = a.double() @ w.double().t() + bias.double() + table.double()[rows]
    err = rel_l2(out, ref)
    print(f"[bound] patch-embedding GEMM S={S} {gemm_mode}: rel-L2 {err:.3g} (bound 2e-5)")
    assert err < 2e-5
    assert_rows_close(f"patch-embedding GEMM S={S} {gemm_mode} per row", out, ref, rtol=1e-4, atol=0.0)
    check(f"patch-embedding GEMM S={S} {gemm_mode}", out, reference(a, w, bias=bias, residual=table, res_row_mod=S)["out"])


@pytest.mark.parametrize("H,W,P", [(32, 48, 16), (36, 48, 12)])
def test_patch_embed_fn_matches_the_reference_embedding(gemm_mode, H, W, P):
    """engine.PatchEmbedFn forward and backward against oracle.reference_port.video_tokens in fp64.  The reference gets
    the video and the conv weight rounded to bf16, as the GEMM reads them, so that what remains is fp32 accumulation.
    P = 12 gives K = 3 * 12 * 12 = 432, not a multiple of 64 (or 32)."""
    from egovlp_b200 import engine
    from oracle import reference_port as rp
    B, T, F, C, D = 2, 3, 4, 3, 256
    N = (H // P) * (W // P)
    S = 1 + T * N
    video = mk((B, T, C, H, W), 30, dtype=F32)
    init = {"cls_token": mk((1, 1, D), 31, dtype=F32), "pos_embed": mk((1, 1 + N, D), 32, dtype=F32),
            "temporal_embed": mk((1, F, D), 33, dtype=F32), "patch_embed.proj.weight": mk((D, C, P, P), 34, 0.05, F32),
            "patch_embed.proj.bias": mk((D,), 35, dtype=F32)}
    p = {k: v.clone().requires_grad_(True) for k, v in init.items()}
    x = engine.PatchEmbedFn.apply(video, p["cls_token"], p["pos_embed"], p["temporal_embed"],
                                  p["patch_embed.proj.weight"], p["patch_embed.proj.bias"], engine.Bf16Cache())
    g = mk((B, S, D), 36, dtype=F32)
    x.backward(g)

    p64 = {"video_model." + k: (v.to(BF16) if k == "patch_embed.proj.weight" else v).double().requires_grad_(True)
           for k, v in init.items()}
    tok, _, _ = rp.video_tokens(video.to(BF16).double(), p64)
    err = rel_l2(x.detach(), tok.detach())
    print(f"[bound] PatchEmbedFn tokens P={P} {gemm_mode}: rel-L2 {err:.3g} (bound 2e-5)")
    assert err < 2e-5
    names = ["cls_token", "pos_embed", "temporal_embed", "patch_embed.proj.bias"]
    leaves = [p64["video_model." + k] for k in names]
    ref = torch.autograd.grad(tok, leaves, g.double(), retain_graph=True)
    terms = torch.autograd.grad(tok, leaves, g.double().abs(), retain_graph=True)   # every term enters with weight +1
    for k, r, t in zip(names, ref, terms):
        assert_sum_bound(f"PatchEmbedFn d{k} P={P} {gemm_mode}", p[k].grad, r, t)
    # the engine rounds the upstream gradient to bf16 before the weight-gradient GEMM
    (rw,) = torch.autograd.grad(tok, [p64["video_model.patch_embed.proj.weight"]], g.to(BF16).double())
    err = rel_l2(p["patch_embed.proj.weight"].grad, rw)
    print(f"[bound] PatchEmbedFn dconv_weight P={P} {gemm_mode}: rel-L2 {err:.3g} (bound 2e-5)")
    assert err < 2e-5


# ---------------------------------------------------------------------------------------------------------- B. text tower
def test_text_embed_fwd_is_an_exact_gather_plus_add(ops):
    B, L, D, V, n_pos = 7, 13, 96, 50, 40
    g = torch.Generator(device="cuda").manual_seed(40)
    ids = torch.randint(0, V, (B, L), generator=g, device="cuda")
    word, pos = mk((V, D), 41, dtype=F32), mk((n_pos, D), 42, dtype=F32)
    out = nan_filled((B * L, D), F32)
    ops.text_embed_fwd(ids, word, pos, out, B, L, D)
    assert_bits_equal("text_embed_fwd", out, (word[ids] + pos[:L]).reshape(B * L, D))


@pytest.mark.parametrize("B,L,distinct", [(16, 128, False), (4, 20, True)])
def test_text_embed_bwd_accumulates_within_the_reduction_bound(ops, B, L, distinct):
    """16 x 128 = 2048 tokens drawn from 5 ids: ~400 atomics land on each of those rows.  Then one batch of all-distinct
    ids.  The outputs accumulate onto a random base; rows of unused ids and positions >= L must keep it bit for bit."""
    D, V, n_pos = 96, 100, 130
    g = torch.Generator(device="cuda").manual_seed(43)
    if distinct:
        ids = torch.randperm(V, generator=g, device="cuda")[:B * L].view(B, L)
    else:
        vocab = torch.tensor([3, 17, 18, 64, 99], device="cuda")
        ids = vocab[torch.randint(0, 5, (B, L), generator=g, device="cuda")]
    dsum = mk((B * L, D), 44, dtype=F32)
    base_w, base_p = mk((V, D), 45, dtype=F32), mk((n_pos, D), 46, dtype=F32)
    dword, dpos = base_w.clone(), base_p.clone()
    ops.text_embed_bwd(ids, dsum, dword, dpos, B, L, D)
    flat = ids.flatten()

    def per_id(t):
        return torch.zeros(V, D, device="cuda", dtype=F64).index_add_(0, flat, t)

    d64 = dsum.double()
    assert_sum_bound(f"text_embed_bwd dword {B}x{L}", dword, base_w.double() + per_id(d64),
                     base_w.double().abs() + per_id(d64.abs()))
    assert_sum_bound(f"text_embed_bwd dpos {B}x{L}", dpos[:L], base_p[:L].double() + d64.view(B, L, D).sum(0),
                     base_p[:L].double().abs() + d64.abs().view(B, L, D).sum(0))
    unused = torch.ones(V, dtype=torch.bool, device="cuda")
    unused[flat] = False
    assert_bits_equal("text_embed_bwd unused ids", dword[unused], base_w[unused])
    assert_bits_equal("text_embed_bwd positions >= L", dpos[L:], base_p[L:])


@pytest.mark.parametrize("cls_only", [False, True])
def test_relu_rows_forward_and_backward_are_exact(ops, cls_only):
    """Token mode (row stride D) and the CLS rows of [B, L, D] (row stride L * D).  x holds exact zeros, where the
    gradient of ReLU is 0 in torch and must be in the kernel too."""
    B, L, D = 6, 11, 96
    x = mk((B * L, D), 50, dtype=F32)
    x[:, ::5] = 0.0
    rows, stride = (B, L * D) if cls_only else (B * L, D)
    xr = x.view(B, L * D)[:, :D] if cls_only else x
    out = nan_filled((rows, D), BF16)
    ops.relu_rows_fwd(x, stride, out, rows, D)
    assert torch.equal(out, torch.relu(xr).to(BF16))
    dh = mk((rows, D), 51, dtype=F32)
    sentinel = 12345.0
    dx = torch.full((B * L, D), sentinel, device="cuda")
    ops.relu_rows_bwd(x, stride, dh, dx, rows, D)
    xg = xr.clone().requires_grad_(True)
    torch.relu(xg).backward(dh)
    assert bool((xg.grad[xr == 0] == 0).all()) and bool((dh[xr == 0] != 0).all())
    got = dx.view(B, L * D)[:, :D] if cls_only else dx
    assert torch.equal(got, xg.grad)
    if cls_only:                  # only the CLS token rows (row index a multiple of L) are written
        assert torch.all(dx.view(B, L, D)[:, 1:] == sentinel)
