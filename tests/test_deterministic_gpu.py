"""Deterministic mode: under torch.use_deterministic_algorithms(True) every reducing kernel of the training step takes
its fixed-order form, so equal inputs give equal bits.

Per kernel: three launches on inputs whose sums are order-sensitive (magnitudes spread over 2^20) give identical bits,
and the result stays within the fp64 bounds the kernel tests use.  The split-K GEMM is held to its exact contract:
out = ((out + P_0) + P_1) + ..., P_s = the same GEMM with one split over split s's k-blocks.
Per model: one seeded training step (forward, loss, backward, fused AdamW) run three times from the same state gives the
same loss, gradients and updated weights, bit for bit."""
import contextlib
import os
import subprocess
import sys

import pytest
import torch
from kernel_checks import BF16, F32, assert_bits_equal, assert_sum_bound, mk

pytestmark = pytest.mark.gpu
F64 = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def deterministic(warn_only=False):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def spread(shape, seed, dtype=F32):
    """N(0, 1) times 2^e, e uniform in [-10, 10): sums over such terms change with the order they are taken in."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, generator=g, device="cuda")
    e = torch.randint(-10, 10, shape, generator=g, device="cuda").float()
    return (x * torch.exp2(e)).to(dtype)


def three_times(fn):
    """fn() -> tuple of tensors, run three times under the flag; asserts bit equality and returns the first result."""
    runs = []
    for _ in range(3):
        with deterministic():
            runs.append(tuple(t.clone() for t in fn()))
    for r in runs[1:]:
        for i, (a, b) in enumerate(zip(runs[0], r)):
            assert_bits_equal(f"output {i} across launches", b, a)
    return runs[0]


# ---------------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("n_out,n_in", [(2304, 768), (768, 768), (3072, 768), (768, 3072), (200, 256)])
@pytest.mark.parametrize("with_colsum", [False, True])
def test_wgrad_is_the_ordered_sum_of_its_split_partials(n_out, n_in, with_colsum):
    """The step's four weight-gradient shapes, and n_out = 200 (not a multiple of the 128-row tile: the tail rows of
    each split's workspace slab)."""
    from egovlp_b200 import engine, ops
    K = 2 * 16 * 197                               # a step's token rows (B = 2): not a multiple of 64
    dy, x = spread((K, n_out), 1, BF16), spread((K, n_in), 2, BF16)
    split = engine._det_split_for(n_out, n_in, K)
    assert split > 1

    def run():
        dw = torch.zeros(n_out, n_in, device="cuda")
        cs = torch.zeros(n_out, device="cuda") if with_colsum else None
        ops.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=split, colsum_a=cs)
        return (dw, cs) if with_colsum else (dw,)

    got = three_times(run)
    num_kb = -(-K // 64)
    kbps = -(-num_kb // split)
    want_w = torch.zeros(n_out, n_in, device="cuda")
    want_c = torch.zeros(n_out, device="cuda")
    for r0 in range(0, K, kbps * 64):
        r1 = min(K, r0 + kbps * 64)
        p = torch.zeros(n_out, n_in, device="cuda")
        pc = torch.zeros(n_out, device="cuda") if with_colsum else None
        with deterministic():
            ops.gemm(dy[r0:r1], x[r0:r1], p, a_mn=True, b_mn=True, accumulate=True, split_k=1, colsum_a=pc)
        want_w = want_w + p
        if with_colsum:
            want_c = want_c + pc
    assert_bits_equal(f"dW {n_out}x{n_in}", got[0], want_w)
    d64, x64 = dy.double(), x.double()
    assert_sum_bound(f"dW {n_out}x{n_in} vs fp64", got[0], d64.T @ x64, d64.abs().T @ x64.abs())
    if with_colsum:
        assert_bits_equal(f"db {n_out}", got[1], want_c)
        assert_sum_bound(f"db {n_out} vs fp64", got[1], d64.sum(0), d64.abs().sum(0))


def test_gemm_output_colsum_has_no_deterministic_form():
    from egovlp_b200 import ops
    a, b = mk((256, 64), 1), mk((64, 64), 2)
    out = torch.zeros(256, 64, device="cuda")
    with deterministic(), pytest.raises(RuntimeError, match="colsum"):
        ops.gemm(a, b, out, accumulate=True, colsum=torch.zeros(64, device="cuda"))


# ---------------------------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize("T,mode", [(3, 0), (4, 0), (8, 0), (16, 0), (4, 1)])
def test_divided_attention_backward_is_bit_reproducible(T, mode, monkeypatch):
    """T = 3: the generic kernels; 4 / 8 / 16: the time kernel (CLS row in four parts); mode 1: space, N = 196.  The
    A/B switches do not change the bits under the flag."""
    from divided_attention_ref import check_against_reference, make_inputs
    from egovlp_b200 import ops
    B, N, H = 2, 196, 2
    qkv, dout = make_inputs(B, T, N, H, seed=5 + T)
    with deterministic():
        out, lse = ops.divided_attn_fwd(qkv, B, T, N, H, mode)
    dq = three_times(lambda: (ops.divided_attn_bwd(qkv, out, dout, lse, B, T, N, H, mode, 0.125),))[0]
    for env in ({"EGOVLP_ATTN_GENERIC": "1"}, {"EGOVLP_ATTN_TIME_BWD_WARPS": "8"}):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        with deterministic():
            again = ops.divided_attn_bwd(qkv, out, dout, lse, B, T, N, H, mode, 0.125)
        assert_bits_equal(f"dqkv with {env}", again, dq)
        for k in env:
            monkeypatch.delenv(k)
    check_against_reference(f"det T={T} mode={mode}", qkv, dout, out, lse, dq, B, T, N, H, mode, 0.125)


# ---------------------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("rows,dy16", [(4096 + 37, False), (1000, True)])
def test_layernorm_backward_sums_are_bit_reproducible(rows, dy16):
    """4133 rows: the pipelined kernel; 1000: the occupancy-driven one.  All three column sums."""
    from egovlp_b200 import ops
    D = 768
    x = spread((rows, D), 3)
    gamma = 1 + 0.1 * mk((D,), 4, dtype=F32)
    mean, rstd = x.mean(1), torch.rsqrt(x.var(1, unbiased=False) + 1e-6)
    dy = spread((rows, D), 5, BF16 if dy16 else F32)

    def run():
        dx = torch.empty(rows, D, device="cuda")
        sums = [torch.zeros(D, device="cuda") for _ in range(3)]
        ops.layernorm_bwd(dy, x, gamma, mean, rstd, dx=dx, dgamma=sums[0], dbeta=sums[1], colsum_dx=sums[2])
        return (dx, *sums)

    dx, dg, db, cs = three_times(run)
    xh = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    d64 = dy.double()
    assert_sum_bound("dgamma", dg, (d64 * xh).sum(0), (d64 * xh).abs().sum(0))
    assert_sum_bound("dbeta", db, d64.sum(0), d64.abs().sum(0))
    assert_sum_bound("colsum_dx", cs, dx.double().sum(0), dx.double().abs().sum(0))
    with torch.no_grad():                  # the plain form computes dx the same way
        dx2 = torch.empty_like(dx)
        ops.layernorm_bwd(dy, x, gamma, mean, rstd, dx=dx2)
    assert_bits_equal("dx", dx2, dx)


@pytest.mark.parametrize("M,N,fp32", [(64 * 197, 768, False), (5000, 3072, True)])
def test_colsum_accum_is_bit_reproducible(M, N, fp32):
    from egovlp_b200 import ops
    dy = spread((M, N), 6, F32 if fp32 else BF16)
    base = spread((N,), 7)

    def run():
        out = base.clone()
        ops.colsum_accum(dy, out)
        return (out,)

    (out,) = three_times(run)
    d64 = dy.double()
    assert_sum_bound("colsum_accum", out, base.double() + d64.sum(0), base.double().abs() + d64.abs().sum(0))


# ---------------------------------------------------------------------------------------------------------- embeddings
def test_patch_embed_reduce_is_bit_reproducible():
    from egovlp_b200 import ops
    B, T, N, D = 2, 16, 196, 768
    S = 1 + T * N
    dx = spread((B, S, D), 8)
    bases = [spread(s, 9 + i) for i, s in enumerate([(D,), (1 + N, D), (T, D), (D,)])]

    def run():
        outs = [b.clone() for b in bases]
        ops.video_embed_bwd(dx, torch.empty(S * D, device="cuda"), *outs, B, T, N, D)
        return tuple(outs)

    got = three_times(run)
    tok = dx.double()[:, 1:].reshape(B, T, N, D)
    assert_sum_bound("dbias", got[3], bases[3].double() + tok.sum((0, 1, 2)),
                     bases[3].double().abs() + tok.abs().sum((0, 1, 2)))


def test_text_embedding_backward_with_repeated_ids_is_bit_reproducible():
    """64 x 32 tokens, most of them the padding id 0 (hundreds per batch), the rest from five ids."""
    from egovlp_b200 import ops
    B, L, D, V = 64, 32, 768, 120
    g = torch.Generator(device="cuda").manual_seed(11)
    ids = torch.tensor([0, 0, 0, 101, 102, 7, 7, 55], device="cuda")[torch.randint(0, 8, (B, L), generator=g,
                                                                                      device="cuda")]
    dsum = spread((B * L, D), 12)
    base_w, base_p = spread((V, D), 13), spread((L + 4, D), 14)

    def run():
        dword, dpos = base_w.clone(), base_p.clone()
        ops.text_embed_bwd(ids, dsum, dword, dpos, B, L, D)
        return dword, dpos

    dword, dpos = three_times(run)
    d64, flat = dsum.double(), ids.flatten()
    per = torch.zeros(V, D, device="cuda", dtype=F64).index_add_(0, flat, d64)
    per_abs = torch.zeros(V, D, device="cuda", dtype=F64).index_add_(0, flat, d64.abs())
    assert_sum_bound("dword", dword, base_w.double() + per, base_w.double().abs() + per_abs)
    assert_sum_bound("dpos", dpos[:L], base_p[:L].double() + d64.view(B, L, D).sum(0),
                     base_p[:L].double().abs() + d64.abs().view(B, L, D).sum(0))
    assert_bits_equal("dpos rows >= L", dpos[L:], base_p[L:])


# ---------------------------------------------------------------------------------------------------------- MaxMargin
@pytest.mark.parametrize("adaptive", [False, True])
@pytest.mark.parametrize("fix_norm", [True, False])
def test_maxmargin_is_bit_reproducible(adaptive, fix_norm):
    from loss_ref import maxmargin_case, maxmargin_reference
    from egovlp_b200 import ops
    G = 512
    x, w = maxmargin_case(G, 21, adaptive)
    x = (x * torch.exp2(torch.randint(-10, 10, (G, G), generator=torch.Generator().manual_seed(3)).float())).cuda()
    w = w.cuda() if w is not None else None
    gscale = torch.tensor([0.75], device="cuda")
    loss, dx = three_times(lambda: (ops.maxmargin_fwd(x, 0.25, fix_norm, w),
                                    ops.maxmargin_bwd(x, 0.25, fix_norm, gscale, w)))
    r = maxmargin_reference(x, 0.25, fix_norm, w, 0.75)
    assert abs(loss.double().item() - r["loss"].item()) <= r["loss_err"].item()
    assert bool(((dx.double() - r["dx"]).abs() <= r["dx_err"] + 1e-30).all())


# ---------------------------------------------------------------------------------------------------------- model step
VIDEO = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "pretrained": True, "time_init": "zeros"}
DISTILBERT = {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"}


def build_model(frames=16, img=224, low_memory=False, drops=True, bert=False, oscc=False):
    """oscc: the Ego4D OSCC fine-tuning model (2-wide projection head on the narrow-head kernels, video only)."""
    import warnings
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.model import FrozenInTime
    video = dict(VIDEO, num_frames=frames, img_size=img, grad_checkpointing=low_memory)
    if drops:
        video.update(drop_rate=0.1, drop_path_rate=0.1)
    text = dict(DISTILBERT, model="bert-base-uncased") if bert else DISTILBERT
    dims = syn.model_dims(num_frames=frames, img=img, **({"text_layers": 12, "text_kind": "bert"} if bert else {}),
                          **({"proj_dim": 2} if oscc else {}))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if oscc:
            net = FrozenInTime(video, text, projection_dim=2)
        else:
            net = FrozenInTime(video, text, projection="minimal", load_checkpoint="")
    net.load_state_dict(syn.seeded_state_dict(dims, seed=0), strict=False)
    return net.cuda().train()


def step_bits(net, B=2, frames=16, img=224, L=16, loss="egonce", seed=0):
    """One seeded training step from a copy of `net`'s state: (loss, {name: grad}, {name: updated weight})."""
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.loss import AdaptiveMaxMarginRankingLoss, EgoNCE
    from egovlp_b200.model.model import sim_matrix
    from egovlp_b200.optim import AdamW
    state = {k: v.clone() for k, v in net.state_dict().items()}
    data = {"video": syn.synthetic_video(B, frames, seed=1, img=img).cuda(),
            "text": {k: v.cuda() for k, v in syn.synthetic_text(B, L, seed=2, ragged=True).items()}}
    verb, noun = [t.cuda() for t in syn.synthetic_tags(B, seed=3)]
    torch.manual_seed(seed)                       # the dropout masks' seeds come from torch's generator
    opt = AdamW(net.parameters(), lr=1e-4, weight_decay=0.01)
    opt.zero_grad(set_to_none=True)
    if loss == "oscc":                            # trainer_oscc.py: CrossEntropy over the 2-wide head, video only
        from egovlp_b200.model.loss import CrossEntropy
        scores = net({"video": data["video"]}, video_only=True)
        t, v = scores, scores
        value = CrossEntropy()(scores, torch.arange(B, device="cuda") % 2)
    elif loss == "egonce":
        t, v = net(data)
        value = EgoNCE().fused(t, v, verb, noun)
    else:
        t, v = net(data)
        w = torch.linspace(0.5, 1.5, B, device="cuda")
        value = AdaptiveMaxMarginRankingLoss(margin=0.2)(sim_matrix(t, v), w)
    value.backward()
    grads = {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}
    opt.step()
    weights = {n: p.detach().clone() for n, p in net.named_parameters()}
    net.load_state_dict(state)
    return value.detach().clone(), grads, weights, (t.detach().clone(), v.detach().clone())


def assert_steps_equal(a, b, tag):
    assert_bits_equal(f"{tag} loss", b[0], a[0])
    assert a[1].keys() == b[1].keys()
    for n in a[1]:
        assert_bits_equal(f"{tag} grad {n}", b[1][n], a[1][n])
    for n in a[2]:
        assert_bits_equal(f"{tag} weight {n}", b[2][n], a[2][n])
    for e, f in zip(a[3], b[3]):
        assert_bits_equal(f"{tag} embeddings", f, e)


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


CASES = {"a": {}, "b": {"low_memory": True}, "c": {"frames": 3}, "d": {"img": 288, "frames": 4},
         "e": {"bert": True, "frames": 4, "L": 200}, "f": {"frames": 4, "loss": "adaptive_maxmargin"},
         "g": {"oscc": True, "drops": False, "B": 4, "loss": "oscc"}}


@pytest.mark.parametrize("case", sorted(CASES))
def test_training_step_is_bit_reproducible(case):
    kw = dict(CASES[case])
    step_kw = {k: kw.pop(k) for k in ("L", "loss", "B") if k in kw}
    net = build_model(**kw)
    frames, img = kw.get("frames", 16), kw.get("img", 224)
    with deterministic():
        runs = [step_bits(net, frames=frames, img=img, **step_kw) for _ in range(3)]
    assert len(runs[0][1]) >= 150 and all(bool(torch.isfinite(g).all()) for g in runs[0][1].values())
    if case == "g":                               # the video tower and the narrow head train, the text tower does not
        assert "vid_proj.0.weight" in runs[0][1] and not any(n.startswith("text_model.") for n in runs[0][1])
    if case == "a":
        assert len(runs[0][1]) == 327
    for r in runs[1:]:
        assert_steps_equal(runs[0], r, f"case {case}")
    if case == "a":
        # warn_only=True takes the same forms
        with deterministic(warn_only=True):
            assert_steps_equal(runs[0], step_bits(net), "warn_only")
        # the flag off: the default kernels agree within test_parity_fullsize_gpu.py's tolerances (embeddings rel-L2
        # 9e-3, loss 1e-3 relative, all 327 gradients together: cosine > 0.997, rel-L2 < 8.5e-2)
        off = step_bits(net)
        assert abs(off[0].item() - runs[0][0].item()) <= 1e-3 * abs(runs[0][0].item()), (off[0], runs[0][0])
        for e_off, e_det in zip(off[3], runs[0][3]):
            assert _rel(e_off, e_det) < 9e-3
        g_off = torch.cat([off[1][n].flatten() for n in sorted(off[1])]).double()
        g_det = torch.cat([runs[0][1][n].flatten() for n in sorted(off[1])]).double()
        cos = (g_off @ g_det / (g_off.norm() * g_det.norm())).item()
        assert cos > 0.997 and _rel(g_off, g_det) < 8.5e-2, (cos, _rel(g_off, g_det))
        # a fresh process computes the same bits
        path = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"egovlp_det_step_{os.getpid()}.pt")
        code = ("import sys, torch; sys.path[:0] = [%r, %r]; import test_deterministic_gpu as t; "
                "net = t.build_model(); torch.use_deterministic_algorithms(True); "
                "torch.save(t.step_bits(net), %r)" % (ROOT, os.path.join(ROOT, "tests"), path))
        subprocess.run([sys.executable, "-c", code], check=True, cwd=ROOT)
        try:
            assert_steps_equal(runs[0], torch.load(path), "fresh process")
        finally:
            os.remove(path)
