"""Training dropouts of the video tower (drop_rate, drop_path_rate; reference model/video_transformer.py:36-52, 135-136,
163-177, 244-251, 320-321), fused into the proj / fc1 / fc2 GEMM epilogues:
  * the epilogue forms apply exactly the masks and per-sample factors that ops.dropout_mask / ops.drop_path_factors
    materialise, on 256- and 128-column tiles, and drop_rows_bf16 (the backward's masked operand) does too;
  * one block against an fp32 port of the reference block whose Dropout / DropPath use those masks: forward output and
    every parameter and input gradient, at tiny dims and TimeSformer-B width, T = 4 and 16, a frame of 289 patches,
    default and low-memory modes; and the tiny tower the same way, pos_drop and the per-block sites included;
  * keep fractions within 6 sigma of the binomial at p = 0.1 and 0.5, whole-clip zeros only on the drop-path branches,
    different seeds give different masks, torch.manual_seed reproduces losses bit for bit (gradients to the
    run-to-run spread of the split-K atomics);
  * with all rates 0, and with any rates under eval(), outputs are those of a tower built without them bit for bit, and
    gradients to the run-to-run spread of the split-K atomics;
  * the low-memory rebuild of tr / sr equals the forward's bit for bit, and its gradients match the default mode's;
  * fp8 inference precision with the tower in train() and dropout on gives the bf16 forward bit for bit."""
from functools import partial

import pytest
import torch
import torch.nn.functional as F
from gemm_ref import check, check_all, reference
from kernel_checks import nan_filled
from torch import nn

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


@pytest.fixture(scope="module", autouse=True)
def fp32_matmul():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False            # the oracle runs in true fp32 on the GPU
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def cos(a, b):
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-300)).item()


def multiplier(d, B, S, width):
    """fp32 [B*S, width] multiplier of an ops.Drop: mask / (1 - p) times the sample's drop-path factor."""
    from egovlp_b200 import ops
    m = ops.dropout_mask(B * S, width, d.p, d.seed, d.site)
    if d.path_rows:
        m = m * ops.drop_path_factors(B, d.path_p, d.seed, d.path_site).repeat_interleave(S)[:, None]
    return m


def block_ref(x, p, heads, T, N, mult, eps=1e-6):
    """fp32 SpaceTimeBlock.forward of the reference (:163-177) with its Dropout / DropPath replaced by the multipliers
    `mult` (time proj, space proj, GELU output, fc2 output; None = identity)."""
    from oracle import reference_port as rp
    B, S, D = x.shape

    def ln(t, name):
        return F.layer_norm(t, (D,), p[name + ".weight"], p[name + ".bias"], eps)

    def lin(t, name):
        return t @ p[name + ".weight"].t() + p[name + ".bias"]

    def att(t, pre, mode):
        return lin(rp.divided_attention_core(lin(t, pre + "qkv"), heads, T, N, mode), pre + "proj")

    def drop(t, m):
        return t if m is None else t * m.view(B, S, -1)

    mt, ms, mg, mf = mult
    tr = x + drop(att(ln(x, "norm3"), "timeattn.", "time"), mt)
    sr = x + drop(att(ln(tr, "norm1"), "attn.", "space"), ms)          # from the block input, as the reference
    h = drop(F.gelu(lin(ln(sr, "norm2"), "mlp.fc1")), mg)
    return sr + drop(lin(h, "mlp.fc2"), mf)


def make_block(D, H, drop, path, seed=0):
    from egovlp_b200.model.video_transformer import SpaceTimeBlock
    torch.manual_seed(seed)
    blk = SpaceTimeBlock(D, H, qkv_bias=True, drop=drop, drop_path=path,
                         norm_layer=partial(nn.LayerNorm, eps=1e-6), time_init="rand")
    with torch.no_grad():                       # non-trivial LayerNorm affines and biases
        for name, prm in blk.named_parameters():
            if prm.dim() == 1:
                prm.add_(0.05 * torch.randn_like(prm))
    return blk.cuda().train()


# ------------------------------------------------------------------------------------------------ epilogue forms
@pytest.mark.parametrize("N", [256, 384])                 # 256- and 128-column tiles
def test_gemm_dropout_forms_apply_the_materialised_masks(N):
    from egovlp_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    M, K, B = 1000, 128, 8                                 # 8 samples of 125 rows; M is not a tile multiple
    a = torch.randn(M, K, device="cuda", generator=g).to(BF16)
    w = (0.1 * torch.randn(N, K, device="cuda", generator=g)).to(BF16)
    bias = 0.1 * torch.randn(N, device="cuda", generator=g)
    resid = torch.randn(M, N, device="cuda", generator=g)
    d = ops.Drop(0.3, 1234, 7, 0.5, 8, M // B)
    m = multiplier(d, B, M // B, N)
    assert (m.view(B, -1) == 0).all(1).any() and not (m.view(B, -1) == 0).all(1).all()

    # proj / fc2 forward: resid + m (a w^T + b); the plain form gives the product
    plain = ops.gemm(a, w, torch.empty(M, N, device="cuda"), bias=bias, residual=torch.zeros_like(resid))
    got = ops.gemm(a, w, nan_filled((M, N), torch.float32), bias=bias, residual=resid, drop=d)
    sel = plain.abs() > 1e-3                                # where the product cannot vanish into the residual's rounding
    assert torch.equal((got == resid)[sel], (m == 0)[sel])
    assert rel(got - resid, plain * m) < 1e-6
    check(f"dropout residual fp32 N={N}", got, reference(a, w, bias=bias, residual=resid, mult=m)["out"])

    # fc1 forward, both training forms: h = m GELU(v); the second output is unmasked
    e = ops.Drop(0.3, 1234, 9)
    me = multiplier(e, B, M // B, N)
    h0, u0 = torch.empty(M, N, device="cuda", dtype=BF16), torch.empty(M, N, device="cuda", dtype=BF16)
    ops.gemm(a, w, h0, bias=bias, act=3, out2=u0)
    for act in (3, 1):
        h, u = nan_filled((M, N), BF16), nan_filled((M, N), BF16)
        ops.gemm(a, w, h, bias=bias, act=act, out2=u, drop=e)
        if act == 3:
            assert torch.equal(u, u0)
        assert torch.equal(h == 0, (me == 0) | (h0 == 0)) and rel(h, h0.float() * me) < 5e-3
        check_all(f"dropout act {act} N={N}", {"out": h, "out2": u},
                  reference(a, w, bias=bias, act=act, out2=True, mult=me))

    # fc2 input gradient with W2 as MN-major B: du = (dy W2) aux m;  low memory: du and h = m GELU(z)
    dy = torch.randn(M, K, device="cuda", generator=g).to(BF16)
    w2 = (0.1 * torch.randn(K, N, device="cuda", generator=g)).to(BF16)
    aux = torch.randn(M, N, device="cuda", generator=g).to(BF16)
    du0 = ops.gemm(dy, w2, torch.empty(M, N, device="cuda", dtype=BF16), b_mn=True, aux=aux, act=4)
    du = ops.gemm(dy, w2, nan_filled((M, N), BF16), b_mn=True, aux=aux, act=4, drop=e)
    assert torch.equal(du == 0, (me == 0) | (du0 == 0)) and rel(du, du0.float() * me) < 5e-3
    check(f"dropout act 4 N={N}", du, reference(dy, w2, b_mn=True, aux=aux, act=4, mult=me)["out"])
    du0, hz0 = torch.empty_like(du), torch.empty_like(du)
    ops.gemm(dy, w2, du0, b_mn=True, aux=aux, act=5, out2=hz0)
    du, hz = nan_filled((M, N), BF16), nan_filled((M, N), BF16)
    ops.gemm(dy, w2, du, b_mn=True, aux=aux, act=5, out2=hz, drop=e)
    assert torch.equal(hz == 0, (me == 0) | (hz0 == 0)) and rel(hz, hz0.float() * me) < 5e-3
    assert torch.equal(du == 0, (me == 0) | (du0 == 0)) and rel(du, du0.float() * me) < 5e-3
    check_all(f"dropout act 5 N={N}", {"out": du, "out2": hz},
              reference(dy, w2, b_mn=True, aux=aux, act=5, out2=True, mult=me))

    # the backward's masked operand, from fp32 and from bf16
    x32 = torch.randn(M, N, device="cuda", generator=g)
    assert torch.equal(ops.drop_rows_bf16(x32, d), (x32 * m).to(BF16))
    x16 = x32.to(BF16)
    assert torch.equal(ops.drop_rows_bf16(x16, d), (x16.float() * m).to(BF16))

    # a descriptor no dropout form takes is refused rather than run without the mask
    with pytest.raises(Exception, match="dropout"):
        ops.gemm(a, w, torch.empty(M, N, device="cuda", dtype=BF16), bias=bias, drop=e)


# ------------------------------------------------------------------------------------------------ one block vs the oracle
CASES = [  # D, H, B, T, N, low_memory
    pytest.param(128, 2, 3, 4, 16, False, id="tiny-T4"),
    pytest.param(128, 2, 3, 4, 16, True, id="tiny-T4-lowmem"),
    pytest.param(128, 2, 2, 16, 9, False, id="tiny-T16"),
    pytest.param(128, 2, 2, 16, 9, True, id="tiny-T16-lowmem"),
    pytest.param(128, 2, 2, 2, 289, False, id="large-frame-N289"),
    pytest.param(128, 2, 2, 2, 289, True, id="large-frame-N289-lowmem"),
    pytest.param(768, 12, 2, 4, 196, False, id="timesformer-b-T4"),
    pytest.param(768, 12, 2, 16, 196, True, id="timesformer-b-T16-lowmem"),
]


@pytest.mark.parametrize("D,H,B,T,N,low", CASES)
def test_block_with_dropout_vs_oracle_fed_with_the_masks(D, H, B, T, N, low):
    from egovlp_b200 import engine
    S = 1 + T * N
    blk = make_block(D, H, drop=0.1, path=0.4)
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(B, S, D, device="cuda", generator=g)
    probe = torch.randn(B, S, D, device="cuda", generator=g)
    seed, index = 987654321, 5
    xi = x.clone().requires_grad_(True)
    y = blk(xi, time_n=N, space_f=T, low_memory=low, drop_seed=seed, block_index=index)
    (y * probe).sum().backward()

    drops = engine.VideoBlockDrop(seed, index, *blk.dropout_rates()).sites(S)
    widths = (D, D, blk.mlp.fc1.out_features, D)
    mult = [multiplier(d, B, S, w) for d, w in zip(drops, widths)]
    p = {k: v.detach().clone().requires_grad_(True) for k, v in blk.named_parameters()}
    xr = x.clone().requires_grad_(True)
    want = block_ref(xr, p, H, T, N, mult)
    (want * probe).sum().backward()
    plain = block_ref(x, {k: v.detach() for k, v in p.items()}, H, T, N, (None,) * 4)
    assert rel(y, want) < 1e-2, rel(y, want)
    assert rel(plain, want) > 3 * rel(y, want)             # the dropout is active and it is what the oracle applies
    worst = min((cos(prm.grad, p[k].grad), k) for k, prm in blk.named_parameters())
    flat_g = torch.cat([prm.grad.flatten() for _, prm in blk.named_parameters()] + [xi.grad.flatten()])
    flat_r = torch.cat([p[k].grad.flatten() for k, _ in blk.named_parameters()] + [xr.grad.flatten()])
    print(f"\n[dropout block D={D} T={T} N={N} low={low}] out rel {rel(y, want):.2e}, input grad cos "
          f"{cos(xi.grad, xr.grad):.6f}, worst parameter grad cos {worst[0]:.6f} ({worst[1]}), all rel "
          f"{rel(flat_g, flat_r):.2e}")
    assert cos(xi.grad, xr.grad) > 0.999
    assert worst[0] > 0.993, worst
    assert cos(flat_g, flat_r) > 0.997 and rel(flat_g, flat_r) < 8.5e-2


# ------------------------------------------------------------------------------------------------ mask statistics
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_fraction_and_whole_clip_zeros(p):
    from egovlp_b200 import engine, ops
    B, S, W = 64, 1 + 8 * 196, 256
    n = B * S * W
    drops = engine.VideoBlockDrop(42, 3, p, p, p, p).sites(S)
    for which, d in zip(("time", "space", "gelu", "fc2"), drops):
        m = multiplier(d, B, S, W)
        per_clip = (m.view(B, -1) != 0).float().mean(1)
        zero_clips = int((per_clip == 0).sum())
        if d.path_rows:                                      # drop-path branches: whole clips drop with rate p
            assert zero_clips > 0 and abs(zero_clips - p * B) < 6 * (B * p * (1 - p)) ** 0.5, (which, zero_clips)
            kept = m.view(B, -1)[per_clip > 0]
        else:
            assert zero_clips == 0, which
            kept = m
        frac = (kept != 0).float().mean().item()
        sigma = (p * (1 - p) / kept.numel()) ** 0.5
        assert abs(frac - (1 - p)) < 6 * sigma, (which, frac)
    a = ops.dropout_mask(1000, W, p, 42, 2)
    assert not torch.equal(a, ops.dropout_mask(1000, W, p, 43, 2)) and not torch.equal(a, ops.dropout_mask(1000, W, p, 42, 3))


def tiny_tower(**rates):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.video_transformer import SpaceTimeTransformer
    net = SpaceTimeTransformer(img_size=32, patch_size=16, embed_dim=128, depth=2, num_heads=2, num_frames=4,
                               time_init="rand", num_classes=0, **rates)     # block 1 has drop-path (block 0 never)
    sd = syn.seeded_state_dict(syn.TINY_DIMS, seed=7, text=False, proj=False)
    net.load_state_dict({k[len("video_model."):]: v for k, v in sd.items()})
    return net.cuda()


def run_tower(net, video, seed=None, low=False):
    if seed is not None:
        torch.manual_seed(seed)
    net.set_grad_checkpointing(low)
    net.zero_grad(set_to_none=True)
    f = net(video)
    loss = (f * torch.linspace(-1, 1, f.numel(), device="cuda").view_as(f)).sum()
    loss.backward()
    return loss.detach(), f.detach(), {k: p.grad.clone() for k, p in net.named_parameters()}


def video_input(B=4):
    from egovlp_b200 import synthetic as syn
    return syn.synthetic_video(B, 4, seed=1, img=32).cuda()


# The split-K weight gradients and the fused bias sums add fp32 partials with atomics, in no fixed order, so two runs of
# the same step differ in the last bits of those gradients with or without dropout: gradients are compared to that
# spread, outputs and losses bit for bit.
GRAD_SPREAD = 1e-5


def assert_grads_match(g, ref, what):
    worst = max((rel(g[k], ref[k]), k) for k in ref)
    assert worst[0] < GRAD_SPREAD, (what, worst)


def test_manual_seed_reproduces_and_seeds_differ():
    video = video_input()
    net = tiny_tower(drop_rate=0.2, drop_path_rate=0.3).train()
    l1, f1, g1 = run_tower(net, video, seed=11)
    l2, f2, g2 = run_tower(net, video, seed=11)
    l3, f3, g3 = run_tower(net, video, seed=12)
    assert torch.equal(l1, l2) and torch.equal(f1, f2)
    assert_grads_match(g2, g1, "same seed")
    assert not torch.equal(f1, f3) and max(rel(g3[k], g1[k]) for k in g1) > 1e-2


def test_rates_zero_and_eval_are_the_plain_tower_bit_for_bit():
    video = video_input()
    base = tiny_tower().train()
    lb, fb, gb = run_tower(base, video, seed=3)
    _, _, gb2 = run_tower(base, video, seed=3)
    assert_grads_match(gb2, gb, "plain tower run to run")
    for net in (tiny_tower(drop_rate=0., attn_drop_rate=0., drop_path_rate=0.).train(),
                tiny_tower(drop_rate=0.3, attn_drop_rate=0.2, drop_path_rate=0.5).eval()):
        for low in (False, True):
            l, f, g = run_tower(net, video, seed=3, low=low)
            lb_, fb_, gb_ = run_tower(base, video, seed=3, low=low)
            assert torch.equal(f, fb_) and torch.equal(l, lb_), low
            assert_grads_match(g, gb_, ("rates 0 / eval", low))
    net = tiny_tower(drop_rate=0.3, drop_path_rate=0.5).train()
    with torch.no_grad():                                  # train() drops under no_grad, eval() does not
        torch.manual_seed(5)
        assert not torch.equal(net(video), fb)
        assert torch.equal(net.eval()(video), base.eval()(video))


@pytest.mark.parametrize("low", [False, True], ids=["default", "lowmem"])
def test_tower_with_dropout_vs_oracle_fed_with_the_masks(low):
    """The whole tiny tower in training: pos_drop at site 0 on the embedded tokens, every block at its own sites under
    the one seed the forward drew (replayed from torch.manual_seed), against the reference port fed with those masks:
    the CLS feature and every gradient, the embeddings' and the patch projection's included."""
    from egovlp_b200 import engine, ops
    from oracle import reference_port as rp
    video = video_input()
    net = tiny_tower(drop_rate=0.2, drop_path_rate=0.4).train()
    probe = torch.linspace(-1, 1, 4 * 128, device="cuda").view(4, 128)
    net.set_grad_checkpointing(low)
    net.zero_grad(set_to_none=True)
    torch.manual_seed(21)
    f = net(video)
    (f * probe).sum().backward()
    torch.manual_seed(21)
    seed = engine.draw_dropout_seed()                       # the seed that forward drew

    p = {k: v.detach().clone().requires_grad_(True) for k, v in net.named_parameters()}
    x, T, N = rp.video_tokens(video, p, prefix="")
    B, S, D = x.shape
    pos = ops.dropout_mask(B * S, D, net.pos_drop.p, seed, engine.VIDEO_SITE_POS).view(B, S, D)
    x = x * pos
    for i, blk in enumerate(net.blocks):
        drops = engine.VideoBlockDrop(seed, i, *blk.dropout_rates()).sites(S)
        mult = [None if d is None else multiplier(d, B, S, w)
                for d, w in zip(drops, (D, D, blk.mlp.fc1.out_features, D))]
        pb = {k[len(f"blocks.{i}."):]: v for k, v in p.items() if k.startswith(f"blocks.{i}.")}
        x = block_ref(x, pb, blk.num_heads, T, N, mult)
    want = F.layer_norm(x, (D,), p["norm.weight"], p["norm.bias"], net.norm.eps)[:, 0]
    (want * probe).sum().backward()
    net.set_grad_checkpointing(False)

    assert rel(f, want) < 1e-2, rel(f, want)
    worst = min((cos(prm.grad, p[k].grad), k) for k, prm in net.named_parameters())
    flat_g = torch.cat([prm.grad.flatten() for _, prm in net.named_parameters()])
    flat_r = torch.cat([p[k].grad.flatten() for k, _ in net.named_parameters()])
    print(f"\n[dropout tower low={low}] feature rel {rel(f, want):.2e}, worst gradient cos {worst[0]:.6f} "
          f"({worst[1]}), all rel {rel(flat_g, flat_r):.2e}")
    assert worst[0] > 0.993, worst
    assert cos(flat_g, flat_r) > 0.997 and rel(flat_g, flat_r) < 8.5e-2
    for k in ("cls_token", "pos_embed", "temporal_embed", "patch_embed.proj.weight", "patch_embed.proj.bias"):
        assert rel(dict(net.named_parameters())[k].grad, p[k].grad) < 2e-2, k


# ------------------------------------------------------------------------------------------------ modes
def test_lowmem_rebuild_with_dropout_is_bit_identical_and_gradients_match():
    from egovlp_b200 import engine
    blk = make_block(768, 12, drop=0.1, path=0.3)
    B, T, N = 2, 16, 196
    S = 1 + T * N
    x = torch.randn(B, S, 768, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    outs, grads = [], []
    for low in (False, True):
        blk.zero_grad(set_to_none=True)
        xi = x.clone().requires_grad_(True)
        y = blk(xi, time_n=N, space_f=T, low_memory=low, drop_seed=77, block_index=2)
        outs.append((y, y.grad_fn))
        (y * x).sum().backward(retain_graph=True)
        grads.append({k: p.grad.clone() for k, p in blk.named_parameters()} | {"x": xi.grad.clone()})
    (y0, f0), (y1, f1) = outs
    assert torch.equal(y0, y1)
    s0, s1 = f0.saved_tensors, f1.saved_tensors
    sr, n2 = engine.SpaceTimeBlockFn.rebuild("sr", s1, f1.eps, f1.cache, f1.drops)
    tr, n1 = engine.SpaceTimeBlockFn.rebuild("tr", s1, f1.eps, f1.cache, f1.drops)
    for name, got, i in (("tr", tr, 7), ("n1", n1, 8), ("sr", sr, 14), ("n2", n2, 15)):
        assert torch.equal(got, s0[i]), name
    assert not torch.equal(engine.SpaceTimeBlockFn.rebuild("sr", s1, f1.eps, f1.cache)[0], sr)   # the mask mattered
    worst = min((cos(grads[1][k], grads[0][k]), k) for k in grads[0])
    assert worst[0] > 0.9995, worst


@pytest.mark.parametrize("rates", [dict(drop_rate=0.2, drop_path_rate=0.3), dict(drop_path_rate=0.3)],
                         ids=["dropout-and-drop-path", "drop-path-only"])
def test_fp8_in_train_with_dropout_runs_the_bf16_forward(rates):
    """Every block runs bf16, block 0 of a drop-path-only tower (which has nothing to drop) included."""
    video = video_input()
    net = tiny_tower(**rates).train()
    with torch.no_grad():
        torch.manual_seed(9)
        ref = net(video)
        net.set_inference_precision("fp8")
        torch.manual_seed(9)
        got = net(video)
    assert torch.equal(got, ref)
