"""The video tower on frames of more than 255 patches (256 to 512 px at patch 16), end to end on the GPU: the patch
embedding against fp64, the tiny tower against the unmodified reference (tests/golden/video_large_grid.npz), the
full-size TimeSformer-B step against the fp32 oracle (with the low-memory mode and fp8 inference at 384 px), and a
FrozenInTime with `img_size = 384` restored from a 224-px checkpoint, trained one step, saved and resumed.

Tolerances are the existing ones: PatchEmbedFn those of test_front_end_kernels_gpu.py, the tiny tower those of
test_model_gpu.py::test_video_tower_tiny_vs_reference_golden, the full-size step those of test_parity_fullsize_gpu.py,
fp8 those of test_fp8_inference_gpu.py and the low-memory mode those of test_activation_memory_gpu.py."""
import json
import warnings

import pytest
import torch
from kernel_checks import BF16, F32, assert_sum_bound, mk, rel_l2

from conftest import load_golden

pytestmark = pytest.mark.gpu
warnings.simplefilter("ignore")

VIDEO = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "pretrained": True, "time_init": "zeros"}
TEXT = {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"}
EMB_TOL, LOSS_TOL = 9e-3, 1e-3


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def cos(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-300)).item()


# ------------------------------------------------------------------------------------------------ patch embedding
@pytest.mark.parametrize("H,W", [(256, 256), (384, 384), (512, 512), (256, 320)])
def test_patch_embed_fn_at_large_frames(H, W):
    """engine.PatchEmbedFn forward and backward against oracle.reference_port.video_tokens in fp64 (the reference gets
    the bf16-rounded video and conv weight the GEMM reads), with the bounds of test_front_end_kernels_gpu.py."""
    from egovlp_b200 import engine
    from oracle import reference_port as rp
    B, T, F, C, D, P = 2, 3, 4, 3, 256, 16
    N = (H // P) * (W // P)
    S = 1 + T * N
    video = mk((B, T, C, H, W), 40, dtype=F32)
    init = {"cls_token": mk((1, 1, D), 41, dtype=F32), "pos_embed": mk((1, 1 + N, D), 42, dtype=F32),
            "temporal_embed": mk((1, F, D), 43, dtype=F32), "patch_embed.proj.weight": mk((D, C, P, P), 44, 0.05, F32),
            "patch_embed.proj.bias": mk((D,), 45, dtype=F32)}
    p = {k: v.clone().requires_grad_(True) for k, v in init.items()}
    x = engine.PatchEmbedFn.apply(video, p["cls_token"], p["pos_embed"], p["temporal_embed"],
                                  p["patch_embed.proj.weight"], p["patch_embed.proj.bias"], engine.Bf16Cache())
    g = mk((B, S, D), 46, dtype=F32)
    x.backward(g)
    p64 = {"video_model." + k: (v.to(BF16) if k == "patch_embed.proj.weight" else v).double().requires_grad_(True)
           for k, v in init.items()}
    tok, _, n = rp.video_tokens(video.to(BF16).double(), p64)
    assert n == N
    err = rel_l2(x.detach(), tok.detach())
    print(f"[bound] PatchEmbedFn tokens {H}x{W}: rel-L2 {err:.3g} (bound 2e-5)")
    assert err < 2e-5
    names = ["cls_token", "pos_embed", "temporal_embed", "patch_embed.proj.bias"]
    leaves = [p64["video_model." + k] for k in names]
    ref = torch.autograd.grad(tok, leaves, g.double(), retain_graph=True)
    terms = torch.autograd.grad(tok, leaves, g.double().abs(), retain_graph=True)
    for k, r, t in zip(names, ref, terms):
        assert_sum_bound(f"PatchEmbedFn d{k} {H}x{W}", p[k].grad, r, t)
    (rw,) = torch.autograd.grad(tok, [p64["video_model.patch_embed.proj.weight"]], g.to(BF16).double())
    err = rel_l2(p["patch_embed.proj.weight"].grad, rw)
    print(f"[bound] PatchEmbedFn dconv_weight {H}x{W}: rel-L2 {err:.3g} (bound 2e-5)")
    assert err < 2e-5


# ------------------------------------------------------------------------------------------------ tiny tower vs golden
@pytest.mark.parametrize("tag", ["n256", "n320"])
def test_tiny_tower_vs_reference_golden(tag):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.video_transformer import SpaceTimeTransformer
    g = load_golden("video_large_grid.npz")
    B, T, seed = int(g["B"]), int(g["T"]), int(g["seed"])
    img = tuple(int(v) for v in g[f"{tag}:img"])
    dims = syn.model_dims(embed_dim=128, depth=2, heads=2, patch=16, img=img, num_frames=4, proj_dim=32)
    sd = syn.seeded_state_dict(dims, seed=seed, text=False, proj=False)
    net = SpaceTimeTransformer(img_size=img, patch_size=16, embed_dim=128, depth=2, num_heads=2, num_frames=4,
                               time_init="zeros", num_classes=0)
    net.load_state_dict({k[len("video_model."):]: v for k, v in sd.items()}, strict=True)
    net.cuda()
    video = syn.synthetic_video(B, T, seed=seed, img=img).cuda()
    with torch.no_grad():
        tok = net.forward_tokens(video).reshape(-1, 128)[g[f"{tag}:token_rows"].cuda()]
    out = net(video)
    e_out, e_tok = rel(out, g[f"{tag}:out"]), rel(tok, g[f"{tag}:tokens"])
    (out * g[f"{tag}:probe"].cuda()).sum().backward()
    params = dict(net.named_parameters())
    worst = []
    for k, ref in g.items():
        if k.startswith(f"{tag}:g:"):
            name = k[len(f"{tag}:g:video_model."):]
            grad = params[name].grad
            got = grad.flatten()[g[f"{tag}:gi:video_model.{name}"].cuda()]
            nrm = abs(grad.norm().item() / g[f"{tag}:n:video_model.{name}"].item() - 1)
            worst.append((cos(got, ref), rel(got, ref), nrm, name))
    print(f"\n[tiny {tag}] out rel {e_out:.2e} tokens rel {e_tok:.2e} worst grad", min(worst), max(w[1] for w in worst))
    assert e_out < 1e-2 and e_tok < 1e-2, (e_out, e_tok)
    assert len(worst) == len(sd)
    for c, r, nrm, name in worst:
        assert c > 0.999 and r < 3e-2 and nrm < 3e-2, (name, c, r, nrm)


# ------------------------------------------------------------------------------------------------ full size vs oracle
def _full(img, num_frames=16, seed=0):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.model import FrozenInTime
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = syn.seeded_state_dict(syn.model_dims(img=img, num_frames=num_frames), seed=seed)
    net = FrozenInTime(dict(VIDEO, num_frames=num_frames, img_size=img), dict(TEXT))
    net.load_state_dict(sd, strict=True)
    net.text_model.config.dropout = net.text_model.config.attention_dropout = 0.0
    return net.cuda(), {k: v.cuda() for k, v in sd.items()}


def _batch(B, T, img, seed):
    from egovlp_b200 import synthetic as syn
    data = {"video": syn.synthetic_video(B, T, seed=seed, img=img).cuda(),
            "text": {k: v.cuda() for k, v in syn.synthetic_text(B, 16, seed=seed, ragged=True).items()}}
    verb, noun = [t.cuda() for t in syn.synthetic_tags(B, seed=seed)]
    return data, verb, noun


def _step(net, data, verb, noun):
    from egovlp_b200.model.loss import EgoNCE
    net.zero_grad(set_to_none=True)
    t, v = net(data)
    loss = EgoNCE().fused(t, v, verb, noun)
    loss.backward()
    return t.detach(), v.detach(), loss.item(), {k: w.grad.detach().clone() for k, w in net.named_parameters()
                                                   if w.grad is not None}


def _grad_stats(grads, ref):
    rows = [(k, cos(g, ref[k]), ref[k].numel()) for k, g in grads.items()
            if ref.get(k) is not None and ref[k].norm().item() > 1e-12 and not k.endswith("k_lin.bias")]
    keys = [k for k, _, _ in rows]
    flat_g = torch.cat([grads[k].double().flatten() for k in keys])
    flat_r = torch.cat([ref[k].double().flatten() for k in keys])
    mats = [r for r in rows if r[2] > 4096]
    return cos(flat_g, flat_r), min(mats, key=lambda r: r[1]), len(rows)


@pytest.mark.parametrize("img,T", [(384, 8), (256, 16)])
def test_full_size_step_vs_fp32_oracle(img, T):
    """TimeSformer-B + DistilBERT + EgoNCE, B = 8 (the batch test_parity_fullsize_gpu.py's bounds were set at): embeddings, loss and the gradients of every tensor against the fp32
    oracle on the GPU.  At 384 px also the low-memory mode (same forward, gradients within the same bounds and close
    to the default's) and fp8 inference (video embeddings within test_fp8_inference_gpu.py's 8e-2)."""
    from oracle import reference_port as rp
    net, params = _full(img)
    B = 8
    data, verb, noun = _batch(B, T, img, seed=60 + T)
    t, v, loss, grads = _step(net, data, verb, noun)
    p = {k: w.clone().requires_grad_(True) for k, w in params.items()}
    tr, vr = rp.frozen_in_time_forward(data, p)
    lr = rp.egonce_loss(rp.sim_matrix(tr, vr), rp.sim_matrix(verb, verb), rp.sim_matrix(noun, noun))
    lr.backward()
    ref = {k: w.grad for k, w in p.items()}
    e_t, e_v, e_l = rel(t, tr), rel(v, vr), abs(loss - lr.item()) / abs(lr.item())
    cos_all, worst_m, n = _grad_stats(grads, ref)
    res = {"img": img, "T": T, "rel_text": e_t, "rel_video": e_v, "rel_loss": e_l, "grad_cos_all": cos_all,
           "worst_matrix": worst_m[:2], "n_tensors": n}
    if img == 384:
        net.video_model.set_grad_checkpointing(True)
        t2, v2, loss2, grads2 = _step(net, data, verb, noun)
        net.video_model.set_grad_checkpointing(False)
        cos_all2, worst_m2, _ = _grad_stats(grads2, ref)
        vs_def = min(cos(grads2[k], grads[k]) for k in grads if grads[k].numel() > 4096)
        res.update(lowmem_forward_equal=bool(torch.equal(v2, v) and loss2 == loss), lowmem_grad_cos_all=cos_all2,
                   lowmem_worst_matrix=worst_m2[:2], lowmem_vs_default=vs_def)
        with torch.no_grad():
            net.video_model.set_inference_precision("fp8")
            v8 = net.compute_video(data["video"])
            net.video_model.set_inference_precision("bf16")
        res["fp8_rel_video"] = rel(v8, vr)
    print("\n[large grid full size]", json.dumps(res))
    assert n >= 318, n
    assert e_t < EMB_TOL and e_v < EMB_TOL and e_l < LOSS_TOL, res
    assert cos_all > 0.997 and worst_m[1] > 0.993, res
    if img == 384:
        assert res["lowmem_forward_equal"], res
        assert cos_all2 > 0.997 and worst_m2[1] > 0.993 and vs_def > 0.998, res
        assert res["fp8_rel_video"] < 8e-2, res


# ------------------------------------------------------------------------------------------------ FrozenInTime at 384
def test_frozen_in_time_384_from_a_224_checkpoint_trains_saves_and_resumes(tmp_path):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.loss import EgoNCE
    from egovlp_b200.model.model import FrozenInTime, resample_pos_embed
    from oracle import reference_port as rp
    sd224 = syn.seeded_state_dict(syn.model_dims(num_frames=4), seed=2)
    path = tmp_path / "trainer224.pth"
    torch.save({"state_dict": {"module." + k: v for k, v in sd224.items()}}, path)
    net = FrozenInTime(dict(VIDEO, num_frames=4, img_size=384), dict(TEXT), load_checkpoint=str(path))
    net.text_model.config.dropout = net.text_model.config.attention_dropout = 0.0
    net.cuda()
    pe = net.video_model.pos_embed.detach().cpu()
    assert pe.shape == (1, 577, 768)
    # resampled where the checkpoint was loaded to (the current CUDA device)
    want = resample_pos_embed(sd224["video_model.pos_embed"].cuda(), (24, 24)).cpu()
    torch.testing.assert_close(pe, want, rtol=0, atol=0)
    data, verb, noun = _batch(2, 4, 384, seed=70)
    params = {k: v.detach().clone() for k, v in net.state_dict().items()}
    t, v = net(data)
    loss = EgoNCE().fused(t, v, verb, noun)
    with torch.no_grad():
        tr, vr = rp.frozen_in_time_forward(data, params)
        lr = rp.egonce_loss(rp.sim_matrix(tr, vr), rp.sim_matrix(verb, verb), rp.sim_matrix(noun, noun))
    e_l = abs(loss.item() - lr.item()) / abs(lr.item())
    print(f"\n[FrozenInTime 384] loss {loss.item():.6f} oracle {lr.item():.6f} rel {e_l:.2e}")
    assert e_l < LOSS_TOL
    opt = torch.optim.AdamW(net.parameters(), lr=1e-4)
    loss.backward()
    opt.step()
    ckpt = tmp_path / "trainer384.pth"
    torch.save({"state_dict": net.state_dict()}, ckpt)
    again = FrozenInTime(dict(VIDEO, num_frames=4, img_size=384), dict(TEXT), load_checkpoint=str(ckpt))
    again.text_model.config.dropout = again.text_model.config.attention_dropout = 0.0
    again.cuda()
    sd, sd2 = net.state_dict(), again.state_dict()
    assert list(sd) == list(sd2) and all(torch.equal(sd[k], sd2[k]) for k in sd)
    with torch.no_grad():
        assert torch.equal(net.compute_video(data["video"]), again.compute_video(data["video"]))
