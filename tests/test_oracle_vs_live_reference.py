"""The oracle against the UNMODIFIED reference on seeded random geometries.  What the reference's own modules computed for
each case is stored in tests/golden/live_reference.npz (written by oracle/make_live_golden.py, which runs them through
oracle/ref_shim.py); this file recomputes every case with the oracle's restatement and compares, fp32 vs fp32,
rounding-level tolerances.  tests/test_oracle_golden.py pins the oracle on further recorded vectors."""
import json
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch

from oracle import reference_port as rp
from egovlp_b200 import synthetic as syn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live_reference.npz")


@pytest.fixture(scope="module")
def ref():
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def meta(ref):
    return json.loads(str(ref["meta"]))


def t(a):
    return torch.from_numpy(np.asarray(a))


def close(a, b, rtol=1e-4, atol=1e-5):
    b = t(b) if not torch.is_tensor(b) else b
    torch.testing.assert_close(a.float(), b.float(), rtol=rtol, atol=atol)


@pytest.mark.parametrize("seed,frames_model,frames_in,img,heads,depth", [
    (1, 4, 4, 32, 2, 1), (2, 8, 5, 32, 2, 2), (3, 4, 1, 48, 2, 1), (4, 16, 16, 32, 2, 1), (5, 4, 2, 64, 2, 1)])
def test_video_tower_random_geometries(ref, meta, seed, frames_model, frames_in, img, heads, depth):
    """SpaceTimeTransformer.forward (model/video_transformer.py:302-338) incl. T < num_frames, 1-frame input, several
    patch grids, non-zero timeattn weights; outputs and gradients of every parameter (a fixed sample of each gradient's
    entries).  (heads >= 2 throughout: with one head the reference's in-place `q *= self.scale` (:106) hits a view and
    raises under autograd -- SURVEY.md quirk 4.)"""
    key = f"video/{seed}"
    dim = 64 * heads
    dims = syn.model_dims(embed_dim=dim, depth=depth, heads=heads, patch=16, img=img, num_frames=frames_model)
    sd = syn.seeded_state_dict(dims, seed=seed, text=False, proj=False)
    video = syn.synthetic_video(2, frames_in, seed=seed, img=img)
    want = t(ref[key + "/out"])
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    got = rp.video_tower(video, p, heads=heads)
    close(got, want)
    probe = torch.randn(want.shape, generator=torch.Generator().manual_seed(seed))
    (got * probe).sum().backward()
    checked = 0
    for n in meta[key]:
        g = p["video_model." + n].grad
        assert g is not None, n
        close(g.flatten()[t(ref[f"{key}/grad_idx/{n}"])], ref[f"{key}/grad/{n}"], rtol=5e-4, atol=5e-5)
        checked += 1
    assert checked >= 20


@pytest.mark.parametrize("seed,B,L", [(1, 3, 7), (2, 1, 1), (3, 4, 12)])
def test_distilbert_random_ragged(ref, seed, B, L):
    d = syn.TINY_DIMS
    sd = syn.seeded_state_dict(d, seed=seed, video=False, proj=False)
    text = syn.synthetic_text(B, L, seed=seed, ragged=True, vocab=d["vocab"])
    close(rp.distilbert_forward(text["input_ids"], text["attention_mask"], sd, heads=d["text_heads"]), ref[f"text/{seed}"])


@pytest.mark.parametrize("seed,G", [(1, 2), (2, 9), (3, 33)])
def test_losses_random(ref, seed, G):
    key = f"loss/{seed}"
    g = torch.Generator().manual_seed(seed)
    a, b = torch.randn(G, 24, generator=g), torch.randn(G, 24, generator=g)
    a[0] = 0                                                     # zero row: the eps clamp of sim_matrix
    verb, noun = syn.synthetic_tags(G, seed=seed)
    w = torch.rand(G, generator=g)
    x_ref = t(ref[key + "/sim"])
    close(rp.sim_matrix(a, b), x_ref, rtol=1e-5, atol=1e-6)
    sv, sn = t(ref[key + "/sim_v"]), t(ref[key + "/sim_n"])
    close(rp.sim_matrix(verb, verb), sv, rtol=1e-5, atol=1e-6)
    close(rp.sim_matrix(noun, noun), sn, rtol=1e-5, atol=1e-6)
    for i, kw in enumerate(({}, {"noun": True, "verb": False}, {"noun": False, "verb": True}, {"temperature": 0.07})):
        xo = x_ref.clone().requires_grad_(True)
        got = rp.egonce_loss(xo, sv, sn, **kw)
        close(got, ref[f"{key}/egonce/{i}"], rtol=1e-5, atol=1e-6)
        got.backward()
        close(xo.grad, ref[f"{key}/egonce_grad/{i}"], rtol=1e-4, atol=1e-7)
    close(rp.norm_softmax_loss(x_ref), ref[key + "/norm_softmax"], rtol=1e-5, atol=1e-6)
    for fix in (True, False):
        close(rp.max_margin_ranking_loss(x_ref, fix_norm=fix), ref[f"{key}/max_margin/{fix}"], rtol=1e-5, atol=1e-6)
        close(rp.adaptive_max_margin_ranking_loss(x_ref, w, fix_norm=fix), ref[f"{key}/adaptive_max_margin/{fix}"],
              rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("seed,R,C", [(1, 1, 1), (2, 5, 17), (3, 12, 300)])
def test_ranking_metrics_random(ref, seed, R, C):
    key = f"rank/{seed}"
    rng = np.random.default_rng(seed)
    sim = rng.permutation(R * C).reshape(R, C).astype(np.float32) / (R * C)     # tie-free
    rel = rng.choice([0.0, 0.0, 0.5, 1.0], size=(R, C))
    rel[np.arange(R), rng.integers(0, C, R)] = 1.0
    np.testing.assert_allclose(rp.ndcg(sim, rel), ref[key + "/ndcg"], rtol=1e-12)
    np.testing.assert_allclose(rp.ndcg(sim, rel, reduction=None), ref[key + "/ndcg_rows"], rtol=1e-12)
    np.testing.assert_allclose(rp.average_precision(sim, rel).mean(), ref[key + "/map"], rtol=1e-12)
    assert np.array_equal(rp.k_counts_of(rel), ref[key + "/k_counts"])


def test_attention_core_matches_var_attention_module(ref):
    """The oracle's divided_attention_core against the reference's VarAttention.forward (:100-137), both modes."""
    B, T, N, H = 2, 3, 4, 2
    x = t(ref["attn/x"])
    w = {k[len("attn/w/"):]: t(v) for k, v in ref.items() if k.startswith("attn/w/")}
    for mode in ("time", "space"):
        qkv = torch.nn.functional.linear(x, w["qkv.weight"], w["qkv.bias"])
        core = rp.divided_attention_core(qkv, H, T, N, mode)
        got = torch.nn.functional.linear(core, w["proj.weight"], w["proj.bias"])
        close(got, ref["attn/out/" + mode], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("fix", ["zeros", "interp", "bilinear"])
@pytest.mark.parametrize("load_f,curr_f", [(4, 16), (16, 4), (8, 8), (1, 4)])
def test_temporal_embed_inflation_matches_reference(ref, meta, fix, load_f, curr_f):
    """FrozenInTime._inflate_positional_embeds (model/model.py:145-187) of the mirror vs the reference's, called on the
    same stand-in object (the method only touches video_params, load_temporal_fix and state_dict())."""
    import types
    from egovlp_b200.model.model import FrozenInTime
    key = f"inflate/{fix}/{load_f}/{curr_f}"
    curr = {"video_model.temporal_embed": torch.zeros(1, curr_f, 12), "video_model.pos_embed": torch.zeros(1, 5, 12)}

    def stand_in():
        return types.SimpleNamespace(video_params={"num_frames": curr_f, "model": "SpaceTimeTransformer"},
                                     load_temporal_fix=fix, state_dict=lambda: curr)

    def loaded():
        gg = torch.Generator().manual_seed(7)
        return {"video_model.temporal_embed": torch.randn(1, load_f, 12, generator=gg),
                "video_model.pos_embed": torch.randn(1, 5, 12, generator=gg), "other": torch.ones(3)}

    got = FrozenInTime._inflate_positional_embeds(stand_in(), loaded())
    if fix == "interp" and load_f < curr_f:
        # the reference passes align_corners=True with mode='nearest' (:172-175), which torch rejects: its 'interp' mode
        # cannot inflate at all.  The mirror keeps the mode usable (plain nearest-neighbour along the frame axis).
        assert meta[key] == "ValueError"
        src = loaded()["video_model.temporal_embed"]
        want_te = torch.nn.functional.interpolate(src.unsqueeze(0), (curr_f, 12), mode="nearest").squeeze(0)
        torch.testing.assert_close(got["video_model.temporal_embed"], want_te, rtol=0, atol=0)
        return
    assert set(got) == set(meta[key])
    for k in meta[key]:
        want = t(ref[f"{key}/{k}"])
        assert got[k].shape == want.shape, k
        torch.testing.assert_close(got[k], want, rtol=0, atol=0)
    bad = loaded()
    bad["video_model.pos_embed"] = torch.zeros(1, 9, 12)
    assert meta[key + "/bad_pos_embed"] == "NotImplementedError"
    with pytest.raises(NotImplementedError):
        FrozenInTime._inflate_positional_embeds(stand_in(), dict(bad))


def test_data_parallel_prefix_fix_matches_reference(meta):
    from egovlp_b200.model.model import state_dict_data_parallel_fix as our_fix
    plain = OrderedDict((k, torch.tensor(float(i))) for i, k in enumerate(["a.w", "a.b", "c"]))
    dp = OrderedDict(("module." + k, v) for k, v in plain.items())
    for (load, curr), want in zip(((plain, plain), (dp, plain), (plain, dp), (dp, dp)), meta["dp_fix"]):
        got = our_fix(OrderedDict(load), curr)
        assert [[k, float(v)] for k, v in got.items()] == want


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_egomcq_accuracy_metrics_matches_reference(meta, seed):
    from egovlp_b200.model.metric import egomcq_accuracy_metrics
    g = torch.Generator().manual_seed(seed)
    Q = 50
    preds = torch.randn(Q, 5, generator=g)
    preds[3, 2] = preds[3, 4] = preds[3].max() + 1            # a tie: argmax must resolve identically
    labels = torch.randint(0, 5, (Q,), generator=g)
    types = torch.randint(1, 3, (Q,), generator=g)
    assert egomcq_accuracy_metrics(preds, labels, types) == meta[f"egomcq/{seed}"]
