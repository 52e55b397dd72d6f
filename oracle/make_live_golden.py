"""Generate tests/golden/live_reference.npz: what the UNMODIFIED reference (via oracle/ref_shim.py) computes for the
seeded cases of tests/test_oracle_vs_live_reference.py, so that those tests compare the oracle with the reference on
any machine.  Needs the reference checkout (EGOVLP_REFERENCE_ROOT):   python oracle/make_live_golden.py

Large gradients are stored as a fixed, seeded sample of their entries (index + value) to keep the file small.
"""
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from egovlp_b200 import synthetic as syn  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference.npz")
GRAD_SAMPLES = 128

VIDEO_CASES = [(1, 4, 4, 32, 2, 1), (2, 8, 5, 32, 2, 2), (3, 4, 1, 48, 2, 1), (4, 16, 16, 32, 2, 1), (5, 4, 2, 64, 2, 1)]
TEXT_CASES = [(1, 3, 7), (2, 1, 1), (3, 4, 12)]
LOSS_CASES = [(1, 2), (2, 9), (3, 33)]
RANK_CASES = [(1, 1, 1), (2, 5, 17), (3, 12, 300)]
EGONCE_KW = ({}, {"noun": True, "verb": False}, {"noun": False, "verb": True}, {"temperature": 0.07})
INFLATE_FIX = ["zeros", "interp", "bilinear"]
INFLATE_FRAMES = [(4, 16), (16, 4), (8, 8), (1, 4)]


def sample_index(numel, seed):
    if numel <= GRAD_SAMPLES:
        return np.arange(numel, dtype=np.int64)
    g = torch.Generator().manual_seed(seed)
    return torch.randperm(numel, generator=g)[:GRAD_SAMPLES].sort().values.numpy()


def video(out, meta):
    _, vt, _ = ref_shim.modules()
    for seed, frames_model, frames_in, img, heads, depth in VIDEO_CASES:
        key = f"video/{seed}"
        dim = 64 * heads
        dims = syn.model_dims(embed_dim=dim, depth=depth, heads=heads, patch=16, img=img, num_frames=frames_model)
        sd = syn.seeded_state_dict(dims, seed=seed, text=False, proj=False)
        net = vt.SpaceTimeTransformer(img_size=img, patch_size=16, embed_dim=dim, depth=depth, num_heads=heads,
                                      num_frames=frames_model, time_init="zeros", num_classes=0)
        net.pre_logits = torch.nn.Identity()
        net.load_state_dict({k[len("video_model."):]: v for k, v in sd.items()}, strict=True)
        net.eval()
        want = net(syn.synthetic_video(2, frames_in, seed=seed, img=img))
        out[key + "/out"] = want.detach().numpy()
        probe = torch.randn(want.shape, generator=torch.Generator().manual_seed(seed))
        (want * probe).sum().backward()
        names = []
        for i, (n, q) in enumerate(net.named_parameters()):
            if q.grad is None:
                continue
            idx = sample_index(q.grad.numel(), seed * 1000 + i)
            out[f"{key}/grad_idx/{n}"] = idx
            out[f"{key}/grad/{n}"] = q.grad.flatten()[idx].numpy()
            names.append(n)
        meta[key] = names


def text(out):
    from transformers import DistilBertConfig, DistilBertModel
    d = syn.TINY_DIMS
    for seed, B, L in TEXT_CASES:
        sd = syn.seeded_state_dict(d, seed=seed, video=False, proj=False)
        cfg = DistilBertConfig(vocab_size=d["vocab"], dim=d["text_dim"], n_layers=d["text_layers"], n_heads=d["text_heads"],
                               hidden_dim=d["text_hidden"], max_position_embeddings=d["max_pos"], dropout=0.0,
                               attention_dropout=0.0)
        net = DistilBertModel(cfg).eval()
        net.load_state_dict({k[len("text_model."):]: v for k, v in sd.items()}, strict=True)
        t = syn.synthetic_text(B, L, seed=seed, ragged=True, vocab=d["vocab"])
        out[f"text/{seed}"] = net(**t).last_hidden_state.detach().numpy()


def losses(out):
    mm, _, ml = ref_shim.modules()
    for seed, G in LOSS_CASES:
        key = f"loss/{seed}"
        g = torch.Generator().manual_seed(seed)
        a, b = torch.randn(G, 24, generator=g), torch.randn(G, 24, generator=g)
        a[0] = 0
        verb, noun = syn.synthetic_tags(G, seed=seed)
        w = torch.rand(G, generator=g)
        x_ref = mm.sim_matrix(a, b)
        out[key + "/sim"] = x_ref.numpy()
        sv, sn = mm.sim_matrix(verb, verb), mm.sim_matrix(noun, noun)
        out[key + "/sim_v"], out[key + "/sim_n"] = sv.numpy(), sn.numpy()
        for i, kw in enumerate(EGONCE_KW):
            xr = x_ref.clone().requires_grad_(True)
            want = ref_shim.cpu_egonce(xr, sv, sn, **kw)
            want.backward()
            out[f"{key}/egonce/{i}"] = want.detach().numpy()
            out[f"{key}/egonce_grad/{i}"] = xr.grad.numpy()
        out[key + "/norm_softmax"] = ml.NormSoftmaxLoss()(x_ref).detach().numpy()
        for fix in (True, False):
            out[f"{key}/max_margin/{fix}"] = ml.MaxMarginRankingLoss(fix_norm=fix)(x_ref).detach().numpy()
            out[f"{key}/adaptive_max_margin/{fix}"] = ml.AdaptiveMaxMarginRankingLoss(fix_norm=fix)(x_ref, w).detach().numpy()


def ranking(out):
    ref_shim.install()
    from utils import nDCG as ref_ndcg, mAP as ref_map
    for seed, R, C in RANK_CASES:
        key = f"rank/{seed}"
        rng = np.random.default_rng(seed)
        sim = rng.permutation(R * C).reshape(R, C).astype(np.float32) / (R * C)
        rel = rng.choice([0.0, 0.0, 0.5, 1.0], size=(R, C))
        rel[np.arange(R), rng.integers(0, C, R)] = 1.0
        out[key + "/ndcg"] = np.asarray(ref_ndcg.calculate_nDCG(sim, rel))
        out[key + "/ndcg_rows"] = np.asarray(ref_ndcg.calculate_nDCG(sim, rel, reduction=None))
        out[key + "/map"] = np.asarray(ref_map.calculate_mAP(sim, rel))
        out[key + "/k_counts"] = np.asarray(ref_ndcg.calculate_k_counts(rel))


def attention(out):
    _, vt, _ = ref_shim.modules()
    torch.manual_seed(0)
    B, T, N, H = 2, 3, 4, 2
    D = 64 * H
    attn = vt.VarAttention(D, num_heads=H, qkv_bias=True)
    x = torch.randn(B, 1 + T * N, D)
    out["attn/x"] = x.numpy()
    for n, p in attn.named_parameters():
        out["attn/w/" + n] = p.detach().numpy()
    for mode, (ef, et, kw) in {"time": ("b (f n) d", "(b n) f d", {"n": N}),
                               "space": ("b (f n) d", "(b f) n d", {"f": T})}.items():
        out["attn/out/" + mode] = attn(x, ef, et, **kw).detach().numpy()


def inflate(out, meta):
    mm, _, _ = ref_shim.modules()
    for fix in INFLATE_FIX:
        for load_f, curr_f in INFLATE_FRAMES:
            key = f"inflate/{fix}/{load_f}/{curr_f}"
            curr = {"video_model.temporal_embed": torch.zeros(1, curr_f, 12), "video_model.pos_embed": torch.zeros(1, 5, 12)}

            def stand_in():
                return types.SimpleNamespace(video_params={"num_frames": curr_f, "model": "SpaceTimeTransformer"},
                                             load_temporal_fix=fix, state_dict=lambda: curr)

            def loaded():
                gg = torch.Generator().manual_seed(7)
                return {"video_model.temporal_embed": torch.randn(1, load_f, 12, generator=gg),
                        "video_model.pos_embed": torch.randn(1, 5, 12, generator=gg), "other": torch.ones(3)}

            try:
                want = mm.FrozenInTime._inflate_positional_embeds(stand_in(), loaded())
            except ValueError:
                meta[key] = "ValueError"
                continue
            meta[key] = sorted(want)
            for k, v in want.items():
                out[f"{key}/{k}"] = v.numpy()
            bad = loaded()
            bad["video_model.pos_embed"] = torch.zeros(1, 9, 12)
            try:
                mm.FrozenInTime._inflate_positional_embeds(stand_in(), dict(bad))
                meta[key + "/bad_pos_embed"] = "no error"
            except NotImplementedError:
                meta[key + "/bad_pos_embed"] = "NotImplementedError"


def data_parallel_fix(meta):
    ref_shim.install()
    from collections import OrderedDict
    from utils.util import state_dict_data_parallel_fix as ref_fix
    plain = OrderedDict((k, torch.tensor(float(i))) for i, k in enumerate(["a.w", "a.b", "c"]))
    dp = OrderedDict(("module." + k, v) for k, v in plain.items())
    cases = []
    for load, curr in ((plain, plain), (dp, plain), (plain, dp), (dp, dp)):
        want = ref_fix(OrderedDict(load), curr)
        cases.append([[k, float(v)] for k, v in want.items()])
    meta["dp_fix"] = cases


def egomcq_metrics(meta):
    ref_shim.install()
    import model.metric as ref_metric
    for seed in (0, 1, 2):
        g = torch.Generator().manual_seed(seed)
        Q = 50
        preds = torch.randn(Q, 5, generator=g)
        preds[3, 2] = preds[3, 4] = preds[3].max() + 1
        labels = torch.randint(0, 5, (Q,), generator=g)
        types_ = torch.randint(1, 3, (Q,), generator=g)
        meta[f"egomcq/{seed}"] = ref_metric.egomcq_accuracy_metrics(preds, labels, types_)


def main():
    out, meta = {}, {}
    video(out, meta)
    text(out)
    losses(out)
    ranking(out)
    attention(out)
    inflate(out, meta)
    data_parallel_fix(meta)
    egomcq_metrics(meta)
    out["meta"] = np.asarray(json.dumps(meta, sort_keys=True))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}  ({os.path.getsize(OUT) / 1024:.1f} KiB, {len(out)} arrays)")


if __name__ == "__main__":
    main()
