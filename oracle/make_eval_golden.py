"""Generate tests/golden/charades.npz: what the UNMODIFIED reference (via oracle/ref_shim.py) computes for the
Charades-Ego metric, the t2v / v2t retrieval ranks and the zero-shot Charades-Ego evaluation flow.  Runs on the host
cores and needs the reference checkout (EGOVLP_REFERENCE_ROOT):   python oracle/make_eval_golden.py

Two shims for numpy 2, in this recording script only: `np.NINF` (removed in numpy 2; model/metric.py:335 uses it) and a
`cols2metrics` in the reference's metric module (called at :124 and :216 but defined nowhere) that returns the raw rank
vector, so the ranks themselves are recorded.

The zero-shot flow restates trainer/trainer_charades.py:_valid_epoch (:192-243) on a reference FrozenInTime built for 16
frames with seeded weights (egovlp_b200.synthetic.seeded_state_dict), 157 synthetic class prompts as ragged token ids
(no tokenizer offline) and 12 synthetic 4-frame clips in batches of 4.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from egovlp_b200 import synthetic as syn  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "charades.npz")
N_CLASSES = 157
# zero-shot flow: weight seed, prompt tokens (seed, length), clips (count, frames, batch, video seed, text seed)
ZS_WSEED, ZS_PROMPT_SEED, ZS_PROMPT_LEN = 41, 42, 12
ZS_CLIPS, ZS_FRAMES, ZS_BATCH, ZS_VSEED, ZS_TSEED = 12, 4, 4, 43, 44


def reference_metric():
    ref_shim.install()
    np.NINF = -np.inf
    import model.metric as ref_metric
    assert ref_metric.__file__.startswith(ref_shim.REFERENCE_ROOT), ref_metric.__file__
    ref_metric.cols2metrics = lambda cols, num_queries: (np.asarray(cols, dtype=np.float64), int(num_queries))
    return ref_metric


def multi_hot(rng, n, per_video, empty_rows=(), cover=True):
    """[n, 157] 0/1 targets: `per_video` random classes per video, every class with a positive when `cover`, the
    `empty_rows` all zero."""
    gt = np.zeros((n, N_CLASSES), dtype=np.float32)
    for i in range(n):
        gt[i, rng.choice(N_CLASSES, per_video, replace=False)] = 1
    full = [i for i in range(n) if i not in set(empty_rows)]
    if cover:
        for c in range(N_CLASSES):
            gt[full[c % len(full)], c] = 1
    gt[list(empty_rows)] = 0
    return gt


def charades_cases(rng):
    """{name: (scores [N, 157] float32, targets [N, 157])}, none with a tie between a positive and a negative."""
    cases = {}
    n = 300
    gt = multi_hot(rng, n, 3, empty_rows=(5, 77, 123, 299))
    scores = (0.1 * rng.standard_normal((n, N_CLASSES)) + 0.08 * gt).astype(np.float32)    # cosine-like, informative
    cases["realistic"] = (scores, gt)
    gt = multi_hot(rng, 40, 2, empty_rows=(0, 1, 2, 39))
    cases["empty_rows"] = ((0.2 * rng.standard_normal((40, N_CLASSES))).astype(np.float32), gt)
    gt = multi_hot(rng, 60, 2)
    gt[:, 17] = 0                                                    # class 17 has no positive: its AP and the mAP are NaN
    gt[3, 17] = 2                                                    # ... even with a non-1 label in it (tp = gt == 1)
    cases["nan_class"] = ((0.2 * rng.standard_normal((60, N_CLASSES))).astype(np.float32), gt)
    # exact ties inside a positive run and inside a negative run only: positives score from one value set, negatives
    # from a disjoint one, so every tie group has one label and its order cannot change the AP
    gt = multi_hot(rng, 80, 4, empty_rows=(9,))
    pos = rng.choice(np.array([0.5, 0.625, 0.75], dtype=np.float32), gt.shape)
    neg = rng.choice(np.array([0.125, 0.25, 0.5625, 0.875], dtype=np.float32), gt.shape)
    cases["ties"] = (np.where(gt == 1, pos, neg).astype(np.float32), gt)
    gt = multi_hot(rng, 1, 10, cover=False)
    cases["n1"] = ((0.2 * rng.standard_normal((1, N_CLASSES))).astype(np.float32), gt)
    return cases


def rank_cases(rng):
    """{name: (sims [Q, V] text x video, query_masks for t2v [Q] or None, caption masks for v2t [Q] or None)}."""
    cases = {}
    s = (0.2 * rng.standard_normal((50, 50)) + 0.3 * np.eye(50)).astype(np.float32)
    cases["q1"] = (s, None, None)
    V, q = 30, 20
    s = (0.2 * rng.standard_normal((V * q, V)) + 0.3 * np.repeat(np.eye(V), q, axis=0)).astype(np.float32)
    cases["q20"] = (s, None, None)
    m = np.ones(V * q, dtype=np.float32)
    m[rng.choice(V * q, 40, replace=False)] = 0
    m[q * 4: q * 5] = 0                                              # every caption of video 4 missing: rank +inf
    cases["q20_masked"] = (s, m, m)
    s = (np.round(2 * rng.standard_normal((V * q, V))) / 4).astype(np.float32)   # quantised: many exact ties
    cases["q20_quantised"] = (s, None, None)
    cases["q20_quantised_f64"] = (s.astype(np.float64) + 0.125, m, m)
    cases["q1_all_equal"] = (np.zeros((40, 40), dtype=np.float32), None, None)
    cases["q20_all_equal"] = (np.full((V * q, V), 0.25, dtype=np.float32), None, None)
    return cases


def zero_shot(out):
    """trainer/trainer_charades.py:_valid_epoch (:176-243) with one data loader and world size 1."""
    mm, _, _ = ref_shim.modules()
    ref_metric = reference_metric()
    net = ref_shim.build_reference_model(num_frames=16)
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=16), seed=ZS_WSEED), strict=True)
    net.eval()                                                                                         # :176
    prompts = syn.synthetic_text(N_CLASSES, ZS_PROMPT_LEN, seed=ZS_PROMPT_SEED, ragged=True)
    clip_text = syn.synthetic_text(ZS_CLIPS, 16, seed=ZS_TSEED, ragged=True)
    video = syn.synthetic_video(ZS_CLIPS, ZS_FRAMES, seed=ZS_VSEED)
    targets = multi_hot(np.random.default_rng(45), ZS_CLIPS, 20, empty_rows=(ZS_CLIPS - 1,))
    with torch.no_grad():
        dict_cls = {"text": prompts, "video": torch.Tensor(1, 4, 3, 224, 224)}                       # :197
        text_embed, _ = net(dict_cls, return_embeds=True)                                              # :198
        text_embeds = text_embed.cpu().detach()                                                        # :199
        vid_embed_arr, target_arr = [], []
        for b0 in range(0, ZS_CLIPS, ZS_BATCH):
            data = {"text": {k: v[b0:b0 + ZS_BATCH] for k, v in clip_text.items()},
                    "video": video[b0:b0 + ZS_BATCH]}
            _, vid_embed = net(data, return_embeds=True)                                               # :210
            vid_embed_arr.append(vid_embed.cpu())                                                      # :215
            target_arr.append(torch.from_numpy(targets[b0:b0 + ZS_BATCH]))                             # :220
    vid_embeds = torch.cat(vid_embed_arr)                                                              # :235
    target_embeds = torch.cat(target_arr)                                                              # :236
    sims = mm.sim_matrix(text_embeds, vid_embeds).numpy().T                                            # :238
    res = ref_metric.charades_metrics(sims, target_embeds.numpy())                                     # :243
    key = "zero_shot/"
    out[key + "prompt_ids"], out[key + "prompt_mask"] = prompts["input_ids"].numpy(), prompts["attention_mask"].numpy()
    out[key + "clip_ids"], out[key + "clip_mask"] = clip_text["input_ids"].numpy(), clip_text["attention_mask"].numpy()
    out[key + "text_embeds"], out[key + "vid_embeds"] = text_embeds.numpy(), vid_embeds.numpy()
    out[key + "sims"], out[key + "targets"] = sims, targets.astype(np.uint8)
    out[key + "mAP"] = np.asarray(res["mAP"])


def main():
    out = {}
    torch.set_num_threads(os.cpu_count())
    ref_metric = reference_metric()
    rng = np.random.default_rng(2024)
    for name, (scores, gt) in charades_cases(rng).items():
        key = f"charades/{name}/"
        out[key + "scores"], out[key + "targets"] = scores, gt.astype(np.uint8)            # 0 / 1 / 2: exact
        fix = scores.copy()
        fix[np.sum(gt, axis=1) == 0, :] = np.NINF                                 # model/metric.py:333-335
        out[key + "aps"] = ref_metric.map(fix, gt)[2]
        out[key + "mAP"] = np.asarray(ref_metric.charades_metrics(scores, gt)["mAP"])
    for name, (sims, qmask, cmask) in rank_cases(rng).items():
        key = f"ranks/{name}/"
        out[key + "sims"] = sims
        if qmask is not None:
            out[key + "query_masks"] = qmask
        out[key + "t2v"], out[key + "t2v_n"] = ref_metric.t2v_metrics(sims.copy(), qmask)
        out[key + "v2t"], out[key + "v2t_n"] = ref_metric.v2t_metrics(sims.copy(), cmask)
    zero_shot(out)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}  ({os.path.getsize(OUT) / 1024:.1f} KiB, {len(out)} arrays)")


if __name__ == "__main__":
    main()
