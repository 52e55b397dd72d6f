"""Metrics of the reference's model/metric.py: the t2v / v2t retrieval ranks (:20-216) on the GPU (ops.gt_ranks),
EgoMCQ (:218-234) with GPU scoring (ops.egomcq_score), EPIC-MIR (:236-299), Charades-Ego mAP (:301-340) on the ranking
kernel and the Ego4D OSCC / PNR fine-tuning metrics (:342-397)."""
import warnings

import numpy as np
import torch

from .. import ops


# ------------------------------------------------------------------------------------------------------------------
# MSR-VTT-style retrieval ranks (model/metric.py:20-216; the NLQ / MQ evaluation configs list them)
# ------------------------------------------------------------------------------------------------------------------

def _sims_dev(sims):
    from ..utils.nDCG import _dev
    s = _dev(sims)
    return s if s.dtype in (torch.float32, torch.float64) else s.double()


def _host(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def cols2metrics(cols, num_queries):
    """The rank vector -> metrics, as Frozen-in-Time defines it (the reference calls it but never defines it): R@k =
    100 * #(rank < k) / num_queries for k in 1, 5, 10, 50; MedR / MeanR = median / mean of the ranks + 1; and the
    geometric mean of R1, R5, R10."""
    import scipy.stats                  # only here: the other metrics of this module do not need scipy
    cols = _host(cols)
    metrics = {}
    for k in (1, 5, 10, 50):
        metrics[f"R{k}"] = 100 * float(np.sum(cols < k)) / num_queries
    metrics["MedR"] = np.median(cols) + 1
    metrics["MeanR"] = np.mean(cols) + 1
    stats = [metrics[x] for x in ("R1", "R5", "R10")]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)         # log(0) of an R@k of 0, as scipy reports it
        metrics["geometric_mean_R1-R5-R10"] = scipy.stats.mstats.gmean(stats)
    return metrics


def t2v_ranks(sims, query_masks=None):
    """0-based rank of every (kept) query's ground-truth video: sims [Q, V], ground truth of query i is video
    i // (Q // V), ties broken optimistically.  -> (fp64 ranks on the device, number of queries)."""
    ranks = ops.gt_ranks(_sims_dev(sims), 0)
    if query_masks is None:
        return ranks, ranks.shape[0]
    keep = torch.as_tensor(_host(query_masks).reshape(-1).astype(bool))
    assert keep.numel() == ranks.shape[0], "invalid query mask shape"
    return ranks[keep.to(ranks.device)], int(keep.sum())


def v2t_ranks(sims, query_masks=None):
    """0-based rank of every video's closest ground-truth caption: sims [N, V] (text x video, transposed here as the
    reference does), captions [i c, (i + 1) c) of video i with c = N // V, ties averaged; query_masks [N] marks
    missing captions.  -> (fp64 ranks on the device, number of videos)."""
    s = _sims_dev(sims).t().contiguous()
    mask = None if query_masks is None else torch.as_tensor((_host(query_masks).reshape(-1) != 0).astype(np.uint8))
    return ops.gt_ranks(s, 1, mask), s.shape[0]


def t2v_metrics(sims, query_masks=None):
    """model/metric.py:20-124 (numpy or torch input, moved to the current CUDA device)."""
    return cols2metrics(*t2v_ranks(sims, query_masks))


def v2t_metrics(sims, query_masks=None):
    """model/metric.py:127-216 (numpy or torch input, moved to the current CUDA device)."""
    return cols2metrics(*v2t_ranks(sims, query_masks))


def egomcq_predict(text_embeds, video_embeds):
    """text [Q, C], video [Q, K, C] -> (scores [Q, K], pred [Q]); cosine similarity, ties -> lowest index."""
    return ops.egomcq_score(text_embeds.float(), video_embeds.float())


def egomcq_accuracy_metrics(preds, labels, types):
    """Same contract as the reference (model/metric.py:218-234): preds [Q, K] scores, labels [Q], types [Q] -> accuracy
    in % per question type, as tensor expressions (one argmax + two masked sums instead of a Python loop over Q).
    The reference pairs the names ["Intra-video", "Inter-video"] with the SORTED unique type ids -- so with a single
    type present it is reported as "Intra-video" whatever its id -- and that pairing is kept."""
    preds, labels, types = torch.as_tensor(preds), torch.as_tensor(labels), torch.as_tensor(types)
    hit = torch.argmax(preds, dim=1).to(labels.device) == labels.reshape(-1)
    metrics = {}
    for type_i, group_i in zip(torch.unique(types), ("Intra-video", "Inter-video")):
        sel = types.reshape(-1) == type_i
        metrics[group_i] = (hit & sel.to(hit.device)).sum().item() / sel.sum().item() * 100
    return metrics


# ------------------------------------------------------------------------------------------------------------------
# EPIC-Kitchens-100 multi-instance retrieval (model/metric.py:236-299)
# ------------------------------------------------------------------------------------------------------------------

def initialise_nDCG_values(relevancy_matrix):
    """model/metric.py:236-246."""
    from ..utils import nDCG
    rel = nDCG._rel(relevancy_matrix)
    vis_k, txt_k = nDCG.calculate_k_counts(rel), nDCG.calculate_k_counts(rel.t().contiguous())
    vis_IDCG, txt_IDCG = nDCG.calculate_IDCG(rel, vis_k), nDCG.calculate_IDCG(rel.t().contiguous(), txt_k)
    return {"v": vis_IDCG, "t": txt_IDCG}, {"v": vis_k, "t": txt_k}


def initialise_jpose_nDCG_values(relevancy_matrix):
    """model/metric.py:248-255."""
    idcg, k_values = initialise_nDCG_values(relevancy_matrix)
    return {"action": {"IDCG": idcg, "k_values": k_values}}


def mir_metrics_core(similarity_matrix, idx_arr, video_id, text_id, relevancy):
    """model/metric.py:257-299 after the annotation files are read: `similarity_matrix` [N, N] cosine similarities of
    text i vs video j in LOADER order, `idx_arr` [N] the dataset index of every loader position, `video_id` [N] /
    `text_id` [Nt] the annotation id columns, `relevancy` [N, Nt].  Everything stays on the GPU."""
    from ..utils import nDCG, mAP
    sim = nDCG._dev(similarity_matrix, torch.float32)
    sim = (sim + 1) / 2
    video_id, idx_list = list(video_id), torch.as_tensor(idx_arr).tolist()
    first = {}
    for pos, v in enumerate(video_id):
        first.setdefault(v, pos)
    indexes = [first[e] for e in text_id if e in first]                  # :266-270 (`list.index` = first occurrence)
    pos_of = {}
    for pos, i in enumerate(idx_list):
        pos_of.setdefault(i, pos)
    order = torch.tensor([pos_of[i] for i in range(len(video_id))], device=sim.device)        # :272-275
    sim = sim[order][:, order]
    sim = sim.t()[:, torch.tensor(indexes, device=sim.device)].contiguous()                  # [videos, unique texts]
    rel = nDCG._rel(relevancy)
    sim_t, rel_t = sim.t().contiguous(), rel.t().contiguous()
    vis_nDCG, txt_nDCG = nDCG.calculate_nDCG(sim, rel), nDCG.calculate_nDCG(sim_t, rel_t)
    vis_mAP, txt_mAP = mAP.calculate_mAP(sim, rel), mAP.calculate_mAP(sim_t, rel_t)
    return {"nDCG_V2T": vis_nDCG * 100, "nDCG_T2V": txt_nDCG * 100, "nDCG_AVG": 100 * (vis_nDCG + txt_nDCG) / 2,
            "mAP_V2T": vis_mAP * 100, "mAP_T2V": txt_mAP * 100, "mAP_AVG": 100 * (vis_mAP + txt_mAP) / 2}


def mir_metrics(similarity_matrix, idx_arr):
    """Same contract as the reference (reads the EPIC annotation files from the same relative paths)."""
    import os
    import pickle
    import pandas as pd
    base = "dataset/epic-kitchens/epic-kitchens-100-annotations-master/retrieval_annotations"
    video_id = pd.read_csv(os.path.join(base, "EPIC_100_retrieval_test.csv")).values[:, 0]
    text_id = pd.read_csv(os.path.join(base, "EPIC_100_retrieval_test_sentence.csv")).values[:, 0]
    with open(os.path.join(base, "relevancy/caption_relevancy_EPIC_100_retrieval_test.pkl"), "rb") as f:
        relevancy = pickle.load(f)
    return mir_metrics_core(similarity_matrix, idx_arr, video_id, text_id, relevancy)


# ------------------------------------------------------------------------------------------------------------------
# Charades-Ego (model/metric.py:301-340)
# ------------------------------------------------------------------------------------------------------------------

CHARADES_MAX_VIDEOS = 16384          # egovlp_rank_metrics ranks at most this many items per query (one CTA in smem)


def charades_class_ap(submission_array, gt_array):
    """Average precision of every class of a [videos, classes] score matrix (fp64 [classes] on the device): videos
    whose ground truth is empty score -inf; within a class, videos rank by score (compared in fp32), equal scores by
    smaller video index first, NaN scores after every real one as numpy's argsort of -score puts them; AP = sum of
    precision@k over the true positives (gt == 1) / their number, NaN for a class without one."""
    from ..utils.nDCG import _dev
    sub = _dev(submission_array, torch.float32)
    gt = _dev(gt_array)
    assert sub.dim() == 2 and gt.shape == sub.shape, "expected [videos, classes] scores and targets"
    if sub.shape[0] > CHARADES_MAX_VIDEOS:
        raise ValueError(f"charades_metrics: {sub.shape[0]} videos, at most {CHARADES_MAX_VIDEOS} are supported")
    empty = gt.sum(dim=1) == 0
    fix = torch.where(empty[:, None], torch.full_like(sub, -float("inf")), sub)
    _, ap = ops.rank_metrics(fix.t().contiguous(), (gt == 1).t().float().contiguous(), tie_mode=0, want_dcg=False)
    return ap


def charades_metrics(submission_array, gt_array):
    """model/metric.py:327-340: {'mAP': mean class AP} as a fraction; a class without a positive makes it NaN."""
    ap = charades_class_ap(submission_array, gt_array).cpu().numpy()
    return {"mAP": np.mean(ap)}


# ------------------------------------------------------------------------------------------------------------------
# Ego4D hand-object benchmarks (model/metric.py:342-397)
# ------------------------------------------------------------------------------------------------------------------

def _rows_argmax(preds):
    """argmax of every row (flattened), ties -> lowest index: torch.argmax(pred) per row as the reference loops do."""
    preds = torch.as_tensor(preds)
    return torch.argmax(preds.reshape(preds.shape[0], -1), dim=1)


def oscc_metrics(preds, labels):
    """model/metric.py:342-353: accuracy in % of the row-wise argmax of `preds` [N, C] against `labels` [N]."""
    pred = _rows_argmax(preds)
    correct = (pred == torch.as_tensor(labels).to(pred.device).reshape(-1)).sum().item()
    return {"accuracy": correct / pred.shape[0] * 100}


def pnr_metrics(preds, labels, sc_labels, fps, parent_start_frames, parent_end_frames, parent_pnr_frames):
    """model/metric.py:355-397: mean keyframe error in seconds over the clips with a state change (`sc_labels == 1`).
    The predicted keyframe maps to `(parent_end - parent_start) / 16 * argmax`, a true division of the frame tensors
    (float32 for integer frame numbers, as in the reference); the error is |mapped - (pnr - start)| / fps in float64.
    No state-change clip gives NaN: the reference's `np.mean(0.0)` fallback (:388-393) is overwritten by
    `np.mean([])` on the next line."""
    pred = _rows_argmax(preds)
    dev = pred.device

    def col(v):
        return torch.as_tensor(v).to(dev).reshape(-1)

    sc, start, end, pnr, rate = (col(v) for v in (sc_labels, parent_start_frames, parent_end_frames,
                                                  parent_pnr_frames, fps))
    keep = sc == 1
    mapped = (end[keep] - start[keep]) / 16 * pred[keep]
    err = (mapped.double() - (pnr[keep].double() - start[keep].double())).abs() / rate[keep].double()
    with warnings.catch_warnings(), np.errstate(invalid="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        return {"keyframe_distance": np.mean(err.cpu().numpy())}
