"""Metrics of the reference's model/metric.py: EgoMCQ (:218-234) with GPU scoring (ops.egomcq_score), EPIC-MIR
(:236-299) and the Ego4D OSCC / PNR fine-tuning metrics (:342-397)."""
import warnings

import numpy as np
import torch

from .. import ops


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
