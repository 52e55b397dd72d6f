"""Host restatement (numpy) of the reference's evaluation metrics for Charades-Ego and the MSR-VTT-style retrieval ranks.
TEST INFRASTRUCTURE ONLY, like oracle/reference_port.py: imported by tests/ and tools/bench_charades.py's host baseline,
never by the product package.  Pinned against the unmodified reference by oracle/make_eval_golden.py ->
tests/golden/charades.npz (tests/test_eval_oracle.py).  Every function names the reference lines it restates.

Tie rules.  The ranks of t2v / v2t are fully determined by the reference (distance subtraction), so they are restated
exactly.  `map` ranks with the reference's `np.argsort(-x)`, whose default sort is not stable: equal scores that
straddle a positive and a negative are unspecified there.  Here the argsort is stable, i.e. equal scores rank by
smaller video index first, the rule the package documents; NaN scores rank after every real one (numpy sorts NaN
last), by video index among themselves."""
import warnings

import numpy as np
import scipy.stats


def map(submission_array, gt_array):                                      # noqa: A001  (the reference's name)
    """model/metric.py:301-325 (m_ap, w_ap, m_aps), with a stable argsort (:306)."""
    m_aps = []
    n_classes = submission_array.shape[1]
    for oc_i in range(n_classes):
        sorted_idxs = np.argsort(-submission_array[:, oc_i], kind="stable")
        tp = gt_array[:, oc_i][sorted_idxs] == 1
        fp = np.invert(tp)
        n_pos = tp.sum()
        if n_pos < 0.1:
            m_aps.append(float("nan"))
            continue
        prec = np.cumsum(tp) / (np.cumsum(fp) + np.cumsum(tp)).astype(float)
        avg_prec = 0
        for i in range(submission_array.shape[0]):
            if tp[i]:
                avg_prec += prec[i]
        m_aps.append(avg_prec / n_pos.astype(float))
    m_aps = np.array(m_aps)
    m_ap = np.mean(m_aps)
    w_ap = m_aps * gt_array.sum(axis=0) / gt_array.sum().sum().astype(float)
    return m_ap, w_ap, m_aps


def charades_fix(submission_array, gt_array):
    """model/metric.py:333-335: videos with an empty ground truth score -inf in every class."""
    fix = submission_array.copy()
    fix[np.sum(gt_array, axis=1) == 0, :] = -np.inf
    return fix


def charades_metrics(submission_array, gt_array):
    """model/metric.py:327-340."""
    m_ap, _, _ = map(charades_fix(submission_array, gt_array), gt_array)
    return {"mAP": m_ap}


def t2v_ranks(sims, query_masks=None):
    """model/metric.py:32-115: 0-based position of query i's ground-truth distance (video i // (Q // V)) among its
    row's sorted distances, first match (break_ties = "optimistically", :66-73); masked queries dropped (:109-115)."""
    num_queries, num_vids = sims.shape
    assert num_queries % num_vids == 0, "the reference's own cols.size assertion (:96-100)"
    q = num_queries // num_vids
    dists = -sims
    sorted_dists = np.sort(dists, axis=1)
    gt = dists[np.arange(num_queries), np.arange(num_queries) // q][:, None]
    match = (sorted_dists - gt) == 0
    assert match.any(axis=1).all(), "the reference's own cols.size assertion (:96-100)"
    cols = np.argmax(match, axis=1).astype(np.float64)
    if query_masks is not None:
        keep = query_masks.reshape(-1).astype(bool)
        cols, num_queries = cols[keep], keep.sum()
    return cols, num_queries


def v2t_ranks(sims, query_masks=None):
    """model/metric.py:143-191: per video, over its captions [ii c, (ii + 1) c), the smallest mean position of the
    caption's distance among the sorted row (break_ties = "averaging"); masked captions become MISSING_VAL = 1e8 in the
    row and are skipped as candidates (:159-179)."""
    sims = sims.T
    num_queries, num_caps = sims.shape
    dists = -sims
    caps_per_video = num_caps // num_queries
    missing = 1e8
    query_ranks = []
    for ii in range(num_queries):
        row_dists = dists[ii, :].copy()
        if query_masks is not None:
            row_dists[np.logical_not(query_masks.reshape(-1))] = missing
        sorted_dists = np.sort(row_dists)
        min_rank = np.inf
        for jj in range(ii * caps_per_video, (ii + 1) * caps_per_video):
            if row_dists[jj] == missing:
                continue
            with np.errstate(invalid="ignore"):
                ranks = np.where((sorted_dists - row_dists[jj]) == 0)[0]
            if ranks.size == 0:                   # a NaN or infinite distance never matches: ranks.mean() = NaN never wins
                continue
            rank = ranks.mean()
            if rank < min_rank:
                min_rank = rank
        query_ranks.append(min_rank)
    return np.array(query_ranks, dtype=np.float64), num_queries


def cols2metrics(cols, num_queries):
    """The reference calls cols2metrics (model/metric.py:124, :216) but never defines it; Frozen-in-Time's definition:
    R@k = 100 #(rank < k) / num_queries, MedR / MeanR = median / mean rank + 1, geometric mean of R1, R5, R10."""
    metrics = {}
    for k in (1, 5, 10, 50):
        metrics[f"R{k}"] = 100 * float(np.sum(cols < k)) / num_queries
    metrics["MedR"] = np.median(cols) + 1
    metrics["MeanR"] = np.mean(cols) + 1
    stats = [metrics[x] for x in ("R1", "R5", "R10")]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        metrics["geometric_mean_R1-R5-R10"] = scipy.stats.mstats.gmean(stats)
    return metrics


def t2v_metrics(sims, query_masks=None):
    """model/metric.py:20-124."""
    return cols2metrics(*t2v_ranks(sims, query_masks))


def v2t_metrics(sims, query_masks=None):
    """model/metric.py:127-216."""
    return cols2metrics(*v2t_ranks(sims, query_masks))
