"""CPU checks of oracle/eval_port.py against tests/golden/charades.npz, recorded from the unmodified reference by
oracle/make_eval_golden.py: Charades-Ego class APs and mAP (1e-12 relative, NaN in the same places) and the t2v / v2t
rank vectors (equal); plus the metric names the shipped configs list, resolved on the package."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import eval_port as ep

CHARADES = ["realistic", "empty_rows", "nan_class", "ties", "n1"]
RANKS = ["q1", "q20", "q20_masked", "q20_quantised", "q20_quantised_f64", "q1_all_equal", "q20_all_equal"]
# every metric name in the reference's configs/{pt,ft,eval}/*.json
CONFIG_METRICS = ["egomcq_accuracy_metrics", "mir_metrics", "charades_metrics", "oscc_metrics", "pnr_metrics",
                  "t2v_metrics", "v2t_metrics"]


@pytest.fixture(scope="module")
def g():
    z = np.load(os.path.join(GOLDEN, "charades.npz"))
    return {k: z[k] for k in z.files}


def assert_rel(got, want, rtol):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    ok = ~np.isnan(want)
    assert np.all(np.abs(got[ok] - want[ok]) <= rtol * np.abs(want[ok])), np.max(np.abs(got[ok] - want[ok]))


@pytest.mark.parametrize("name", CHARADES)
def test_charades_oracle_matches_reference(g, name):
    key = f"charades/{name}/"
    scores, gt = g[key + "scores"], g[key + "targets"].astype(np.float32)
    _, _, aps = ep.map(ep.charades_fix(scores, gt), gt)
    assert_rel(aps, g[key + "aps"], 1e-12)
    assert_rel(ep.charades_metrics(scores, gt)["mAP"], g[key + "mAP"], 1e-12)
    if name == "nan_class":
        assert np.isnan(aps[17]) and np.isnan(ep.charades_metrics(scores, gt)["mAP"])


@pytest.mark.parametrize("name", RANKS)
def test_rank_oracle_matches_reference(g, name):
    key = f"ranks/{name}/"
    sims = g[key + "sims"]
    qm = g.get(key + "query_masks")
    ranks, n = ep.t2v_ranks(sims, qm)
    assert np.array_equal(ranks, g[key + "t2v"]) and n == g[key + "t2v_n"]
    ranks, n = ep.v2t_ranks(sims, qm)
    assert np.array_equal(ranks, g[key + "v2t"]) and n == g[key + "v2t_n"]


def test_zero_shot_mAP_oracle_matches_reference(g):
    res = ep.charades_metrics(g["zero_shot/sims"], g["zero_shot/targets"].astype(np.float32))
    assert_rel(res["mAP"], g["zero_shot/mAP"], 1e-12)


def test_cols2metrics_definition():
    cols = np.array([0.0, 0.5, 3.0, 7.0, 12.0, 60.0, np.inf])
    m = ep.cols2metrics(cols, 7)
    assert m["R1"] == 100 * 2 / 7 and m["R5"] == 100 * 3 / 7 and m["R10"] == 100 * 4 / 7 and m["R50"] == 100 * 5 / 7
    assert m["MedR"] == 8.0 and m["MeanR"] == np.inf
    assert abs(m["geometric_mean_R1-R5-R10"] - (m["R1"] * m["R5"] * m["R10"]) ** (1 / 3)) < 1e-12


def test_package_cols2metrics_equals_the_oracle():
    from egovlp_b200.model import metric
    rng = np.random.default_rng(3)
    for cols in (rng.integers(0, 80, 200).astype(np.float64), np.full(10, 4.5), np.array([0.0]), np.arange(30.0)):
        want = ep.cols2metrics(cols, cols.size)
        for got in (metric.cols2metrics(cols, cols.size), metric.cols2metrics(torch.from_numpy(cols), cols.size)):
            assert got == want or all(np.isclose(got[k], want[k], rtol=0, atol=0) for k in want), (got, want)


def test_config_metric_names_resolve_after_install():
    import egovlp_b200
    egovlp_b200.install_as_reference_model()
    try:
        import model.metric as mmetric
        for name in CONFIG_METRICS:
            assert callable(getattr(mmetric, name)), name
    finally:
        for k in [k for k in sys.modules if k == "model" or k.startswith("model.")]:
            del sys.modules[k]
