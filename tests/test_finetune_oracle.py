"""CPU checks of the Ego4D OSCC / PNR fine-tuning pieces against tests/golden/finetune.npz, recorded from the unmodified
reference by oracle/make_finetune_golden.py: the oracle's cross-entropy (edge cases included), the OSCC and PNR step
losses through the full-size video tower with narrow heads, and the package's oscc / pnr metrics (exactly, NaN included);
plus the reference module names the unchanged fine-tuning trainers look up."""
import sys

import numpy as np
import pytest
import torch

from conftest import load_golden
from egovlp_b200 import synthetic as syn
from oracle import finetune_port as fp, reference_port as rp

CE_BIG_SEED = 4096


@pytest.fixture(scope="module")
def g():
    return load_golden("finetune.npz")


def close(a, b, rtol=2e-5, atol=2e-6):
    torch.testing.assert_close(a.float(), b.float(), rtol=rtol, atol=atol, equal_nan=True)


def big_ce_case():
    x = 3 * torch.randn(4096, 16, generator=torch.Generator().manual_seed(CE_BIG_SEED))
    t = torch.randint(0, 16, (4096,), generator=torch.Generator().manual_seed(CE_BIG_SEED + 1))
    return x, t


@pytest.mark.parametrize("name", ["ignored", "all_ignored", "c1", "huge", "big"])
def test_cross_entropy_oracle_matches_reference(g, name):
    key = f"ce/{name}/"
    x, t = big_ce_case() if name == "big" else (g[key + "x"], g[key + "t"])
    xr = x.clone().requires_grad_(True)
    loss = fp.cross_entropy(xr, t)
    close(loss.detach(), g[key + "loss"])
    if name == "all_ignored":
        assert torch.isnan(loss)
        return
    loss.backward()
    if name == "big":
        close(xr.grad[:64], g[key + "dx[:64]"], rtol=1e-5, atol=1e-9)
        close(xr.grad.norm(), g[key + "dx_norm"])
    else:
        close(xr.grad, g[key + "dx"], rtol=1e-5, atol=1e-8)


def test_cross_entropy_oracle_bad_target_is_nan():
    assert torch.isnan(fp.cross_entropy(torch.randn(3, 4), torch.tensor([0, 4, 1])))
    assert torch.isnan(fp.cross_entropy(torch.randn(3, 4), torch.tensor([0, -1, 1])))


@pytest.mark.parametrize("task,C,wseed,B,T,vseed", [("oscc", 2, 11, 4, 8, 21), ("pnr", 16, 12, 4, 4, 22)])
def test_step_oracle_matches_reference(g, task, C, wseed, B, T, vseed):
    """Full-size video tower (12 blocks, model built for 16 frames) + the C-wide head + the trainer's loss expression."""
    key = f"{task}/"
    p = {k: v.requires_grad_(True)
         for k, v in syn.seeded_state_dict(syn.model_dims(num_frames=16, proj_dim=C), seed=wseed).items()}
    video = syn.synthetic_video(B, T, seed=vseed)
    state = g[key + "state"]
    logits = rp.compute_video(video, p)
    close(logits, g[key + "logits"], rtol=2e-4, atol=2e-5)
    if task == "oscc":
        loss = fp.oscc_step_loss([logits], [state])
    else:
        loss = fp.pnr_step_loss([logits], [g[key + "labels"]], [state])
    close(loss, g[key + "loss"], rtol=1e-4)
    loss.backward()
    n = 0
    for k, ref in g.items():
        if not k.startswith(key + "g:"):
            continue
        name = k[len(key) + 2:]
        if name.endswith("[:2]"):
            got = p[name[:-4]].grad
            got = got.reshape(got.shape[0], -1)[:2]
        else:
            got = p[name].grad
        close(got, ref.reshape(got.shape), rtol=2e-3, atol=1e-6)
        n += 1
    assert n >= 8
    norms = {k[len(key) + 2:]: v for k, v in g.items() if k.startswith(key + "n:")}
    assert len(norms) == sum(1 for k in p if k.startswith(("video_model.", "vid_proj.")))
    for name, ref in norms.items():
        close(p[name].grad.norm(), ref, rtol=2e-3, atol=1e-7)


def test_metrics_equal_reference_exactly(g):
    from egovlp_b200.model import metric
    preds, labels = g["oscc_metrics/preds"], g["oscc_metrics/labels"]
    want = {"accuracy": float(g["oscc_metrics/accuracy"])}
    assert metric.oscc_metrics(preds, labels) == want and fp.oscc_metrics(preds, labels) == want
    args = [g["pnr_metrics/" + k] for k in ("preds", "labels", "sc_labels", "fps", "start", "end", "pnr")]
    want = float(g["pnr_metrics/keyframe_distance"])
    for fn in (metric.pnr_metrics, fp.pnr_metrics):
        got = fn(*args)["keyframe_distance"]
        assert isinstance(got, np.floating) and float(got) == want, (got, want)
    assert np.isnan(float(g["pnr_metrics/empty_keyframe_distance"]))
    empty = list(args)
    empty[2] = torch.zeros_like(args[2])
    for fn in (metric.pnr_metrics, fp.pnr_metrics):
        assert np.isnan(fn(*empty)["keyframe_distance"])


def test_metrics_accept_the_tensor_forms_trainers_pass():
    from egovlp_b200.model import metric
    preds = torch.tensor([[0.0, 1.0], [2.0, 2.0], [1.0, -1.0]])
    assert metric.oscc_metrics(preds, torch.tensor([1, 1, 0]))["accuracy"] == 2 / 3 * 100      # the tie goes to 0
    assert metric.oscc_metrics(preds.numpy(), [1, 0, 0])["accuracy"] == 100.0
    # float frame numbers: the reference's arithmetic stays in their dtype for the mapped keyframe
    out = metric.pnr_metrics(torch.eye(16)[:2] * 5, None, torch.tensor([1, 1]), torch.tensor([30.0, 25.0]),
                             torch.tensor([10.0, 0.0]), torch.tensor([42.0, 16.0]), torch.tensor([12.0, 3.0]))
    assert out["keyframe_distance"] == np.mean([abs(0 - 2) / 30.0, abs(1 - 3) / 25.0])


def test_install_as_reference_model_exposes_finetune_names():
    import egovlp_b200
    egovlp_b200.install_as_reference_model()
    try:
        import model.loss as ml
        import model.metric as mmetric
        assert ml.CrossEntropy.__module__ == "egovlp_b200.model.loss"
        assert mmetric.oscc_metrics.__module__ == "egovlp_b200.model.metric"
        assert callable(mmetric.pnr_metrics)
        # config.initialize('loss', module_loss) with configs/ft/oscc.json's {"type": "CrossEntropy", "args": {}}
        crit = getattr(ml, "CrossEntropy")(**{})
        with pytest.raises(NotImplementedError):
            crit(torch.randn(4, 2), torch.rand(4, 2))                  # class probabilities: not a form the trainers pass
        with pytest.raises(NotImplementedError):
            crit(torch.randn(4, 2, 3), torch.zeros(4, 3, dtype=torch.int64))
    finally:
        for k in [k for k in sys.modules if k == "model" or k.startswith("model.")]:
            del sys.modules[k]
