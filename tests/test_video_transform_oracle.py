"""CPU checks of the GPU video-transform path's host half and of its float64 oracle, against
tests/golden/video_transforms.npz (recorded from the unmodified reference by oracle/make_transform_golden.py)."""
import os
import random

import numpy as np
import pytest
import torch

from egovlp_b200 import transforms as vt
from oracle import transform_port as tp

ORACLE_TOL = 1e-5


@pytest.fixture(scope="module")
def gold():
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "video_transforms.npz"))
    return {k: z[k] for k in z.files}


def golden_cases(gold):
    k = 0
    while f"case{k}:meta" in gold:
        H, W, T, F, R, cc, seed = (int(v) for v in gold[f"case{k}:meta"])
        frames = tp.synthetic_clip(T, H, W, seed)
        if (H, W, T) == (224, 224, 1):
            frames[:] = 0
        yield k, frames, F, R, cc, gold[f"case{k}:params"], gold[f"case{k}:idx"], gold[f"case{k}:val"]
        k += 1


def test_oracle_matches_reference_golden(gold):
    n = 0
    for k, frames, F, R, cc, params, idx, val in golden_cases(gold):
        out = tp.transform_clip(frames, params, F, R, cc)
        err = np.abs(out.reshape(-1)[idx] - val).max()
        assert err <= ORACLE_TOL, (k, err)
        T = frames.shape[0]
        assert (out[T:] == 0).all(), k
        pad = idx >= T * (out.size // F)
        assert (val[pad] == 0).all(), k
        n += 1
    assert n >= 20


def test_train_draws_match_reference(gold):
    """The package's draws equal the reference transform's, clip after clip, and leave both RNGs in its state."""
    sizes, params, rng = gold["draws:sizes"], gold["draws:params"], gold["draws:rng"]
    seed = int(gold["draws:seed"])
    torch.manual_seed(seed)
    random.seed(seed)
    tsfm = vt.init_video_transform_dict(input_res=112, center_crop=128)["train"]
    fallback = 0
    for n, (H, W) in enumerate(sizes):
        got = tsfm(torch.zeros(1, int(H), int(W), 3, dtype=torch.uint8))["params"]
        assert got[0] == vt.TRAIN
        assert tuple(got[1:]) == tuple(int(v) for v in params[n]), (n, H, W, got, params[n])
        assert tp.rng_fingerprint() == tuple(int(v) for v in rng[n]), n
        fallback += (H, W) == (40, 900)
    assert len(sizes) >= 200 and fallback > 0


def test_golden_train_params_follow_from_seed(gold):
    for k, frames, F, R, cc, params, idx, val in golden_cases(gold):
        if params[0] != vt.TRAIN:
            continue
        seed = int(gold[f"case{k}:meta"][-1])
        torch.manual_seed(seed)
        random.seed(seed)
        got = vt.init_video_transform_dict(input_res=R, center_crop=cc)["train"](frames)["params"]
        assert tuple(got) == tuple(int(v) for v in params), k


def test_eval_and_options():
    d = vt.init_video_transform_dict()
    assert d["val"](np.zeros((2, 5, 7, 3), np.uint8))["params"] == (vt.EVAL, 0, 0, 0, 0, 0)
    with pytest.raises(NotImplementedError):
        vt.init_video_transform_dict(color_jitter=(0.4, 0, 0))
    cfg = dict(input_res=224, center_crop=256, randcrop_scale=(0.5, 1.0), color_jitter=(0, 0, 0),
               norm_mean=(0.485, 0.456, 0.406), norm_std=(0.229, 0.224, 0.225))
    vt.init_video_transform_dict(**cfg)
    vt.DeviceVideoTransform(16, **cfg)                          # one config dict serves both halves
    with pytest.raises(NotImplementedError):
        vt.DeviceVideoTransform(16, **{**cfg, "color_jitter": (0, 0.2, 0)})
    with pytest.raises(ValueError):
        d["train"](torch.zeros(2, 5, 7, 3))                     # fp32 frames: the GPU path takes decoded uint8
    with pytest.raises(ValueError):
        d["test"](torch.zeros(2, 3, 5, 7, dtype=torch.uint8))   # channels-first


def test_collate_packs_ragged_clips():
    shapes = [(3, 5, 7), (1, 2, 9), (4, 6, 4)]
    items = []
    for b, (T, H, W) in enumerate(shapes):
        f = torch.from_numpy(tp.synthetic_clip(T, H, W, b))
        if b == 2:
            f = f.transpose(1, 2).contiguous().transpose(1, 2)  # a non-contiguous view packs as its values
        items.append({"video": {"frames": f, "params": (vt.TRAIN, 0, 1, H - 1, W - 2, b % 2)},
                      "text": f"caption {b}", "label": torch.tensor(b)})
    out = vt.collate_video_clips(items)
    frames, desc = out["video"]["frames"], out["video"]["desc"]
    assert desc.dtype == np.int64 and desc.shape == (3, 10)
    assert frames.dtype == torch.uint8 and frames.numel() == sum(T * H * W * 3 for T, H, W in shapes)
    off = 0
    for b, (T, H, W) in enumerate(shapes):
        assert tuple(desc[b]) == (off, T, H, W, vt.TRAIN, 0, 1, H - 1, W - 2, b % 2)
        n = T * H * W * 3
        assert torch.equal(frames[off:off + n].view(T, H, W, 3), items[b]["video"]["frames"])
        off += n
    assert out["text"] == ["caption 0", "caption 1", "caption 2"]
    assert torch.equal(out["label"], torch.tensor([0, 1, 2]))


def test_oracle_weights_are_convex_and_shift_free():
    for n_in, n_out in [(256, 224), (224, 256), (455, 112), (40, 128), (5, 5)]:
        for m in (tp.aa_weights(n_in, n_out), tp.bilinear_weights(n_in, n_out)):
            assert (m >= 0).all() and np.allclose(m.sum(1), 1.0, atol=1e-6)
    assert np.array_equal(tp.aa_weights(7, 7), np.eye(7))
    assert tp.eval_geometry(256, 455, 256) == (256, 455, 0, 100)    # round(99.5) = 100 (halves to even)
    assert tp.eval_geometry(480, 640, 256) == (256, 341, 0, 42)     # round(42.5) = 42
