"""float64 restatement of the reference's video transforms (data_loader/transforms.py:34-61 with torchvision 0.26's tensor
ops) and of the reader tail around them (base/base_dataset.py:117-140: `.float() / 255`, transform, zero-padded `final`).

Each resize is a per-axis weight matrix [out, in]: a frame is `Wy @ img @ Wx^T` per channel.  The weights are the
float32 values torch computes (their coordinate rounding is part of the reference's result); the /255, the sums and the
normalisation are float64.
  train: crop (i, j, h, w) -> F.interpolate(bilinear, align_corners=False, antialias=False) -> optional hflip
  eval:  Resize(center_crop) -> CenterCrop(center_crop) -> Resize(R), torch's antialiased bilinear (triangle filter)
The parameter draws are the package's own (`egovlp_b200.transforms.resized_crop_params`); the golden file checks both
against the unmodified reference.
"""
import math

import numpy as np
import torch

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def synthetic_clip(T, H, W, seed):
    """Deterministic noise frames uint8 [T, H, W, 3] (an integer hash of (seed, t, y, x, c); no RNG library)."""
    t, y, x, c = np.ogrid[:T, :H, :W, :3]
    with np.errstate(over="ignore"):                                 # wrap-around multiplication is the hash
        v = (np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15) + t.astype(np.uint64) * np.uint64(0xD1B54A32D192ED03)
             + y.astype(np.uint64) * np.uint64(0xAEF17502108EF2D9)
             + x.astype(np.uint64) * np.uint64(0x94D049BB133111EB) + c.astype(np.uint64) * np.uint64(0xBF58476D1CE4E5B9))
        v ^= v >> np.uint64(31)
        v *= np.uint64(0x94D049BB133111EB)
        v ^= v >> np.uint64(29)
    return (v >> np.uint64(56)).astype(np.uint8)


def bilinear_weights(n_in, n_out):
    """F.interpolate(mode='bilinear', align_corners=False, antialias=False) along one axis, with the weights torch
    computes for the reference's fp32 [C, T, h, w] crop view: source coordinate scale * (o + 0.5) - 0.5 with
    scale = float32(n_in / n_out), rounded once to float32 (torch's CPU kernel evaluates it as a fused multiply-add on
    this layout).  A one-ulp difference in the coordinate moves an output by up to ~ulp(n_in) (7.6e-6 at n_in ~ 200,
    3.4e-5 after the division by std), more than the 1e-5 the outputs are compared at, so it is restated exactly."""
    m = np.zeros((n_out, n_in))
    f32 = np.float32
    scale = f32(n_in) / f32(n_out)
    for o in range(n_out):
        src = max(float(f32(float(scale) * (o + 0.5) - 0.5)), 0.0)   # exact in float64, one rounding to float32
        i0 = min(int(math.floor(src)), n_in - 1)
        i1 = i0 + (1 if i0 < n_in - 1 else 0)
        l1 = min(max(f32(src) - f32(i0), f32(0.0)), f32(1.0))
        m[o, i0] += float(f32(1.0) - l1)
        m[o, i1] += float(l1)
    return m


def aa_weights(n_in, n_out):
    """torch's antialiased bilinear (_upsample_bilinear2d_aa, align_corners=False) along one axis, with its float32
    weights (triangle filter at (x - center + 0.5) * invscale, divided by their float32 sum); identity if the size is
    unchanged (torchvision returns the image as is)."""
    if n_in == n_out:
        return np.eye(n_in)
    f32 = np.float32
    scale = f32(n_in) / f32(n_out)
    support = scale if scale >= 1.0 else f32(1.0)
    inv = f32(1.0) / scale if scale >= 1.0 else f32(1.0)
    m = np.zeros((n_out, n_in))
    for o in range(n_out):
        center = scale * (f32(o) + f32(0.5))
        lo = max(int(float(center - support) + 0.5), 0)
        hi = min(int(float(center + support) + 0.5), n_in)
        a = np.abs((np.arange(lo, hi, dtype=f32) - center + f32(0.5)) * inv)
        w = np.where(a < 1, f32(1.0) - a, f32(0.0)).astype(f32)
        total = f32(0.0)
        for v in w:
            total = f32(total + v)
        m[o, lo:hi] = w / total
    return m


def eval_geometry(H, W, center_crop):
    """torchvision Resize(center_crop) output size (short side -> center_crop, long -> int(cc * long / short)) and the
    CenterCrop offsets int(round((dim - cc) / 2)) (Python's round: halves to even)."""
    if W <= H:
        dw, dh = center_crop, int(center_crop * H / W)
    else:
        dh, dw = center_crop, int(center_crop * W / H)
    return dh, dw, int(round((dh - center_crop) / 2.0)), int(round((dw - center_crop) / 2.0))


def eval_axis_weights(n_in, center_crop, R, d1, c0):
    w1 = aa_weights(n_in, d1)[c0:c0 + center_crop]
    return aa_weights(center_crop, R) @ w1


def clip_weights(H, W, params, R, center_crop):
    """(Wy [R, H], Wx [R, W]) of one clip; params = (mode, i, j, h, w, flip), mode 0 train / 1 eval."""
    mode, i, j, h, w, flip = (int(p) for p in params)
    if mode == 0:
        wy = np.zeros((R, H))
        wx = np.zeros((R, W))
        wy[:, i:i + h] = bilinear_weights(h, R)
        wx[:, j:j + w] = bilinear_weights(w, R)
        return wy, (wx[::-1] if flip else wx)
    dh, dw, c0y, c0x = eval_geometry(H, W, center_crop)
    return eval_axis_weights(H, center_crop, R, dh, c0y), eval_axis_weights(W, center_crop, R, dw, c0x)


def transform_clip(frames, params, F, R, center_crop, mean=MEAN, std=STD):
    """uint8 [T, H, W, 3] -> float64 [F, 3, R, R]: resampled frames / 255, (v - mean) / std per channel (mean / std as
    the float32 values torch uses), frames t >= T exactly 0."""
    frames = np.asarray(frames)
    T, H, W, _ = frames.shape
    wy, wx = clip_weights(H, W, params, R, center_crop)
    img = frames.astype(np.float64) / 255.0                         # [T, H, W, 3]
    res = np.einsum("rh,thwc,sw->tcrs", wy, img, wx, optimize=True)
    m = np.asarray(mean, dtype=np.float32).astype(np.float64)[None, :, None, None]
    s = np.asarray(std, dtype=np.float32).astype(np.float64)[None, :, None, None]
    out = np.zeros((F, 3, R, R))
    out[:T] = (res - m) / s
    return out


def transform_batch(clips, params, F, R, center_crop, mean=MEAN, std=STD):
    return np.stack([transform_clip(c, p, F, R, center_crop, mean, std) for c, p in zip(clips, params)])


def host_transform_clip(frames, params, F, R, center_crop, mean=MEAN, std=STD):
    """The reference's host path in fp32, from torchvision's own ops with the clip's drawn parameters: the reader's
    `.float() / 255` and [C, T, H, W] transpose, then train: `_functional_video.resized_crop` (bilinear) + `hflip`,
    eval: Resize(cc) -> CenterCrop(cc) -> Resize(R) (torchvision's defaults), then NormalizeVideo, then the
    zero-padded `final` copy.  Needs torchvision (imported here only)."""
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from torchvision import transforms as T
        from torchvision.transforms import _functional_video as FV
    mode, i, j, h, w, flip = (int(p) for p in params)
    x = torch.as_tensor(np.asarray(frames)).permute(0, 3, 1, 2).float() / 255        # cv2 reader: [T, C, H, W]
    x = x.transpose(0, 1)
    if mode == 0:
        x = FV.resized_crop(x, i, j, h, w, (R, R), "bilinear")
        x = FV.hflip(x) if flip else x
    else:
        x = T.Compose([T.Resize(center_crop), T.CenterCrop(center_crop), T.Resize(R)])(x)
    x = FV.normalize(x, mean, std).transpose(0, 1)
    out = torch.zeros(F, 3, R, R)
    out[:x.shape[0]] = x
    return out


def rng_fingerprint():
    """(torch, python) RNG state digests, to check that a sequence of draws leaves both generators where it should."""
    import hashlib
    import random
    t = hashlib.sha1(torch.get_rng_state().numpy().tobytes()).digest()[:8]
    p = hashlib.sha1(repr(random.getstate()).encode()).digest()[:8]
    return int.from_bytes(t, "little", signed=True), int.from_bytes(p, "little", signed=True)
