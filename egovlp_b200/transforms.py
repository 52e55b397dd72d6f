"""Dataset video transforms on the GPU (data_loader/transforms.py:34-61 of the reference).

The reference's dataset workers convert every decoded clip to fp32 at source resolution (`.float() / 255`), run the
transform on the host and copy the result into a zero-padded `[num_frames, 3, R, R]` tensor (base/base_dataset.py:117-140,
220-243).  Here the worker only draws the clip's random parameters and hands over its raw uint8 frames:

    tsfm = init_video_transform_dict(...)[split]      # in the worker: tsfm(uint8 [T, H, W, 3]) -> {"frames", "params"}
    loader = DataLoader(ds, collate_fn=collate_video_clips, pin_memory=True, ...)
    for batch in DevicePrefetcher(loader, "cuda", transform=DeviceVideoTransform(num_frames)):
        batch["video"]                                  # fp32 [B, num_frames, 3, R, R], as the reference's loader gives

and one sm_90a kernel (egovlp_video_transform) does the crop, resize, flip, /255, normalisation and zero padding.

The `train` object draws its parameters with the same RNG calls, in the same order, as the reference's `Compose`
(RandomResizedCropVideo -> RandomHorizontalFlipVideo -> ColorJitter), so a worker seeded by the DataLoader yields the
crops and flips the reference would, and leaves the torch and python RNGs in the same state.  The draws are restated
here from torchvision's definitions; torchvision is not imported.
"""
import math
import random

import numpy as np
import torch
from torch.utils.data import default_collate

TRAIN, EVAL = 0, 1
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def _as_clip(frames):
    frames = torch.as_tensor(frames)
    if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] != 3 or frames.shape[0] < 1:
        raise ValueError(f"expected decoded uint8 frames [T >= 1, H, W, 3], got {frames.dtype} {tuple(frames.shape)}")
    return frames


def resized_crop_params(height, width, scale, ratio=(3.0 / 4.0, 4.0 / 3.0)):
    """The crop box (i, j, h, w) of torchvision's RandomResizedCrop.get_params, with its torch RNG draws: up to ten
    (area, log-aspect) tries, then the ratio-clamped centre crop."""
    area = height * width
    log_ratio = torch.log(torch.tensor(ratio))
    for _ in range(10):
        target_area = area * torch.empty(1).uniform_(scale[0], scale[1]).item()
        aspect_ratio = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1])).item()
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if 0 < w <= width and 0 < h <= height:
            i = torch.randint(0, height - h + 1, size=(1,)).item()
            j = torch.randint(0, width - w + 1, size=(1,)).item()
            return i, j, h, w
    in_ratio = float(width) / float(height)
    if in_ratio < min(ratio):
        w = width
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = height
        w = int(round(h * max(ratio)))
    else:
        w, h = width, height
    return (height - h) // 2, (width - w) // 2, h, w


class TrainClipParams:
    """RandomResizedCropVideo(input_res, scale) -> RandomHorizontalFlipVideo() -> ColorJitter(0, 0, 0): draws the crop
    box, the flip (python `random`) and ColorJitter's operation order (`torch.randperm(4)`, applied to nothing)."""

    def __init__(self, input_res, randcrop_scale):
        self.input_res, self.scale = input_res, tuple(randcrop_scale)

    def __call__(self, frames):
        frames = _as_clip(frames)
        i, j, h, w = resized_crop_params(frames.shape[1], frames.shape[2], self.scale)
        flip = random.random() < 0.5
        torch.randperm(4)
        return {"frames": frames, "params": (TRAIN, i, j, h, w, int(flip))}


class EvalClipParams:
    """Resize(center_crop) -> CenterCrop(center_crop) -> Resize(input_res): no random draws; the geometry follows from
    the frame size, on the GPU."""

    def __call__(self, frames):
        return {"frames": _as_clip(frames), "params": (EVAL, 0, 0, 0, 0, 0)}


def init_video_transform_dict(input_res=224, center_crop=256, randcrop_scale=(0.5, 1.0), color_jitter=(0, 0, 0),
                              norm_mean=IMAGENET_MEAN, norm_std=IMAGENET_STD):
    """Worker-side half of the reference's `init_video_transform_dict` (same signature and defaults).  `input_res`,
    `center_crop`, `norm_mean` and `norm_std` take effect in the device half, `DeviceVideoTransform`, which must be
    given the same values."""
    if any(c != 0 for c in color_jitter):
        raise NotImplementedError("colour jitter on the GPU path: only color_jitter=(0, 0, 0) is supported")
    ev = EvalClipParams()
    return {"train": TrainClipParams(input_res, randcrop_scale), "val": ev, "test": ev}


def collate_video_clips(batch, key="video"):
    """Packs the clips under `key` ({"frames": uint8 [T, H, W, 3], "params"}) of a batch into one uint8 buffer and an
    int64 descriptor table [B, 10] of (byte offset, T, H, W, mode, i, j, h, w, flip) rows; the other keys go through
    `default_collate`.  The table stays a host numpy array (the kernel's binding checks it before launch, and the
    device feed leaves it on the host); `DataLoader(pin_memory=True)` pins the buffer."""
    clips = [item[key] for item in batch]
    sizes = [c["frames"].numel() for c in clips]
    frames = torch.empty(sum(sizes), dtype=torch.uint8)
    desc = np.zeros((len(clips), 10), dtype=np.int64)
    off = 0
    for b, (c, n) in enumerate(zip(clips, sizes)):
        f = c["frames"]
        frames[off:off + n].view(f.shape).copy_(f)
        desc[b, :4] = (off, *f.shape[:3])
        desc[b, 4:] = c["params"]
        off += n
    out = default_collate([{k: v for k, v in item.items() if k != key} for item in batch])
    out[key] = {"frames": frames, "desc": desc}
    return out


def apply_video_transform(packed, num_frames, input_res=224, center_crop=256, norm_mean=IMAGENET_MEAN,
                          norm_std=IMAGENET_STD):
    """Runs the transform kernel on a packed batch (`collate_video_clips`) whose frames are on the GPU (a host buffer
    is copied to the current device first).  Returns fp32 [B, num_frames, 3, input_res, input_res]."""
    from . import ops
    frames = packed["frames"]
    if not frames.is_cuda:
        frames = frames.to(torch.cuda.current_device(), non_blocking=True)
    return ops.video_transform(frames, packed["desc"], num_frames, input_res, center_crop, norm_mean, norm_std)


class DeviceVideoTransform:
    """Batch transform for `DevicePrefetcher(transform=...)`: replaces batch[key] (packed clips) by the kernel's
    fp32 clip tensor.  Takes the same transform keys as `init_video_transform_dict`, so one config dict serves both
    halves; `randcrop_scale` acts in the worker (the drawn crop boxes arrive in the descriptor table)."""

    def __init__(self, num_frames, input_res=224, center_crop=256, randcrop_scale=(0.5, 1.0), color_jitter=(0, 0, 0),
                 norm_mean=IMAGENET_MEAN, norm_std=IMAGENET_STD, key="video"):
        if any(c != 0 for c in color_jitter):
            raise NotImplementedError("colour jitter on the GPU path: only color_jitter=(0, 0, 0) is supported")
        self.num_frames, self.key = num_frames, key
        self.cfg = dict(input_res=input_res, center_crop=center_crop, norm_mean=norm_mean, norm_std=norm_std)

    def __call__(self, batch):
        batch = dict(batch)
        batch[self.key] = apply_video_transform(batch[self.key], self.num_frames, **self.cfg)
        return batch
