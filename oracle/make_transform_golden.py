"""Generate tests/golden/video_transforms.npz: what the UNMODIFIED reference's `init_video_transform_dict`
(data_loader/transforms.py:34-61, torchvision 0.26) and its reader tail (base/base_dataset.py:117-140 and the cv2 reader
:220-243: uint8 frames -> `.float() / 255` -> [C, T, H, W] -> transform -> [T, C, H, W] -> zero-padded `final`)
produce.  Runs on the host cores and needs the reference checkout (EGOVLP_REFERENCE_ROOT):
    python oracle/make_transform_golden.py

Recorded:
  * `case{k}:*` -- one clip per case (frames `transform_port.synthetic_clip(T, H, W, seed)`), every split, with
    torch and python `random` seeded to `seed` before the transform.  `params` is the crop box and flip the reference
    drew (read by wrapping torchvision's `resized_crop` / `hflip`, which the reference calls).  Most cases use
    input_res 112 / center_crop 128, five the full 224 / 256 (including 224x224 frames, whose first eval
    resize upsamples 224 -> 256); `idx` / `val` are a seeded sample of the output's flat
    entries (the whole outputs would be several MB), plus every zero-padded frame's first entry.
  * `draws:*` -- a few hundred train draws in sequence under one seed, on mixed frame sizes (the 10-try fallback
    included): the reference's (i, j, h, w, flip) and, after each clip, digests of the torch and python RNG states.
  * `aa_vs_no_aa` -- max |difference| of the eval output with torchvision's antialiased resize (0.26) against the
    non-antialiased resize torchvision 0.13.1 did on tensors, on the Ego4D / Charades / EPIC frame sizes.
"""
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle import transform_port as tp  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "video_transforms.npz")
SAMPLE = 2048
# (H, W, T, F, split, full_size, seed)
SIZES = [(256, 455), (455, 256), (480, 640), (256, 256), (224, 224), (301, 199), (40, 900)]
CASES = ([(h, w, 3, 4, s, False, 100 + 10 * k + n) for k, (h, w) in enumerate(SIZES)
          for n, s in enumerate(("train", "val", "test"))]
         + [(256, 455, 4, 4, "train", True, 201), (256, 455, 2, 3, "test", True, 202), (480, 640, 1, 2, "val", True, 203),
            (224, 224, 1, 4, "test", False, 204), (224, 224, 1, 4, "train", False, 205),
            (224, 224, 2, 3, "test", True, 206), (224, 224, 3, 3, "val", True, 207)])   # first resize upsamples
N_DRAWS, DRAW_SEED = 300, 7
DRAW_SIZES = SIZES + [(1080, 1920), (600, 40), (2, 2), (3, 700)]


def reference_transforms(**kw):
    ref_shim.install()
    from data_loader.transforms import init_video_transform_dict
    ref_t = sys.modules["data_loader.transforms"]      # the package re-exports torchvision's `transforms` under that name
    assert ref_t.__file__.startswith(ref_shim.REFERENCE_ROOT), ref_t.__file__
    return init_video_transform_dict(**kw)


class Spy:
    """Records the crop box / flip the reference's train transform applies (wraps the torchvision functions it calls)."""

    def __init__(self):
        import torchvision.transforms._functional_video as fv
        self.fv, self.box, self.flip = fv, None, 0
        self.real_rc, self.real_flip = fv.resized_crop, fv.hflip

        def rc(clip, i, j, h, w, *a, **k):
            self.box = (i, j, h, w)
            return self.real_rc(clip, i, j, h, w, *a, **k)

        def hf(clip):
            self.flip = 1
            return self.real_flip(clip)
        fv.resized_crop, fv.hflip = rc, hf

    def take(self):
        box, flip, self.box, self.flip = self.box, self.flip, None, 0
        return box, flip


def reader_tail(tsfm, frames_u8, F, R):
    imgs = torch.from_numpy(frames_u8).permute(0, 3, 1, 2).float() / 255      # cv2 reader: [T, C, H, W]
    imgs = tsfm(imgs.transpose(0, 1)).transpose(0, 1)
    final = torch.zeros([F, 3, R, R])
    final[:imgs.shape[0]] = imgs
    return final


def main():
    rec = {}
    spy = Spy()
    dicts = {False: reference_transforms(input_res=112, center_crop=128),
             True: reference_transforms(input_res=224, center_crop=256)}
    for k, (H, W, T, F, split, full, seed) in enumerate(CASES):
        R, cc = (224, 256) if full else (112, 128)
        frames = tp.synthetic_clip(T, H, W, seed)
        if (H, W, T) == (224, 224, 1):
            frames[:] = 0                                    # the `lax` loader's black 1-frame fallback clip
        torch.manual_seed(seed)
        random.seed(seed)
        out = reader_tail(dicts[full][split], frames, F, R).numpy()
        box, flip = spy.take()
        params = (0, *box, flip) if split == "train" else (1, 0, 0, 0, 0, 0)
        rng = np.random.default_rng(seed)
        idx = np.unique(np.concatenate([rng.choice(out.size, SAMPLE, replace=False),
                                        np.arange(T, F) * (out.size // F)])).astype(np.int64)
        rec.update({f"case{k}:meta": np.array([H, W, T, F, R, cc, seed], np.int64),
                    f"case{k}:split": np.array(split), f"case{k}:params": np.array(params, np.int64),
                    f"case{k}:idx": idx, f"case{k}:val": out.reshape(-1)[idx]})
        print(f"case {k}: {H}x{W} T={T} F={F} {split} R={R} params={params}")

    tsfm = dicts[False]["train"]
    torch.manual_seed(DRAW_SEED)
    random.seed(DRAW_SEED)
    rs = np.random.default_rng(DRAW_SEED)
    sizes, draws, fps = [], [], []
    for n in range(N_DRAWS):
        H, W = DRAW_SIZES[rs.integers(len(DRAW_SIZES))]
        tsfm(torch.zeros(3, 1, H, W))
        box, flip = spy.take()
        sizes.append((H, W))
        draws.append((*box, flip))
        fps.append(tp.rng_fingerprint())
    rec.update({"draws:seed": np.array(DRAW_SEED), "draws:sizes": np.array(sizes, np.int64),
                "draws:params": np.array(draws, np.int64), "draws:rng": np.array(fps, np.int64)})
    print("fallback draws:", sum(1 for (H, W), d in zip(sizes, draws) if (H, W) == (40, 900)))

    # torchvision 0.13.1 resized tensors without antialias: size of the difference on the eval path
    import torchvision.transforms as T
    diffs = []
    for H, W in [(256, 455), (480, 640), (256, 340)]:
        x = torch.from_numpy(tp.synthetic_clip(2, H, W, 9)).permute(3, 0, 1, 2).float() / 255
        outs = []
        for aa in (True, False):
            f = T.Compose([T.Resize(256, antialias=aa), T.CenterCrop(256), T.Resize(224, antialias=aa)])
            outs.append(dicts[True]["test"].transforms[-1](f(x)))
        diffs.append((H, W, (outs[0] - outs[1]).abs().max().item()))
        print(f"eval {H}x{W}: max |antialias - no antialias| after normalisation = {diffs[-1][2]:.4f}")
    rec["aa_vs_no_aa"] = np.array(diffs, np.float64)
    np.savez_compressed(OUT, **rec)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
