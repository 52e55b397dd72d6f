"""Record tests/golden/video_large_grid.npz from the UNMODIFIED reference SpaceTimeTransformer (via oracle/ref_shim.py)
on the CPU: a tiny tower on frames of more than 255 patches, which the video tower's spatial attention runs on its
tiled kernel.

Run in the build container only (needs the reference):   python oracle/make_large_grid_golden.py

Geometry: embed_dim 128, depth 2, 2 heads, num_frames 4, every weight seeded (the temporal attention non-zero), with
T = 3 < num_frames frames of 256 x 256 px (N = 256) and of 256 x 320 px (N = 320), patch 16.  Per geometry it keeps
the CLS features, 64 seeded rows of the last block's token outputs, 64 seeded elements of every parameter gradient and
every gradient's norm, for the loss sum(features * probe).  Weights, frames and probe are re-derived from the seeds
(egovlp_b200.synthetic), so the file stays small.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from egovlp_b200 import synthetic as syn  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "video_large_grid.npz")
GEOMETRIES = {"n256": (256, 256), "n320": (256, 320)}
B, T, SEED, SAMPLE = 2, 3, 11, 64


def dims(img):
    return syn.model_dims(embed_dim=128, depth=2, heads=2, patch=16, img=img, num_frames=4, proj_dim=32)


def sample_index(numel, tag):
    """SAMPLE seeded element indices of a tensor of `numel` elements (all of them when it is smaller)."""
    g = torch.Generator().manual_seed(sum(map(ord, tag)))
    return torch.randperm(numel, generator=g)[:SAMPLE]


def record(tag, img):
    _, vt, _ = ref_shim.modules()
    sd = syn.seeded_state_dict(dims(img), seed=SEED, text=False, proj=False)
    net = vt.SpaceTimeTransformer(img_size=img, patch_size=16, embed_dim=128, depth=2, num_heads=2, num_frames=4,
                                  time_init="zeros", num_classes=0)
    net.pre_logits = torch.nn.Identity()
    print(tag, "load:", net.load_state_dict({k[len("video_model."):]: v for k, v in sd.items()}, strict=True))
    net.eval()
    tokens = {}
    net.blocks[-1].register_forward_hook(lambda m, i, o: tokens.setdefault("x", o))
    video = syn.synthetic_video(B, T, seed=SEED, img=img)
    out = net(video)
    probe = torch.randn(out.shape, generator=torch.Generator().manual_seed(SEED + 1))
    (out * probe).sum().backward()
    x = tokens["x"].detach()
    rows = sample_index(x.shape[0] * x.shape[1], tag + ":tokens")
    res = {f"{tag}:out": out, f"{tag}:probe": probe, f"{tag}:token_rows": rows,
           f"{tag}:tokens": x.reshape(-1, x.shape[-1])[rows]}
    for n, p in net.named_parameters():
        if p.grad is None:
            continue
        idx = sample_index(p.numel(), f"{tag}:{n}")
        res[f"{tag}:gi:video_model.{n}"] = idx
        res[f"{tag}:g:video_model.{n}"] = p.grad.flatten()[idx]
        res[f"{tag}:n:video_model.{n}"] = p.grad.norm()
    return res


def main():
    torch.manual_seed(0)
    torch.set_num_threads(os.cpu_count())
    arrs = {"seed": SEED, "B": B, "T": T}
    for tag, img in GEOMETRIES.items():
        arrs[f"{tag}:img"] = np.asarray(img)
        arrs.update(record(tag, img))
    arrs = {k: (v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in arrs.items()}
    np.savez_compressed(OUT, **arrs)
    print(f"wrote {OUT}  ({os.path.getsize(OUT) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
