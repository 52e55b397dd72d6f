"""egovlp_video_transform (csrc/video_transform.cu) against the float64 oracle (oracle/transform_port.py) and the
reference's own outputs (tests/golden/video_transforms.npz).

Bound: 1e-5 absolute after normalisation.  Each output is a convex combination of values in [0, 1] summed in fp32 with
the reference's fp32 weights, then divided by std ~ 0.225: fp32 rounding gives ~1e-7 before the division.  An
off-by-one tap on these noise frames errs by >= 1e-2."""
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

from oracle import transform_port as tp

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _note(name, err):
    print(f"[video_transform] {name}: worst |err| {err:.3e} = {err / TOL:.3f} of the bound")


@pytest.fixture(scope="module")
def vt():
    from egovlp_b200 import transforms
    return transforms


def _batch(vt, clips, params):
    items = [{"video": {"frames": torch.from_numpy(c), "params": tuple(int(v) for v in p)}} for c, p in
             zip(clips, params)]
    return vt.collate_video_clips(items)["video"]


def _run(vt, clips, params, F, R, cc):
    packed = _batch(vt, clips, params)
    out = vt.apply_video_transform(packed, F, input_res=R, center_crop=cc)
    torch.cuda.synchronize()
    return out, packed


def _check(vt, name, clips, params, F, R, cc):
    out, _ = _run(vt, clips, params, F, R, cc)
    ref = tp.transform_batch(clips, params, F, R, cc)
    err = np.abs(out.cpu().double().numpy() - ref).max()
    _note(name, err)
    assert err <= TOL, (name, err)
    for b, c in enumerate(clips):
        pad = out[b, c.shape[0]:]
        assert torch.equal(pad, torch.zeros_like(pad)), (name, b)     # bitwise +0.0
        assert not torch.signbit(pad).any()
    return out


def test_train_boxes_against_oracle(vt):
    H, W, R = 96, 130, 64
    boxes = [(0, 0, H, W), (0, 0, 20, 30), (H - 20, W - 30, 20, 30), (0, W - 1, H, 1), (H - 1, 0, 1, W),
             (5, 7, 1, 1), (30, 40, 40, 50), (0, 0, 64, 64), (10, 20, 17, 20), (H - 64, W - 64, 64, 64)]
    params = [(0, *b, f) for b in boxes for f in (0, 1)]
    clips = [tp.synthetic_clip(2, H, W, 10 + k) for k in range(len(params))]
    _check(vt, "train boxes (edges, full frame, upsampling, 1-pixel, flips)", clips, params, 3, R, 80)


def test_train_full_size(vt):
    clips = [tp.synthetic_clip(4, 256, 455, 1), tp.synthetic_clip(3, 480, 640, 2)]
    params = [(0, 12, 100, 230, 300, 1), (0, 0, 0, 480, 640, 0)]
    _check(vt, "train 224 from Ego4D / Charades frames", clips, params, 4, 224, 256)


@pytest.mark.parametrize("HW", [(256, 455), (455, 256), (480, 640), (256, 256), (224, 224), (301, 199), (40, 900)])
def test_eval_against_oracle(vt, HW):
    H, W = HW
    clips = [tp.synthetic_clip(2, H, W, H + W)]
    _check(vt, f"eval {H}x{W}", clips, [(1, 0, 0, 0, 0, 0)], 3, 224, 256)


def test_mixed_batch_64x16(vt):
    rng = np.random.default_rng(5)
    sizes = [(64, 114), (114, 64), (120, 160), (64, 64), (56, 56), (75, 50), (20, 300)]
    F, R, cc = 16, 56, 64
    clips, params = [], []
    for b in range(64):
        H, W = sizes[b % len(sizes)]
        T = (1, F - 1, F)[b % 3]
        clips.append(tp.synthetic_clip(T, H, W, 1000 + b))
        if b % 2:
            params.append((1, 0, 0, 0, 0, 0))
        else:
            h, w = int(rng.integers(1, H + 1)), int(rng.integers(1, W + 1))
            params.append((0, int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1)), h, w, b % 4 == 0))
    _check(vt, "mixed batch B=64 F=16", clips, params, F, R, cc)


def _golden():
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "video_transforms.npz"))
    return {k: z[k] for k in z.files}


def test_same_seeds_end_to_end_match_reference_golden(vt):
    """The package's seeded draws + the kernel reproduce the reference transform's recorded outputs."""
    g = _golden()
    k, worst = 0, 0.0
    while f"case{k}:meta" in g:
        H, W, T, F, R, cc, seed = (int(v) for v in g[f"case{k}:meta"])
        frames = tp.synthetic_clip(T, H, W, seed)
        if (H, W, T) == (224, 224, 1):
            frames[:] = 0
        split = "train" if g[f"case{k}:params"][0] == 0 else "test"
        torch.manual_seed(seed)
        random.seed(seed)
        item = vt.init_video_transform_dict(input_res=R, center_crop=cc)[split](frames)
        assert tuple(item["params"]) == tuple(int(v) for v in g[f"case{k}:params"])
        out = vt.apply_video_transform(vt.collate_video_clips([{"video": item}])["video"], F, input_res=R,
                                       center_crop=cc)
        flat = out.reshape(-1).cpu().numpy()
        idx, val = g[f"case{k}:idx"], g[f"case{k}:val"]
        err = np.abs(flat[idx].astype(np.float64) - val).max()
        worst = max(worst, err)
        assert err <= TOL, (k, err)
        assert (flat[T * (flat.size // F):] == 0).all()
        k += 1
    _note("reference golden (seeded draws + kernel)", worst)
    assert k >= 20


def test_bitwise_reproducible(vt):
    clips = [tp.synthetic_clip(3, 480, 640, 3), tp.synthetic_clip(2, 256, 455, 4)]
    params = [(1, 0, 0, 0, 0, 0), (0, 3, 50, 200, 260, 1)]
    a, _ = _run(vt, clips, params, 4, 224, 256)
    b, _ = _run(vt, clips, params, 4, 224, 256)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_writes_nothing_outside_the_output(vt):
    from egovlp_b200 import ops
    clips = [tp.synthetic_clip(2, 70, 90, 6), tp.synthetic_clip(1, 50, 40, 7)]
    params = [(0, 3, 4, 40, 50, 1), (1, 0, 0, 0, 0, 0)]
    packed = _batch(vt, clips, params)
    B, F, R, G = 2, 3, 40, 4096
    n = B * F * 3 * R * R
    buf = torch.full((n + 2 * G,), 12345.0, device="cuda")
    frames = packed["frames"].cuda()
    desc = torch.from_numpy(packed["desc"]).cuda()
    mean = (C.c_float * 3)(*tp.MEAN)
    std = (C.c_float * 3)(*tp.STD)
    ops.call("egovlp_video_transform", ops._ptr(frames), C.c_longlong(frames.numel()), ops._ptr(desc), B, F, R, 48,
             mean, std, C.c_void_p(buf.data_ptr() + 4 * G), ops._stream())
    torch.cuda.synchronize()
    assert (buf[:G] == 12345.0).all() and (buf[G + n:] == 12345.0).all()
    out = buf[G:G + n].view(B, F, 3, R, R)
    assert not (out == 12345.0).any()
    ref = tp.transform_batch(clips, params, F, R, 48)
    assert np.abs(out.cpu().double().numpy() - ref).max() <= TOL


def test_invalid_descriptors_raise(vt):
    from egovlp_b200 import ops
    from egovlp_b200._lib import EgovlpError
    clip = tp.synthetic_clip(2, 30, 40, 8)
    packed = _batch(vt, [clip], [(0, 0, 0, 30, 40, 0)])
    frames = packed["frames"].cuda()
    good = packed["desc"]

    def run(desc, F=4, R=32, cc=36, buf=frames):
        return ops.video_transform(buf, desc, F, R, cc, tp.MEAN, tp.STD)

    run(good)
    for col, val in [(5, -1), (6, 1), (7, 31), (8, 0), (7, 0), (2, 0), (3, 0), (1, 5), (1, 0), (0, 1), (0, -1),
                     (4, 2), (2, 70000)]:
        d = good.copy()
        d[0, col] = val
        with pytest.raises(EgovlpError):
            run(d)
    with pytest.raises(EgovlpError):
        run(good, buf=frames[:-1].contiguous())                  # clip extends past the buffer
    eval_big = good.copy()
    eval_big[0, :5] = (0, 1, 30, 40, 1)
    run(eval_big, cc=36)
    with pytest.raises(EgovlpError):
        run(eval_big, cc=2)                                      # 15x down-scale: more taps than the kernel holds
    with pytest.raises(EgovlpError):
        run(good, R=1000)
    with pytest.raises(EgovlpError):
        run(good[:, :9])


def test_patch_im2col_of_gpu_and_host_transformed_frames_agree(vt):
    """The model's first op sees the same bf16 patches from the GPU transform as from the reference's host-transformed
    fp32 frames (torchvision's ops on the `.float() / 255` frames, with the same drawn parameters): equal, or one bf16
    ulp apart where the two fp32 values straddle a bf16 rounding boundary, or (for values within 1e-5 of zero) within
    the fp32 absolute error."""
    pytest.importorskip("torchvision")
    from egovlp_b200 import ops
    clips = [tp.synthetic_clip(4, 256, 455, 11), tp.synthetic_clip(3, 480, 640, 12), tp.synthetic_clip(2, 224, 224, 13)]
    params = [(0, 10, 80, 240, 320, 1), (1, 0, 0, 0, 0, 0), (1, 0, 0, 0, 0, 0)]
    F, R, P = 4, 224, 16
    gpu, _ = _run(vt, clips, params, F, R, 256)
    host = torch.stack([tp.host_transform_clip(c, p, F, R, 256) for c, p in zip(clips, params)]).cuda()
    err = (gpu - host).abs().max().item()
    _note("against torchvision's host-transformed fp32 frames", err)
    assert err <= TOL
    S, K = 1 + F * (R // P) ** 2, 3 * P * P
    pa = torch.empty(len(clips) * S, K, dtype=torch.bfloat16, device="cuda")
    pb = torch.empty_like(pa)
    ops.patch_im2col(gpu.contiguous(), pa, P)
    ops.patch_im2col(host.contiguous(), pb, P)
    def ordered(x):                               # bf16 bits -> integers in value order (ulp distance = difference)
        b = x.view(torch.int16).int()
        return torch.where(b < 0, -(b & 0x7FFF), b)
    d = (ordered(pa) - ordered(pb)).abs()
    # Near zero (|v| << 1) the fp32 values differ by their absolute rounding error (~1e-7, from sums of terms of size
    # ~1), which is many bf16 ulps of the tiny result; there the patches agree to within that absolute error.
    near_zero = (pa.float() - pb.float()).abs() <= TOL
    assert bool(((d <= 1) | near_zero).all()), int(d[~near_zero].max())
    print(f"[video_transform] patch_im2col: {(d == 0).float().mean().item():.6f} equal, "
          f"{(d == 1).float().mean().item():.6f} one bf16 ulp apart, {(d > 1).float().mean().item():.2e} more "
          f"(all |v| < {TOL})")


def test_prefetcher_transform_equals_direct_call(vt):
    from egovlp_b200.data import DevicePrefetcher
    batches = []
    for n in range(3):
        clips = [tp.synthetic_clip(1 + (n + b) % 4, 100 + 10 * b, 140 - 5 * n, 40 + 10 * n + b) for b in range(3)]
        params = [(0, 1, 2, 60, 70, b % 2) if (n + b) % 2 else (1, 0, 0, 0, 0, 0) for b in range(3)]
        items = [{"video": {"frames": torch.from_numpy(c), "params": p}, "idx": torch.tensor(b)}
                 for b, (c, p) in enumerate(zip(clips, params))]
        batches.append(vt.collate_video_clips(items))
    for b in batches:
        b["video"]["frames"] = b["video"]["frames"].pin_memory()
    tsfm = vt.DeviceVideoTransform(4, input_res=64, center_crop=72)
    got = [(b["video"].clone(), b["idx"].clone()) for b in DevicePrefetcher(batches, "cuda", transform=tsfm)]
    for (v, i), b in zip(got, batches):
        want = vt.apply_video_transform(b["video"], 4, input_res=64, center_crop=72)
        assert torch.equal(v.view(torch.int32), want.view(torch.int32))
        assert torch.equal(i.cpu(), b["idx"])
    plain = [b for b in DevicePrefetcher(batches, "cuda")]
    assert plain[0]["video"]["frames"].is_cuda and plain[0]["video"]["frames"].dtype == torch.uint8
