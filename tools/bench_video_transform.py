"""Times egovlp_video_transform (CUDA events), the host transform it replaces (one core), the H2D bytes of both feeds,
and the cfg3 training step fed each way through DevicePrefetcher.

    python tools/bench_video_transform.py [--iters 50] [--steps 8] [--warmup 3] [--no-e2e] [--out DIR]

Kernel time: CUDA events around back-to-back raw `egovlp_video_transform` launches on device-resident frames and
descriptor table, so the binding's host work (table checks, table copy, allocation) is not in it; `op_ms` is the same
through `transforms.apply_video_transform`, host work included.

Bytes model (the least HBM traffic the kernel needs): the source pixels its weights touch (train: the crop box; eval:
the rows / columns the composed resize reads), uint8, once, plus the fp32 output once, 12 R^2 bytes per output frame.
Share of the HBM bound = (bytes / 3.35 TB/s, H100 SXM data sheet) / kernel time.  H2D bytes count whole frames.

End to end: the cfg3 step (FrozenInTime 16 x 224^2 + DistilBERT L = 16 + EgoNCE + AdamW, batch 32, seeded weights, as
`bench.py`) fed through `DevicePrefetcher` by (a) host-transformed pinned fp32 [32, 16, 3, 224, 224] frames and (b) the
raw pinned uint8 256x455 frames + `DeviceVideoTransform` on the copy stream; the legs alternate, twice each.  The host
transform's own cost is not in (a); it is the per-clip one-core figure.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egovlp_b200 import ops  # noqa: E402
from egovlp_b200 import transforms as vt  # noqa: E402
from oracle import transform_port as tp  # noqa: E402

HBM = 3.35e12
R, CC = 224, 256
# name, clips, frames, (H, W), split
CASES = [("cfg3 train (Ego4D 256x455)", 32, 16, (256, 455), "train"),
         ("Charades train 480x640, B=4", 4, 16, (480, 640), "train"),
         ("Charades train 480x640, B=32", 32, 16, (480, 640), "train"),
         ("EgoMCQ test (Ego4D 256x455)", 32, 16, (256, 455), "test")]
STEP_RATES = {"cfg3 at 112 clips/s": 112, "cfg3 at 175 clips/s": 175, "cfg2 at 488 clips/s": 488}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def packed_batch(B, F, HW, split, seed=0):
    torch.manual_seed(seed)
    tsfm = vt.init_video_transform_dict(input_res=R, center_crop=CC)[split]
    items = [{"video": tsfm(tp.synthetic_clip(F, *HW, seed + b))} for b in range(B)]
    packed = vt.collate_video_clips(items)["video"]
    packed["frames"] = packed["frames"].pin_memory()
    return packed


def kernel_bytes(packed, F):
    """Source bytes the kernel's weights touch + output bytes (module docstring)."""
    src = 0
    for off, T, H, W, *params in packed["desc"].tolist():
        wy, wx = tp.clip_weights(H, W, params, R, CC)
        src += T * int((wy != 0).any(0).sum()) * int((wx != 0).any(0).sum()) * 3
    return src + len(packed["desc"]) * F * 12 * R * R


def events_ms(fn, iters):
    for _ in range(5):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def time_kernel(packed, F, iters):
    frames = packed["frames"].cuda()
    desc = torch.from_numpy(packed["desc"]).cuda()
    B = desc.shape[0]
    out = torch.empty(B, F, 3, R, R, device="cuda")
    mean, std = (C.c_float * 3)(*tp.MEAN), (C.c_float * 3)(*tp.STD)
    args = (ops._ptr(frames), C.c_longlong(frames.numel()), ops._ptr(desc), B, F, R, CC, mean, std, ops._ptr(out),
            ops._stream())
    kernel = events_ms(lambda: ops.call("egovlp_video_transform", *args), iters)
    dev = {"frames": frames, "desc": packed["desc"]}
    op = events_ms(lambda: vt.apply_video_transform(dev, F), iters)
    return kernel, op


def host_ms_per_clip(HW, F, params, reps=3):
    try:
        import torchvision  # noqa: F401
    except ImportError:
        return None
    u8 = tp.synthetic_clip(F, *HW, 1)
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        tp.host_transform_clip(u8, params, F, R, CC)
        best = min(best, time.perf_counter() - t0)
    torch.set_num_threads(threads)
    return best * 1e3


def e2e(steps, warmup, B=32, T=16, L=16):
    """clips/s of the cfg3 step fed host-transformed fp32 vs raw uint8 + the GPU transform (module docstring)."""
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.data import DevicePrefetcher
    from egovlp_b200.distributed import egoclip_step_loss
    from egovlp_b200.model.loss import EgoNCE
    from egovlp_b200.model.model import FrozenInTime
    from egovlp_b200.optim import AdamW
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": T,
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=T), seed=0), strict=True)
    net.to(dev)
    loss_fn, opt = EgoNCE(), AdamW(net.parameters(), lr=3e-5)
    txt = syn.synthetic_text(B, L, seed=0)
    verb, noun = syn.synthetic_tags(B, seed=0)
    rest = {"text": {"input_ids": txt["input_ids"].pin_memory(), "attention_mask": txt["attention_mask"].pin_memory()},
            "verb_vec": verb.pin_memory(), "noun_vec": noun.pin_memory()}
    packed = packed_batch(B, T, (256, 455), "train", seed=3)
    host_fp32 = torch.stack([tp.host_transform_clip(packed["frames"].numpy()[o:o + t * h * w * 3].reshape(t, h, w, 3),
                                                    p, T, R, CC)
                             for o, t, h, w, *p in packed["desc"].tolist()]).pin_memory()
    feeds = {"host-transformed fp32": ({**rest, "video": host_fp32}, None),
             "raw uint8 + GPU transform": ({**rest, "video": packed}, vt.DeviceVideoTransform(T))}

    def step(data):
        opt.zero_grad(set_to_none=True)
        loss = egoclip_step_loss(net, loss_fn, data)
        loss.backward()
        opt.step()
        return loss.item()

    def run(name):
        batch, tsfm = feeds[name]
        it = iter(DevicePrefetcher((batch for _ in range(warmup + steps)), dev, transform=tsfm))
        for _ in range(warmup):
            step(next(it))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            step(next(it))                                  # loss.item(): the step ends in a device synchronise
        return B * steps / (time.perf_counter() - t0)

    res = {name: [] for name in feeds}
    for _ in range(2):
        for name in feeds:
            res[name].append(run(name))
    h2d_rest = sum(t.numel() * t.element_size() for t in (*rest["text"].values(), rest["verb_vec"], rest["noun_vec"]))
    return {name: {"clips_per_s": v, "h2d_bytes_per_step": h2d_rest + (host_fp32.numel() * 4 if "fp32" in name
                                                                        else packed["frames"].numel())}
            for name, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    res = {"card": card(), "cases": []}
    print(res["card"])
    for name, B, F, HW, split in CASES:
        packed = packed_batch(B, F, HW, split)
        kernel_ms, op_ms = time_kernel(packed, F, a.iters)
        nbytes = kernel_bytes(packed, F)
        host = host_ms_per_clip(HW, F, packed["desc"][0, 4:].tolist())
        row = {"case": name, "kernel_ms": kernel_ms, "op_ms": op_ms, "kernel_bytes_MB": nbytes / 1e6,
               "GB/s": nbytes / kernel_ms / 1e6, "hbm_share": nbytes / HBM * 1e3 / kernel_ms,
               "h2d_uint8_MB": packed["frames"].numel() / 1e6, "h2d_fp32_224_MB": B * F * 12 * R * R / 1e6,
               "host_ms_per_clip_1core": host,
               "host_cores_needed": None if host is None else {k: host * r / 1e3 for k, r in STEP_RATES.items()}}
        res["cases"].append(row)
        print(json.dumps(row))
    if not a.no_e2e:
        res["e2e_cfg3"] = e2e(a.steps, a.warmup)
        print(json.dumps({"e2e_cfg3": res["e2e_cfg3"]}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_video_transform.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
