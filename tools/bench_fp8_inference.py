"""bf16 vs fp8 (e4m3) inference of the video tower (`set_inference_precision`), alternated in one process:

  * cfg5: the EgoMCQ step of bench.py --workload cfg5 (640 clips x 4 frames through the towers + scoring);
  * dense: `dense_video_features` over a long synthetic clip, 16-frame windows, batch 64;
  * the GEMM forms the flag switches (timeattn.qkv / attn.qkv: N = 2304, mlp.fc1: N = 3072, K = 768), bf16 vs e4m3,
    at both workloads' token counts M (CUDA events, TFLOP/s from the shapes).

Each end-to-end pair runs bf16 then fp8 `--pairs` times; every call is timed with CUDA events after a warm-up of both
modes.  Also reported: how far the fp8 outputs are from the bf16 ones, the card name, power limit and median SM clock of
the run.  Seeded synthetic weights and inputs."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
warnings.simplefilter("ignore")

import bench  # noqa: E402  (SM clock sampler of the headline benchmark)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().split(",")[:2]]
        return name, power
    except (OSError, ValueError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(), None


def event_ms(fn, reps=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def gemm_forms(M, reps):
    from egovlp_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    K = 768
    x = torch.randn(M, K, generator=g, device="cuda")
    a16 = x.to(torch.bfloat16)
    a8, sa = ops.quantize_rows_e4m3(x)
    del x
    res = {}
    for name, N, act in (("qkv", 2304, 0), ("fc1", 3072, 1)):
        w = torch.randn(N, K, generator=g, device="cuda") * 0.02
        bias = torch.zeros(N, device="cuda")
        w16 = w.to(torch.bfloat16)
        w8, sw = ops.quantize_rows_e4m3(w)
        out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        kw = dict(col_scale=0.125, col_scale_ncols=768) if act == 0 else {}
        f16 = lambda: ops.gemm(a16, w16, out, bias=bias, act=act, **kw)            # noqa: E731
        f8 = lambda: ops.gemm_e4m3(a8, sa, w8, sw, out, bias=bias, act=act, **kw)  # noqa: E731
        for f in (f16, f8):
            event_ms(f, 3)
        t16, t8 = [], []
        for _ in range(3):                                  # alternated
            t16.append(event_ms(f16, reps)[0])
            t8.append(event_ms(f8, reps)[0])
        flop = 2.0 * M * N * K
        m16, m8 = statistics.median(t16), statistics.median(t8)
        res[name] = {"M": M, "N": N, "K": K, "bf16_ms": m16, "e4m3_ms": m8, "bf16_tflops": flop / m16 / 1e9,
                     "e4m3_tflops": flop / m8 / 1e9, "speedup": m16 / m8}
        del out, w, w16, w8
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=5, help="alternated bf16 / fp8 pairs per workload")
    ap.add_argument("--dense-frames", type=int, default=16 * 64 * 2, help="frames of the synthetic dense-feature clip")
    ap.add_argument("--gemm-reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_inference.py measures the CUDA path: no CUDA device")
    from egovlp_b200 import features, synthetic as syn
    from egovlp_b200.model.metric import egomcq_predict
    from egovlp_b200.model.model import FrozenInTime
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 16,
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=16), seed=0), strict=True)
    net.to(dev).eval()
    net.set_device(dev)
    tower = net.video_model

    B, T, L = 640, 4, 16
    txt = syn.synthetic_text(B // 5, L, seed=0)
    data = {"video": syn.synthetic_video(B, T, seed=0).to(dev),
            "text": {"input_ids": txt["input_ids"].to(dev), "attention_mask": txt["attention_mask"].to(dev)}}

    def cfg5():
        with torch.no_grad():
            t, v = net(data)
            return egomcq_predict(t, v.view(t.shape[0], 5, -1))

    frames = syn.synthetic_video(1, args.dense_frames, seed=1)[0]

    def dense():
        return features.dense_video_features(net, frames, 16, batch=64)

    line = {"tool": "tools/bench_fp8_inference.py", "pairs": args.pairs}
    sampler = bench.ClockSampler(dev.index)
    t0 = time.time()
    for name, fn, clips in (("cfg5", cfg5, B), ("dense16_b64", dense, args.dense_frames // 16)):
        outs = {}
        for mode in ("bf16", "fp8"):                        # warm-up (and weight quantisation) of both modes
            tower.set_inference_precision(mode)
            outs[mode] = event_ms(fn)[1]
        times = {"bf16": [], "fp8": []}
        if name == "cfg5":
            sampler.start()
        for _ in range(args.pairs):
            for mode in ("bf16", "fp8"):
                tower.set_inference_precision(mode)
                times[mode].append(event_ms(fn)[0])
        tower.set_inference_precision("bf16")
        m16, m8 = statistics.median(times["bf16"]), statistics.median(times["fp8"])
        entry = {"clips": clips, "bf16_ms": times["bf16"], "fp8_ms": times["fp8"], "bf16_clips_per_s": clips / m16 * 1e3,
                 "fp8_clips_per_s": clips / m8 * 1e3, "speedup_median": m16 / m8,
                 "fp8_faster_in_every_pair": all(b > f for b, f in zip(times["bf16"], times["fp8"]))}
        if name == "cfg5":
            (s16, p16), (s8, p8) = outs["bf16"], outs["fp8"]
            entry.update({"max_abs_score_diff": (s16 - s8).abs().max().item(),
                          "argmax_agree": (p16 == p8).float().mean().item()})
        else:
            entry["feature_rel_l2_vs_bf16"] = rel(outs["fp8"], outs["bf16"])
        line[name] = entry
    clocks = sampler.stop()
    del data
    torch.cuda.empty_cache()
    line["gemm"] = {"cfg5_M": gemm_forms(B * (1 + T * 196), args.gemm_reps),
                    "dense_M": gemm_forms(64 * (1 + 16 * 196), args.gemm_reps)}
    name, power = card()
    line.update({"gpu": name, "power_limit": power, "sm_clock_mhz_median": clocks.get("sm_mhz"),
                 "sm_clock_max_mhz": clocks.get("sm_max_mhz"), "throttle_reasons": clocks.get("reasons"),
                 "wall_s": time.time() - t0})
    print(json.dumps(line))


if __name__ == "__main__":
    main()
