"""Per-form timing of the GEMM calls one video block (SpaceTimeBlockFn) makes at the headline step's size.

    python tools/bench_gemm.py [--M 100384] [--iters 20] [--json out.json] [--wgrad-decomp]

cfg3 = 32 clips x (1 + 16 x 196) tokens = 100,384 rows.  Every call of engine.py's forward and input-gradient GEMMs is
timed with CUDA events, with the same dtypes, epilogue arguments and b_mn flags, plus the weight gradients with
engine._split_for's split.  A form that reads or writes more than one bf16 output's worth of epilogue bytes is also timed
with the plain bf16 epilogue on the same A.B: the difference is what its epilogue costs on top.  Each specialised form is
checked bit for bit against the generic epilogue (EGOVLP_GEMM_GENERIC_EPI=1) at this size.  The block's six weight
gradients are summed with their TFLOP/s; --wgrad-decomp also times each of them without the fused bias gradient,
through the K-major form on transposed copies (the operand path's share) and at the splits around the engine's choice.
EGOVLP_B200_LIB=<path> runs another build of the library (A/B comparisons)."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egovlp_b200 import engine, ops  # noqa: E402

D, HID = 768, 3072
BF16, F32 = torch.bfloat16, torch.float32


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unavailable"
    except (OSError, subprocess.TimeoutExpired):
        return "unavailable"


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--M", type=int, default=32 * (1 + 16 * 196))
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--wgrad-decomp", action="store_true",
                    help="also time each weight gradient without the bias gradient, through the K-major form on "
                         "transposed copies, and at the splits around the engine's choice")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gemm.py measures on the GPU"
    M, dev = args.M, "cuda"
    g = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape, dt=BF16, scale=0.05):
        return (torch.randn(*shape, device=dev, generator=g) * scale).to(dt)

    x768, x3072 = rnd(M, D, scale=1.0), rnd(M, HID, scale=1.0)
    dy768, dy2304, dy3072 = rnd(M, D, scale=1.0), rnd(M, 3 * D, scale=1.0), rnd(M, HID, scale=1.0)
    w_qkv, w_proj, w_fc1, w_fc2 = rnd(3 * D, D), rnd(D, D), rnd(HID, D), rnd(D, HID)
    b_qkv, b_proj, b_fc1, b_fc2 = (rnd(n, dt=F32) for n in (3 * D, D, HID, D))
    res = rnd(M, D, dt=F32, scale=1.0)
    u = rnd(M, HID, scale=1.0)
    sms = engine._sm_count(torch.cuda.current_device())

    # (name, calls per block, A, B, out shape/dtype, gemm kwargs, epilogue HBM bytes, specialised)
    def fwd(name, n, a, w, out_dt, kw, ebytes):
        return (name, n, a, w, (M, w.shape[0]), out_dt, kw, ebytes, True)

    def dgrad(name, n, a, w, out_dt, kw, ebytes):
        return (name, n, a, w, (M, w.shape[1]), out_dt, dict(kw, b_mn=True), ebytes, True)

    forms = [
        fwd("qkv fwd (bias, q-scale -> bf16)", 2, x768, w_qkv, BF16,
            dict(bias=b_qkv, col_scale=0.125, col_scale_ncols=D), M * 3 * D * 2),
        fwd("proj fwd (bias + fp32 residual)", 2, x768, w_proj, F32, dict(bias=b_proj, residual=res), M * D * 8),
        fwd("fc1 fwd (GELU, GELU')", 1, x768, w_fc1, BF16, dict(bias=b_fc1, act=3, out2="out2"), M * HID * 4),
        fwd("fc2 fwd (bias + fp32 residual)", 1, x3072, w_fc2, F32, dict(bias=b_fc2, residual=res), M * D * 8),
        dgrad("fc2 dgrad (x GELU')", 1, dy768, w_fc2, BF16, dict(aux=u, act=4), M * HID * 4),
        dgrad("fc1 dgrad", 1, dy3072, w_fc1, BF16, {}, M * D * 2),
        dgrad("proj dgrad", 2, dy768, w_proj, BF16, {}, M * D * 2),
        dgrad("qkv dgrad", 2, dy2304, w_qkv, BF16, {}, M * D * 2),
    ]
    rows, report = [], {"gpu": gpu_info(), "M": M, "lib": os.environ.get("EGOVLP_B200_LIB") or "in-tree",
                        "forms": []}
    surcharge_block, ms_block, mismatches = 0.0, 0.0, []
    for name, n, a, w, shape, out_dt, kw, ebytes, _ in forms:
        out = torch.empty(*shape, device=dev, dtype=out_dt)
        kw = dict(kw)
        if kw.get("out2") == "out2":
            kw["out2"] = torch.empty(*shape, device=dev, dtype=BF16)
        call = lambda: ops.gemm(a, w, out, **kw)  # noqa: E731
        ms = timed(call, args.iters)
        flop = 2.0 * M * shape[1] * a.shape[1]
        plain_ms = None
        if ebytes > M * shape[1] * 2:
            o16 = torch.empty(*shape, device=dev, dtype=BF16)
            plain = dict(b_mn=True) if kw.get("b_mn") else {}
            plain_ms = timed(lambda: ops.gemm(a, w, o16, **plain), args.iters)
            surcharge_block += n * (ms - plain_ms)
        ms_block += n * ms
        # bit-identical to the generic epilogue at this size
        os.environ["EGOVLP_GEMM_GENERIC_EPI"] = "1"
        call()
        ref = [out.clone()] + ([kw["out2"].clone()] if "out2" in kw else [])
        os.environ["EGOVLP_GEMM_GENERIC_EPI"] = "0"
        out.fill_(float("nan"))
        call()
        got = [out] + ([kw["out2"]] if "out2" in kw else [])
        same = all(torch.equal(r, q) for r, q in zip(ref, got))
        if not same:
            mismatches.append(name)
        rows.append((name, n, ms, flop / ms / 1e9, ebytes / 1e6, plain_ms, same))
        report["forms"].append(dict(name=name, calls_per_block=n, ms=ms, tflops=flop / ms / 1e9, epilogue_mb=ebytes / 1e6,
                                    plain_bf16_ms=plain_ms, bitwise_equal_generic=same))
    os.environ.pop("EGOVLP_GEMM_GENERIC_EPI", None)
    # weight gradients (MN-major dy and x, split-K fp32 adds into dW), the engine's split rule
    wgrad_block, decomp = 0.0, []
    for name, n, dy, x, n_out, n_in, colsum in [("fc2 wgrad", 1, dy768, x3072, D, HID, False),
                                                ("fc1 wgrad (+ bias grad)", 1, dy3072, x768, HID, D, True),
                                                ("proj wgrad", 2, dy768, x768, D, D, False),
                                                ("qkv wgrad (+ bias grad)", 2, dy2304, x768, 3 * D, D, True)]:
        split = engine._split_for(n_out, n_in, M, sms)
        dw = torch.zeros(n_out, n_in, device=dev, dtype=F32)
        db = torch.zeros(n_out, device=dev, dtype=F32) if colsum else None
        ms = timed(lambda: ops.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=split, colsum_a=db),
                   args.iters)
        flop = 2.0 * M * n_out * n_in
        ms_block += n * ms
        wgrad_block += n * ms
        rows.append((f"{name} split {split}", n, ms, flop / ms / 1e9, n_out * n_in * 4 / 1e6, None, None))
        report["forms"].append(dict(name=name, split=split, calls_per_block=n, ms=ms, tflops=flop / ms / 1e9))
        if args.wgrad_decomp:
            # where the wgrad time goes: without the fused bias gradient; the same product through the K-major form
            # (transposed copies made here, outside the timed region; the forward / dgrad operand path) at the same
            # split; and the MN/MN form at the splits around the engine's choice (wave fill, flush count)
            d = dict(name=name, split=split)
            mn = lambda s: lambda: ops.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=s)  # noqa: E731
            d["no_colsum_ms"] = timed(mn(split), args.iters)
            dyt, xt = dy.t().contiguous(), x.t().contiguous()
            d["kmajor_ms"] = timed(lambda: ops.gemm(dyt, xt, dw, accumulate=True, split_k=split), args.iters)
            del dyt, xt
            d["splits_ms"] = {s: timed(mn(s), args.iters) for s in range(max(1, split - 3), split + 4)}
            decomp.append(d)
    report["wgrad_decomposition"] = decomp

    print(f"GPU: {report['gpu']}   (name, power limit, SM clock, max SM clock)")
    print(f"M = {M}, library: {report['lib']}")
    print(f"{'form':40s} {'x/blk':>5s} {'ms':>8s} {'TFLOP/s':>8s} {'epi MB':>8s} {'plain ms':>9s} {'surcharge':>9s}  bitwise")
    for name, n, ms, tf, mb, plain_ms, same in rows:
        pl = f"{plain_ms:9.3f}" if plain_ms is not None else " " * 9
        sc = f"{ms - plain_ms:9.3f}" if plain_ms is not None else " " * 9
        eq = "" if same is None else ("yes" if same else "NO")
        print(f"{name:40s} {n:5d} {ms:8.3f} {tf:8.1f} {mb:8.1f} {pl} {sc}  {eq}")
    print(f"per block: GEMMs {ms_block:.3f} ms, epilogue surcharge {surcharge_block:.3f} ms; "
          f"x 12 blocks: {12 * ms_block:.1f} ms, surcharge {12 * surcharge_block:.1f} ms")
    # the block's six weight gradients (qkv and proj twice, fc1, fc2) do the FLOPs of its forward GEMMs
    wgrad_flop = 2.0 * M * (2 * 3 * D * D + 2 * D * D + D * HID + HID * D)
    print(f"per block: weight gradients {wgrad_block:.3f} ms = {wgrad_flop / wgrad_block / 1e9:.1f} TFLOP/s")
    for d in decomp:
        sp = "  ".join(f"{s}:{t:.3f}" for s, t in d["splits_ms"].items())
        print(f"  {d['name']:28s} split {d['split']}: no colsum {d['no_colsum_ms']:.3f} ms, K-major operands "
              f"{d['kmajor_ms']:.3f} ms, by split  {sp}")
    report.update(block_ms=ms_block, block_surcharge_ms=surcharge_block, mismatches=mismatches,
                  wgrad_block_ms=wgrad_block, wgrad_block_tflops=wgrad_flop / wgrad_block / 1e9)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)
    if mismatches:
        sys.exit(f"specialised epilogue differs from the generic one: {mismatches}")


if __name__ == "__main__":
    main()
