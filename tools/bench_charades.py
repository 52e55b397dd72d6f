"""Charades-Ego on one GPU: the zero-shot evaluation, the metrics and the fine-tuning step, each as the reference's
trainer runs it (tools/charades_sequence.py restates trainer/trainer_charades.py call for call).

    python tools/bench_charades.py [--clips N] [--steps K] [--warmup W] [--no-eager]

  * zero-shot evaluation, clips/s: 157 class prompts plus N synthetic 16-frame clips through `_valid_epoch`'s sequence
    (prompt forward, per-batch video forward, host-side cat, host `sim_matrix`, `.numpy().T`, `charades_metrics`) at
    batch 4 (configs/eval/charades.json) and 32, next to the same sequence on the oracle in eager PyTorch on the same
    GPU (fp32 and bf16 autocast);
  * metric time: `charades_metrics` ([N, 157] scores) and `t2v_metrics` ([N, N] similarities) from host numpy arrays,
    on the GPU kernels and in the reference's numpy algorithm on the host (oracle/eval_port.py), N = 1000 and 10000;
  * fine-tuning step, clips/s: the trainer's step (model(data) -> gather -> sim_matrix -> NormSoftmaxLoss -> backward ->
    fused AdamW -> loss.item()) at batch 4 and 32, timed between CUDA events after the warm-up steps.

Prints ONE JSON line, with the card name, power limit and median SM clock of each timed GPU section.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (SM clock sampler of the headline benchmark)
from tools.bench_finetune import card, timed  # noqa: E402

FRAMES, N_CLASSES, PROMPT_LEN, TEXT_LEN = 16, 157, 12, 16
VIDEO = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": FRAMES, "pretrained": True,
         "time_init": "zeros"}
TEXT = {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"}


def model(device):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.model import FrozenInTime
    net = FrozenInTime(VIDEO, TEXT)
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=FRAMES), seed=0))
    return net.to(device)


def eval_inputs(clips, batch):
    from egovlp_b200 import synthetic as syn
    prompts = syn.synthetic_text(N_CLASSES, PROMPT_LEN, seed=1, ragged=True)
    rng = np.random.default_rng(2)
    batches = []
    for b0 in range(0, clips, batch):
        b = min(batch, clips - b0)
        target = torch.from_numpy((rng.random((b, N_CLASSES)) < 0.05).astype(np.float32))
        batches.append({"video": syn.synthetic_video(b, FRAMES, seed=b0), "target": target,
                        "text": syn.synthetic_text(b, TEXT_LEN, seed=b0, ragged=True)})
    return prompts, batches


def sampled(fn, device):
    """fn() under the SM clock sampler -> (fn's result, clocks)."""
    s = bench.ClockSampler(device.index)
    s.start()
    out = fn()
    return out, s.stop()


def zero_shot_ours(net, clips, batch, device):
    from egovlp_b200.model import metric
    from egovlp_b200.model.model import sim_matrix
    from tools.charades_sequence import valid_epoch
    prompts, batches = eval_inputs(clips, batch)
    dummy = torch.zeros(1, 4, 3, 224, 224)
    valid_epoch(net, prompts, batches[:1], device, sim_matrix, [metric.charades_metrics], dummy)      # warm-up
    torch.cuda.synchronize()

    def run():
        t0 = time.perf_counter()
        valid_epoch(net, prompts, batches, device, sim_matrix, [metric.charades_metrics], dummy)
        return time.perf_counter() - t0

    sec, clocks = sampled(run, device)
    return {"batch": batch, "clips": clips, "clips_per_s": clips / sec, "wall_s": sec,
            "sm_clock_mhz_median": clocks.get("sm_mhz"), "throttle_reasons": clocks.get("reasons")}


def zero_shot_eager(clips, batch, device, autocast):
    """The same sequence on the oracle's towers in eager PyTorch (torch.no_grad), then the reference's numpy metric."""
    from egovlp_b200 import synthetic as syn
    from oracle import eval_port as ep, reference_port as rp
    torch.backends.cuda.matmul.allow_tf32 = False
    p = {k: v.to(device) for k, v in syn.seeded_state_dict(syn.model_dims(num_frames=FRAMES), seed=0).items()}
    prompts, batches = eval_inputs(clips, batch)

    def run():
        t0 = time.perf_counter()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            text = rp.compute_text({k: v.to(device) for k, v in prompts.items()}, p).float().cpu()
            vids, targets = [], []
            for b in batches:
                vids.append(rp.compute_video(b["video"].to(device), p).float().cpu())
                targets.append(b["target"])
        sims = rp.sim_matrix(text, torch.cat(vids)).numpy().T
        ep.charades_metrics(sims, torch.cat(targets).numpy())
        return time.perf_counter() - t0

    try:
        run()
        sec = run()
    except torch.cuda.OutOfMemoryError:
        sec = None
    del p
    torch.cuda.empty_cache()
    return None if sec is None else {"clips_per_s": clips / sec, "wall_s": sec}


def metric_times(device, repeats=5):
    from egovlp_b200.model import metric
    from oracle import eval_port as ep
    out = {}
    for n in (1000, 10000):
        rng = np.random.default_rng(n)
        scores = (0.1 * rng.standard_normal((n, N_CLASSES))).astype(np.float32)
        gt = (rng.random((n, N_CLASSES)) < 0.05).astype(np.float32)
        sims = (0.1 * rng.standard_normal((n, n)) + 0.2 * np.eye(n)).astype(np.float32)
        row = {}
        for name, fn, ofn, args in (("charades_metrics", metric.charades_metrics, ep.charades_metrics, (scores, gt)),
                                    ("t2v_metrics", metric.t2v_metrics, ep.t2v_metrics, (sims,))):
            fn(*args)                                                                        # warm-up
            gpu = []
            for _ in range(repeats):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(*args)                                                                    # ends on host values
                gpu.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            ofn(*args)
            host = time.perf_counter() - t0
            row[name] = {"gpu_ms_median": statistics.median(gpu) * 1e3, "host_numpy_ms": host * 1e3}
        out[f"N={n}"] = row
    return out


def finetune_step(net, batch, steps, warmup, device):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.loss import NormSoftmaxLoss
    from egovlp_b200.model.model import sim_matrix
    from egovlp_b200.optim import AdamW
    from tools.charades_sequence import train_step
    net.train()
    opt = AdamW(net.parameters(), lr=3e-5)
    loss_fn = NormSoftmaxLoss()
    host = {"video": syn.synthetic_video(batch, FRAMES, seed=7).pin_memory(),
            "text": syn.synthetic_text(batch, TEXT_LEN, seed=7, ragged=True)}

    def step():
        return train_step(net, loss_fn, opt, host, device, sim_matrix)

    s = bench.ClockSampler(device.index)
    sec, loss = timed(step, steps, warmup, s)
    clocks = s.stop()
    return {"batch": batch, "clips_per_s": batch / sec, "step_ms": sec * 1e3, "loss": loss,
            "sm_clock_mhz_median": clocks.get("sm_mhz"), "throttle_reasons": clocks.get("reasons")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=256, help="synthetic 16-frame clips of the zero-shot evaluation")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-eager", action="store_true", help="skip the eager PyTorch comparison")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_charades.py measures the CUDA path: no CUDA device")
    device = torch.device("cuda", torch.cuda.current_device())
    t0 = time.time()
    net = model(device)
    line = {"frames": FRAMES, "classes": N_CLASSES, "zero_shot": {}, "finetune": {}}
    for batch in (4, 32):
        line["zero_shot"][f"b{batch}"] = zero_shot_ours(net, args.clips, batch, device)
    for batch in (4, 32):
        line["finetune"][f"b{batch}"] = finetune_step(net, batch, args.steps, max(3, args.warmup), device)
    del net
    torch.cuda.empty_cache()
    if not args.no_eager:
        line["zero_shot"]["eager_pytorch_same_gpu"] = {
            f"b{batch}": {mode: zero_shot_eager(args.clips, batch, device, ac)
                          for mode, ac in (("fp32", False), ("bf16_autocast", True))}
            for batch in (4, 32)}
    line["metrics"] = metric_times(device)
    name, power = card()
    line.update({"gpu": name, "power_limit": power, "wall_s": time.time() - t0})
    print(json.dumps(line))


if __name__ == "__main__":
    main()
