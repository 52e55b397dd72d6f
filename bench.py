"""Headline benchmark: clips/sec of the TimeSformer-B + DistilBERT dual-encoder step on H100.

    python bench.py --gpus N --steps K --warmup W [--workload cfg3]      (N > 1: launched by torch.distributed.run)
    python bench.py --impl reference ...                                  (the reference algorithm on the host CPU cores)
    python bench.py ... --dump-outputs DIR                                (also write the last timed step's results)

Workloads = BASELINE.json `configs` (per-GPU shapes; weak scaling in N):
  cfg3 (default, the headline)  16f x 224^2, per-GPU batch 32, L=16, EgoNCE over G = 32 N: zero_grad -> FrozenInTime forward
                                -> ONE packed embedding/tag all-gather -> fused similarity + EgoNCE -> backward -> DDP
                                gradient all-reduce -> AdamW
  cfg2                          the same step at 4 frames (the reference's 4f pretraining shape), per-GPU batch 64
  cfg4                          EPIC-Kitchens MIR fine-tune step: 16f, per-GPU batch 32, MaxMarginRankingLoss on the gathered
                                similarity matrix (trainer/trainer_epic.py:118-131) + the 4096^2 dual-softmax rescoring
  cfg5                          EgoMCQ inference: per GPU 128 queries x 5 candidate clips x 4f through both towers, cosine
                                scoring + argmax (trainer/trainer_egoclip.py:204-215); 8 GPUs = 1024 queries per batch
Prints ONE JSON line (contract in the task statement / DESIGN.md section 7).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
warnings.simplefilter("ignore")

WORKLOADS = {
    "cfg2": dict(kind="train", frames=4, batch=64, loss="egonce",
                 metric="clips/sec, 4-frame TimeSformer-B + DistilBERT + EgoNCE training step"),
    # batch 32: the step saves ~1.45 GB of activations per 16-frame clip, so 64 clips would not fit an 80 GB H100
    "cfg3": dict(kind="train", frames=16, batch=32, loss="egonce",
                 metric="clips/sec, 16-frame TimeSformer-B + DistilBERT + EgoNCE training step"),
    "cfg4": dict(kind="train", frames=16, batch=32, loss="maxmargin",
                 metric="clips/sec, 16-frame EPIC-Kitchens MIR fine-tune step (MaxMarginRankingLoss)"),
    "cfg5": dict(kind="egomcq", frames=4, batch=640, loss=None,
                 metric="clips/sec, EgoMCQ inference (5 candidate 4-frame clips per query, cosine scoring + argmax)"),
}


# algorithmic FLOPs (SURVEY.md section 8d; multiply-add = 2)
def flops_per_clip(T, L, N=196, D=768, H=12, HID=3072, depth=12, text_layers=6):
    S = 1 + T * N
    blk = S * (2 * 2 * D * 3 * D + 2 * 2 * D * D + 2 * 2 * D * HID) + H * N * 4 * 64 * T * (T + 1) + \
        H * T * 4 * 64 * N * (N + 1) + 2 * H * 4 * 64 * S
    patch = 2 * T * N * D * D
    video = depth * blk + patch + 2 * D * 256
    text = text_layers * (L * (8 * D * D + 4 * D * HID) + H * 4 * 64 * L * L)
    return 3 * (video + text) - patch, video, text


def measured_peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        p = json.load(open(path))
        return p, "measured (MEASURED_PEAKS.json)"
    # H100 SXM data sheet (700 W board): dense bf16 989 TFLOP/s, HBM3 3.35 TB/s -- limits, not reached rates
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0}, "H100 SXM data sheet"


def host_cores():
    """CPU threads this process may really use: affinity mask capped by the cgroup CPU quota (os.cpu_count() reports
    the host's cores even inside a CPU-limited container, and oversubscribing torch threads is catastrophic)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period))))
    except (OSError, ValueError):
        try:
            quota = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            period = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if quota > 0:
                n = min(n, max(1, quota // period))
        except (OSError, ValueError):
            pass
    return max(1, min(n, 32))   # beyond ~32 threads the fp32 eager path at this size scales negatively


class ClockSampler:
    """nvidia-smi SM clock / throttle reasons sampled during the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "200", "-i", str(self.index)], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except OSError:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm = sorted(int(r[1]) for r in self.rows if len(r) >= 8 and r[1].isdigit())
        reasons = set()
        for r in self.rows:
            if len(r) >= 8:
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[4:8]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
        mx = [int(r[2]) for r in self.rows if len(r) >= 8 and r[2].isdigit()]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


# ----------------------------------------------------------------------------------------------------------------------
# baselines: the reference's algorithm (oracle port) on the host cores, and in eager PyTorch on the same GPU
# ----------------------------------------------------------------------------------------------------------------------
def _oracle_step_fn(wl, T, L, batch, device, autocast=False, seed=0):
    """One step of workload `wl` through the oracle port (torch, functional) on `device`; returns (step fn, clips/step)."""
    from oracle import reference_port as rp
    from egovlp_b200 import synthetic as syn
    dims = syn.model_dims(num_frames=max(T, 4))
    train = wl["kind"] == "train"
    params = {k: v.to(device).requires_grad_(train) for k, v in syn.seeded_state_dict(dims, seed=seed).items()}
    if train:
        opt = torch.optim.AdamW(list(params.values()), lr=3e-5, eps=1e-6, weight_decay=0.0)
        data = {"video": syn.synthetic_video(batch, T, seed=seed).to(device),
                "text": {k: v.to(device) for k, v in syn.synthetic_text(batch, L, seed=seed).items()}}
        verb, noun = [t.to(device) for t in syn.synthetic_tags(batch, seed=seed)]

        def step():
            opt.zero_grad(set_to_none=True)
            with torch.autocast(device.type, dtype=torch.bfloat16, enabled=autocast):
                t, v = rp.frozen_in_time_forward(data, params)
            x = rp.sim_matrix(t.float(), v.float())
            if wl["loss"] == "egonce":
                loss = rp.egonce_loss(x, rp.sim_matrix(verb, verb), rp.sim_matrix(noun, noun))
            else:
                loss = rp.max_margin_ranking_loss(x)
            loss.backward()
            opt.step()
            return loss.item()
        return step, batch
    q = max(1, batch // 5)
    text = {k: v.to(device) for k, v in syn.synthetic_text(q, L, seed=seed).items()}
    video = syn.synthetic_video(q * 5, T, seed=seed).to(device)

    def step():
        with torch.no_grad(), torch.autocast(device.type, dtype=torch.bfloat16, enabled=autocast):
            t = rp.compute_text(text, params)
            v = rp.compute_video(video, params)
        return rp.egomcq_predict(t.float(), v.float().view(q, 5, -1))[1].sum().item()
    return step, q * 5


def cpu_reference_rate(wl, T, L, steps, warmup):
    """The reference algorithm (oracle port, torch fp32, all host threads) on a bounded sample of the workload."""
    cores = host_cores()
    torch.set_num_threads(cores)
    batch = 2 if wl["kind"] == "train" else 5
    step, clips = _oracle_step_fn(wl, T, L, batch, torch.device("cpu"))
    for _ in range(warmup):
        step()
    t0 = time.perf_counter()
    done = 0
    while done < steps and (done == 0 or time.perf_counter() - t0 < 45.0):     # bounded: ~10-45 s of CPU work
        step()
        done += 1
    dt = time.perf_counter() - t0
    what = "fwd+bwd+AdamW" if wl["kind"] == "train" else "forward + scoring"
    return (clips * done / dt, dt / done, cores,
            f"oracle port, fp32, {clips} clips x {T}f x 224^2 + {L} tokens, {what}, {done} timed steps on {cores} threads")


def gpu_eager_baseline(wl, T, L, device, budget_s=12.0):
    """SURVEY.md 8d's "meaningful denominator": the reference's algorithm in eager PyTorch ON THIS GPU (oracle port;
    fp32 = the reference's own precision, then TF32 and bf16 autocast), a few clips, bounded time."""
    out = {"what": "oracle port (reference algorithm, eager PyTorch) on the same GPU", "unit": "clips/s"}
    batch = 8 if wl["kind"] == "train" else 40
    for mode in ("fp32", "tf32", "bf16_autocast"):
        torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
        try:
            step, clips = _oracle_step_fn(wl, T, L, batch, device, autocast=(mode == "bf16_autocast"))
            step(); step()
            torch.cuda.synchronize(device)
            t0, n = time.perf_counter(), 0
            while n < 3 or (n < 20 and time.perf_counter() - t0 < budget_s / 3):
                step()                                   # .item() inside: synchronous
                n += 1
            out[mode] = clips * n / (time.perf_counter() - t0)
        except torch.cuda.OutOfMemoryError:
            out[mode] = None
        finally:
            step = None
            torch.cuda.empty_cache()
    torch.backends.cuda.matmul.allow_tf32 = False
    out["batch"] = batch
    return out


def run_reference(args, wl):
    rank = int(os.environ.get("RANK", 0))
    if rank != 0:
        return
    steps = max(1, min(args.steps, 4))
    warm = max(1, min(args.warmup, 1))
    value, s_per_step, cores, sample = cpu_reference_rate(wl, args.frames, args.text_len, steps, warm)
    world = int(os.environ.get("WORLD_SIZE", 1))
    line = {"impl": "reference", "metric": wl["metric"], "workload": args.workload,
            "value": value, "unit": "clips/s", "n_gpus": args.gpus, "steps": steps, "warmup": warm,
            "ms_per_step": s_per_step * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic (seeded video/text/tags, seeded random-init weights)",
            "config": workload_config(args, wl, 1, cpu_sample=True),
            "cpu_baseline": {"value": value, "unit": "clips/s", "cores": cores, "kind": "port", "sample": sample},
            "e2e": {"value": value, "unit": "clips/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "note": ("ONE CPU process on rank 0 (the other ranks exit): the reference arm does not scale with --gpus"
                     if world > 1 or args.gpus > 1 else "one CPU process")}
    print(json.dumps(line), flush=True)


def workload_config(args, wl, world, cpu_sample=False):
    what = {"cfg2": "EgoClip pretraining step", "cfg3": "EgoClip pretraining step",
            "cfg4": "EPIC-Kitchens MIR fine-tune step", "cfg5": "EgoMCQ inference"}[args.workload]
    loss = {"egonce": "EgoNCE", "maxmargin": "MaxMarginRankingLoss", None: "cosine scoring + argmax"}[wl["loss"]]
    cfg = {"workload": f"{args.workload}: {what}: TimeSformer-B {args.frames}f x 224^2 p16 (divided space-time attention) "
                       f"+ DistilBERT L={args.text_len} + {loss}, per-GPU batch {args.batch}"
                       + (" [CPU arm: bounded sample of 2 clips (training) / 5 clips (inference) per step]" if cpu_sample else ""),
           "global_batch": args.batch * world, "frames": args.frames, "text_len": args.text_len,
           "parallelism": f"dp{world}",
           "l2_policy": "per-step working set (tens of GB of activations) >> 50 MB L2; no explicit flush needed"}
    if wl["kind"] == "train":
        cfg["optimizer"] = "AdamW (HF semantics) lr 3e-5"
    return cfg


def dump_outputs(path, out, net, train):
    """What the last timed step computed, as path/<name>.npy.  Training: the loss and, per parameter in named order, 4096
    entries at fixed seeded positions of the weights AdamW has just updated (5 MB in all); EgoMCQ: scores and argmax."""
    import numpy as np
    os.makedirs(path, exist_ok=True)
    if train:
        np.save(os.path.join(path, "loss.npy"), np.array([out.item()], dtype=np.float64))
        parts = []
        for i, (_, p) in enumerate(net.named_parameters()):
            idx = torch.randint(0, p.numel(), (4096,), generator=torch.Generator().manual_seed(i)).to(p.device)
            parts.append(p.detach().flatten()[idx].float().cpu())
        np.save(os.path.join(path, "weights_sample.npy"), torch.cat(parts).numpy())
    else:
        scores, pred = out
        np.save(os.path.join(path, "scores.npy"), scores.float().cpu().numpy())
        np.save(os.path.join(path, "predictions.npy"), pred.cpu().numpy().astype(np.float64))


# ----------------------------------------------------------------------------------------------------------------------
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="cfg3", choices=sorted(WORKLOADS))
    ap.add_argument("--batch", type=int, default=None, help="per-GPU clips per step (default: the workload's)")
    ap.add_argument("--frames", type=int, default=None)
    ap.add_argument("--text-len", type=int, default=16)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-gpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-ddp-comm", action="store_true", help="diagnostic: DDP no_sync (no gradient all-reduce)")
    ap.add_argument("--ddp-bf16-compress", action="store_true", help="bf16 gradient-compression DDP comm hook")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last timed step's results to DIR/<name>.npy (training: the loss "
                         "and a fixed seeded sample of the updated weights; EgoMCQ: scores and predictions)")
    ap.add_argument("--ddp-bucket-mb", type=int, default=0,
                    help="DDP bucket_cap_mb (default: EGOVLP_DDP_BUCKET_MB or 2048 = ONE gradient bucket all-reduced after "
                         "the backward; 25 = torch's default overlapped buckets)")
    args = ap.parse_args()
    wl = WORKLOADS[args.workload]
    args.batch = args.batch or wl["batch"]
    args.frames = args.frames or wl["frames"]
    if args.impl == "reference":
        return run_reference(args, wl)

    import torch.distributed as dist
    from egovlp_b200 import _lib, ops, synthetic as syn
    from egovlp_b200.distributed import AllGatherLocalGrad, egoclip_step_loss
    from egovlp_b200.model.loss import EgoNCE, MaxMarginRankingLoss
    from egovlp_b200.model.metric import egomcq_predict
    from egovlp_b200.model.model import FrozenInTime, sim_matrix
    from egovlp_b200.optim import AdamW

    world = int(os.environ.get("WORLD_SIZE", 1))
    rank = int(os.environ.get("RANK", 0))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    assert args.warmup >= 3 or args.steps <= 2, "use at least 3 warm-up steps for a reportable number"
    torch.manual_seed(0)                                     # text-tower dropout seeds: identical runs for identical args

    B, T, L = args.batch, args.frames, args.text_len
    train = wl["kind"] == "train"
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": max(T, 4),
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=max(T, 4)), seed=0), strict=True)
    net.to(dev)
    model = net
    if not train:
        net.eval()
    elif world > 1:
        # One bucket = one fp32 all-reduce (724 MB, ~2 ms over NVLink / NVSwitch) AFTER the backward: overlapped 25 MB
        # buckets make NCCL's CTAs compete with the persistent one-CTA-per-SM GEMMs of the backward (whose static tile
        # schedule then waits for the delayed SMs) and cost more than they hide -- measured, see DESIGN.md section 8.
        bucket_mb = args.ddp_bucket_mb or int(os.environ.get("EGOVLP_DDP_BUCKET_MB", "2048"))
        model = torch.nn.parallel.DistributedDataParallel(net, device_ids=[local], gradient_as_bucket_view=True,
                                                          bucket_cap_mb=bucket_mb)
        if args.ddp_bf16_compress:
            from torch.distributed.algorithms.ddp_comm_hooks import default_hooks
            model.register_comm_hook(None, default_hooks.bf16_compress_hook)
    loss_fn = EgoNCE() if wl["loss"] == "egonce" else MaxMarginRankingLoss()
    opt = AdamW(net.parameters(), lr=3e-5) if train else None

    seed = rank                                              # identical weights, per-rank data
    n_text = B if train else B // 5                          # EgoMCQ: one query text per 5 candidate clips
    txt = syn.synthetic_text(n_text, L, seed=seed)
    host = {"video": syn.synthetic_video(B, T, seed=seed).pin_memory(),
            "ids": txt["input_ids"].pin_memory(), "mask": txt["attention_mask"].pin_memory()}
    if train:
        verb_h, noun_h = syn.synthetic_tags(B, seed=seed)
        host["verb"], host["noun"] = verb_h.pin_memory(), noun_h.pin_memory()

    def batch_of(video):
        d = {"video": video, "text": {"input_ids": host["ids"], "attention_mask": host["mask"]}}
        if train:
            d["verb_vec"], d["noun_vec"] = host["verb"], host["noun"]
        return d

    def to_device(d):
        return {k: ({kk: vv.to(dev, non_blocking=True) for kk, vv in v.items()} if isinstance(v, dict)
                    else v.to(dev, non_blocking=True)) for k, v in d.items()}

    resident = to_device(batch_of(host["video"]))
    h2d_bytes = sum(t.numel() * t.element_size() for t in host.values())

    def train_step(data):
        opt.zero_grad(set_to_none=True)
        if wl["loss"] == "egonce":
            loss = egoclip_step_loss(model, loss_fn, data)
        else:                                                # trainer/trainer_epic.py:118-131
            t, v = model(data)
            loss = loss_fn(sim_matrix(AllGatherLocalGrad.apply(t), AllGatherLocalGrad.apply(v)))
        if args.no_ddp_comm and world > 1:
            with model.no_sync():
                loss.backward()
        else:
            loss.backward()
        opt.step()
        return loss

    def egomcq_step(data):
        with torch.no_grad():
            t, v = net(data)                                 # [Q, 256], [5 Q, 256]
            return egomcq_predict(t, v.view(t.shape[0], 5, -1))      # scores [Q, 5], predictions [Q]

    step = train_step if train else egomcq_step

    def result_to_host(out):
        return out.item() if train else out[1].cpu()         # loss value / the [Q] predictions

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(n, fn):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = None
        for _ in range(n):
            out = fn()
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return ms.item(), out

    for _ in range(args.warmup):
        out = step(resident)
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    _lib.reset_launch_count()
    ops.profile(True)
    ms_total, out = timed(args.steps, lambda: step(resident))
    prof = ops.profile(False)
    launches = _lib.launch_count()
    clocks = sampler.stop() if rank == 0 else None
    result = result_to_host(out)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, out, net, train)
    ms_per_step = ms_total / args.steps
    value = B * world * args.steps / (ms_total / 1e3)

    e2e = None
    if not args.no_e2e:
        from egovlp_b200.data import DevicePrefetcher

        def run_e2e(video):
            n = args.steps + 1
            it = iter(DevicePrefetcher((batch_of(video) for _ in range(n)), dev))   # every batch: pinned host -> device
            result_to_host(step(next(it)))                               # untimed first step
            ms, _ = timed(args.steps, lambda: result_to_host(step(next(it))))   # D2H read of the result every step
            return ms

        ms_e2e = run_e2e(host["video"])
        d2h = 4 if train else 8 * n_text
        e2e = {"value": B * world * args.steps / (ms_e2e / 1e3), "unit": "clips/s", "h2d_bytes_per_step": h2d_bytes,
               "d2h_bytes_per_step": d2h, "ms_per_step": ms_e2e / args.steps,
               "note": "per step: pinned-host fp32 video/ids/mask" + ("/tags" if train else "") + " -> device (one batch in "
                       "flight on a copy stream, egovlp_b200.data.DevicePrefetcher), model(data) public API, "
                       + ("loss.item()" if train else "predictions copied to the host")}
        # same step fed with uint8 frames (normalisation fused into the patch-embedding kernel): 4x fewer H2D bytes
        mean = torch.tensor(syn.IMAGENET_MEAN).view(1, 1, 3, 1, 1)
        std = torch.tensor(syn.IMAGENET_STD).view(1, 1, 3, 1, 1)
        video_u8 = ((host["video"] * std + mean).clamp(0, 1) * 255).round().to(torch.uint8).pin_memory()
        ms_u8 = run_e2e(video_u8)
        e2e["uint8_frames"] = {"value": B * world * args.steps / (ms_u8 / 1e3), "ms_per_step": ms_u8 / args.steps,
                               "h2d_bytes_per_step": h2d_bytes - host["video"].numel() * 3}

    trainer_seq = None
    if train and wl["loss"] == "egonce" and not args.no_e2e:
        # the reference trainer's literal call sequence (tools/trainer_sequence.py): blocking fp32 copies from pageable-
        # style host tensors, 4 list-API all_gathers, 3 sim_matrix launches, EgoNCE(x, sim_v, sim_n), .item() twice
        from tools.trainer_sequence import trainer_step
        hb = {"video": host["video"], "text": {"input_ids": host["ids"], "attention_mask": host["mask"]},
              "verb_vec": host["verb"], "noun_vec": host["noun"]}
        n_seq = max(2, min(args.steps, 4))
        trainer_step(model, loss_fn, opt, hb, dev, sim_matrix)
        ms_seq, loss_seq = timed(n_seq, lambda: trainer_step(model, loss_fn, opt, hb, dev, sim_matrix))
        trainer_seq = {"value": B * world * n_seq / (ms_seq / 1e3), "unit": "clips/s", "ms_per_step": ms_seq / n_seq,
                       "steps": n_seq, "loss": loss_seq,
                       "what": "trainer/trainer_egoclip.py:118-160 call for call through the reference-facing API "
                               "(blocking fp32 .to(device), AllGather_multi x4, sim_matrix x3, EgoNCE(x, sim_v, sim_n), "
                               "loss.item() x2), same model / optimizer"}

    extra = {}
    if args.workload == "cfg4" and rank == 0:
        g = torch.Generator().manual_seed(3)
        sim = (torch.nn.functional.normalize(torch.randn(4096, 256, generator=g), dim=1) @
               torch.nn.functional.normalize(torch.randn(4096, 256, generator=g), dim=1).t()).to(dev)
        ops.dual_softmax(sim)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.dual_softmax(sim)
        e1.record()
        torch.cuda.synchronize()
        extra["dual_softmax_4096x4096_ms"] = e0.elapsed_time(e1) / 10

    if rank == 0:
        peaks, peak_src = measured_peaks()
        f_step, f_video, f_text = flops_per_clip(T, L)
        f_clip = f_step if train else f_video + f_text / 5.0
        peak_tf = peaks["bf16_tflops_sustained"]
        peak_hbm = peaks["hbm_gbs"]
        g_flops, g_ms, g_calls = prof.get("gemm", (0.0, 0.0, 0))
        achieved = g_flops / (g_ms / 1e3) / 1e12 if g_ms > 0 else None
        hbm = {}
        for kind, (nbytes, ms, calls) in sorted(prof.items()):
            if kind == "gemm" or ms <= 0:
                continue
            gbs = nbytes / (ms / 1e3) / 1e9
            hbm[kind] = {"bound": "hbm", "achieved": gbs, "peak": peak_hbm, "unit": "GB/s", "frac": gbs / peak_hbm,
                         "algorithmic_bytes_per_launch": nbytes / calls, "ms_per_launch": ms / calls,
                         "launches_per_step": calls / args.steps, "share_of_step": ms / ms_total}
        line = {"metric": wl["metric"], "workload": args.workload,
                "value": value, "unit": "clips/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "bf16", "data": "synthetic (seeded video/text/tags, seeded random-init weights"
                + ("; text-tower dropout 0.1 active as in the reference's train mode)" if train else "; eval mode)"),
                "config": workload_config(args, wl, world),
                ("loss" if train else "pred_checksum"): (result if train else int(result.sum())),
                "step_flop_fraction_of_peak": value / world * f_clip / (peak_tf * 1e12),
                "gflop_per_clip_step": f_clip / 1e9,
                "roofline": {"bound": "tensor", "kernel": "gemm_bf16_wgmma_kernel (all fwd/dgrad/wgrad launches)",
                             "achieved": achieved, "peak": peak_tf, "unit": "TFLOP/s",
                             "frac": achieved / peak_tf if achieved else None,
                             "algorithmic_flop_per_launch": g_flops / g_calls if g_calls else None,
                             "launches_per_step": g_calls / args.steps, "share_of_step": g_ms / ms_total,
                             "peak_source": peak_src + ", sustained bf16 (kernel timed inside a long step)"},
                "roofline_hbm": hbm, "roofline_hbm_peak_source": peak_src + ", copy bandwidth",
                "clocks": clocks, "e2e": e2e, "gpu_launches": launches,
                # share of the timed region covered by the CUDA-event intervals of the profiled kernels (GEMM + attention +
                # LayerNorm): close to 1 = the step is GPU-bound, the ~700 ctypes C-ABI calls per step stay ahead of the GPU
                "gpu_busy_fraction_profiled_kernels": sum(ms for _, ms, _ in prof.values()) / ms_total}
        if trainer_seq is not None:
            line["trainer_sequence"] = trainer_seq
        line.update(extra)
        if world > 1 and train:
            line["ddp_bucket_cap_mb"] = bucket_mb
        if args.no_ddp_comm or args.ddp_bf16_compress:
            line["ddp_variant"] = "no_sync (diagnostic)" if args.no_ddp_comm else "bf16_compress_hook"
        if world == 1:
            net.zero_grad(set_to_none=True)
            torch.cuda.empty_cache()
            if not args.no_gpu_baseline:
                line["gpu_eager_baseline"] = gpu_eager_baseline(wl, T, L, dev)
            if not args.no_cpu_baseline:
                v, s, cores, sample = cpu_reference_rate(wl, T, L, steps=2, warmup=1)
                line["cpu_baseline"] = {"value": v, "unit": "clips/s", "cores": cores, "kind": "port", "sample": sample}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
