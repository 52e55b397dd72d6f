"""Peak memory and clips/s of the cfg3 training step (16 frames, L = 16, EgoNCE, fused AdamW, seeded synthetic inputs) with
and without the video tower's selective activation recompute (`set_grad_checkpointing`), on one GPU.

    python tools/bench_activation_memory.py [--batches 32,48,64] [--steps 8] [--warmup 3]

Runs B = 32 in the two modes alternately, twice each, then every other batch once per mode.  The default mode is skipped
where the shapes say it cannot fit the card (its 12 blocks save 38,520 bytes per token; 21,624 in the low-memory mode).
Prints one JSON line per case: torch.cuda.max_memory_allocated after a reset, clips/s between CUDA events after the warm-up
steps, the saved bytes per token of one block counted from its saved tensors, the card name, power limit and median SM
clock of the run.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (SM clock sampler of the headline benchmark)
from bench_finetune import card  # noqa: E402

FRAMES, TEXT_LEN, TOKENS_PER_CLIP, DEPTH = 16, 16, 1 + 16 * 196, 12
SAVED = {False: 38520, True: 21624}       # bytes per token per block, from the shapes


def fits(B, low, total):
    """Shape arithmetic: the saved activations of the 12 blocks, one block backward's transients (~30 KB per token) and
    ~4 GB of weights, gradients, Adam state and the text tower."""
    tokens = B * TOKENS_PER_CLIP
    return DEPTH * SAVED[low] * tokens + 30e3 * tokens + 4e9 <= total


def run_case(net, opt, B, low, steps, warmup, device):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.distributed import egoclip_step_loss
    from egovlp_b200.model.loss import EgoNCE
    net.video_model.set_grad_checkpointing(low)
    txt = syn.synthetic_text(B, TEXT_LEN, seed=0)
    verb, noun = syn.synthetic_tags(B, seed=0)
    data = {"video": syn.synthetic_video(B, FRAMES, seed=0).to(device),
            "text": {k: v.to(device) for k, v in txt.items()}, "verb_vec": verb.to(device), "noun_vec": noun.to(device)}
    loss_fn = EgoNCE()
    saved = []

    def count_saved(module, args, out):          # one block's saved tensors, parameters excluded
        if not saved and out.grad_fn is not None:
            sv = out.grad_fn.saved_tensors
            saved.append(sum(t.numel() * t.element_size() for t in sv[:20] if t is not None) / sv[0].shape[0])

    hook = net.video_model.blocks[0].register_forward_hook(count_saved)

    def step():
        opt.zero_grad(set_to_none=True)
        loss = egoclip_step_loss(net, loss_fn, data)
        loss.backward()
        opt.step()
        return loss

    try:
        for _ in range(warmup):
            step()
        hook.remove()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        sampler = bench.ClockSampler(device.index)
        sampler.start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            loss = step()
        e1.record()
        torch.cuda.synchronize()
        clocks = sampler.stop()
        ms = e0.elapsed_time(e1)
        return {"batch": B, "low_memory": low, "clips_per_s": B * steps / (ms / 1e3), "ms_per_step": ms / steps,
                "peak_allocated_gb": torch.cuda.max_memory_allocated() / 1e9, "saved_bytes_per_token_block": saved[0],
                "loss": loss.item(), "steps": steps, "warmup": warmup, "sm_clock_mhz_median": clocks.get("sm_mhz")}
    except torch.OutOfMemoryError as e:
        return {"batch": B, "low_memory": low, "error": "out of memory: " + str(e).split("\n")[0]}
    finally:
        hook.remove()
        del data
        opt.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="32,48,64")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert args.steps >= 8 and args.warmup >= 3, "time at least 8 steps after 3 warm-up steps"
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.model import FrozenInTime
    from egovlp_b200.optim import AdamW
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    device = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": FRAMES,
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=FRAMES), seed=0), strict=True)
    net.to(device)
    opt = AdamW(net.parameters(), lr=3e-5)
    total = torch.cuda.get_device_properties(device).total_memory
    name, power = card()
    batches = [int(b) for b in args.batches.split(",")]
    cases = []
    if 32 in batches:
        cases += [(32, False), (32, True), (32, False), (32, True)]        # alternated in one session
    for B in batches:
        if B != 32:
            cases += [(B, False), (B, True)]
    for B, low in cases:
        if not fits(B, low, total):
            line = {"batch": B, "low_memory": low,
                    "skipped": f"needs more than the card's {total / 1e9:.1f} GB by the shape arithmetic"}
        else:
            line = run_case(net, opt, B, low, args.steps, args.warmup, device)
        line.update({"gpu": name, "power_limit": power, "free_gb_after": torch.cuda.mem_get_info()[0] / 1e9})
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
