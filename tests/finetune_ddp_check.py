"""Multi-rank parity of the Ego4D OSCC fine-tuning step, launched by tests/test_finetune_distributed_gpu.py (or by hand) as

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/finetune_ddp_check.py

On N NCCL ranks, full-size video tower (model built for 16 frames, 4-frame input) with the 2-wide OSCC head, the step
of trainer/trainer_oscc.py:333-338 under DistributedDataParallel(find_unused_parameters=True) as base/base_trainer.py
wraps it: model(data, video_only=True) -> AllGather_multi of the scores and of the state labels (local-slice backward) ->
CrossEntropy.  The loss is bit-identical on every rank and equals the single-process full-batch loss; DDP's averaged
gradient x world equals the full-batch gradient.  Rank 0 writes finetune_ddp_check_N.json to EGOVLP_RECORD_DIR (default:
a temporary directory)."""
import json
import os
import sys
import tempfile
import warnings

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
warnings.simplefilter("ignore")

from ddp_check import rel  # noqa: E402


def main():
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.distributed import AllGatherLocalGrad
    from egovlp_b200.model.loss import CrossEntropy
    from egovlp_b200.model.model import FrozenInTime

    world, rank, local = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    B, T, C = 4, 4, 2
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 16,
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"}, projection_dim=C)
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=16, proj_dim=C), seed=3), strict=True)
    net.to(dev)
    crit = CrossEntropy()

    def batch(r):
        state = torch.randint(0, 2, (B,), generator=torch.Generator().manual_seed(200 + r))
        return syn.synthetic_video(B, T, seed=200 + r).to(dev), state.to(dev)

    def grads():
        return {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}

    # ---- single-process full batch (no collective): every rank computes it redundantly
    full = [batch(r) for r in range(world)]
    net.zero_grad(set_to_none=True)
    loss_full = crit(net({"video": torch.cat([v for v, _ in full])}, video_only=True), torch.cat([s for _, s in full]))
    loss_full.backward()
    g_full = grads()

    # ---- the trainer's step under DDP
    ddp = torch.nn.parallel.DistributedDataParallel(net, device_ids=[local], find_unused_parameters=True)
    net.zero_grad(set_to_none=True)
    video, state = batch(rank)
    scores = AllGatherLocalGrad.apply(ddp({"video": video}, video_only=True))
    loss_ddp = crit(scores, AllGatherLocalGrad.apply(state))
    loss_ddp.backward()
    g_ddp = grads()
    losses = [torch.zeros((), device=dev) for _ in range(world)]
    dist.all_gather(losses, loss_ddp.detach())
    same_on_all_ranks = all(torch.equal(x, losses[0]) for x in losses)
    rel_loss_full = abs(loss_ddp.item() - loss_full.item()) / abs(loss_full.item())
    keys = [k for k in g_full if g_full[k].norm() > 1e-10]
    big = [k for k in keys if g_full[k].numel() > 4096]
    worst = max((rel(g_ddp[k] * world, g_full[k]), k) for k in big)
    all_rel = rel(torch.cat([g_ddp[k].flatten().double() * world for k in keys]),
                  torch.cat([g_full[k].flatten().double() for k in keys]))
    text_untouched = not any(k.startswith(("text_model.", "txt_proj.")) for k in g_ddp)
    out = {"world": world, "loss_full_batch": loss_full.item(), "loss_ddp": loss_ddp.item(),
           "loss_identical_on_all_ranks": same_on_all_ranks, "rel_loss_vs_full_batch": rel_loss_full,
           "worst_matrix_grad_rel_ddp_x_world_vs_full": worst, "all_grads_rel_ddp_x_world_vs_full": all_rel,
           "n_grad_tensors": len(g_full), "text_tower_without_grads": text_untouched}
    # same bound as tests/ddp_check.py for the whole gradient: two executions differ by the order of the video tower's
    # fp32 atomics (split-K, CLS rows); a wrong 1/world factor or a missing local slice would show up as O(1)
    ok = (same_on_all_ranks and rel_loss_full < 1e-5 and text_untouched and all_rel < 1.2e-2 and worst[0] < 6e-2
          and len(g_ddp) == len(g_full))
    flag = torch.tensor([1.0 if ok else 0.0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        out["ok"] = bool(flag.item() == 1.0)
        out_dir = os.environ.get("EGOVLP_RECORD_DIR") or os.path.join(tempfile.gettempdir(), "egovlp_records")
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, f"finetune_ddp_check_{world}.json"), "w") as f:
            json.dump(out, f, indent=1)
        print(json.dumps(out), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1.0 else 1)


if __name__ == "__main__":
    main()
