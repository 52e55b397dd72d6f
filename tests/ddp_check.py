"""Multi-rank parity script, launched by tests/test_distributed_gpu.py (or by hand) as

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/ddp_check.py

Checks on N NCCL ranks (N = 1 works too), full-size FrozenInTime towers (4-frame input), dropout off:
  1. fused step (model -> ONE packed all-gather -> EgoNCE.fused) under DDP: the loss is bit-identical on every rank and
     equals the single-process full-batch loss; DDP's averaged gradient x world == the full-batch gradient
     (SURVEY.md 8a quirk 8: gather backward keeps the local slice only);
  2. the reference trainer's literal call sequence (tools/trainer_sequence.py: 4x list-API all_gather, 3x sim_matrix,
     EgoNCE(x, sim_v, sim_n)) gives the same loss and the same gradients as the fused step.
Rank 0 writes ddp_check_N.json to EGOVLP_RECORD_DIR (default: a temporary directory)."""
import json
import os
import sys
import tempfile
import warnings

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
warnings.simplefilter("ignore")


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


class _NoStep:
    """Optimizer stand-in for the trainer sequence: clears gradients before the step, keeps them afterwards."""

    def __init__(self, net):
        self.net, self.calls = net, 0

    def zero_grad(self):
        self.calls += 1
        if self.calls % 2 == 1:
            self.net.zero_grad(set_to_none=True)

    def step(self):
        pass


def main():
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.distributed import egoclip_step_loss
    from egovlp_b200.model.loss import EgoNCE
    from egovlp_b200.model.model import FrozenInTime, sim_matrix
    from tools.trainer_sequence import trainer_step

    world, rank, local = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    B, T, L = 4, 4, 12
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 4,
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=4), seed=0), strict=True)
    net.text_model.config.dropout = net.text_model.config.attention_dropout = 0.0
    net.to(dev)
    loss_fn = EgoNCE()

    def batch(r):
        verb, noun = syn.synthetic_tags(B, seed=100 + r, zero_noun_row=False)
        return {"video": syn.synthetic_video(B, T, seed=100 + r), "text": syn.synthetic_text(B, L, seed=100 + r, ragged=True),
                "verb_vec": verb, "noun_vec": noun}

    def to_dev(b):
        return {"video": b["video"].to(dev), "text": {k: v.to(dev) for k, v in b["text"].items()},
                "verb_vec": b["verb_vec"].to(dev), "noun_vec": b["noun_vec"].to(dev)}

    names = [k for k, _ in net.named_parameters()]

    def grads():
        return {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}

    # ---- single-process full batch (no collective): every rank computes it redundantly
    full = [batch(r) for r in range(world)]
    cat = {"video": torch.cat([b["video"] for b in full]).to(dev),
           "text": {k: torch.cat([b["text"][k] for b in full]).to(dev) for k in ("input_ids", "attention_mask")}}
    verb_all = torch.cat([b["verb_vec"] for b in full]).to(dev)
    noun_all = torch.cat([b["noun_vec"] for b in full]).to(dev)
    net.zero_grad(set_to_none=True)
    t, v = net(cat)
    loss_full = loss_fn.fused(t, v, verb_all, noun_all)
    loss_full.backward()
    g_full = grads()

    # ---- fused step under DDP
    ddp = torch.nn.parallel.DistributedDataParallel(net, device_ids=[local], gradient_as_bucket_view=True)
    net.zero_grad(set_to_none=True)
    loss_ddp = egoclip_step_loss(ddp, loss_fn, to_dev(batch(rank)))
    loss_ddp.backward()
    g_ddp = grads()
    losses = [torch.zeros((), device=dev) for _ in range(world)]
    dist.all_gather(losses, loss_ddp.detach())
    same_on_all_ranks = all(torch.equal(x, losses[0]) for x in losses)
    rel_loss_full = abs(loss_ddp.item() - loss_full.item()) / abs(loss_full.item())
    # matrices are compared tensor by tensor; small vectors (biases, LayerNorm, cls_token: sums of nearly cancelling
    # per-clip terms whose fp32 atomic order differs run to run) through a looser bound and the global vector
    big = [k for k in g_full if g_full[k].numel() > 4096 and g_full[k].norm() > 1e-10]
    # (k_lin.bias gradients are analytically zero -- softmax shift invariance -- i.e. pure rounding noise)
    small = [k for k in g_full if g_full[k].numel() <= 4096 and g_full[k].norm() > 1e-10 and not k.endswith("k_lin.bias")]
    flat = lambda gd, ks, s=1.0: torch.cat([gd[k].flatten().double() * s for k in ks])
    worst_ddp = max((rel(g_ddp[k] * world, g_full[k]), k) for k in big)
    worst_ddp_vec = max((rel(g_ddp[k] * world, g_full[k]), k) for k in small)
    all_ddp = rel(flat(g_ddp, big + small, world), flat(g_full, big + small))

    # ---- the reference trainer's literal sequence under DDP
    shim = _NoStep(net)
    loss_seq = trainer_step(ddp, loss_fn, shim, batch(rank), dev, sim_matrix)
    g_seq = grads()
    rel_loss_seq = abs(loss_seq - loss_ddp.item()) / abs(loss_ddp.item())
    worst_seq = max((rel(g_seq[k], g_ddp[k]), k) for k in big)
    worst_seq_vec = max((rel(g_seq[k], g_ddp[k]), k) for k in small)
    all_seq = rel(flat(g_seq, big + small), flat(g_ddp, big + small))

    out = {"world": world, "loss_full_batch": loss_full.item(), "loss_fused_ddp": loss_ddp.item(), "loss_trainer_sequence": loss_seq,
           "loss_identical_on_all_ranks": same_on_all_ranks, "rel_loss_vs_full_batch": rel_loss_full,
           "worst_matrix_grad_rel_ddp_x_world_vs_full": worst_ddp, "worst_vector_grad_rel_ddp_x_world_vs_full": worst_ddp_vec,
           "all_grads_rel_ddp_x_world_vs_full": all_ddp, "rel_loss_sequence_vs_fused": rel_loss_seq,
           "worst_matrix_grad_rel_sequence_vs_fused": worst_seq, "worst_vector_grad_rel_sequence_vs_fused": worst_seq_vec,
           "all_grads_rel_sequence_vs_fused": all_seq, "n_grad_tensors": len(g_full), "n_params": len(names)}
    ok = (same_on_all_ranks and rel_loss_full < 1e-5 and rel_loss_seq < 1e-6 and len(g_full) == len(names)
          # two executions of the same math differ by the order of fp32 atomics (split-K, CLS rows) amplified through
          # bf16 re-rounding -- measured on 2 ranks: 4e-3 on the whole gradient between two executions of the SAME
          # DDP step, 1.2e-2 between DDP x world and the single-process full batch, 3e-2 on the cancellation-heavy
          # pos_embed / cls_token sums; a wrong 1/world factor or a missing local slice would show up as O(1)
          and worst_ddp[0] < 6e-2 and worst_seq[0] < 6e-2 and worst_ddp_vec[0] < 0.15 and worst_seq_vec[0] < 0.15
          and all_ddp < 2.5e-2 and all_seq < 2.5e-2)
    flag = torch.tensor([1.0 if ok else 0.0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        out["ok"] = bool(flag.item() == 1.0)
        out_dir = os.environ.get("EGOVLP_RECORD_DIR") or os.path.join(tempfile.gettempdir(), "egovlp_records")
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, f"ddp_check_{world}.json"), "w") as f:
            json.dump(out, f, indent=1)
        print(json.dumps(out), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1.0 else 1)


if __name__ == "__main__":
    main()
