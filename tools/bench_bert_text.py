"""What a BERT text tower costs: the tower alone, and the cfg3 EgoClip training step with it.

    python tools/bench_bert_text.py [--part tower|step|all] [--text-len 16] [--steps 8] [--rounds 3]
                                    [--dump-outputs DIR] [--json out.json]

Tower (B = 32, L in 16 / 64 / 128 / 512; distilbert-base, bert-base, bert-large, seeded weights): forward + backward
of the CUDA tower (engine.TextTowerFn / BertTowerFn) with dropout off and on (p = 0.1 / 0.1), its no_grad forward,
and the HuggingFace module (DistilBertModel / BertModel, the CLS row / pooler_output) run eagerly on the same GPU in
fp32 and under bf16 autocast, forward + backward.  CUDA-event times per call, mean over the timed iterations.

Step: the cfg3 step as bench.py builds it (16 frames, batch 32, EgoNCE, fused AdamW, seeded weights), once with the
DistilBERT text tower and once with a bert-base-uncased one, the two models alternated in `--rounds` rounds of
`--steps` timed steps after 3 warm-up steps each.  `--dump-outputs DIR` writes each model's last loss and bench.py's
weight sample to DIR/<tower>_*.npy.  The card name, power limit and SM clocks are read in the same run.
"""
import argparse
import json
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_text_attn import card  # noqa: E402

ARCHS = {"distilbert-base": dict(text_dim=768, text_layers=6, text_heads=12, text_hidden=3072),
         "bert-base": dict(text_dim=768, text_layers=12, text_heads=12, text_hidden=3072, text_kind="bert"),
         "bert-large": dict(text_dim=1024, text_layers=24, text_heads=16, text_hidden=4096, text_kind="bert")}


def time_ms(fn, iters, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def hf_module(arch, dims):
    from transformers import BertConfig, BertModel, DistilBertConfig, DistilBertModel
    if arch == "distilbert-base":
        return DistilBertModel(DistilBertConfig(dropout=0.0, attention_dropout=0.0)), lambda o: o.last_hidden_state[:, 0]
    cfg = BertConfig(hidden_size=dims["text_dim"], num_hidden_layers=dims["text_layers"],
                     num_attention_heads=dims["text_heads"], intermediate_size=dims["text_hidden"],
                     hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    return BertModel(cfg), lambda o: o.pooler_output


def bench_tower(iters):
    from egovlp_b200 import engine, synthetic as syn
    rows = []
    for arch, a in ARCHS.items():
        dims = syn.model_dims(**a)
        sd = syn.seeded_state_dict(dims, seed=0, video=False, proj=True)
        keys = [k for k in sd if k.startswith("text_model.")] + ["txt_proj.1.weight", "txt_proj.1.bias"]
        p = [sd[k].cuda().requires_grad_(True) for k in keys]
        fn = engine.BertTowerFn if a.get("text_kind") == "bert" else engine.TextTowerFn
        cache = engine.Bf16Cache()
        hf, head = hf_module(arch, dims)
        hf = hf.cuda()
        for L in (16, 64, 128, 512):
            text = {k: v.cuda() for k, v in syn.synthetic_text(32, L, seed=L).items()}
            ids, mask = text["input_ids"], text["attention_mask"]

            def fwd_bwd(drop):
                out = fn.apply(ids, mask, a["text_heads"], 1e-12, False, cache, drop, *p)
                out.sum().backward()

            def fwd():
                with torch.no_grad():
                    fn.apply(ids, mask, a["text_heads"], 1e-12, False, cache, None, *p)

            def eager(autocast):
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                    out = head(hf(input_ids=ids, attention_mask=mask))
                out.float().sum().backward()

            r = {"arch": arch, "L": L, "B": 32,
                 "cuda_fwd_bwd_ms": time_ms(lambda: fwd_bwd(None), iters),
                 "cuda_fwd_bwd_dropout_ms": time_ms(lambda: fwd_bwd((0.1, 0.1)), iters),
                 "cuda_fwd_nograd_ms": time_ms(fwd, iters),
                 "hf_fp32_fwd_bwd_ms": time_ms(lambda: eager(False), max(3, iters // 4), warm=1),
                 "hf_bf16_autocast_fwd_bwd_ms": time_ms(lambda: eager(True), max(3, iters // 4), warm=1)}
            print(json.dumps(r), flush=True)
            rows.append(r)
            for t in p:
                t.grad = None
            hf.zero_grad(set_to_none=True)
        del hf, p, cache
        torch.cuda.empty_cache()
    return rows


def bench_step(text_len, steps, rounds, dump):
    import numpy as np
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.distributed import egoclip_step_loss
    from egovlp_b200.model.loss import EgoNCE
    from egovlp_b200.model.model import FrozenInTime
    from egovlp_b200.optim import AdamW
    torch.manual_seed(0)
    B, T = 32, 16
    video = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": T, "pretrained": True,
             "time_init": "zeros"}
    txt = syn.synthetic_text(B, text_len, seed=0)
    verb, noun = syn.synthetic_tags(B, seed=0)
    data = {"video": syn.synthetic_video(B, T, seed=0).cuda(),
            "text": {"input_ids": txt["input_ids"].cuda(), "attention_mask": txt["attention_mask"].cuda()},
            "verb_vec": verb.cuda(), "noun_vec": noun.cuda()}
    runs = {}
    for name, model, extra in (("distilbert", "distilbert-base-uncased", {}),
                               ("bert", "bert-base-uncased", dict(text_layers=12, text_kind="bert"))):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            net = FrozenInTime(video, {"model": model, "pretrained": True, "input": "text"})
        net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=T, **extra), seed=0), strict=True)
        net.cuda()
        runs[name] = dict(net=net, opt=AdamW(net.parameters(), lr=3e-5), ms=[], loss=None)
    loss_fn = EgoNCE()

    def step(r):
        r["opt"].zero_grad(set_to_none=True)
        loss = egoclip_step_loss(r["net"], loss_fn, data)
        loss.backward()
        r["opt"].step()
        return loss

    for r in runs.values():
        for _ in range(3):
            step(r)
    torch.cuda.synchronize()
    for _ in range(rounds):
        for r in runs.values():
            out = []
            r["ms"].append(time_ms(lambda: out.append(step(r)), steps, warm=0))
            r["loss"] = out[-1].item()
    res = {"text_len": text_len, "batch": B, "frames": T, "steps_per_round": steps, "rounds": rounds}
    for name, r in runs.items():
        ms = sorted(r["ms"])
        res[name] = {"ms_per_step_rounds": r["ms"], "clips_per_s_median": B / (ms[len(ms) // 2] / 1e3),
                     "last_loss": r["loss"]}
        if dump:
            os.makedirs(dump, exist_ok=True)
            np.save(os.path.join(dump, f"{name}_loss.npy"), np.array([r["loss"]], dtype=np.float64))
            parts = []
            for i, (_, p) in enumerate(r["net"].named_parameters()):
                idx = torch.randint(0, p.numel(), (4096,), generator=torch.Generator().manual_seed(i)).to(p.device)
                parts.append(p.detach().flatten()[idx].float().cpu())
            np.save(os.path.join(dump, f"{name}_weights_sample.npy"), torch.cat(parts).numpy())
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", default="all", choices=["tower", "step", "all"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--text-len", type=int, default=16)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    out = {"card": card()}
    print(json.dumps(out), flush=True)
    if args.part in ("tower", "all"):
        out["tower"] = bench_tower(args.iters)
    if args.part in ("step", "all"):
        out["step"] = bench_step(args.text_len, args.steps, args.rounds, args.dump_outputs)
    out["card_after"] = card()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
