"""Error budget of the bf16 path (VERDICT r1, "what's weak" 1): which rounding puts the CUDA path's embeddings / loss /
gradients where they are relative to the fp32 reference.

The fp32 oracle's graph is re-run on the GPU with bf16 rounding INJECTED at one site at a time (and at all sites), on the
headline geometry (16 frames, 12 blocks, full DistilBERT), and every variant is compared with the plain fp32 run; the CUDA
path's own distance to fp32 is measured next to it.  With every switch off the instrumented graph must reproduce the
oracle bit for bit (asserted), which ties the instrumented copy to oracle/reference_port.py.

Rounding sites (all of them are inputs of a tensor-core MMA, i.e. inherent to a bf16 contraction, except `resid`):
  forward   w      weights of every Linear / the patch conv            x     activation operand of every Linear
            qkv    q (pre-scaled), k, v as stored by the qkv GEMM       p     softmax numerators before P @ V
  backward  dy     output gradient of every Linear (dgrad + wgrad operand)
            dx     input gradient of every Linear as written by its dgrad GEMM (LayerNorm-input grads, da, du)
            resid  the two block-internal residual gradients (d space_residual, d time_residual) kept in bf16 only

    python tools/error_budget.py [--batch 4] [--out error_budget.json]
"""
import argparse
import json
import os
import sys
import warnings

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
warnings.simplefilter("ignore")

SITES_FWD = ("w", "x", "qkv", "p")
SITES_BWD = ("dy", "dx", "resid")


def r16(t):
    return t.to(torch.bfloat16).to(torch.float32)


class _RoundGrad(torch.autograd.Function):
    @staticmethod
    def forward(ctx, t):
        return t.view_as(t)

    @staticmethod
    def backward(ctx, g):
        return r16(g)


def rg(t, on):
    return _RoundGrad.apply(t) if on else t


class Graph:
    """The oracle's graph (oracle/reference_port.py, same line-for-line structure) with optional rounding."""

    def __init__(self, sites):
        self.s = set(sites)

    def linear(self, x, w, b):
        x = rg(x, "dx" in self.s)
        xx = r16(x) if "x" in self.s else x
        ww = r16(w) if "w" in self.s else w
        if "x" in self.s:                     # straight-through: the rounding is a storage format, not a function
            xx = x + (xx - x).detach()
        if "w" in self.s:
            ww = w + (ww - w).detach()
        y = xx @ ww.t() + b
        return rg(y, "dy" in self.s)

    def softmax_av(self, q, k, v):
        p = torch.softmax(q @ k.transpose(-1, -2), dim=-1)
        if "p" in self.s:
            p = p + (r16(p) - p).detach()
        return p @ v

    def attention(self, x, p, prefix, heads, frames, patches, mode):
        qkv = self.linear(x, p[prefix + "qkv.weight"], p[prefix + "qkv.bias"])
        B, S, D3 = qkv.shape
        D = D3 // 3
        d = D // heads
        qkv = qkv.reshape(B, S, 3, heads, d).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0] * d ** -0.5, qkv[1], qkv[2]
        if "qkv" in self.s:
            q, k, v = [t + (r16(t) - t).detach() for t in (q, k, v)]
        cls_out = self.softmax_av(q[:, :, :1], k, v)

        def group(t):
            t = t.reshape(B, heads, frames, patches, d)
            return t.transpose(2, 3) if mode == "time" else t

        qg, kg, vg = group(q[:, :, 1:]), group(k[:, :, 1:]), group(v[:, :, 1:])
        n_groups = qg.shape[2]
        kc = k[:, :, :1].unsqueeze(2).expand(B, heads, n_groups, 1, d)
        vc = v[:, :, :1].unsqueeze(2).expand(B, heads, n_groups, 1, d)
        og = self.softmax_av(qg, torch.cat([kc, kg], dim=3), torch.cat([vc, vg], dim=3))
        if mode == "time":
            og = og.transpose(2, 3)
        out = torch.cat([cls_out, og.reshape(B, heads, frames * patches, d)], dim=2)
        out = out.permute(0, 2, 1, 3).reshape(B, S, D)
        return self.linear(out, p[prefix + "proj.weight"], p[prefix + "proj.bias"])

    def block(self, x, p, prefix, heads, frames, patches, eps=1e-6):
        D = x.shape[-1]
        ln = lambda t, n: F.layer_norm(t, (D,), p[prefix + n + ".weight"], p[prefix + n + ".bias"], eps)
        t_res = x + self.attention(ln(x, "norm3"), p, prefix + "timeattn.", heads, frames, patches, "time")
        t_res = rg(t_res, "resid" in self.s)
        s_res = x + self.attention(ln(t_res, "norm1"), p, prefix + "attn.", heads, frames, patches, "space")
        s_res = rg(s_res, "resid" in self.s)
        h = F.gelu(self.linear(ln(s_res, "norm2"), p[prefix + "mlp.fc1.weight"], p[prefix + "mlp.fc1.bias"]))
        return s_res + self.linear(h, p[prefix + "mlp.fc2.weight"], p[prefix + "mlp.fc2.bias"])

    def video(self, video, p, heads=12):
        from oracle import reference_port as rp
        B, T, C, H, W = video.shape
        w = p["video_model.patch_embed.proj.weight"]
        D, _, ph, pw = w.shape
        gh, gw = H // ph, W // pw
        n = gh * gw
        patches = video.reshape(B * T, C, gh, ph, gw, pw).permute(0, 2, 4, 1, 3, 5).reshape(B * T * n, C * ph * pw)
        tok = self.linear(patches, w.reshape(D, -1), p["video_model.patch_embed.proj.bias"]).reshape(B, T * n, D)
        pos, tmp = p["video_model.pos_embed"][0], p["video_model.temporal_embed"][0, :T]
        tok = tok + (pos[1:].unsqueeze(0) + tmp.unsqueeze(1)).reshape(1, T * n, D)
        cls = (p["video_model.cls_token"][0, 0] + pos[0]).expand(B, 1, D)
        x = torch.cat([cls, tok], dim=1)
        depth = 1 + max(int(k.split("blocks.")[1].split(".")[0]) for k in p if k.startswith("video_model.blocks."))
        for i in range(depth):
            x = self.block(x, p, f"video_model.blocks.{i}.", heads, T, n)
        x = F.layer_norm(x, (D,), p["video_model.norm.weight"], p["video_model.norm.bias"], 1e-6)[:, 0]
        return self.linear(x, p["vid_proj.0.weight"], p["vid_proj.0.bias"])

    def text(self, text, p, heads=12):
        ids, mask = text["input_ids"], text["attention_mask"]
        B, L = ids.shape
        pre = "text_model."
        we, pe = p[pre + "embeddings.word_embeddings.weight"], p[pre + "embeddings.position_embeddings.weight"]
        D = we.shape[1]
        d = D // heads
        x = F.layer_norm(we[ids] + pe[:L].unsqueeze(0), (D,), p[pre + "embeddings.LayerNorm.weight"],
                         p[pre + "embeddings.LayerNorm.bias"], 1e-12)
        bias = torch.zeros(B, 1, 1, L, device=x.device).masked_fill(mask.reshape(B, 1, 1, L) == 0, float("-inf"))
        n_layers = 1 + max(int(k.split("transformer.layer.")[1].split(".")[0]) for k in p if "transformer.layer." in k)
        for i in range(n_layers):
            lp = f"{pre}transformer.layer.{i}."
            hd = lambda t: t.reshape(B, L, heads, d).transpose(1, 2)
            q = hd(self.linear(x, p[lp + "attention.q_lin.weight"], p[lp + "attention.q_lin.bias"])) / d ** 0.5
            k = hd(self.linear(x, p[lp + "attention.k_lin.weight"], p[lp + "attention.k_lin.bias"]))
            v = hd(self.linear(x, p[lp + "attention.v_lin.weight"], p[lp + "attention.v_lin.bias"]))
            if "qkv" in self.s:
                q, k, v = [t + (r16(t) - t).detach() for t in (q, k, v)]
            w = torch.softmax(q @ k.transpose(-1, -2) + bias, dim=-1)       # text attention P stays fp32 in text.cu
            ctx = (w @ v).transpose(1, 2).reshape(B, L, D)
            sa = self.linear(ctx, p[lp + "attention.out_lin.weight"], p[lp + "attention.out_lin.bias"])
            x = F.layer_norm(sa + x, (D,), p[lp + "sa_layer_norm.weight"], p[lp + "sa_layer_norm.bias"], 1e-12)
            h = F.gelu(self.linear(x, p[lp + "ffn.lin1.weight"], p[lp + "ffn.lin1.bias"]))
            h = self.linear(h, p[lp + "ffn.lin2.weight"], p[lp + "ffn.lin2.bias"])
            x = F.layer_norm(h + x, (D,), p[lp + "output_layer_norm.weight"], p[lp + "output_layer_norm.bias"], 1e-12)
        return self.linear(torch.relu(x[:, 0]), p["txt_proj.1.weight"], p["txt_proj.1.bias"])


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def run_graph(sites, data, verb, noun, params, want_grad):
    from oracle import reference_port as rp
    g = Graph(sites)
    p = {k: v.clone().requires_grad_(want_grad) for k, v in params.items()}
    with torch.set_grad_enabled(want_grad):
        t, v = g.text(data["text"], p), g.video(data["video"], p)
        loss = rp.egonce_loss(rp.sim_matrix(t, v), rp.sim_matrix(verb, verb), rp.sim_matrix(noun, noun))
        if want_grad:
            loss.backward()
    grad = torch.cat([p[k].grad.flatten() for k in sorted(p) if p[k].grad is not None]) if want_grad else None
    return t.detach(), v.detach(), loss.item(), grad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--out", default="error_budget.json")
    args = ap.parse_args()
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.loss import EgoNCE
    from egovlp_b200.model.model import FrozenInTime
    from oracle import reference_port as rp
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0)
    B, T, L = args.batch, args.frames, 16
    sd = syn.seeded_state_dict(syn.model_dims(num_frames=T), seed=0)
    params = {k: v.to(dev) for k, v in sd.items()}
    data = {"video": syn.synthetic_video(B, T, seed=5).to(dev),
            "text": {k: v.to(dev) for k, v in syn.synthetic_text(B, L, seed=5, ragged=True).items()}}
    verb, noun = [t.to(dev) for t in syn.synthetic_tags(B, seed=5)]

    t0, v0, l0, g0 = run_graph((), data, verb, noun, params, True)
    # the instrumented graph with every switch off IS the oracle
    p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    tr, vr = rp.frozen_in_time_forward(data, p)
    lr = rp.egonce_loss(rp.sim_matrix(tr, vr), rp.sim_matrix(verb, verb), rp.sim_matrix(noun, noun))
    assert rel(t0, tr) < 1e-6 and rel(v0, vr) < 1e-6 and abs(lr.item() - l0) < 1e-6 * abs(l0), "instrumented graph != oracle"

    rows = {}
    for name, sites in [(s, (s,)) for s in SITES_FWD] + [("all forward", SITES_FWD)]:
        t, v, l, _ = run_graph(sites, data, verb, noun, params, False)
        rows[name] = {"rel_text_emb": rel(t, t0), "rel_video_emb": rel(v, v0), "rel_loss": abs(l - l0) / abs(l0)}
    for name, sites in [(s, (s,)) for s in SITES_BWD] + [("all backward", SITES_BWD),
                                                         ("all forward + backward", SITES_FWD + SITES_BWD)]:
        t, v, l, g = run_graph(sites, data, verb, noun, params, True)
        rows[name] = {"rel_text_emb": rel(t, t0), "rel_video_emb": rel(v, v0), "rel_loss": abs(l - l0) / abs(l0),
                      "rel_grad_all": rel(g, g0)}

    # the CUDA path on the same inputs
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": T,
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    net.load_state_dict(sd, strict=True)
    net.text_model.config.dropout = net.text_model.config.attention_dropout = 0.0
    net.to(dev)
    t, v = net(data)
    loss = EgoNCE().fused(t, v, verb, noun)
    loss.backward()
    named = dict(net.named_parameters())
    g = torch.cat([named[k].grad.flatten() for k in sorted(named) if named[k].grad is not None])
    rows["CUDA path (measured)"] = {"rel_text_emb": rel(t, t0), "rel_video_emb": rel(v, v0),
                                    "rel_loss": abs(loss.item() - l0) / abs(l0), "rel_grad_all": rel(g, g0)}
    out = {"shape": {"batch": B, "frames": T, "text_len": L, "blocks": 12}, "loss_fp32": l0, "rows": rows}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    w = max(len(k) for k in rows)
    print(f"{'site':{w}}  text-emb   video-emb  loss       grad(all)")
    for k, r in rows.items():
        print(f"{k:{w}}  {r['rel_text_emb']:.2e}   {r['rel_video_emb']:.2e}   {r['rel_loss']:.2e}   "
              + (f"{r['rel_grad_all']:.2e}" if "rel_grad_all" in r else "-"))


if __name__ == "__main__":
    main()
