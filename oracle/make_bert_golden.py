"""Generate tests/golden/bert_tiny.npz from the UNMODIFIED reference's `bert*` text tower (model/model.py:34-35,
:117-138), run on the CPU through oracle/ref_shim.py.

    python -m oracle.make_bert_golden

FrozenInTime is built with text_params.model = 'bert-base-uncased' while `AutoModel.from_pretrained` returns a tiny
BertModel (vocab 120, hidden 128, 2 layers, 2 heads, FFN 256, 512 positions, dropout 0) holding
egovlp_b200.synthetic.seeded_state_dict(BERT_TINY_DIMS, seed=SEED); txt_proj gets the same mapping's weights.
Stored (outputs only; the weights are regenerated from the seed):
  * compute_text and compute_text_tokens on ragged batches at L = 9 and L = 200, with projection 'minimal', and the
    pooled output with projection='';
  * under the probe loss sum_L <compute_text(text_L), probe_L>, GRAD_SAMPLES seeded entries of the gradient of every
    text parameter and of txt_proj (every entry of tensors that small), and each gradient's L2 norm;
  * the state_dict keys and shapes of a full-size bert-base-uncased FrozenInTime (JSON), so the key check runs
    without the reference.
"""
import contextlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from egovlp_b200 import synthetic as syn  # noqa: E402
from oracle import ref_shim  # noqa: E402

BERT_TINY_DIMS = dict(syn.TINY_DIMS, max_pos=512, text_kind="bert")
SEED = 8
GRAD_SAMPLES = 256
CASES = ((5, 9, 1), (4, 200, 2))                      # (B, L, input seed): ragged, row 0 full length


@contextlib.contextmanager
def bert_constructors(factory):
    """ref_shim's patched constructors with `AutoModel.from_pretrained` returning factory()."""
    mm, _, _ = ref_shim.modules()
    with ref_shim._patched_constructors():
        patched = mm.AutoModel.from_pretrained
        mm.AutoModel.from_pretrained = lambda *a, **k: factory()
        try:
            yield mm
        finally:
            mm.AutoModel.from_pretrained = patched


def tiny_bert(sd):
    from transformers import BertConfig, BertModel
    d = BERT_TINY_DIMS
    cfg = BertConfig(vocab_size=d["vocab"], hidden_size=d["text_dim"], num_hidden_layers=d["text_layers"],
                     num_attention_heads=d["text_heads"], intermediate_size=d["text_hidden"],
                     max_position_embeddings=d["max_pos"], hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    net = BertModel(cfg)
    net.load_state_dict({k[len("text_model."):]: v for k, v in sd.items() if k.startswith("text_model.")}, strict=True)
    return net


def reference_model(sd, projection):
    video_params = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 4,
                    "pretrained": True, "time_init": "zeros"}
    text_params = {"model": "bert-base-uncased", "pretrained": True, "input": "text"}
    with bert_constructors(lambda: tiny_bert(sd)) as mm:
        net = mm.FrozenInTime(video_params, text_params, projection_dim=BERT_TINY_DIMS["proj_dim"],
                              load_checkpoint=None, projection=projection)
    if projection == "minimal":
        net.txt_proj[1].weight.data.copy_(sd["txt_proj.1.weight"])
        net.txt_proj[1].bias.data.copy_(sd["txt_proj.1.bias"])
    return net


def inputs():
    return [syn.synthetic_text(B, L, seed=s, ragged=True, vocab=BERT_TINY_DIMS["vocab"]) for B, L, s in CASES]


def probes():
    g = torch.Generator().manual_seed(31)
    return [torch.randn(B, BERT_TINY_DIMS["proj_dim"], generator=g) for B, _, _ in CASES]


def grad_index(name, n):
    """The sampled flat indices of a gradient: all of them up to GRAD_SAMPLES entries, else a seeded draw."""
    if n <= GRAD_SAMPLES:
        return torch.arange(n)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    return torch.randperm(n, generator=g)[:GRAD_SAMPLES].sort().values


def main():
    from transformers import BertConfig, BertModel
    sd = syn.seeded_state_dict(BERT_TINY_DIMS, seed=SEED, video=False, proj=True)
    out = {"seed": SEED}
    texts = inputs()
    net = reference_model(sd, "minimal")
    bare = reference_model(sd, "")
    loss = 0
    for (B, L, _), text, probe in zip(CASES, texts, probes()):
        out[f"l{L}/input_ids"], out[f"l{L}/attention_mask"] = text["input_ids"].numpy(), text["attention_mask"].numpy()
        t = net.compute_text(text)
        with torch.no_grad():
            out[f"l{L}/tokens"] = net.compute_text_tokens(text).numpy()
            out[f"l{L}/pooled"] = bare.compute_text(text).numpy()
        out[f"l{L}/text"] = t.detach().numpy()
        loss = loss + (t * probe).sum()
    loss.backward()
    params = dict(net.named_parameters())
    names = [k for k in sd if k.startswith("text_model.") or k.startswith("txt_proj.")]
    for k in names:
        gr = params[k].grad
        gr = torch.zeros_like(params[k]) if gr is None else gr
        idx = grad_index(k, gr.numel())
        out[f"grad/{k}/idx"] = idx.numpy()
        out[f"grad/{k}/val"] = gr.flatten()[idx].numpy()
        out[f"grad/{k}/norm"] = np.float64(gr.double().norm())
    with bert_constructors(lambda: BertModel(BertConfig())) as mm:
        full = mm.FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 4,
                                "pretrained": True, "time_init": "zeros"},
                               {"model": "bert-base-uncased", "pretrained": True, "input": "text"},
                               projection_dim=256, load_checkpoint=None, projection="minimal")
    keys = json.dumps([[k, list(v.shape)] for k, v in full.state_dict().items()])
    out["bert_base_keys_json"] = np.frombuffer(keys.encode(), dtype=np.uint8)          # UTF-8 bytes of the JSON
    path = os.path.join(ROOT, "tests", "golden", "bert_tiny.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB), {len(full.state_dict())} bert-base FrozenInTime keys")


if __name__ == "__main__":
    main()
