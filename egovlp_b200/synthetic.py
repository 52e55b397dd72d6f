"""Seeded synthetic weights and inputs (SURVEY.md section 8d) — no dataset, tokenizer or checkpoint needed.

`seeded_state_dict` produces a full FrozenInTime state_dict (reference key names and shapes,
SURVEY.md section 8b) from a CPU torch.Generator, so the reference module, the oracle and the
CUDA model can be loaded with identical weights on any machine of the same image.  All
temporal-attention weights are drawn non-zero (the reference's time_init='zeros' would hide
temporal-kernel bugs, SURVEY.md section 8a quirk 3).
"""
from collections import OrderedDict

import torch

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def model_dims(embed_dim=768, depth=12, heads=12, mlp_ratio=4, patch=16, img=224, num_frames=16,
               text_dim=768, text_layers=6, text_heads=12, text_hidden=3072, vocab=30522, max_pos=512,
               proj_dim=256, text_kind=None):
    """`text_kind='bert'`: a BERT text tower (token-type table, BERT key names, pooler); None = DistilBERT."""
    dims = dict(embed_dim=embed_dim, depth=depth, heads=heads, mlp_hidden=int(embed_dim * mlp_ratio), patch=patch,
                img=img, num_frames=num_frames, text_dim=text_dim, text_layers=text_layers, text_heads=text_heads,
                text_hidden=text_hidden, vocab=vocab, max_pos=max_pos, proj_dim=proj_dim)
    if text_kind is not None:
        dims["text_kind"] = text_kind
    return dims


# small geometry used by the tests: head_dim stays 64 (the attention kernels are specialised for it)
TINY_DIMS = model_dims(embed_dim=128, depth=2, heads=2, patch=16, img=32, num_frames=4, text_dim=128, text_layers=2,
                       text_heads=2, text_hidden=256, vocab=120, max_pos=32, proj_dim=32)


def _bert_shapes(dims, s):
    """transformers BertModel keys (token types 2, pooler) under text_model., in its registration order."""
    E, TH = dims["text_dim"], dims["text_hidden"]
    s["text_model.embeddings.word_embeddings.weight"] = (dims["vocab"], E)
    s["text_model.embeddings.position_embeddings.weight"] = (dims["max_pos"], E)
    s["text_model.embeddings.token_type_embeddings.weight"] = (2, E)
    s["text_model.embeddings.LayerNorm.weight"] = (E,)
    s["text_model.embeddings.LayerNorm.bias"] = (E,)
    for i in range(dims["text_layers"]):
        lp = f"text_model.encoder.layer.{i}."
        for lin in ("self.query", "self.key", "self.value", "output.dense"):
            s[lp + f"attention.{lin}.weight"] = (E, E)
            s[lp + f"attention.{lin}.bias"] = (E,)
        s[lp + "attention.output.LayerNorm.weight"] = (E,)
        s[lp + "attention.output.LayerNorm.bias"] = (E,)
        s[lp + "intermediate.dense.weight"] = (TH, E)
        s[lp + "intermediate.dense.bias"] = (TH,)
        s[lp + "output.dense.weight"] = (E, TH)
        s[lp + "output.dense.bias"] = (E,)
        s[lp + "output.LayerNorm.weight"] = (E,)
        s[lp + "output.LayerNorm.bias"] = (E,)
    s["text_model.pooler.dense.weight"] = (E, E)
    s["text_model.pooler.dense.bias"] = (E,)


def state_dict_shapes(dims, video=True, text=True, proj=True):
    """Ordered {key: shape} in the reference's registration order.  dims["img"]: an int, or an (H, W) pair."""
    D, H, P = dims["embed_dim"], dims["mlp_hidden"], dims["patch"]
    img = dims["img"] if isinstance(dims["img"], (tuple, list)) else (dims["img"], dims["img"])
    n = (img[0] // P) * (img[1] // P)
    s = OrderedDict()
    if text and dims.get("text_kind") == "bert":
        _bert_shapes(dims, s)
    elif text:
        E, TH = dims["text_dim"], dims["text_hidden"]
        s["text_model.embeddings.word_embeddings.weight"] = (dims["vocab"], E)
        s["text_model.embeddings.position_embeddings.weight"] = (dims["max_pos"], E)
        s["text_model.embeddings.LayerNorm.weight"] = (E,)
        s["text_model.embeddings.LayerNorm.bias"] = (E,)
        for i in range(dims["text_layers"]):
            lp = f"text_model.transformer.layer.{i}."
            for lin in ("q_lin", "k_lin", "v_lin", "out_lin"):
                s[lp + f"attention.{lin}.weight"] = (E, E)
                s[lp + f"attention.{lin}.bias"] = (E,)
            s[lp + "sa_layer_norm.weight"] = (E,)
            s[lp + "sa_layer_norm.bias"] = (E,)
            s[lp + "ffn.lin1.weight"] = (TH, E)
            s[lp + "ffn.lin1.bias"] = (TH,)
            s[lp + "ffn.lin2.weight"] = (E, TH)
            s[lp + "ffn.lin2.bias"] = (E,)
            s[lp + "output_layer_norm.weight"] = (E,)
            s[lp + "output_layer_norm.bias"] = (E,)
    if video:
        s["video_model.cls_token"] = (1, 1, D)
        s["video_model.pos_embed"] = (1, n + 1, D)
        s["video_model.temporal_embed"] = (1, dims["num_frames"], D)
        s["video_model.patch_embed.proj.weight"] = (D, 3, P, P)
        s["video_model.patch_embed.proj.bias"] = (D,)
        for i in range(dims["depth"]):
            bp = f"video_model.blocks.{i}."
            s[bp + "norm1.weight"] = (D,)
            s[bp + "norm1.bias"] = (D,)
            for a in ("attn", "timeattn"):
                s[bp + a + ".qkv.weight"] = (3 * D, D)
                s[bp + a + ".qkv.bias"] = (3 * D,)
                s[bp + a + ".proj.weight"] = (D, D)
                s[bp + a + ".proj.bias"] = (D,)
            s[bp + "norm2.weight"] = (D,)
            s[bp + "norm2.bias"] = (D,)
            s[bp + "mlp.fc1.weight"] = (H, D)
            s[bp + "mlp.fc1.bias"] = (H,)
            s[bp + "mlp.fc2.weight"] = (D, H)
            s[bp + "mlp.fc2.bias"] = (D,)
            s[bp + "norm3.weight"] = (D,)
            s[bp + "norm3.bias"] = (D,)
        s["video_model.norm.weight"] = (D,)
        s["video_model.norm.bias"] = (D,)
    if proj:
        s["txt_proj.1.weight"] = (dims["proj_dim"], dims["text_dim"])
        s["txt_proj.1.bias"] = (dims["proj_dim"],)
        s["vid_proj.0.weight"] = (dims["proj_dim"], D)
        s["vid_proj.0.bias"] = (dims["proj_dim"],)
    return s


def seeded_state_dict(dims, seed=0, video=True, text=True, proj=True, dtype=torch.float32):
    """Deterministic weights: matrices ~ N(0, fan_in^-1/2 * 0.8) (keeps activations O(1) through depth),
    LayerNorm weight ~ 1 + 0.1 N, biases / embeddings ~ 0.02 N, word embeddings ~ 0.05 N."""
    g = torch.Generator().manual_seed(1234567 + seed)
    out = OrderedDict()
    for k, shp in state_dict_shapes(dims, video, text, proj).items():
        r = torch.randn(shp, generator=g, dtype=torch.float32)
        leaf = k.rsplit(".", 2)
        if k.endswith("LayerNorm.weight") or "norm" in leaf[-2] and k.endswith(".weight"):
            t = 1.0 + 0.1 * r
        elif k.endswith(".bias"):
            t = 0.02 * r
        elif "word_embeddings" in k or "position_embeddings" in k or "token_type_embeddings" in k:
            t = 0.05 * r
        elif k.endswith(("cls_token", "pos_embed", "temporal_embed")):
            t = 0.02 * r
        else:
            fan_in = 1
            for d_ in shp[1:]:
                fan_in *= d_
            t = r * (0.8 / fan_in ** 0.5)
        out[k] = t.to(dtype)
    return out


def synthetic_video(B, T, seed=0, img=224, device="cpu"):
    """rand -> ImageNet-normalised, values about U(-2.1, 2.6) (data_loader/transforms.py:38-41).  img: an int, or an
    (H, W) pair."""
    g = torch.Generator().manual_seed(77 + seed)
    hw = tuple(img) if isinstance(img, (tuple, list)) else (img, img)
    v = torch.rand(B, T, 3, *hw, generator=g)
    mean = torch.tensor(IMAGENET_MEAN).view(1, 1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD).view(1, 1, 3, 1, 1)
    return ((v - mean) / std).to(device)


def synthetic_text(B, L, seed=0, ragged=False, vocab=30522, device="cpu"):
    """input_ids with CLS=101 first, SEP=102 last valid; attention_mask ones or ragged (lengths 3..L)."""
    g = torch.Generator().manual_seed(991 + seed)
    hi = min(30000, vocab)
    lo = min(1000, hi - 1)
    ids = torch.randint(lo, hi, (B, L), generator=g)
    mask = torch.ones(B, L, dtype=torch.int64)
    lens = torch.full((B,), L, dtype=torch.int64)
    if ragged:
        lens = torch.randint(min(3, L), L + 1, (B,), generator=g)
        lens[0] = L
    for b in range(B):
        n = int(lens[b])
        ids[b, 0] = min(101, vocab - 2)
        ids[b, n - 1] = min(102, vocab - 1)
        ids[b, n:] = 0
        mask[b, n:] = 0
    return {"input_ids": ids.to(device), "attention_mask": mask.to(device)}


def synthetic_tags(B, seed=0, n_verb=118, n_noun=582, device="cpu", zero_noun_row=True):
    """Multi-hot verb (1 per sample) / noun (1-3 per sample) vectors, Zipf-like so a few % of pairs
    are positives; optionally one all-zero noun row to exercise sim_matrix's eps clamp."""
    g = torch.Generator().manual_seed(4242 + seed)

    def zipf(n, count):
        w = 1.0 / torch.arange(1, n + 1, dtype=torch.float32)
        return torch.multinomial(w / w.sum(), count, replacement=False, generator=g)

    verb = torch.zeros(B, n_verb)
    noun = torch.zeros(B, n_noun)
    for b in range(B):
        verb[b, zipf(n_verb, 1)] = 1.0
        k = int(torch.randint(1, 4, (1,), generator=g))
        noun[b, zipf(n_noun, k)] = 1.0
    if zero_noun_row and B > 2:
        noun[B - 1] = 0.0
    return verb.to(device), noun.to(device)
