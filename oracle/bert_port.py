"""CPU / GPU restatement (torch fp32, functional) of the reference's `bert*` text tower.  TEST INFRASTRUCTURE ONLY.

The reference builds it with `AutoModel.from_pretrained(text_params['model'])` and embeds a caption with
`text_model(input_ids, attention_mask=...)['pooler_output']` (model/model.py:34-35, :117-131); its
compute_text_tokens returns the same pooled tensor ("not implement for bert", :129-131).  The BertModel graph
(transformers modeling_bert.py: BertEmbeddings, post-LN BertLayer, BertPooler) is restated here from the published
architecture and pinned against the unmodified reference run through oracle/ref_shim.py
(``oracle/make_bert_golden.py`` -> ``tests/golden/bert_tiny.npz``).  DistilBERT stays in oracle/reference_port.py.

Weights are a flat mapping with the reference's FrozenInTime key names (``text_model.embeddings...``,
``text_model.encoder.layer.{i}...``, ``text_model.pooler.dense...``, ``txt_proj.1...``).
"""
import math

import torch
import torch.nn.functional as F

from oracle import reference_port as rp


def bert_forward(input_ids, attention_mask, p, heads=12, prefix="text_model.", eps=1e-12, dropout=None):
    """BertModel: returns (last_hidden_state [B, L, D], pooler_output [B, D]).

    No token_type_ids are passed by the reference, so every token adds row 0 of the token-type table.  `dropout` =
    None (eval / p = 0) or a dict of MULTIPLIERS (mask / (1 - p)) for BERT's four train-mode dropout sites: "emb"
    [B, L, D] on the embedding LayerNorm output, ("att", layer) [B, H, L, L] on the attention probabilities,
    ("so", layer) [B, L, D] on the attention output dense (BertSelfOutput), ("ffn", layer) [B, L, D] on the FFN output
    dense (BertOutput)."""
    B, L = input_ids.shape
    we = p[prefix + "embeddings.word_embeddings.weight"]
    pe = p[prefix + "embeddings.position_embeddings.weight"]
    te = p[prefix + "embeddings.token_type_embeddings.weight"]
    D = we.shape[1]
    d = D // heads
    x = we[input_ids] + pe[:L].unsqueeze(0) + te[0]
    x = F.layer_norm(x, (D,), p[prefix + "embeddings.LayerNorm.weight"], p[prefix + "embeddings.LayerNorm.bias"], eps)
    if dropout is not None:
        x = x * dropout["emb"]
    key_bias = torch.zeros(B, 1, 1, L, dtype=x.dtype, device=x.device)
    key_bias = key_bias.masked_fill(attention_mask.reshape(B, 1, 1, L) == 0, float("-inf"))
    n_layers = 1 + max(int(k.split("encoder.layer.")[1].split(".")[0]) for k in p if "encoder.layer." in k)
    for i in range(n_layers):
        lp = f"{prefix}encoder.layer.{i}."

        def heads_of(t):
            return t.reshape(B, L, heads, d).transpose(1, 2)

        q = heads_of(rp._linear(x, p[lp + "attention.self.query.weight"], p[lp + "attention.self.query.bias"]))
        k = heads_of(rp._linear(x, p[lp + "attention.self.key.weight"], p[lp + "attention.self.key.bias"]))
        v = heads_of(rp._linear(x, p[lp + "attention.self.value.weight"], p[lp + "attention.self.value.bias"]))
        w = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d) + key_bias, dim=-1)
        if dropout is not None:
            w = w * dropout[("att", i)]
        ctx = (w @ v).transpose(1, 2).reshape(B, L, D)
        so = rp._linear(ctx, p[lp + "attention.output.dense.weight"], p[lp + "attention.output.dense.bias"])
        if dropout is not None:
            so = so * dropout[("so", i)]
        x = F.layer_norm(so + x, (D,), p[lp + "attention.output.LayerNorm.weight"],
                         p[lp + "attention.output.LayerNorm.bias"], eps)
        h = F.gelu(rp._linear(x, p[lp + "intermediate.dense.weight"], p[lp + "intermediate.dense.bias"]))
        h = rp._linear(h, p[lp + "output.dense.weight"], p[lp + "output.dense.bias"])
        if dropout is not None:
            h = h * dropout[("ffn", i)]
        x = F.layer_norm(h + x, (D,), p[lp + "output.LayerNorm.weight"], p[lp + "output.LayerNorm.bias"], eps)
    pooled = torch.tanh(rp._linear(x[:, 0], p[prefix + "pooler.dense.weight"], p[prefix + "pooler.dense.bias"]))
    return x, pooled


def compute_text(text, p, heads=12, dropout=None, kind="bert", projection="minimal", eps=1e-12):
    """FrozenInTime.compute_text (model/model.py:117-126) for either tower: kind='bert' -> pooler_output, otherwise
    DistilBERT's CLS row (oracle/reference_port.py); then txt_proj = ReLU -> Linear, or nothing for projection=''."""
    if kind == "bert":
        h = bert_forward(text["input_ids"], text["attention_mask"], p, heads, eps=eps, dropout=dropout)[1]
    else:
        h = rp.distilbert_forward(text["input_ids"], text["attention_mask"], p, heads, eps=eps, dropout=dropout)[:, 0]
    if projection == "":
        return h
    return rp._linear(torch.relu(h), p["txt_proj.1.weight"], p["txt_proj.1.bias"])


def compute_text_tokens(text, p, heads=12, dropout=None, kind="bert", projection="minimal", eps=1e-12):
    """FrozenInTime.compute_text_tokens (model/model.py:128-138): for BERT the reference returns the pooled, projected
    [B, P] tensor, exactly compute_text's result."""
    if kind == "bert":
        return compute_text(text, p, heads, dropout, kind, projection, eps)
    h = rp.distilbert_forward(text["input_ids"], text["attention_mask"], p, heads, eps=eps, dropout=dropout)
    if projection == "":
        return h
    return rp._linear(torch.relu(h), p["txt_proj.1.weight"], p["txt_proj.1.bias"])


def frozen_in_time_forward(data, p, heads=12, text_heads=12, kind="bert"):
    """FrozenInTime.forward (model/model.py:100-115) with the given text tower; returns (text, video)."""
    return compute_text(data["text"], p, text_heads, kind=kind), rp.compute_video(data["video"], p, heads)
