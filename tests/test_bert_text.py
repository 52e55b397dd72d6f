"""BERT text tower (`text_params['model'] = 'bert*'`), host side: the fp32 oracle (oracle/bert_port.py) against the
unmodified reference's recording tests/golden/bert_tiny.npz, FrozenInTime's construction, state_dict keys and
refusals.  The CUDA path is checked in test_bert_text_gpu.py."""
import json
import warnings

import pytest
import torch

from conftest import load_golden


def tiny_dims():
    from egovlp_b200 import synthetic as syn
    return dict(syn.TINY_DIMS, max_pos=512, text_kind="bert")


def close(a, b, rtol=1e-4, atol=1e-5):
    torch.testing.assert_close(a.float(), b.float(), rtol=rtol, atol=atol)


VIDEO = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 4, "pretrained": True,
         "time_init": "zeros"}


def build(name, **kw):
    from egovlp_b200.model.model import FrozenInTime
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return FrozenInTime(VIDEO, {"model": name, "pretrained": True, "input": "text"}, **kw)


def test_oracle_vs_reference_bert_golden():
    """bert_port.compute_text / compute_text_tokens (both projections) and the gradient of every text parameter and
    txt_proj reproduce the reference's FrozenInTime with a tiny BertModel at L = 9 and 200 (ragged), at the fp32
    tolerances of test_oracle_vs_live_reference.py."""
    from egovlp_b200 import synthetic as syn
    from oracle import bert_port as bp
    g = load_golden("bert_tiny.npz")
    sd = syn.seeded_state_dict(tiny_dims(), seed=int(g["seed"]), video=False, proj=True)
    sd = {k: v.clone().requires_grad_(True) for k, v in sd.items() if not k.startswith("vid_proj")}
    pgen = torch.Generator().manual_seed(31)
    loss = 0
    for B, L in ((5, 9), (4, 200)):
        text = {"input_ids": g[f"l{L}/input_ids"], "attention_mask": g[f"l{L}/attention_mask"]}
        t = bp.compute_text(text, sd, heads=2)
        close(t, g[f"l{L}/text"])
        with torch.no_grad():
            close(bp.compute_text_tokens(text, sd, heads=2), g[f"l{L}/tokens"])
            close(bp.compute_text(text, sd, heads=2, projection=""), g[f"l{L}/pooled"])
        loss = loss + (t * torch.randn(B, 32, generator=pgen)).sum()
    loss.backward()
    for k, v in sd.items():
        gr = v.grad if v.grad is not None else torch.zeros_like(v)
        close(gr.flatten()[g[f"grad/{k}/idx"].long()], g[f"grad/{k}/val"], rtol=5e-4, atol=5e-5)
        # (+1e-6: the key biases' gradients are rounding noise, zero analytically by softmax shift invariance)
        assert abs(gr.double().norm().item() - g[f"grad/{k}/norm"].item()) <= 5e-4 * g[f"grad/{k}/norm"].item() + 1e-6, k


def test_frozen_in_time_bert_base_keys_are_the_references():
    """A bert-base-uncased FrozenInTime builds on the CPU (random init without local files) with the reference's 426
    state_dict keys and shapes, in order, and a reference-keyed state dict loads with strict=True."""
    from egovlp_b200 import synthetic as syn
    g = load_golden("bert_tiny.npz")
    want = [(k, tuple(s)) for k, s in json.loads(bytes(g["bert_base_keys_json"].numpy()).decode())]
    net = build("bert-base-uncased")
    got = [(k, tuple(v.shape)) for k, v in net.state_dict().items()]
    assert len(got) == 426 and got == want
    dims = syn.model_dims(num_frames=4, text_layers=12, text_kind="bert")
    assert list(syn.state_dict_shapes(dims).items()) == want
    net.load_state_dict(syn.seeded_state_dict(dims, seed=1), strict=True)
    assert net.text_model.config.layer_norm_eps == 1e-12


@pytest.mark.parametrize("name, dims", [("bert-base-cased", (768, 12, 12, 3072, 28996)),
                                        ("bert-large-uncased", (1024, 24, 16, 4096, 30522))])
def test_named_architectures_without_files(name, dims):
    from egovlp_b200.model.model import _build_bert
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        tm = _build_bert(name)
    assert any("randomly initialised" in str(x.message) for x in w)
    c = tm.config
    assert (c.hidden_size, c.num_hidden_layers, c.num_attention_heads, c.intermediate_size, c.vocab_size) == dims


def test_bert_large_state_dict_has_618_tensors():
    from egovlp_b200 import synthetic as syn
    dims = syn.model_dims(text_dim=1024, text_layers=24, text_heads=16, text_hidden=4096, text_kind="bert")
    assert len(syn.state_dict_shapes(dims)) == 618


def test_refusals():
    """Names the reference cannot embed, and BERT configs the CUDA tower does not run, raise NotImplementedError at
    construction, naming the field."""
    from transformers import BertConfig, BertModel
    from egovlp_b200.model import model as mm
    with pytest.raises(NotImplementedError, match="roberta-base"):
        build("roberta-base")
    with pytest.raises(NotImplementedError, match="no local files"):
        build("bert-tiny-unknown")
    base = dict(vocab_size=120, hidden_size=128, num_hidden_layers=1, num_attention_heads=2, intermediate_size=256)
    mm._check_bert(BertModel(BertConfig(**base)))
    bad = [(dict(num_attention_heads=4), "num_attention_heads"), (dict(hidden_act="relu"), "hidden_act"),
           (dict(position_embedding_type="relative_key"), "position_embedding_type"),
           (dict(is_decoder=True), "is_decoder")]
    for change, field in bad:
        with pytest.raises(NotImplementedError, match=field):
            mm._check_bert(BertModel(BertConfig(**dict(base, **change))))
    with pytest.raises(NotImplementedError, match="hidden_size"):
        mm._check_bert(BertModel(BertConfig(**dict(base, hidden_size=1088, num_attention_heads=17))))
    with pytest.raises(NotImplementedError, match="pooler"):
        mm._check_bert(BertModel(BertConfig(**base), add_pooling_layer=False))
