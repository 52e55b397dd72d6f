"""Text tower above 128 tokens, up to DistilBERT's 512 positions: the tiled text attention (text_attn_long_*,
csrc/text_attention.cu) and the tower that dispatches to it for L > 128.

  * the fp32 oracle against HF DistilBertModel on tests/golden/distilbert_long.npz (CPU);
  * the kernel against float64, element by element, at the bounds of tests/divided_attention_ref.py, over ragged,
    holed and nearly empty masks, with a planted score maximum in the last valid key tile;
  * bitwise reproducibility, batch-position independence, the documented dropout keep mask regenerated on the host,
    argument refusals and the position-table check of the tower;
  * the tower against the golden and, at DistilBERT-base geometry, against the fp32 oracle on the GPU; dropout through
    the tower; one FrozenInTime training step with a 300-token caption."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from divided_attention_ref import Q_SCALE, SENTINEL, SLACK, U, _with_sentinels
from kernel_checks import BF16, F32, F64, assert_bits_equal, assert_elementwise_bound, nan_filled

P_ORDER_LAYER = ("attention.q_lin", "attention.k_lin", "attention.v_lin", "attention.out_lin")


@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


def long_dims():
    """The golden's geometry: the tiny test DistilBERT (dim 128, 2 heads, 2 layers) with 512 positions."""
    from egovlp_b200 import synthetic as syn
    return dict(syn.TINY_DIMS, max_pos=512)


def param_order(n_layers, proj=True):
    order = ["text_model.embeddings.word_embeddings.weight", "text_model.embeddings.position_embeddings.weight",
             "text_model.embeddings.LayerNorm.weight", "text_model.embeddings.LayerNorm.bias"]
    for i in range(n_layers):
        lp = f"text_model.transformer.layer.{i}."
        for lin in P_ORDER_LAYER:
            order += [lp + lin + ".weight", lp + lin + ".bias"]
        order += [lp + "sa_layer_norm.weight", lp + "sa_layer_norm.bias", lp + "ffn.lin1.weight", lp + "ffn.lin1.bias",
                  lp + "ffn.lin2.weight", lp + "ffn.lin2.bias", lp + "output_layer_norm.weight",
                  lp + "output_layer_norm.bias"]
    return order + (["txt_proj.1.weight", "txt_proj.1.bias"] if proj else [])


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def cos(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-300)).item()


# ------------------------------------------------------------------------------------------------ oracle vs golden
def test_oracle_vs_distilbert_long_golden():
    """oracle/reference_port.distilbert_forward reproduces HF DistilBertModel at L = 512 and 200 (ragged lengths 512,
    300, 129, 65, 7 and a holed mask), every hidden state, at fp32 rounding level."""
    from egovlp_b200 import synthetic as syn
    from oracle import reference_port as rp
    g = load_golden("distilbert_long.npz")
    sd = syn.seeded_state_dict(long_dims(), seed=int(g["seed"]), video=False, proj=False)
    for L, tag in ((512, "l512"), (200, "l200")):
        ids, mask = g["input_ids"][:, :L], g["attention_mask"][:, :L]
        bi, li = g[f"{tag}_rows_b"].long(), g[f"{tag}_rows_l"].long()
        emb = sd["text_model.embeddings.word_embeddings.weight"][ids] + sd["text_model.embeddings.position_embeddings.weight"][:L]
        hs = [torch.nn.functional.layer_norm(emb, (emb.shape[-1],), sd["text_model.embeddings.LayerNorm.weight"],
                                             sd["text_model.embeddings.LayerNorm.bias"], 1e-12)]
        for n in (1, 2):
            part = {k: v for k, v in sd.items() if "transformer.layer." not in k or int(k.split("layer.")[1].split(".")[0]) < n}
            hs.append(rp.distilbert_forward(ids, mask, part, heads=2))
        for i, h in enumerate(hs):
            torch.testing.assert_close(h[:, 0], g[f"{tag}_cls"][i], rtol=1e-4, atol=1e-5)
            torch.testing.assert_close(h[bi, li], g[f"{tag}_rows"][i], rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------------ host Philox
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(key, ctr):
    """common.cuh philox4x32_10 on uint64 numpy arrays of counters -> the four 32-bit words."""
    k0, k1 = np.uint64(key & 0xFFFFFFFF), np.uint64(key >> 32)
    c0, c1 = ctr & _M32, ctr >> np.uint64(32)
    c2, c3 = np.full_like(ctr, 0x2B7E1516), np.full_like(ctr, 0x28AED2A6)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
    return c0, c1, c2, c3


def keep_mask(seed, site, p, B, H, L):
    """The documented keep mask of text_attn_long_*: bool [B, H, L(i), L(j)]."""
    key = (seed ^ ((0x9E3779B97F4A7C15 * (site + 1)) & 0xFFFFFFFFFFFFFFFF)) & 0xFFFFFFFFFFFFFFFF
    t = float(np.float32(p)) * 4294967296.0
    thresh = 0xFFFFFFFF if t >= 4294967295.0 else int(t)
    b, h, i, jg = np.meshgrid(np.arange(B, dtype=np.uint64), np.arange(H, dtype=np.uint64), np.arange(L, dtype=np.uint64),
                              np.arange((L + 3) // 4, dtype=np.uint64), indexing="ij")
    words = philox4x32_10(key, ((b * np.uint64(4096) + h) * np.uint64(512) + i) * np.uint64(128) + jg)
    keep = np.stack([w >= np.uint64(thresh) for w in words], -1).reshape(B, H, L, -1)[..., :L]
    return torch.from_numpy(keep)


def multiplier(seed, site, p, B, H, L):
    return keep_mask(seed, site, p, B, H, L).double() / (1 - p)


# ------------------------------------------------------------------------------------------------ kernel harness
def reference(qkv, dout, mask, B, L, H, q_scale, mult=None):
    """float64 masked attention (dropout multipliers `mult` [B, H, L, L] on the probabilities) and the magnitude sums
    of the bounds (DESIGN section 6 forms, as tests/divided_attention_ref.py)."""
    x = qkv.to(F64).view(B, L, 3, H, 64).permute(2, 0, 3, 1, 4)
    q, k, v = x[0], x[1], x[2]
    do = dout.to(F64).view(B, L, H, 64).permute(0, 2, 1, 3)
    valid = mask.bool().view(B, 1, 1, L)
    s = (q @ k.transpose(-1, -2)).masked_fill(~valid, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    m = mult.to(qkv.device) if mult is not None else torch.ones((), dtype=F64, device=qkv.device)
    pd = p * m
    o = pd @ v
    pv = pd @ v.abs()
    dp = (do @ v.transpose(-1, -2)) * m
    delta = (do * o).sum(-1, keepdim=True)
    ds = p * (dp - delta)
    e = (do.abs() * (pv + 2 * o.abs())).sum(-1, keepdim=True)
    w = p * ((dp - delta).abs() + e)
    lse_t = (q.abs() @ k.abs().transpose(-1, -2)).masked_fill(~valid, 0.0).amax(-1)
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(B * L, H * 64)
    return {"out": rows(o), "out_t": rows(pv), "lse": lse, "lse_t": lse_t,
            "dq": rows(q_scale * (ds @ k)), "dq_t": rows(q_scale * (w @ k.abs())),
            "dk": rows(ds.transpose(-1, -2) @ q), "dk_t": rows(w.transpose(-1, -2) @ q.abs()),
            "dv": rows(pd.transpose(-1, -2) @ do), "dv_t": rows(pd.transpose(-1, -2) @ do.abs())}


def make_inputs(B, L, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = 64 * H
    x = torch.randn(B * L, 3 * D, generator=g, device="cuda")
    x[:, :D] *= Q_SCALE
    return x.to(BF16), torch.randn(B * L, D, generator=g, device="cuda").to(BF16)


def plant_last_tile_maxima(qkv, mask, B, L, H, score=18.0):
    """Every third query row points at its sample's last valid key (in the last valid key tile), `score` above the
    rest: the running maximum changes in the last tile, so the online rescaling is exercised."""
    x = qkv.float().view(B, L, 3, H, 64)
    for b in range(B):
        last = int(mask[b].nonzero().max())
        kk = x[b, last, 1]                                         # [H, 64]
        x[b, ::3, 0] = (kk * (score / kk.pow(2).sum(-1, keepdim=True)))[None]
    return x.reshape(B * L, 3 * H * 64).to(BF16)


def masks_for(L):
    """full; one valid key; lengths around 64-key tile edges; holes (a non-prefix pattern); 5 valid keys."""
    j = torch.arange(L)
    rows = [torch.ones(L, dtype=torch.int64), (j == (L - 1) // 2).long()]
    for n in (63, 64, 65, L - 1):
        rows.append((j < max(1, min(L, n))).long())
    holes = ((j % 7 != 3) & ~((j >= 64) & (j < 128))).long()
    holes[0] = 1
    rows += [holes, (j < 5).long()]
    return torch.stack(rows).cuda()


def run_long(ops, qkv, dout, mask, B, L, H, q_scale=Q_SCALE, p=0.0, seed=0, site=0):
    """Forward into NaN-filled buffers with sentinel rows, backward likewise; checks every element of the outputs was
    written and no sentinel changed; returns (out, lse [B, H, L], dqkv)."""
    D = 64 * H
    M = B * L
    out_buf, lse_buf, dq_buf = _with_sentinels(M, D, BF16), _with_sentinels(B * H, L, F32), _with_sentinels(M, 3 * D, BF16)
    ops.text_attn_long_fwd(qkv, mask, out_buf, lse_buf, B, L, H, p, seed, site)
    out, lse = out_buf[:M], lse_buf[:B * H].view(B, H, L)
    ops.text_attn_long_bwd(qkv, mask, out, lse, dout, dq_buf, B, L, H, q_scale, p, seed, site)
    torch.cuda.synchronize()
    for name, buf, rows in (("out", out_buf, M), ("lse", lse_buf, B * H), ("dqkv", dq_buf, M)):
        assert not buf[:rows].isnan().any(), f"{name}: {int(buf[:rows].isnan().sum())} elements left unwritten"
        assert bool((buf[rows:] == SENTINEL).all()), f"{name}: a row past the output was written"
    return out, lse, dq_buf[:M]


def check(tag, qkv, dout, mask, out, lse, dqkv, B, L, H, mult=None):
    D = 64 * H
    r = reference(qkv, dout, mask, B, L, H, Q_SCALE, mult)
    assert_elementwise_bound(f"out {tag}", out, r["out"], SLACK * U * (r["out_t"] + 2 * r["out"].abs()))
    assert_elementwise_bound(f"lse {tag}", lse, r["lse"], SLACK * (2e-5 * r["lse_t"] + 1e-6 * (1 + r["lse"].abs())))
    for i, name in enumerate(("dq", "dk", "dv")):
        assert_elementwise_bound(f"{name} {tag}", dqkv[:, i * D:(i + 1) * D], r[name],
                                 SLACK * U * (r[name + "_t"] + r[name].abs()))
    pad = (mask.view(-1) == 0)
    assert bool((dqkv[pad, D:] == 0).all()), f"{tag}: dk / dv of padded keys not exactly 0"


LS = [1, 63, 64, 65, 128, 129, 192, 255, 256, 257, 384, 511, 512]


@pytest.mark.gpu
@pytest.mark.parametrize("H", [1, 12])
@pytest.mark.parametrize("L", LS)
def test_text_attn_long_vs_fp64(ops, L, H):
    mask = masks_for(L)
    B = mask.shape[0]
    qkv, dout = make_inputs(B, L, H, seed=L * 31 + H)
    qkv = plant_last_tile_maxima(qkv, mask, B, L, H)
    out, lse, dqkv = run_long(ops, qkv, dout, mask, B, L, H)
    check(f"L={L} H={H}", qkv, dout, mask, out, lse, dqkv, B, L, H)


@pytest.mark.gpu
def test_text_attn_long_one_caption_padded_to_512(ops):
    """One sample of 5 valid keys next to a full one at L = 512: its 7 empty key tiles are skipped, same bounds."""
    B, L, H = 2, 512, 12
    mask = torch.ones(B, L, dtype=torch.int64, device="cuda")
    mask[1, 5:] = 0
    qkv, dout = make_inputs(B, L, H, seed=5)
    out, lse, dqkv = run_long(ops, qkv, dout, mask, B, L, H)
    check("padded to 512", qkv, dout, mask, out, lse, dqkv, B, L, H)


@pytest.mark.gpu
def test_text_attn_long_empty_mask_gives_nan_rows_only_there(ops):
    """A sample without a valid key (never produced by a tokenizer) must not fault nor touch its neighbours: NaN rows
    in out and lse, zero gradients, the other samples as computed alone."""
    B, L, H = 3, 200, 2
    D = 64 * H
    mask = torch.ones(B, L, dtype=torch.int64, device="cuda")
    mask[1] = 0
    qkv, dout = make_inputs(B, L, H, seed=9)
    out, lse = torch.empty(B * L, D, device="cuda", dtype=BF16), torch.empty(B, H, L, device="cuda")
    ops.text_attn_long_fwd(qkv, mask, out, lse, B, L, H)
    dq = torch.empty(B * L, 3 * D, device="cuda", dtype=BF16)
    ops.text_attn_long_bwd(qkv, mask, out, lse, dout, dq, B, L, H, Q_SCALE)
    rows = slice(L, 2 * L)
    assert bool(out[rows].isnan().all()) and bool(lse[1].isnan().all())
    assert bool((dq[rows] == 0).all())
    keep = torch.tensor([0, 2], device="cuda")
    sub = lambda t: t.view(B, L, -1)[keep].reshape(2 * L, -1)
    o2, l2, d2 = run_long(ops, sub(qkv), sub(dout), mask[keep], 2, L, H)
    assert_bits_equal("out beside an empty sample", sub(out), o2)
    assert_bits_equal("dqkv beside an empty sample", sub(dq), d2)


@pytest.mark.gpu
@pytest.mark.parametrize("L", [129, 300, 512])
def test_text_attn_long_bitwise_reproducible_and_batch_position_independent(ops, L):
    B, H = 8, 12
    j = torch.arange(L, device="cuda")
    lens = torch.tensor([L, 3, L - 1, 64, 65, 130, 7, L // 2], device="cuda")
    mask = (j[None] < lens[:, None]).long()
    qkv, dout = make_inputs(B, L, H, seed=L)
    a, b = run_long(ops, qkv, dout, mask, B, L, H), run_long(ops, qkv, dout, mask, B, L, H)
    for name, x, y in zip(("out", "lse", "dqkv"), a, b):
        assert_bits_equal(f"{name} run to run L={L}", x, y)
    for s in (0, 5):
        one = run_long(ops, qkv.view(B, L, -1)[s].contiguous(), dout.view(B, L, -1)[s].contiguous(),
                       mask[s:s + 1].contiguous(), 1, L, H)
        assert_bits_equal(f"out sample {s} alone L={L}", one[0], a[0].view(B, L, -1)[s])
        assert_bits_equal(f"lse sample {s} alone L={L}", one[1][0], a[1][s])
        assert_bits_equal(f"dqkv sample {s} alone L={L}", one[2], a[2].view(B, L, -1)[s])
    # a caller's p = 0 with any (seed, site) is the dropout-free call
    c = run_long(ops, qkv, dout, mask, B, L, H, p=0.0, seed=123456789, site=9)
    for name, x, y in zip(("out", "lse", "dqkv"), a, c):
        assert_bits_equal(f"{name} p=0 L={L}", x, y)


# ------------------------------------------------------------------------------------------------ dropout
def extract_keep(ops, B, L, H, p, seed, site):
    """The kernel's keep mask [B, H, L, L] read back through the forward: q = k = 0 makes the softmax uniform over the
    valid keys; a 64-key window of valid keys with v = one-hot of the key's offset makes output column d of row i equal
    keep(i, j0 + d) / (1 - p) / 64."""
    D = 64 * H
    qkv = torch.zeros(B * L, 3 * D, device="cuda", dtype=BF16)
    keep = torch.zeros(B, H, L, L, dtype=torch.bool)
    j = torch.arange(L, device="cuda")
    for j0 in range(0, L, 64):
        n = min(64, L - j0)
        v = qkv.view(B, L, 3, H, 64)[:, :, 2]
        v.zero_()
        v[:, j0:j0 + n, :, :] = torch.eye(64, device="cuda", dtype=BF16)[:n, None, :]
        mask = ((j >= j0) & (j < j0 + n)).long()[None].expand(B, L).contiguous()
        out, lse = torch.empty(B * L, D, device="cuda", dtype=BF16), torch.empty(B, H, L, device="cuda")
        ops.text_attn_long_fwd(qkv, mask, out, lse, B, L, H, p, seed, site)
        o = out.float().view(B, L, H, 64)[..., :n].permute(0, 2, 1, 3) * n   # kept -> 1 / (1 - p), dropped -> 0
        keep[..., j0:j0 + n] = (o > 0.5).cpu()
    return keep


@pytest.mark.gpu
def test_attention_dropout_mask_is_the_documented_philox_stream_with_proper_statistics(ops):
    B, L, H, p, seed, site = 2, 512, 4, 0.1, 0x1234_5678_9ABC, 3
    kern = extract_keep(ops, B, L, H, p, seed, site)
    host = keep_mask(seed, site, p, B, H, L)
    assert torch.equal(kern, host), f"{int((kern != host).sum())} of {kern.numel()} keep bits differ from the host Philox"
    n = host.numel()                                                       # 2.1M draws
    rate = host.double().mean().item()
    assert abs(rate - (1 - p)) < 3 * (p * (1 - p) / n) ** 0.5, rate
    for other in (keep_mask(seed, site + 1, p, B, H, L), keep_mask(seed + 1, site, p, B, H, L)):
        agree = (other == host).double().mean().item()                      # independent: (1-p)^2 + p^2
        want = (1 - p) ** 2 + p ** 2
        assert abs(agree - want) < 3 * (want * (1 - want) / n) ** 0.5 + 1e-4, agree
    blocks = host.view(-1, 4096).double().mean(1)                           # no structure along the index
    assert (blocks - (1 - p)).abs().max().item() < 0.03


@pytest.mark.gpu
@pytest.mark.parametrize("L", [129, 512])
def test_text_attn_long_dropout_vs_fp64_with_the_host_mask(ops, L):
    B, H, p, seed, site = 3, 2, 0.2, 987654321, 5
    j = torch.arange(L, device="cuda")
    mask = (j[None] < torch.tensor([L, L - 70, 9], device="cuda")[:, None]).long()
    qkv, dout = make_inputs(B, L, H, seed=77 + L)
    out, lse, dqkv = run_long(ops, qkv, dout, mask, B, L, H, p=p, seed=seed, site=site)
    mult = multiplier(seed, site, p, B, H, L)
    check(f"dropout L={L}", qkv, dout, mask, out, lse, dqkv, B, L, H, mult=mult)
    again = run_long(ops, qkv, dout, mask, B, L, H, p=p, seed=seed, site=site)
    for name, x, y in zip(("out", "lse", "dqkv"), (out, lse, dqkv), again):
        assert_bits_equal(f"{name} dropout run to run L={L}", x, y)


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.gpu
@pytest.mark.parametrize("L,p", [(0, 0.0), (513, 0.0), (64, 1.0), (200, -0.1), (200, float("nan"))])
def test_text_attn_long_refuses_bad_arguments_and_writes_nothing(ops, L, p):
    from egovlp_b200._lib import EgovlpError
    B, H = 2, 2
    Ln = max(L, 1)
    qkv = torch.zeros(B * Ln, 3 * 64 * H, device="cuda", dtype=BF16)
    mask = torch.ones(B, Ln, dtype=torch.int64, device="cuda")
    out, lse = nan_filled((B * Ln, 64 * H), BF16), nan_filled((B, H, Ln), F32)
    dq, dout = nan_filled((B * Ln, 3 * 64 * H), BF16), torch.zeros(B * Ln, 64 * H, device="cuda", dtype=BF16)
    with pytest.raises(EgovlpError):
        ops.text_attn_long_fwd(qkv, mask, out, lse, B, L, H, p)
    with pytest.raises(EgovlpError):
        ops.text_attn_long_bwd(qkv, mask, out, lse, dout, dq, B, L, H, Q_SCALE, p)
    torch.cuda.synchronize()
    assert bool(out.isnan().all()) and bool(lse.isnan().all()) and bool(dq.isnan().all())


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["tiny", "full"])
def test_tower_refuses_captions_longer_than_the_position_table_before_any_launch(size):
    from egovlp_b200 import _lib, engine, synthetic as syn
    dims = syn.TINY_DIMS if size == "tiny" else syn.model_dims()
    L = dims["max_pos"] + 1                                                   # 33 / 513
    sd = syn.seeded_state_dict(dims, seed=1, video=False, proj=True)
    order = param_order(dims["text_layers"])
    args = [sd[k].cuda() for k in order]
    text = syn.synthetic_text(2, L, seed=0, vocab=dims["vocab"])
    ids, mask = text["input_ids"].cuda(), text["attention_mask"].cuda()
    for tokens_mode in (False, True):
        before = _lib.launch_count()
        with pytest.raises(_lib.EgovlpError, match="position embeddings"):
            engine.TextTowerFn.apply(ids, mask, dims["text_heads"], 1e-12, tokens_mode, engine.Bf16Cache(), None, *args)
        assert _lib.launch_count() == before


# ------------------------------------------------------------------------------------------------ the tower
@pytest.mark.gpu
def test_text_tower_long_vs_reference_golden():
    """The tiny DistilBERT geometry with 512 positions through TextTowerFn: hidden states (projection '') against
    the HF recording at L = 512 and 200, then compute_text / compute_text_tokens with txt_proj and the gradients
    against the oracle, at the tolerances of test_model_gpu.py::test_text_tower_tiny_vs_oracle."""
    from egovlp_b200 import engine, synthetic as syn
    from oracle import reference_port as rp
    g = load_golden("distilbert_long.npz")
    dims = long_dims()
    sd = syn.seeded_state_dict(dims, seed=int(g["seed"]), video=False, proj=True)
    sd = {k: v for k, v in sd.items() if not k.startswith("vid_proj")}
    cache = engine.Bf16Cache()
    p_gpu = {k: v.clone().cuda().requires_grad_(True) for k, v in sd.items()}
    bare = [p_gpu[k] for k in param_order(2, proj=False)] + [None, None]
    for L, tag in ((512, "l512"), (200, "l200")):
        ids, mask = g["input_ids"][:, :L].cuda(), g["attention_mask"][:, :L].cuda()
        with torch.no_grad():
            tok = engine.TextTowerFn.apply(ids, mask, 2, 1e-12, True, cache, None, *bare)
            cls = engine.TextTowerFn.apply(ids, mask, 2, 1e-12, False, cache, None, *bare)
        bi, li = g[f"{tag}_rows_b"].long(), g[f"{tag}_rows_l"].long()
        assert rel(tok[bi.cuda(), li.cuda()], g[f"{tag}_rows"][-1]) < 1e-2, tag
        assert rel(cls, g[f"{tag}_cls"][-1]) < 1e-2, tag
    L = 512
    text = {"input_ids": g["input_ids"][:, :L], "attention_mask": g["attention_mask"][:, :L]}
    p_cpu = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref_tok = rp.compute_text_tokens(text, p_cpu, heads=2)
    ref_cls = rp.compute_text(text, p_cpu, heads=2)
    probe = torch.randn(ref_cls.shape, generator=torch.Generator().manual_seed(3))
    (ref_cls * probe).sum().backward()
    order = param_order(2)
    args = [p_gpu[k] for k in order]
    ids, mask = text["input_ids"].cuda(), text["attention_mask"].cuda()
    tok = engine.TextTowerFn.apply(ids, mask, 2, 1e-12, True, cache, None, *args)
    assert rel(tok, ref_tok) < 1e-2
    cls = engine.TextTowerFn.apply(ids, mask, 2, 1e-12, False, cache, None, *args)
    assert rel(cls, ref_cls) < 1e-2
    (cls * probe.cuda()).sum().backward()
    for k in order:
        ref = p_cpu[k].grad
        if ref is None or k.endswith("k_lin.bias"):      # analytically zero (softmax shift invariance)
            continue
        assert cos(p_gpu[k].grad, ref) > 0.995, (k, cos(p_gpu[k].grad, ref))


@pytest.mark.gpu
@pytest.mark.parametrize("L", [512, 129])
def test_full_size_text_tower_long_vs_fp32_oracle(L):
    """DistilBERT-base geometry (768, 12 heads, 6 layers, seeded weights), B = 8 ragged with one full-length row:
    compute_text / compute_text_tokens within the full-size bound of DESIGN section 6 (rel-L2 < 9e-3) of the fp32
    oracle run on the GPU with TF32 off; gradients of every text-tower parameter and txt_proj by cosine."""
    from egovlp_b200 import engine, synthetic as syn
    from oracle import reference_port as rp
    dims = syn.model_dims()
    sd = syn.seeded_state_dict(dims, seed=21, video=False, proj=True)
    sd = {k: v.cuda() for k, v in sd.items() if not k.startswith("vid_proj")}
    text = {k: v.cuda() for k, v in syn.synthetic_text(8, L, seed=L, ragged=True).items()}
    order = param_order(dims["text_layers"])
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        p_ref = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
        ref_tok = rp.compute_text_tokens(text, p_ref, heads=12).detach()
        ref_cls = rp.compute_text(text, p_ref, heads=12)
        probe = torch.randn(ref_cls.shape, generator=torch.Generator().manual_seed(4)).cuda()
        (ref_cls * probe).sum().backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    p_gpu = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    cache = engine.Bf16Cache()
    args = [p_gpu[k] for k in order]
    with torch.no_grad():
        tok = engine.TextTowerFn.apply(text["input_ids"], text["attention_mask"], 12, 1e-12, True, cache, None, *args)
    e_tok = rel(tok, ref_tok)
    cls = engine.TextTowerFn.apply(text["input_ids"], text["attention_mask"], 12, 1e-12, False, cache, None, *args)
    e_cls = rel(cls, ref_cls)
    (cls * probe).sum().backward()
    got, want, worst = [], [], (1.0, None)
    for k in order:
        if k.endswith("k_lin.bias"):
            continue
        a, b = p_gpu[k].grad, p_ref[k].grad
        got.append(a.flatten()); want.append(b.flatten())
        if a.dim() == 2:
            worst = min(worst, (cos(a, b), k))
    whole = cos(torch.cat(got), torch.cat(want))
    print(f"[parity] L={L}: tokens rel {e_tok:.3g}, cls rel {e_cls:.3g}, grad cos {whole:.5f}, worst matrix {worst}")
    assert e_tok < 9e-3 and e_cls < 9e-3, (e_tok, e_cls)
    assert whole > 0.997 and worst[0] > 0.993, (whole, worst)


@pytest.mark.gpu
def test_text_tower_dropout_at_300_vs_oracle_fed_with_the_masks():
    """Train-mode dropout above 128 tokens: reproducible under torch.manual_seed, different from p = 0, and equal to
    the oracle fed with the masks -- attention from the host Philox of text_attn_long, embedding / FFN from the
    egovlp_dropout stream (as test_dropout_gpu.py)."""
    from egovlp_b200 import engine, ops, synthetic as syn
    from oracle import reference_port as rp
    dims = long_dims()
    sd = {k: v for k, v in syn.seeded_state_dict(dims, seed=4, video=False, proj=True).items() if not k.startswith("vid_proj")}
    B, L, D, H, p_hid, p_att = 4, 300, dims["text_dim"], dims["text_heads"], 0.1, 0.2
    text = syn.synthetic_text(B, L, seed=2, ragged=True, vocab=120)
    order = param_order(dims["text_layers"])
    p_gpu = {k: v.clone().cuda().requires_grad_(True) for k, v in sd.items()}
    ids, mask = text["input_ids"].cuda(), text["attention_mask"].cuda()
    cache = engine.Bf16Cache()

    def run(seed_for_torch):
        torch.manual_seed(seed_for_torch)
        return engine.TextTowerFn.apply(ids, mask, H, 1e-12, False, cache, (p_hid, p_att), *[p_gpu[k] for k in order])

    det = engine.TextTowerFn.apply(ids, mask, H, 1e-12, False, cache, None, *[p_gpu[k] for k in order])
    a, b, c = run(7), run(7), run(8)
    assert torch.equal(a, b) and not torch.equal(a, c) and not torch.equal(a, det)
    torch.manual_seed(7)
    seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    ones = torch.ones(B * L * D, device="cuda")
    drop = {"emb": ops.dropout(ones, p_hid, seed, 0, y32=torch.empty_like(ones))[0].view(B, L, D).cpu()}
    for i in range(dims["text_layers"]):
        drop[("att", i)] = multiplier(seed, 1 + 2 * i, p_att, B, H, L).float()
        drop[("ffn", i)] = ops.dropout(ones, p_hid, seed, 2 + 2 * i, y32=torch.empty_like(ones))[0].view(B, L, D).cpu()
    p_cpu = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    want = rp.compute_text(text, p_cpu, heads=H, dropout=drop)
    assert rel(a, want) < 1e-2, rel(a, want)
    assert rel(det, want) > 5e-2
    probe = torch.randn(want.shape, generator=torch.Generator().manual_seed(3))
    (want * probe).sum().backward()
    (a * probe.cuda()).sum().backward()
    for k in order:
        ref = p_cpu[k].grad
        if ref is None or k.endswith("k_lin.bias"):
            continue
        assert cos(p_gpu[k].grad, ref) > 0.995, (k, cos(p_gpu[k].grad, ref))


@pytest.mark.gpu
def test_frozen_in_time_training_step_with_a_300_token_caption():
    """One FrozenInTime step (seeded full-size weights, 4 clips x 4 frames, EgoNCE, fused AdamW) on a batch whose
    longest caption has 300 tokens: completes, and its loss is the fp32 oracle's within 1e-3 relative."""
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.loss import EgoNCE
    from egovlp_b200.model.model import FrozenInTime
    from egovlp_b200.optim import AdamW
    from oracle import reference_port as rp
    sd = syn.seeded_state_dict(syn.model_dims(num_frames=4), seed=5)
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 4,
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    net.load_state_dict(sd, strict=True)
    net.text_model.config.dropout = net.text_model.config.attention_dropout = 0.0
    net.cuda()
    text = {k: v.cuda() for k, v in syn.synthetic_text(4, 300, seed=3, ragged=True).items()}
    assert int(text["attention_mask"].sum(1).max()) == 300
    data = {"video": syn.synthetic_video(4, 4, seed=1).cuda(), "text": text}
    verb, noun = [t.cuda() for t in syn.synthetic_tags(4, seed=2)]
    opt = AdamW(net.parameters(), lr=3e-5)
    opt.zero_grad(set_to_none=True)
    t, v = net(data)
    loss = EgoNCE().fused(t, v, verb, noun)
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    assert all(bool(p.isfinite().all()) for p in net.parameters())
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            p = {k: v.cuda() for k, v in sd.items()}
            tr, vr = rp.frozen_in_time_forward(data, p)
            want = rp.egonce_loss(rp.sim_matrix(tr, vr), rp.sim_matrix(verb, verb), rp.sim_matrix(noun, noun))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    assert abs(loss.item() - want.item()) <= 1e-3 * abs(want.item()), (loss.item(), want.item())
