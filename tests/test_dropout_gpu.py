"""Train-mode dropout of the DistilBERT text tower (HF modeling_distilbert.py; the reference keeps
`text_model.train()`, model/model.py:36).  RNG parity with torch is impossible, so the test separates the two halves:
the MASKS are checked bit for bit against the documented Philox streams regenerated on the host (tests/philox_ref.py)
and as an RNG (rate, scaling, determinism, site independence), and the ARITHMETIC around them is checked against the
fp32 oracle fed with the host's masks.  The attention dropout of the L <= 128 kernel is checked element by element in
test_text_attention_gpu.py."""
import pytest
import torch
from kernel_checks import BF16, F32, assert_bits_equal, nan_filled
from philox_ref import drop_path_keep, flat_keep, flat_multiplier, multiplier, short_attn_keep

pytestmark = pytest.mark.gpu


def test_dropout_kernel_is_a_proper_mask():
    from egovlp_b200 import ops
    n, p, seed = 1 << 20, 0.1, 1234567891011
    ones = torch.ones(n, device="cuda")
    y, y16 = ops.dropout(ones, p, seed, 3, y32=torch.empty_like(ones), y16=torch.empty(n, device="cuda", dtype=torch.bfloat16))
    kept = y != 0
    assert abs(kept.float().mean().item() - (1 - p)) < 3e-3                     # 1M draws: sigma = 3e-4
    torch.testing.assert_close(y[kept], torch.full_like(y[kept], 1 / (1 - p)))
    assert torch.equal(y16, y.bfloat16())
    y2, _ = ops.dropout(ones, p, seed, 3, y32=torch.empty_like(ones))
    assert torch.equal(y, y2)                                                    # same (seed, site) -> same mask
    other_site, _ = ops.dropout(ones, p, seed, 4, y32=torch.empty_like(ones))
    other_seed, _ = ops.dropout(ones, p, seed + 1, 3, y32=torch.empty_like(ones))
    for o in (other_site, other_seed):                                           # independent streams
        agree = ((o != 0) == kept).float().mean().item()
        assert abs(agree - (0.81 + 0.01)) < 5e-3
    # no visible structure along the element index: every 4096-block keeps ~90 %
    blocks = kept.view(-1, 4096).float().mean(1)
    assert (blocks - 0.9).abs().max().item() < 0.03
    x, add = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    z, _ = ops.dropout(x, p, seed, 3, add=add, y32=torch.empty_like(x))
    torch.testing.assert_close(z, x * y + add)
    same, _ = ops.dropout(x, 0.0, seed, 3, y32=torch.empty_like(x))
    assert torch.equal(same, x)


# bit 63 set in two of the seeds; site 2^32 - 1 is the one whose key wraps to the seed itself
SEEDS = (0x8000_0000_0000_0001, 0xFEDC_BA98_7654_3210, 1234567891011)
SITES = (0, 72, 0xFFFFFFFF)


def _kept_value(ops, p):
    """The fp32 value a kept element of a vector of ones becomes: the kernel's own 1 / (1 - p)."""
    ones = torch.ones(1024, device="cuda")
    y = ops.dropout(ones, p, 0, 0, y32=torch.empty_like(ones))[0]
    keep = flat_keep(1024, p, 0, 0).cuda()
    assert bool(keep.any()), "no kept element to read 1 / (1 - p) from"
    return y[keep][0].item()


@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_dropout_keep_bits_and_arithmetic_are_the_documented_ones(p):
    """egovlp_dropout against tests/philox_ref.py's flat stream, every element: keep bits for n = 4, 1020 and 2^20 + 4,
    seeds with bit 63 set, sites 0, 72 and 2^32 - 1; y32 = fl(x inv) and, with add, fl(fl(x inv) + add) bit for bit
    (an FMUL and an FADD: a build that contracted them into one FFMA would fail here); y16 = bf16(y32) (normal-range
    inputs, so FTZ does not enter)."""
    from egovlp_b200 import ops
    inv = _kept_value(ops, p)
    for n in (4, 1020, (1 << 20) + 4):
        g = torch.Generator(device="cuda").manual_seed(n)
        x, add = torch.randn(n, device="cuda", generator=g), torch.randn(n, device="cuda", generator=g)
        for seed in SEEDS:
            for site in SITES:
                keep = flat_keep(n, p, seed, site).cuda()
                ones = torch.ones(n, device="cuda")
                m = ops.dropout(ones, p, seed, site, y32=torch.empty_like(ones))[0]
                assert torch.equal(m != 0, keep), (n, hex(seed), site, int(((m != 0) != keep).sum()))
                assert bool((m[keep] == inv).all())
                y32, y16 = ops.dropout(x, p, seed, site, y32=nan_filled((n,), F32), y16=nan_filled((n,), BF16))
                prod = torch.where(keep, x * torch.tensor(inv, device="cuda"), torch.zeros_like(x))   # fl(x inv)
                assert_bits_equal(f"dropout y32 n={n} site={site}", y32, prod)
                assert_bits_equal(f"dropout y16 n={n} site={site}", y16, prod.to(BF16))
                z32, z16 = ops.dropout(x, p, seed, site, add=add, y32=nan_filled((n,), F32), y16=nan_filled((n,), BF16))
                want = prod + add
                if not torch.equal(z32, want):
                    fused = torch.where(keep, x.double() * inv + add.double(), add.double()).float()
                    hint = (" (it equals the fused fma(x, inv, add): the FMUL and FADD were contracted into an FFMA)"
                            if torch.equal(z32, fused) else "")
                    raise AssertionError(f"dropout with add n={n}: y32 is not fl(fl(x inv) + add){hint}")
                assert_bits_equal(f"dropout + add y16 n={n} site={site}", z16, want.to(BF16))


@pytest.mark.parametrize("width", [768, 3072])
@pytest.mark.parametrize("rows", [1, 197, 3137])
def test_dropout_mask_and_drop_path_factors_are_the_host_streams(width, rows):
    """ops.dropout_mask (the reference of the GEMM dropout forms in test_video_dropout_gpu.py) at the video widths and
    ragged row counts equals the host flat stream of the [rows, width] tensor; ops.drop_path_factors equals the host
    per-sample words."""
    from egovlp_b200 import ops
    p, seed, site = 0.3, 0x8765_4321_0FED_CBA9, 17
    inv = _kept_value(ops, p)
    m = ops.dropout_mask(rows, width, p, seed, site)
    keep = flat_keep(rows * width, p, seed, site).view(rows, width).cuda()
    assert torch.equal(m != 0, keep) and bool((m[keep] == inv).all())
    n = rows % 61 + 3
    f = ops.drop_path_factors(n, 0.4, seed, site + 1)
    kp = drop_path_keep(n, 0.4, seed, site + 1).cuda()
    assert torch.equal(f != 0, kp) and bool((f[kp] == _kept_value(ops, 0.4)).all())


@pytest.mark.parametrize("x_bf16", [False, True], ids=["fp32", "bf16"])
def test_drop_rows_bf16_is_the_documented_product_with_the_host_masks(x_bf16):
    """drop_rows_bf16 = bf16(fl(x * s)) with s = fl((1 / (1 - p)) f_b) for kept elements (0 otherwise), f_b the
    drop-path factor of the row's sample: keep bits and factors from the host streams, over 8 samples of 125 rows."""
    from egovlp_b200 import ops
    M, W, B = 1000, 384, 8
    d = ops.Drop(0.3, 0x8000_0000_1234_5678, 7, 0.5, 8, M // B)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(M, W, device="cuda", generator=g)
    x = x.to(BF16) if x_bf16 else x
    keep = flat_keep(M * W, d.p, d.seed, d.site).view(M, W).cuda()
    path = drop_path_keep(B, d.path_p, d.seed, d.path_site).cuda()
    assert bool(path.any()) and not bool(path.all())
    f = torch.where(path, torch.tensor(_kept_value(ops, d.path_p), device="cuda"), torch.zeros((), device="cuda"))
    s = torch.tensor(_kept_value(ops, d.p), device="cuda") * f.repeat_interleave(M // B)[:, None]
    want = (x.float() * torch.where(keep, s, torch.zeros_like(s))).to(BF16)
    assert_bits_equal(f"drop_rows_bf16 from {'bf16' if x_bf16 else 'fp32'}", ops.drop_rows_bf16(x, d), want)


def test_text_tower_with_dropout_vs_oracle_fed_with_the_drawn_masks():
    """The tiny DistilBERT in training against the oracle fed with every site's multiplier from the host Philox
    (tests/philox_ref.py): embeddings and FFN outputs the flat stream, attention the short-attention stream.  L = 128
    (positions table widened to 128) runs a lane's 3rd and 4th key with dropout on; there the output checked is the
    CLS hidden state, without txt_proj: its ReLU is a kink at 0 that about 2 of the 640 CLS features (within bf16
    rounding of 0) cross between the tower and the oracle, and each such flip moves the gradient of every parameter
    beneath it by far more than rounding does (measured on an H100: lowest cosine 0.994 through txt_proj, 0.99996
    without)."""
    for L in (9, 128):
        _tower_with_dropout_vs_oracle(L)


def _tower_with_dropout_vs_oracle(L):
    from egovlp_b200 import engine, synthetic as syn
    from oracle import reference_port as rp
    from test_model_gpu import rel, cos
    dims = syn.TINY_DIMS if L <= syn.TINY_DIMS["max_pos"] else dict(syn.TINY_DIMS, max_pos=L)
    sd = {k: v for k, v in syn.seeded_state_dict(dims, seed=4, video=False, proj=True).items() if not k.startswith("vid_proj")}
    text = syn.synthetic_text(5, L, seed=1, ragged=True, vocab=120)
    B, D, H, p_hid, p_att = 5, dims["text_dim"], dims["text_heads"], 0.1, 0.2
    order = ["text_model.embeddings.word_embeddings.weight", "text_model.embeddings.position_embeddings.weight",
             "text_model.embeddings.LayerNorm.weight", "text_model.embeddings.LayerNorm.bias"]
    for i in range(dims["text_layers"]):
        lp = f"text_model.transformer.layer.{i}."
        for lin in ("attention.q_lin", "attention.k_lin", "attention.v_lin", "attention.out_lin"):
            order += [lp + lin + ".weight", lp + lin + ".bias"]
        order += [lp + "sa_layer_norm.weight", lp + "sa_layer_norm.bias", lp + "ffn.lin1.weight", lp + "ffn.lin1.bias",
                  lp + "ffn.lin2.weight", lp + "ffn.lin2.bias", lp + "output_layer_norm.weight", lp + "output_layer_norm.bias"]
    proj = L == 9
    if proj:
        order += ["txt_proj.1.weight", "txt_proj.1.bias"]
    p_gpu = {k: v.clone().cuda().requires_grad_(True) for k, v in sd.items()}
    ids, mask = text["input_ids"].cuda(), text["attention_mask"].cuda()
    cache = engine.Bf16Cache()

    def run(seed_for_torch):
        torch.manual_seed(seed_for_torch)
        return engine.TextTowerFn.apply(ids, mask, H, 1e-12, False, cache, (p_hid, p_att), *args())

    def args():
        return [p_gpu[k] for k in order] + ([] if proj else [None, None])

    det = engine.TextTowerFn.apply(ids, mask, H, 1e-12, False, cache, None, *args())
    a, b, c = run(7), run(7), run(8)
    assert torch.equal(a, b) and not torch.equal(a, c) and not torch.equal(a, det)     # reproducible, seeded, active
    # the seed the forward drew, and from it the multipliers of every site
    torch.manual_seed(7)
    seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    drop = {"emb": flat_multiplier((B, L, D), p_hid, seed, 0).float()}
    for i in range(dims["text_layers"]):
        drop[("att", i)] = multiplier(short_attn_keep(p_att, seed, 1 + 2 * i, B, H, L), p_att).float()
        drop[("ffn", i)] = flat_multiplier((B, L, D), p_hid, seed, 2 + 2 * i).float()
    p_cpu = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    want = (rp.compute_text(text, p_cpu, heads=H, dropout=drop) if proj else
            rp.distilbert_forward(text["input_ids"], text["attention_mask"], p_cpu, H, dropout=drop)[:, 0])
    assert rel(a, want) < 1e-2, (L, rel(a, want))
    assert rel(det, want) > 5e-2, L                                                    # and it is not the p = 0 output
    probe = torch.randn(want.shape, generator=torch.Generator().manual_seed(3))
    (want * probe).sum().backward()
    (a * probe.cuda()).sum().backward()
    for k in order:
        ref = p_cpu[k].grad
        if ref is None or k.endswith("k_lin.bias"):
            continue
        assert cos(p_gpu[k].grad, ref) > 0.995, (L, k, cos(p_gpu[k].grad, ref))
