"""e4m3 (fp8) inference of the video tower (`SpaceTimeTransformer.set_inference_precision("fp8")`):
  1. the e4m3 GEMM (qkv form: bias + q column scale; fc1 form: bias + GELU) against fp64 from the same dequantised
     operands, bitwise reproducible, unsupported shapes refused;
  2. the LayerNorm forward's e4m3 output (warp kernel below 4096 rows, pipelined kernel above): row scales, rounding,
     and the other outputs bit-identical to the plain call;
  3. the weight quantiser bit for bit against torch's float8_e4m3fn conversion;
  4. the tower against the fp32 oracle at 4 and 16 frames, and the cfg5 EgoMCQ argmax on the fp8 path;
  5. mode semantics: batch invariance, training untouched by the flag, bf16 restored bit for bit, `p.data` updates seen.
All accuracy figures come from the seeded synthetic weights (real ViT activations have outlier channels that per-row
scales handle less well)."""
import json
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu
warnings.simplefilter("ignore")
E4M3, BF16, F32 = torch.float8_e4m3fn, torch.bfloat16, torch.float32
Q_SCALE = 0.125
VIDEO = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 16, "pretrained": True,
         "time_init": "zeros"}
TEXT = {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"}


@pytest.fixture(scope="module")
def ops():
    from egovlp_b200 import ops
    return ops


def randn(shape, seed, device="cuda"):
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randn(shape, generator=g, device=device)


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def cos(a, b):
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-300)).item()


def bf16_ulp(x):
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))) - 7)


def quantized_operand(ops, rows, K, seed):
    """e4m3 rows with per-row scales spanning four decades (so that the scales matter)."""
    w = randn((rows, K), seed) * torch.exp2(randn((rows, 1), seed + 1) * 3)
    return ops.quantize_rows_e4m3(w)


# ------------------------------------------------------------------------------------------------ 1. e4m3 GEMM
@pytest.mark.parametrize("K", [768, 3072])
@pytest.mark.parametrize("N", [384, 2304, 3072])
@pytest.mark.parametrize("act", [0, 1])
def test_gemm_e4m3_against_fp64_of_the_dequantised_operands(ops, N, K, act):
    Ms = [1, 63, 64, 65, 1000, 502_400] if K == 768 else [1, 65, 1000, 8192]
    b8, bs = quantized_operand(ops, N, K, 11)
    bias = randn((N,), 12)
    bd = b8.double() * bs.double()[:, None]
    for M in Ms:
        a8, as_ = quantized_operand(ops, M, K, 13 + M)
        out = torch.empty(M, N, dtype=BF16, device="cuda")
        kw = dict(bias=bias, act=act) if act else dict(bias=bias, col_scale=Q_SCALE, col_scale_ncols=N // 3)
        ops.gemm_e4m3(a8, as_, b8, bs, out, **kw)
        again = torch.empty_like(out)
        ops.gemm_e4m3(a8, as_, b8, bs, again, **kw)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), again.view(torch.int16)), f"not reproducible at M={M}"
        rows = torch.arange(M, device="cuda")
        if M > 4096:                                       # fp64 check on a sample: both ends and random rows
            g = torch.Generator(device="cuda").manual_seed(M)
            rows = torch.cat([rows[:256], rows[-256:], torch.randint(0, M, (1024,), generator=g, device="cuda")])
        ad = a8[rows].double() * as_[rows].double()[:, None]
        pre = ad @ bd.T + bias.double()
        mag = ad.abs() @ bd.abs().T
        if act:
            ref = torch.nn.functional.gelu(pre)
            tol = 1.2e-3 * mag                              # |GELU'| <= 1.13
        else:
            cs = torch.ones(N, dtype=torch.float64, device="cuda")
            cs[:N // 3] = Q_SCALE
            ref, tol = pre * cs, 1e-3 * mag * cs
        err = (out[rows].double() - ref).abs()
        bound = tol + bf16_ulp(ref)
        worst = (err / bound).max().item()
        assert worst <= 1.0, f"M={M} N={N} K={K} act={act}: error {worst:.3f} x the bound"


def test_gemm_e4m3_refuses_unsupported_shapes(ops):
    from egovlp_b200._lib import EgovlpError
    a8, as_ = quantized_operand(ops, 64, 768, 1)
    b8, bs = quantized_operand(ops, 320, 768, 2)           # N % 128 != 0
    with pytest.raises(EgovlpError, match="bad shape"):
        ops.gemm_e4m3(a8, as_, b8, bs, torch.empty(64, 320, dtype=BF16, device="cuda"))
    a8, as_ = quantized_operand(ops, 64, 24, 3)            # K % 16 != 0
    b8, bs = quantized_operand(ops, 128, 24, 4)
    with pytest.raises(EgovlpError, match="bad shape"):
        ops.gemm_e4m3(a8, as_, b8, bs, torch.empty(64, 128, dtype=BF16, device="cuda"))
    a8, as_ = quantized_operand(ops, 64, 768, 5)
    b8, bs = quantized_operand(ops, 128, 768, 6)
    with pytest.raises(EgovlpError, match="epilogues"):
        ops.gemm_e4m3(a8, as_, b8, bs, torch.empty(64, 128, dtype=BF16, device="cuda"), act=3)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ 2. LayerNorm
@pytest.mark.parametrize("rows,D", [(1000, 768), (8192, 768), (5000, 384), (77, 1000)])
def test_layernorm_e4m3_output(ops, rows, D):
    x = randn((rows, D), 21) * 3 + 1
    x[7] = 0.5                                             # constant row: y = beta
    gamma, beta = randn((D,), 22), randn((D,), 23) * 0.1
    eps = 1e-6
    y16, y32 = torch.empty(rows, D, dtype=BF16, device="cuda"), torch.empty(rows, D, device="cuda")
    mean, rstd = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
    ops.layernorm_fwd(x, gamma, beta, eps, y16=y16, y32=y32, mean=mean, rstd=rstd)
    z16, z32 = torch.empty_like(y16), torch.empty_like(y32)
    zm, zr = torch.empty_like(mean), torch.empty_like(rstd)
    y8, scale = torch.empty(rows, D, dtype=E4M3, device="cuda"), torch.empty(rows, device="cuda")
    ops.layernorm_fwd(x, gamma, beta, eps, y16=z16, y32=z32, mean=zm, rstd=zr, y8=y8, row_scale=scale)
    torch.cuda.synchronize()
    for a, b in ((y16, z16), (y32, z32), (mean, zm), (rstd, zr)):
        assert torch.equal(a, b)
    amax = y32.abs().amax(dim=1)
    # true division (torch divides by a scalar through its reciprocal)
    assert torch.equal(scale, torch.where(amax > 0, amax / torch.full_like(amax, 448.0), torch.ones_like(amax)))
    deq = y8.double() * scale.double()[:, None]
    xd = x.double()
    ref = (xd - xd.mean(1, keepdim=True)) / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + eps) * gamma.double() \
        + beta.double()
    s = scale.double()[:, None]
    # e4m3 rounding: half an ulp = 2^-4 relative for normals (|v| >= 2^-6 before scaling), half the subnormal step 2^-9
    # below; plus the fp32 LayerNorm's own distance from fp64
    bound = torch.maximum(ref.abs() * 2.0 ** -4, 2.0 ** -10 * s) + 1e-5 * (ref.abs() + s)
    assert ((deq - ref).abs() <= bound).all(), ((deq - ref).abs() / bound).max().item()


def test_layernorm_e4m3_refuses_small_d(ops):
    from egovlp_b200._lib import EgovlpError
    x = randn((16, 256), 1)
    with pytest.raises(EgovlpError, match="bad D"):
        ops.layernorm_fwd(x, torch.ones(256, device="cuda"), torch.zeros(256, device="cuda"), 1e-6,
                          y8=torch.empty(16, 256, dtype=E4M3, device="cuda"),
                          row_scale=torch.empty(16, device="cuda"))


# ------------------------------------------------------------------------------------------------ 3. weights
def test_weight_quantiser_matches_torch_float8(ops):
    w = randn((2304, 768), 31) * 0.02
    w[3] = 0.0                                             # zero row: scale 1, all-zero bytes
    w[5] = 1e-4 * randn((768,), 32)
    w[5, 100] = 7.5                                        # one large value: everything else near or below subnormal
    w[9] *= 1e-3
    q, s = ops.quantize_rows_e4m3(w)
    torch.cuda.synchronize()
    wc = w.cpu()
    amax = wc.abs().amax(dim=1)
    one = torch.ones_like(amax)
    inv = torch.where(amax > 0, torch.full_like(amax, 448.0) / amax, one)
    want_q = (wc * inv[:, None]).to(E4M3)
    want_s = torch.where(amax > 0, amax / torch.full_like(amax, 448.0), one)
    assert torch.equal(s.cpu(), want_s)
    assert torch.equal(q.cpu().view(torch.uint8), want_q.view(torch.uint8))
    assert s[3].item() == 1.0 and q[3].view(torch.uint8).sum().item() == 0


# ------------------------------------------------------------------------------------------------ 4. tower accuracy
@pytest.fixture(scope="module")
def setup():
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.model import FrozenInTime
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = syn.seeded_state_dict(syn.model_dims(num_frames=16), seed=0)
    net = FrozenInTime(dict(VIDEO), dict(TEXT))
    net.load_state_dict(sd, strict=True)
    net.text_model.config.dropout = net.text_model.config.attention_dropout = 0.0
    net.cuda()
    net.set_device(torch.device("cuda"))
    params = {k: v.cuda() for k, v in sd.items()}
    yield net, params
    net.video_model.set_inference_precision("bf16")


@pytest.mark.parametrize("B,T", [(16, 4), (8, 16)])
def test_tower_against_fp32_oracle(setup, B, T):
    from egovlp_b200 import synthetic as syn
    from oracle import reference_port as rp
    net, params = setup
    clips = syn.synthetic_video(B, T, seed=40 + T).cuda()
    with torch.no_grad():
        net.video_model.set_inference_precision("fp8")
        v8 = net.compute_video(clips)
        net.video_model.set_inference_precision("bf16")
        v16 = net.compute_video(clips)
        vr = torch.cat([rp.compute_video(clips[i:i + 8], params) for i in range(0, B, 8)])
    e8, e16 = rel(v8, vr), rel(v16, vr)
    print(f"\n[fp8 tower B={B} T={T}] rel-L2 fp8 {e8:.3e}  bf16 {e16:.3e}")
    # Measured on an H100: 6.5-6.7e-2 at both shapes, above the 5e-2 first estimated from e4m3's 3-bit mantissa.  The
    # test below shows the excess is the operand rounding, not the accumulator.  DESIGN.md section 6 records it.
    assert e16 < 9e-3 and e8 < 8e-2, (e8, e16)


def test_tower_error_is_operand_rounding_not_fp8_accumulation(setup, monkeypatch):
    """The same e4m3 operands and scales, but multiplied in fp32 (exact e4m3 products, fp32 sums, TF32 off) instead of
    on the e4m3 tensor cores: if the tensor cores' reduced-precision fp8 accumulation caused the tower's error, this
    tower would be much closer to the fp32 oracle than the fp8 one."""
    from egovlp_b200 import ops as ops_mod, synthetic as syn
    from oracle import reference_port as rp
    net, params = setup
    B, T = 16, 4
    clips = syn.synthetic_video(B, T, seed=40 + T).cuda()

    def gemm_e4m3_fp32(a8, a_scale, b8, b_scale, out, *, bias=None, act=0, alpha=1.0, col_scale=1.0,
                       col_scale_ncols=0):
        v = (a8.float() @ b8.float().T) * a_scale[:, None] * b_scale[None, :] * alpha
        if bias is not None:
            v = v + bias
        if act:
            v = torch.nn.functional.gelu(v)
        else:
            v[:, :col_scale_ncols] *= col_scale
        out.copy_(v)
        return out

    net.video_model.set_inference_precision("fp8")
    try:
        with torch.no_grad():
            v8 = net.compute_video(clips).clone()
            monkeypatch.setattr(ops_mod, "gemm_e4m3", gemm_e4m3_fp32)
            v_emul = net.compute_video(clips).clone()
            monkeypatch.undo()
            vr = torch.cat([rp.compute_video(clips[i:i + 8], params) for i in range(0, B, 8)])
    finally:
        net.video_model.set_inference_precision("bf16")
    e8, e_emul, d = rel(v8, vr), rel(v_emul, vr), rel(v8, v_emul)
    print(f"\n[fp8 accumulation] rel-L2 vs fp32: tensor cores {e8:.3e}, fp32-accumulated {e_emul:.3e}; "
          f"between the two {d:.3e}")
    # Measured: 6.66e-2 on the tensor cores, 6.69e-2 fp32-accumulated.  The two towers are 3.4e-2 apart from each
    # other: a last-bit difference in an accumulator can move a LayerNorm output across an e4m3 rounding boundary (a
    # 6 % step), so two summation orders diverge through the blocks while each stays as far from fp32 as the other.
    assert e_emul > 0.8 * e8, (e8, e_emul, d)


def test_cfg5_egomcq_on_the_fp8_path(setup):
    """The cfg5 EgoMCQ check of test_parity_fullsize_gpu.py with the video tower in fp8."""
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.metric import egomcq_predict
    from oracle import reference_port as rp
    net, params = setup
    Q, K, T, L, CH = 1024, 5, 4, 16, 128
    text = {k: v.cuda() for k, v in syn.synthetic_text(Q, L, seed=9, ragged=True).items()}
    v_gpu, v_ref = [], []
    net.video_model.set_inference_precision("fp8")
    try:
        with torch.no_grad():
            t_gpu = net.compute_text(text)
            t_ref = torch.cat([rp.compute_text({k: x[i:i + 256] for k, x in text.items()}, params)
                               for i in range(0, Q, 256)])
            for c in range(0, Q * K, CH):
                clips = syn.synthetic_video(CH, T, seed=1000 + c).cuda()
                v_gpu.append(net.compute_video(clips))
                v_ref.append(torch.cat([rp.compute_video(clips[i:i + 32], params) for i in range(0, CH, 32)]))
            v_gpu, v_ref = torch.cat(v_gpu).view(Q, K, -1), torch.cat(v_ref).view(Q, K, -1)
            s_gpu, pred = egomcq_predict(t_gpu, v_gpu)
            s_ref, pred_ref = rp.egomcq_predict(t_ref, v_ref)
    finally:
        net.video_model.set_inference_precision("bf16")
    err = (s_gpu - s_ref).abs().max().item()
    top2 = s_ref.topk(2, dim=1).values
    margin = top2[:, 0] - top2[:, 1]
    decided = margin > 2 * err
    agree = pred == pred_ref
    print("\n[cfg5 EgoMCQ fp8]", json.dumps({"max_abs_score_err": err, "n_decided": int(decided.sum()),
                                             "agree_decided": int((agree & decided).sum()),
                                             "agree_all": int(agree.sum()), "rel_video_emb": rel(v_gpu, v_ref)}))
    assert err < 6e-2
    assert bool(agree[decided].all())


# ------------------------------------------------------------------------------------------------ 5. semantics
def test_dense_features_are_batch_invariant_in_fp8(setup):
    from egovlp_b200 import features, synthetic as syn
    net, _ = setup
    frames = syn.synthetic_video(1, 40, seed=5)[0]
    net.video_model.set_inference_precision("fp8")
    try:
        small = features.dense_video_features(net, frames, 4, batch=4)
        big = features.dense_video_features(net, frames, 4, batch=64)
    finally:
        net.video_model.set_inference_precision("bf16")
    assert torch.equal(small, big)


def test_training_step_ignores_the_flag_and_bf16_is_restored(setup):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.loss import EgoNCE
    net, _ = setup
    B, T = 4, 4
    data = {"video": syn.synthetic_video(B, T, seed=7).cuda(),
            "text": {k: v.cuda() for k, v in syn.synthetic_text(B, 16, seed=7).items()}}
    verb, noun = [t.cuda() for t in syn.synthetic_tags(B, seed=7)]

    def step():
        from egovlp_b200 import ops
        net.zero_grad(set_to_none=True)
        ops.profile(True)
        t, v = net(data)
        loss = EgoNCE().fused(t, v, verb, noun)
        loss.backward()
        kinds = ops.profile(False)
        return (t.detach().clone(), v.detach().clone(), loss.detach().clone(),
                {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None}, kinds)

    def inference():
        from egovlp_b200 import ops
        ops.profile(True)
        with torch.no_grad():
            e = net.compute_video(data["video"]).clone()
        return e, ops.profile(False)

    e16, _ = inference()
    t16, v16, l16, g16, k16 = step()
    net.video_model.set_inference_precision("fp8")
    try:
        t8, v8, l8, g8, k8 = step()
        e8, k_inf = inference()
    finally:
        net.video_model.set_inference_precision("bf16")
    net.zero_grad(set_to_none=True)
    # The flagged training step runs the bf16 path: the same launches of every profiled kind with the same algorithmic
    # FLOPs / bytes (no e4m3 GEMM, no e4m3 LayerNorm output), and the same forward bit for bit.  The gradients are not
    # bitwise reproducible run to run (split-K weight-gradient and CLS-row atomics at B = 4 put two unflagged steps
    # 1 - cos = 2e-6 to 3e-5 apart, measured), so the gradients get a fixed, loose bound; the two checks above carry the
    # claim.
    work = lambda rec: {k: (w, n) for k, (w, _, n) in rec.items()}               # noqa: E731
    assert work(k8) == work(k16), (work(k8), work(k16))
    assert torch.equal(t16, t8) and torch.equal(v16, v8) and torch.equal(l16, l8)
    assert g16.keys() == g8.keys()
    flat = lambda g: torch.cat([g[k].double().flatten() for k in sorted(g)])        # noqa: E731
    c = cos(flat(g8), flat(g16))
    print(f"\n[training with the flag] gradient cosine to the unflagged step 1 - {1 - c:.2e}")
    assert c > 1 - 1e-3, c
    assert k_inf["gemm_e4m3"][2] == 36                     # 12 blocks x (two qkv + fc1) in inference
    assert not torch.equal(e8, e16)
    with torch.no_grad():
        assert torch.equal(net.compute_video(data["video"]), e16)


def test_weight_updates_through_data_are_seen_by_fp8(setup):
    from egovlp_b200 import synthetic as syn
    net, _ = setup
    video = syn.synthetic_video(2, 4, seed=3).cuda()
    tower = net.video_model
    tower.set_inference_precision("fp8")
    w = tower.blocks[3].mlp.fc1.weight
    saved = w.detach().clone()

    class DataSGD(torch.optim.Optimizer):
        def __init__(self, params):
            super().__init__(params, {})

        def step(self):
            for g in self.param_groups:
                for p in g["params"]:
                    p.data.mul_(1.5)

    try:
        with torch.no_grad():
            before = net.compute_video(video).clone()
            ver = w._version
            DataSGD([w]).step()                            # no version bump: the optimizer-step hook catches it
            assert w._version == ver
            after = net.compute_video(video).clone()
        assert rel(after, before) > 1e-3
        w.data.copy_(saved)                                # caught by the refresh of a training forward
        with torch.enable_grad():
            net.compute_video(video)
        with torch.no_grad():
            assert torch.equal(net.compute_video(video), before)
    finally:
        w.data.copy_(saved)
        tower.set_inference_precision("bf16")
        with torch.enable_grad():
            net.compute_video(video)
