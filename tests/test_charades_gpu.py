"""Charades-Ego fine-tuning / evaluation and the t2v / v2t retrieval ranks on the CUDA path:
  * `egovlp_gt_ranks` against oracle/eval_port.py bit for bit (t2v up to 5000 x 5000, v2t 1000 videos x 20 captions,
    quantised scores, masks, fp32 and fp64) and its error paths; the metrics built on it; the golden rank vectors;
  * `charades_metrics` on the ranking kernel against the reference golden (tests/golden/charades.npz) and against the
    oracle's tie rule where equal scores straddle a positive and a negative; NaN / +-inf scores ranked as numpy sorts
    them (the ranking kernel in both tie modes, with padded sort slots); the 16384-video cap;
  * `sim_matrix` on host tensors: bit-identical to the device call, with gradients;
  * the zero-shot `_valid_epoch` flow (tools/charades_sequence.py) against the golden, and the Charades training step
    at the config's geometry (4 clips x 16 frames) against the fp32 oracle on the GPU, and two steps with a learning
    rate change between them."""
import types

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import eval_port as ep

pytestmark = pytest.mark.gpu
EMB_TOL, STEP_LOSS_TOL = 9e-3, 1e-3      # full-size bf16-operand tolerances (DESIGN.md section 6)
VIDEO = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 16, "pretrained": True,
         "time_init": "zeros"}
TEXT = {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"}
CHARADES_EXACT = ["realistic", "empty_rows", "nan_class", "ties", "n1"]
RANKS = ["q1", "q20", "q20_masked", "q20_quantised", "q20_quantised_f64", "q1_all_equal", "q20_all_equal"]


def _bound(name, worst, bound):
    print(f"[bound] {name}: {worst:.3e} = {worst / bound:.3f} of the bound {bound:g}")
    assert worst <= bound, name


def rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def cos(a, b):
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-300)).item()


def max_rel(got, want):
    """max |got - want| / |want| over the non-NaN entries; NaN positions must agree."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    ok = ~np.isnan(want)
    err = np.abs(got[ok] - want[ok])
    return float(np.max(np.where(err == 0, 0.0, err / np.maximum(np.abs(want[ok]), 1e-300)), initial=0.0))


# ------------------------------------------------------------------------------------------------------ gt ranks
def _sims(rng, shape, dtype, quantised):
    s = rng.standard_normal(shape)
    s = np.round(4 * s) / 8 if quantised else 0.3 * s
    return s.astype(dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("Q,V,quantised", [(5000, 5000, False), (5000, 5000, True), (2000, 100, True),
                                           (7, 7, False), (60, 3, False)])
def test_t2v_ranks_equal_the_oracle(Q, V, quantised, dtype):
    from egovlp_b200.model import metric
    rng = np.random.default_rng(Q + V + quantised)
    sims = _sims(rng, (Q, V), dtype, quantised)
    got, n = metric.t2v_ranks(sims)
    want, wn = ep.t2v_ranks(sims)
    assert n == wn and np.array_equal(got.cpu().numpy(), want)
    mask = (rng.random(Q) > 0.1).astype(np.float32)
    got, n = metric.t2v_ranks(torch.from_numpy(sims).cuda(), mask)
    want, wn = ep.t2v_ranks(sims, mask)
    assert n == wn and np.array_equal(got.cpu().numpy(), want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("V,c,quantised,masked", [(1000, 20, False, False), (1000, 20, True, True), (300, 64, True, False),
                                                  (50, 1, False, True), (40, 25, True, True)])
def test_v2t_ranks_equal_the_oracle(V, c, quantised, masked, dtype):
    from egovlp_b200.model import metric
    rng = np.random.default_rng(V * c + quantised)
    sims = _sims(rng, (V * c + 3, V), dtype, quantised)          # 3 trailing captions: c = N // V as the reference
    mask = None
    if masked:
        mask = (rng.random(sims.shape[0]) > 0.15).astype(np.float32)
        mask[:c] = 0                                             # every caption of video 0 missing: rank +inf
        sims[c + 1, :] = np.nan                                  # NaN only in a masked caption: replaced, no error
        mask[c + 1] = 0
    got, n = metric.v2t_ranks(sims, mask)
    want, wn = ep.v2t_ranks(sims, mask)
    assert n == wn and np.array_equal(got.cpu().numpy(), want)


def test_gt_ranks_error_paths():
    from egovlp_b200 import ops
    from egovlp_b200._lib import EgovlpError, lib
    from egovlp_b200.model import metric
    assert lib().egovlp_gt_ranks_max_candidates() == 64
    s = torch.rand(40, 10, device="cuda")
    s[7, 3] = float("nan")
    with pytest.raises(EgovlpError, match="NaN"):
        metric.t2v_metrics(s)
    with pytest.raises(EgovlpError, match="NaN"):
        metric.v2t_metrics(s)
    with pytest.raises(EgovlpError, match="multiple"):
        metric.t2v_metrics(torch.rand(41, 10, device="cuda"))
    with pytest.raises(EgovlpError, match="candidates"):
        metric.v2t_metrics(torch.rand(2 * 65, 2, device="cuda"))
    s = torch.rand(20, 10, device="cuda", dtype=torch.float64)
    s[4, 2] = float("inf")                                       # query 4's ground truth (column 2) is infinite
    with pytest.raises(EgovlpError, match="non-finite"):
        ops.gt_ranks(s, 0)
    assert metric.v2t_metrics(torch.rand(2 * 64, 2, device="cuda"))["R50"] >= 0          # 64 candidates are allowed
    s = torch.rand(20, 10, device="cuda")
    s[4, 2] = float("inf")                                       # both conditions in one call: both are reported
    s[9, 7] = float("nan")
    with pytest.raises(EgovlpError, match="NaN.*non-finite"):
        ops.gt_ranks(s, 0)


def test_retrieval_metrics_equal_the_oracle():
    from egovlp_b200.model import metric
    rng = np.random.default_rng(8)
    for sims, mask in ((_sims(rng, (3000, 150), np.float32, True), None),
                       (_sims(rng, (1000, 1000), np.float32, False), (rng.random(1000) > 0.2).astype(np.float32))):
        for fn, ofn in ((metric.t2v_metrics, ep.t2v_metrics), (metric.v2t_metrics, ep.v2t_metrics)):
            got, want = fn(sims, mask), ofn(sims, mask)
            assert got.keys() == want.keys()
            for k in ("R1", "R5", "R10", "R50", "MedR", "MeanR"):
                assert got[k] == want[k], (fn.__name__, k, got[k], want[k])
            g, w = got["geometric_mean_R1-R5-R10"], want["geometric_mean_R1-R5-R10"]
            assert abs(g - w) <= 1e-12 * abs(w), (g, w)


@pytest.mark.parametrize("name", RANKS)
def test_golden_rank_vectors_reproduced(name):
    from egovlp_b200.model import metric
    g = load_golden("charades.npz")
    key = f"ranks/{name}/"
    sims, qm = g[key + "sims"].numpy(), g.get(key + "query_masks")
    qm = None if qm is None else qm.numpy()
    got, n = metric.t2v_ranks(sims, qm)
    assert n == int(g[key + "t2v_n"]) and np.array_equal(got.cpu().numpy(), g[key + "t2v"].numpy())
    got, n = metric.v2t_ranks(sims, qm)
    assert n == int(g[key + "v2t_n"]) and np.array_equal(got.cpu().numpy(), g[key + "v2t"].numpy())


# ------------------------------------------------------------------------------------------------------ charades mAP
@pytest.mark.parametrize("name", CHARADES_EXACT)
def test_charades_metrics_vs_reference_golden(name):
    from egovlp_b200.model import metric
    g = load_golden("charades.npz")
    key = f"charades/{name}/"
    scores, gt = g[key + "scores"].numpy(), g[key + "targets"].numpy().astype(np.float32)
    aps = metric.charades_class_ap(scores, gt).cpu().numpy()
    m_ap = metric.charades_metrics(scores, gt)["mAP"]
    _bound(f"charades {name} class AP rel", max_rel(aps, g[key + "aps"].numpy()), 1e-9)
    _bound(f"charades {name} mAP rel", max_rel([m_ap], [float(g[key + "mAP"])]), 1e-9)
    if name == "nan_class":
        assert np.isnan(aps[17]) and np.isnan(m_ap) and np.isfinite(np.delete(aps, 17)).all()


def test_charades_straddling_ties_follow_the_documented_rule():
    """Equal scores across a positive and a negative: smaller video index first (the oracle's stable argsort)."""
    from egovlp_b200.model import metric
    rng = np.random.default_rng(11)
    n = 500
    gt = (rng.random((n, 157)) < 0.03).astype(np.float32)
    gt[rng.choice(n, 20, replace=False)] = 0
    scores = (np.round(rng.standard_normal((n, 157)) * 3) / 8).astype(np.float32)    # ~20 distinct values
    got = metric.charades_class_ap(torch.from_numpy(scores).cuda(), torch.from_numpy(gt).cuda()).cpu().numpy()
    _, _, want = ep.map(ep.charades_fix(scores, gt), gt)
    _bound("charades straddling ties class AP rel", max_rel(got, want), 1e-9)
    # a real -inf score on a positive of a non-empty row ranks after every finite score, among the empty rows' -inf
    # by video index, and ahead of the kernel's padding (700 videos -> 1024 sort slots)
    n = 700
    gt = (rng.random((n, 157)) < 0.02).astype(np.float32)
    gt[::7] = 0
    gt[3, :] = 1
    scores = rng.standard_normal((n, 157)).astype(np.float32)
    scores[3, :] = -np.inf
    got = metric.charades_class_ap(scores, gt).cpu().numpy()
    _, _, want = ep.map(ep.charades_fix(scores, gt), gt)
    _bound("charades -inf positives class AP rel", max_rel(got, want), 1e-9)
    assert np.all(np.nan_to_num(got) > 0)


@pytest.mark.parametrize("cols", [300, 511, 512, 700])
def test_rank_metrics_order_nan_and_inf_as_numpy(cols):
    """egovlp_rank_metrics with NaN / +-inf similarities and padded sort slots (cols is not a power of two): NaN ranks
    after every real value for the argsort of -sim (mAP.py, charades_metrics) and before every real value for the
    reversed ascending argsort (nDCG.py), as numpy sorts it; the real columns always fill the first `cols` ranks."""
    from egovlp_b200 import ops
    from oracle import reference_port as rp
    rng = np.random.default_rng(cols)
    rows = 40
    sim = rng.standard_normal((rows, cols)).astype(np.float32)
    for r in range(rows):
        k = r % 6
        sim[r, rng.choice(cols, k, replace=False)] = np.nan
        sim[r, rng.choice(cols, r % 3, replace=False)] = -np.inf
        sim[r, rng.choice(cols, r % 2, replace=False)] = np.inf
    sim[0, :] = np.nan                                                      # an all-NaN row
    rel = (rng.random((rows, cols)) < 0.1).astype(np.float64)
    rel[np.isnan(sim) & (rng.random((rows, cols)) < 0.5)] = 1.0             # positives among the NaNs
    k_counts = rp.k_counts_of(rel)
    dcg, ap = ops.rank_metrics(torch.from_numpy(sim).cuda(), torch.from_numpy(rel).cuda(), None, tie_mode=0)
    _bound(f"rank_metrics NaN/inf AP (argsort of -sim) rel, cols={cols}",
           max_rel(ap.cpu().numpy(), rp.average_precision(sim, rel)), 1e-12)
    dcg, _ = ops.rank_metrics(torch.from_numpy(sim).cuda(), torch.from_numpy(rel).cuda(), None, tie_mode=1,
                              want_ap=False)
    _bound(f"rank_metrics NaN/inf DCG (reversed ascending argsort) rel, cols={cols}",
           max_rel(dcg.cpu().numpy(), rp.dcg(sim, rel, k_counts)), 1e-12)


def test_charades_nan_scores_rank_last_as_numpy():
    """A diverged model's NaN scores: ranked after every real score (-inf of empty rows included), as the reference's
    np.argsort(-x) puts them, never displacing a video from the ranking."""
    from egovlp_b200.model import metric
    rng = np.random.default_rng(13)
    n = 700
    gt = (rng.random((n, 157)) < 0.03).astype(np.float32)
    gt[::11] = 0
    scores = (0.2 * rng.standard_normal((n, 157))).astype(np.float32)
    scores[rng.random((n, 157)) < 0.02] = np.nan
    scores[5, :] = np.nan
    gt[5, :3] = 1
    got = metric.charades_class_ap(scores, gt).cpu().numpy()
    _, _, want = ep.map(ep.charades_fix(scores, gt), gt)
    _bound("charades NaN scores class AP rel", max_rel(got, want), 1e-9)
    assert np.isfinite(got).all()


def test_charades_video_cap_raises():
    from egovlp_b200.model import metric
    metric.charades_metrics(np.zeros((16384, 3), np.float32), np.ones((16384, 3), np.float32))
    with pytest.raises(ValueError, match="16384"):
        metric.charades_metrics(np.zeros((16385, 3), np.float32), np.ones((16385, 3), np.float32))


# ------------------------------------------------------------------------------------------------------ sim_matrix
def test_sim_matrix_on_host_tensors():
    from egovlp_b200.model.model import sim_matrix
    g = torch.Generator().manual_seed(2)
    a, b = torch.randn(157, 256, generator=g), torch.randn(37, 256, generator=g)
    a[5] = 0                                                                        # the eps clamp
    probe = torch.randn(157, 37, generator=g)
    ah, bh = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    out_h = sim_matrix(ah, bh)
    (out_h * probe).sum().backward()
    ad, bd = a.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    out_d = sim_matrix(ad, bd)
    (out_d * probe.cuda()).sum().backward()
    assert out_h.device.type == "cpu" and torch.equal(out_h.detach(), out_d.detach().cpu())
    assert ah.grad.device.type == "cpu" and torch.equal(ah.grad, ad.grad.cpu()) and torch.equal(bh.grad, bd.grad.cpu())
    with torch.no_grad():
        sims = sim_matrix(a, b).numpy().T                                            # the trainers' literal use
    assert sims.shape == (37, 157) and np.array_equal(sims, out_d.detach().cpu().numpy().T)
    with pytest.raises(RuntimeError, match="same device"):
        sim_matrix(a, b.cuda())


# ------------------------------------------------------------------------------------------------------ trainer flows
def _model(seed):
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.model import FrozenInTime
    net = FrozenInTime(VIDEO, TEXT)
    net.load_state_dict(syn.seeded_state_dict(syn.model_dims(num_frames=16), seed=seed), strict=True)
    net.text_model.config.dropout = net.text_model.config.attention_dropout = 0.0
    return net.cuda()


def test_zero_shot_valid_epoch_vs_reference_golden():
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model import metric
    from egovlp_b200.model.model import sim_matrix
    from tools.charades_sequence import valid_epoch
    g = load_golden("charades.npz")
    key = "zero_shot/"
    net = _model(41)
    prompts = {"input_ids": g[key + "prompt_ids"], "attention_mask": g[key + "prompt_mask"]}
    video = syn.synthetic_video(12, 4, seed=43)
    targets = g[key + "targets"].float()
    batches = [{"video": video[i:i + 4], "target": targets[i:i + 4],
                "text": {"input_ids": g[key + "clip_ids"][i:i + 4], "attention_mask": g[key + "clip_mask"][i:i + 4]}}
               for i in range(0, 12, 4)]
    res, sims, text_embeds, vid_embeds = valid_epoch(net, prompts, batches, torch.device("cuda"), sim_matrix,
                                                     [metric.charades_metrics])
    e_t, e_v = rel(text_embeds, g[key + "text_embeds"]), rel(vid_embeds, g[key + "vid_embeds"])
    _bound("zero-shot class-prompt text embeddings rel-L2", e_t, EMB_TOL)
    _bound("zero-shot video embeddings rel-L2", e_v, EMB_TOL)
    assert sims.shape == (12, 157) and isinstance(sims, np.ndarray)
    want = ep.charades_metrics(sims, targets.numpy())["mAP"]
    _bound("zero-shot mAP vs oracle on the same sims rel", max_rel([res["charades_metrics"]["mAP"]], [want]), 1e-9)
    print(f"[zero-shot] mAP {res['charades_metrics']['mAP']:.6f} (reference on its own sims "
          f"{float(g[key + 'mAP']):.6f})")
    # the class-prompt embeddings are the text tower's alone: equal to compute_text, whatever the dummy video holds
    with torch.no_grad():
        direct = net.compute_text({k: v.cuda() for k, v in prompts.items()}).cpu()
    assert torch.equal(text_embeds, direct)
    _, _, text_nan, _ = valid_epoch(net, prompts, batches[:1], torch.device("cuda"), sim_matrix, [],
                                    dummy_video=torch.full((1, 4, 3, 224, 224), float("nan")))
    assert torch.equal(text_nan, direct)


class _GradProbe:
    """An optimizer stand-in for tools.charades_sequence.train_step that records the gradients at `step()`."""

    def __init__(self, named):
        self.named, self.param_groups, self.grads = named, [{"lr": 0.0}], None

    def zero_grad(self):
        for p in self.named.values():
            p.grad = None

    def step(self):
        self.grads = {k: p.grad.detach().clone() for k, p in self.named.items() if p.grad is not None}


def _step_batch(seed):
    from egovlp_b200 import synthetic as syn
    return {"video": syn.synthetic_video(4, 16, seed=seed),
            "text": syn.synthetic_text(4, 16, seed=seed, ragged=True)}


def _oracle_loss(p, batch):
    from oracle import reference_port as rp
    data = {"video": batch["video"].cuda(), "text": {k: v.cuda() for k, v in batch["text"].items()}}
    t, v = rp.frozen_in_time_forward(data, p)
    return rp.norm_softmax_loss(rp.sim_matrix(t, v)), t, v


def test_charades_step_b4_t16_vs_fp32_oracle():
    """configs/ft/charades.json: 4 clips x 16 frames, NormSoftmaxLoss; embeddings, loss and every gradient."""
    from egovlp_b200.model.loss import NormSoftmaxLoss
    from egovlp_b200.model.model import sim_matrix
    from tools.charades_sequence import train_step
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    net = _model(51)
    batch = _step_batch(52)
    net.train()
    with torch.no_grad():
        t_got, v_got = net({"video": batch["video"].cuda(), "text": {k: v.cuda() for k, v in batch["text"].items()}})
    probe = _GradProbe(dict(net.named_parameters()))
    loss = train_step(net, NormSoftmaxLoss(), probe, batch, torch.device("cuda"), sim_matrix)
    p = {k: v.detach().clone().requires_grad_(True) for k, v in net.state_dict().items()}
    lr, t, v = _oracle_loss(p, batch)
    lr.backward()
    rows = [(k, cos(probe.grads[k], q.grad), q.grad.numel()) for k, q in p.items()
            if q.grad is not None and q.grad.norm() > 1e-12]
    assert all(k in probe.grads for k, _, _ in rows) and len(rows) >= 250
    c_all = cos(torch.cat([probe.grads[k].double().flatten() for k, _, _ in rows]),
                torch.cat([p[k].grad.double().flatten() for k, _, _ in rows]))
    worst_m = min((r for r in rows if r[2] > 4096), key=lambda r: r[1])
    _bound("charades step text embeddings rel-L2", rel(t_got, t), EMB_TOL)
    _bound("charades step video embeddings rel-L2", rel(v_got, v), EMB_TOL)
    _bound("charades step loss rel", abs(loss - lr.item()) / abs(lr.item()), STEP_LOSS_TOL)
    print(f"[charades step] whole-gradient cosine {c_all:.5f} over {len(rows)} tensors, lowest matrix cosine "
          f"{worst_m[1]:.5f} ({worst_m[0]})")
    assert c_all > 0.997 and worst_m[1] > 0.993


def _update_norm(params, before):
    return sum(((q.detach() - b).double().norm() ** 2).item() for q, b in zip(params, before)) ** 0.5


def test_charades_two_steps_with_lr_schedule_vs_oracle_torch_adamw():
    """Two trainer steps with `_adjust_learning_rate` between them (epoch 1 reaches milestone 1: lr x 0.1); the
    package's fused HF-AdamW against torch.optim.AdamW with HF's defaults on the fp32 oracle.
      * The update norm of each step tells whether the new lr reached the optimizer: the first Adam steps move each
        weight by about lr (m / sqrt(v) is about sign(g) while the gradient barely changes), so the second step's norm
        must be a tenth of the first's, for both optimizers.  Their norms are printed, not compared with each other: HF
        AdamW adds eps to sqrt(v) before the bias correction and torch.optim.AdamW after it, so at the same eps they damp
        small-gradient weights differently (on an H100 the package's first update norm measured 12 % below torch's).
      * Each step's loss is compared with the oracle's at the step tolerance, both computed from the same weights: after
        the first update the oracle's weights are set to the package's.  Without that the second loss would carry the
        difference of the two updates: an update of 1e-7 moves a weight's bf16 GEMM copy only where it crosses a
        rounding boundary, by a whole bf16 ulp, so which copies move follows the run-to-run noise of the gradients'
        fp32 atomics (the second loss varied by 1.2e-3 relative between runs on an H100).  lr keeps seeded-weight
        steps in the linear regime (see test_finetune_gpu.py)."""
    from egovlp_b200.model.loss import NormSoftmaxLoss
    from egovlp_b200.model.model import sim_matrix
    from egovlp_b200.optim import AdamW
    from tools.charades_sequence import adjust_learning_rate, train_step
    torch.backends.cuda.matmul.allow_tf32 = False
    args = types.SimpleNamespace(learning_rate1=1e-7, schedule=[1])
    net = _model(61)
    batch = _step_batch(62)
    p = {k: v.detach().clone().requires_grad_(True) for k, v in net.named_parameters()}
    ours, ref = list(net.parameters()), list(p.values())
    opt = AdamW(ours, lr=args.learning_rate1)
    ref_opt = torch.optim.AdamW(ref, lr=args.learning_rate1, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0)
    net.train()
    got, want, d_got, d_want = [], [], [], []
    for step in range(2):
        before = [q.detach().clone() for q in ours]
        got.append(train_step(net, NormSoftmaxLoss(), opt, batch, torch.device("cuda"), sim_matrix))
        d_got.append(_update_norm(ours, before))
        before = [q.detach().clone() for q in ref]
        ref_opt.zero_grad()
        lr, _, _ = _oracle_loss(p, batch)
        lr.backward()
        ref_opt.step()
        want.append(lr.item())
        d_want.append(_update_norm(ref, before))
        del before
        if step == 0:
            with torch.no_grad():
                for k, q in net.named_parameters():
                    p[k].copy_(q)
            adjust_learning_rate(opt, 1, args)
            adjust_learning_rate(ref_opt, 1, args)
            assert opt.param_groups[0]["lr"] == ref_opt.param_groups[0]["lr"] == pytest.approx(1e-8, rel=1e-12)
    print(f"[charades two steps] losses {got} vs oracle {want}; update norms {d_got} vs oracle {d_want}")
    for i, (a, b) in enumerate(zip(got, want)):
        _bound(f"charades step {i} loss rel (lr schedule)", abs(a - b) / abs(b), STEP_LOSS_TOL)
    assert got[1] < got[0]
    for name, d in (("package", d_got), ("oracle", d_want)):
        r = d[1] / d[0]
        print(f"[charades lr schedule] {name}: update norm ratio step1/step0 {r:.4f} (lr ratio 0.1)")
        assert 0.08 < r < 0.12, (name, d)
