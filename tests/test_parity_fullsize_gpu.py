"""Numeric parity at the headline shapes: the CUDA path (bf16 tensor-core operands, fp32 accumulation / residual stream)
against the fp32 oracle (oracle/reference_port.py) executed ON THE GPU with TF32 off, on identical seeded inputs.

  (i)   cfg3 per-GPU shape scaled to fit the oracle's activation memory: B=8 clips x 16 frames x 224^2, L=16 ragged,
        12 blocks, EgoNCE over G=8 -- embeddings, loss, and cosine / norm of the gradients of ALL 327 tensors;
  (ii)  cfg2: B=64 clips x 4 frames, EgoNCE over G=64 -- embeddings and loss;
  (iii) cfg5: EgoMCQ, 1024 queries x 5 candidate clips x 4 frames through the bf16 towers -- argmax against the fp32
        oracle run through ITS towers (not shared embeddings), with the top-2 margin analysis;
  (iv)  weights updated through `p.data` (transformers.AdamW 4.x style) are seen by the next forward.

Tolerances come from the error budget of DESIGN.md section 6 (tools/error_budget.py: bf16 rounding of the MMA operands
alone puts the embeddings 3-6e-3 from fp32 at this depth); the measured values are printed and written as parity_*.json
records to EGOVLP_RECORD_DIR.  The north_star's 1e-3 holds for the loss, not for 12-block bf16
embeddings -- see DESIGN.md section 6 for the evidence."""
import json
import os
import tempfile
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu
warnings.simplefilter("ignore")

EMB_TOL = 9e-3          # rel-L2 of [B,256] embeddings vs fp32 (budget: 3-6e-3 measured, x1.5)
LOSS_TOL = 1e-3         # relative, the north_star's figure
# parity records go where EGOVLP_RECORD_DIR points (default: a temporary directory), never into the source tree
OUT = os.environ.get("EGOVLP_RECORD_DIR") or os.path.join(tempfile.gettempdir(), "egovlp_records")


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def cos(a, b):
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-300)).item()


def _record(name, payload):
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, f"parity_{name}.json"), "w") as f:
        json.dump(payload, f, indent=1)


@pytest.fixture(scope="module")
def setup():
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.model import FrozenInTime
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = syn.seeded_state_dict(syn.model_dims(num_frames=16), seed=0)
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 16,
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    net.load_state_dict(sd, strict=True)
    net.text_model.config.dropout = net.text_model.config.attention_dropout = 0.0       # deterministic parity path
    net.cuda()
    params = {k: v.cuda() for k, v in sd.items()}
    return net, params


def _batch(B, T, L, seed, ragged=True):
    from egovlp_b200 import synthetic as syn
    data = {"video": syn.synthetic_video(B, T, seed=seed).cuda(),
            "text": {k: v.cuda() for k, v in syn.synthetic_text(B, L, seed=seed, ragged=ragged).items()}}
    verb, noun = [t.cuda() for t in syn.synthetic_tags(B, seed=seed)]
    return data, verb, noun


def test_cfg3_shape_b8_t16_embeddings_loss_and_all_327_gradients(setup):
    from egovlp_b200.model.loss import EgoNCE
    from oracle import reference_port as rp
    net, params = setup
    B, T, L = 8, 16, 16
    data, verb, noun = _batch(B, T, L, seed=5)
    net.zero_grad(set_to_none=True)
    t, v = net(data)
    loss = EgoNCE().fused(t, v, verb, noun)
    loss.backward()
    p = {k: w.clone().requires_grad_(True) for k, w in params.items()}
    tr, vr = rp.frozen_in_time_forward(data, p)
    lr = rp.egonce_loss(rp.sim_matrix(tr, vr), rp.sim_matrix(verb, verb), rp.sim_matrix(noun, noun))
    lr.backward()
    e_t, e_v = rel(t, tr), rel(v, vr)
    e_l = abs(loss.item() - lr.item()) / abs(lr.item())
    rows = []
    for k, w in net.named_parameters():
        g, gr = w.grad, p[k].grad
        if gr is None or gr.norm().item() < 1e-12 or k.endswith("k_lin.bias"):
            continue                 # k-bias gradients are analytically zero (softmax shift invariance): pure rounding noise
        rows.append((k, cos(g, gr), g.double().norm().item() / gr.double().norm().item(), gr.numel()))
    mats = [r for r in rows if r[3] > 4096]
    vecs = [r for r in rows if r[3] <= 4096]
    worst_m = min(mats, key=lambda r: r[1])
    worst_v = min(vecs, key=lambda r: r[1])
    norm_m = max(abs(r[2] - 1) for r in mats)
    norm_v = max(abs(r[2] - 1) for r in vecs)
    # gradient of everything at once: cosine of the concatenation of all 327 tensors
    flat_g = torch.cat([w.grad.double().flatten() for k, w in net.named_parameters() if p[k].grad is not None])
    flat_r = torch.cat([p[k].grad.double().flatten() for k, w in net.named_parameters() if p[k].grad is not None])
    cos_all = cos(flat_g, flat_r)
    rel_all = rel(flat_g, flat_r)
    payload = {"shape": [B, T, L], "rel_text_emb": e_t, "rel_video_emb": e_v, "loss": loss.item(), "loss_ref": lr.item(),
               "rel_loss": e_l, "n_tensors": len(rows), "grad_cos_all": cos_all, "grad_rel_all": rel_all,
               "worst_matrix": worst_m[:3], "worst_vector": worst_v[:3], "max_norm_dev_matrix": norm_m,
               "max_norm_dev_vector": norm_v,
               "lowest_cos": sorted([(r[1], r[0]) for r in rows])[:8]}
    _record("cfg3_b8_t16", payload)
    print("\n[cfg3 B=8 T=16]", json.dumps(payload))
    assert len(rows) >= 318, len(rows)
    assert e_t < EMB_TOL and e_v < EMB_TOL, (e_t, e_v)
    assert e_l < LOSS_TOL, (loss.item(), lr.item())
    # gradients: the error budget (tools/error_budget.py) puts the whole-gradient distance of a bf16-operand step at
    # 5-6e-2
    assert cos_all > 0.997 and rel_all < 8.5e-2, (cos_all, rel_all)
    assert worst_m[1] > 0.993, worst_m
    assert worst_v[1] > 0.98, worst_v
    assert norm_m < 0.03, norm_m


def test_cfg2_b64_t4_embeddings_and_loss(setup):
    from egovlp_b200.model.loss import EgoNCE
    from oracle import reference_port as rp
    net, params = setup
    B, T, L = 64, 4, 16
    data, verb, noun = _batch(B, T, L, seed=6)
    with torch.no_grad():
        t, v = net(data)
        loss = EgoNCE().fused(t, v, verb, noun)
        tr = rp.compute_text(data["text"], params)
        vr = torch.cat([rp.compute_video(data["video"][i:i + 16], params) for i in range(0, B, 16)])
        lr = rp.egonce_loss(rp.sim_matrix(tr, vr), rp.sim_matrix(verb, verb), rp.sim_matrix(noun, noun))
    e_t, e_v, e_l = rel(t, tr), rel(v, vr), abs(loss.item() - lr.item()) / abs(lr.item())
    payload = {"shape": [B, T, L], "rel_text_emb": e_t, "rel_video_emb": e_v, "loss": loss.item(), "loss_ref": lr.item(),
               "rel_loss": e_l}
    _record("cfg2_b64_t4", payload)
    print("\n[cfg2 B=64 T=4]", json.dumps(payload))
    assert e_t < EMB_TOL and e_v < EMB_TOL, (e_t, e_v)
    assert e_l < LOSS_TOL, (loss.item(), lr.item())


def test_cfg5_egomcq_argmax_through_the_towers(setup):
    """1024 queries x 5 candidates x 4 frames: bf16 towers + egomcq kernel vs the fp32 oracle's towers + argmax."""
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.metric import egomcq_predict
    from oracle import reference_port as rp
    net, params = setup
    Q, K, T, L, CH = 1024, 5, 4, 16, 128
    text = {k: v.cuda() for k, v in syn.synthetic_text(Q, L, seed=9, ragged=True).items()}
    v_gpu, v_ref = [], []
    with torch.no_grad():
        t_gpu = net.compute_text(text)
        t_ref = torch.cat([rp.compute_text({k: x[i:i + 256] for k, x in text.items()}, params) for i in range(0, Q, 256)])
        for c in range(0, Q * K, CH):                         # clips generated chunk-wise (5120 x 4f = 12 GB in fp32)
            clips = syn.synthetic_video(CH, T, seed=1000 + c).cuda()
            v_gpu.append(net.compute_video(clips))
            v_ref.append(torch.cat([rp.compute_video(clips[i:i + 32], params) for i in range(0, CH, 32)]))
        v_gpu, v_ref = torch.cat(v_gpu).view(Q, K, -1), torch.cat(v_ref).view(Q, K, -1)
        s_gpu, pred = egomcq_predict(t_gpu, v_gpu)
        s_ref, pred_ref = rp.egomcq_predict(t_ref, v_ref)
    err = (s_gpu - s_ref).abs().max().item()                  # worst score error of the bf16 path
    top2 = s_ref.topk(2, dim=1).values
    margin = (top2[:, 0] - top2[:, 1])
    decided = margin > 2 * err                                # a flip needs two scores to move by > margin / 2 each
    agree = (pred == pred_ref)
    payload = {"queries": Q, "max_abs_score_err": err, "min_top2_margin": margin.min().item(),
               "median_top2_margin": margin.median().item(), "n_decided": int(decided.sum()),
               "agree_all": int(agree.sum()), "agree_decided": int((agree & decided).sum()),
               "rel_text_emb": rel(t_gpu, t_ref), "rel_video_emb": rel(v_gpu, v_ref)}
    _record("cfg5_egomcq", payload)
    print("\n[cfg5 EgoMCQ]", json.dumps(payload))
    assert err < 2e-2
    assert bool(agree[decided].all()), "argmax differs on a query whose top-2 margin exceeds the score error bound"
    # synthetic clips make near-ties the rule (median top-2 margin 5e-3 vs a worst score error of 1.8e-3; measured: 631 of
    # 1024 queries decided, 631 / 631 of them agree, 1003 / 1024 overall): every disagreement must sit inside the error bound
    assert bool((~agree <= ~decided).all()) and agree.float().mean().item() > 0.95
    # same embeddings on both sides -> bit-exact indices (the kernel itself, incl. tie rule)
    assert torch.equal(egomcq_predict(t_ref, v_ref)[1], pred_ref)


def test_weights_updated_through_data_are_seen(setup):
    """ADVICE r1: an optimizer writing p.data (no version bump) must not leave stale bf16 GEMM operands behind."""
    from egovlp_b200 import synthetic as syn
    net, _ = setup
    video = syn.synthetic_video(2, 4, seed=3).cuda()
    with torch.no_grad():
        before = net.compute_video(video).clone()
    w = net.video_model.blocks[3].mlp.fc1.weight
    saved = w.detach().clone()
    ver = w._version
    w.data.mul_(1.5)                                          # transformers.AdamW 4.x / apex style update
    assert w._version == ver
    try:
        with torch.enable_grad():
            after_train = net.compute_video(video)            # training forward: multi-tensor refresh
        assert rel(after_train, before) > 1e-3
        # a torch.optim optimizer stepping through .data is caught by the global post-step hook even under no_grad
        w.data.copy_(saved)

        class DataSGD(torch.optim.Optimizer):
            def __init__(self, params):
                super().__init__(params, {})

            def step(self):
                for g in self.param_groups:
                    for p in g["params"]:
                        p.data.mul_(1.5)

        DataSGD([w]).step()
        assert w._version == ver
        with torch.no_grad():
            after_eval = net.compute_video(video)
        assert rel(after_eval, after_train) < 1e-6
    finally:
        w.data.copy_(saved)
        with torch.enable_grad():
            net.compute_video(video)
    with torch.no_grad():
        assert rel(net.compute_video(video), before) < 1e-6
