"""CPU-only checks: the C-ABI library loads and exports every symbol include/egovlp_b200.h declares, the model
mirror keeps the reference's state_dict / constructor contract, the product path fails loudly without a GPU,
and the gather keeps the reference's local-slice backward (gloo, world_size 2)."""
import os
import subprocess
import sys
import warnings

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
warnings.simplefilter("ignore")


def test_library_exports_every_declared_symbol():
    from egovlp_b200 import _lib
    syms = _lib.declared_symbols()
    assert len(syms) >= 30 and "egovlp_gemm_bf16" in syms and "egovlp_divided_attn_bwd" in syms
    lib = _lib.lib()
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing
    assert lib.egovlp_abi_version() == 1


def test_argument_errors_are_reported_not_swallowed():
    import ctypes as C
    from egovlp_b200 import _lib
    with pytest.raises(_lib.EgovlpError, match="null pointer"):
        _lib.call("egovlp_layernorm_fwd", None, C.c_longlong(0), None, None, None, None, None, None, None, None, 4, 768,
                  C.c_float(1e-6), None)
    assert _lib.lib().egovlp_divided_attn_workspace_floats(2, 16, 196, 12, 0) == 2 * 12 * 28 * 4 * 66
    assert _lib.lib().egovlp_divided_attn_workspace_floats(2, 16, 196, 12, 1) == 2 * 12 * 16 * 4 * 66
    assert _lib.lib().egovlp_divided_attn_workspace_floats(2, 400, 196, 12, 0) == -1     # unsupported geometry


@pytest.mark.parametrize("field,value,msg", [
    ("bias", 0x40004, "8-byte aligned"), ("residual", 0x50004, "8-byte aligned"), ("colsum", 0x60004, "8-byte aligned"),
    ("out", 0x30004, "8-byte aligned"),                        # fp32 out (out_mode 1)
    ("aux", 0x70002, "4-byte aligned"), ("out2", 0x80002, "4-byte aligned"), ("out", 0x30002, "4-byte aligned"),
    ("ldr", 769, "even"), ("ldaux", 769, "even"), ("ldo2", 769, "even")])
def test_gemm_refuses_misaligned_epilogue_tensors(field, value, msg):
    """The generic epilogue moves bias / residual / fp32 out / colsum as float2 and aux / bf16 out / out2 as bf16x2:
    egovlp_gemm_bf16 must refuse a base or row stride that would misalign them, before any launch.  The addresses are
    made up, so this runs only where no GPU could be reached by a check that failed to refuse."""
    if torch.cuda.is_available():
        pytest.skip("made-up device addresses: not passed where a GPU is visible")
    import ctypes as C
    from egovlp_b200 import _lib
    M, N, K = 256, 768, 768
    e = _lib.GemmEpilogue()
    e.bias, e.residual, e.aux, e.out, e.out2 = 0x40000, 0x50000, 0x70000, 0x30000, 0x80000
    e.ldr = e.ldaux = e.ldo = e.ldo2 = N
    e.act, e.alpha, e.col_scale = 5, 1.0, 1.0                  # act 5 reads aux and writes out2
    e.out_mode = 1 if (field, msg) == ("out", "8-byte aligned") else 0
    setattr(e, field, value)
    with pytest.raises(_lib.EgovlpError, match=msg):
        _lib.call("egovlp_gemm_bf16", C.c_void_p(0x10000), 0, C.c_longlong(K), C.c_void_p(0x20000), 0,
                  C.c_longlong(K), M, N, K, C.byref(e), 1, None)


@pytest.mark.parametrize("field,value", [("x", 0x10004), ("add", 0x20008), ("y32", 0x30004), ("y16", 0x40004),
                                         ("y16", 0x40002)])
def test_dropout_refuses_misaligned_pointers(field, value):
    """egovlp_dropout reads x / add and writes y32 as float4, y16 as four bf16 at once: a base off 16 (8) bytes must be
    refused before any launch.  Made-up addresses, so only where no GPU is visible."""
    if torch.cuda.is_available():
        pytest.skip("made-up device addresses: not passed where a GPU is visible")
    import ctypes as C
    from egovlp_b200 import _lib
    ptrs = {"x": 0x10000, "add": 0x20000, "y32": 0x30000, "y16": 0x40000}
    ptrs[field] = value
    with pytest.raises(_lib.EgovlpError, match="aligned"):
        _lib.call("egovlp_dropout", *(C.c_void_p(ptrs[k]) for k in ("x", "add", "y32", "y16")), C.c_longlong(1024),
                  C.c_float(0.1), C.c_ulonglong(1), C.c_uint(0), None)


def test_text_attn_bwd_refuses_a_mask_that_is_not_contiguous_int64(monkeypatch):
    """The kernel reads the mask as int64 [B, L]: an int32 or strided mask would be read past its end or at the wrong
    keys, so ops.text_attn_bwd refuses it, as the forward does, before the C call."""
    from egovlp_b200 import ops
    reached = []
    monkeypatch.setattr(ops, "call", lambda name, *args: reached.append(name))
    monkeypatch.setattr(ops, "_stream", lambda: None)
    B, L, H = 2, 8, 1
    qkv, dqkv = torch.zeros(B * L, 3 * 64 * H, dtype=torch.bfloat16), torch.zeros(B * L, 3 * 64 * H, dtype=torch.bfloat16)
    dout = torch.zeros(B * L, 64 * H, dtype=torch.bfloat16)
    for bad in (torch.ones(B, L, dtype=torch.int32), torch.ones(L, B, dtype=torch.int64).t()):
        with pytest.raises(AssertionError):
            ops.text_attn_bwd(qkv, bad, dout, dqkv, B, L, H, 0.125)
    assert not reached
    ops.text_attn_bwd(qkv, torch.ones(B, L, dtype=torch.int64), dout, dqkv, B, L, H, 0.125)
    assert reached == ["egovlp_text_attn_bwd"]


def test_state_dict_contract_matches_reference_keys():
    from egovlp_b200 import synthetic as syn
    from egovlp_b200.model.model import FrozenInTime
    net = FrozenInTime({"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 16,
                        "pretrained": True, "time_init": "zeros"},
                       {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"})
    shapes = syn.state_dict_shapes(syn.model_dims(num_frames=16))
    sd = net.state_dict()
    assert set(sd) == set(shapes) and len(sd) == 327
    assert all(tuple(sd[k].shape) == tuple(v) for k, v in shapes.items())
    assert sum(p.numel() for p in net.parameters()) == 180_934_400
    # time_init='zeros' rule of the reference (video_transformer.py:90-96)
    ta = net.video_model.blocks[0].timeattn
    assert ta.qkv.weight.abs().sum() == 0 and torch.all(ta.proj.weight == 1) and ta.proj.bias.abs().sum() == 0
    assert "Trainable parameters: 180934400" in str(net)
    with pytest.raises(NotImplementedError):
        FrozenInTime({"model": "SpaceTimeTransformer"}, {"model": "distilbert-base-uncased", "pretrained": False})


def test_temporal_embed_inflation_and_dp_prefix():
    from egovlp_b200.model.model import FrozenInTime, state_dict_data_parallel_fix
    net = FrozenInTime({"model": "SpaceTimeTransformer", "num_frames": 16, "pretrained": True},
                       {"model": "distilbert-base-uncased", "pretrained": True}, load_temporal_fix="zeros")
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    sd["video_model.temporal_embed"] = torch.randn(1, 4, 768)
    out = net._inflate_positional_embeds(dict(sd))
    assert out["video_model.temporal_embed"].shape == (1, 16, 768)
    assert torch.equal(out["video_model.temporal_embed"][:, :4], sd["video_model.temporal_embed"])
    assert out["video_model.temporal_embed"][:, 4:].abs().sum() == 0
    net.load_temporal_fix = "bilinear"
    assert net._inflate_positional_embeds(dict(sd))["video_model.temporal_embed"].shape == (1, 16, 768)
    sd["video_model.temporal_embed"] = torch.randn(1, 32, 768)
    assert net._inflate_positional_embeds(dict(sd))["video_model.temporal_embed"].shape == (1, 16, 768)
    wrapped = {"module." + k: v for k, v in net.state_dict().items()}
    assert set(state_dict_data_parallel_fix(wrapped, net.state_dict())) == set(net.state_dict())


def test_product_path_fails_loudly_without_gpu():
    """No CPU / PyTorch fallback: on a machine without CUDA the forward raises instead of computing elsewhere."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from egovlp_b200.model.loss import NormSoftmaxLoss
    from egovlp_b200.model.model import sim_matrix
    with pytest.raises((AssertionError, RuntimeError)):
        sim_matrix(torch.randn(4, 8), torch.randn(4, 8))
    with pytest.raises((AssertionError, RuntimeError)):
        NormSoftmaxLoss()(torch.randn(4, 4))


def test_install_as_reference_model_aliases():
    import egovlp_b200
    egovlp_b200.install_as_reference_model()
    import model.model as mm
    import model.loss as ml
    assert mm.FrozenInTime.__module__ == "egovlp_b200.model.model" and hasattr(ml, "EgoNCE") and hasattr(mm, "sim_matrix")
    for k in [k for k in sys.modules if k == "model" or k.startswith("model.")]:
        del sys.modules[k]


def test_egomcq_metric_contract():
    from egovlp_b200.model.metric import egomcq_accuracy_metrics
    preds = torch.tensor([[0.1, 0.9, 0, 0, 0], [0.8, 0.1, 0, 0, 0], [0.2, 0.2, 0.9, 0, 0], [0.5, 0.5, 0.1, 0, 0]])
    labels = torch.tensor([1, 0, 0, 0])
    types = torch.tensor([1, 1, 2, 2])
    m = egomcq_accuracy_metrics(preds, labels, types)
    assert m == {"Intra-video": 100.0, "Inter-video": 50.0}      # sorted type ids zipped with the fixed name list


GLOO_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["EGOVLP_ROOT"])
from egovlp_b200.distributed import AllGatherLocalGrad, PackedGather
from oracle import reference_port as rp
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", rank=rank, world_size=world)
g = torch.Generator().manual_seed(5)
B, C = 3, 8
t_all, v_all = torch.randn(world * B, C, generator=g), torch.randn(world * B, C, generator=g)
verb_all = (torch.rand(world * B, 6, generator=g) > 0.6).float()
noun_all = (torch.rand(world * B, 10, generator=g) > 0.6).float()
sl = slice(rank * B, (rank + 1) * B)
t, v = t_all[sl].clone().requires_grad_(True), v_all[sl].clone().requires_grad_(True)
# (1) reference-style four separate gathers
tg, vg = AllGatherLocalGrad.apply(t), AllGatherLocalGrad.apply(v)
assert torch.equal(tg.detach(), t_all) and torch.equal(vg.detach(), v_all)
loss = rp.egonce_loss(rp.sim_matrix(tg, vg), rp.sim_matrix(verb_all, verb_all), rp.sim_matrix(noun_all, noun_all))
loss.backward()
# single-process full-batch oracle: local-slice backward == rows of the full gradient
tf, vf = t_all.clone().requires_grad_(True), v_all.clone().requires_grad_(True)
full = rp.gathered_step_loss([tf], [vf], [verb_all], [noun_all])
full.backward()
assert abs(loss.item() - full.item()) < 1e-6
assert torch.allclose(t.grad, tf.grad[sl], atol=1e-6) and torch.allclose(v.grad, vf.grad[sl], atol=1e-6)
# (2) ONE packed collective gives the same tensors and the same local-slice gradients
t2, v2 = t_all[sl].clone().requires_grad_(True), v_all[sl].clone().requires_grad_(True)
a, b, c, d = PackedGather.apply(t2, v2, verb_all[sl], noun_all[sl])
assert torch.equal(a.detach(), t_all) and torch.equal(b.detach(), v_all) and torch.equal(c, verb_all) and torch.equal(d, noun_all)
rp.egonce_loss(rp.sim_matrix(a, b), rp.sim_matrix(c, c), rp.sim_matrix(d, d)).backward()
assert torch.allclose(t2.grad, t.grad, atol=1e-7) and torch.allclose(v2.grad, v.grad, atol=1e-7)
# every rank sees the same loss
l = torch.tensor([loss.item()]); ls = [torch.zeros(1) for _ in range(world)]
dist.all_gather(ls, l)
assert all(abs(x.item() - loss.item()) < 1e-7 for x in ls)
dist.destroy_process_group()
print("OK", rank)
'''


def test_gather_semantics_gloo_world2(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(GLOO_WORKER)
    env = dict(os.environ, EGOVLP_ROOT=ROOT, MASTER_ADDR="127.0.0.1", MASTER_PORT="29541", WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r)), stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=180)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(outs)
    assert all("OK" in o for o in outs)


def test_bench_flop_model_matches_the_survey_and_the_oracle_counter():
    """bench.py's algorithmic-FLOP model (the numerator of every roofline fraction it prints) equals SURVEY.md 8d's
    figures, and its forward part equals torch's FLOP counter run on the oracle at a small shape."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(os.path.dirname(os.path.dirname(__file__)), "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    step, video, text = bench.flops_per_clip(16, 16)
    assert abs(video / 1e9 - 739.177) < 0.01 and abs(text / 1e9 - 1.364) < 0.01 and abs(step / 1e9 - 2217.9) < 0.1
    step4, video4, _ = bench.flops_per_clip(4, 16)
    assert abs(video4 / 1e9 - 184.617) < 0.01 and abs(step4 / 1e9 - 557.0) < 0.1
    a = type("A", (), {"frames": 16, "text_len": 16, "batch": 64, "workload": "cfg3"})()
    cfg = bench.workload_config(a, bench.WORKLOADS["cfg3"], 8)
    assert cfg["global_batch"] == 512 and cfg["parallelism"] == "dp8" and cfg["workload"].startswith("cfg3")
    assert set(bench.WORKLOADS) == {"cfg2", "cfg3", "cfg4", "cfg5"}
    # forward FLOPs of the tiny tower, counted by torch on the oracle, against the same formula
    from torch.utils.flop_counter import FlopCounterMode
    from oracle import reference_port as rp
    from egovlp_b200 import synthetic as syn
    d = syn.TINY_DIMS
    sd = syn.seeded_state_dict(d, seed=0, text=False, proj=False)
    vid = syn.synthetic_video(1, 4, seed=0, img=32)
    with FlopCounterMode(display=False) as fc:
        rp.video_tower(vid, sd, heads=2)
    N = (32 // 16) ** 2
    _, want, _ = bench.flops_per_clip(4, 8, N=N, D=128, H=2, HID=4 * 128, depth=2)
    want -= 2 * 128 * 256                                     # no projection head in video_tower()
    want -= 2 * 4 * N * 128 * 128 - 2 * 4 * N * 128 * (3 * 16 * 16)   # patch embed of a 16x16x3 patch: K = 768, not D
    assert abs(fc.get_total_flops() - want) / want < 0.02, (fc.get_total_flops(), want)


def test_wgrad_split_k_fills_whole_waves(monkeypatch):
    """engine._split_for: the split-K factor of a weight-gradient GEMM (128 x 256 tiles, 64-row k-blocks, one CTA per SM).
    At the step's shapes the units must fill >= 95 % of the waves they occupy, the kernel must not have to drop empty
    splits, and tiny contractions must still spread over the grid; EGOVLP_WGRAD_SPLIT=legacy restores round(400 / tiles)."""
    from egovlp_b200 import engine
    monkeypatch.delenv("EGOVLP_WGRAD_SPLIT", raising=False)
    engine._split_for.cache_clear()
    n_sm = 132                                              # H100 SXM
    for n_out, n_in in ((2304, 768), (768, 768), (3072, 768), (768, 3072), (256, 768), (768, 256)):
        for rows in (64 * 3137, 64 * 785, 32 * 3137, 8 * 3137):
            s = engine._split_for(n_out, n_in, rows, n_sm)
            tiles = -(-n_out // 128) * -(-n_in // 256)
            num_kb = -(-rows // 64)
            assert 1 <= s <= 64
            kbs = -(-num_kb // s)
            assert -(-num_kb // kbs) == s                       # no empty splits
            units = tiles * s
            assert units / (-(-units // n_sm) * n_sm) >= 0.9, (n_out, n_in, rows, s)
    # 1024 text tokens: 16 k-blocks only -- still more than one unit per tile
    assert engine._split_for(768, 768, 1024, n_sm) > 1
    # fc1 weight gradient at 64 clips x 16 frames: 9 splits (648 units = 4.91 waves), not 6 (432 units = 3.27 waves)
    assert engine._split_for(3072, 768, 64 * 3137, n_sm) == 9
    monkeypatch.setenv("EGOVLP_WGRAD_SPLIT", "legacy")
    engine._split_for.cache_clear()
    assert engine._split_for(3072, 768, 64 * 3137, n_sm) == 6
    engine._split_for.cache_clear()
