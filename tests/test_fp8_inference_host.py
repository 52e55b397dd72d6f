"""CPU-only checks of the fp8 inference option: the config key and the setter are accepted, a bad value raises, the
state_dict is unchanged, and the e4m3 C-ABI entries reject bad shapes before touching the device."""
import ctypes as C
import warnings

import pytest

warnings.simplefilter("ignore")
VIDEO = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 4, "pretrained": True,
         "time_init": "zeros"}
TEXT = {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"}


def test_inference_precision_option():
    import torch
    from egovlp_b200.model.model import FrozenInTime
    torch.manual_seed(0)
    base = FrozenInTime(dict(VIDEO), dict(TEXT))
    assert base.video_model.inference_precision == "bf16"
    torch.manual_seed(0)
    net = FrozenInTime(dict(VIDEO, inference_precision="fp8"), dict(TEXT))
    assert net.video_model.inference_precision == "fp8"
    a, b = base.state_dict(), net.state_dict()
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    net.video_model.set_inference_precision("bf16")
    assert net.video_model.inference_precision == "bf16"
    with pytest.raises(ValueError):
        net.video_model.set_inference_precision("int8")
    with pytest.raises(ValueError):
        FrozenInTime(dict(VIDEO, inference_precision="fp16"), dict(TEXT))


def test_e4m3_entries_reject_bad_arguments():
    from egovlp_b200 import _lib
    p = C.c_void_p(256)                          # never dereferenced: the checks come first
    e = _lib.GemmEpilogue()
    e.out, e.ldo = 256, 320
    with pytest.raises(_lib.EgovlpError, match="bad shape"):
        _lib.call("egovlp_gemm_e4m3", p, C.c_longlong(768), p, C.c_longlong(768), p, p, 64, 320, 768, C.byref(e), None)
    with pytest.raises(_lib.EgovlpError, match="bad shape"):
        _lib.call("egovlp_gemm_e4m3", p, C.c_longlong(32), p, C.c_longlong(32), p, p, 64, 384, 24, C.byref(e), None)
    e.act = 3
    with pytest.raises(_lib.EgovlpError, match="epilogues"):
        _lib.call("egovlp_gemm_e4m3", p, C.c_longlong(768), p, C.c_longlong(768), p, p, 64, 384, 768, C.byref(e), None)
    with pytest.raises(_lib.EgovlpError, match="bad D"):
        _lib.call("egovlp_layernorm_fwd_e4m3", p, C.c_longlong(256), p, p, None, None, None, None, p, p, 16, 256,
                  C.c_float(1e-6), None)
    with pytest.raises(_lib.EgovlpError, match="bad args"):
        _lib.call("egovlp_quantize_rows_e4m3", p, C.c_longlong(6), p, p, 4, 6, None)
