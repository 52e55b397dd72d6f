"""ctypes binding of the C-ABI in include/egovlp_b200.h.  No CPU fallback: a missing library or a
non-zero return code raises."""
import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
# EGOVLP_B200_LIB: A/B a differently built library from the tools/ benchmarks (never a fallback: it must exist too)
LIB_PATH = os.environ.get("EGOVLP_B200_LIB") or os.path.join(_PKG, "lib", "libegovlp_b200.so")
_lib = None


class GemmEpilogue(C.Structure):
    _fields_ = [("bias", C.c_void_p), ("residual", C.c_void_p), ("aux", C.c_void_p), ("out", C.c_void_p),
                ("out2", C.c_void_p), ("ldr", C.c_longlong), ("ldaux", C.c_longlong), ("ldo", C.c_longlong),
                ("ldo2", C.c_longlong), ("out_mode", C.c_int), ("act", C.c_int), ("alpha", C.c_float),
                ("col_scale", C.c_float), ("col_scale_ncols", C.c_int), ("res_row_mod", C.c_int), ("colsum", C.c_void_p),
                ("colsum_a", C.c_void_p), ("drop_p", C.c_float), ("drop_site", C.c_uint), ("drop_seed", C.c_ulonglong),
                ("path_p", C.c_float), ("path_site", C.c_uint), ("path_rows", C.c_int), ("det_ws", C.c_void_p)]


class EgovlpError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EgovlpError(f"{LIB_PATH} is missing: build it with `python -m egovlp_b200.build` "
                              "(there is no CPU / PyTorch fallback for the hot path)")
        _lib = C.CDLL(LIB_PATH)
        _lib.egovlp_last_error.restype = C.c_char_p
        _lib.egovlp_divided_attn_workspace_floats.restype = C.c_longlong
        _lib.egovlp_egonce_fused_workspace_floats.restype = C.c_longlong
        _lib.egovlp_narrow_linear_workspace_floats.restype = C.c_longlong
        _lib.egovlp_space_attn_long_workspace_floats.restype = C.c_longlong
        for name in ("egovlp_gemm_det_workspace_floats", "egovlp_layernorm_bwd_det_workspace_floats",
                     "egovlp_colsum_det_workspace_floats", "egovlp_divided_attn_bwd_det_workspace_floats",
                     "egovlp_maxmargin_det_workspace_floats"):
            getattr(_lib, name).restype = C.c_longlong
    return _lib


# kernels launched per C-ABI call (memsets excluded) -- bench.py reports the count as `gpu_launches`
_KERNELS_PER_CALL = {"egovlp_egonce_fused_max_g": 0, "egovlp_divided_attn_fwd": 2, "egovlp_divided_attn_bwd": 2, "egovlp_video_embed_bwd": 2,
                     "egovlp_divided_attn_bwd_det": 2, "egovlp_video_embed_bwd_det": 3, "egovlp_layernorm_bwd_det": 2,
                     "egovlp_colsum_accum_det": 2, "egovlp_text_embed_bwd_det": 2, "egovlp_maxmargin_fwd_det": 2,
                     "egovlp_nce_fwd": 2, "egovlp_dual_softmax": 2, "egovlp_cross_entropy_fwd": 2,
                     "egovlp_narrow_linear_bwd": 3, "egovlp_text_attn_long_bwd": 3, "egovlp_space_attn_long_fwd": 2,
                     "egovlp_space_attn_long_bwd": 4}
_launches = 0


def reset_launch_count():
    global _launches
    _launches = 0


def launch_count():
    return _launches


def count_launches(n):
    """Kernels a call launched beyond its entry in _KERNELS_PER_CALL (those that depend on the arguments)."""
    global _launches
    _launches += n


def call(name, *args):
    global _launches
    fn = getattr(lib(), name)
    rc = fn(*args)
    _launches += _KERNELS_PER_CALL.get(name, 1)
    if rc != 0:
        raise EgovlpError(f"{name} failed ({rc}): {lib().egovlp_last_error().decode()}")


def declared_symbols():
    """Function names declared in include/egovlp_b200.h (used by the symbol-export test)."""
    import re
    hdr = os.path.join(os.path.dirname(_PKG), "include", "egovlp_b200.h")
    text = open(hdr).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(egovlp_[a-z0-9_]+)\s*\(", text)))
