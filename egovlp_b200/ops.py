"""Tensor-level wrappers over the C-ABI (include/egovlp_b200.h).  torch is used only for device memory and
the current stream; every computation happens in libegovlp_b200.so."""
import ctypes as C

import torch

from ._lib import GemmEpilogue, call, count_launches, lib

BF16, F32, E4M3 = torch.bfloat16, torch.float32, torch.float8_e4m3fn


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def deterministic():
    """torch.are_deterministic_algorithms_enabled(), read at every call as torch reads it: while it is set, every op
    below that reduces across CTAs takes its deterministic form (partials in a workspace, merged in an order that
    depends on the shapes only), so equal inputs give equal bits.  An op without such a form raises RuntimeError."""
    return torch.are_deterministic_algorithms_enabled()


_det_cache = {}       # (device index, stream) -> the fp32 workspace of the deterministic forms, grown on demand


def _det_ws(n_floats, device):
    """Workspace of a deterministic form: one buffer per (device, stream), grown on demand and shared by the calls on
    that stream (stream order keeps them apart).  The kernels write every element they read back, so the buffer is
    allocated once instead of per call: under torch's deterministic mode a fresh torch.empty is NaN-filled, which for
    the weight gradients alone would be 9 x 9.4 MB of fill per fc1 / fc2 call."""
    assert n_floats >= 0, "deterministic form: unsupported shape"
    device = torch.device(device)
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _det_cache.get(key)
    if buf is None or buf.numel() < n_floats:
        _det_cache[key] = buf = torch.empty(max(int(n_floats), 1), dtype=F32, device=device)
    return buf


def _chk(t, dtype, name):
    assert t.is_cuda and t.dtype == dtype, f"{name}: expected cuda {dtype}, got {t.device} {t.dtype}"


_prof = None         # bench.py's live roofline probe: {kind: [(work, start event, end event), ...]}


def profile(enable):
    """CUDA events (on the launching stream) around every GEMM / divided-attention / LayerNorm launch.
    profile(True) starts recording; profile(False) returns {kind: (work, milliseconds, launches)} where `work` is the
    algorithmic FLOPs (kind 'gemm') or algorithmic HBM bytes (the HBM-bound kinds) of the recorded launches."""
    global _prof
    if enable:
        _prof = {}
        return None
    rec, _prof = _prof or {}, None
    torch.cuda.synchronize()
    return {k: (sum(r[0] for r in v), sum(r[1].elapsed_time(r[2]) for r in v), len(v)) for k, v in rec.items()}


def profile_gemm(enable):
    """GEMM-only view of `profile` (tools/): profile_gemm(False) -> (flops, milliseconds, launches)."""
    res = profile(enable)
    return None if enable else res.get("gemm", (0.0, 0.0, 0))


class _Probe:
    """`with _Probe(kind, work):` records one launch when profiling is on (no-op otherwise)."""
    __slots__ = ("kind", "work", "e0")

    def __init__(self, kind, work):
        self.kind, self.work, self.e0 = kind, work, None

    def __enter__(self):
        if _prof is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *exc):
        if self.e0 is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            _prof.setdefault(self.kind, []).append((self.work, self.e0, e1))
        return False


def gemm(a, b, out, *, a_mn=False, b_mn=False, bias=None, residual=None, aux=None, out2=None, act=0, alpha=1.0,
         col_scale=1.0, col_scale_ncols=0, accumulate=False, split_k=1, res_row_mod=0, colsum=None, colsum_a=None,
         drop=None):
    """out = epi(A @ B^T).  a: [M,K] (or [K,M] if a_mn), b: [N,K] (or [K,N] if b_mn); 2-D, last-dim contiguous.
    out: bf16 or fp32 [M,N]; accumulate=True -> fp32 atomic add into `out` (required for split_k>1).
    drop: None or a `Drop`: the epilogue's dropout forms (include/egovlp_b200.h, egovlp_gemm_epilogue.drop_*).
    Under `deterministic()`, accumulate / colsum_a take the workspace form (egovlp_gemm_epilogue.det_ws): out +=
    P_0 + ... + P_{s-1} left to right over the splits' partial tiles."""
    _chk(a, BF16, "a"); _chk(b, BF16, "b")
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    (K, M) = a.shape if a_mn else a.shape[::-1]
    (Kb, N) = b.shape if b_mn else b.shape[::-1]
    assert K == Kb, (a.shape, b.shape, a_mn, b_mn)
    assert out.shape == (M, N) and out.stride(1) == 1 and out.dtype in (BF16, F32)
    e = GemmEpilogue()
    e.bias = bias.data_ptr() if bias is not None else None
    e.residual = residual.data_ptr() if residual is not None else None
    e.aux = aux.data_ptr() if aux is not None else None
    e.out = out.data_ptr()
    e.out2 = out2.data_ptr() if out2 is not None else None
    e.ldr = residual.stride(0) if residual is not None else 0
    e.ldaux = aux.stride(0) if aux is not None else 0
    e.ldo = out.stride(0)
    e.ldo2 = out2.stride(0) if out2 is not None else 0
    if bias is not None:
        _chk(bias, F32, "bias"); assert bias.numel() == N
    if residual is not None:
        _chk(residual, F32, "residual")
        assert residual.shape == ((res_row_mod or M), N) and residual.stride(1) == 1
    if aux is not None:
        _chk(aux, BF16, "aux"); assert aux.shape == (M, N)
    if out2 is not None:
        _chk(out2, BF16, "out2"); assert out2.shape == (M, N)
    if accumulate:
        assert out.dtype == F32
        e.out_mode = 2
    else:
        e.out_mode = 0 if out.dtype == BF16 else 1
    e.act, e.alpha, e.col_scale, e.col_scale_ncols = act, alpha, col_scale, col_scale_ncols
    e.res_row_mod = res_row_mod
    if colsum is not None:
        _chk(colsum, F32, "colsum"); assert colsum.numel() == N
    e.colsum = colsum.data_ptr() if colsum is not None else None
    if colsum_a is not None:                 # wgrad form only: column sums of A accumulated from the smem tiles
        _chk(colsum_a, F32, "colsum_a"); assert a_mn and b_mn and colsum_a.numel() == M
    e.colsum_a = colsum_a.data_ptr() if colsum_a is not None else None
    ws = None
    det = deterministic()
    if det and colsum is not None:
        raise RuntimeError("egovlp gemm: the output column sums (colsum) have no deterministic form; "
                           "use colsum_accum on the output instead")
    # one split without colsum_a adds each element once: the atomic form is already deterministic
    if det and ((accumulate and split_k > 1) or colsum_a is not None):
        ws = _det_ws(lib().egovlp_gemm_det_workspace_floats(M, N, K, split_k), out.device)
        e.det_ws = ws.data_ptr()
    if drop is not None:
        e.drop_p, e.drop_seed, e.drop_site = drop.p, drop.seed, drop.site
        e.path_p, e.path_site, e.path_rows = drop.path_p, drop.path_site, drop.path_rows
    with _Probe("gemm", 2.0 * M * N * K):
        call("egovlp_gemm_bf16", _ptr(a), int(a_mn), C.c_longlong(a.stride(0)), _ptr(b), int(b_mn),
             C.c_longlong(b.stride(0)), M, N, K, C.byref(e), split_k, _stream())
    if ws is not None:              # the ordered merge passes of the deterministic form
        count_launches(int(accumulate) + int(colsum_a is not None))
    return out


def layernorm_fwd(x, gamma, beta, eps, *, add=None, sum_out=None, y16=None, y32=None, mean=None, rstd=None, y8=None,
                  row_scale=None):
    """x fp32 [rows, D] (row stride free).  Returns nothing; writes the provided outputs.  y8 (float8_e4m3fn [rows, D])
    with row_scale (fp32 [rows]): the output as the A operand of `gemm_e4m3` (no `add` / `sum_out` then)."""
    _chk(x, F32, "x")
    rows, D = x.shape
    assert x.stride(1) == 1
    for t in (add, sum_out, y32):
        assert t is None or (t.dtype == F32 and t.is_contiguous() and t.shape == (rows, D))
    assert y16 is None or (y16.dtype == BF16 and y16.is_contiguous() and y16.shape == (rows, D))
    assert (y8 is None) == (row_scale is None), "y8 and row_scale go together"
    nbytes = rows * D * (4 + 4 * (add is not None) + 4 * (sum_out is not None) + 2 * (y16 is not None) + 4 * (y32 is not None)
                         + (y8 is not None))
    if y8 is not None:
        assert add is None and sum_out is None
        _chk(y8, E4M3, "y8"); _chk(row_scale, F32, "row_scale")
        assert y8.is_contiguous() and y8.shape == (rows, D) and row_scale.is_contiguous() and row_scale.numel() == rows
        with _Probe("layernorm_fwd", nbytes):
            call("egovlp_layernorm_fwd_e4m3", _ptr(x), C.c_longlong(x.stride(0)), _ptr(gamma), _ptr(beta), _ptr(y16),
                 _ptr(y32), _ptr(mean), _ptr(rstd), _ptr(y8), _ptr(row_scale), rows, D, C.c_float(eps), _stream())
        return
    with _Probe("layernorm_fwd", nbytes):
        call("egovlp_layernorm_fwd", _ptr(x), C.c_longlong(x.stride(0)), _ptr(add), _ptr(sum_out), _ptr(gamma),
             _ptr(beta), _ptr(y16), _ptr(y32), _ptr(mean), _ptr(rstd), rows, D, C.c_float(eps), _stream())


def layernorm_bwd(dy, x, gamma, mean, rstd, *, add1=None, add2=None, dx=None, dx16=None, dgamma=None, dbeta=None,
                  colsum_dx=None):
    """dx = LNbwd(dy) + add1 + add2.  dy / add1 / add2 may each be fp32 or bf16."""
    _chk(x, F32, "x")
    rows, D = x.shape
    assert dy.is_cuda and dy.dtype in (F32, BF16) and dy.shape == (rows, D) and dy.stride(1) == 1 and x.stride(1) == 1
    for t in (add1, add2):
        assert t is None or (t.dtype in (F32, BF16) and t.is_contiguous() and t.shape == (rows, D))
    assert dx is None or (dx.dtype == F32 and dx.shape == (rows, D) and dx.stride(1) == 1)
    assert dx16 is None or (dx16.dtype == BF16 and dx16.is_contiguous() and dx16.shape == (rows, D))
    nbytes = rows * D * (dy.element_size() + 4 + sum(t.element_size() for t in (add1, add2) if t is not None)
                         + 4 * (dx is not None) + 2 * (dx16 is not None))
    args = (_ptr(dy), int(dy.dtype == BF16), C.c_longlong(dy.stride(0)), _ptr(x), C.c_longlong(x.stride(0)),
            _ptr(gamma), _ptr(mean), _ptr(rstd), _ptr(add1), int(add1 is not None and add1.dtype == BF16), _ptr(add2),
            int(add2 is not None and add2.dtype == BF16), _ptr(dx), C.c_longlong(dx.stride(0) if dx is not None else D),
            _ptr(dx16), _ptr(dgamma), _ptr(dbeta), _ptr(colsum_dx), rows, D)
    with _Probe("layernorm_bwd", nbytes):
        if deterministic() and (dgamma is not None or dbeta is not None or colsum_dx is not None):
            ws = _det_ws(lib().egovlp_layernorm_bwd_det_workspace_floats(rows, D), x.device)
            call("egovlp_layernorm_bwd_det", *args, _ptr(ws), _stream())
        else:
            call("egovlp_layernorm_bwd", *args, _stream())


def gemm_e4m3(a8, a_scale, b8, b_scale, out, *, bias=None, act=0, alpha=1.0, col_scale=1.0, col_scale_ncols=0):
    """out bf16 [M, N] = epi((a8 @ b8^T) * a_scale[:, None] * b_scale[None, :]); a8 [M, K] / b8 [N, K] float8_e4m3fn,
    K-major; epi = bias, then the column scale (act 0) or GELU (act 1) -- see egovlp_gemm_e4m3."""
    _chk(a8, E4M3, "a8"); _chk(b8, E4M3, "b8"); _chk(a_scale, F32, "a_scale"); _chk(b_scale, F32, "b_scale")
    _chk(out, BF16, "out")
    assert a8.dim() == 2 and b8.dim() == 2 and a8.stride(1) == 1 and b8.stride(1) == 1
    (M, K), (N, Kb) = a8.shape, b8.shape
    assert K == Kb and out.shape == (M, N) and out.stride(1) == 1, (a8.shape, b8.shape, out.shape)
    assert a_scale.is_contiguous() and a_scale.numel() == M and b_scale.is_contiguous() and b_scale.numel() == N
    e = GemmEpilogue()
    if bias is not None:
        _chk(bias, F32, "bias"); assert bias.numel() == N
        e.bias = bias.data_ptr()
    e.out, e.ldo, e.out_mode = out.data_ptr(), out.stride(0), 0
    e.act, e.alpha, e.col_scale, e.col_scale_ncols = act, alpha, col_scale, col_scale_ncols
    with _Probe("gemm_e4m3", 2.0 * M * N * K):
        call("egovlp_gemm_e4m3", _ptr(a8), C.c_longlong(a8.stride(0)), _ptr(b8), C.c_longlong(b8.stride(0)),
             _ptr(a_scale), _ptr(b_scale), M, N, K, C.byref(e), _stream())
    return out


def quantize_rows_e4m3(w, q=None, scale=None):
    """fp32 [N, K] -> (float8_e4m3fn [N, K], fp32 [N] per-row scales), see egovlp_quantize_rows_e4m3."""
    _chk(w, F32, "w")
    assert w.dim() == 2 and w.stride(1) == 1
    N, K = w.shape
    q = torch.empty(N, K, dtype=E4M3, device=w.device) if q is None else q
    scale = torch.empty(N, dtype=F32, device=w.device) if scale is None else scale
    _chk(q, E4M3, "q"); _chk(scale, F32, "scale")
    assert q.is_contiguous() and q.shape == (N, K) and scale.is_contiguous() and scale.numel() == N
    call("egovlp_quantize_rows_e4m3", _ptr(w), C.c_longlong(w.stride(0)), _ptr(q), _ptr(scale), N, K, _stream())
    return q, scale


def cast_bf16(src, dst=None):
    _chk(src, F32, "src")
    assert src.is_contiguous()
    if dst is None:
        dst = torch.empty(src.shape, dtype=BF16, device=src.device)
    call("egovlp_cast_f32_to_bf16", _ptr(src), _ptr(dst), C.c_longlong(src.numel()), _stream())
    return dst


class _CastDesc(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("numel", C.c_longlong)]


def build_cast_table(pairs):
    """Device-side descriptor / chunk tables for `cast_multi`: pairs = [(fp32 src, bf16 dst), ...] (contiguous)."""
    chunk = lib().egovlp_adamw_chunk_elems()
    descs = (_CastDesc * len(pairs))()
    ct, co = [], []
    for i, (src, dst) in enumerate(pairs):
        _chk(src, F32, "src"); _chk(dst, BF16, "dst")
        assert src.is_contiguous() and dst.is_contiguous() and src.numel() == dst.numel()
        descs[i] = _CastDesc(src.data_ptr(), dst.data_ptr(), src.numel())
        n = (src.numel() + chunk - 1) // chunk
        ct += [i] * n
        co += list(range(n))
    dev = pairs[0][0].device
    raw = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).to(dev)
    return raw, torch.tensor(ct, dtype=torch.int32, device=dev), torch.tensor(co, dtype=torch.int32, device=dev)


def cast_multi(raw, chunk_tensor, chunk_offset):
    """fp32 -> bf16 for every (src, dst) pair of a table from `build_cast_table`, one launch."""
    call("egovlp_cast_multi_f32_to_bf16", _ptr(raw), _ptr(chunk_tensor), _ptr(chunk_offset), chunk_tensor.numel(),
         _stream())


def colsum_accum(dy, out):
    """out[n] += sum_m dy[m,n]; dy bf16/fp32 [M,N]."""
    assert dy.dim() == 2 and dy.stride(1) == 1 and out.dtype == F32 and out.numel() == dy.shape[1]
    args = (_ptr(dy), int(dy.dtype == F32), C.c_longlong(dy.stride(0)), _ptr(out), dy.shape[0], dy.shape[1])
    if deterministic():
        ws = _det_ws(lib().egovlp_colsum_det_workspace_floats(dy.shape[0], dy.shape[1], int(dy.dtype == F32)), dy.device)
        call("egovlp_colsum_accum_det", *args, _ptr(ws), _stream())
    else:
        call("egovlp_colsum_accum", *args, _stream())


def divided_attn_fwd(qkv, B, T, N, H, mode):
    """qkv bf16 [B*S, 3*64*H] (q pre-scaled) -> (out bf16 [B*S, D], lse fp32 [B, H, S]).  mode: 0 time, 1 space."""
    _chk(qkv, BF16, "qkv")
    S, D = 1 + T * N, 64 * H
    assert qkv.is_contiguous() and qkv.shape == (B * S, 3 * D)
    out = torch.empty(B * S, D, dtype=BF16, device=qkv.device)
    lse = torch.empty(B, H, S, dtype=F32, device=qkv.device)
    n_ws = lib().egovlp_divided_attn_workspace_floats(B, T, N, H, mode)
    assert n_ws > 0, "unsupported attention geometry"
    ws = torch.empty(n_ws, dtype=F32, device=qkv.device)
    # algorithmic bytes: read q|k|v once (3 x 2 D), write the output (2 D) and the lse (4 H) per token
    with _Probe("attn_time_fwd" if mode == 0 else "attn_space_fwd", B * S * (8 * D + 4 * H)):
        call("egovlp_divided_attn_fwd", _ptr(qkv), _ptr(out), _ptr(lse), _ptr(ws), B, T, N, H, mode, _stream())
    return out, lse


def divided_attn_bwd(qkv, out, dout, lse, B, T, N, H, mode, q_scale, dqkv=None):
    _chk(qkv, BF16, "qkv"); _chk(out, BF16, "out"); _chk(dout, BF16, "dout"); _chk(lse, F32, "lse")
    assert qkv.is_contiguous() and out.is_contiguous() and dout.is_contiguous() and lse.is_contiguous()
    if dqkv is None:
        dqkv = torch.empty_like(qkv)
    det = deterministic()
    if det:      # one CLS-row slot per group (and part), summed in order
        ws = _det_ws(lib().egovlp_divided_attn_bwd_det_workspace_floats(B, T, N, H, mode), qkv.device)
    else:
        ws = torch.empty(B * H * 3 * 64, dtype=F32, device=qkv.device)
    S, D = 1 + T * N, 64 * H
    # algorithmic bytes: read q|k|v, out, dout and the lse once, write dq|dk|dv
    with _Probe("attn_time_bwd" if mode == 0 else "attn_space_bwd", B * S * (16 * D + 4 * H)):
        call("egovlp_divided_attn_bwd_det" if det else "egovlp_divided_attn_bwd", _ptr(qkv), _ptr(out), _ptr(dout),
             _ptr(lse), _ptr(dqkv), _ptr(ws), B, T, N, H, mode, C.c_float(q_scale), _stream())
    return dqkv


def _space_long_ws(B, T, N, H, device):
    n_ws = lib().egovlp_space_attn_long_workspace_floats(B, T, N, H)
    assert n_ws > 0, f"space_attn_long: unsupported geometry B={B} T={T} N={N} H={H}"
    return torch.empty(n_ws, dtype=F32, device=device)


def space_attn_long_fwd(qkv, B, T, N, H):
    """divided_attn_fwd(mode=1) for frames of up to 1024 patches, on the tiled kernel: qkv bf16 [B*S, 3*64*H]
    (q pre-scaled) -> (out bf16 [B*S, D], lse fp32 [B, H, S])."""
    _chk(qkv, BF16, "qkv")
    S, D = 1 + T * N, 64 * H
    assert qkv.is_contiguous() and qkv.shape == (B * S, 3 * D)
    out = torch.empty(B * S, D, dtype=BF16, device=qkv.device)
    lse = torch.empty(B, H, S, dtype=F32, device=qkv.device)
    ws = _space_long_ws(B, T, N, H, qkv.device)
    with _Probe("attn_space_long_fwd", B * S * (8 * D + 4 * H)):
        call("egovlp_space_attn_long_fwd", _ptr(qkv), _ptr(out), _ptr(lse), _ptr(ws), B, T, N, H, _stream())
    return out, lse


def space_attn_long_bwd(qkv, out, dout, lse, B, T, N, H, q_scale, dqkv=None):
    """Backward of space_attn_long_fwd (out / lse: its outputs) -> dqkv bf16 [B*S, 3*64*H]."""
    _chk(qkv, BF16, "qkv"); _chk(out, BF16, "out"); _chk(dout, BF16, "dout"); _chk(lse, F32, "lse")
    assert qkv.is_contiguous() and out.is_contiguous() and dout.is_contiguous() and lse.is_contiguous()
    if dqkv is None:
        dqkv = torch.empty_like(qkv)
    S, D = 1 + T * N, 64 * H
    ws = _space_long_ws(B, T, N, H, qkv.device)
    with _Probe("attn_space_long_bwd", B * S * (16 * D + 4 * H)):
        call("egovlp_space_attn_long_bwd", _ptr(qkv), _ptr(out), _ptr(dout), _ptr(lse), _ptr(dqkv), _ptr(ws), B, T,
             N, H, C.c_float(q_scale), _stream())
    return dqkv


# ---------------------------------------------------------------- video front end
def patch_im2col(video, patches, P):
    _chk(video, F32, "video")
    B, T, Cc, H, W = video.shape
    assert video.is_contiguous() and patches.dtype == BF16 and patches.is_contiguous()
    call("egovlp_patch_im2col", _ptr(video), _ptr(patches), B, T, Cc, H, W, P, _stream())


def patch_im2col_u8(video, patches, P, mean, std):
    assert video.is_cuda and video.dtype == torch.uint8 and video.is_contiguous()
    B, T, Cc, H, W = video.shape
    m3, s3 = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
    call("egovlp_patch_im2col_u8", _ptr(video), _ptr(patches), B, T, Cc, H, W, P, m3, s3, _stream())


def video_transform(frames, desc, F, R, center_crop, mean, std):
    """Dataset video transforms on the GPU (egovlp_video_transform): frames = packed uint8 clips on CUDA (clip b is
    [T, H, W, 3] at byte offset desc[b, 0]); desc = host int64 [B, 10] rows (offset, T, H, W, mode, i, j, h, w, flip),
    mode 0 = train (crop box + flip), 1 = eval.  Returns fp32 [B, F, 3, R, R]; frames t >= T are 0.0.  The table is
    checked here, before launch: a row the kernel would have to refuse raises EgovlpError."""
    import numpy as np
    from ._lib import EgovlpError
    _chk(frames, torch.uint8, "frames")
    assert frames.dim() == 1 and frames.is_contiguous()
    d = np.asarray(desc.numpy() if torch.is_tensor(desc) else desc)
    if d.ndim != 2 or d.shape[1] != 10 or d.shape[0] < 1 or d.dtype.kind not in "iu":
        raise EgovlpError(f"video_transform: descriptor table must be integer [B >= 1, 10], got {d.dtype} {d.shape}")
    d = d.astype(np.int64)
    off, T, H, W, mode, i, j, h, w, flip = d.T
    B = d.shape[0]
    bad = []
    def rows(mask, what):
        if mask.any():
            bad.append(f"{what} (clips {np.flatnonzero(mask)[:8].tolist()})")
    rows((H < 1) | (W < 1) | (H > 65535) | (W > 65535), "frame size outside [1, 65535]")
    rows((T < 1) | (T > F), f"frame count outside [1, F={F}]")
    rows((mode != 0) & (mode != 1), "mode not 0 (train) or 1 (eval)")
    ok = (H >= 1) & (W >= 1) & (H <= 65535) & (W <= 65535) & (T >= 1) & (T <= F)
    end = off + np.where(ok, T * H * W * 3, 0)
    rows(ok & ((off < 0) | (end > frames.numel())), f"clip outside the {frames.numel()}-byte frame buffer")
    tr = mode == 0
    rows(tr & ((h < 1) | (w < 1)), "crop box h or w < 1")
    rows(tr & ((i < 0) | (j < 0) | (i + h > H) | (j + w > W)), "crop box outside its frame")
    ev = (mode == 1) & ok
    if ev.any():
        # Source pixels one output index can weigh along an axis (bounded; see egovlp_video_transform_max_taps).
        shrt, lng = np.minimum(H, W), np.maximum(H, W)
        nlong = center_crop * lng // shrt
        d1 = [np.where(W <= H, nlong, center_crop), np.where(W <= H, center_crop, nlong)]
        sup2 = max(center_crop / R, 1.0)
        taps = 0
        for src, dst in zip((H, W), d1):
            sc1 = src / np.maximum(dst, 1)
            taps = np.maximum(taps, 2 * sc1 * sup2 + 2 * np.maximum(sc1, 1.0) + 2)
        rows(ev & (taps > lib().egovlp_video_transform_max_taps()),
             "source too large for the eval resize (short side above ~7 x center_crop)")
    if not 1 <= R <= lib().egovlp_video_transform_max_res() or center_crop < 1:
        bad.append(f"R = {R} outside [1, {lib().egovlp_video_transform_max_res()}] or center_crop = {center_crop} < 1")
    if bad:
        raise EgovlpError("video_transform: " + "; ".join(bad))
    desc_dev = torch.from_numpy(np.ascontiguousarray(d)).to(frames.device, non_blocking=True)
    out = torch.empty(B, F, 3, R, R, dtype=F32, device=frames.device)
    m = (C.c_float * 3)(*mean)
    s = (C.c_float * 3)(*std)
    call("egovlp_video_transform", _ptr(frames), C.c_longlong(frames.numel()), _ptr(desc_dev), B, F, R, center_crop,
         m, s, _ptr(out), _stream())
    return out


def video_pos_table(cls_token, pos_embed, temporal_embed, conv_bias, table, T, N, D):
    call("egovlp_video_pos_table", _ptr(cls_token), _ptr(pos_embed), _ptr(temporal_embed), _ptr(conv_bias),
         _ptr(table), T, N, D, _stream())


def video_embed_bwd(dx, tmp, dcls, dpos, dtemporal, dbias, B, T, N, D):
    if deterministic():
        ws = _det_ws(T * D, dx.device)
        call("egovlp_video_embed_bwd_det", _ptr(dx), _ptr(tmp), _ptr(dcls), _ptr(dpos), _ptr(dtemporal), _ptr(dbias),
             _ptr(ws), B, T, N, D, _stream())
        return
    call("egovlp_video_embed_bwd", _ptr(dx), _ptr(tmp), _ptr(dcls), _ptr(dpos), _ptr(dtemporal), _ptr(dbias), B, T, N,
         D, _stream())


# ---------------------------------------------------------------- text tower pieces
def text_embed_fwd(ids, word, pos, out, B, L, D):
    assert ids.dtype == torch.int64 and ids.is_contiguous()
    call("egovlp_text_embed_fwd", _ptr(ids), _ptr(word), _ptr(pos), _ptr(out), B, L, D, _stream())


def text_embed_bwd(ids, dsum, dword, dpos, B, L, D):
    if deterministic():
        # a stable sort groups each vocabulary row's tokens, in token order (int64 plumbing, deterministic in torch)
        sorted_ids, perm = torch.sort(ids.reshape(-1), stable=True)
        call("egovlp_text_embed_bwd_det", _ptr(sorted_ids), _ptr(perm), _ptr(dsum), _ptr(dword), _ptr(dpos), B, L, D,
             _stream())
        return
    call("egovlp_text_embed_bwd", _ptr(ids), _ptr(dsum), _ptr(dword), _ptr(dpos), B, L, D, _stream())


def text_attn_fwd(qkv, mask, out, B, L, H, p_drop=0.0, seed=0, site=0):
    assert mask.dtype == torch.int64 and mask.is_contiguous()
    call("egovlp_text_attn_fwd", _ptr(qkv), _ptr(mask), _ptr(out), B, L, H, C.c_float(p_drop), C.c_ulonglong(seed),
         C.c_uint(site), _stream())


def text_attn_bwd(qkv, mask, dout, dqkv, B, L, H, q_scale, p_drop=0.0, seed=0, site=0):
    call("egovlp_text_attn_bwd", _ptr(qkv), _ptr(mask), _ptr(dout), _ptr(dqkv), B, L, H, C.c_float(q_scale),
         C.c_float(p_drop), C.c_ulonglong(seed), C.c_uint(site), _stream())


def text_attn_long_fwd(qkv, mask, out, lse, B, L, H, p_drop=0.0, seed=0, site=0):
    """Tiled text attention (L <= 512): out bf16 [B*L, H*64], lse fp32 [B, H, L] (kept for the backward)."""
    assert mask.dtype == torch.int64 and mask.is_contiguous()
    _chk(lse, F32, "lse")
    assert lse.numel() >= B * H * L
    call("egovlp_text_attn_long_fwd", _ptr(qkv), _ptr(mask), _ptr(out), _ptr(lse), B, L, H, C.c_float(p_drop),
         C.c_ulonglong(seed), C.c_uint(site), _stream())


def text_attn_long_bwd(qkv, mask, out, lse, dout, dqkv, B, L, H, q_scale, p_drop=0.0, seed=0, site=0):
    """Backward of text_attn_long_fwd (out / lse: its outputs) -> dqkv bf16 [B*L, 3*H*64]."""
    assert mask.dtype == torch.int64 and mask.is_contiguous()
    ws = torch.empty(B * H * L, dtype=F32, device=qkv.device)     # delta_i = rowsum(dO * O)
    call("egovlp_text_attn_long_bwd", _ptr(qkv), _ptr(mask), _ptr(out), _ptr(lse), _ptr(dout), _ptr(dqkv), _ptr(ws),
         B, L, H, C.c_float(q_scale), C.c_float(p_drop), C.c_ulonglong(seed), C.c_uint(site), _stream())


def dropout(x, p, seed, site, add=None, y32=None, y16=None):
    """y = dropout_p(x) (+ add) with the (seed, site) Philox mask; returns (y32, y16) (whichever were given)."""
    _chk(x, F32, "x")
    assert x.is_contiguous() and (y32 is not None or y16 is not None)
    call("egovlp_dropout", _ptr(x), _ptr(add), _ptr(y32), _ptr(y16), C.c_longlong(x.numel()), C.c_float(p),
         C.c_ulonglong(seed), C.c_uint(site), _stream())
    return y32, y16


class Drop:
    """One dropout site of a [rows, W] tensor with an optional per-sample drop-path: element (r, c) is kept with the
    (seed, site) Philox mask of `egovlp_dropout` and scaled by 1 / (1 - p), times the drop-path factor of sample
    r // path_rows drawn at (seed, path_site) with rate path_p (path_rows = 0: none)."""
    __slots__ = ("p", "seed", "site", "path_p", "path_site", "path_rows")

    def __init__(self, p, seed, site, path_p=0.0, path_site=0, path_rows=0):
        self.p, self.seed, self.site = float(p), int(seed), int(site)
        self.path_p, self.path_site, self.path_rows = float(path_p), int(path_site), int(path_rows)


def drop_rows_bf16(x, drop, y=None):
    """y bf16 [rows, W] = x * keep / (1 - p) * drop-path factor of the row's sample: the gradient of a branch that a GEMM
    dropout form masked with `drop`.  x fp32 or bf16 [rows, W], contiguous."""
    assert x.dtype in (F32, BF16) and x.is_cuda and x.is_contiguous() and x.dim() == 2
    y = torch.empty(x.shape, dtype=BF16, device=x.device) if y is None else y
    _chk(y, BF16, "y")
    assert y.shape == x.shape and y.is_contiguous()
    call("egovlp_drop_rows_bf16", _ptr(x), int(x.dtype == BF16), _ptr(y), C.c_longlong(x.shape[0]), x.shape[1],
         C.c_float(drop.p), C.c_ulonglong(drop.seed), C.c_uint(drop.site), C.c_float(drop.path_p),
         C.c_uint(drop.path_site), drop.path_rows, _stream())
    return y


def dropout_mask(rows, width, p, seed, site, device="cuda"):
    """fp32 [rows, width] multipliers (0 or 1 / (1 - p)) of the (seed, site) element mask of a [rows, width] tensor: the
    mask of `dropout` and of the GEMM dropout forms."""
    ones = torch.ones(rows * width, dtype=F32, device=device)
    return dropout(ones, p, seed, site, y32=torch.empty_like(ones))[0].view(rows, width)


def drop_path_factors(n, p, seed, site, device="cuda"):
    """fp32 [n] per-sample drop-path factors (0 or 1 / (1 - p)) drawn at (seed, site)."""
    return dropout_mask(1, (n + 3) // 4 * 4, p, seed, site, device)[0, :n]


def relu_rows_fwd(x, row_stride, out, rows, D):
    call("egovlp_relu_rows_fwd", _ptr(x), C.c_longlong(row_stride), _ptr(out), rows, D, _stream())


def relu_rows_bwd(x, row_stride, dh, dx, rows, D):
    call("egovlp_relu_rows_bwd", _ptr(x), C.c_longlong(row_stride), _ptr(dh), _ptr(dx), rows, D, _stream())


def text_pooler_fwd(h, row_stride, w, b, y, relu16, B, D):
    """BERT pooler: y fp32 [B, D] = tanh(W h_CLS + b) from the CLS rows h[r * row_stride + :D]; relu16 (bf16 [B, D] or
    None) = relu(y)."""
    _chk(h, F32, "h"); _chk(w, F32, "w"); _chk(b, F32, "b"); _chk(y, F32, "y")
    if relu16 is not None:
        _chk(relu16, BF16, "relu16")
    call("egovlp_text_pooler_fwd", _ptr(h), C.c_longlong(row_stride), _ptr(w), _ptr(b), _ptr(y), _ptr(relu16), B, D,
         _stream())


def text_pooler_bwd(g, y, relu, h, row_stride, w, dw, db, dh, B, D):
    """Backward of text_pooler_fwd from the gradient at relu(y) (relu=True) or at y: writes dw, db and the CLS rows of dh."""
    for t, name in ((g, "g"), (y, "y"), (h, "h"), (w, "w"), (dw, "dw"), (db, "db"), (dh, "dh")):
        _chk(t, F32, name)
    call("egovlp_text_pooler_bwd", _ptr(g), _ptr(y), int(bool(relu)), _ptr(h), C.c_longlong(row_stride), _ptr(w),
         _ptr(dw), _ptr(db), _ptr(dh), B, D, _stream())


# ---------------------------------------------------------------- narrow projection heads (C % 32 != 0)
def narrow_linear_fwd(act16, w16, bias, out):
    """out fp32 [rows, C] = act16 [rows, K] @ w16 [C, K]^T + bias (fp32 [C])."""
    _chk(act16, BF16, "act16"); _chk(w16, BF16, "w16"); _chk(out, F32, "out")
    rows, K = act16.shape
    Cc = w16.shape[0]
    assert act16.is_contiguous() and w16.is_contiguous() and w16.shape == (Cc, K)
    assert out.is_contiguous() and out.shape == (rows, Cc)
    if bias is not None:
        _chk(bias, F32, "bias"); assert bias.is_contiguous() and bias.numel() == Cc
    call("egovlp_narrow_linear_fwd", _ptr(act16), _ptr(w16), _ptr(bias), _ptr(out), rows, Cc, K, _stream())
    return out


def narrow_linear_bwd(dout, d16, act16, w16):
    """-> (dW fp32 [C, K] = d16^T act16, db fp32 [C] = colsum(dout), d_act fp32 [rows, K] = d16 w16)."""
    _chk(dout, F32, "dout"); _chk(d16, BF16, "d16"); _chk(act16, BF16, "act16"); _chk(w16, BF16, "w16")
    rows, K = act16.shape
    Cc = w16.shape[0]
    for t in (dout, d16, act16, w16):
        assert t.is_contiguous()
    assert dout.shape == (rows, Cc) and d16.shape == (rows, Cc) and w16.shape == (Cc, K)
    dev = act16.device
    dw = torch.empty(Cc, K, dtype=F32, device=dev)
    db = torch.empty(Cc, dtype=F32, device=dev)
    dact = torch.empty(rows, K, dtype=F32, device=dev)
    n_ws = lib().egovlp_narrow_linear_workspace_floats(rows, Cc, K)
    ws = torch.empty(n_ws, dtype=F32, device=dev) if n_ws > 0 else None
    call("egovlp_narrow_linear_bwd", _ptr(dout), _ptr(d16), _ptr(act16), _ptr(w16), _ptr(dw), _ptr(db), _ptr(dact),
         _ptr(ws), rows, Cc, K, _stream())
    return dw, db, dact


# ---------------------------------------------------------------- similarity / losses (fp32)
def rownorm_fwd(a, eps=1e-8):
    _chk(a, F32, "a")
    a = a.contiguous()
    an, norm = torch.empty_like(a), torch.empty(a.shape[0], dtype=F32, device=a.device)
    call("egovlp_rownorm_fwd", _ptr(a), _ptr(an), _ptr(norm), a.shape[0], a.shape[1], C.c_float(eps), _stream())
    return an, norm


def rownorm_bwd(dan, an, norm, eps=1e-8):
    da = torch.empty_like(an)
    call("egovlp_rownorm_bwd", _ptr(dan.contiguous()), _ptr(an), _ptr(norm), _ptr(da), an.shape[0], an.shape[1],
         C.c_float(eps), _stream())
    return da


def sgemm(a, b, *, trans_a=False, trans_b=True, out=None, alpha=1.0, beta=0.0):
    """fp32 C = op(a) @ op(b)^T-style product on CUDA cores.  Default: a[M,K] @ b[N,K]^T.
    trans_a: a is [K,M]; trans_b=False: b is [K,N]."""
    _chk(a, F32, "a"); _chk(b, F32, "b")
    M, K = (a.shape[1], a.shape[0]) if trans_a else a.shape
    N = b.shape[0] if trans_b else b.shape[1]
    sam, sak = (a.stride(1), a.stride(0)) if trans_a else (a.stride(0), a.stride(1))
    sbn, sbk = (b.stride(0), b.stride(1)) if trans_b else (b.stride(1), b.stride(0))
    if out is None:
        out = torch.empty(M, N, dtype=F32, device=a.device)
    call("egovlp_sgemm_f32", _ptr(a), C.c_longlong(sam), C.c_longlong(sak), _ptr(b), C.c_longlong(sbn),
         C.c_longlong(sbk), _ptr(out), C.c_longlong(out.stride(0)), M, N, K, C.c_float(alpha), C.c_float(beta), _stream())
    return out


def positives_mask_from_tags(verb, noun, mode):
    """uint8 [G,G] positives mask (diag | shared verb & shared noun) from multi-hot vectors."""
    G = (verb if verb is not None else noun).shape[0]
    dev = (verb if verb is not None else noun).device
    mask = torch.empty(G, G, dtype=torch.uint8, device=dev)
    vb = nb = None
    nv = nn_ = 0
    if verb is not None:
        nv = verb.shape[1]
        vb = torch.empty(G, (nv + 31) // 32, dtype=torch.int32, device=dev)
        call("egovlp_pack_multihot", _ptr(verb.contiguous().float()), _ptr(vb), G, nv, _stream())
    if noun is not None:
        nn_ = noun.shape[1]
        nb = torch.empty(G, (nn_ + 31) // 32, dtype=torch.int32, device=dev)
        call("egovlp_pack_multihot", _ptr(noun.contiguous().float()), _ptr(nb), G, nn_, _stream())
    call("egovlp_mask_from_bits", _ptr(vb), nv, _ptr(nb), nn_, _ptr(mask), G, mode, _stream())
    return mask


def positives_mask_from_sims(sim_v, sim_n, G, mode, device=None):
    """uint8 [G,G] positives mask; mode 0 (identity) needs `device` since it has no input tensor to take it from."""
    src = sim_v if sim_v is not None else sim_n
    dev = src.device if src is not None else torch.device(device)
    assert dev.type == "cuda", f"positives mask: CUDA tensors expected, got {dev} (there is no CPU path)"
    mask = torch.empty(G, G, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        call("egovlp_mask_from_sims", _ptr(sim_v), _ptr(sim_n), _ptr(mask), G, mode, _stream())
    return mask


def nce_fwd(x, mask, inv_temp):
    _chk(x, F32, "x")
    G = x.shape[0]
    assert x.shape == (G, G) and x.is_contiguous() and mask.shape == (G, G)
    stats = torch.empty(4 * G, dtype=F32, device=x.device)
    loss = torch.empty((), dtype=F32, device=x.device)
    call("egovlp_nce_fwd", _ptr(x), _ptr(mask), G, C.c_float(inv_temp), _ptr(stats), _ptr(loss), _stream())
    return loss, stats


def nce_bwd(x, mask, stats, inv_temp, gscale):
    dx = torch.empty_like(x)
    call("egovlp_nce_bwd", _ptr(x), _ptr(mask), _ptr(stats), x.shape[0], C.c_float(inv_temp), _ptr(gscale), _ptr(dx),
         _stream())
    return dx


def pack_rows4(a, b, c, d):
    """[a | b | c | d] along dim 1 (fp32, row-major) in one launch: the send buffer of the packed all-gather."""
    for t in (a, b, c, d):
        _chk(t, F32, "pack_rows4 input"); assert t.dim() == 2 and t.is_contiguous() and t.shape[0] == a.shape[0]
    out = torch.empty(a.shape[0], a.shape[1] + b.shape[1] + c.shape[1] + d.shape[1], dtype=F32, device=a.device)
    call("egovlp_pack_rows4", _ptr(a), a.shape[1], _ptr(b), b.shape[1], _ptr(c), c.shape[1], _ptr(d), d.shape[1], _ptr(out),
         a.shape[0], _stream())
    return out


_fused_ws = {}


def egonce_fused_supported(G, C, n_verb=0, n_noun=0, mode=0):
    """Whether the fused EgoNCE kernel takes G rows of width C with these tag widths (those `mode` uses)."""
    return bool(lib().egovlp_egonce_fused_supported(G, C, n_verb, n_noun, mode))


def _rows_view(t, name):
    _chk(t, F32, name)
    assert t.dim() == 2 and t.stride(1) == 1, f"{name}: rows with unit inner stride expected"
    return t


def egonce_fused_fwd(text, video, verb, noun, inv_temp, mode, eps=1e-8):
    """ONE kernel: normalise rows -> cosine similarities (smem only) -> positives from tag bits -> masked LSEs -> loss.
    text / video [G, C], verb [G, nv] / noun [G, nn] (or None per `mode`): row-strided fp32 views, read in place.
    -> (loss, saved = (norm_text, norm_video, tag_bits, stats))."""
    text, video = _rows_view(text, "text"), _rows_view(video, "video")
    G, Cc = text.shape
    assert video.shape == (G, Cc)
    nv = verb.shape[1] if verb is not None else 0
    nn_ = noun.shape[1] if noun is not None else 0
    if verb is not None: _rows_view(verb, "verb")
    if noun is not None: _rows_view(noun, "noun")
    dev = text.device
    na, nb = torch.empty(G, dtype=F32, device=dev), torch.empty(G, dtype=F32, device=dev)
    bits = torch.empty(G, max(1, (nv + 31) // 32 + (nn_ + 31) // 32), dtype=torch.int32, device=dev)
    stats = torch.empty(4 * G, dtype=F32, device=dev)
    loss = torch.empty((), dtype=F32, device=dev)
    key = (dev.index, G)
    ws = _fused_ws.get(key)
    if ws is None:                      # zero once: the kernel leaves its ticket word zero after every launch
        ws = _fused_ws[key] = torch.zeros(lib().egovlp_egonce_fused_workspace_floats(G), dtype=F32, device=dev)
    call("egovlp_egonce_fused_fwd", _ptr(text), C.c_longlong(text.stride(0)), _ptr(video), C.c_longlong(video.stride(0)),
         _ptr(verb), C.c_longlong(verb.stride(0) if verb is not None else 0), nv, _ptr(noun),
         C.c_longlong(noun.stride(0) if noun is not None else 0), nn_, G, Cc, C.c_float(inv_temp), int(mode), C.c_float(eps),
         _ptr(na), _ptr(nb), _ptr(bits), _ptr(stats), _ptr(ws), _ptr(loss), _stream())
    return loss, (na, nb, bits, stats)


def egonce_fused_bwd(text, video, saved, n_verb, n_noun, inv_temp, mode, gscale, row0, n_local, eps=1e-8):
    """-> (d_text, d_video) [n_local, C] of rows [row0, row0 + n_local) only."""
    na, nb, bits, stats = saved
    G, Cc = text.shape
    d_text = torch.empty(n_local, Cc, dtype=F32, device=text.device)
    d_video = torch.empty(n_local, Cc, dtype=F32, device=text.device)
    call("egovlp_egonce_fused_bwd", _ptr(text), C.c_longlong(text.stride(0)), _ptr(video), C.c_longlong(video.stride(0)),
         _ptr(na), _ptr(nb), _ptr(bits), n_verb, n_noun, _ptr(stats), G, Cc, C.c_float(inv_temp), int(mode), C.c_float(eps),
         _ptr(gscale), row0, n_local, _ptr(d_text), _ptr(d_video), _stream())
    return d_text, d_video


def maxmargin_fwd(x, margin, fix_norm, row_weight=None):
    _chk(x, F32, "x")
    if row_weight is not None:
        _chk(row_weight, F32, "row_weight")
        assert row_weight.shape == (x.shape[0],) and row_weight.is_contiguous()
    loss = torch.empty((), dtype=F32, device=x.device)
    if deterministic():
        ws = _det_ws(lib().egovlp_maxmargin_det_workspace_floats(x.shape[0]), x.device)
        call("egovlp_maxmargin_fwd_det", _ptr(x), _ptr(row_weight), x.shape[0], C.c_float(margin), int(fix_norm),
             _ptr(loss), _ptr(ws), _stream())
        return loss
    call("egovlp_maxmargin_fwd", _ptr(x), _ptr(row_weight), x.shape[0], C.c_float(margin), int(fix_norm), _ptr(loss),
         _stream())
    return loss


def maxmargin_bwd(x, margin, fix_norm, gscale, row_weight=None):
    dx = torch.empty_like(x)
    call("egovlp_maxmargin_bwd_det" if deterministic() else "egovlp_maxmargin_bwd", _ptr(x), _ptr(row_weight), x.shape[0], C.c_float(margin), int(fix_norm), _ptr(gscale),
         _ptr(dx), _stream())
    return dx


def cross_entropy_fwd(x, target, ignore_index=-100):
    """x fp32 [G, C] (row stride free), target int64 [G] -> (loss fp32 scalar, lse fp32 [G], stats fp32 [2] =
    (loss, n_valid))."""
    x = _rows_view(x, "logits")
    assert target.is_cuda and target.dtype == torch.int64 and target.is_contiguous() and target.shape == (x.shape[0],)
    G, Cc = x.shape
    lse = torch.empty(G, dtype=F32, device=x.device)
    row_loss = torch.empty(G, dtype=F32, device=x.device)
    stats = torch.empty(2, dtype=F32, device=x.device)
    call("egovlp_cross_entropy_fwd", _ptr(x), C.c_longlong(x.stride(0) if G > 0 else Cc), _ptr(target), G, Cc,
         int(ignore_index), _ptr(lse), _ptr(row_loss), _ptr(stats), _stream())
    return stats[0], lse, stats


def cross_entropy_bwd(x, target, lse, stats, gscale, ignore_index=-100):
    """-> dx fp32 [G, C] = gscale * (softmax(x) - onehot(target)) / n_valid (0 on ignored rows)."""
    G, Cc = x.shape
    dx = torch.empty(G, Cc, dtype=F32, device=x.device)
    call("egovlp_cross_entropy_bwd", _ptr(x), C.c_longlong(x.stride(0) if G > 0 else Cc), _ptr(target), _ptr(lse),
         _ptr(stats), G, Cc, int(ignore_index), _ptr(gscale), _ptr(dx), _stream())
    return dx


def rank_metrics(sim, rel, k_counts=None, tie_mode=0, want_dcg=True, want_ap=True):
    """Per-query ranking metrics (egovlp_rank_metrics): sim fp32 [R, C], rel fp32/fp64 [R, C], optional int32
    k_counts [R, C] -> (dcg fp64 [R] | None, ap fp64 [R] | None)."""
    _chk(sim, F32, "sim")
    assert rel.is_cuda and rel.dtype in (torch.float32, torch.float64) and rel.shape == sim.shape and sim.dim() == 2
    sim, rel = sim.contiguous(), rel.contiguous()
    R, Cc = sim.shape
    if k_counts is not None:
        assert k_counts.is_cuda and k_counts.shape == sim.shape
        k_counts = k_counts.to(torch.int32).contiguous()
    dcg = torch.empty(R, dtype=torch.float64, device=sim.device) if want_dcg else None
    ap = torch.empty(R, dtype=torch.float64, device=sim.device) if want_ap else None
    if R == 0:
        return dcg, ap
    call("egovlp_rank_metrics", _ptr(sim), C.c_longlong(sim.stride(0)), _ptr(rel), int(rel.dtype == torch.float64),
         C.c_longlong(rel.stride(0)), _ptr(k_counts), R, Cc, int(tie_mode), _ptr(dcg), _ptr(ap), _stream())
    return dcg, ap


def gt_ranks(sims, mode, col_mask=None):
    """Ground-truth ranks (egovlp_gt_ranks): sims fp32/fp64 [rows, cols] on CUDA -> fp64 [rows], 0-based.  mode 0 (t2v):
    [queries, videos], ties optimistic; mode 1 (v2t): [videos, captions], ties averaged, min over each video's captions,
    col_mask [captions] (0 = missing caption).  Synchronises; raises EgovlpError on a NaN row or an invalid shape."""
    assert sims.is_cuda and sims.dtype in (torch.float32, torch.float64) and sims.dim() == 2
    sims = sims if sims.stride(1) == 1 else sims.contiguous()
    rows, cols = sims.shape
    if col_mask is not None:
        assert mode == 1 and col_mask.numel() == cols
        col_mask = col_mask.reshape(-1).to(device=sims.device, dtype=torch.uint8).contiguous()
    ranks = torch.empty(rows, dtype=torch.float64, device=sims.device)
    status = torch.empty(1, dtype=torch.int32, device=sims.device)
    call("egovlp_gt_ranks", _ptr(sims), int(sims.dtype == torch.float64), C.c_longlong(sims.stride(0)), rows, cols,
         int(mode), _ptr(col_mask), _ptr(ranks), _ptr(status), _stream())
    return ranks


def dual_softmax(sim, temp=500.0):
    _chk(sim, F32, "sim")
    sim = sim.contiguous()
    out = torch.empty_like(sim)
    call("egovlp_dual_softmax", _ptr(sim), _ptr(out), sim.shape[0], sim.shape[1], C.c_float(temp), _stream())
    return out


def egomcq_score(text, video, eps=1e-8):
    _chk(text, F32, "text"); _chk(video, F32, "video")
    Q, K, Cc = video.shape
    scores = torch.empty(Q, K, dtype=F32, device=text.device)
    pred = torch.empty(Q, dtype=torch.int64, device=text.device)
    call("egovlp_egomcq_score", _ptr(text.contiguous()), _ptr(video.contiguous()), _ptr(scores), _ptr(pred), Q, K, Cc,
         C.c_float(eps), _stream())
    return scores, pred
