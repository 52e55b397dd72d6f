"""fp64 reference and GPU harness of the divided space-time attention tests (test_divided_attention_gpu.py, which
derives the bounds used here, and test_kernels_gpu.py::test_divided_attention_fwd_bwd)."""
import torch
from kernel_checks import BF16, F32, F64, assert_elementwise_bound, nan_filled

U = 2.0 ** -8        # bf16 unit roundoff
SLACK = 1.25         # fp32 accumulation
Q_SCALE = 0.125      # engine.Q_SCALE: head_dim ** -0.5
SENTINEL_ROWS = 3
SENTINEL = -3.0

# path -> environment.  "default": the dispatch the engine uses; "generic": the group-id kernels for every geometry;
# "tc": + the wgmma space-attention forward (128 < N + 1 <= 208); "w8": the 8-warp time backward.
PATH_ENV = {
    "default": {"EGOVLP_ATTN_GENERIC": "0", "EGOVLP_ATTN_TC": "0", "EGOVLP_ATTN_TIME_BWD_WARPS": "4"},
    "generic": {"EGOVLP_ATTN_GENERIC": "1", "EGOVLP_ATTN_TC": "0", "EGOVLP_ATTN_TIME_BWD_WARPS": "4"},
    "tc": {"EGOVLP_ATTN_GENERIC": "0", "EGOVLP_ATTN_TC": "1", "EGOVLP_ATTN_TIME_BWD_WARPS": "4"},
    "w8": {"EGOVLP_ATTN_GENERIC": "0", "EGOVLP_ATTN_TC": "0", "EGOVLP_ATTN_TIME_BWD_WARPS": "8"},
}


def time_fast(T, N):
    """The specialised time kernels: T in {4, 8, 16} with full 112-row groups (112 / T patches, so N >= 112 / T)."""
    return T in (4, 8, 16) and N >= 112 // T


def paths_for(T, N, mode):
    """Every path the geometry admits, each once (a time geometry off the fast path is already generic by default)."""
    paths = ["default"]
    if mode == 1 or time_fast(T, N):
        paths.append("generic")
    if mode == 1 and 128 < N + 1 <= 208:
        paths.append("tc")
    if mode == 0 and time_fast(T, N):
        paths.append("w8")
    return paths


# ---------------------------------------------------------------------------------------------------------- reference
def _group_core(q, k, v, do, q_scale):
    """Softmax attention of queries q [..., M, 64] over keys k / values v [..., K, 64], upstream gradient do, in the
    dtype given (float64): out, lse, the analytic backward and the magnitude sums of the bounds."""
    s = q @ k.transpose(-1, -2)
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    o = p @ v
    pv = p @ v.abs()                                               # sum_j P_ij |v_jd|
    dp = do @ v.transpose(-1, -2)
    delta = (do * o).sum(-1, keepdim=True)
    ds = p * (dp - delta)
    e = (do.abs() * (pv + 2 * o.abs())).sum(-1, keepdim=True)     # E_i
    w = p * ((dp - delta).abs() + e)
    pt = p.transpose(-1, -2)
    return {"out": o, "lse": lse, "out_t": pv, "lse_t": (q.abs() @ k.abs().transpose(-1, -2)).amax(-1),
            "dq": q_scale * (ds @ k), "dq_t": q_scale * (w @ k.abs()),
            "dk": ds.transpose(-1, -2) @ q, "dk_t": w.transpose(-1, -2) @ q.abs(),
            "dv": pt @ do, "dv_t": pt @ do.abs()}


def reference(qkv, dout, B, T, N, H, mode, q_scale):
    """float64 divided attention of qkv [B*S, 3*D] (q as stored) with upstream gradient dout [B*S, D], per group.
    Returns out, dq, dk, dv [B*S, D], lse [B, H, S] and, under the same names + "_t", the sums the bounds use."""
    S, D = 1 + T * N, 64 * H
    x = qkv.to(F64).view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)          # [3, B, H, S, 64]
    q, k, v = x[0], x[1], x[2]
    do = dout.to(F64).view(B, S, H, 64).permute(0, 2, 1, 3)

    def group(t):          # patch rows [B, H, S, 64] -> [B, H, groups, members, 64]
        t = t[:, :, 1:].reshape(B, H, T, N, 64)
        return t.transpose(2, 3) if mode == 0 else t

    def ungroup(t):        # the inverse, -> [B, H, S - 1, 64]
        return (t.transpose(2, 3) if mode == 0 else t).reshape(B, H, T * N, 64)

    ng = N if mode == 0 else T
    kc = k[:, :, None, :1].expand(B, H, ng, 1, 64)
    vc = v[:, :, None, :1].expand(B, H, ng, 1, 64)
    grp = _group_core(group(q), torch.cat([kc, group(k)], 3), torch.cat([vc, group(v)], 3), group(do), q_scale)
    cls = _group_core(q[:, :, :1], k, v, do[:, :, :1], q_scale)          # the CLS query over all S keys

    res = {}
    for name in ("out", "out_t", "dq", "dq_t"):                            # per query row
        t = torch.cat([cls[name], ungroup(grp[name])], 2)
        res[name] = t.permute(0, 2, 1, 3).reshape(B * S, D)
    for name in ("lse", "lse_t"):
        lg = grp[name].transpose(2, 3) if mode == 0 else grp[name]
        res[name] = torch.cat([cls[name], lg.reshape(B, H, T * N)], 2)
    for name in ("dk", "dk_t", "dv", "dv_t"):                              # per key row: summed over every query
        t = cls[name].clone()
        t[:, :, :1] += grp[name][:, :, :, :1].sum(2)
        t[:, :, 1:] += ungroup(grp[name][:, :, :, 1:])
        res[name] = t.permute(0, 2, 1, 3).reshape(B * S, D)
    return res


def make_inputs(B, T, N, H, seed, q_scale=Q_SCALE, device="cuda"):
    """qkv [B*S, 3*D] bf16 with q pre-scaled by q_scale (as the QKV GEMM's epilogue does), dout [B*S, D] bf16.
    Scores q.k have a standard deviation of 8 q_scale (1 at the engine's scale)."""
    S, D = 1 + T * N, 64 * H
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(B * S, 3 * D, generator=g, device=device)
    x[:, :D] *= q_scale
    dout = torch.randn(B * S, D, generator=g, device=device)
    return x.to(BF16), dout.to(BF16)


def plant_maxima(qkv, B, T, N, H, mode, score=18.0):
    """Sharp scores: point chosen query rows at one key each, so that key's score is `score` above the others.
      * every 5th patch row (per group member index) at the CLS key;
      * every 3rd other patch row at the last member of its own attention group (the last valid key of the kernels'
        group: the last key chunk);
      * the CLS query at the last patch token, in the last frame (space) / the last, partly filled group (time)."""
    S, D = 1 + T * N, 64 * H
    x = qkv.float().view(B, S, 3, H, 64)
    tok = torch.arange(1, S, device=qkv.device)
    f, n = (tok - 1) // N, (tok - 1) % N
    member = n if mode == 1 else f                   # index within the attention group
    last = 1 + (f * N + N - 1 if mode == 1 else (T - 1) * N + n)
    to_cls = member % 5 == 0
    to_last = ~to_cls & (member % 3 == 1)

    def aim(rows, keys):
        kk = x[:, keys, 1]                               # [B, rows, H, 64]
        x[:, rows, 0] = kk * (score / kk.pow(2).sum(-1, keepdim=True))

    aim(tok[to_cls], torch.zeros_like(tok[to_cls]))
    aim(tok[to_last], last[to_last])
    aim(torch.tensor([0], device=qkv.device), torch.tensor([S - 1], device=qkv.device))
    return x.reshape(B * S, 3 * D).to(BF16)



def set_path(monkeypatch, path):
    for k, v in PATH_ENV[path].items():
        monkeypatch.setenv(k, v)


def _with_sentinels(shape_rows, cols, dtype):
    """NaN-filled [rows + SENTINEL_ROWS, cols] buffer whose last SENTINEL_ROWS rows hold SENTINEL."""
    buf = nan_filled((shape_rows + SENTINEL_ROWS, cols), dtype)
    buf[shape_rows:] = SENTINEL
    return buf


def run_attention(ops, qkv, dout, B, T, N, H, mode, q_scale):
    """Forward through the C entry point into caller-owned buffers, then the backward into a dqkv= view; returns
    (out [B*S, D], lse [B, H, S], dqkv [B*S, 3*D]) after checking that every element was written and no sentinel
    changed."""
    from egovlp_b200._lib import lib
    S, D = 1 + T * N, 64 * H
    M = B * S
    out_buf = _with_sentinels(M, D, BF16)
    lse_buf = _with_sentinels(B * H, S, F32)
    ws = torch.empty(lib().egovlp_divided_attn_workspace_floats(B, T, N, H, mode), dtype=F32, device="cuda")
    ops.call("egovlp_divided_attn_fwd", ops._ptr(qkv), ops._ptr(out_buf), ops._ptr(lse_buf), ops._ptr(ws), B, T, N, H,
             mode, ops._stream())
    out, lse = out_buf[:M], lse_buf[:B * H].view(B, H, S)
    dq_buf = _with_sentinels(M, 3 * D, BF16)
    ops.divided_attn_bwd(qkv, out, dout, lse, B, T, N, H, mode, q_scale, dqkv=dq_buf[:M])
    torch.cuda.synchronize()
    for name, buf, rows in (("out", out_buf, M), ("lse", lse_buf, B * H), ("dqkv", dq_buf, M)):
        assert not buf[:rows].isnan().any(), f"{name}: {int(buf[:rows].isnan().sum())} elements left unwritten"
        assert bool((buf[rows:] == SENTINEL).all()), f"{name}: a row past the output was written"
    return out, lse, dq_buf[:M]


def check_against_reference(tag, qkv, dout, out, lse, dqkv, B, T, N, H, mode, q_scale):
    """Every element of out, lse and dq | dk | dv within its bound; returns the reference."""
    D = 64 * H
    r = reference(qkv, dout, B, T, N, H, mode, q_scale)
    assert_elementwise_bound(f"out {tag}", out, r["out"], SLACK * U * (r["out_t"] + 2 * r["out"].abs()))
    assert_elementwise_bound(f"lse {tag}", lse, r["lse"], SLACK * (2e-5 * r["lse_t"] + 1e-6 * (1 + r["lse"].abs())))
    for i, name in enumerate(("dq", "dk", "dv")):
        got = dqkv[:, i * D:(i + 1) * D]
        assert_elementwise_bound(f"{name} {tag}", got, r[name], SLACK * U * (r[name + "_t"] + r[name].abs()))
    return r


def check_case(ops, monkeypatch, B, T, N, H, mode, path, seed, q_scale=Q_SCALE, sharp=False):
    """Run one case on one path and hold every output to its bound; returns (out, dqkv, reference)."""
    set_path(monkeypatch, path)
    qkv, dout = make_inputs(B, T, N, H, seed, q_scale)
    if sharp:
        qkv = plant_maxima(qkv, B, T, N, H, mode)
    out, lse, dqkv = run_attention(ops, qkv, dout, B, T, N, H, mode, q_scale)
    tag = f"{'space' if mode else 'time'} B={B} T={T} N={N} H={H} {path}" + (" sharp" if sharp else "")
    return out, dqkv, check_against_reference(tag, qkv, dout, out, lse, dqkv, B, T, N, H, mode, q_scale)
