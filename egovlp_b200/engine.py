"""Host-side step engine: torch.autograd.Function wrappers that sequence the CUDA kernels of the hot path.

torch supplies device buffers, the current stream and the autograd graph (so DDP / optimizers of the unchanged
reference trainer keep working); every FLOP below runs in libegovlp_b200.so through `ops`.

Numerics layout: residual stream and LayerNorm statistics in fp32, GEMM operands in bf16 (fp32 accumulation in
wgmma registers), attention probabilities never leave the SM, losses in fp32.  fp32 master parameters are the autograd
leaves; their bf16 GEMM copies come from `Bf16Cache` (refreshed when a parameter's version changes).
"""
import functools
import os
import threading
import weakref

import torch

from . import ops
from ._lib import EgovlpError

BF16, F32 = torch.bfloat16, torch.float32
Q_SCALE = 0.125            # head_dim ** -0.5 for head_dim = 64 (model/video_transformer.py:87)


def _empty(shape, dtype, like):
    return torch.empty(shape, dtype=dtype, device=like.device)


class _ZeroArena:
    """One zero-filled fp32 buffer per block backward, carved into the ~20 accumulators (split-K weight gradients, bias /
    LayerNorm gradient vectors) that each used to cost a fill launch of its own.  Views keep the buffer alive."""

    def __init__(self, n_floats, like):
        self.buf = torch.zeros(n_floats, dtype=F32, device=like.device)
        self.off = 0

    def take(self, shape):
        n = 1
        for d in shape:
            n *= int(d)
        if self.off + n > self.buf.numel():
            return None
        v = self.buf[self.off:self.off + n].view(shape)
        self.off += (n + 63) // 64 * 64                     # 256-byte aligned carve-outs
        return v


_tls = threading.local()        # per autograd thread (= per device): the arena of the block backward in progress


def _zeros(shape, like):
    arena = getattr(_tls, "arena", None)
    if arena is not None and arena.buf.device == like.device:
        v = arena.take(shape)
        if v is not None:
            return v
    return torch.zeros(shape, dtype=F32, device=like.device)


# Generation counter of "some optimizer stepped": bumped by a global torch.optim post-step hook, so that bf16 copies
# are rebuilt even when the optimizer wrote through `p.data` (transformers.AdamW 4.x, apex), which does not bump
# `p._version`.  The fused egovlp_b200.optim.AdamW rewrites the copies itself (same kernel pass) and is exempt, so that
# `get()` right after its step (an evaluation forward) casts nothing; `refresh()` in a training forward re-casts anyway.
_GEN = 0


def _on_optimizer_step(optimizer, args, kwargs):
    global _GEN
    if not getattr(optimizer, "_egovlp_fused", False):
        _GEN += 1


try:                                                          # torch >= 2.0
    from torch.optim.optimizer import register_optimizer_step_post_hook as _reg_hook
    _reg_hook(_on_optimizer_step)
except ImportError:                                           # pragma: no cover
    pass


class _CastEntry:
    __slots__ = ("ref", "t16", "version", "ptr", "gen", "scale")

    def __init__(self, p, t16, scale=None):
        self.ref, self.t16, self.scale = weakref.ref(p), t16, scale         # scale: e4m3 entries only
        self.version, self.ptr, self.gen = -1, 0, -1

    def stamp(self, p):
        self.version, self.ptr, self.gen = p._version, p.data_ptr(), _GEN

    def current(self, p):
        return (self.ref() is p and self.version == p._version and self.ptr == p.data_ptr() and self.gen == _GEN
                and self.t16.device == p.device)


_SHADOWS = {}          # id(param) -> _CastEntry: lets the fused AdamW write the bf16 copy in its own pass


def _prune_shadows():
    """Drop the entries of parameters that no longer exist, so that a dead model's bf16 copies are freed with it instead
    of staying referenced here until the process ends (a process that builds several models in turn, such as the test
    suite, would otherwise keep every one's copies on the device)."""
    for key in [k for k, e in _SHADOWS.items() if e.ref() is None]:
        del _SHADOWS[key]


def shadow_entry(p):
    ent = _SHADOWS.get(id(p))
    return ent if ent is not None and ent.ref() is p and ent.t16.device == p.device else None


class Bf16Cache:
    """bf16 GEMM-operand copies of the fp32 master parameters.

    * `get(p)` returns the copy, re-casting when the parameter object, its storage, its version or the global
      optimizer generation changed (entries hold a weak reference, so a recycled `id()` cannot alias a dead parameter).
    * `refresh()` -- called at the top of every TRAINING forward -- re-casts every known copy in ONE launch
      (egovlp_cast_multi_f32_to_bf16), so an update made through `p.data` by any optimizer / EMA is always seen by the
      next training step.  That includes copies the fused AdamW has just written: a write through `p.data` after its
      step leaves no trace (`p._version` stays put), so no copy can be trusted to be current at that point.
    * `get_e4m3(p)` returns (e4m3 [N, K], fp32 [N] per-row scales) of a 2-D weight for the fp8 inference GEMMs, under the
      same invalidation rules; `refresh()` marks those entries stale, so they are re-quantised by the next fp8 forward."""

    def __init__(self):
        self._store = {}
        self._cats = {}
        self._table = None
        self._e4m3 = {}

    def _entry(self, p, t16_factory):
        ent = self._store.get(id(p))
        if ent is None or ent.ref() is not p or ent.t16.device != p.device:
            ent = _CastEntry(p, t16_factory())
            self._store[id(p)] = ent
            _prune_shadows()
            _SHADOWS[id(p)] = ent
            self._table = None
        if not ent.current(p):
            ops.cast_bf16(p.detach().contiguous(), ent.t16)
            ent.stamp(p)
        return ent

    def get(self, p, shape=None):
        t = self._entry(p, lambda: torch.empty(p.shape, dtype=BF16, device=p.device)).t16
        return t.view(shape) if shape is not None else t

    def get_e4m3(self, p):
        ent = self._e4m3.get(id(p))
        if ent is None or ent.ref() is not p or ent.t16.device != p.device:
            ent = _CastEntry(p, torch.empty(p.shape, dtype=ops.E4M3, device=p.device),
                             torch.empty(p.shape[0], dtype=F32, device=p.device))
            self._e4m3[id(p)] = ent
        if not ent.current(p):
            ops.quantize_rows_e4m3(p.detach().contiguous(), ent.t16, ent.scale)
            ent.stamp(p)
        return ent.t16, ent.scale

    def cat(self, name, params):
        """bf16 concat along dim 0 of several parameters (DistilBERT q/k/v -> one [3D, D] operand): every part is a cache
        entry whose copy is a slice of one buffer, so `refresh()` keeps the concatenation current too."""
        buf = self._cats.get(name)
        rows = sum(p.shape[0] for p in params)
        if buf is None or buf.device != params[0].device or buf.shape[0] != rows:
            buf = torch.empty((rows,) + tuple(params[0].shape[1:]), dtype=BF16, device=params[0].device)
            self._cats[name] = buf
            for p in params:
                self._store.pop(id(p), None)
        r = 0
        for p in params:
            sl = buf[r:r + p.shape[0]]
            self._entry(p, lambda sl=sl: sl)
            r += p.shape[0]
        return buf

    def refresh(self):
        """Bring every cached copy up to date with one multi-tensor cast."""
        for key, ent in list(self._e4m3.items()):
            if ent.ref() is None:
                del self._e4m3[key]
            else:
                ent.version = -1
        live = []
        for key, ent in list(self._store.items()):
            p = ent.ref()
            if p is None or ent.t16.device != p.device:
                del self._store[key]
                if _SHADOWS.get(key) is ent:
                    del _SHADOWS[key]
                self._table = None
                continue
            live.append((p, ent))
        if not live:
            return
        key = tuple((p.data_ptr(), ent.t16.data_ptr(), p.numel()) for p, ent in live)
        if self._table is None or self._table[0] != key:
            self._table = (key,) + ops.build_cast_table([(p.detach(), ent.t16) for p, ent in live])
        ops.cast_multi(*self._table[1:])
        for p, ent in live:
            ent.stamp(p)

    def clear(self):
        for key, ent in self._store.items():
            if _SHADOWS.get(key) is ent:
                del _SHADOWS[key]
        self._store.clear()
        self._cats.clear()
        self._e4m3.clear()
        self._table = None


# By-products of an fp32 gradient tensor handed between consecutive Functions: its bf16 twin (saves one cast pass per
# block) and its column sums (the next block's fc2 bias gradient; saves one read of the tensor per block).  An entry
# holds the fp32 tensor itself, so its storage cannot be recycled for another tensor while the entry exists, and the
# tensor's version, so a gradient that autograd accumulated into in place (a block output with two consumers) is
# recognised and simply recomputed.  One slot per device; cleared when a video forward / backward starts.
_twin = {}
_twin_lock = threading.Lock()


def _publish_twin(t32, t16, colsum=None):
    with _twin_lock:
        _twin[t32.device.index] = (t32, t32._version, t16, colsum)


def _clear_twin(device):
    with _twin_lock:
        _twin.pop(device.index, None)


def _take_twin(t32):
    with _twin_lock:
        ent = _twin.pop(t32.device.index, None)
    if ent is None:
        return None, None
    src, version, t16, colsum = ent
    same = (src.data_ptr() == t32.data_ptr() and src.numel() == t32.numel() and src._version == version
            and t32.dtype == src.dtype and t32.is_contiguous())
    return (t16, colsum) if same else (None, None)


def _byproducts_of(t32):
    """-> (bf16 twin, column sums [D]) of an fp32 [M, D] gradient, from the producer if it published them."""
    t16, colsum = _take_twin(t32)
    if t16 is None:
        t16 = ops.cast_bf16(t32.contiguous())
    if colsum is None:
        colsum = bgrad(t32)
    return t16, colsum


def _bf16_of(t32):
    t16, _ = _take_twin(t32)
    if t16 is None:
        t16 = ops.cast_bf16(t32.contiguous())
    return t16


@functools.lru_cache(maxsize=None)
def _sm_count(device_index):
    return torch.cuda.get_device_properties(device_index).multi_processor_count


@functools.lru_cache(maxsize=None)
def _split_for(n_out, n_in, k_rows, n_sm=132):
    """Split-K factor of a weight-gradient GEMM (one persistent CTA per SM, 128 x 256 tiles, 64-row k-blocks): the split
    whose (tiles x splits) units fill whole waves of the grid.  Cost model = waves x (k-blocks per unit + 4 for the
    pipeline fill and the atomic epilogue that the next unit cannot hide); the smallest split within 3 % of the best
    (fewer fp32 atomics).  round(400 / tiles) leaves the 72-tile fc1 gradient at 6 splits = 3.27 waves on 132 SMs
    (0.82 of the occupied waves filled); this rule picks 9 (4.91 waves, 0.98 filled)."""
    tiles = ((n_out + 127) // 128) * ((n_in + 255) // 256)
    num_kb = (k_rows + 63) // 64
    if os.environ.get("EGOVLP_WGRAD_SPLIT", "waves") == "legacy":       # A/B knob: the round-1 rule
        return max(1, min(num_kb, round(400 / tiles)))
    costs = {}
    for s in range(1, min(num_kb, 64) + 1):
        kbs = -(-num_kb // s)
        if -(-num_kb // kbs) != s:          # the kernel drops empty splits: same as a smaller s
            continue
        if s > 1 and kbs < 2:
            break
        costs[s] = -(-tiles * s // n_sm) * (kbs + 4)
    floor = min(costs.values())
    return min(s for s, c in costs.items() if c <= 1.03 * floor)


def wgrad(dy16, x16, n_out, n_in, bias_grad=None):
    """dW[n_out, n_in] = dy^T x (contraction over token rows), fp32, split-K atomics.  `bias_grad` (fp32 [n_out],
    zero-initialised) additionally receives colsum(dy), summed from the dy tiles while they are in shared memory."""
    dw = _zeros((n_out, n_in), dy16)
    ops.gemm(dy16, x16, dw, a_mn=True, b_mn=True, accumulate=True, split_k=_split_for(n_out, n_in, dy16.shape[0], _sm_count(dy16.device.index)),
             colsum_a=bias_grad)
    return dw


def wgrad_and_bgrad(dy16, x16, n_out, n_in):
    """(dW, db) of a Linear from its bf16 output gradient: one GEMM when the fused column sums apply (n_in % 256 == 0;
    +1.0 % on the step, A/B on one box: 280.5 / 282.7 vs 278.5 / 278.9 clips/s; EGOVLP_WGRAD_COLSUM=0 disables), else
    GEMM + a column-sum pass over dy."""
    if _WGRAD_COLSUM and n_in % 256 == 0 and n_out % 8 == 0:
        db = _zeros((n_out,), dy16)
        return wgrad(dy16, x16, n_out, n_in, bias_grad=db), db
    return wgrad(dy16, x16, n_out, n_in), bgrad(dy16)


_WGRAD_COLSUM = os.environ.get("EGOVLP_WGRAD_COLSUM", "1") != "0"
# Mlp pair: fc1 saves GELU'(pre-activation) (GEMM act 3) and the fc2 input-gradient GEMM multiplies by it (act 4);
# EGOVLP_GELU_DERIV=0 = the round-1 pair (pre-activation saved, GELU' recomputed in the dgrad epilogue), for A/B runs
_ACT_FWD, _ACT_BWD = (3, 4) if os.environ.get("EGOVLP_GELU_DERIV", "1") != "0" else (1, 2)


def bgrad(dy):
    db = _zeros((dy.shape[1],), dy)
    ops.colsum_accum(dy, db)
    return db


def _wgrad_with_bgrad(dy16, x16, n_out, n_in, db):
    """(dW, db) of a Linear: `db` when its bias gradient was already summed elsewhere, else summed here from dy16."""
    return (wgrad(dy16, x16, n_out, n_in), db) if db is not None else wgrad_and_bgrad(dy16, x16, n_out, n_in)


def _linear_fwd(act16, w16, b, out):
    """out = act16 w16^T + b for the projection heads (model/model.py:72-79): the wgmma GEMM, or for the widths it cannot
    take (C % 32 != 0, e.g. the OSCC / PNR fine-tuning heads of width 2 / 16) the narrow-head kernels."""
    if w16.shape[0] % 32:
        ops.narrow_linear_fwd(act16, w16, b, out)
    else:
        ops.gemm(act16, w16, out, bias=b)


def _linear_bwd(dout, act16, w16):
    """-> (dW, db, d_act fp32) of `_linear_fwd` from its fp32 output gradient; both products take d16 = bf16(dout)."""
    n_out, n_in = w16.shape
    d16 = ops.cast_bf16(dout)
    if n_out % 32:
        return ops.narrow_linear_bwd(dout, d16, act16, w16)
    g_w, g_b = wgrad(d16, act16, n_out, n_in), bgrad(dout)
    dact = _empty((act16.shape[0], n_in), F32, dout)
    ops.gemm(d16, w16, dact, b_mn=True)
    return g_w, g_b, dact


# ----------------------------------------------------------------------------------------------------------
# video tower
# ----------------------------------------------------------------------------------------------------------
def draw_dropout_seed():
    """The Philox seed of one training forward, from torch's CPU generator (torch.manual_seed makes a run reproducible)."""
    return int(torch.randint(0, 2 ** 62, (1,)).item())


# Philox sites of the video tower's training dropouts, all keyed by the one seed its forward draws (masks of the [B*S,
# width] tensors, element (row, column), as egovlp_dropout draws them; drop-path factors per sample): site 0 = pos_drop
# on the embedded tokens; block i uses 1 + 6 i + one of the offsets below.
VIDEO_SITE_POS = 0
(VIDEO_SITE_TIME_PROJ, VIDEO_SITE_SPACE_PROJ, VIDEO_SITE_GELU, VIDEO_SITE_FC2, VIDEO_SITE_PATH_SPACE,
 VIDEO_SITE_PATH_MLP) = range(6)


def video_block_site(block, offset):
    return 1 + 6 * block + offset


class VideoBlockDrop:
    """The dropouts of one SpaceTimeBlock in training (model/video_transformer.py:36-52, 135-136, 163-177): proj_drop of
    timeattn and attn, the Mlp's two dropouts and the drop-path of the space and MLP branches, at the block's sites.
    `sites(S)` -> the ops.Drop of (time proj output, space proj output, GELU output, fc2 output), None where inactive."""

    def __init__(self, seed, block, p_time, p_space, p_mlp, p_path):
        self.seed, self.block = int(seed), int(block)
        self.p_time, self.p_space, self.p_mlp, self.p_path = float(p_time), float(p_space), float(p_mlp), float(p_path)

    def sites(self, S):
        site = functools.partial(video_block_site, self.block)
        path = self.p_path > 0
        return (ops.Drop(self.p_time, self.seed, site(VIDEO_SITE_TIME_PROJ)) if self.p_time > 0 else None,
                ops.Drop(self.p_space, self.seed, site(VIDEO_SITE_SPACE_PROJ), self.p_path, site(VIDEO_SITE_PATH_SPACE),
                         S if path else 0) if self.p_space > 0 or path else None,
                ops.Drop(self.p_mlp, self.seed, site(VIDEO_SITE_GELU)) if self.p_mlp > 0 else None,
                ops.Drop(self.p_mlp, self.seed, site(VIDEO_SITE_FC2), self.p_path, site(VIDEO_SITE_PATH_MLP),
                         S if path else 0) if self.p_mlp > 0 or path else None)


class PatchEmbedFn(torch.autograd.Function):
    """VideoPatchEmbed + cls/pos/temporal embedding assembly (model/video_transformer.py:72-77, 304-321), and the
    training pos_drop (:244, 320-321) when `drop` (an ops.Drop) is given."""

    @staticmethod
    def forward(ctx, video, cls_token, pos_embed, temporal_embed, w, b, cache, norm=None, drop=None):
        B, T, C, H, W = video.shape
        D, _, P, _ = w.shape
        _clear_twin(w.device)
        N = (H // P) * (W // P)
        S = 1 + T * N
        K = C * P * P
        patches = _empty((B * S, K), BF16, w)
        if video.dtype == torch.uint8:          # raw frames: dataset normalisation fused into the unfold
            mean, std = norm if norm is not None else ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
            ops.patch_im2col_u8(video.contiguous(), patches, P, mean, std)
        else:
            video = video.contiguous().float()
            ops.patch_im2col(video, patches, P)
        table = _empty((S, D), F32, w)
        ops.video_pos_table(cls_token.detach().contiguous(), pos_embed.detach().contiguous(),
                            temporal_embed.detach().contiguous(), b.detach(), table, T, N, D)
        x = _empty((B * S, D), F32, w)
        ops.gemm(patches, cache.get(w, (D, K)), x, bias=b.detach(), residual=table, res_row_mod=S)
        if drop is not None:                    # into a new buffer: the dropout kernel's input and output are restrict
            x = ops.dropout(x, drop.p, drop.seed, drop.site, y32=torch.empty_like(x))[0]
        ctx.dims, ctx.drop = (B, T, N, D, K, temporal_embed.shape[1]), drop
        ctx.save_for_backward(patches)
        return x.view(B, S, D)

    @staticmethod
    def backward(ctx, dx):
        (patches,) = ctx.saved_tensors
        B, T, N, D, K, F = ctx.dims
        dx = dx.contiguous().view(-1, D)
        drop = ctx.drop
        if drop is None:
            dx16 = _bf16_of(dx)
        else:                   # the gradient of the embedding is the masked one; a published twin is of the unmasked
            _take_twin(dx)
            dx16 = _empty(dx.shape, BF16, dx)
            dx = ops.dropout(dx, drop.p, drop.seed, drop.site, y32=torch.empty_like(dx), y16=dx16)[0]
        if K % 32 == 0:
            dw = wgrad(dx16, patches, D, K)
        else:           # the GEMM's N must be a multiple of 32 (K = 432 at P = 12): form dW^T = patches^T dx instead
            dw = wgrad(patches, dx16, K, D).t()
        dcls, dpos = _zeros((1, 1, D), dx), _zeros((1, N + 1, D), dx)
        dtemp, dbias = _zeros((1, F, D), dx), _zeros((D,), dx)
        tmp = _empty(((1 + T * N) * D,), F32, dx)
        ops.video_embed_bwd(dx, tmp, dcls, dpos, dtemp, dbias, B, T, N, D)
        P = int(round((K // 3) ** 0.5))
        return None, dcls, dpos, dtemp, dw.reshape(D, 3, P, P), dbias, None, None, None


def _ln16(inp, w, b, eps):
    """-> (bf16 LayerNorm(inp), mean, rstd) of an fp32 [M, D] input (deterministic: a rebuild is bit-identical)."""
    M, D = inp.shape
    y = _empty((M, D), BF16, inp)
    mean, rstd = _empty((M,), F32, inp), _empty((M,), F32, inp)
    ops.layernorm_fwd(inp, w.detach(), b.detach(), eps, y16=y, mean=mean, rstd=rstd)
    return y, mean, rstd


def _ln8(inp, w, b, eps):
    """-> ((e4m3 LayerNorm(inp), its per-row scales), None, None): the A operand of the fp8 inference GEMMs."""
    M, D = inp.shape
    y8, scale = _empty((M, D), ops.E4M3, inp), _empty((M,), F32, inp)
    ops.layernorm_fwd(inp, w.detach(), b.detach(), eps, y8=y8, row_scale=scale)
    return (y8, scale), None, None


def _proj_residual(a, pw, pb, resid, cache, drop=None):
    """fp32 resid + proj(a): the attention output projection on the bias + fp32 residual GEMM form (with `drop`, an
    ops.Drop: resid + the dropped projection)."""
    out = _empty(resid.shape, F32, a)
    ops.gemm(a, cache.get(pw), out, bias=pb.detach(), residual=resid, drop=drop)
    return out


# Most patches per frame the one-CTA-per-frame spatial attention (divided_attn_*, mode 1) takes; larger frames, up to
# 1024 patches (512 x 512 px at patch 16), run the tiled kernel (space_attn_long_*).  EGOVLP_ATTN_GENERIC and
# EGOVLP_ATTN_TC select among the divided-attention kernels only, so they do not apply above this.
SPACE_ATTN_SHORT_MAX_N = 255
SPACE_ATTN_LONG_MAX_N = 1024


def check_video_grid(B, T, N, D, HID):
    """Refuse, before any launch, a frame the spatial attention cannot take, and a large-frame batch whose widest
    activation ([B*S, max(3*D, HID)]: qkv or the MLP hidden) has 2^31 elements or more, the range the tower is verified
    in above N = 255."""
    if N > SPACE_ATTN_LONG_MAX_N:
        raise ValueError(f"video tower: {N} patches per frame; the spatial attention takes at most "
                         f"{SPACE_ATTN_LONG_MAX_N} (512 x 512 px at patch 16)")
    if N > SPACE_ATTN_SHORT_MAX_N and B * (1 + T * N) * max(3 * D, HID) >= 2 ** 31:
        raise ValueError(f"video tower: B={B} clips of {T} frames x {N} patches give activations of 2^31 elements or "
                         f"more ({B * (1 + T * N)} tokens x {max(3 * D, HID)}); split the batch")


class SpaceTimeBlockFn(torch.autograd.Function):
    """SpaceTimeBlock.forward (model/video_transformer.py:163-177) incl. both VarAttention calls and the Mlp.

    params: norm1.{w,b}, attn.qkv.{w,b}, attn.proj.{w,b}, timeattn.qkv.{w,b}, timeattn.proj.{w,b},
            norm2.{w,b}, mlp.fc1.{w,b}, mlp.fc2.{w,b}, norm3.{w,b}      (18 tensors, reference order)
    dims: (B, T, N, H, grad_mode, low_memory, fp8).  fp8 = e4m3 inference (set_inference_precision): a forward that
    records no autograd runs the qkv and fc1 GEMMs on e4m3 operands -- the LayerNorm writes its output as e4m3 with
    per-row scales, the weights come per-output-channel scaled from the cache; a training forward ignores the flag (the
    backward needs the bf16 operands).  low_memory = selective activation recompute for training: the forward
    saves x, qkv, the attention outputs, the softmax and LayerNorm statistics and the bf16 fc1 pre-activation z (21,624
    instead of 38,520 bytes per token at D = 768); the backward rebuilds the residuals tr / sr and the LayerNorm outputs
    from them with the forward's own kernels (bit-identical), and GELU(z) / GELU'(z) inside the fc2 input-gradient GEMM.
    dims[7] = a VideoBlockDrop or None: the block's training dropouts, fused into the proj / fc1 / fc2 GEMM epilogues
    (EPI_*_DROP); the backward and the low-memory rebuild regenerate the masks from the seed, so none is saved.  A
    forward with dropout runs the bf16 GEMMs even when fp8 is asked for.
    """

    @staticmethod
    def forward(ctx, x, dims, eps, cache, *p):
        (n1w, n1b, sqw, sqb, spw, spb, tqw, tqb, tpw, tpb, n2w, n2b, f1w, f1b, f2w, f2b, n3w, n3b) = p
        B, T, N, H, grad_mode, low_memory, fp8, drop = dims
        D = H * 64
        S = 1 + T * N
        M = B * S
        HID = f1w.shape[0]
        check_video_grid(B, T, N, D, HID)
        x2 = x.contiguous().view(M, D)
        # `grad_mode` = torch.is_grad_enabled() at the call site: inside Function.forward grad mode is always off and
        # needs_input_grad reflects requires_grad of the parameters even under torch.no_grad()
        train = grad_mode and any(ctx.needs_input_grad)
        drops = drop.sites(S) if drop is not None else (None, None, None, None)
        d_time, d_space, d_gelu, d_fc2 = drops
        fp8 = fp8 and not train and drop is None
        ln = _ln8 if fp8 else _ln16

        def attention(inp, qw, qb, pw, pb, mode, resid, d):
            qkv = _empty((M, 3 * D), BF16, x2)
            if fp8:
                ops.gemm_e4m3(*inp, *cache.get_e4m3(qw), qkv, bias=qb.detach(), col_scale=Q_SCALE, col_scale_ncols=D)
            else:
                ops.gemm(inp, cache.get(qw), qkv, bias=qb.detach(), col_scale=Q_SCALE, col_scale_ncols=D)
            if mode == 1 and N > SPACE_ATTN_SHORT_MAX_N:
                a, lse = ops.space_attn_long_fwd(qkv, B, T, N, H)
            else:
                a, lse = ops.divided_attn_fwd(qkv, B, T, N, H, mode)
            return qkv, a, lse, _proj_residual(a, pw, pb, resid, cache, d)

        n3, mean3, rstd3 = ln(x2, n3w, n3b, eps)
        qkv_t, a_t, lse_t, tr = attention(n3, tqw, tqb, tpw, tpb, 0, x2, d_time)  # time_residual = x + time_output
        n1, mean1, rstd1 = ln(tr, n1w, n1b, eps)
        qkv_s, a_s, lse_s, sr = attention(n1, sqw, sqb, spw, spb, 1, x2, d_space)  # space_residual = x + space_output
        n2, mean2, rstd2 = ln(sr, n2w, n2b, eps)
        h = _empty((M, HID), BF16, x2)
        # training: u = GELU'(fc1 output) for the backward, or in the low-memory mode z = the fc1 output itself (act 1
        # with out2: h is bit-identical to act 3's)
        # (the GELU-output dropout has the act 3 / act 1 + out2 forms only: a dropping forward keeps u even in inference;
        # its backward is the act 3 / 4 pair whatever EGOVLP_GELU_DERIV says)
        u = _empty((M, HID), BF16, x2) if train or d_gelu is not None else None
        act_fwd, act_bwd = (3, 4) if d_gelu is not None else (_ACT_FWD, _ACT_BWD)
        act = (1 if low_memory else act_fwd) if train or d_gelu is not None else 1
        if fp8:
            ops.gemm_e4m3(*n2, *cache.get_e4m3(f1w), h, bias=f1b.detach(), act=1)
        else:
            ops.gemm(n2, cache.get(f1w), h, bias=f1b.detach(), act=act, out2=u, drop=d_gelu)
        y = _empty((M, D), F32, x2)
        ops.gemm(h, cache.get(f2w), y, bias=f2b.detach(), residual=sr, drop=d_fc2)
        if train:
            ctx.dims, ctx.cache, ctx.eps = (B, T, N, H, HID), cache, eps
            ctx.drops, ctx.act_bwd = drops, act_bwd
            if low_memory:          # the None slots are rebuilt by the backward (see `rebuild`)
                ctx.save_for_backward(x2, None, mean3, rstd3, qkv_t, a_t, lse_t, None, None, mean1, rstd1, qkv_s, a_s,
                                      lse_s, None, None, mean2, rstd2, u, None, *p)
            else:
                ctx.save_for_backward(x2, n3, mean3, rstd3, qkv_t, a_t, lse_t, tr, n1, mean1, rstd1, qkv_s, a_s, lse_s,
                                      sr, n2, mean2, rstd2, u, h, *p)
        return y.view(B, S, D)

    @staticmethod
    def rebuild(which, sv, eps, cache, drops=(None, None, None, None)):
        """Rebuild what the low-memory forward did not save, from its saved tensors `sv` (ctx.saved_tensors):
        'sr' -> (space_residual, bf16 norm2(sr)), 'tr' -> (time_residual, bf16 norm1(tr)), 'n3' -> bf16 norm3(x).
        The proj GEMM and the LayerNorm forward are deterministic, so the results equal the forward's bit for bit; with
        dropout, `drops` = the forward's ctx.drops regenerates its masks."""
        x2, a_t, a_s, p = sv[0], sv[5], sv[12], sv[20:]
        (n1w, n1b, sqw, sqb, spw, spb, tqw, tqb, tpw, tpb, n2w, n2b, f1w, f1b, f2w, f2b, n3w, n3b) = p
        if which == "sr":
            r = _proj_residual(a_s, spw, spb, x2, cache, drops[1])
            return r, _ln16(r, n2w, n2b, eps)[0]
        if which == "tr":
            r = _proj_residual(a_t, tpw, tpb, x2, cache, drops[0])
            return r, _ln16(r, n1w, n1b, eps)[0]
        if which == "n3":
            return _ln16(x2, n3w, n3b, eps)[0]
        raise ValueError(which)

    @staticmethod
    def backward(ctx, dy):
        sv = ctx.saved_tensors
        (x2, n3, mean3, rstd3, qkv_t, a_t, lse_t, tr, n1, mean1, rstd1, qkv_s, a_s, lse_s, sr, n2, mean2, rstd2, u,
         h) = sv[:20]
        (n1w, n1b, sqw, sqb, spw, spb, tqw, tqb, tpw, tpb, n2w, n2b, f1w, f1b, f2w, f2b, n3w, n3b) = sv[20:]
        B, T, N, H, HID = ctx.dims
        cache = ctx.cache
        D = H * 64
        M = x2.shape[0]
        dy = dy.contiguous().view(M, D)
        _tls.arena = _ZeroArena(2 * D * HID + 8 * D * D + HID + 24 * D + 32 * 64, dy)
        try:
            return SpaceTimeBlockFn._backward(ctx, dy, sv, B, T, N, H, HID, D, M, cache)
        finally:
            _tls.arena = None

    @staticmethod
    def _backward(ctx, dy, sv, B, T, N, H, HID, D, M, cache):
        (x2, n3, mean3, rstd3, qkv_t, a_t, lse_t, tr, n1, mean1, rstd1, qkv_s, a_s, lse_s, sr, n2, mean2, rstd2, u,
         h) = sv[:20]
        (n1w, n1b, sqw, sqb, spw, spb, tqw, tqb, tpw, tpb, n2w, n2b, f1w, f1b, f2w, f2b, n3w, n3b) = sv[20:]
        d_time, d_space, d_gelu, d_fc2 = ctx.drops
        # a dropped branch takes dy * mask * drop-path factor / (1 - p) as the bf16 operand of its dgrad, wgrad and bias
        # gradient; the residual stream keeps dy
        if d_fc2 is None:
            dy16, g_f2b = _byproducts_of(dy)                 # fc2 bias gradient = colsum(dy)
        else:
            _take_twin(dy)                                   # its twin and column sums are those of the unmasked dy
            dy16, g_f2b = ops.drop_rows_bf16(dy, d_fc2), None
        low_memory = h is None         # rebuild sr / n2, tr / n1 and n3 as they are consumed; free each after its last use
        if low_memory:
            sr, n2 = SpaceTimeBlockFn.rebuild("sr", sv, ctx.eps, cache, ctx.drops)

        # ---- MLP:  y = sr + fc2(gelu(fc1(LN2(sr))))   (with dropout: fc2 reads the dropped GELU output h, and its input
        # gradient is multiplied by the same mask)
        if low_memory:             # u = z: du = (dy W2) * gelu'(z), and the same pass writes h = gelu(z) for the wgrad
            du, h = _empty((M, HID), BF16, dy), _empty((M, HID), BF16, dy)
            ops.gemm(dy16, cache.get(f2w), du, b_mn=True, aux=u, act=5, out2=h, drop=d_gelu)
            g_f2w, g_f2b = _wgrad_with_bgrad(dy16, h, D, HID, g_f2b)
            del h
        else:
            g_f2w, g_f2b = _wgrad_with_bgrad(dy16, h, D, HID, g_f2b)
            du = _empty((M, HID), BF16, dy)
            ops.gemm(dy16, cache.get(f2w), du, b_mn=True, aux=u, act=ctx.act_bwd, drop=d_gelu)   # (dy W2) * gelu'
        g_f1w, g_f1b = wgrad_and_bgrad(du, n2, HID, D)       # fc1 bias gradient = colsum(du), summed inside the wgrad GEMM
        del n2
        dn2 = _empty((M, D), BF16, dy)                       # LayerNorm-input gradients travel as bf16
        ops.gemm(du, cache.get(f1w), dn2, b_mn=True)
        del du
        # gradients that stay inside the block (d space_residual, d time_residual) are kept in bf16 only
        dsr16 = _empty((M, D), BF16, dy)
        g_n2w, g_n2b = _zeros((D,), dy), _zeros((D,), dy)
        # bias grad of attn.proj = colsum(d space_residual), or with dropout colsum of the masked gradient
        g_spb = _zeros((D,), dy) if d_space is None else None
        ops.layernorm_bwd(dn2, sr, n2w.detach(), mean2, rstd2, add1=dy, dx16=dsr16, dgamma=g_n2w, dbeta=g_n2b,
                          colsum_dx=g_spb)
        del dn2, sr

        def attention_bwd(dres16, qkv, a, lse, inp16, qw, pw, mode, g_pb):
            dres = dres16
            g_pw, g_pb = _wgrad_with_bgrad(dres16, a, D, D, g_pb)
            da = _empty((M, D), BF16, dres)
            ops.gemm(dres16, cache.get(pw), da, b_mn=True)
            if mode == 1 and N > SPACE_ATTN_SHORT_MAX_N:
                dqkv = ops.space_attn_long_bwd(qkv, a, da, lse, B, T, N, H, Q_SCALE)
            else:
                dqkv = ops.divided_attn_bwd(qkv, a, da, lse, B, T, N, H, mode, Q_SCALE)
            g_qw, g_qb = wgrad_and_bgrad(dqkv, inp16, 3 * D, D)
            dinp = _empty((M, D), BF16, dres)
            ops.gemm(dqkv, cache.get(qw), dinp, b_mn=True)
            return g_qw, g_qb, g_pw, g_pb, dinp

        # ---- space attention:  sr = x + proj(attn(LN1(tr)))
        if low_memory:
            tr, n1 = SpaceTimeBlockFn.rebuild("tr", sv, ctx.eps, cache, ctx.drops)
        gs16 = dsr16 if d_space is None else ops.drop_rows_bf16(dsr16, d_space)
        g_sqw, g_sqb, g_spw, g_spb, dn1 = attention_bwd(gs16, qkv_s, a_s, lse_s, n1, sqw, spw, 1, g_spb)
        del n1, gs16
        dtr16 = _empty((M, D), BF16, dy)
        g_n1w, g_n1b = _zeros((D,), dy), _zeros((D,), dy)
        # bias grad of timeattn.proj = colsum(d time_residual), or with dropout colsum of the masked gradient
        g_tpb = _zeros((D,), dy) if d_time is None else None
        ops.layernorm_bwd(dn1, tr, n1w.detach(), mean1, rstd1, dx16=dtr16, dgamma=g_n1w, dbeta=g_n1b, colsum_dx=g_tpb)
        del dn1, tr
        # ---- time attention:  tr = x + proj(timeattn(LN3(x)))
        if low_memory:
            n3 = SpaceTimeBlockFn.rebuild("n3", sv, ctx.eps, cache)
        gt16 = dtr16 if d_time is None else ops.drop_rows_bf16(dtr16, d_time)
        g_tqw, g_tqb, g_tpw, g_tpb, dn3 = attention_bwd(gt16, qkv_t, a_t, lse_t, n3, tqw, tpw, 0, g_tpb)
        del gt16
        del n3
        dx, dx16 = _empty((M, D), F32, dy), _empty((M, D), BF16, dy)
        g_n3w, g_n3b = _zeros((D,), dy), _zeros((D,), dy)
        dx_colsum = _zeros((D,), dy)                         # = the fc2 bias gradient of the block below
        ops.layernorm_bwd(dn3, x2, n3w.detach(), mean3, rstd3, add1=dsr16, add2=dtr16, dx=dx, dx16=dx16, dgamma=g_n3w,
                          dbeta=g_n3b, colsum_dx=dx_colsum)
        _publish_twin(dx, dx16, dx_colsum)
        S = 1 + T * N
        return (dx.view(B, S, D), None, None, None, g_n1w, g_n1b, g_sqw, g_sqb, g_spw, g_spb, g_tqw, g_tqb, g_tpw,
                g_tpb, g_n2w, g_n2b, g_f1w, g_f1b, g_f2w, g_f2b, g_n3w, g_n3b)


class ClsHeadFn(torch.autograd.Function):
    """norm(x)[:, 0] -> optional Linear projection (model/video_transformer.py:330; model/model.py:77-79,141-142).
    LayerNorm is applied to the B CLS rows only (the reference normalises all S rows, then slices)."""

    @staticmethod
    def forward(ctx, x, eps, cache, nw, nb, pw, pb):
        B, S, D = x.shape
        x = x.contiguous()
        cls_rows = x.view(B, S * D)[:, :D]                      # row stride S*D
        y16 = _empty((B, D), BF16, x)
        y32 = _empty((B, D), F32, x)
        mean, rstd = _empty((B,), F32, x), _empty((B,), F32, x)
        ops.layernorm_fwd(cls_rows, nw.detach(), nb.detach(), eps, y16=y16, y32=y32, mean=mean, rstd=rstd)
        ctx.has_proj = pw is not None
        ctx.shape, ctx.cache = (B, S, D), cache
        if pw is None:
            ctx.save_for_backward(x, mean, rstd, nw)
            return y32
        out = _empty((B, pw.shape[0]), F32, x)
        _linear_fwd(y16, cache.get(pw), pb.detach(), out)
        ctx.save_for_backward(x, mean, rstd, nw, y16, pw)
        return out

    @staticmethod
    def backward(ctx, dout):
        B, S, D = ctx.shape
        dout = dout.contiguous().float()
        _clear_twin(dout.device)
        g_pw = g_pb = None
        if ctx.has_proj:
            x, mean, rstd, nw, y16, pw = ctx.saved_tensors
            g_pw, g_pb, dn = _linear_bwd(dout, y16, ctx.cache.get(pw))
        else:
            x, mean, rstd, nw = ctx.saved_tensors
            dn = dout
        dx = _zeros((B, S, D), dout)
        g_nw, g_nb = _zeros((D,), dout), _zeros((D,), dout)
        ops.layernorm_bwd(dn, x.view(B, S * D)[:, :D], nw.detach(), mean, rstd, dx=dx.view(B, S * D)[:, :D],
                          dgamma=g_nw, dbeta=g_nb)
        return dx, None, None, g_nw, g_nb, g_pw, g_pb


# ----------------------------------------------------------------------------------------------------------
# text tower (DistilBERT / BERT) + ReLU/Linear projection
# ----------------------------------------------------------------------------------------------------------
# Longest caption the one-CTA-per-(sample, head) text attention (text_attn_*) takes; longer ones, up to the 512
# positions of DistilBERT, run the tiled kernel (text_attn_long_*), which also keeps the rows' lse for the backward.
TEXT_ATTN_SHORT_MAX_L = 128


def _text_tower_fwd(ctx, bert, input_ids, attention_mask, heads, eps, tokens_mode, cache, drop, p):
    """Forward of TextTowerFn (bert=False) and BertTowerFn (bert=True); see their docstrings for `p`."""
    grad_mode = True
    if isinstance(tokens_mode, tuple):
        tokens_mode, grad_mode = tokens_mode
    if bert:
        word, pos, tt, elw, elb = p[:5]
        qw_pool, qb_pool, pw, pb = p[-4:]
        layer_p = p[5:-4]
        tokens_mode = False          # the reference's compute_text_tokens returns the pooled output for BERT
    else:
        word, pos, elw, elb = p[:4]
        pw, pb = p[-2:]
        layer_p = p[4:-2]
    layers = [layer_p[16 * i: 16 * (i + 1)] for i in range(len(layer_p) // 16)]
    n_layers = len(layers)
    B, L = input_ids.shape
    if L > pos.shape[0]:
        raise EgovlpError(f"text tower: sequence length {L} exceeds the {pos.shape[0]} position embeddings "
                          "(max_position_embeddings); truncate the captions to that length")
    D = word.shape[1]
    M = B * L
    long_attn = L > TEXT_ATTN_SHORT_MAX_L
    ids = input_ids.contiguous().to(torch.int64)
    mask = attention_mask.contiguous().to(torch.int64)
    dev = word
    train = grad_mode and any(ctx.needs_input_grad)
    saved, lses = [], []
    p_hid, p_att = (float(drop[0]), float(drop[1])) if drop else (0.0, 0.0)
    seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if (p_hid > 0 or p_att > 0) else 0

    emb = _empty((M, D), F32, dev)
    # BERT: every token adds token-type row 0 (the reference passes no token_type_ids), folded into the positions
    pos_tab = (pos.detach()[:L] + tt.detach()[0]) if bert else pos.detach()
    ops.text_embed_fwd(ids, word.detach(), pos_tab, emb, B, L, D)
    x, x16 = _empty((M, D), F32, dev), _empty((M, D), BF16, dev)
    mean, rstd = _empty((M,), F32, dev), _empty((M,), F32, dev)
    ops.layernorm_fwd(emb, elw.detach(), elb.detach(), eps, y16=x16, y32=x, mean=mean, rstd=rstd)
    if p_hid > 0:
        ops.dropout(x, p_hid, seed, 0, y32=x, y16=x16)                                # embeddings dropout (in place)
    saved += [emb, mean, rstd]
    for li, lp in enumerate(layers):
        (qw, qb, kw, kb, vw, vb, ow, ob, sw, sb, l1w, l1b, l2w, l2b, fw, fb) = lp
        wqkv = cache.cat(("text_qkv_w", li, id(qw)), (qw, kw, vw))
        bqkv = torch.cat([qb.detach(), kb.detach(), vb.detach()])
        HID = l1w.shape[0]
        qkv = _empty((M, 3 * D), BF16, dev)
        ops.gemm(x16, wqkv, qkv, bias=bqkv, col_scale=Q_SCALE, col_scale_ncols=D)
        ctxv = _empty((M, D), BF16, dev)
        if long_attn:
            lse = _empty((B, heads, L), F32, dev)
            ops.text_attn_long_fwd(qkv, mask, ctxv, lse, B, L, heads, p_att, seed, 1 + 2 * li)
            lses.append(lse)
        else:
            ops.text_attn_fwd(qkv, mask, ctxv, B, L, heads, p_att, seed, 1 + 2 * li)
        sa = _empty((M, D), F32, dev)
        if bert and p_hid > 0:
            ops.gemm(ctxv, cache.get(ow), sa, bias=ob.detach())
            ops.dropout(sa, p_hid, seed, 1 + 2 * n_layers + li, add=x, y32=sa)          # BertSelfOutput: dropout + x
        else:
            ops.gemm(ctxv, cache.get(ow), sa, bias=ob.detach(), residual=x)           # sa_output + x
        x1, x1_16 = _empty((M, D), F32, dev), _empty((M, D), BF16, dev)
        m1, r1 = _empty((M,), F32, dev), _empty((M,), F32, dev)
        ops.layernorm_fwd(sa, sw.detach(), sb.detach(), eps, y16=x1_16, y32=x1, mean=m1, rstd=r1)
        hh, u = _empty((M, HID), BF16, dev), (_empty((M, HID), BF16, dev) if train else None)
        ops.gemm(x1_16, cache.get(l1w), hh, bias=l1b.detach(), act=_ACT_FWD if train else 1, out2=u)
        ff = _empty((M, D), F32, dev)
        if p_hid > 0:
            ops.gemm(hh, cache.get(l2w), ff, bias=l2b.detach())
            ops.dropout(ff, p_hid, seed, 2 + 2 * li, add=x1, y32=ff)                   # dropout(ffn_output) + sa_output
        else:
            ops.gemm(hh, cache.get(l2w), ff, bias=l2b.detach(), residual=x1)          # ffn_output + sa_output
        xn, xn16 = _empty((M, D), F32, dev), _empty((M, D), BF16, dev)
        m2, r2 = _empty((M,), F32, dev), _empty((M,), F32, dev)
        ops.layernorm_fwd(ff, fw.detach(), fb.detach(), eps, y16=xn16, y32=xn, mean=m2, rstd=r2)
        saved += [x16, qkv, ctxv, sa, m1, r1, x1_16, u, hh, ff, m2, r2]
        x, x16 = xn, xn16
    rows, stride = (M, D) if tokens_mode else (B, L * D)
    pooled = None
    if bert:                       # pooler_output = tanh(dense(h_CLS)), and relu of it when txt_proj follows
        pooled = _empty((B, D), F32, dev)
        r16 = _empty((B, D), BF16, dev) if pw is not None else None
        ops.text_pooler_fwd(x, L * D, qw_pool.detach(), qb_pool.detach(), pooled, r16, B, D)
        out = pooled
        if pw is not None:
            out = _empty((B, pw.shape[0]), F32, dev)
            _linear_fwd(r16, cache.get(pw), pb.detach(), out)
    elif pw is None:               # projection='' (nn.Identity, model/model.py:80-82): the hidden state itself
        r16 = None
        out = x if tokens_mode else x.view(B, L * D)[:, :D].clone()
    else:
        r16 = _empty((rows, D), BF16, dev)
        ops.relu_rows_fwd(x, stride, r16, rows, D)
        out = _empty((rows, pw.shape[0]), F32, dev)
        _linear_fwd(r16, cache.get(pw), pb.detach(), out)
    if train:
        ctx.meta = (B, L, D, heads, tokens_mode, n_layers, len(saved), p_hid, p_att, seed, bert)
        ctx.cache = cache
        ctx.has_proj = pw is not None
        ctx.n_lse = len(lses)
        ctx.save_for_backward(ids, mask, x, r16, pooled, *saved, *lses, *p[:len(p) - (0 if pw is not None else 2)])
    return out.view(B, L, -1) if tokens_mode else out


def _text_tower_bwd(ctx, dout):
    B, L, D, heads, tokens_mode, n_layers, n_saved, p_hid, p_att, seed, bert = ctx.meta
    cache = ctx.cache
    sv = ctx.saved_tensors
    ids, mask, x_last, r16, pooled = sv[:5]
    saved = list(sv[5:5 + n_saved])
    lses = sv[5 + n_saved:5 + n_saved + ctx.n_lse]          # one per layer when L > TEXT_ATTN_SHORT_MAX_L
    p = sv[5 + n_saved + ctx.n_lse:]
    head = 5 if bert else 4
    if bert:
        word, pos, tt, elw, elb = p[:5]
    else:
        word, pos, elw, elb = p[:4]
    layers = [p[head + 16 * i: head + 16 * (i + 1)] for i in range(n_layers)]
    M = B * L
    rows, stride = (M, D) if tokens_mode else (B, L * D)
    g_pw = g_pb = None
    if ctx.has_proj:
        pw, pb = p[-2:]
        Pd = pw.shape[0]
        dout = dout.contiguous().float().view(rows, Pd)
        g_pw, g_pb, dr = _linear_bwd(dout, r16, cache.get(pw))
    if bert:
        qw_pool = p[head + 16 * n_layers]
        g_in = dr if ctx.has_proj else dout.contiguous().float().view(B, D)
        dx = _zeros((M, D), g_in)
        g_qw_pool, g_qb_pool = _empty((D, D), F32, g_in), _empty((D,), F32, g_in)
        ops.text_pooler_bwd(g_in, pooled, ctx.has_proj, x_last, L * D, qw_pool.detach(), g_qw_pool, g_qb_pool, dx, B, D)
        dout = g_in
    elif ctx.has_proj:
        dx = _zeros((M, D), dout)
        ops.relu_rows_bwd(x_last, stride, dr, dx, rows, D)
    else:
        dout = dout.contiguous().float().view(rows, D)
        if tokens_mode:
            dx = dout
        else:
            dx = _zeros((M, D), dout)
            dx.view(B, L * D)[:, :D].copy_(dout)
    grads = []
    for li in reversed(range(n_layers)):
        (qw, qb, kw, kb, vw, vb, ow, ob, sw, sb, l1w, l1b, l2w, l2b, fw, fb) = layers[li]
        x16, qkv, ctxv, sa, m1, r1, x1_16, u, hh, ff, m2, r2 = saved[3 + 12 * li: 3 + 12 * (li + 1)]
        HID = l1w.shape[0]
        dff, dff16 = _empty((M, D), F32, dout), _empty((M, D), BF16, dout)
        g_fw, g_fb = _zeros((D,), dout), _zeros((D,), dout)
        ops.layernorm_bwd(dx, ff, fw.detach(), m2, r2, dx=dff, dx16=dff16, dgamma=g_fw, dbeta=g_fb)
        dffn, dffn16 = dff, dff16                      # gradient of the FFN output (before its dropout)
        if p_hid > 0:
            dffn, dffn16 = _empty((M, D), F32, dout), _empty((M, D), BF16, dout)
            ops.dropout(dff, p_hid, seed, 2 + 2 * li, y32=dffn, y16=dffn16)
        g_l2w, g_l2b = wgrad(dffn16, hh, D, HID), bgrad(dffn)
        du = _empty((M, HID), BF16, dout)
        ops.gemm(dffn16, cache.get(l2w), du, b_mn=True, aux=u, act=_ACT_BWD)
        g_l1w, g_l1b = wgrad(du, x1_16, HID, D), bgrad(du)
        dx1 = _empty((M, D), F32, dout)
        ops.gemm(du, cache.get(l1w), dx1, b_mn=True, residual=dff)                     # + residual path
        dsa, dsa16 = _empty((M, D), F32, dout), _empty((M, D), BF16, dout)
        g_sw, g_sb = _zeros((D,), dout), _zeros((D,), dout)
        ops.layernorm_bwd(dx1, sa, sw.detach(), m1, r1, dx=dsa, dx16=dsa16, dgamma=g_sw, dbeta=g_sb)
        dso, dso16 = dsa, dsa16                        # gradient of the attention output dense (before its dropout)
        if bert and p_hid > 0:
            dso, dso16 = _empty((M, D), F32, dout), _empty((M, D), BF16, dout)
            ops.dropout(dsa, p_hid, seed, 1 + 2 * n_layers + li, y32=dso, y16=dso16)
        g_ow, g_ob = wgrad(dso16, ctxv, D, D), bgrad(dso)
        dctx = _empty((M, D), BF16, dout)
        ops.gemm(dso16, cache.get(ow), dctx, b_mn=True)
        dqkv = _empty((M, 3 * D), BF16, dout)
        if lses:
            ops.text_attn_long_bwd(qkv, mask, ctxv, lses[li], dctx, dqkv, B, L, heads, Q_SCALE, p_att, seed,
                                   1 + 2 * li)
        else:
            ops.text_attn_bwd(qkv, mask, dctx, dqkv, B, L, heads, Q_SCALE, p_att, seed, 1 + 2 * li)
        g_wqkv, g_bqkv = wgrad(dqkv, x16, 3 * D, D), bgrad(dqkv)
        wqkv = cache.cat(("text_qkv_w", li, id(qw)), (qw, kw, vw))
        dxin = _empty((M, D), F32, dout)
        ops.gemm(dqkv, wqkv, dxin, b_mn=True, residual=dsa)                            # x feeds qkv and the residual
        dx = dxin
        gq, gk, gv = g_wqkv[:D], g_wqkv[D:2 * D], g_wqkv[2 * D:]
        bq, bk, bv = g_bqkv[:D], g_bqkv[D:2 * D], g_bqkv[2 * D:]
        grads = [gq, bq, gk, bk, gv, bv, g_ow, g_ob, g_sw, g_sb, g_l1w, g_l1b, g_l2w, g_l2b, g_fw, g_fb] + grads
    emb, mean, rstd = saved[:3]
    if p_hid > 0:
        ops.dropout(dx, p_hid, seed, 0, y32=dx)                                       # embeddings dropout, backward
    demb = _empty((M, D), F32, dout)
    g_elw, g_elb = _zeros((D,), dout), _zeros((D,), dout)
    ops.layernorm_bwd(dx, emb, elw.detach(), mean, rstd, dx=demb, dgamma=g_elw, dbeta=g_elb)
    g_word, g_pos = torch.zeros_like(word), torch.zeros_like(pos)
    ops.text_embed_bwd(ids, demb, g_word, g_pos, B, L, D)
    if not bert:
        return (None, None, None, None, None, None, None, g_word, g_pos, g_elw, g_elb, *grads, g_pw, g_pb)
    g_tt = torch.zeros_like(tt)
    g_tt[0] = g_pos[:L].sum(0)                         # token-type row 0 was added to every position row
    return (None, None, None, None, None, None, None, g_word, g_pos, g_tt, g_elw, g_elb, *grads, g_qw_pool, g_qb_pool,
            g_pw, g_pb)


class TextTowerFn(torch.autograd.Function):
    """DistilBertModel(...).last_hidden_state -> (CLS | all tokens) -> ReLU -> Linear  (model/model.py:117-138).

    params: word_emb, pos_emb, emb_ln.{w,b}, then per layer
            q.{w,b}, k.{w,b}, v.{w,b}, out.{w,b}, sa_ln.{w,b}, lin1.{w,b}, lin2.{w,b}, out_ln.{w,b}   (16 / layer),
            finally txt_proj.{w,b}.
    `drop` = (p_hidden, p_attention): HuggingFace DistilBERT's train-mode dropouts -- on the embedding LayerNorm output,
    on the attention probabilities and on the FFN output (modeling_distilbert.py; the reference calls
    `self.text_model.train()`, model/model.py:36).  Masks come from a counter-based Philox stream keyed by one seed
    drawn per forward from torch's CPU generator (so `torch.manual_seed` makes a run reproducible); the backward
    regenerates them.  Philox sites: 0 = embeddings, 1 + 2 * layer = attention probabilities, 2 + 2 * layer = FFN
    output.  (0, 0) = eval mode / the deterministic parity path."""

    @staticmethod
    def forward(ctx, input_ids, attention_mask, heads, eps, tokens_mode, cache, drop, *p):
        """`tokens_mode`: False / True, or a (tokens_mode, grad_mode) pair -- see SpaceTimeBlockFn.forward."""
        return _text_tower_fwd(ctx, False, input_ids, attention_mask, heads, eps, tokens_mode, cache, drop, p)

    @staticmethod
    def backward(ctx, dout):
        return _text_tower_bwd(ctx, dout)


class BertTowerFn(torch.autograd.Function):
    """BertModel(input_ids, attention_mask=...)['pooler_output'] -> ReLU -> Linear  (model/model.py:117-138, the
    `bert*` branch).  The encoder layers run exactly as TextTowerFn's; BERT adds token-type row 0 to every embedding
    (the reference passes no token_type_ids), a dropout on the attention output dense, and the pooler
    tanh(dense(h_CLS)) in place of the CLS row.  tokens_mode gives the pooled result too, as the reference's
    compute_text_tokens does for BERT.

    params: word_emb, pos_emb, token_type_emb, emb_ln.{w,b}, then per layer
            query.{w,b}, key.{w,b}, value.{w,b}, attention.output.dense.{w,b}, attention.output.LayerNorm.{w,b},
            intermediate.dense.{w,b}, output.dense.{w,b}, output.LayerNorm.{w,b}   (16 / layer),
            then pooler.dense.{w,b}, finally txt_proj.{w,b} (None, None for projection='').
    `drop` = (hidden_dropout_prob, attention_probs_dropout_prob), applied as HF BERT does in train mode.  Philox sites
    (n = number of layers): 0 = embeddings, 1 + 2 * layer = attention probabilities, 2 + 2 * layer = FFN output,
    1 + 2 * n + layer = attention output dense."""

    @staticmethod
    def forward(ctx, input_ids, attention_mask, heads, eps, tokens_mode, cache, drop, *p):
        return _text_tower_fwd(ctx, True, input_ids, attention_mask, heads, eps, tokens_mode, cache, drop, p)

    @staticmethod
    def backward(ctx, dout):
        return _text_tower_bwd(ctx, dout)


# ----------------------------------------------------------------------------------------------------------
# similarity + losses
# ----------------------------------------------------------------------------------------------------------
class SimMatrixFn(torch.autograd.Function):
    """sim_matrix (model/model.py:189-197): cosine similarity with the norm clamped at eps, fp32."""

    @staticmethod
    def forward(ctx, a, b, eps):
        a, b = a.contiguous().float(), b.contiguous().float()
        an, na = ops.rownorm_fwd(a, eps)
        bn, nb = ops.rownorm_fwd(b, eps)
        ctx.eps = eps
        ctx.save_for_backward(an, na, bn, nb)
        return ops.sgemm(an, bn)

    @staticmethod
    def backward(ctx, dx):
        an, na, bn, nb = ctx.saved_tensors
        dx = dx.contiguous().float()
        dan = ops.sgemm(dx, bn, trans_b=False)                    # dX @ bn
        dbn = ops.sgemm(dx, an, trans_a=True, trans_b=False)      # dX^T @ an
        return ops.rownorm_bwd(dan, an, na, ctx.eps), ops.rownorm_bwd(dbn, bn, nb, ctx.eps), None


class NceLossFn(torch.autograd.Function):
    """EgoNCE / InfoNCE on a similarity matrix with a uint8 positives mask (model/loss.py:13-25, 34-53)."""

    @staticmethod
    def forward(ctx, x, mask, temperature):
        x = x.contiguous().float()
        loss, stats = ops.nce_fwd(x, mask, 1.0 / temperature)
        ctx.inv_temp = 1.0 / temperature
        ctx.save_for_backward(x, mask, stats)
        return loss

    @staticmethod
    def backward(ctx, g):
        x, mask, stats = ctx.saved_tensors
        return ops.nce_bwd(x, mask, stats, ctx.inv_temp, g.contiguous().float()), None, None


class FusedEgoNceFn(torch.autograd.Function):
    """sim_matrix + EgoNCE / InfoNCE from the gathered embeddings and multi-hot tags in ONE kernel per direction
    (csrc/loss_fused.cu; reference trainer/trainer_egoclip.py:130-135).  `text` / `video` [G, C], `verb` / `noun`
    [G, n] are fp32 row-strided views (e.g. column slices of the packed all-gather buffer, read in place).  Gradients
    are produced for rows [row0, row0 + n_local) only and returned zero-padded to [G, C] when n_local < G is not the
    whole matrix -- `GatherEgoNceFn` below hands the local slice out directly instead."""

    @staticmethod
    def forward(ctx, text, video, verb, noun, temperature, mode):
        loss, saved = ops.egonce_fused_fwd(text, video, verb, noun, 1.0 / temperature, mode)
        ctx.args = (1.0 / temperature, mode, verb.shape[1] if verb is not None else 0,
                    noun.shape[1] if noun is not None else 0)
        ctx.save_for_backward(text, video, *saved)
        return loss

    @staticmethod
    def backward(ctx, g):
        text, video, *saved = ctx.saved_tensors
        inv_temp, mode, nv, nn_ = ctx.args
        dt, dv = ops.egonce_fused_bwd(text, video, saved, nv, nn_, inv_temp, mode, g.contiguous().float(), 0,
                                      text.shape[0])
        return dt, dv, None, None, None, None


class GatherEgoNceFn(torch.autograd.Function):
    """The exchange step of the data-parallel training step, fused with the loss: local embeddings + tags -> ONE packed
    all-gather (one pack launch, one ncclAllGather) -> the fused EgoNCE kernel on column views of the gathered buffer ->
    loss; the backward kernel emits d text / d video of THIS rank's rows only (the reference's AllGather_multi backward,
    trainer/trainer_egoclip.py:23-27).  `gather(packed_local) -> packed_all` is the collective (identity at world 1)."""

    @staticmethod
    def forward(ctx, text, video, verb, noun, temperature, mode, gather, rank):
        B, Ct = text.shape
        Cv, nv, nn_ = video.shape[1], verb.shape[1], noun.shape[1]
        assert Ct == Cv
        packed = ops.pack_rows4(text.contiguous().float(), video.contiguous().float(), verb.contiguous().float(),
                                noun.contiguous().float())
        allp = gather(packed)                              # [world * B, Ct + Cv + nv + nn], rank-major
        t, v = allp[:, :Ct], allp[:, Ct:Ct + Cv]
        vb, nb_ = allp[:, Ct + Cv:Ct + Cv + nv], allp[:, Ct + Cv + nv:]
        loss, saved = ops.egonce_fused_fwd(t, v, vb, nb_, 1.0 / temperature, mode)
        ctx.args = (1.0 / temperature, mode, nv, nn_, Ct, Cv, rank * B, B)
        ctx.save_for_backward(allp, *saved)
        return loss

    @staticmethod
    def backward(ctx, g):
        allp, *saved = ctx.saved_tensors
        inv_temp, mode, nv, nn_, Ct, Cv, row0, B = ctx.args
        dt, dv = ops.egonce_fused_bwd(allp[:, :Ct], allp[:, Ct:Ct + Cv], saved, nv, nn_, inv_temp, mode,
                                      g.contiguous().float(), row0, B)
        return dt, dv, None, None, None, None, None, None


class MaxMarginFn(torch.autograd.Function):
    """MaxMarginRankingLoss (model/loss.py:63-90) and, with `row_weight`, AdaptiveMaxMarginRankingLoss
    (model/loss.py:100-133); no host-side index building.  The weight gets no gradient (the reference feeds the
    dataset's relevancy, a constant)."""

    @staticmethod
    def forward(ctx, x, margin, fix_norm, row_weight=None):
        x = x.contiguous().float()
        w = None if row_weight is None else row_weight.detach().contiguous().float()
        ctx.args = (margin, fix_norm)
        ctx.has_w = w is not None
        ctx.save_for_backward(*((x, w) if w is not None else (x,)))
        return ops.maxmargin_fwd(x, margin, fix_norm, w)

    @staticmethod
    def backward(ctx, g):
        x = ctx.saved_tensors[0]
        w = ctx.saved_tensors[1] if ctx.has_w else None
        return ops.maxmargin_bwd(x, ctx.args[0], ctx.args[1], g.contiguous().float(), w), None, None, None


class CrossEntropyFn(torch.autograd.Function):
    """nn.CrossEntropyLoss() with its defaults (model/loss.py:135-141): mean over the rows whose target is not
    `ignore_index` of the max-subtracted LSE minus the target logit, fp32.  `x` [G, C] is read in place when its rows are
    unit-stride."""

    @staticmethod
    def forward(ctx, x, target, ignore_index):
        x = x if (x.dtype == F32 and x.stride(1) == 1) else x.float().contiguous()
        target = target.contiguous()
        loss, lse, stats = ops.cross_entropy_fwd(x, target, ignore_index)
        ctx.ignore_index = ignore_index
        ctx.save_for_backward(x, target, lse, stats)
        return loss

    @staticmethod
    def backward(ctx, g):
        x, target, lse, stats = ctx.saved_tensors
        return ops.cross_entropy_bwd(x, target, lse, stats, g.contiguous().float(), ctx.ignore_index), None, None
