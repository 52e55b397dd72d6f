"""Space-time video transformer ("frozen-in-time" TimeSformer-B variant) on the project's H100 kernels.

API mirror of the reference's model/video_transformer.py (SpaceTimeTransformer, SpaceTimeBlock, VarAttention,
Mlp, VideoPatchEmbed): same constructor arguments, attribute names and state_dict keys, so checkpoints and the
config-driven factory keep working.  The nn.Linear / nn.LayerNorm / nn.Conv2d members are parameter containers
(default initialisation identical to the reference's); their math runs in egovlp_b200.engine.
"""
from functools import partial

import torch
from torch import nn

from .. import engine, ops


def _to_2tuple(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def _check_rate(name, p):
    assert 0. <= p < 1., f"{name} must lie in [0, 1), got {p}"


class DropPath(nn.Module):
    """Stochastic depth per sample (timm's DropPath, which the reference imports): in training a residual branch is
    zeroed for a whole clip with probability drop_prob and kept clips are scaled by 1 / (1 - drop_prob).  No parameters;
    SpaceTimeBlock applies it inside the proj / fc2 GEMM epilogues."""

    def __init__(self, drop_prob=0.):
        super().__init__()
        _check_rate("drop_path", drop_prob)
        self.drop_prob = float(drop_prob)

    def extra_repr(self):
        return f"drop_prob={self.drop_prob}"


class Mlp(nn.Module):
    """fc1 -> GELU(erf) -> dropout -> fc2 -> dropout (reference :36-52).  The two dropouts (rate `drop`, active in
    training) run in the fc1 and fc2 GEMM epilogues of SpaceTimeBlock."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.):
        super().__init__()
        _check_rate("drop", drop)
        assert act_layer is nn.GELU, "the fc1 epilogue implements GELU(erf) only"
        hidden = hidden_features or in_features
        # parameter containers only (keys mlp.fc1.*, mlp.fc2.*): GELU and the two GEMMs run in the fused epilogues
        self.fc1, self.fc2 = nn.Linear(in_features, hidden), nn.Linear(hidden, out_features or in_features)
        self.drop = nn.Dropout(drop)


class VideoPatchEmbed(nn.Module):
    """Video to patch embedding (reference :55-77)."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, num_frames=8):
        super().__init__()
        img_size, patch_size = _to_2tuple(img_size), _to_2tuple(patch_size)
        self.img_size, self.patch_size = img_size, patch_size
        self.num_patches = (img_size[1] // patch_size[1]) * (img_size[0] // patch_size[0]) * num_frames
        self.num_frames, self.embed_dim = num_frames, embed_dim
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)


class VarAttention(nn.Module):
    """qkv / proj parameter holder with the reference's `initialize='zeros'` rule (:80-98).  `proj_drop`: dropout on
    the projected output in training, applied in the proj GEMM epilogue.  `attn_drop` is accepted and has no effect, as
    in the reference, whose VarAttention builds `attn_drop` but never calls it (:97, 100-137)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0., proj_drop=0.,
                 initialize='random'):
        super().__init__()
        _check_rate("attn_drop", attn_drop)
        _check_rate("proj_drop", proj_drop)
        assert qkv_bias, "qkv_bias=False is not implemented (reference builds the tower with qkv_bias=True)"
        assert dim // num_heads == 64 and qk_scale is None, "kernels are specialised for head_dim 64"
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj_drop = nn.Dropout(proj_drop)
        if initialize == 'zeros':                      # reference :90-96: the temporal branch starts as the zero map
            with torch.no_grad():
                for t, v in ((self.qkv.weight, 0.), (self.qkv.bias, 0.), (self.proj.weight, 1.), (self.proj.bias, 0.)):
                    t.fill_(v)


class SpaceTimeBlock(nn.Module):
    """Reference :140-177.  In training, `drop` drops the time and space proj outputs and the Mlp's GELU and fc2
    outputs, and `drop_path` drops the space and MLP branches per clip (the time branch has no drop-path, as in the
    reference); `attn_drop` has no effect (see VarAttention).  eval() never drops."""

    def __init__(self, dim, num_heads, mlp_ratio=4., qkv_bias=False, qk_scale=None, drop=0., attn_drop=0.,
                 drop_path=0., act_layer=nn.GELU, norm_layer=nn.LayerNorm, time_init='zeros',
                 attention_style='frozen-in-time'):
        super().__init__()
        _check_rate("drop_path", drop_path)
        if attention_style != 'frozen-in-time':
            raise NotImplementedError
        self.norm1 = norm_layer(dim)
        self.attn = VarAttention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale, attn_drop=attn_drop,
                                 proj_drop=drop)
        self.timeattn = VarAttention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale,
                                     attn_drop=attn_drop, proj_drop=drop, initialize=time_init)
        self.drop_path = DropPath(drop_path) if drop_path > 0. else nn.Identity()
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(in_features=dim, hidden_features=int(dim * mlp_ratio), act_layer=act_layer, drop=drop)
        self.norm3 = norm_layer(dim)
        self.attention_style = attention_style
        self.num_heads = num_heads

    def kernel_params(self):
        return (self.norm1.weight, self.norm1.bias, self.attn.qkv.weight, self.attn.qkv.bias, self.attn.proj.weight,
                self.attn.proj.bias, self.timeattn.qkv.weight, self.timeattn.qkv.bias, self.timeattn.proj.weight,
                self.timeattn.proj.bias, self.norm2.weight, self.norm2.bias, self.mlp.fc1.weight, self.mlp.fc1.bias,
                self.mlp.fc2.weight, self.mlp.fc2.bias, self.norm3.weight, self.norm3.bias)

    def dropout_rates(self):
        """(time proj, space proj, Mlp, drop-path) rates."""
        p_path = self.drop_path.drop_prob if isinstance(self.drop_path, DropPath) else 0.
        return self.timeattn.proj_drop.p, self.attn.proj_drop.p, self.mlp.drop.p, p_path

    def forward(self, x, einops_from_space=None, einops_to_space=None, einops_from_time=None, einops_to_time=None,
                time_n=None, space_f=None, cache=None, low_memory=False, fp8=False, drop_seed=None, block_index=0):
        """x [B, 1 + space_f*time_n, D] fp32.  The einops pattern arguments of the reference signature are
        accepted and ignored: the token layout is fixed to the reference's 'b (f n) d'.  `low_memory`: selective
        activation recompute in training (see SpaceTimeTransformer.set_grad_checkpointing); `fp8`: e4m3 inference GEMMs
        (see SpaceTimeTransformer.set_inference_precision).  In training with a rate > 0 the dropout masks are drawn
        from `drop_seed` (a new seed from torch's generator when None) at the Philox sites of block `block_index`
        (engine.video_block_site)."""
        B = x.shape[0]
        eps = self.norm1.eps
        cache = cache if cache is not None else _default_cache(self)
        drop = None
        rates = self.dropout_rates()
        if self.training and any(r > 0 for r in rates):
            seed = engine.draw_dropout_seed() if drop_seed is None else drop_seed
            drop = engine.VideoBlockDrop(seed, block_index, *rates)
        dims = (B, space_f, time_n, self.num_heads, torch.is_grad_enabled(), bool(low_memory), bool(fp8), drop)
        return engine.SpaceTimeBlockFn.apply(x, dims, eps, cache, *self.kernel_params())


def _default_cache(module):
    c = getattr(module, "_bf16_cache", None)
    if c is None:
        c = engine.Bf16Cache()
        object.__setattr__(module, "_bf16_cache", c)
    return c


class SpaceTimeTransformer(nn.Module):
    """Same constructor as the reference (:196-199).  forward(x[B,T,3,H,W]) -> [B, embed_dim] (CLS feature), or
    head(features) when a classifier head is set.  `img_size` (an int or an (H, W) pair) sets the pos_embed grid:
    any frame of at most 1024 patches runs, e.g. 224 to 512 px or 256 x 320 at patch 16.  Above 255 patches per frame
    the spatial attention runs on its tiled kernel, which the EGOVLP_ATTN_GENERIC / EGOVLP_ATTN_TC switches do not
    select; such batches are refused when an activation would reach 2^31 elements (engine.check_video_grid).

    Regularisation in training, as the reference (:244-251, 320-321): `drop_rate` = dropout on the embedded tokens
    (pos_drop), on the time and space proj outputs and on the Mlp's GELU and fc2 outputs; `drop_path_rate` = stochastic
    depth, block i dropping its space and MLP branches per clip with rate linspace(0, drop_path_rate, depth)[i].
    `attn_drop_rate` is accepted and has no effect, as in the reference.  The masks follow `self.training`, not grad
    mode, and come from a counter-based Philox stream under one seed drawn per forward from torch's CPU generator (so
    torch.manual_seed reproduces a run); they are fused into the GEMM epilogues and regenerated by the backward."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, num_classes=1000, embed_dim=768, depth=12,
                 num_heads=12, mlp_ratio=4., qkv_bias=True, qk_scale=None, representation_size=None,
                 drop_rate=0., attn_drop_rate=0., drop_path_rate=0., hybrid_backbone=None, norm_layer=None,
                 num_frames=8, time_init='rand', attention_style='frozen-in-time'):
        super().__init__()
        for name, p in (("drop_rate", drop_rate), ("attn_drop_rate", attn_drop_rate), ("drop_path_rate", drop_path_rate)):
            _check_rate(name, p)
        if hybrid_backbone is not None:
            raise NotImplementedError('hybrid backbone not implemented')
        if representation_size:
            raise NotImplementedError('representation_size is not implemented (reference never sets it)')
        self.num_classes = num_classes
        self.num_features = self.embed_dim = embed_dim
        self.num_frames = num_frames
        norm_layer = norm_layer or partial(nn.LayerNorm, eps=1e-6)
        self.patch_embed = VideoPatchEmbed(img_size=img_size, patch_size=patch_size, in_chans=in_chans,
                                           embed_dim=embed_dim, num_frames=num_frames)
        self.patches_per_frame = self.patch_embed.num_patches // num_frames
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, self.patches_per_frame + 1, embed_dim))
        self.temporal_embed = nn.Parameter(torch.zeros(1, num_frames, embed_dim))
        self.pos_drop = nn.Dropout(p=drop_rate)
        dpr = [v.item() for v in torch.linspace(0, drop_path_rate, depth)]      # stochastic depth decay rule (:246)
        self.blocks = nn.ModuleList([
            SpaceTimeBlock(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias,
                           qk_scale=qk_scale, drop=drop_rate, attn_drop=attn_drop_rate, drop_path=dpr[i],
                           norm_layer=norm_layer, time_init=time_init, attention_style=attention_style)
            for i in range(depth)])
        self.norm = norm_layer(embed_dim)
        self.pre_logits = nn.Identity()
        self.head = nn.Linear(self.num_features, num_classes) if num_classes > 0 else nn.Identity()
        nn.init.trunc_normal_(self.pos_embed, std=.02)
        nn.init.trunc_normal_(self.cls_token, std=.02)
        if num_frames == 1:                            # reference :268-270: image mode re-initialises every layer
            for m in self.modules():
                if isinstance(m, nn.Linear):
                    nn.init.trunc_normal_(m.weight, std=.02)
                    if m.bias is not None:
                        nn.init.zeros_(m.bias)
                elif isinstance(m, nn.LayerNorm):
                    nn.init.zeros_(m.bias)
                    nn.init.ones_(m.weight)
        self.einops_from_space, self.einops_to_space = 'b (f n) d', '(b f) n d'
        self.einops_from_time, self.einops_to_time = 'b (f n) d', '(b n) f d'
        self.grad_checkpointing = False
        self.inference_precision = "bf16"
        object.__setattr__(self, "_bf16_cache", engine.Bf16Cache())

    def pos_embed_grid(self):
        """(rows, cols) of patches per frame that pos_embed is laid out for."""
        pe = self.patch_embed
        return pe.img_size[0] // pe.patch_size[0], pe.img_size[1] // pe.patch_size[1]

    def set_grad_checkpointing(self, enable=True):
        """Trade compute for activation memory in training.  This is selective recompute, not timm's re-run of whole
        blocks: each block keeps its input, the qkv and attention outputs, the softmax / LayerNorm statistics and the bf16
        fc1 pre-activation (0.56x the activation bytes), and its backward rebuilds the two attention residuals, the three
        LayerNorm outputs and GELU / GELU' of the pre-activation from them.  The forward, inference and the state_dict
        are unchanged; the MLP gradients are rounded slightly differently (GELU is taken of the bf16 pre-activation)."""
        self.grad_checkpointing = bool(enable)

    def set_inference_precision(self, precision="bf16"):
        """Trade a bounded accuracy loss for speed in inference.  "fp8": forwards that record no autograd (evaluation,
        feature extraction under torch.no_grad()) run each block's three LayerNorm-fed GEMMs -- timeattn.qkv, attn.qkv
        and mlp.fc1, 62.5 % of the block's GEMM FLOPs -- on e4m3 tensor-core operands: the LayerNorm output with one
        scale per token row, the weights with one scale per output channel (re-quantised whenever the parameter
        changes).  Rows stay independent, so results do not depend on the batch size.  Every other GEMM, the text
        tower, and every training forward of the tower (grad mode on and a parameter or input of a block requiring a
        gradient) stay bf16; a tower frozen with requires_grad_(False) runs in fp8 even while a head on top trains.  A tower
        in train() with a dropout rate > 0 drops even under torch.no_grad(), and such forwards run bf16 too.  "bf16" (the
        default) restores the bf16 path bit for bit.  The state_dict is unchanged."""
        if precision not in ("bf16", "fp8"):
            raise ValueError(f"inference precision must be 'bf16' or 'fp8', got {precision!r}")
        self.inference_precision = precision

    def forward_tokens(self, x, _refresh=True):
        """All tokens after the 12 blocks, [B, S, D] fp32 (before the final norm)."""
        B, F, C, H, W = x.shape
        assert F <= self.num_frames
        cache = self._bf16_cache
        if _refresh and torch.is_grad_enabled():
            cache.refresh()                            # training forward: bf16 weight copies follow ANY optimizer
        pe = self.patch_embed
        n = (H // pe.patch_size[0]) * (W // pe.patch_size[1])
        if self.blocks:
            engine.check_video_grid(B, F, n, self.embed_dim, self.blocks[0].mlp.fc1.out_features)
        # uint8 frames are normalised on the fly with `input_norm` = (mean, std) (default: ImageNet, as the reference's
        # data_loader/transforms.py); float frames are taken as already normalised (the reference contract).
        # training dropouts: one Philox seed for the whole tower, drawn only when some rate is active
        seed = pos_drop = None
        if self.training and (self.pos_drop.p > 0 or any(r > 0 for b in self.blocks for r in b.dropout_rates())):
            seed = engine.draw_dropout_seed()
            if self.pos_drop.p > 0:
                pos_drop = ops.Drop(self.pos_drop.p, seed, engine.VIDEO_SITE_POS)
        x = engine.PatchEmbedFn.apply(x, self.cls_token, self.pos_embed, self.temporal_embed, pe.proj.weight,
                                      pe.proj.bias, cache, getattr(self, "input_norm", None), pos_drop)
        # a forward that drops anywhere runs bf16 in every block (the fp8 GEMMs have no mask; block 0 of a drop-path-only
        # tower has nothing to drop but stays bf16 too)
        fp8 = self.inference_precision == "fp8" and seed is None
        for i, blk in enumerate(self.blocks):
            x = blk(x, time_n=n, space_f=F, cache=cache, low_memory=self.grad_checkpointing, fp8=fp8, drop_seed=seed,
                    block_index=i)
        return x

    def forward_features(self, x, proj=None, _refresh=True):
        """norm(x)[:, 0]; when `proj` (an nn.Linear) is given its projection is fused behind the CLS LayerNorm."""
        x = self.forward_tokens(x, _refresh)
        pw, pb = (proj.weight, proj.bias) if proj is not None else (None, None)
        return engine.ClsHeadFn.apply(x, self.norm.eps, self._bf16_cache, self.norm.weight, self.norm.bias, pw, pb)

    def forward(self, x):
        if isinstance(self.head, nn.Linear):
            return self.forward_features(x, proj=self.head)
        return self.forward_features(x)
