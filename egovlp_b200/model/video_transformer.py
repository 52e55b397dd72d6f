"""Space-time video transformer ("frozen-in-time" TimeSformer-B variant) on the project's H100 kernels.

API mirror of the reference's model/video_transformer.py (SpaceTimeTransformer, SpaceTimeBlock, VarAttention,
Mlp, VideoPatchEmbed): same constructor arguments, attribute names and state_dict keys, so checkpoints and the
config-driven factory keep working.  The nn.Linear / nn.LayerNorm / nn.Conv2d members are parameter containers
(default initialisation identical to the reference's); their math runs in egovlp_b200.engine.
"""
from functools import partial

import torch
from torch import nn

from .. import engine


def _to_2tuple(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


class Mlp(nn.Module):
    """fc1 -> GELU(erf) -> fc2 (reference :36-52); dropout p must be 0 (all shipped configs)."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.):
        super().__init__()
        assert drop == 0., "dropout inside the video tower is not implemented (reference configs use 0)"
        assert act_layer is nn.GELU, "the fc1 epilogue implements GELU(erf) only"
        hidden = hidden_features or in_features
        # parameter containers only (keys mlp.fc1.*, mlp.fc2.*): GELU and the two GEMMs run in the fused epilogues
        self.fc1, self.fc2 = nn.Linear(in_features, hidden), nn.Linear(hidden, out_features or in_features)


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
    """qkv / proj parameter holder with the reference's `initialize='zeros'` rule (:80-98)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0., proj_drop=0.,
                 initialize='random'):
        super().__init__()
        assert attn_drop == 0. and proj_drop == 0., "attention dropout is not implemented (reference configs use 0)"
        assert qkv_bias, "qkv_bias=False is not implemented (reference builds the tower with qkv_bias=True)"
        assert dim // num_heads == 64 and qk_scale is None, "kernels are specialised for head_dim 64"
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        if initialize == 'zeros':                      # reference :90-96: the temporal branch starts as the zero map
            with torch.no_grad():
                for t, v in ((self.qkv.weight, 0.), (self.qkv.bias, 0.), (self.proj.weight, 1.), (self.proj.bias, 0.)):
                    t.fill_(v)


class SpaceTimeBlock(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio=4., qkv_bias=False, qk_scale=None, drop=0., attn_drop=0.,
                 drop_path=0., act_layer=nn.GELU, norm_layer=nn.LayerNorm, time_init='zeros',
                 attention_style='frozen-in-time'):
        super().__init__()
        assert drop_path == 0., "stochastic depth is not implemented (reference configs use 0)"
        if attention_style != 'frozen-in-time':
            raise NotImplementedError
        self.norm1 = norm_layer(dim)
        self.attn = VarAttention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale, attn_drop=attn_drop,
                                 proj_drop=drop)
        self.timeattn = VarAttention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale,
                                     attn_drop=attn_drop, proj_drop=drop, initialize=time_init)
        self.drop_path = nn.Identity()
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

    def forward(self, x, einops_from_space=None, einops_to_space=None, einops_from_time=None, einops_to_time=None,
                time_n=None, space_f=None, cache=None, low_memory=False, fp8=False):
        """x [B, 1 + space_f*time_n, D] fp32.  The einops pattern arguments of the reference signature are
        accepted and ignored: the token layout is fixed to the reference's 'b (f n) d'.  `low_memory`: selective
        activation recompute in training (see SpaceTimeTransformer.set_grad_checkpointing); `fp8`: e4m3 inference GEMMs
        (see SpaceTimeTransformer.set_inference_precision)."""
        B = x.shape[0]
        eps = self.norm1.eps
        cache = cache if cache is not None else _default_cache(self)
        dims = (B, space_f, time_n, self.num_heads, torch.is_grad_enabled(), bool(low_memory), bool(fp8))
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
    select; such batches are refused when an activation would reach 2^31 elements (engine.check_video_grid)."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, num_classes=1000, embed_dim=768, depth=12,
                 num_heads=12, mlp_ratio=4., qkv_bias=True, qk_scale=None, representation_size=None,
                 drop_rate=0., attn_drop_rate=0., drop_path_rate=0., hybrid_backbone=None, norm_layer=None,
                 num_frames=8, time_init='rand', attention_style='frozen-in-time'):
        super().__init__()
        assert drop_rate == 0. and attn_drop_rate == 0. and drop_path_rate == 0.
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
        self.blocks = nn.ModuleList([
            SpaceTimeBlock(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias,
                           qk_scale=qk_scale, drop=drop_rate, attn_drop=attn_drop_rate, drop_path=0.,
                           norm_layer=norm_layer, time_init=time_init, attention_style=attention_style)
            for _ in range(depth)])
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
        gradient) stay bf16; a tower frozen with requires_grad_(False) runs in fp8 even while a head on top trains.  "bf16" (the
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
        x = engine.PatchEmbedFn.apply(x, self.cls_token, self.pos_embed, self.temporal_embed, pe.proj.weight,
                                      pe.proj.bias, cache, getattr(self, "input_norm", None))
        for blk in self.blocks:
            x = blk(x, time_n=n, space_f=F, cache=cache, low_memory=self.grad_checkpointing,
                    fp8=self.inference_precision == "fp8")
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
