"""Host side of the video tower's training dropouts: the constructor takes the reference's rates, the stochastic-depth
rule is the reference's linspace, attn_drop_rate changes nothing the kernels see, the state_dict keys stay, and the
`video_params` keys reach the tower."""
import pytest
import torch

from egovlp_b200 import engine
from egovlp_b200.model.model import _build_video_tower
from egovlp_b200.model.video_transformer import DropPath, SpaceTimeBlock, SpaceTimeTransformer, VarAttention, Mlp

TINY = dict(img_size=32, patch_size=16, embed_dim=128, depth=4, num_heads=2, num_frames=4, num_classes=0)


def tower(seed=0, **rates):
    torch.manual_seed(seed)
    return SpaceTimeTransformer(**TINY, **rates)


def test_constructors_take_the_rates_and_refuse_ones_outside_0_1():
    net = tower(drop_rate=0.1, attn_drop_rate=0.2, drop_path_rate=0.3)
    assert net.pos_drop.p == 0.1
    for blk in net.blocks:
        assert blk.attn.proj_drop.p == blk.timeattn.proj_drop.p == blk.mlp.drop.p == 0.1
        assert blk.attn.attn_drop.p == blk.timeattn.attn_drop.p == 0.2
    Mlp(128, 512, drop=0.5)
    VarAttention(128, 2, qkv_bias=True, attn_drop=0.5, proj_drop=0.5)
    SpaceTimeBlock(128, 2, qkv_bias=True, drop=0.5, attn_drop=0.5, drop_path=0.5)
    for bad in (-0.1, 1.0):
        for kw in ("drop_rate", "attn_drop_rate", "drop_path_rate"):
            with pytest.raises(AssertionError):
                tower(**{kw: bad})
        with pytest.raises(AssertionError):
            SpaceTimeBlock(128, 2, qkv_bias=True, drop_path=bad)


def test_drop_path_rates_are_the_references_linspace():
    net = tower(drop_path_rate=0.3)
    dpr = [x.item() for x in torch.linspace(0, 0.3, TINY["depth"])]       # reference :246
    assert not isinstance(net.blocks[0].drop_path, DropPath)                # block 0 never drops
    for blk, r in zip(net.blocks, dpr):
        assert blk.dropout_rates()[3] == r
        if r > 0:
            assert isinstance(blk.drop_path, DropPath) and blk.drop_path.drop_prob == r


def test_attn_drop_rate_changes_neither_the_math_nor_the_state_dict():
    plain, other = tower(), tower(attn_drop_rate=0.4)
    sd0, sd1 = plain.state_dict(), other.state_dict()
    assert list(sd0) == list(sd1) and all(torch.equal(sd0[k], sd1[k]) for k in sd0)
    assert all(b0.dropout_rates() == b1.dropout_rates() == (0., 0., 0., 0.) for b0, b1 in zip(plain.blocks, other.blocks))
    assert all(not any(p.numel() for p in m.parameters(recurse=False)) for m in other.modules()
               if isinstance(m, (torch.nn.Dropout, DropPath)))


def test_state_dict_keys_are_unchanged_by_the_rates():
    assert list(tower().state_dict()) == list(tower(drop_rate=0.1, attn_drop_rate=0.1, drop_path_rate=0.1).state_dict())


def test_video_params_keys_reach_the_tower():
    vp = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 4, "img_size": 32}
    net = _build_video_tower(vp, from_scratch=False)
    assert net.pos_drop.p == 0 and all(b.dropout_rates() == (0., 0., 0., 0.) for b in net.blocks)
    net = _build_video_tower(dict(vp, drop_rate=0.1, attn_drop_rate=0.2, drop_path_rate=0.2), from_scratch=False)
    assert net.pos_drop.p == 0.1 and net.blocks[0].attn.attn_drop.p == 0.2
    assert [b.dropout_rates() for b in net.blocks] == [(0.1, 0.1, 0.1, r.item()) for r in torch.linspace(0, 0.2, 12)]


def test_site_layout():
    assert engine.VIDEO_SITE_POS == 0
    assert [engine.video_block_site(2, k) for k in range(6)] == list(range(13, 19))
    t, s, g, f = engine.VideoBlockDrop(5, 2, 0.1, 0.2, 0.3, 0.4).sites(17)
    assert (t.site, t.p, t.path_rows) == (13, 0.1, 0)
    assert (s.site, s.p, s.path_site, s.path_p, s.path_rows) == (14, 0.2, 17, 0.4, 17)
    assert (g.site, g.p, g.path_rows) == (15, 0.3, 0)
    assert (f.site, f.p, f.path_site, f.path_p, f.path_rows) == (16, 0.3, 18, 0.4, 17)
    assert engine.VideoBlockDrop(5, 0, 0., 0., 0., 0.).sites(17) == (None, None, None, None)
