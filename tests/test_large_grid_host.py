"""CPU-only checks of frames above 255 patches: the `img_size` key of video_params, the bicubic pos_embed resampling
on load (ViT-B/16 file and trainer checkpoints), the reference's refusal without the key, unchanged state_dict keys,
the refusal of oversized batches, the new C-ABI entries' refusals, and the oracle against
tests/golden/video_large_grid.npz (recorded from the unmodified reference by oracle/make_large_grid_golden.py)."""
import warnings

import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden

warnings.simplefilter("ignore")
VIDEO = {"model": "SpaceTimeTransformer", "arch_config": "base_patch16_224", "num_frames": 4, "pretrained": True,
         "time_init": "zeros"}
TEXT = {"model": "distilbert-base-uncased", "pretrained": True, "input": "text"}
REFUSED = 'Loading models with different spatial resolution / patch number not yet implemented, sorry.'


def expected_pos_embed(pe224, rows, cols):
    """What loading a 14 x 14 pos_embed into a rows x cols tower must give, computed here from F.interpolate."""
    D = pe224.shape[-1]
    grid = pe224[:, 1:].float().reshape(1, 14, 14, D).permute(0, 3, 1, 2)
    grid = F.interpolate(grid, size=(rows, cols), mode="bicubic", align_corners=False)
    return torch.cat([pe224[:, :1], grid.permute(0, 2, 3, 1).reshape(1, rows * cols, D)], 1)


def test_img_size_key_sets_the_grid_and_keeps_the_state_dict_keys():
    from egovlp_b200.model.model import FrozenInTime
    base = FrozenInTime(dict(VIDEO), dict(TEXT))
    assert base.video_model.pos_embed.shape == (1, 197, 768)
    assert base.video_model.pos_embed_grid() == (14, 14)
    net = FrozenInTime(dict(VIDEO, img_size=384), dict(TEXT))
    assert net.video_model.pos_embed.shape == (1, 577, 768)
    assert net.video_model.pos_embed_grid() == (24, 24)
    sd, sd_base = net.state_dict(), base.state_dict()
    assert list(sd) == list(sd_base)
    assert all(sd[k].shape == sd_base[k].shape for k in sd if k != "video_model.pos_embed")
    assert FrozenInTime(dict(VIDEO, img_size=224), dict(TEXT)).video_model.pos_embed.shape == (1, 197, 768)
    for bad in ("384", 384.0, 8, True):
        with pytest.raises(ValueError, match="img_size"):
            FrozenInTime(dict(VIDEO, img_size=bad), dict(TEXT))


def test_rectangular_tower_grid():
    from egovlp_b200.model.video_transformer import SpaceTimeTransformer
    net = SpaceTimeTransformer(img_size=(256, 320), embed_dim=128, depth=1, num_heads=2, num_frames=2, num_classes=0)
    assert net.pos_embed.shape == (1, 321, 128) and net.pos_embed_grid() == (16, 20)


def test_resample_pos_embed_is_bicubic_with_the_cls_entry_kept():
    from egovlp_b200.model.model import resample_pos_embed
    pe = torch.randn(1, 197, 64, generator=torch.Generator().manual_seed(1))
    for rows, cols in ((24, 24), (16, 20), (14, 14), (32, 32)):
        got = resample_pos_embed(pe, (rows, cols))
        assert got.shape == (1, 1 + rows * cols, 64)
        assert torch.equal(got[:, 0], pe[:, 0])
        torch.testing.assert_close(got, expected_pos_embed(pe, rows, cols), rtol=0, atol=0)
    torch.testing.assert_close(resample_pos_embed(pe, (14, 14)), pe, rtol=1e-6, atol=1e-6)   # identity grid
    with pytest.raises(NotImplementedError, match="square"):
        resample_pos_embed(torch.zeros(1, 1 + 16 * 20, 8), (24, 24))


def test_checkpoint_of_another_grid(tmp_path):
    """A 224-px trainer checkpoint loads into an img_size = 384 model with the resampled pos_embed; every other tensor
    loads unchanged.  Without the key, the reference's refusal stays, word for word."""
    from egovlp_b200.model.model import FrozenInTime
    src = FrozenInTime(dict(VIDEO), dict(TEXT))
    with torch.no_grad():
        src.video_model.pos_embed.normal_(0, 0.02, generator=torch.Generator().manual_seed(3))
    path = tmp_path / "ckpt224.pth"
    torch.save({"state_dict": {"module." + k: v for k, v in src.state_dict().items()}}, path)
    net = FrozenInTime(dict(VIDEO, img_size=384), dict(TEXT), load_checkpoint=str(path))
    pe = src.video_model.pos_embed.detach()
    torch.testing.assert_close(net.video_model.pos_embed.detach(), expected_pos_embed(pe, 24, 24), rtol=0, atol=0)
    sd, sd_src = net.state_dict(), src.state_dict()
    assert list(sd) == list(sd_src)
    assert all(torch.equal(sd[k], sd_src[k]) for k in sd if k != "video_model.pos_embed")
    # the same checkpoint into the same grid: untouched
    same = FrozenInTime(dict(VIDEO, img_size=224), dict(TEXT), load_checkpoint=str(path))
    assert torch.equal(same.video_model.pos_embed, src.video_model.pos_embed)
    # without the key: a 384 checkpoint into the default (224) tower is refused as the reference refuses it
    path384 = tmp_path / "ckpt384.pth"
    torch.save({"state_dict": net.state_dict()}, path384)
    with pytest.raises(NotImplementedError) as e:
        FrozenInTime(dict(VIDEO), dict(TEXT), load_checkpoint=str(path384))
    assert str(e.value) == REFUSED


def test_vit_file_is_resampled_on_from_scratch_init(tmp_path, monkeypatch):
    from egovlp_b200.model import model as mm
    from egovlp_b200.model.video_transformer import SpaceTimeTransformer
    vit = SpaceTimeTransformer(num_frames=1, num_classes=0).state_dict()     # timm ViT-B/16 key names and shapes
    vit.pop("temporal_embed")
    path = tmp_path / "vit.pth"
    torch.save(vit, path)
    monkeypatch.setattr(mm, "_VIT_B16_FILE", str(path))
    net = mm.FrozenInTime(dict(VIDEO, img_size=320), dict(TEXT))
    torch.testing.assert_close(net.video_model.pos_embed.detach(), expected_pos_embed(vit["pos_embed"], 20, 20),
                               rtol=0, atol=0)
    assert torch.equal(net.video_model.blocks[3].mlp.fc1.weight, vit["blocks.3.mlp.fc1.weight"])


def test_oversized_large_grid_batches_are_refused_before_any_launch():
    """Above 255 patches per frame the tower is verified up to activations of 2^31 elements; larger batches and frames
    above 1024 patches are refused from the shapes alone (meta tensors: nothing is computed)."""
    from egovlp_b200 import engine
    from egovlp_b200.model.video_transformer import SpaceTimeTransformer
    net = SpaceTimeTransformer(img_size=512, depth=1, num_frames=16, num_classes=0)
    with torch.no_grad():
        for B, T, px in ((43, 16, 512), (57, 16, 512), (8, 2, 528)):
            video = torch.empty(B, T, 3, px, px, device="meta")
            with pytest.raises(ValueError, match="2\\^31|at most 1024"):
                net.forward_tokens(video)
    engine.check_video_grid(42, 16, 1024, 768, 3072)          # 42 x 16385 x 3072 < 2^31: accepted
    engine.check_video_grid(1000, 16, 196, 768, 3072)         # N <= 255: the existing kernels, no new limit
    with pytest.raises(ValueError, match="2\\^31"):
        engine.check_video_grid(43, 16, 1024, 768, 3072)


def test_space_attn_long_workspace_refuses_bad_shapes():
    from egovlp_b200 import _lib
    ws = _lib.lib().egovlp_space_attn_long_workspace_floats
    assert ws(2, 16, 1024, 12) == 2 * 12 * (1 + 16 * 1024) + 2 * 12 * 16 * 192
    for bad in ((2, 16, 1025, 12), (2, 16, 0, 12), (0, 16, 256, 12), (2, 0, 256, 12), (2, 16, 256, 0)):
        assert ws(*bad) == -1, bad


def test_oracle_reproduces_the_large_grid_golden():
    """oracle.reference_port (shape-generic) against the unmodified reference at N = 256 and 320, fp32 vs fp32."""
    from egovlp_b200 import synthetic as syn
    from oracle import reference_port as rp
    g = load_golden("video_large_grid.npz")
    B, T, seed = int(g["B"]), int(g["T"]), int(g["seed"])
    for tag in ("n256", "n320"):
        img = tuple(int(v) for v in g[f"{tag}:img"])
        dims = syn.model_dims(embed_dim=128, depth=2, heads=2, patch=16, img=img, num_frames=4, proj_dim=32)
        sd = syn.seeded_state_dict(dims, seed=seed, text=False, proj=False)
        p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
        video = syn.synthetic_video(B, T, seed=seed, img=img)
        x, Tn, n = rp.video_tokens(video, p)
        assert n == (img[0] // 16) * (img[1] // 16)
        for i in range(2):
            x = rp.space_time_block(x, p, f"video_model.blocks.{i}.", 2, Tn, n, 1e-6)
        out = F.layer_norm(x, (128,), p["video_model.norm.weight"], p["video_model.norm.bias"], 1e-6)[:, 0]
        torch.testing.assert_close(out, g[f"{tag}:out"], rtol=1e-4, atol=1e-5)
        tok = x.detach().reshape(-1, 128)[g[f"{tag}:token_rows"]]
        torch.testing.assert_close(tok, g[f"{tag}:tokens"], rtol=1e-4, atol=1e-5)
        (out * g[f"{tag}:probe"]).sum().backward()
        checked = 0
        for k, v in g.items():
            if k.startswith(f"{tag}:g:"):
                name = k[len(f"{tag}:g:"):]
                grad = p[name].grad
                torch.testing.assert_close(grad.flatten()[g[f"{tag}:gi:{name}"]], v, rtol=2e-4, atol=2e-5)
                torch.testing.assert_close(grad.norm(), g[f"{tag}:n:{name}"], rtol=2e-4, atol=2e-6)
                checked += 1
        assert checked == len(sd)
