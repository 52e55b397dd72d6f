"""Deterministic mode (torch.use_deterministic_algorithms), host side: the partitions of the deterministic reductions
are functions of the shapes alone, and the workspaces the library asks for match what its kernels index."""
import pytest

from egovlp_b200 import engine
from egovlp_b200._lib import lib

# the step's weight gradients (n_out, n_in) at D = 768: qkv, proj, fc1, fc2
WGRAD_SHAPES = [(2304, 768), (768, 768), (3072, 768), (768, 3072)]
TOKENS = [64 * 3137, 2 * 3137, 2 * 16 * 197, 1000, 37]


@pytest.mark.parametrize("n_out,n_in", WGRAD_SHAPES)
def test_det_split_is_a_function_of_the_shapes(n_out, n_in, monkeypatch):
    for k in TOKENS:
        # the rule of an H100 SXM (132 SMs), on every card (PCIe: 114) and whatever EGOVLP_WGRAD_SPLIT says
        want = engine._waves_split(-(-n_out // 128) * -(-n_in // 256), -(-k // 64), 132)
        assert engine._det_split_for(n_out, n_in, k) == want == engine._split_for(n_out, n_in, k, 132)
        monkeypatch.setenv("EGOVLP_WGRAD_SPLIT", "legacy")
        engine._det_split_for.cache_clear()
        assert engine._det_split_for(n_out, n_in, k) == want
        monkeypatch.delenv("EGOVLP_WGRAD_SPLIT")
        engine._det_split_for.cache_clear()


def test_default_split_rule_is_unchanged():
    """The default rule still follows the card's SM count: the values it gave before the deterministic mode existed,
    per token count, at 132 and 114 SMs."""
    want = {(2304, 768): [7, 2, 2, 2, 2, 2, 2, 2, 1, 1], (768, 768): [7, 19, 7, 6, 7, 6, 6, 6, 1, 1],
            (3072, 768): [9, 11, 3, 3, 3, 3, 1, 1, 1, 1], (768, 3072): [9, 11, 3, 3, 3, 3, 1, 1, 1, 1]}
    for (o, i), w in want.items():
        assert [engine._split_for(o, i, k, sm) for k in TOKENS for sm in (132, 114)] == w


@pytest.mark.parametrize("M,N,K,split", [(2304, 768, 64 * 3137, 4), (768, 3072, 1000, 9), (200, 256, 130, 3),
                                         (136, 96, 64, 5), (768, 768, 37, 1)])
def test_gemm_det_workspace_matches_the_kernel_layout(M, N, K, split):
    num_kb = -(-K // 64)
    s = max(1, min(split, num_kb))
    kbps = -(-num_kb // s)
    s = -(-num_kb // kbps)                       # no empty splits
    Mp = -(-M // 128) * 128
    nnb = N // 256 if N % 256 == 0 else -(-N // 128)
    assert lib().egovlp_gemm_det_workspace_floats(M, N, K, split) == s * Mp * N + s * nnb * Mp
    assert lib().egovlp_gemm_det_workspace_floats(0, N, K, split) == -1


@pytest.mark.parametrize("rows,D", [(1, 768), (4095, 768), (4096, 768), (64 * 3137, 768), (2 * 16 * 3, 256)])
def test_layernorm_det_workspace_covers_both_grids(rows, D):
    pipe = min(-(-rows // 4), 2 * 132)
    gen = min(-(-rows // 4), 12 * 132)
    assert lib().egovlp_layernorm_bwd_det_workspace_floats(rows, D) == 3 * max(pipe, gen) * D


@pytest.mark.parametrize("M,N,fp32", [(64 * 3137, 768, 0), (1000, 3072, 1), (7, 32, 0), (200000, 256, 1)])
def test_colsum_det_workspace_is_sized_for_132_sms(M, N, fp32):
    vec = 4 if fp32 else 8
    cb = -(-(N // vec) // 32)
    rb = max(1, min(-(-M // 64), -(-(132 * 8) // cb)))
    rpb = -(-M // rb)
    rb = -(-M // rpb)
    assert lib().egovlp_colsum_det_workspace_floats(M, N, fp32) == rb * N


@pytest.mark.parametrize("B,T,N,H,mode,parts", [(2, 16, 196, 12, 0, 4), (2, 8, 196, 12, 0, 4), (2, 4, 196, 2, 0, 4),
                                                (2, 3, 196, 2, 0, 1), (2, 16, 196, 12, 1, 1), (1, 5, 7, 1, 0, 1)])
def test_attention_det_workspace_has_a_slot_per_group_and_part(B, T, N, H, mode, parts):
    if mode == 1:
        groups = T
    else:
        pg = min(N, 112 // T) if (T <= 16 and 16 % T == 0) else min(N, 127 // T)
        groups = -(-N // pg)
    assert lib().egovlp_divided_attn_bwd_det_workspace_floats(B, T, N, H, mode) == B * H * groups * parts * 3 * 64


def test_maxmargin_det_workspace_is_the_forward_grid():
    for G in (2, 16, 64, 512, 4096):
        assert lib().egovlp_maxmargin_det_workspace_floats(G) == min(1024, -(-G * G // 256))
    assert lib().egovlp_maxmargin_det_workspace_floats(1) == -1
