"""tests/philox_ref.py, the host reference every dropout test compares the kernels' masks with, pinned on the CPU:
Random123's published philox4x32-10 known answers, the project's fixed counter words, the key (with the uint32 wrap
of site + 1), the threshold, and the stream layouts written out for single elements."""
import numpy as np
import pytest
import torch
from philox_ref import (CTR_HI, drop_path_keep, dropout_key, dropout_threshold, flat_keep, long_attn_keep, philox4x32,
                        philox4x32_10, short_attn_keep)

M = 0xFFFFFFFF


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((M, M, M, M), (M, M), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox4x32_10_known_answers(ctr, key, want):
    """Random123's kat_vectors for philox4x32-10."""
    assert tuple(int(w) for w in philox4x32(ctr, key)) == want


def test_project_form_is_philox_with_fixed_high_counter_words():
    rng = np.random.default_rng(0)
    keys = [0, 1, 0xFFFFFFFFFFFFFFFF, 0x8000000000000001, int(rng.integers(0, 2 ** 63)) * 2 + 1]
    ctrs = np.array([0, 1, 3, 0xFFFFFFFF, 0x100000000, 0xFFFFFFFFFFFFFFFF] + list(rng.integers(0, 2 ** 63, 20)),
                    dtype=np.uint64)
    for key in keys:
        got = philox4x32_10(key, ctrs)
        for n, c in enumerate(ctrs):
            c = int(c)
            want = philox4x32((c & M, c >> 32, CTR_HI[0], CTR_HI[1]), (key & M, key >> 32))
            assert tuple(int(w[n]) for w in got) == tuple(int(w) for w in want), (hex(key), hex(c))


def test_dropout_threshold():
    assert dropout_threshold(0.0) == 0
    assert dropout_threshold(0.1) == 429496736            # float32(0.1) = 0.100000001490116...
    assert dropout_threshold(0.5) == 1 << 31
    below_one = float(np.nextafter(np.float32(1), np.float32(0)))
    assert dropout_threshold(below_one) == 0xFFFFFF00      # (1 - 2^-24) * 2^32, exact
    assert dropout_threshold(1.0) == 0xFFFFFFFF


def test_dropout_key_wraps_site_plus_one_in_uint32():
    seed = 0x8123456789ABCDEF
    assert dropout_key(seed, 0xFFFFFFFF) == seed            # uint32(site + 1) = 0
    assert dropout_key(seed, 0) == seed ^ 0x9E3779B97F4A7C15
    assert dropout_key(seed, 72) == seed ^ ((0x9E3779B97F4A7C15 * 73) % 2 ** 64)
    assert all(0 <= dropout_key(seed, s) < 2 ** 64 for s in (1, 2 ** 31, 2 ** 32 - 2))


def test_stream_layouts_element_by_element():
    seed, site, p = 0xF00DFACE12345678, 9, 0.3
    key, t = dropout_key(seed, site), dropout_threshold(p)
    word = lambda ctr, w: int(philox4x32_10(key, np.array([ctr], dtype=np.uint64))[w][0])
    flat = flat_keep(4 * 5 + 3, p, seed, site)
    for e in (0, 1, 2, 3, 4, 13, 22):
        assert bool(flat[e]) == (word(e // 4, e % 4) >= t), e
    path = drop_path_keep(11, p, seed, site)
    assert torch.equal(path, flat_keep(11, p, seed, site))   # the flat stream of a vector of samples
    B, H, L = 2, 3, 5
    short = short_attn_keep(p, seed, site, B, H, L)
    long = long_attn_keep(p, seed, site, B, H, L)
    for b, h, i, j in ((0, 0, 0, 0), (1, 2, 4, 4), (1, 0, 3, 1), (0, 2, 2, 3)):
        assert bool(short[b, h, i, j]) == (word(((b * H + h) * L + i) * L + j, 0) >= t)
        assert bool(long[b, h, i, j]) == (word(((b * 4096 + h) * 512 + i) * 128 + j // 4, j % 4) >= t)
    assert not short_attn_keep(0.0, seed, site, B, H, L).logical_not().any()      # p = 0 keeps everything
