"""Host (numpy) reference of the dropout random streams (csrc/common.cuh) and of the keep masks the kernels draw from
them, the one Philox implementation the tests use (test_philox_ref_host.py pins it to Random123's known answers).

  philox4x32_10(key, ctr)   Random123's philox4x32-10 on a 64-bit key and a 64-bit counter, with the counter's words
                            2 and 3 fixed at 0x2B7E1516 and 0x28AED2A6 (`philox4x32`: the general four-word form)
  dropout_key(seed, site)   seed ^ (0x9E3779B97F4A7C15 * (uint32(site + 1)))  (mod 2^64; site + 1 wraps in uint32)
  dropout_threshold(p)      floor(float64(float32(p)) * 2^32), at most 0xFFFFFFFF; a word < threshold is DROPPED

The documented stream layouts (DESIGN section 3), each a function of (seed, site, p) and the shape:
  flat          element 4g + w of a flat tensor is kept iff word w of philox(key, g) >= threshold: egovlp_dropout,
                ops.dropout_mask, the GEMM dropout forms (element (m, n) of [M, N] is element m * N + n) and
                drop_rows_kernel
  drop-path     sample b's factor: word b & 3 of philox(key, b >> 2) (the flat stream of a vector of samples)
  short attn    text_attn_* (L <= 128): (b, h, i, j) is kept iff word 0 of philox(key, ((b * H + h) * L + i) * L + j)
                >= threshold
  long attn     text_attn_long_* (L <= 512): word j & 3 of philox(key, ((b * 4096 + h) * 512 + i) * 128 + (j >> 2))
Multipliers are keep / (1 - float32(p)) in float64: the exact value of what the kernels scale by (their own fp32
1 / (1 - p) is within 3 fp32 roundings of it)."""
import numpy as np
import torch

_M32 = np.uint64(0xFFFFFFFF)
_M64 = (1 << 64) - 1
KEY_MUL = 0x9E3779B97F4A7C15
CTR_HI = (0x2B7E1516, 0x28AED2A6)        # counter words 2 and 3 of the project's form


def philox4x32(ctr, key):
    """Random123 philox4x32-10: ctr = four uint64 arrays (or ints) holding 32-bit words, key = two 32-bit words.
    Returns the four output words as uint64 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _M32 for c in ctr)
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = np.uint64(key[0] & 0xFFFFFFFF), np.uint64(key[1] & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2       # 32 x 32 -> 64 bits, exact in uint64
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
    return c0, c1, c2, c3


def philox4x32_10(key, ctr):
    """common.cuh philox4x32_10(key, ctr) on a uint64 array of counters -> its four 32-bit words (uint64 arrays)."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    return philox4x32((ctr & _M32, ctr >> np.uint64(32), CTR_HI[0], CTR_HI[1]), (key & 0xFFFFFFFF, key >> 32))


def dropout_key(seed, site):
    return (int(seed) ^ (KEY_MUL * ((int(site) + 1) & 0xFFFFFFFF))) & _M64


def dropout_threshold(p):
    t = float(np.float32(p)) * 4294967296.0
    return 0xFFFFFFFF if t >= 4294967295.0 else int(t)


def _keep(words, p):
    return words >= np.uint64(dropout_threshold(p))


def flat_keep(n, p, seed, site):
    """bool [n]: the flat stream's keep bits of elements 0 .. n - 1."""
    words = philox4x32_10(dropout_key(seed, site), np.arange((n + 3) // 4, dtype=np.uint64))
    return torch.from_numpy(_keep(np.stack(words, -1).reshape(-1)[:n], p))


def flat_multiplier(shape, p, seed, site):
    """float64 multipliers (0 or 1 / (1 - p)) of a contiguous tensor of `shape` under the flat stream."""
    return multiplier(flat_keep(int(np.prod(shape)), p, seed, site).view(shape), p)


def drop_path_keep(n, p, seed, site):
    """bool [n]: whether sample b keeps its branch (its factor is 1 / (1 - p), else 0)."""
    b = np.arange(n, dtype=np.uint64)
    words = np.stack(philox4x32_10(dropout_key(seed, site), b >> np.uint64(2)), -1)
    return torch.from_numpy(_keep(words[np.arange(n), (b & np.uint64(3)).astype(np.int64)], p))


def short_attn_keep(p, seed, site, B, H, L):
    """bool [B, H, L(i), L(j)]: the keep mask of text_attn_fwd / text_attn_bwd."""
    ctr = np.arange(B * H * L * L, dtype=np.uint64)          # ((b * H + h) * L + i) * L + j, in that order
    return torch.from_numpy(_keep(philox4x32_10(dropout_key(seed, site), ctr)[0], p).reshape(B, H, L, L))


def long_attn_keep(p, seed, site, B, H, L):
    """bool [B, H, L(i), L(j)]: the keep mask of text_attn_long_*."""
    b, h, i, jg = np.meshgrid(np.arange(B, dtype=np.uint64), np.arange(H, dtype=np.uint64), np.arange(L, dtype=np.uint64),
                              np.arange((L + 3) // 4, dtype=np.uint64), indexing="ij")
    words = philox4x32_10(dropout_key(seed, site), ((b * np.uint64(4096) + h) * np.uint64(512) + i) * np.uint64(128) + jg)
    return torch.from_numpy(np.stack([_keep(w, p) for w in words], -1).reshape(B, H, L, -1)[..., :L])


def multiplier(keep, p):
    """float64 keep / (1 - float32(p))."""
    return keep.double() / (1 - float(np.float32(p)))
