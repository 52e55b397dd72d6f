// Text-tower self-attention for long captions (128 < L <= 512; any L in 1..512 is accepted): tiled, online-softmax
// attention on the tensor cores with a key-padding mask and in-kernel attention dropout, forward and backward.
//
// Same contract as text_attn_* (text.cu): qkv bf16 [B*L, 3D] read in place (q pre-scaled by the QKV GEMM epilogue),
// attention_mask int64 [B, L] (0 = padded key, any 0/1 pattern), out bf16 [B*L, D] with the heads merged.  Head dim 64.
//
// Tiling: one CTA (4 warps, 16 rows each) per (64-row tile, head, sample).  The other operand streams through a
// two-stage cp.async ring of 64-row tiles; rows >= L are zero-filled by the copy (src-size 0), so a tile never reads
// the next sample's rows, and keys >= L are masked whatever the tile holds.  The CTA builds a bitmap of its sample's
// valid keys in the prologue and skips every 64-key tile without one -- in the forward and in both backward passes
// -- so a batch padded to 512 for one long caption costs what its valid key tiles cost.
// Math: bf16 mma.sync m16n8k16 with fp32 accumulation, fp32 online softmax in exp2 (as the divided attention).
//
// Backward, with no floating-point atomics (bitwise reproducible run to run):
//   1. row pass:   delta_i = sum_d dO_id * O_id                          -> workspace fp32 [B, H, L]
//   2. key pass:   per 64-key tile, dV = P'^T dO and dK = dS^T Q over all query tiles, P recomputed from lse
//   3. query pass: per 64-query tile, dQ = q_scale * dS K over the valid key tiles
// where P' = P * keep / (1 - p) and dS = P * (dP' - delta), dP' = (dO V^T) * keep / (1 - p).
//
// Dropout keep mask (HF DistilBERT: `weights = dropout(softmax(scores))`): element (b, h, i, j) is kept iff word
// (j & 3) of philox4x32_10(dropout_key(seed, site), ((b * 4096 + h) * 512 + i) * 128 + (j >> 2)) is
// >= dropout_threshold(p).  One Philox call serves four consecutive keys; the mask does not depend on B, H or L.
#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

constexpr int HD = 64;
constexpr int TILE = 64;                   // rows per tile (queries or keys)
constexpr int MAX_L = 512;
constexpr int NTHREADS = 128;              // 4 warps x 16 rows
constexpr int TILE_BYTES = TILE * HD * 2;  // one 64 x 64 bf16 tile
constexpr float LOG2E = 1.4426950408889634f;

// ---- cp.async ----
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// 64 rows (row0.., of sample b) x 64 bf16 columns at column col of a [B*L, ld] matrix -> swizzled tile; rows >= L
// are zero-filled and their addresses never read
__device__ __forceinline__ void load_tile(uint32_t tile, const bf16* base, long long ld, int col, int b, int L,
                                          int row0) {
  for (int idx = threadIdx.x; idx < TILE * 8; idx += NTHREADS) {
    const int r = idx >> 3, c = idx & 7, row = row0 + r;
    const bool valid = row < L;
    const bf16* src = base + ((long long)b * L + (valid ? row : 0)) * ld + col + c * 8;
    cp_async16(sw_addr(tile, r, c), src, valid);
  }
}

// bitmap of sample b's valid keys (bit j of kb[j >> 5]; bits >= L are 0) and of its 64-key tiles with a valid key
__device__ __forceinline__ uint32_t key_bitmap(const long long* __restrict__ mask, int b, int L, uint32_t* kb) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j0 = warp * 32; j0 < MAX_L; j0 += NTHREADS) {
    const int j = j0 + lane;
    const uint32_t w = __ballot_sync(0xffffffffu, j < L && mask[(long long)b * L + j] != 0);
    if (lane == 0) kb[j0 >> 5] = w;
  }
  __syncthreads();
  uint32_t tiles = 0;
#pragma unroll
  for (int kt = 0; kt < MAX_L / TILE; ++kt)
    if (kb[2 * kt] | kb[2 * kt + 1]) tiles |= 1u << kt;
  return tiles;
}

// ---- dropout ----
struct Drop {
  bool on;
  uint32_t thresh;
  float inv_keep;
  unsigned long long key;
};
__device__ __forceinline__ Drop make_drop(float p, unsigned long long seed, uint32_t site) {
  return Drop{p > 0.f, dropout_threshold(p), p > 0.f ? 1.f / (1.f - p) : 1.f, dropout_key(seed, site)};
}
// keep bits of keys 4*jg .. 4*jg+3 of row i (bit w = key 4*jg + w)
__device__ __forceinline__ uint32_t keep4(const Drop& d, int b, int h, int i, int jg) {
  const uint4 r = philox4x32_10(d.key, (((unsigned long long)b * 4096ull + h) * 512ull + i) * 128ull + jg);
  return (uint32_t)(r.x >= d.thresh) | ((uint32_t)(r.y >= d.thresh) << 1) | ((uint32_t)(r.z >= d.thresh) << 2) |
         ((uint32_t)(r.w >= d.thresh) << 3);
}
// Keep bits of one m16n8 accumulator with rows = queries i0.. (16) and columns = keys j0.. (8, j0 % 8 == 0), as
// bits 0..3 in the order of the fragment's c[0..3]: lane computes (row lane & 15, key group lane >> 4) and the quad
// fetches its two rows' nibbles.
__device__ __forceinline__ uint32_t keep_qk(const Drop& d, int b, int h, int i0, int j0, int lane) {
  const uint32_t nib = keep4(d, b, h, i0 + (lane & 15), (j0 >> 2) + (lane >> 4));
  const int gq = lane >> 2, t = lane & 3, src = gq + 16 * (t >> 1), sh = 2 * (t & 1);
  const uint32_t n0 = __shfl_sync(0xffffffffu, nib, src), n1 = __shfl_sync(0xffffffffu, nib, src + 8);
  return ((n0 >> sh) & 3u) | (((n1 >> sh) & 3u) << 2);
}
// The same with rows = keys j0.. (16, j0 % 4 == 0) and columns = queries i0.. (8): lane computes (query lane & 7,
// key group lane >> 3).
__device__ __forceinline__ uint32_t keep_kq(const Drop& d, int b, int h, int j0, int i0, int lane) {
  const uint32_t nib = keep4(d, b, h, i0 + (lane & 7), (j0 >> 2) + (lane >> 3));
  const int gq = lane >> 2, t = lane & 3, w = gq & 3, s0 = (gq >> 2) * 8 + 2 * t, s1 = s0 + 16;
  const uint32_t a = __shfl_sync(0xffffffffu, nib, s0), bb = __shfl_sync(0xffffffffu, nib, s0 + 1);
  const uint32_t c = __shfl_sync(0xffffffffu, nib, s1), e = __shfl_sync(0xffffffffu, nib, s1 + 1);
  return ((a >> w) & 1u) | (((bb >> w) & 1u) << 1) | (((c >> w) & 1u) << 2) | (((e >> w) & 1u) << 3);
}

__device__ __forceinline__ bool key_ok(const uint32_t* kb, int j) { return (kb[j >> 5] >> (j & 31)) & 1u; }

// ------------------------------------------------------------------------------------------------------------
// forward: grid (ceil(L / 64), H, B)
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
text_attn_long_fwd_kernel(const bf16* __restrict__ qkv, const long long* __restrict__ mask, bf16* __restrict__ out,
                          float* __restrict__ lse, int L, int H, float p_drop, unsigned long long seed, uint32_t site) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint32_t kb[MAX_L / 32];
  const uint32_t sq = smem_u32(smem), sk = sq + TILE_BYTES, sv = sk + 2 * TILE_BYTES;   // k, v: two stages each
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z, D = H * HD;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const Drop drop = make_drop(p_drop, seed, site);

  load_tile(sq, qkv, 3 * D, h * HD, b, L, qt * TILE);
  uint32_t tiles = key_bitmap(mask, b, L, kb);
  int kt = tiles ? __ffs(tiles) - 1 : -1;
  if (kt >= 0) {
    load_tile(sk, qkv, 3 * D, D + h * HD, b, L, kt * TILE);
    load_tile(sv, qkv, 3 * D, 2 * D + h * HD, b, L, kt * TILE);
    tiles &= tiles - 1;
  }
  cp_async_commit();

  const int r0 = warp * 16, i0 = qt * TILE + r0;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }

  for (int stage = 0; kt >= 0; stage ^= 1) {
    const int next = tiles ? __ffs(tiles) - 1 : -1;
    if (next >= 0) {
      load_tile(sk + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, D + h * HD, b, L, next * TILE);
      load_tile(sv + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, 2 * D + h * HD, b, L, next * TILE);
      tiles &= tiles - 1;
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const uint32_t kt_s = sk + stage * TILE_BYTES, vt_s = sv + stage * TILE_BYTES;
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t qf[4];
      load_a_frag(sq, r0, kk, lane, qf);
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        uint32_t bf[4];
        load_b_frag_nk(kt_s, 16 * p, kk, lane, bf);
        mma_bf16(s[2 * p], qf, bf[0], bf[1]);
        mma_bf16(s[2 * p + 1], qf, bf[2], bf[3]);
      }
    }
    // key mask (padding and j >= L)
    float cm0 = -INFINITY, cm1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t bits = kb[2 * kt + (j >> 2)] >> ((j & 3) * 8 + 2 * t);
      if (!(bits & 1u)) s[j][0] = s[j][2] = -INFINITY;
      if (!(bits & 2u)) s[j][1] = s[j][3] = -INFINITY;
      cm0 = fmaxf(cm0, fmaxf(s[j][0], s[j][1]));
      cm1 = fmaxf(cm1, fmaxf(s[j][2], s[j][3]));
    }
    cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 1)); cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 2));
    cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 1)); cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 2));
    const float mn0 = fmaxf(m0, cm0), mn1 = fmaxf(m1, cm1);
    const float ms0 = (mn0 == -INFINITY) ? 0.f : mn0, ms1 = (mn1 == -INFINITY) ? 0.f : mn1;
    const float a0 = exp2f((m0 - ms0) * LOG2E), a1 = exp2f((m1 - ms1) * LOG2E);   // m = -inf -> 0
    m0 = mn0; m1 = mn1;
    l0 *= a0; l1 *= a1;
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] *= a0; o[j][1] *= a0; o[j][2] *= a1; o[j][3] *= a1; }
    uint32_t pf[4][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p0 = exp2f((s[j][0] - ms0) * LOG2E), p1 = exp2f((s[j][1] - ms0) * LOG2E);
      float p2 = exp2f((s[j][2] - ms1) * LOG2E), p3 = exp2f((s[j][3] - ms1) * LOG2E);
      l0 += p0 + p1; l1 += p2 + p3;   // the softmax denominator counts every key; dropout acts on the probabilities
      if (drop.on) {
        const uint32_t kp = keep_qk(drop, b, h, i0, kt * TILE + j * 8, lane);
        p0 = (kp & 1u) ? p0 * drop.inv_keep : 0.f;
        p1 = (kp & 2u) ? p1 * drop.inv_keep : 0.f;
        p2 = (kp & 4u) ? p2 * drop.inv_keep : 0.f;
        p3 = (kp & 8u) ? p3 * drop.inv_keep : 0.f;
      }
      pf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0, p1);
      pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int dp = 0; dp < 4; ++dp) {
        uint32_t bf[4];
        load_b_frag_kn(vt_s, kk * 16, dp, lane, bf);
        mma_bf16(o[2 * dp], pf[kk], bf[0], bf[1]);
        mma_bf16(o[2 * dp + 1], pf[kk], bf[2], bf[3]);
      }
    }
    __syncthreads();   // this stage is refilled by the next iteration
    kt = next;
  }
  cp_async_wait<0>();   // a sample without a valid key issued its q tile only

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  // a sample without any valid key: NaN rows, as the L <= 128 kernel gives them
  const float i0v = l0 > 0.f ? 1.f / l0 : __int_as_float(0x7fc00000), i1v = l1 > 0.f ? 1.f / l1 : __int_as_float(0x7fc00000);
  const int q0 = i0 + gq, q1 = i0 + gq + 8;
  if (q0 < L) {
    bf16* dst = out + ((long long)b * L + q0) * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(o[j][0] * i0v, o[j][1] * i0v);
    if (t == 0) lse[((long long)b * H + h) * L + q0] = l0 > 0.f ? m0 + logf(l0) : __int_as_float(0x7fc00000);
  }
  if (q1 < L) {
    bf16* dst = out + ((long long)b * L + q1) * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(o[j][2] * i1v, o[j][3] * i1v);
    if (t == 0) lse[((long long)b * H + h) * L + q1] = l1 > 0.f ? m1 + logf(l1) : __int_as_float(0x7fc00000);
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward 1: delta[b, h, i] = sum_d dO[b*L + i, h*64 + d] * O[b*L + i, h*64 + d]   (8 threads per (row, head))
// ------------------------------------------------------------------------------------------------------------
__global__ void text_attn_long_delta_kernel(const bf16* __restrict__ out, const bf16* __restrict__ dout,
                                            float* __restrict__ delta, int B, int L, int H) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long rh = g >> 3;
  const int c = (int)(g & 7);
  const bool ok = rh < (long long)B * L * H;
  float d = 0.f;
  if (ok) {
    const long long off = rh * HD + c * 8;   // row-major [B*L, H*64]: (row, head) pairs are consecutive 64-blocks
    const uint4 ov = *reinterpret_cast<const uint4*>(out + off), dv = *reinterpret_cast<const uint4*>(dout + off);
    const uint32_t ou[4] = {ov.x, ov.y, ov.z, ov.w}, du[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 a = unpack_bf16x2(ou[i]), e = unpack_bf16x2(du[i]);
      d += a.x * e.x + a.y * e.y;
    }
  }
  d += __shfl_xor_sync(0xffffffffu, d, 1); d += __shfl_xor_sync(0xffffffffu, d, 2); d += __shfl_xor_sync(0xffffffffu, d, 4);
  if (ok && c == 0) {
    const int h = (int)(rh % H);
    const long long row = rh / H, b = row / L, i = row % L;
    delta[(b * H + h) * L + i] = d;
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward 2: dK, dV of one 64-key tile; grid (ceil(L / 64), H, B).  Each warp owns 16 keys and walks every query
// tile (padded query rows attend too) in 32-query chunks: S^T = K Q^T, dP^T = V dO^T.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
text_attn_long_bwd_kv_kernel(const bf16* __restrict__ qkv, const long long* __restrict__ mask,
                             const float* __restrict__ lse, const float* __restrict__ delta,
                             const bf16* __restrict__ dout, bf16* __restrict__ dqkv, int L, int H, float p_drop,
                             unsigned long long seed, uint32_t site) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint32_t kb[MAX_L / 32];
  __shared__ float s_lse[2][TILE], s_del[2][TILE];
  const uint32_t sk = smem_u32(smem), sv = sk + TILE_BYTES, sq = sv + TILE_BYTES, sdo = sq + 2 * TILE_BYTES;
  const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z, D = H * HD;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const Drop drop = make_drop(p_drop, seed, site);
  const int k0r = warp * 16, j0 = kt * TILE + k0r;

  const uint32_t tiles = key_bitmap(mask, b, L, kb);
  if (!((tiles >> kt) & 1u)) {   // no valid key in this tile: dK = dV = 0
    for (int idx = threadIdx.x; idx < TILE * 16; idx += NTHREADS) {
      const int r = idx >> 4, c = idx & 15, row = kt * TILE + r;
      if (row < L)
        *reinterpret_cast<uint4*>(dqkv + ((long long)b * L + row) * 3 * D + (1 + (c >> 3)) * D + h * HD + (c & 7) * 8) =
            make_uint4(0u, 0u, 0u, 0u);
    }
    return;
  }
  const int nqt = (L + TILE - 1) / TILE;
  auto load_q = [&](int qt, int st) {
    load_tile(sq + st * TILE_BYTES, qkv, 3 * D, h * HD, b, L, qt * TILE);
    load_tile(sdo + st * TILE_BYTES, dout, D, h * HD, b, L, qt * TILE);
    if (threadIdx.x < TILE) {
      const int i = qt * TILE + threadIdx.x;
      const long long o = ((long long)b * H + h) * L + i;
      s_lse[st][threadIdx.x] = i < L ? lse[o] * LOG2E : INFINITY;   // +inf: query rows >= L get P = 0
      s_del[st][threadIdx.x] = i < L ? delta[o] : 0.f;
    }
  };
  load_tile(sk, qkv, 3 * D, D + h * HD, b, L, kt * TILE);
  load_tile(sv, qkv, 3 * D, 2 * D + h * HD, b, L, kt * TILE);
  load_q(0, 0);
  cp_async_commit();
  const bool kv0 = key_ok(kb, j0 + gq), kv1 = key_ok(kb, j0 + gq + 8);

  float dk[8][4], dv[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) { dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = 0.f; dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f; }

  for (int qt = 0; qt < nqt; ++qt) {
    const int st = qt & 1;
    if (qt + 1 < nqt) {
      load_q(qt + 1, st ^ 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const uint32_t q_s = sq + st * TILE_BYTES, do_s = sdo + st * TILE_BYTES;
#pragma unroll 1
    for (int c0 = 0; c0 < 8; c0 += 4) {   // 32 queries
      float s[4][4], dp[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; dp[j][0] = dp[j][1] = dp[j][2] = dp[j][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        uint32_t af[4], bf[4];
        load_a_frag(sk, k0r, kk, lane, af);
#pragma unroll
        for (int p = 0; p < 2; ++p) {
          load_b_frag_nk(q_s, (c0 + 2 * p) * 8, kk, lane, bf);
          mma_bf16(s[2 * p], af, bf[0], bf[1]);
          mma_bf16(s[2 * p + 1], af, bf[2], bf[3]);
        }
        load_a_frag(sv, k0r, kk, lane, af);
#pragma unroll
        for (int p = 0; p < 2; ++p) {
          load_b_frag_nk(do_s, (c0 + 2 * p) * 8, kk, lane, bf);
          mma_bf16(dp[2 * p], af, bf[0], bf[1]);
          mma_bf16(dp[2 * p + 1], af, bf[2], bf[3]);
        }
      }
      uint32_t pf[2][4], dsf[2][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = (c0 + j) * 8 + 2 * t;   // query within the tile
        const float lq0 = s_lse[st][col], lq1 = s_lse[st][col + 1], dq0 = s_del[st][col], dq1 = s_del[st][col + 1];
        const float p0 = kv0 ? exp2f(s[j][0] * LOG2E - lq0) : 0.f;
        const float p1 = kv0 ? exp2f(s[j][1] * LOG2E - lq1) : 0.f;
        const float p2 = kv1 ? exp2f(s[j][2] * LOG2E - lq0) : 0.f;
        const float p3 = kv1 ? exp2f(s[j][3] * LOG2E - lq1) : 0.f;
        float pd0 = p0, pd1 = p1, pd2 = p2, pd3 = p3;
        float g0 = dp[j][0], g1 = dp[j][1], g2 = dp[j][2], g3 = dp[j][3];
        if (drop.on) {
          const uint32_t kp = keep_kq(drop, b, h, j0, qt * TILE + (c0 + j) * 8, lane);
          const float k0 = (kp & 1u) ? drop.inv_keep : 0.f, k1 = (kp & 2u) ? drop.inv_keep : 0.f;
          const float k2 = (kp & 4u) ? drop.inv_keep : 0.f, k3 = (kp & 8u) ? drop.inv_keep : 0.f;
          pd0 *= k0; pd1 *= k1; pd2 *= k2; pd3 *= k3;
          g0 *= k0; g1 *= k1; g2 *= k2; g3 *= k3;
        }
        pf[j >> 1][(j & 1) * 2] = pack_bf16x2(pd0, pd1);
        pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(pd2, pd3);
        dsf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0 * (g0 - dq0), p1 * (g1 - dq1));
        dsf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2 * (g2 - dq0), p3 * (g3 - dq1));
      }
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        const int q0r = (c0 + 2 * kk) * 8;
#pragma unroll
        for (int dpi = 0; dpi < 4; ++dpi) {
          uint32_t bf[4];
          load_b_frag_kn(do_s, q0r, dpi, lane, bf);
          mma_bf16(dv[2 * dpi], pf[kk], bf[0], bf[1]);
          mma_bf16(dv[2 * dpi + 1], pf[kk], bf[2], bf[3]);
          load_b_frag_kn(q_s, q0r, dpi, lane, bf);
          mma_bf16(dk[2 * dpi], dsf[kk], bf[0], bf[1]);
          mma_bf16(dk[2 * dpi + 1], dsf[kk], bf[2], bf[3]);
        }
      }
    }
    __syncthreads();   // this stage is refilled by the next iteration
  }
  const int r0 = j0 + gq, r1 = j0 + gq + 8;
  if (r0 < L) {
    bf16* dst = dqkv + ((long long)b * L + r0) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(dst + D + j * 8) = pack_bf16x2(dk[j][0], dk[j][1]);
      *reinterpret_cast<uint32_t*>(dst + 2 * D + j * 8) = pack_bf16x2(dv[j][0], dv[j][1]);
    }
  }
  if (r1 < L) {
    bf16* dst = dqkv + ((long long)b * L + r1) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(dst + D + j * 8) = pack_bf16x2(dk[j][2], dk[j][3]);
      *reinterpret_cast<uint32_t*>(dst + 2 * D + j * 8) = pack_bf16x2(dv[j][2], dv[j][3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward 3: dQ of one 64-query tile over the valid key tiles; grid (ceil(L / 64), H, B)
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
text_attn_long_bwd_q_kernel(const bf16* __restrict__ qkv, const long long* __restrict__ mask,
                            const float* __restrict__ lse, const float* __restrict__ delta,
                            const bf16* __restrict__ dout, bf16* __restrict__ dqkv, int L, int H, float q_scale,
                            float p_drop, unsigned long long seed, uint32_t site) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint32_t kb[MAX_L / 32];
  const uint32_t sq = smem_u32(smem), sdo = sq + TILE_BYTES, sk = sdo + TILE_BYTES, sv = sk + 2 * TILE_BYTES;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z, D = H * HD;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const Drop drop = make_drop(p_drop, seed, site);
  const int r0 = warp * 16, i0 = qt * TILE + r0, q0 = i0 + gq, q1 = q0 + 8;

  load_tile(sq, qkv, 3 * D, h * HD, b, L, qt * TILE);
  load_tile(sdo, dout, D, h * HD, b, L, qt * TILE);
  uint32_t tiles = key_bitmap(mask, b, L, kb);
  int kt = tiles ? __ffs(tiles) - 1 : -1;
  if (kt >= 0) {
    load_tile(sk, qkv, 3 * D, D + h * HD, b, L, kt * TILE);
    load_tile(sv, qkv, 3 * D, 2 * D + h * HD, b, L, kt * TILE);
    tiles &= tiles - 1;
  }
  cp_async_commit();
  const long long ro = ((long long)b * H + h) * L;
  const float ls0 = q0 < L ? lse[ro + q0] * LOG2E : 0.f, ls1 = q1 < L ? lse[ro + q1] * LOG2E : 0.f;
  const float de0 = q0 < L ? delta[ro + q0] : 0.f, de1 = q1 < L ? delta[ro + q1] : 0.f;

  float dq[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) { dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f; }

  for (int stage = 0; kt >= 0; stage ^= 1) {
    const int next = tiles ? __ffs(tiles) - 1 : -1;
    if (next >= 0) {
      load_tile(sk + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, D + h * HD, b, L, next * TILE);
      load_tile(sv + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, 2 * D + h * HD, b, L, next * TILE);
      tiles &= tiles - 1;
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const uint32_t k_s = sk + stage * TILE_BYTES, v_s = sv + stage * TILE_BYTES;
#pragma unroll 1
    for (int c0 = 0; c0 < 8; c0 += 4) {   // 32 keys
      float s[4][4], dp[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; dp[j][0] = dp[j][1] = dp[j][2] = dp[j][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        uint32_t af[4], bf[4];
        load_a_frag(sq, r0, kk, lane, af);
#pragma unroll
        for (int p = 0; p < 2; ++p) {
          load_b_frag_nk(k_s, (c0 + 2 * p) * 8, kk, lane, bf);
          mma_bf16(s[2 * p], af, bf[0], bf[1]);
          mma_bf16(s[2 * p + 1], af, bf[2], bf[3]);
        }
        load_a_frag(sdo, r0, kk, lane, af);
#pragma unroll
        for (int p = 0; p < 2; ++p) {
          load_b_frag_nk(v_s, (c0 + 2 * p) * 8, kk, lane, bf);
          mma_bf16(dp[2 * p], af, bf[0], bf[1]);
          mma_bf16(dp[2 * p + 1], af, bf[2], bf[3]);
        }
      }
      uint32_t dsf[2][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int jl = (c0 + j) * 8;   // key within the tile
        const uint32_t bits = kb[2 * kt + (jl >> 5)] >> ((jl & 31) + 2 * t);
        const float p0 = (bits & 1u) ? exp2f(s[j][0] * LOG2E - ls0) : 0.f;
        const float p1 = (bits & 2u) ? exp2f(s[j][1] * LOG2E - ls0) : 0.f;
        const float p2 = (bits & 1u) ? exp2f(s[j][2] * LOG2E - ls1) : 0.f;
        const float p3 = (bits & 2u) ? exp2f(s[j][3] * LOG2E - ls1) : 0.f;
        float g0 = dp[j][0], g1 = dp[j][1], g2 = dp[j][2], g3 = dp[j][3];
        if (drop.on) {
          const uint32_t kp = keep_qk(drop, b, h, i0, kt * TILE + jl, lane);
          g0 = (kp & 1u) ? g0 * drop.inv_keep : 0.f;
          g1 = (kp & 2u) ? g1 * drop.inv_keep : 0.f;
          g2 = (kp & 4u) ? g2 * drop.inv_keep : 0.f;
          g3 = (kp & 8u) ? g3 * drop.inv_keep : 0.f;
        }
        dsf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0 * (g0 - de0), p1 * (g1 - de0));
        dsf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2 * (g2 - de1), p3 * (g3 - de1));
      }
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
        for (int dpi = 0; dpi < 4; ++dpi) {
          uint32_t bf[4];
          load_b_frag_kn(k_s, (c0 + 2 * kk) * 8, dpi, lane, bf);
          mma_bf16(dq[2 * dpi], dsf[kk], bf[0], bf[1]);
          mma_bf16(dq[2 * dpi + 1], dsf[kk], bf[2], bf[3]);
        }
      }
    }
    __syncthreads();   // this stage is refilled by the next iteration
    kt = next;
  }
  cp_async_wait<0>();
  if (q0 < L) {
    bf16* dst = dqkv + ((long long)b * L + q0) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(dq[j][0] * q_scale, dq[j][1] * q_scale);
  }
  if (q1 < L) {
    bf16* dst = dqkv + ((long long)b * L + q1) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(dq[j][2] * q_scale, dq[j][3] * q_scale);
  }
}

constexpr size_t FWD_SMEM = 5 * TILE_BYTES;   // q + two stages of k, v
constexpr size_t BWD_SMEM = 6 * TILE_BYTES;   // kv pass: k, v + two stages of q, dO;  q pass: q, dO + two of k, v

}  // namespace
}  // namespace egovlp

using namespace egovlp;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int egovlp_text_attn_long_fwd(const void* qkv, const long long* attention_mask, void* out, float* lse, int B,
                                         int L, int H, float p_drop, unsigned long long seed, unsigned int site,
                                         void* stream) {
  EGOVLP_CHECK_ARG(qkv && attention_mask && out && lse, "text_attn_long_fwd: null pointer");
  EGOVLP_CHECK_ARG(B > 0 && B <= 65535 && H > 0 && H <= 4096, "text_attn_long_fwd: B=%d H=%d unsupported", B, H);
  EGOVLP_CHECK_ARG(L > 0 && L <= MAX_L, "text_attn_long: L=%d unsupported (1..512)", L);
  EGOVLP_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, "text_attn_long: p_drop=%f outside [0, 1)", p_drop);
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(text_attn_long_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)FWD_SMEM));
  const dim3 grid((L + TILE - 1) / TILE, H, B);
  text_attn_long_fwd_kernel<<<grid, NTHREADS, FWD_SMEM, ST(stream)>>>(
      reinterpret_cast<const bf16*>(qkv), attention_mask, reinterpret_cast<bf16*>(out), lse, L, H, p_drop, seed, site);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

extern "C" int egovlp_text_attn_long_bwd(const void* qkv, const long long* attention_mask, const void* out,
                                         const float* lse, const void* dout, void* dqkv, float* workspace, int B,
                                         int L, int H, float q_scale, float p_drop, unsigned long long seed,
                                         unsigned int site, void* stream) {
  EGOVLP_CHECK_ARG(qkv && attention_mask && out && lse && dout && dqkv && workspace,
                   "text_attn_long_bwd: null pointer");
  EGOVLP_CHECK_ARG(B > 0 && B <= 65535 && H > 0 && H <= 4096, "text_attn_long_bwd: B=%d H=%d unsupported", B, H);
  EGOVLP_CHECK_ARG(L > 0 && L <= MAX_L, "text_attn_long: L=%d unsupported (1..512)", L);
  EGOVLP_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, "text_attn_long: p_drop=%f outside [0, 1)", p_drop);
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(text_attn_long_bwd_kv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)BWD_SMEM));
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(text_attn_long_bwd_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)BWD_SMEM));
  const bf16* q = reinterpret_cast<const bf16*>(qkv);
  const bf16* o = reinterpret_cast<const bf16*>(out);
  const bf16* g = reinterpret_cast<const bf16*>(dout);
  bf16* dq = reinterpret_cast<bf16*>(dqkv);
  const long long nthr = (long long)B * L * H * 8;
  text_attn_long_delta_kernel<<<(unsigned)((nthr + 255) / 256), 256, 0, ST(stream)>>>(o, g, workspace, B, L, H);
  EGOVLP_CHECK_LAUNCH();
  const dim3 grid((L + TILE - 1) / TILE, H, B);
  text_attn_long_bwd_kv_kernel<<<grid, NTHREADS, BWD_SMEM, ST(stream)>>>(q, attention_mask, lse, workspace, g, dq, L, H,
                                                                        p_drop, seed, site);
  EGOVLP_CHECK_LAUNCH();
  text_attn_long_bwd_q_kernel<<<grid, NTHREADS, BWD_SMEM, ST(stream)>>>(q, attention_mask, lse, workspace, g, dq, L, H,
                                                                       q_scale, p_drop, seed, site);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
