// Tiled, online-softmax attention on the tensor cores at head dim 64, forward and backward: the one implementation
// behind the long-caption text attention (text_attention.cu) and the large-frame spatial attention
// (space_attention.cu).
//
// A group is the set of rows that attend to one another: rows r = 0 .. rows - 1 are its queries and its keys alike.
// Tiling: one CTA (4 warps, 16 rows each) per (64-row tile, head, blockIdx.z); the other operand streams through a
// two-stage cp.async ring of 64-row tiles; tile rows past the group are zero-filled by the copy (src-size 0), so a tile
// never reads another group's rows, and their results are never stored.
// Math: bf16 mma.sync m16n8k16 with fp32 accumulation, fp32 online softmax in exp2 (as the divided attention).
//
// Backward, with no floating-point atomics (bitwise reproducible run to run):
//   1. row pass:   delta_i = sum_d dO_id * O_id                                  -> fp32 [B, H, S rows a sample]
//   2. key pass:   per 64-key tile, dV = P'^T dO and dK = dS^T Q over the group's query tiles, P recomputed from lse
//   3. query pass: per 64-query tile, dQ = q_scale * dS K over the group's key tiles
// where P' = P * keep / (1 - p) and dS = P * (dP' - delta), dP' = (dO V^T) * keep / (1 - p) (keep = 1 without dropout).
//
// A user describes its groups with a layout policy P, a class the kernels construct per CTA from their argument
// P::Args (which holds H), the head blockIdx.y and a P::Smem in static shared memory:
//   rows, row(r)          the group's row count and the matrix row (of qkv, out, dout, dqkv) that holds row r
//   stat(r)               row r's entry of lse and delta
//   key_tiles()           bit kt set: the passes visit 64-key tile kt (the key pass writes zero dK, dV for the others)
//   masked(kt)            the forward applies key_bits() on tile kt (the query pass does on every tile)
//   key_bits(kt, jl, t)   bits 0, 1: keys kt*64 + jl + 2t and kt*64 + jl + 2t + 1 are attended
//   key_ok(j)             key j is attended
//   skips_pair00()        query row 0 does not attend key row 0 in this group
//   kCls                  row 0's results go to fp32 partials through cls_fwd / cls_dkv / cls_dq instead of its rows
//   kDropout              attention dropout: drop.{on, inv_keep} and the keep bits keep_qk / keep_kq
// A row that attends no key gets NaN out and lse.
#pragma once
#include "common.cuh"

namespace egovlp {
namespace {

constexpr int HD = 64;
constexpr int TILE = 64;                   // rows per tile (queries or keys)
constexpr int NTHREADS = 128;              // 4 warps x 16 rows
constexpr int TILE_BYTES = TILE * HD * 2;  // one 64 x 64 bf16 tile
constexpr float LOG2E = 1.4426950408889634f;
constexpr size_t FWD_SMEM = 5 * TILE_BYTES;   // q + two stages of k, v
constexpr size_t BWD_SMEM = 6 * TILE_BYTES;   // kv pass: k, v + two stages of q, dO;  q pass: q, dO + two of k, v

// ---- cp.async ----
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// rows r0 .. r0 + 63 of the group x 64 bf16 columns at column col of a matrix with row stride ld -> swizzled tile;
// rows past the group are zero-filled and their addresses never read
template <class P>
__device__ __forceinline__ void load_tile(uint32_t tile, const bf16* base, long long ld, int col, const P& g, int r0) {
  for (int idx = threadIdx.x; idx < TILE * 8; idx += NTHREADS) {
    const int r = idx >> 3, c = idx & 7, row = r0 + r;
    const bool valid = row < g.rows;
    const bf16* src = base + g.row(valid ? row : 0) * ld + col + c * 8;
    cp_async16(sw_addr(tile, r, c), src, valid);
  }
}

// ------------------------------------------------------------------------------------------------------------
// forward: grid (ceil(rows / 64), H, groups / H)
// ------------------------------------------------------------------------------------------------------------
template <class P>
__global__ void __launch_bounds__(NTHREADS)
tiled_attn_fwd_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ out, float* __restrict__ lse,
                      const typename P::Args a) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ typename P::Smem psm;
  const uint32_t sq = smem_u32(smem), sk = sq + TILE_BYTES, sv = sk + 2 * TILE_BYTES;   // k, v: two stages each
  const int qt = blockIdx.x, h = blockIdx.y, D = a.H * HD;
  const P g(a, h, psm);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  // query row 0 is warp 0, lane 0's first row; key row 0 is column 0 of the first key tile
  const bool skip00 = g.skips_pair00() && qt == 0 && warp == 0 && lane == 0;

  load_tile(sq, qkv, 3 * D, h * HD, g, qt * TILE);
  uint32_t tiles = g.key_tiles();
  int kt = tiles ? __ffs(tiles) - 1 : -1;
  if (kt >= 0) {
    load_tile(sk, qkv, 3 * D, D + h * HD, g, kt * TILE);
    load_tile(sv, qkv, 3 * D, 2 * D + h * HD, g, kt * TILE);
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
      load_tile(sk + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, D + h * HD, g, next * TILE);
      load_tile(sv + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, 2 * D + h * HD, g, next * TILE);
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
    if (kt == 0 && skip00) s[0][0] = -INFINITY;
    const bool masked = g.masked(kt);
    float cm0 = -INFINITY, cm1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (masked) {
        const uint32_t bits = g.key_bits(kt, j * 8, t);
        if (!(bits & 1u)) s[j][0] = s[j][2] = -INFINITY;
        if (!(bits & 2u)) s[j][1] = s[j][3] = -INFINITY;
      }
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
      if constexpr (P::kDropout) {
        if (g.drop.on) {
          const uint32_t kp = g.keep_qk(i0, kt * TILE + j * 8, lane);
          p0 = (kp & 1u) ? p0 * g.drop.inv_keep : 0.f;
          p1 = (kp & 2u) ? p1 * g.drop.inv_keep : 0.f;
          p2 = (kp & 4u) ? p2 * g.drop.inv_keep : 0.f;
          p3 = (kp & 8u) ? p3 * g.drop.inv_keep : 0.f;
        }
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
  cp_async_wait<0>();   // a group without a key tile issued its q tile only

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0v = l0 > 0.f ? 1.f / l0 : __int_as_float(0x7fc00000), i1v = l1 > 0.f ? 1.f / l1 : __int_as_float(0x7fc00000);
  const int q0 = i0 + gq, q1 = i0 + gq + 8;
  const bool cls = P::kCls && q0 == 0;
  if constexpr (P::kCls) {
    if (cls) g.cls_fwd(o, m0, l0, t);
  }
  if (!cls && q0 < g.rows) {
    bf16* dst = out + g.row(q0) * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(o[j][0] * i0v, o[j][1] * i0v);
    if (t == 0) lse[g.stat(q0)] = l0 > 0.f ? m0 + logf(l0) : __int_as_float(0x7fc00000);
  }
  if (q1 < g.rows) {
    bf16* dst = out + g.row(q1) * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(o[j][2] * i1v, o[j][3] * i1v);
    if (t == 0) lse[g.stat(q1)] = l1 > 0.f ? m1 + logf(l1) : __int_as_float(0x7fc00000);
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward 1: delta[b, h, i] = sum_d dO[b*S + i, h*64 + d] * O[b*S + i, h*64 + d] over the rows * H (row, head) pairs
// of a [rows, H*64] matrix, S rows a sample   (8 threads per (row, head))
// ------------------------------------------------------------------------------------------------------------
__global__ void tiled_attn_delta_kernel(const bf16* __restrict__ out, const bf16* __restrict__ dout,
                                        float* __restrict__ delta, long long rows, int S, int H) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long rh = g >> 3;
  const int c = (int)(g & 7);
  const bool ok = rh < rows * H;
  float d = 0.f;
  if (ok) {
    const long long off = rh * HD + c * 8;   // row-major [rows, H*64]: (row, head) pairs are consecutive 64-blocks
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
    const long long row = rh / H, b = row / S, i = row - b * S;
    delta[(b * H + h) * S + i] = d;
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward 2: dK, dV of one 64-key tile; grid (ceil(rows / 64), H, groups / H).  Each warp owns 16 keys and walks
// every query tile of the group (query rows that attend no key too) in 32-query chunks: S^T = K Q^T, dP^T = V dO^T.
// ------------------------------------------------------------------------------------------------------------
template <class P>
__global__ void __launch_bounds__(NTHREADS)
tiled_attn_bwd_kv_kernel(const bf16* __restrict__ qkv, const float* __restrict__ lse, const float* __restrict__ delta,
                         const bf16* __restrict__ dout, bf16* __restrict__ dqkv, const typename P::Args a) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ typename P::Smem psm;
  __shared__ float s_lse[2][TILE], s_del[2][TILE];
  const uint32_t sk = smem_u32(smem), sv = sk + TILE_BYTES, sq = sv + TILE_BYTES, sdo = sq + 2 * TILE_BYTES;
  const int kt = blockIdx.x, h = blockIdx.y, D = a.H * HD;
  const P g(a, h, psm);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int k0r = warp * 16, j0 = kt * TILE + k0r;
  // key row 0 is warp 0, lane 0's first row; query row 0 is column 0 of the first query tile
  const bool skip00 = g.skips_pair00() && kt == 0 && warp == 0 && lane == 0;

  if (!((g.key_tiles() >> kt) & 1u)) {   // no attended key in this tile: dK = dV = 0
    for (int idx = threadIdx.x; idx < TILE * 16; idx += NTHREADS) {
      const int r = idx >> 4, c = idx & 15, row = kt * TILE + r;
      if (row < g.rows)
        *reinterpret_cast<uint4*>(dqkv + g.row(row) * 3 * D + (1 + (c >> 3)) * D + h * HD + (c & 7) * 8) =
            make_uint4(0u, 0u, 0u, 0u);
    }
    return;
  }
  const int nqt = (g.rows + TILE - 1) / TILE;
  auto load_q = [&](int qt, int st) {
    load_tile(sq + st * TILE_BYTES, qkv, 3 * D, h * HD, g, qt * TILE);
    load_tile(sdo + st * TILE_BYTES, dout, D, h * HD, g, qt * TILE);
    if (threadIdx.x < TILE) {
      const int i = qt * TILE + threadIdx.x;
      const bool ok = i < g.rows;
      s_lse[st][threadIdx.x] = ok ? lse[g.stat(i)] * LOG2E : INFINITY;   // +inf: rows past the group get P = 0
      s_del[st][threadIdx.x] = ok ? delta[g.stat(i)] : 0.f;
    }
  };
  load_tile(sk, qkv, 3 * D, D + h * HD, g, kt * TILE);
  load_tile(sv, qkv, 3 * D, 2 * D + h * HD, g, kt * TILE);
  load_q(0, 0);
  cp_async_commit();
  const bool kv0 = g.key_ok(j0 + gq), kv1 = g.key_ok(j0 + gq + 8);

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
        const bool pair00 = skip00 && qt == 0 && c0 == 0 && j == 0;
        const float p0 = kv0 && !pair00 ? exp2f(s[j][0] * LOG2E - lq0) : 0.f;
        const float p1 = kv0 ? exp2f(s[j][1] * LOG2E - lq1) : 0.f;
        const float p2 = kv1 ? exp2f(s[j][2] * LOG2E - lq0) : 0.f;
        const float p3 = kv1 ? exp2f(s[j][3] * LOG2E - lq1) : 0.f;
        float pd0 = p0, pd1 = p1, pd2 = p2, pd3 = p3;
        float g0 = dp[j][0], g1 = dp[j][1], g2 = dp[j][2], g3 = dp[j][3];
        if constexpr (P::kDropout) {
          if (g.drop.on) {
            const uint32_t kp = g.keep_kq(j0, qt * TILE + (c0 + j) * 8, lane);
            const float k0 = (kp & 1u) ? g.drop.inv_keep : 0.f, k1 = (kp & 2u) ? g.drop.inv_keep : 0.f;
            const float k2 = (kp & 4u) ? g.drop.inv_keep : 0.f, k3 = (kp & 8u) ? g.drop.inv_keep : 0.f;
            pd0 *= k0; pd1 *= k1; pd2 *= k2; pd3 *= k3;
            g0 *= k0; g1 *= k1; g2 *= k2; g3 *= k3;
          }
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
  const bool cls = P::kCls && r0 == 0;
  if constexpr (P::kCls) {
    if (cls) g.cls_dkv(dk, dv, t);
  }
  if (!cls && r0 < g.rows) {
    bf16* dst = dqkv + g.row(r0) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(dst + D + j * 8) = pack_bf16x2(dk[j][0], dk[j][1]);
      *reinterpret_cast<uint32_t*>(dst + 2 * D + j * 8) = pack_bf16x2(dv[j][0], dv[j][1]);
    }
  }
  if (r1 < g.rows) {
    bf16* dst = dqkv + g.row(r1) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(dst + D + j * 8) = pack_bf16x2(dk[j][2], dk[j][3]);
      *reinterpret_cast<uint32_t*>(dst + 2 * D + j * 8) = pack_bf16x2(dv[j][2], dv[j][3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward 3: dQ of one 64-query tile over the group's key tiles; grid (ceil(rows / 64), H, groups / H)
// ------------------------------------------------------------------------------------------------------------
template <class P>
__global__ void __launch_bounds__(NTHREADS)
tiled_attn_bwd_q_kernel(const bf16* __restrict__ qkv, const float* __restrict__ lse, const float* __restrict__ delta,
                        const bf16* __restrict__ dout, bf16* __restrict__ dqkv, float q_scale,
                        const typename P::Args a) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ typename P::Smem psm;
  const uint32_t sq = smem_u32(smem), sdo = sq + TILE_BYTES, sk = sdo + TILE_BYTES, sv = sk + 2 * TILE_BYTES;
  const int qt = blockIdx.x, h = blockIdx.y, D = a.H * HD;
  const P g(a, h, psm);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int r0 = warp * 16, i0 = qt * TILE + r0, q0 = i0 + gq, q1 = q0 + 8;
  const bool skip00 = g.skips_pair00() && qt == 0 && warp == 0 && lane == 0;

  load_tile(sq, qkv, 3 * D, h * HD, g, qt * TILE);
  load_tile(sdo, dout, D, h * HD, g, qt * TILE);
  uint32_t tiles = g.key_tiles();
  int kt = tiles ? __ffs(tiles) - 1 : -1;
  if (kt >= 0) {
    load_tile(sk, qkv, 3 * D, D + h * HD, g, kt * TILE);
    load_tile(sv, qkv, 3 * D, 2 * D + h * HD, g, kt * TILE);
    tiles &= tiles - 1;
  }
  cp_async_commit();
  const float ls0 = q0 < g.rows ? lse[g.stat(q0)] * LOG2E : 0.f;
  const float ls1 = q1 < g.rows ? lse[g.stat(q1)] * LOG2E : 0.f;
  const float de0 = q0 < g.rows ? delta[g.stat(q0)] : 0.f;
  const float de1 = q1 < g.rows ? delta[g.stat(q1)] : 0.f;

  float dq[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) { dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f; }

  for (int stage = 0; kt >= 0; stage ^= 1) {
    const int next = tiles ? __ffs(tiles) - 1 : -1;
    if (next >= 0) {
      load_tile(sk + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, D + h * HD, g, next * TILE);
      load_tile(sv + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, 2 * D + h * HD, g, next * TILE);
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
        const uint32_t bits = g.key_bits(kt, jl, t);
        const bool pair00 = skip00 && kt == 0 && c0 == 0 && j == 0;
        const float p0 = (bits & 1u) && !pair00 ? exp2f(s[j][0] * LOG2E - ls0) : 0.f;
        const float p1 = (bits & 2u) ? exp2f(s[j][1] * LOG2E - ls0) : 0.f;
        const float p2 = (bits & 1u) ? exp2f(s[j][2] * LOG2E - ls1) : 0.f;
        const float p3 = (bits & 2u) ? exp2f(s[j][3] * LOG2E - ls1) : 0.f;
        float g0 = dp[j][0], g1 = dp[j][1], g2 = dp[j][2], g3 = dp[j][3];
        if constexpr (P::kDropout) {
          if (g.drop.on) {
            const uint32_t kp = g.keep_qk(i0, kt * TILE + jl, lane);
            g0 = (kp & 1u) ? g0 * g.drop.inv_keep : 0.f;
            g1 = (kp & 2u) ? g1 * g.drop.inv_keep : 0.f;
            g2 = (kp & 4u) ? g2 * g.drop.inv_keep : 0.f;
            g3 = (kp & 8u) ? g3 * g.drop.inv_keep : 0.f;
          }
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
  const bool cls = P::kCls && q0 == 0;
  if constexpr (P::kCls) {
    if (cls) g.cls_dq(dq, t);
  }
  if (!cls && q0 < g.rows) {
    bf16* dst = dqkv + g.row(q0) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(dq[j][0] * q_scale, dq[j][1] * q_scale);
  }
  if (q1 < g.rows) {
    bf16* dst = dqkv + g.row(q1) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(dq[j][2] * q_scale, dq[j][3] * q_scale);
  }
}

}  // namespace
}  // namespace egovlp
