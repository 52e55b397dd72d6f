// Spatial attention of the video tower for large frames (model/video_transformer.py:109-130, space mode): tiled,
// online-softmax attention on the tensor cores, forward and backward, for 1 <= N <= 1024 patches per frame.  The
// divided attention (attention.cu) holds a whole frame in one CTA and stops at N = 255; the engine calls these kernels
// above that.
//
// Same contract as egovlp_divided_attn_* with mode = 1: qkv bf16 [B*S, 3D] read in place (q pre-scaled), S = 1 + T*N,
// row 1 + f*N + n = patch n of frame f, row 0 = the sample's CLS token; out bf16 [B*S, D] with the heads merged, lse
// fp32 [B, H, S].  Head dim 64.
//
// A group is (b, head, frame).  Its rows are indexed r = 0 .. N: r = 0 is the CLS token, r = 1 + n patch n of the frame.
// Queries and keys share that index, so the CLS key is the extra key ahead of the frame's first 64-key tile and the CLS
// query the extra query ahead of its first 64-query tile.  Every pair (r, j) with r, j <= N is attended except the CLS
// query on the CLS key in frames f > 0: over the T groups the CLS query then sees every key of the sample once.
//
// Tiling: one CTA (4 warps, 16 rows each) per (64-row tile, head, frame of a sample); the other operand streams
// through a two-stage cp.async ring of 64-row tiles; rows past N are zero-filled by the copy and masked.
// Math: bf16 mma.sync m16n8k16 with fp32 accumulation, fp32 online softmax in exp2 (as the divided attention).
//
// The CLS rows, with no floating-point atomics (everything is bitwise reproducible run to run):
//   forward:  each group writes the CLS query's un-normalised (max, sum, acc) partial; space_cls_merge_kernel merges
//             the T partials of a (b, head) in frame order and writes out row 0 and lse[b, h, 0];
//   backward: each group writes its fp32 partial of the CLS row's dq, dk and dv; space_cls_grad_kernel sums the T
//             partials in frame order.
// Backward: 1. row pass  delta_i = sum_d dO_id O_id for every row (CLS included)   -> workspace fp32 [B, H, S]
//           2. key pass  per 64-key tile, dV = P^T dO and dK = dS^T Q over the group's query tiles
//           3. query pass per 64-query tile, dQ = q_scale dS K over the group's key tiles
// with P recomputed from lse (the CLS query's lse is the merged one, over all S keys) and dS = P (dP - delta).
#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

constexpr int HD = 64;
constexpr int TILE = 64;                   // rows per tile (queries or keys)
constexpr int MAX_N = 1024;
constexpr int NTHREADS = 128;              // 4 warps x 16 rows
constexpr int TILE_BYTES = TILE * HD * 2;  // one 64 x 64 bf16 tile
constexpr int PART = 66;                   // CLS-query partial: acc[64], max, sum
constexpr float LOG2E = 1.4426950408889634f;

// ---- cp.async ----
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Where a group's rows live: row r of group (b, f) is matrix row  r ? fN + r : bS  (bS = b*S, fN = b*S + f*N), and
// entry  r ? fn + r : 0  of the sample's [S] slice of lse / delta (fn = f*N).
struct Grp {
  long long bS, fN;
  int fn, f, rows;   // rows = N + 1
};
__device__ __forceinline__ Grp make_grp(int bf, int T, int N) {
  const int b = bf / T, f = bf - b * T;
  const long long bS = (long long)b * (1 + (long long)T * N);
  return Grp{bS, bS + (long long)f * N, f * N, f, N + 1};
}
__device__ __forceinline__ long long grp_row(const Grp& g, int r) { return r ? g.fN + r : g.bS; }
__device__ __forceinline__ int grp_tok(const Grp& g, int r) { return r ? g.fn + r : 0; }

// rows r0 .. r0 + 63 of the group x 64 bf16 columns at column col of a matrix with row stride ld -> swizzled tile;
// rows past the group are zero-filled and their addresses never read
__device__ __forceinline__ void load_tile(uint32_t tile, const bf16* base, long long ld, int col, const Grp& g,
                                          int r0) {
  for (int idx = threadIdx.x; idx < TILE * 8; idx += NTHREADS) {
    const int r = idx >> 3, c = idx & 7, row = r0 + r;
    const bool valid = row < g.rows;
    const bf16* src = base + grp_row(g, valid ? row : 0) * ld + col + c * 8;
    cp_async16(sw_addr(tile, r, c), src, valid);
  }
}

// ------------------------------------------------------------------------------------------------------------
// forward: grid (ceil((N + 1) / 64), H, B*T)
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
space_attn_long_fwd_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ out, float* __restrict__ lse,
                           float* __restrict__ cls_part, int T, int N, int H) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sq = smem_u32(smem), sk = sq + TILE_BYTES, sv = sk + 2 * TILE_BYTES;   // k, v: two stages each
  const int qt = blockIdx.x, h = blockIdx.y, D = H * HD, S = 1 + T * N;
  const Grp g = make_grp(blockIdx.z, T, N);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int nt = (g.rows + TILE - 1) / TILE;
  // the CLS query (row 0: warp 0, lane 0's first row) skips the CLS key (column 0) in every frame but the first
  const bool skip_cls_key = qt == 0 && warp == 0 && lane == 0 && g.f > 0;

  load_tile(sq, qkv, 3 * D, h * HD, g, qt * TILE);
  load_tile(sk, qkv, 3 * D, D + h * HD, g, 0);
  load_tile(sv, qkv, 3 * D, 2 * D + h * HD, g, 0);
  cp_async_commit();

  const int r0 = warp * 16, i0 = qt * TILE + r0;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }

  for (int kt = 0; kt < nt; ++kt) {
    const int stage = kt & 1;
    if (kt + 1 < nt) {
      load_tile(sk + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, D + h * HD, g, (kt + 1) * TILE);
      load_tile(sv + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, 2 * D + h * HD, g, (kt + 1) * TILE);
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
    if (kt == nt - 1) {   // keys past the group
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = kt * TILE + j * 8 + 2 * t;
        if (c >= g.rows) s[j][0] = s[j][2] = -INFINITY;
        if (c + 1 >= g.rows) s[j][1] = s[j][3] = -INFINITY;
      }
    }
    if (kt == 0 && skip_cls_key) s[0][0] = -INFINITY;
    float cm0 = -INFINITY, cm1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
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
      const float p0 = exp2f((s[j][0] - ms0) * LOG2E), p1 = exp2f((s[j][1] - ms0) * LOG2E);
      const float p2 = exp2f((s[j][2] - ms1) * LOG2E), p3 = exp2f((s[j][3] - ms1) * LOG2E);
      l0 += p0 + p1; l1 += p2 + p3;
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
  }

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const int q0 = i0 + gq, q1 = i0 + gq + 8;
  const long long lrow = ((long long)blockIdx.z / T * H + h) * S;   // this (b, h)'s lse slice
  if (q0 == 0) {   // the CLS query: un-normalised partial for space_cls_merge_kernel
    float* dst = cls_part + (((long long)blockIdx.z / T * H + h) * T + g.f) * PART;
#pragma unroll
    for (int j = 0; j < 8; ++j) { dst[j * 8 + 2 * t] = o[j][0]; dst[j * 8 + 2 * t + 1] = o[j][1]; }
    if (t == 0) { dst[64] = m0; dst[65] = l0; }
  } else if (q0 < g.rows) {
    const float inv = 1.f / l0;
    bf16* dst = out + grp_row(g, q0) * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(o[j][0] * inv, o[j][1] * inv);
    if (t == 0) lse[lrow + grp_tok(g, q0)] = m0 + logf(l0);
  }
  if (q1 < g.rows) {
    const float inv = 1.f / l1;
    bf16* dst = out + grp_row(g, q1) * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(o[j][2] * inv, o[j][3] * inv);
    if (t == 0) lse[lrow + grp_tok(g, q1)] = m1 + logf(l1);
  }
}

// merge the T partials of the CLS query in frame order: one warp per (b, h)
__global__ void space_cls_merge_kernel(const float* __restrict__ part, bf16* __restrict__ out, float* __restrict__ lse,
                                       int BH, int H, int T, int S) {
  const int bh = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (bh >= BH) return;
  const int lane = threadIdx.x & 31;
  const float* p = part + (long long)bh * T * PART;
  float M = -INFINITY;
  for (int f = 0; f < T; ++f) M = fmaxf(M, p[f * PART + 64]);
  float L = 0.f, o0 = 0.f, o1 = 0.f;
  for (int f = 0; f < T; ++f) {
    const float w = exp2f((p[f * PART + 64] - M) * LOG2E);   // every frame's maximum is finite (N >= 1 keys)
    L += p[f * PART + 65] * w;
    o0 += p[f * PART + 2 * lane] * w;
    o1 += p[f * PART + 2 * lane + 1] * w;
  }
  const int b = bh / H, h = bh - b * H;
  const float inv = 1.f / L;
  *reinterpret_cast<uint32_t*>(out + (long long)b * S * (H * HD) + h * HD + 2 * lane) = pack_bf16x2(o0 * inv, o1 * inv);
  if (lane == 0) lse[(long long)bh * S] = M + logf(L);
}

// ------------------------------------------------------------------------------------------------------------
// backward 1: delta[b, h, i] = sum_d dO[b*S + i, h*64 + d] * O[b*S + i, h*64 + d]   (8 threads per (row, head))
// ------------------------------------------------------------------------------------------------------------
__global__ void space_attn_long_delta_kernel(const bf16* __restrict__ out, const bf16* __restrict__ dout,
                                             float* __restrict__ delta, long long rows, int S, int H) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long rh = g >> 3;
  const int c = (int)(g & 7);
  const bool ok = rh < rows * H;
  float d = 0.f;
  if (ok) {
    const long long off = rh * HD + c * 8;   // row-major [B*S, H*64]: (row, head) pairs are consecutive 64-blocks
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
// backward 2: dK, dV of one 64-key tile; grid (ceil((N + 1) / 64), H, B*T).  Each warp owns 16 keys and walks the
// group's query tiles in 32-query chunks: S^T = K Q^T, dP^T = V dO^T.  The CLS key's rows go to an fp32 partial.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
space_attn_long_bwd_kv_kernel(const bf16* __restrict__ qkv, const float* __restrict__ lse,
                              const float* __restrict__ delta, const bf16* __restrict__ dout,
                              bf16* __restrict__ dqkv, float* __restrict__ dcls, int T, int N, int H) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ float s_lse[2][TILE], s_del[2][TILE];
  const uint32_t sk = smem_u32(smem), sv = sk + TILE_BYTES, sq = sv + TILE_BYTES, sdo = sq + 2 * TILE_BYTES;
  const int kt = blockIdx.x, h = blockIdx.y, D = H * HD, S = 1 + T * N;
  const Grp g = make_grp(blockIdx.z, T, N);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int k0r = warp * 16, j0 = kt * TILE + k0r;
  const int nt = (g.rows + TILE - 1) / TILE;
  const long long lrow = ((long long)blockIdx.z / T * H + h) * S;
  // the CLS key (row 0: warp 0, lane 0's first row) is not attended by the CLS query (column 0) in frames f > 0
  const bool skip_cls_query = kt == 0 && warp == 0 && lane == 0 && g.f > 0;

  auto load_q = [&](int qt, int st) {
    load_tile(sq + st * TILE_BYTES, qkv, 3 * D, h * HD, g, qt * TILE);
    load_tile(sdo + st * TILE_BYTES, dout, D, h * HD, g, qt * TILE);
    if (threadIdx.x < TILE) {
      const int i = qt * TILE + threadIdx.x;
      const bool ok = i < g.rows;
      s_lse[st][threadIdx.x] = ok ? lse[lrow + grp_tok(g, i)] * LOG2E : INFINITY;   // +inf: rows past N get P = 0
      s_del[st][threadIdx.x] = ok ? delta[lrow + grp_tok(g, i)] : 0.f;
    }
  };
  load_tile(sk, qkv, 3 * D, D + h * HD, g, kt * TILE);
  load_tile(sv, qkv, 3 * D, 2 * D + h * HD, g, kt * TILE);
  load_q(0, 0);
  cp_async_commit();
  const bool kv0 = j0 + gq < g.rows, kv1 = j0 + gq + 8 < g.rows;

  float dk[8][4], dv[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) { dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = 0.f; dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f; }

  for (int qt = 0; qt < nt; ++qt) {
    const int st = qt & 1;
    if (qt + 1 < nt) {
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
        const bool cls_pair = skip_cls_query && qt == 0 && c0 == 0 && j == 0;
        const float p0 = kv0 && !cls_pair ? exp2f(s[j][0] * LOG2E - lq0) : 0.f;
        const float p1 = kv0 ? exp2f(s[j][1] * LOG2E - lq1) : 0.f;
        const float p2 = kv1 ? exp2f(s[j][2] * LOG2E - lq0) : 0.f;
        const float p3 = kv1 ? exp2f(s[j][3] * LOG2E - lq1) : 0.f;
        pf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0, p1);
        pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
        dsf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0 * (dp[j][0] - dq0), p1 * (dp[j][1] - dq1));
        dsf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2 * (dp[j][2] - dq0), p3 * (dp[j][3] - dq1));
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
  if (r0 == 0) {   // the CLS key: this frame's partial of its dk, dv
    float* dst = dcls + (((long long)blockIdx.z / T * H + h) * T + g.f) * 3 * HD;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      dst[HD + j * 8 + 2 * t] = dk[j][0]; dst[HD + j * 8 + 2 * t + 1] = dk[j][1];
      dst[2 * HD + j * 8 + 2 * t] = dv[j][0]; dst[2 * HD + j * 8 + 2 * t + 1] = dv[j][1];
    }
  } else if (r0 < g.rows) {
    bf16* dst = dqkv + grp_row(g, r0) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(dst + D + j * 8) = pack_bf16x2(dk[j][0], dk[j][1]);
      *reinterpret_cast<uint32_t*>(dst + 2 * D + j * 8) = pack_bf16x2(dv[j][0], dv[j][1]);
    }
  }
  if (r1 < g.rows) {
    bf16* dst = dqkv + grp_row(g, r1) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(dst + D + j * 8) = pack_bf16x2(dk[j][2], dk[j][3]);
      *reinterpret_cast<uint32_t*>(dst + 2 * D + j * 8) = pack_bf16x2(dv[j][2], dv[j][3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward 3: dQ of one 64-query tile over the group's key tiles; grid (ceil((N + 1) / 64), H, B*T).  The CLS query's
// rows go to an fp32 partial.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
space_attn_long_bwd_q_kernel(const bf16* __restrict__ qkv, const float* __restrict__ lse,
                             const float* __restrict__ delta, const bf16* __restrict__ dout,
                             bf16* __restrict__ dqkv, float* __restrict__ dcls, int T, int N, int H, float q_scale) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sq = smem_u32(smem), sdo = sq + TILE_BYTES, sk = sdo + TILE_BYTES, sv = sk + 2 * TILE_BYTES;
  const int qt = blockIdx.x, h = blockIdx.y, D = H * HD, S = 1 + T * N;
  const Grp g = make_grp(blockIdx.z, T, N);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int r0 = warp * 16, i0 = qt * TILE + r0, q0 = i0 + gq, q1 = q0 + 8;
  const int nt = (g.rows + TILE - 1) / TILE;
  const long long lrow = ((long long)blockIdx.z / T * H + h) * S;
  const bool skip_cls_key = qt == 0 && warp == 0 && lane == 0 && g.f > 0;

  load_tile(sq, qkv, 3 * D, h * HD, g, qt * TILE);
  load_tile(sdo, dout, D, h * HD, g, qt * TILE);
  load_tile(sk, qkv, 3 * D, D + h * HD, g, 0);
  load_tile(sv, qkv, 3 * D, 2 * D + h * HD, g, 0);
  cp_async_commit();
  const float ls0 = q0 < g.rows ? lse[lrow + grp_tok(g, q0)] * LOG2E : 0.f;
  const float ls1 = q1 < g.rows ? lse[lrow + grp_tok(g, q1)] * LOG2E : 0.f;
  const float de0 = q0 < g.rows ? delta[lrow + grp_tok(g, q0)] : 0.f;
  const float de1 = q1 < g.rows ? delta[lrow + grp_tok(g, q1)] : 0.f;

  float dq[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) { dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f; }

  for (int kt = 0; kt < nt; ++kt) {
    const int stage = kt & 1;
    if (kt + 1 < nt) {
      load_tile(sk + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, D + h * HD, g, (kt + 1) * TILE);
      load_tile(sv + (stage ^ 1) * TILE_BYTES, qkv, 3 * D, 2 * D + h * HD, g, (kt + 1) * TILE);
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
        const int c = kt * TILE + (c0 + j) * 8 + 2 * t;   // key of the group
        const bool k0ok = c < g.rows && !(skip_cls_key && c == 0), k1ok = c + 1 < g.rows;
        const float p0 = k0ok ? exp2f(s[j][0] * LOG2E - ls0) : 0.f;
        const float p1 = k1ok ? exp2f(s[j][1] * LOG2E - ls0) : 0.f;
        const float p2 = c < g.rows ? exp2f(s[j][2] * LOG2E - ls1) : 0.f;
        const float p3 = k1ok ? exp2f(s[j][3] * LOG2E - ls1) : 0.f;
        dsf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0 * (dp[j][0] - de0), p1 * (dp[j][1] - de0));
        dsf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2 * (dp[j][2] - de1), p3 * (dp[j][3] - de1));
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
  }
  if (q0 == 0) {   // the CLS query: this frame's partial of its dq (q_scale applied by space_cls_grad_kernel)
    float* dst = dcls + (((long long)blockIdx.z / T * H + h) * T + g.f) * 3 * HD;
#pragma unroll
    for (int j = 0; j < 8; ++j) { dst[j * 8 + 2 * t] = dq[j][0]; dst[j * 8 + 2 * t + 1] = dq[j][1]; }
  } else if (q0 < g.rows) {
    bf16* dst = dqkv + grp_row(g, q0) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(dq[j][0] * q_scale, dq[j][1] * q_scale);
  }
  if (q1 < g.rows) {
    bf16* dst = dqkv + grp_row(g, q1) * 3 * D + h * HD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(dq[j][2] * q_scale, dq[j][3] * q_scale);
  }
}

// dqkv[b*S, which*D + h*64 + d] = bf16(sum over frames, in order, of dcls[b, h, f, which, d]) (x q_scale for dq)
__global__ void space_cls_grad_kernel(const float* __restrict__ dcls, bf16* __restrict__ dqkv, int B, int T, int H,
                                      int S, float q_scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H * 3 * HD) return;
  const int d = i % HD, which = (i / HD) % 3, bh = i / (3 * HD), b = bh / H, h = bh - b * H;
  const float* p = dcls + (long long)bh * T * 3 * HD + which * HD + d;
  float v = 0.f;
  for (int f = 0; f < T; ++f) v += p[(long long)f * 3 * HD];
  dqkv[(long long)b * S * 3 * H * HD + which * H * HD + h * HD + d] = __float2bfloat16(which == 0 ? v * q_scale : v);
}

constexpr size_t FWD_SMEM = 5 * TILE_BYTES;   // q + two stages of k, v
constexpr size_t BWD_SMEM = 6 * TILE_BYTES;   // kv pass: k, v + two stages of q, dO;  q pass: q, dO + two of k, v

int check_shape(const char* who, int B, int T, int N, int H) {
  EGOVLP_CHECK_ARG(N >= 1 && N <= MAX_N, "%s: N=%d unsupported (1..%d patches per frame)", who, N, MAX_N);
  EGOVLP_CHECK_ARG(B >= 1 && T >= 1 && H >= 1 && H <= 65535 && (long long)B * T <= 65535,
                   "%s: B=%d T=%d H=%d unsupported (B*T <= 65535, H <= 65535)", who, B, T, H);
  return EGOVLP_OK;
}

}  // namespace
}  // namespace egovlp

using namespace egovlp;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" long long egovlp_space_attn_long_workspace_floats(int B, int T, int N, int H) {
  if (N < 1 || N > MAX_N || B < 1 || T < 1 || H < 1) return -1;
  // backward: delta [B, H, S] + the CLS rows' partials [B, H, T, 3, 64]; the forward's [B, H, T, 66] fits in it
  return (long long)B * H * (1 + (long long)T * N) + (long long)B * H * T * 3 * HD;
}

extern "C" int egovlp_space_attn_long_fwd(const void* qkv, void* out, float* lse, float* workspace, int B, int T,
                                          int N, int H, void* stream) {
  EGOVLP_CHECK_ARG(qkv && out && lse && workspace, "space_attn_long_fwd: null pointer");
  if (int rc = check_shape("space_attn_long_fwd", B, T, N, H)) return rc;
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(space_attn_long_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)FWD_SMEM));
  bf16* o = reinterpret_cast<bf16*>(out);
  const dim3 grid((N + 1 + TILE - 1) / TILE, H, B * T);
  space_attn_long_fwd_kernel<<<grid, NTHREADS, FWD_SMEM, ST(stream)>>>(reinterpret_cast<const bf16*>(qkv), o, lse,
                                                                      workspace, T, N, H);
  EGOVLP_CHECK_LAUNCH();
  const int BH = B * H;
  space_cls_merge_kernel<<<(BH + 3) / 4, 128, 0, ST(stream)>>>(workspace, o, lse, BH, H, T, 1 + T * N);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

extern "C" int egovlp_space_attn_long_bwd(const void* qkv, const void* out, const void* dout, const float* lse,
                                          void* dqkv, float* workspace, int B, int T, int N, int H, float q_scale,
                                          void* stream) {
  EGOVLP_CHECK_ARG(qkv && out && dout && lse && dqkv && workspace, "space_attn_long_bwd: null pointer");
  if (int rc = check_shape("space_attn_long_bwd", B, T, N, H)) return rc;
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(space_attn_long_bwd_kv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)BWD_SMEM));
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(space_attn_long_bwd_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)BWD_SMEM));
  const int S = 1 + T * N;
  const bf16* q = reinterpret_cast<const bf16*>(qkv);
  const bf16* g = reinterpret_cast<const bf16*>(dout);
  bf16* dq = reinterpret_cast<bf16*>(dqkv);
  float* delta = workspace;
  float* dcls = workspace + (long long)B * H * S;
  const long long rows = (long long)B * S, nthr = rows * H * 8;
  space_attn_long_delta_kernel<<<(unsigned)((nthr + 255) / 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const bf16*>(out), g, delta, rows, S, H);
  EGOVLP_CHECK_LAUNCH();
  const dim3 grid((N + 1 + TILE - 1) / TILE, H, B * T);
  space_attn_long_bwd_kv_kernel<<<grid, NTHREADS, BWD_SMEM, ST(stream)>>>(q, lse, delta, g, dq, dcls, T, N, H);
  EGOVLP_CHECK_LAUNCH();
  space_attn_long_bwd_q_kernel<<<grid, NTHREADS, BWD_SMEM, ST(stream)>>>(q, lse, delta, g, dq, dcls, T, N, H, q_scale);
  EGOVLP_CHECK_LAUNCH();
  const int n = B * H * 3 * HD;
  space_cls_grad_kernel<<<(n + 255) / 256, 256, 0, ST(stream)>>>(dcls, dq, B, T, H, S, q_scale);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
