// LayerNorm forward / backward: one warp per row, float4 loads, warp-shuffle reductions, fp32 statistics.
// HBM-bound: fwd reads 4D (+4D add) and writes 2D (+4D) bytes per row; bwd reads 8D (+adds), writes 4D (+2D).
// Replaces nn.LayerNorm (model/video_transformer.py:146,156,159,228,253; DistilBERT LayerNorms) and its autograd.
#include <stdlib.h>

#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

constexpr int LN_WARPS = 8;

// Forward: one row per warp, 8 rows per CTA (a persistent, register-prefetching variant measured slower: 36 % vs
// 55 % of the HBM copy bandwidth at M = 50k rows -- occupancy beats explicit prefetch here).
// Q8 (compile time, so that the other instantiations are unchanged): also y8 = the row in e4m3 with its scale in
// row_scale (see e4m3_row_scale), from the fp32 values already in registers: the row amax is one more warp reduction.
template <int NV, bool Q8>  // NV float4 per lane: covers D <= NV*128
__global__ void __launch_bounds__(LN_WARPS * 32)
layernorm_fwd_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ add,
                     float* __restrict__ sum_out, const float* __restrict__ gamma, const float* __restrict__ beta,
                     bf16* __restrict__ y16, float* __restrict__ y32, float* __restrict__ mean_out,
                     float* __restrict__ rstd_out, int rows, int D, float eps, uint8_t* __restrict__ y8,
                     float* __restrict__ row_scale) {
  const int row = blockIdx.x * LN_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* xr = x + (long long)row * ldx;
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < D) {
      v[i] = *reinterpret_cast<const float4*>(xr + c);
      if (add) {
        const float4 a = *reinterpret_cast<const float4*>(add + (long long)row * D + c);
        v[i].x += a.x; v[i].y += a.y; v[i].z += a.z; v[i].w += a.w;
      }
      if (sum_out) *reinterpret_cast<float4*>(sum_out + (long long)row * D + c) = v[i];
      s += v[i].x + v[i].y + v[i].z + v[i].w;
    } else {
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  // 1/D correctly rounded and explicit roundings: the same arithmetic as the pipelined kernel (whose D is a constant),
  // so a row's result does not depend on which kernel the row count selects
  const float inv_d = __frcp_rn((float)D);
  const float mean = __fmul_rn(warp_sum(s), inv_d);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < D) {
      const float a = v[i].x - mean, b = v[i].y - mean, cc = v[i].z - mean, d = v[i].w - mean;
      q += a * a + b * b + cc * cc + d * d;
    }
  }
  const float rstd = rsqrtf(__fmaf_rn(warp_sum(q), inv_d, eps));
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < D) {
      const float4 g = *reinterpret_cast<const float4*>(gamma + c);
      const float4 b = *reinterpret_cast<const float4*>(beta + c);
      const float o0 = (v[i].x - mean) * rstd * g.x + b.x, o1 = (v[i].y - mean) * rstd * g.y + b.y;
      const float o2 = (v[i].z - mean) * rstd * g.z + b.z, o3 = (v[i].w - mean) * rstd * g.w + b.w;
      if (y16) *reinterpret_cast<uint2*>(y16 + (long long)row * D + c) = make_uint2(pack_bf16x2(o0, o1), pack_bf16x2(o2, o3));
      if (y32) *reinterpret_cast<float4*>(y32 + (long long)row * D + c) = make_float4(o0, o1, o2, o3);
      if constexpr (Q8) {
        v[i] = make_float4(o0, o1, o2, o3);
        amax = fmaxf(amax, fmaxf(fmaxf(fabsf(o0), fabsf(o1)), fmaxf(fabsf(o2), fabsf(o3))));
      }
    }
  }
  if constexpr (Q8) {
    float scale, inv;
    e4m3_row_scale(warp_max(amax), scale, inv);
    if (lane == 0) row_scale[row] = scale;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 32 + lane) * 4;
      if (c < D)
        *reinterpret_cast<uint32_t*>(y8 + (long long)row * D + c) =
            pack_e4m3x4(v[i].x * inv, v[i].y * inv, v[i].z * inv, v[i].w * inv);
    }
  }
}

// Backward.  4 warps / CTA, one row per warp iteration.  The d(gamma) / d(beta) partial sums live in warp-private
// shared memory (each lane owns fixed float4 slots, so no synchronisation) instead of 48 registers: that brings
// the kernel to <= 80 registers and 6 CTAs (24 warps) per SM, which is what a pure streaming kernel needs.
constexpr int LNB_WARPS = 4;

__device__ __forceinline__ float4 load4_f32_or_bf16(const void* p, bool is16, long long off) {
  if (is16) {
    const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const bf16*>(p) + off);
    const float2 lo = unpack_bf16x2(u.x), hi = unpack_bf16x2(u.y);
    return make_float4(lo.x, lo.y, hi.x, hi.y);
  }
  return *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p) + off);
}

template <int NV>
__global__ void __launch_bounds__(LNB_WARPS * 32, 6)
layernorm_bwd_kernel(const void* __restrict__ dy_, int dy16, long long lddy, const float* __restrict__ x, long long ldx,
                     const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                     const void* __restrict__ add1, int add1_16, const void* __restrict__ add2, int add2_16,
                     float* __restrict__ dx, long long lddx, bf16* __restrict__ dx16, float* __restrict__ dgamma,
                     float* __restrict__ dbeta, float* __restrict__ colsum_dx, int rows, int D,
                     float* __restrict__ part) {
  __shared__ float4 acc_g[LNB_WARPS][NV * 32];
  __shared__ float4 acc_b[LNB_WARPS][NV * 32];
  __shared__ float4 acc_o[LNB_WARPS][NV * 32];   // column sums of the output (bias gradient of the producing Linear)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool want_param_grads = dgamma != nullptr || dbeta != nullptr;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    acc_g[warp][i * 32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
    acc_b[warp][i * 32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
    acc_o[warp][i * 32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int row = blockIdx.x * LNB_WARPS + warp; row < rows; row += gridDim.x * LNB_WARPS) {
    const float mu = mean[row], rs = rstd[row];
    float4 dyv[NV], xh[NV];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 32 + lane) * 4;
      if (c < D) {
        dyv[i] = load4_f32_or_bf16(dy_, dy16, (long long)row * lddy + c);
        const float4 xv = *reinterpret_cast<const float4*>(x + (long long)row * ldx + c);
        xh[i] = make_float4((xv.x - mu) * rs, (xv.y - mu) * rs, (xv.z - mu) * rs, (xv.w - mu) * rs);
      }
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 32 + lane) * 4;
      if (c < D) {
        if (want_param_grads) {
          float4 ag = acc_g[warp][i * 32 + lane], ab = acc_b[warp][i * 32 + lane];
          ag.x += dyv[i].x * xh[i].x; ag.y += dyv[i].y * xh[i].y; ag.z += dyv[i].z * xh[i].z; ag.w += dyv[i].w * xh[i].w;
          ab.x += dyv[i].x; ab.y += dyv[i].y; ab.z += dyv[i].z; ab.w += dyv[i].w;
          acc_g[warp][i * 32 + lane] = ag;
          acc_b[warp][i * 32 + lane] = ab;
        }
        const float4 g4 = __ldg(reinterpret_cast<const float4*>(gamma + c));
        dyv[i].x *= g4.x; dyv[i].y *= g4.y; dyv[i].z *= g4.z; dyv[i].w *= g4.w;
        s1 += dyv[i].x + dyv[i].y + dyv[i].z + dyv[i].w;
        s2 += dyv[i].x * xh[i].x + dyv[i].y * xh[i].y + dyv[i].z * xh[i].z + dyv[i].w * xh[i].w;
      }
    }
    const float inv_d = __frcp_rn((float)D);      // as in the pipelined kernel
    const float c1 = __fmul_rn(warp_sum(s1), inv_d), c2 = __fmul_rn(warp_sum(s2), inv_d);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 32 + lane) * 4;
      if (c < D) {
        float4 o = make_float4(rs * (dyv[i].x - c1 - xh[i].x * c2), rs * (dyv[i].y - c1 - xh[i].y * c2),
                               rs * (dyv[i].z - c1 - xh[i].z * c2), rs * (dyv[i].w - c1 - xh[i].w * c2));
        const long long off = (long long)row * D + c;
        if (add1) { const float4 a = load4_f32_or_bf16(add1, add1_16, off); o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w; }
        if (add2) { const float4 a = load4_f32_or_bf16(add2, add2_16, off); o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w; }
        if (colsum_dx) {
          float4 ao = acc_o[warp][i * 32 + lane];
          ao.x += o.x; ao.y += o.y; ao.z += o.z; ao.w += o.w;
          acc_o[warp][i * 32 + lane] = ao;
        }
        if (dx) *reinterpret_cast<float4*>(dx + (long long)row * lddx + c) = o;
        if (dx16) *reinterpret_cast<uint2*>(dx16 + off) = make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
      }
    }
  }
  if (!want_param_grads && !colsum_dx) return;
  __syncthreads();
  const float* fg = reinterpret_cast<const float*>(&acc_g[0][0]);
  const float* fb = reinterpret_cast<const float*>(&acc_b[0][0]);
  const float* fo = reinterpret_cast<const float*>(&acc_o[0][0]);
  for (int c = threadIdx.x; c < D; c += LNB_WARPS * 32) {
    float sg = 0.f, sb = 0.f, so = 0.f;
#pragma unroll
    for (int w = 0; w < LNB_WARPS; ++w) { sg += fg[w * NV * 128 + c]; sb += fb[w * NV * 128 + c]; so += fo[w * NV * 128 + c]; }
    if (part) {          // deterministic form: this CTA's partials, merged in CTA order by ordered_sum
      part[(0ll * gridDim.x + blockIdx.x) * D + c] = sg;
      part[(1ll * gridDim.x + blockIdx.x) * D + c] = sb;
      part[(2ll * gridDim.x + blockIdx.x) * D + c] = so;
      continue;
    }
    if (dgamma) atomicAdd(dgamma + c, sg);
    if (dbeta) atomicAdd(dbeta + c, sb);
    if (colsum_dx) atomicAdd(colsum_dx + c, so);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Pipelined variants for the hot shapes (contiguous rows, D a multiple of 128): a persistent CTA streams tiles of
// PIPE_R rows through a PIPE_STAGES-deep shared-memory ring filled by 1-D bulk async copies (cp.async.bulk, one per input
// stream and tile, completion on an mbarrier) -- the bytes in flight per SM (2 CTAs x 2 tiles x <= 30 KB) no longer
// depend on how many warps fit, which is what capped the occupancy-driven kernels above at 55-59 % of the HBM copy
// rate.  One warp normalises one row of a tile; d(gamma) / d(beta) / column sums stay in registers for the whole
// kernel and are reduced once per CTA.
// ------------------------------------------------------------------------------------------------------------
constexpr int PIPE_R = 4;          // rows per tile = consumer warps
constexpr int PIPE_STAGES = 3;

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ float4 lds4_f32_or_bf16(const uint8_t* p, bool is16, int c) {   // c = element index
  if (is16) {
    const uint2 u = *reinterpret_cast<const uint2*>(p + c * 2);
    const float2 lo = unpack_bf16x2(u.x), hi = unpack_bf16x2(u.y);
    return make_float4(lo.x, lo.y, hi.x, hi.y);
  }
  return *reinterpret_cast<const float4*>(p + c * 4);
}

template <int NV>
__global__ void __launch_bounds__(PIPE_R * 32, 2)
layernorm_bwd_pipe_kernel(const uint8_t* __restrict__ dy, int dy16, const float* __restrict__ x,
                          const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                          const uint8_t* __restrict__ add1, int add1_16, const uint8_t* __restrict__ add2, int add2_16,
                          float* __restrict__ dx, bf16* __restrict__ dx16, float* __restrict__ dgamma,
                          float* __restrict__ dbeta, float* __restrict__ colsum_dx, int rows, float* __restrict__ part) {
  constexpr int D = NV * 128;
  extern __shared__ __align__(128) uint8_t ln_smem[];
  __shared__ __align__(8) unsigned long long full_bar[PIPE_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int dyB = dy16 ? 2 : 4, a1B = add1 ? (add1_16 ? 2 : 4) : 0, a2B = add2 ? (add2_16 ? 2 : 4) : 0;
  const uint32_t off_x = PIPE_R * D * dyB, off_a1 = off_x + PIPE_R * D * 4, off_a2 = off_a1 + PIPE_R * D * a1B;
  const uint32_t stage_bytes = off_a2 + PIPE_R * D * a2B;
  const uint32_t sbase = smem_u32(ln_smem);
  const int tiles = (rows + PIPE_R - 1) / PIPE_R;
  const bool want_param_grads = dgamma != nullptr || dbeta != nullptr;

  if (threadIdx.x == 0) {
    for (int s = 0; s < PIPE_STAGES; ++s) mbar_init(smem_u32(&full_bar[s]), 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto issue = [&](int k) {                               // k-th tile of this CTA -> ring slot k % PIPE_STAGES
    const long long tile = (long long)blockIdx.x + (long long)k * gridDim.x;
    if (tile >= tiles) return;
    const long long r0 = tile * PIPE_R;
    const uint32_t nr = (uint32_t)min((long long)PIPE_R, rows - r0);
    const uint32_t bar = smem_u32(&full_bar[k % PIPE_STAGES]), dst = sbase + (k % PIPE_STAGES) * stage_bytes;
    mbar_expect_tx(bar, nr * D * (dyB + 4 + a1B + a2B));
    bulk_g2s(dst, dy + r0 * D * dyB, nr * D * dyB, bar);
    bulk_g2s(dst + off_x, x + r0 * D, nr * D * 4, bar);
    if (add1) bulk_g2s(dst + off_a1, add1 + r0 * D * a1B, nr * D * a1B, bar);
    if (add2) bulk_g2s(dst + off_a2, add2 + r0 * D * a2B, nr * D * a2B, bar);
  };
  if (threadIdx.x == 0)
    for (int k = 0; k < PIPE_STAGES - 1; ++k) issue(k);

  float4 ag[NV], ab[NV], ao[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) ag[i] = ab[i] = ao[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 g4[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) g4[i] = __ldg(reinterpret_cast<const float4*>(gamma + (i * 32 + lane) * 4));

  int k = 0;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++k) {
    if (threadIdx.x == 0) issue(k + PIPE_STAGES - 1);     // its slot was released by the barrier ending iteration k - 1
    const int row = (int)(tile * PIPE_R) + warp;
    float mu = 0.f, rs = 0.f;
    if (row < rows) { mu = __ldg(mean + row); rs = __ldg(rstd + row); }
    mbar_wait(smem_u32(&full_bar[k % PIPE_STAGES]), (k / PIPE_STAGES) & 1);
    if (row < rows) {
      const uint8_t* st = ln_smem + (k % PIPE_STAGES) * stage_bytes;
      const uint8_t* s_dy = st + warp * D * dyB;
      const uint8_t* s_x = st + off_x + warp * D * 4;
      float4 dyv[NV], xh[NV];
      float s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = (i * 32 + lane) * 4;
        dyv[i] = lds4_f32_or_bf16(s_dy, dy16, c);
        const float4 xv = *reinterpret_cast<const float4*>(s_x + c * 4);
        xh[i] = make_float4((xv.x - mu) * rs, (xv.y - mu) * rs, (xv.z - mu) * rs, (xv.w - mu) * rs);
        if (want_param_grads) {
          ag[i].x += dyv[i].x * xh[i].x; ag[i].y += dyv[i].y * xh[i].y; ag[i].z += dyv[i].z * xh[i].z; ag[i].w += dyv[i].w * xh[i].w;
          ab[i].x += dyv[i].x; ab[i].y += dyv[i].y; ab[i].z += dyv[i].z; ab[i].w += dyv[i].w;
        }
        dyv[i].x *= g4[i].x; dyv[i].y *= g4[i].y; dyv[i].z *= g4[i].z; dyv[i].w *= g4[i].w;
        s1 += dyv[i].x + dyv[i].y + dyv[i].z + dyv[i].w;
        s2 += dyv[i].x * xh[i].x + dyv[i].y * xh[i].y + dyv[i].z * xh[i].z + dyv[i].w * xh[i].w;
      }
      const float c1 = __fmul_rn(warp_sum(s1), 1.f / D), c2 = __fmul_rn(warp_sum(s2), 1.f / D);
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = (i * 32 + lane) * 4;
        float4 o = make_float4(rs * (dyv[i].x - c1 - xh[i].x * c2), rs * (dyv[i].y - c1 - xh[i].y * c2),
                               rs * (dyv[i].z - c1 - xh[i].z * c2), rs * (dyv[i].w - c1 - xh[i].w * c2));
        if (add1) { const float4 a = lds4_f32_or_bf16(st + off_a1 + warp * D * a1B, add1_16, c); o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w; }
        if (add2) { const float4 a = lds4_f32_or_bf16(st + off_a2 + warp * D * a2B, add2_16, c); o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w; }
        if (colsum_dx) { ao[i].x += o.x; ao[i].y += o.y; ao[i].z += o.z; ao[i].w += o.w; }
        const long long off = (long long)row * D + c;
        if (dx) *reinterpret_cast<float4*>(dx + off) = o;
        if (dx16) *reinterpret_cast<uint2*>(dx16 + off) = make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
      }
    }
    __syncthreads();                                       // every warp is done with this slot: it may be refilled
  }
  if (!want_param_grads && !colsum_dx) return;
  // per-CTA reduction of the register accumulators through the (now idle) ring, then one atomic per column
  float4* red = reinterpret_cast<float4*>(ln_smem);        // [3][PIPE_R][NV * 32] float4 = 36 KB at D = 768 <= 3 stages
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    red[(0 * PIPE_R + warp) * NV * 32 + i * 32 + lane] = ag[i];
    red[(1 * PIPE_R + warp) * NV * 32 + i * 32 + lane] = ab[i];
    red[(2 * PIPE_R + warp) * NV * 32 + i * 32 + lane] = ao[i];
  }
  __syncthreads();
  const float* fr = reinterpret_cast<const float*>(red);
  for (int c = threadIdx.x; c < D; c += PIPE_R * 32) {
    float sg = 0.f, sb = 0.f, so = 0.f;
#pragma unroll
    for (int w = 0; w < PIPE_R; ++w) {
      sg += fr[(0 * PIPE_R + w) * D + c]; sb += fr[(1 * PIPE_R + w) * D + c]; so += fr[(2 * PIPE_R + w) * D + c];
    }
    if (part) {
      part[(0ll * gridDim.x + blockIdx.x) * D + c] = sg;
      part[(1ll * gridDim.x + blockIdx.x) * D + c] = sb;
      part[(2ll * gridDim.x + blockIdx.x) * D + c] = so;
      continue;
    }
    if (dgamma) atomicAdd(dgamma + c, sg);
    if (dbeta) atomicAdd(dbeta + c, sb);
    if (colsum_dx) atomicAdd(colsum_dx + c, so);
  }
}

constexpr int PIPE_FR = 8;         // forward: rows per tile = warps

template <int NV, bool Q8>      // Q8: as layernorm_fwd_kernel
__global__ void __launch_bounds__(PIPE_FR * 32, 2)
layernorm_fwd_pipe_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                          bf16* __restrict__ y16, float* __restrict__ y32, float* __restrict__ mean_out,
                          float* __restrict__ rstd_out, int rows, float eps, uint8_t* __restrict__ y8,
                          float* __restrict__ row_scale) {
  constexpr int D = NV * 128;
  constexpr uint32_t STAGE = PIPE_FR * D * 4;
  extern __shared__ __align__(128) uint8_t ln_smem[];
  __shared__ __align__(8) unsigned long long full_bar[PIPE_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t sbase = smem_u32(ln_smem);
  const int tiles = (rows + PIPE_FR - 1) / PIPE_FR;
  if (threadIdx.x == 0) {
    for (int s = 0; s < PIPE_STAGES; ++s) mbar_init(smem_u32(&full_bar[s]), 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto issue = [&](int k) {
    const long long tile = (long long)blockIdx.x + (long long)k * gridDim.x;
    if (tile >= tiles) return;
    const long long r0 = tile * PIPE_FR;
    const uint32_t nr = (uint32_t)min((long long)PIPE_FR, rows - r0);
    const uint32_t bar = smem_u32(&full_bar[k % PIPE_STAGES]);
    mbar_expect_tx(bar, nr * D * 4);
    bulk_g2s(sbase + (k % PIPE_STAGES) * STAGE, x + r0 * D, nr * D * 4, bar);
  };
  if (threadIdx.x == 0)
    for (int k = 0; k < PIPE_STAGES - 1; ++k) issue(k);
  float4 g4[NV], b4[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    g4[i] = __ldg(reinterpret_cast<const float4*>(gamma + (i * 32 + lane) * 4));
    b4[i] = __ldg(reinterpret_cast<const float4*>(beta + (i * 32 + lane) * 4));
  }
  int k = 0;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++k) {
    if (threadIdx.x == 0) issue(k + PIPE_STAGES - 1);
    const int row = (int)(tile * PIPE_FR) + warp;
    mbar_wait(smem_u32(&full_bar[k % PIPE_STAGES]), (k / PIPE_STAGES) & 1);
    if (row < rows) {
      const uint8_t* s_x = ln_smem + (k % PIPE_STAGES) * STAGE + warp * D * 4;
      float4 v[NV];
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        v[i] = *reinterpret_cast<const float4*>(s_x + (i * 32 + lane) * 16);
        s += v[i].x + v[i].y + v[i].z + v[i].w;
      }
      const float mu = __fmul_rn(warp_sum(s), 1.f / D);
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const float a = v[i].x - mu, b = v[i].y - mu, c = v[i].z - mu, d = v[i].w - mu;
        q += a * a + b * b + c * c + d * d;
      }
      const float rs = rsqrtf(__fmaf_rn(warp_sum(q), 1.f / D, eps));
      if (lane == 0) {
        if (mean_out) mean_out[row] = mu;
        if (rstd_out) rstd_out[row] = rs;
      }
      float amax = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const long long off = (long long)row * D + (i * 32 + lane) * 4;
        const float o0 = (v[i].x - mu) * rs * g4[i].x + b4[i].x, o1 = (v[i].y - mu) * rs * g4[i].y + b4[i].y;
        const float o2 = (v[i].z - mu) * rs * g4[i].z + b4[i].z, o3 = (v[i].w - mu) * rs * g4[i].w + b4[i].w;
        if (y16) *reinterpret_cast<uint2*>(y16 + off) = make_uint2(pack_bf16x2(o0, o1), pack_bf16x2(o2, o3));
        if (y32) *reinterpret_cast<float4*>(y32 + off) = make_float4(o0, o1, o2, o3);
        if constexpr (Q8) {
          v[i] = make_float4(o0, o1, o2, o3);
          amax = fmaxf(amax, fmaxf(fmaxf(fabsf(o0), fabsf(o1)), fmaxf(fabsf(o2), fabsf(o3))));
        }
      }
      if constexpr (Q8) {
        float scale, inv;
        e4m3_row_scale(warp_max(amax), scale, inv);
        if (lane == 0) row_scale[row] = scale;
#pragma unroll
        for (int i = 0; i < NV; ++i)
          *reinterpret_cast<uint32_t*>(y8 + (long long)row * D + (i * 32 + lane) * 4) =
              pack_e4m3x4(v[i].x * inv, v[i].y * inv, v[i].z * inv, v[i].w * inv);
      }
    }
    __syncthreads();
  }
}

// The pipelined kernels take contiguous rows (ld == D), D = NV * 128 and 16-byte aligned bases; EGOVLP_LN_PIPE=0 keeps
// the occupancy-driven kernels (A/B, and the shapes above stay covered by them anyway).
inline bool ln_pipe_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("EGOVLP_LN_PIPE"); on = !(e && e[0] == '0'); }
  return on == 1;
}
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
inline bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

// Views whose base is not 16-byte (src) / 8-byte (dst) aligned, such as the slices of a Bf16Cache.cat buffer, take
// the scalar path, as in cast_multi_kernel.
__global__ void cast_f32_to_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x * 4;
  const bool vec = (reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
    if (vec && i + 3 < n) {
      const float4 v = *reinterpret_cast<const float4*>(src + i);
      *reinterpret_cast<uint2*>(dst + i) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
    } else {
      for (long long j = i; j < min(n, i + 4); ++j) dst[j] = __float2bfloat16(src[j]);   // this thread's 4 only
    }
  }
}

// out[n] += sum_m dy[m,n].  Block = 32 (16-byte column vectors) x 8 (rows); every warp load is 512 contiguous bytes,
// 4 independent row loads in flight per thread; smem reduce over the 8 row-lanes, one atomicAdd per column per block.
template <bool FP32>
__global__ void __launch_bounds__(256)
colsum_kernel(const void* __restrict__ dy, long long ld, float* __restrict__ out, int M, int N, int rows_per_block,
              float* __restrict__ part) {
  constexpr int VEC = FP32 ? 4 : 8;
  __shared__ float red[8][32 * VEC + 1];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int col = (blockIdx.x * 32 + tx) * VEC;
  const int r0 = blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
  float acc[VEC];
#pragma unroll
  for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
  if (col < N) {
    auto add_row = [&](int r) {
      if (FP32) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(dy) + (long long)r * ld + col));
        acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w;
      } else {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(dy) + (long long)r * ld + col));
        const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
        acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
        acc[4 % VEC] += c.x; acc[5 % VEC] += c.y; acc[6 % VEC] += d.x; acc[7 % VEC] += d.y;
      }
    };
    int r = r0 + ty;
    for (; r + 24 < r1; r += 32) { add_row(r); add_row(r + 8); add_row(r + 16); add_row(r + 24); }
    for (; r < r1; r += 8) add_row(r);
  }
#pragma unroll
  for (int k = 0; k < VEC; ++k) red[ty][tx * VEC + k] = acc[k];
  __syncthreads();
  for (int c = threadIdx.x; c < 32 * VEC; c += 256) {
    const int gc = blockIdx.x * 32 * VEC + c;
    if (gc < N) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += red[w][c];
      if (part) part[(long long)blockIdx.y * N + gc] = t;      // deterministic form: merged in row-block order
      else atomicAdd(out + gc, t);
    }
  }
}

template <int NV, bool Q8 = false>
int launch_ln_fwd(const float* x, long long ldx, const float* add, float* sum_out, const float* gamma,
                  const float* beta, void* y16, float* y32, float* mean, float* rstd, int rows, int D, float eps,
                  cudaStream_t st, uint8_t* y8 = nullptr, float* row_scale = nullptr) {
  if (ln_pipe_enabled() && D == NV * 128 && ldx == D && !add && !sum_out && rows >= 4096 && aligned16(x)) {
    auto kern = layernorm_fwd_pipe_kernel<NV, Q8>;
    const int smem = PIPE_STAGES * PIPE_FR * D * 4;
    static bool attr = false;
    if (!attr) { EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); attr = true; }
    const int tiles = (rows + PIPE_FR - 1) / PIPE_FR;
    kern<<<min(tiles, 2 * num_sms()), PIPE_FR * 32, smem, st>>>(x, gamma, beta, reinterpret_cast<bf16*>(y16), y32, mean, rstd,
                                                                 rows, eps, y8, row_scale);
    EGOVLP_CHECK_LAUNCH();
    return EGOVLP_OK;
  }
  const int grid = (rows + LN_WARPS - 1) / LN_WARPS;
  layernorm_fwd_kernel<NV, Q8><<<grid, LN_WARPS * 32, 0, st>>>(x, ldx, add, sum_out, gamma, beta,
                                                              reinterpret_cast<bf16*>(y16), y32, mean, rstd, rows, D, eps,
                                                              y8, row_scale);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

template <int NV>
int launch_ln_bwd(const void* dy, int dy16, long long lddy, const float* x, long long ldx, const float* gamma,
                  const float* mean, const float* rstd, const void* add1, int add1_16, const void* add2, int add2_16,
                  float* dx, long long lddx, void* dx16, float* dgamma, float* dbeta, float* colsum_dx, int rows, int D,
                  cudaStream_t st, float* part) {
  // part (deterministic form): per-CTA partials [3][grid][D], merged in CTA order; the kernel choice ignores
  // EGOVLP_LN_PIPE and the grid is sized for DET_SMS, so both follow from the shapes, the strides and the 16-byte
  // alignment of dy / x / add1 / add2 (the pipelined kernel's bulk copies need it) alone
  const bool det = part != nullptr;
  const int sms = det ? DET_SMS : num_sms();
  auto merge = [&](int grid) -> int {
    if (!det) return EGOVLP_OK;
    return ordered_sum(part, grid, D, dgamma, dbeta, colsum_dx, st);
  };
  if ((det || ln_pipe_enabled()) && D == NV * 128 && ldx == D && lddy == D && (!dx || lddx == D) && rows >= 4096 && aligned16(dy) &&
      aligned16(x) && aligned16(add1) && aligned16(add2)) {
    auto kern = layernorm_bwd_pipe_kernel<NV>;
    const int per_elem = (dy16 ? 2 : 4) + 4 + (add1 ? (add1_16 ? 2 : 4) : 0) + (add2 ? (add2_16 ? 2 : 4) : 0);
    const int smem = max(PIPE_STAGES * PIPE_R * D * per_elem, 3 * PIPE_R * D * 4);
    static int attr = 0;
    if (attr < smem) { EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); attr = smem; }
    const int tiles = (rows + PIPE_R - 1) / PIPE_R;
    const int grid = min(tiles, 2 * sms);
    kern<<<grid, PIPE_R * 32, smem, st>>>(
        reinterpret_cast<const uint8_t*>(dy), dy16, x, gamma, mean, rstd, reinterpret_cast<const uint8_t*>(add1), add1_16,
        reinterpret_cast<const uint8_t*>(add2), add2_16, dx, reinterpret_cast<bf16*>(dx16), dgamma, dbeta, colsum_dx, rows,
        part);
    EGOVLP_CHECK_LAUNCH();
    return merge(grid);
  }
  const int grid = min((rows + LNB_WARPS - 1) / LNB_WARPS, sms * 12);
  layernorm_bwd_kernel<NV><<<grid, LNB_WARPS * 32, 0, st>>>(dy, dy16, lddy, x, ldx, gamma, mean, rstd, add1, add1_16, add2,
                                                           add2_16, dx, lddx, reinterpret_cast<bf16*>(dx16), dgamma,
                                                           dbeta, colsum_dx, rows, D, part);
  EGOVLP_CHECK_LAUNCH();
  return merge(grid);
}

}  // namespace
}  // namespace egovlp

using namespace egovlp;

extern "C" int egovlp_layernorm_fwd(const float* x, long long ldx, const float* add, float* sum_out,
                                    const float* gamma, const float* beta, void* y_bf16, float* y_f32, float* mean,
                                    float* rstd, int rows, int D, float eps, void* stream) {
  EGOVLP_CHECK_ARG(x && gamma && beta && (y_bf16 || y_f32), "layernorm_fwd: null pointer");
  EGOVLP_CHECK_ARG(rows >= 0 && D > 0 && D % 4 == 0 && D <= 1024 && ldx % 4 == 0, "layernorm_fwd: bad D=%d ldx=%lld", D, ldx);
  // every kernel moves whole vectors (float4, 4 x bf16): a base off that alignment is refused here instead of faulting
  EGOVLP_CHECK_ARG(aligned16(x) && aligned16(add) && aligned16(sum_out) && aligned16(gamma) && aligned16(beta) &&
                   aligned16(y_f32) && aligned8(y_bf16),
                   "layernorm_fwd: fp32 operands must be 16-byte aligned and bf16 ones 8-byte aligned");
  if (rows == 0) return EGOVLP_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int nv = (D + 127) / 128;
#define LN_FWD_CASE(n) case n: return launch_ln_fwd<n>(x, ldx, add, sum_out, gamma, beta, y_bf16, y_f32, mean, rstd, rows, D, eps, st)
  switch (nv) { LN_FWD_CASE(1); LN_FWD_CASE(2); LN_FWD_CASE(3); LN_FWD_CASE(4); LN_FWD_CASE(5); LN_FWD_CASE(6); LN_FWD_CASE(7); LN_FWD_CASE(8); }
#undef LN_FWD_CASE
  return EGOVLP_ERR_UNSUPPORTED;
}

extern "C" int egovlp_layernorm_fwd_e4m3(const float* x, long long ldx, const float* gamma, const float* beta,
                                         void* y_bf16, float* y_f32, float* mean, float* rstd, uint8_t* y8,
                                         float* row_scale, int rows, int D, float eps, void* stream) {
  EGOVLP_CHECK_ARG(x && gamma && beta && y8 && row_scale, "layernorm_fwd_e4m3: null pointer");
  // D <= 256 is not instantiated: the D = 256 form spills (ptxas keeps it at 32 registers)
  EGOVLP_CHECK_ARG(rows >= 0 && D > 256 && D % 4 == 0 && D <= 1024 && ldx % 4 == 0,
                   "layernorm_fwd_e4m3: bad D=%d ldx=%lld (256 < D <= 1024, D %% 4 == 0)", D, ldx);
  EGOVLP_CHECK_ARG((reinterpret_cast<uintptr_t>(y8) & 3) == 0, "layernorm_fwd_e4m3: y8 must be 4B aligned");
  EGOVLP_CHECK_ARG(aligned16(x) && aligned16(gamma) && aligned16(beta) && aligned16(y_f32) && aligned8(y_bf16),
                   "layernorm_fwd_e4m3: fp32 operands must be 16-byte aligned and bf16 ones 8-byte aligned");
  if (rows == 0) return EGOVLP_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int nv = (D + 127) / 128;
#define LN_FWD8_CASE(n) case n: return launch_ln_fwd<n, true>(x, ldx, nullptr, nullptr, gamma, beta, y_bf16, y_f32, mean, rstd, rows, D, eps, st, y8, row_scale)
  switch (nv) { LN_FWD8_CASE(3); LN_FWD8_CASE(4); LN_FWD8_CASE(5); LN_FWD8_CASE(6); LN_FWD8_CASE(7); LN_FWD8_CASE(8); }
#undef LN_FWD8_CASE
  return EGOVLP_ERR_UNSUPPORTED;
}

static int layernorm_bwd_impl(const void* dy, int dy_is_bf16, long long lddy, const float* x, long long ldx,
                              const float* gamma, const float* mean, const float* rstd, const void* add1,
                              int add1_is_bf16, const void* add2, int add2_is_bf16, float* dx, long long lddx,
                              void* dx_bf16, float* dgamma, float* dbeta, float* colsum_dx, int rows, int D, float* part,
                              void* stream) {
  EGOVLP_CHECK_ARG(dy && x && gamma && mean && rstd && (dx || dx_bf16), "layernorm_bwd: null pointer");
  EGOVLP_CHECK_ARG(rows >= 0 && D > 0 && D % 4 == 0 && D <= 1024 && ldx % 4 == 0 && lddy % 4 == 0 && lddx % 4 == 0, "layernorm_bwd: bad D=%d", D);
  EGOVLP_CHECK_ARG((dy_is_bf16 ? aligned8(dy) : aligned16(dy)) && (add1_is_bf16 ? aligned8(add1) : aligned16(add1)) &&
                   (add2_is_bf16 ? aligned8(add2) : aligned16(add2)) && aligned16(x) && aligned16(gamma) &&
                   aligned16(dx) && aligned8(dx_bf16),
                   "layernorm_bwd: fp32 operands must be 16-byte aligned and bf16 ones 8-byte aligned");
  if (rows == 0) return EGOVLP_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int nv = (D + 127) / 128;
#define LN_BWD_CASE(n) case n: return launch_ln_bwd<n>(dy, dy_is_bf16, lddy, x, ldx, gamma, mean, rstd, add1, add1_is_bf16, add2, add2_is_bf16, dx, lddx, dx_bf16, dgamma, dbeta, colsum_dx, rows, D, st, part)
  switch (nv) { LN_BWD_CASE(1); LN_BWD_CASE(2); LN_BWD_CASE(3); LN_BWD_CASE(4); LN_BWD_CASE(5); LN_BWD_CASE(6); LN_BWD_CASE(7); LN_BWD_CASE(8); }
#undef LN_BWD_CASE
  return EGOVLP_ERR_UNSUPPORTED;
}

extern "C" int egovlp_layernorm_bwd(const void* dy, int dy_is_bf16, long long lddy, const float* x, long long ldx,
                                    const float* gamma, const float* mean, const float* rstd, const void* add1,
                                    int add1_is_bf16, const void* add2, int add2_is_bf16, float* dx, long long lddx,
                                    void* dx_bf16, float* dgamma, float* dbeta, float* colsum_dx, int rows, int D,
                                    void* stream) {
  return layernorm_bwd_impl(dy, dy_is_bf16, lddy, x, ldx, gamma, mean, rstd, add1, add1_is_bf16, add2, add2_is_bf16, dx,
                            lddx, dx_bf16, dgamma, dbeta, colsum_dx, rows, D, nullptr, stream);
}

// the largest grid either backward kernel takes for these shapes in the deterministic form, x 3 sums x D
extern "C" long long egovlp_layernorm_bwd_det_workspace_floats(int rows, int D) {
  if (rows < 0 || D <= 0) return -1;
  const long long pipe = min((rows + PIPE_R - 1) / PIPE_R, 2 * DET_SMS);
  const long long gen = min((rows + LNB_WARPS - 1) / LNB_WARPS, 12 * DET_SMS);
  return 3ll * max(pipe, gen) * D;
}

extern "C" int egovlp_layernorm_bwd_det(const void* dy, int dy_is_bf16, long long lddy, const float* x, long long ldx,
                                        const float* gamma, const float* mean, const float* rstd, const void* add1,
                                        int add1_is_bf16, const void* add2, int add2_is_bf16, float* dx, long long lddx,
                                        void* dx_bf16, float* dgamma, float* dbeta, float* colsum_dx, int rows, int D,
                                        float* ws, void* stream) {
  EGOVLP_CHECK_ARG(ws || (!dgamma && !dbeta && !colsum_dx), "layernorm_bwd_det: null workspace");
  // without any column sum there is nothing to reduce: the plain kernel is deterministic as it stands
  const bool sums = dgamma || dbeta || colsum_dx;
  return layernorm_bwd_impl(dy, dy_is_bf16, lddy, x, ldx, gamma, mean, rstd, add1, add1_is_bf16, add2, add2_is_bf16, dx,
                            lddx, dx_bf16, dgamma, dbeta, colsum_dx, rows, D, sums ? ws : nullptr, stream);
}

extern "C" int egovlp_cast_f32_to_bf16(const float* src, void* dst_bf16, long long n, void* stream) {
  EGOVLP_CHECK_ARG(src && dst_bf16 && n >= 0, "cast: bad args");
  if (n == 0) return EGOVLP_OK;
  const long long blocks = (n / 4 + 255) / 256;
  long long g = blocks < 1 ? 1 : blocks;
  if (g > (long long)num_sms() * 16) g = (long long)num_sms() * 16;
  const int grid = (int)g;
  cast_f32_to_bf16_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(src, reinterpret_cast<bf16*>(dst_bf16), n);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

// One warp per row: the row amax, then the row in e4m3 with its scale (the weight operands of the e4m3 GEMM, one scale
// per output channel).
__global__ void quantize_rows_e4m3_kernel(const float* __restrict__ w, long long ldw, uint8_t* __restrict__ q,
                                          float* __restrict__ scale, int rows, int K) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* wr = w + (long long)row * ldw;
  float amax = 0.f;
  for (int c = lane * 4; c < K; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(wr + c);
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  float s, inv;
  e4m3_row_scale(warp_max(amax), s, inv);
  if (lane == 0) scale[row] = s;
  for (int c = lane * 4; c < K; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(wr + c);
    *reinterpret_cast<uint32_t*>(q + (long long)row * K + c) =
        pack_e4m3x4(__fmul_rn(v.x, inv), __fmul_rn(v.y, inv), __fmul_rn(v.z, inv), __fmul_rn(v.w, inv));
  }
}

extern "C" int egovlp_quantize_rows_e4m3(const float* w, long long ldw, uint8_t* q, float* scale, int rows, int K,
                                         void* stream) {
  EGOVLP_CHECK_ARG(w && q && scale && rows >= 0 && K > 0 && K % 4 == 0 && ldw >= K && ldw % 4 == 0,
                   "quantize_rows_e4m3: bad args (K=%d ldw=%lld)", K, ldw);
  EGOVLP_CHECK_ARG(((reinterpret_cast<uintptr_t>(w) & 15) | (reinterpret_cast<uintptr_t>(q) & 3)) == 0,
                   "quantize_rows_e4m3: w must be 16B and q 4B aligned");
  if (rows == 0) return EGOVLP_OK;
  quantize_rows_e4m3_kernel<<<(rows + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(w, ldw, q, scale, rows, K);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

// The row-block split (sized for DET_SMS when `part` is given: deterministic form, part = [row_blocks][N])
static void colsum_grid(int M, int N, int vec, int sms, int& row_blocks, int& rows_per_block) {
  const int col_blocks = (N / vec + 31) / 32;
  row_blocks = max(1, min((M + 63) / 64, (sms * 8 + col_blocks - 1) / col_blocks));
  rows_per_block = (M + row_blocks - 1) / row_blocks;
  row_blocks = (M + rows_per_block - 1) / rows_per_block;
}

static int colsum_impl(const void* dy, int dy_is_fp32, long long ld, float* out, int M, int N, float* part, void* stream) {
  EGOVLP_CHECK_ARG(dy && out && M >= 0 && N > 0, "colsum: bad args");
  if (M == 0) return EGOVLP_OK;
  const int vec = dy_is_fp32 ? 4 : 8;
  EGOVLP_CHECK_ARG(N % vec == 0 && ld % vec == 0 && (reinterpret_cast<uintptr_t>(dy) & 15) == 0,
                   "colsum: N=%d / ld=%lld must be multiples of %d and the base 16B aligned", N, ld, vec);
  int row_blocks, rows_per_block;
  colsum_grid(M, N, vec, part ? DET_SMS : num_sms(), row_blocks, rows_per_block);
  dim3 grid((N / vec + 31) / 32, row_blocks);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dy_is_fp32) colsum_kernel<true><<<grid, 256, 0, st>>>(dy, ld, out, M, N, rows_per_block, part);
  else colsum_kernel<false><<<grid, 256, 0, st>>>(dy, ld, out, M, N, rows_per_block, part);
  EGOVLP_CHECK_LAUNCH();
  return part ? ordered_sum(part, row_blocks, N, out, st) : EGOVLP_OK;
}

extern "C" int egovlp_colsum_accum(const void* dy, int dy_is_fp32, long long ld, float* out, int M, int N,
                                   void* stream) {
  return colsum_impl(dy, dy_is_fp32, ld, out, M, N, nullptr, stream);
}

extern "C" long long egovlp_colsum_det_workspace_floats(int M, int N, int dy_is_fp32) {
  if (M < 0 || N <= 0) return -1;
  if (M == 0) return 0;
  int row_blocks, rows_per_block;
  colsum_grid(M, N, dy_is_fp32 ? 4 : 8, DET_SMS, row_blocks, rows_per_block);
  return (long long)row_blocks * N;
}

extern "C" int egovlp_colsum_accum_det(const void* dy, int dy_is_fp32, long long ld, float* out, int M, int N, float* ws,
                                       void* stream) {
  EGOVLP_CHECK_ARG(ws, "colsum_det: null workspace");
  return colsum_impl(dy, dy_is_fp32, ld, out, M, N, ws, stream);
}
