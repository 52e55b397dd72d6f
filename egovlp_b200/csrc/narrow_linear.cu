// Narrow projection heads: out[rows, C] = act[rows, K] W[C, K]^T + b for widths C the wgmma GEMM cannot take
// (its N must be a multiple of 32 and its TMA descriptors need 16-byte row strides, which a [rows, C] bf16 gradient
// of C = 2 or 16 does not have).  These are the fine-tuning heads of Ego4D OSCC (projection_dim 2,
// configs/ft/oscc.json) and PNR (projection_dim 16, configs/ft/pnr.json): vid_proj = Linear(768, C) behind the CLS
// LayerNorm and txt_proj = ReLU -> Linear(768, C) (model/model.py:72-79).
//
// Same operands and roundings as the wide path: bf16 activations and bf16 weight copy in, fp32 accumulation, fp32 bias
// and output; the backward takes d16 = bf16(dout) for both products and the fp32 dout for the bias gradient.
// The work is tiny (2 rows x C x K MACs per row), so these are plain CUDA-core kernels.  No atomics: every output
// element is summed by one thread or one warp in a fixed order (the weight gradient's row splits are merged by a
// second pass in split order), so results are bitwise reproducible from run to run.
#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

constexpr int FWD_ROWS = 8;       // activation rows per CTA (staged in shared memory, reused by every column)
constexpr int FWD_COLS = 32;      // output columns per CTA (4 per warp)
constexpr int WG_COLS = 8;        // weight-gradient rows (output columns c) per thread
constexpr int WG_THREADS = 128;   // each thread owns 2 adjacent k

__device__ __forceinline__ void unpack8(const uint4 u, float* f) {
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}

// one warp per output column: lanes stride K in 8-element vectors, partial sums of the CTA's FWD_ROWS rows, then a
// butterfly reduction (fixed order)
__global__ void __launch_bounds__(256)
narrow_fwd_kernel(const uint4* __restrict__ act, const uint4* __restrict__ w, const float* __restrict__ bias,
                  float* __restrict__ out, int rows, int C, int K8) {
  extern __shared__ uint4 xs[];                                   // [FWD_ROWS][K8]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r0 = blockIdx.x * FWD_ROWS, nr = min(FWD_ROWS, rows - r0);
  for (int idx = tid; idx < FWD_ROWS * K8; idx += blockDim.x) {
    const int r = idx / K8;
    xs[idx] = r < nr ? act[(long long)(r0 + r) * K8 + idx % K8] : make_uint4(0, 0, 0, 0);
  }
  __syncthreads();
  const int c_end = min(C, (int)(blockIdx.y + 1) * FWD_COLS);
  for (int c = blockIdx.y * FWD_COLS + warp; c < c_end; c += 8) {
    float acc[FWD_ROWS];
#pragma unroll
    for (int r = 0; r < FWD_ROWS; ++r) acc[r] = 0.f;
    for (int v = lane; v < K8; v += 32) {
      float wf[8];
      unpack8(w[(long long)c * K8 + v], wf);
#pragma unroll
      for (int r = 0; r < FWD_ROWS; ++r) {
        float xf[8];
        unpack8(xs[r * K8 + v], xf);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[r] = fmaf(xf[e], wf[e], acc[r]);
      }
    }
    const float b = bias ? bias[c] : 0.f;
#pragma unroll
    for (int r = 0; r < FWD_ROWS; ++r) {
      const float s = warp_sum(acc[r]);
      if (lane == 0 && r < nr) out[(long long)(r0 + r) * C + c] = s + b;
    }
  }
}

// dW partial of one row split: dst[c, k] = sum_{r in split} d16[r, c] act[r, k]   (thread = 2 k x WG_COLS c)
__global__ void __launch_bounds__(WG_THREADS)
narrow_wgrad_kernel(const bf16* __restrict__ d16, const uint32_t* __restrict__ act, float* __restrict__ dst, int rows,
                    int C, int K, int rows_per_split) {
  const int k2 = blockIdx.x * WG_THREADS + threadIdx.x;
  if (2 * k2 >= K) return;
  const int c0 = blockIdx.y * WG_COLS;
  const int r_begin = blockIdx.z * rows_per_split, r_end = min(rows, r_begin + rows_per_split);
  float acc[WG_COLS][2];
#pragma unroll
  for (int j = 0; j < WG_COLS; ++j) acc[j][0] = acc[j][1] = 0.f;
  for (int r = r_begin; r < r_end; ++r) {
    const float2 a = unpack_bf16x2(act[(long long)r * (K / 2) + k2]);
#pragma unroll
    for (int j = 0; j < WG_COLS; ++j) {
      if (c0 + j < C) {
        const float d = __bfloat162float(d16[(long long)r * C + c0 + j]);
        acc[j][0] = fmaf(d, a.x, acc[j][0]);
        acc[j][1] = fmaf(d, a.y, acc[j][1]);
      }
    }
  }
  float* base = dst + (long long)blockIdx.z * C * K;
#pragma unroll
  for (int j = 0; j < WG_COLS; ++j)
    if (c0 + j < C) *reinterpret_cast<float2*>(base + (long long)(c0 + j) * K + 2 * k2) = make_float2(acc[j][0], acc[j][1]);
}

// dW[i] = sum over the row splits of their partials, in split order
__global__ void narrow_wgrad_merge_kernel(const float* __restrict__ part, float* __restrict__ dw, long long n, int splits) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int p = 0; p < splits; ++p) s += part[p * n + i];
  dw[i] = s;
}

// d_act[r, k] = sum_c d16[r, c] W[c, k]   (thread = 2 k of one row)
__global__ void __launch_bounds__(128)
narrow_dgrad_kernel(const bf16* __restrict__ d16, const uint32_t* __restrict__ w, float* __restrict__ dact, int C, int K) {
  const int k2 = blockIdx.x * 128 + threadIdx.x, r = blockIdx.y;
  if (2 * k2 >= K) return;
  float a0 = 0.f, a1 = 0.f;
  for (int c = 0; c < C; ++c) {
    const float d = __bfloat162float(d16[(long long)r * C + c]);
    const float2 wv = unpack_bf16x2(w[(long long)c * (K / 2) + k2]);
    a0 = fmaf(d, wv.x, a0);
    a1 = fmaf(d, wv.y, a1);
  }
  *reinterpret_cast<float2*>(dact + (long long)r * K + 2 * k2) = make_float2(a0, a1);
}

// db[c] = sum_r dout[r, c]: one warp per column (lanes stride the rows, then a butterfly reduction)
__global__ void narrow_bgrad_kernel(const float* __restrict__ dout, float* __restrict__ db, int rows, int C) {
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c >= C) return;
  float s = 0.f;
  for (int r = lane; r < rows; r += 32) s += dout[(long long)r * C + c];
  s = warp_sum(s);
  if (lane == 0) db[c] = s;
}

// row splits of the weight gradient: enough CTAs to cover the SMs about twice, at least 32 rows per split
int wgrad_splits(int rows, int C, int K) {
  const int ctas = ((K / 2 + WG_THREADS - 1) / WG_THREADS) * ((C + WG_COLS - 1) / WG_COLS);
  const int want = (2 * num_sms() + ctas - 1) / ctas;
  return max(1, min(want, (rows + 31) / 32));
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace
}  // namespace egovlp

using namespace egovlp;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int egovlp_narrow_linear_fwd(const void* act, const void* w, const float* bias, float* out, int rows, int C,
                                        int K, void* stream) {
  EGOVLP_CHECK_ARG(act && w && out && rows >= 0 && C > 0 && K > 0, "narrow_linear_fwd: bad args");
  EGOVLP_CHECK_ARG(K % 8 == 0 && K <= 2048 && aligned16(act) && aligned16(w),
                   "narrow_linear_fwd: K=%d must be a multiple of 8 (<= 2048) and act / w 16B aligned", K);
  if (rows == 0) return EGOVLP_OK;
  const int K8 = K / 8;
  dim3 grid((rows + FWD_ROWS - 1) / FWD_ROWS, (C + FWD_COLS - 1) / FWD_COLS);
  narrow_fwd_kernel<<<grid, 256, FWD_ROWS * K8 * sizeof(uint4), ST(stream)>>>(
      reinterpret_cast<const uint4*>(act), reinterpret_cast<const uint4*>(w), bias, out, rows, C, K8);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

extern "C" long long egovlp_narrow_linear_workspace_floats(int rows, int C, int K) {
  if (rows <= 0 || C <= 0 || K <= 0) return 0;
  const int s = wgrad_splits(rows, C, K);
  return s > 1 ? (long long)s * C * K : 0;
}

extern "C" int egovlp_narrow_linear_bwd(const float* dout, const void* dout_bf16, const void* act, const void* w,
                                        float* dw, float* db, float* dact, float* workspace, int rows, int C, int K,
                                        void* stream) {
  EGOVLP_CHECK_ARG(dout_bf16 && act && w && rows > 0 && C > 0 && K > 0, "narrow_linear_bwd: bad args");
  EGOVLP_CHECK_ARG(K % 8 == 0 && aligned16(act) && aligned16(w) && (!dw || aligned16(dw)) && (!dact || aligned16(dact)),
                   "narrow_linear_bwd: K=%d must be a multiple of 8 and act / w / dw / dact 16B aligned", K);
  EGOVLP_CHECK_ARG(!db || dout, "narrow_linear_bwd: the bias gradient needs the fp32 dout");
  const bf16* d16 = reinterpret_cast<const bf16*>(dout_bf16);
  if (dw) {
    const int splits = wgrad_splits(rows, C, K);
    EGOVLP_CHECK_ARG(splits == 1 || workspace, "narrow_linear_bwd: workspace of %lld floats required",
                     (long long)splits * C * K);
    const int rows_per_split = (rows + splits - 1) / splits;
    dim3 grid((K / 2 + WG_THREADS - 1) / WG_THREADS, (C + WG_COLS - 1) / WG_COLS, (rows + rows_per_split - 1) / rows_per_split);
    narrow_wgrad_kernel<<<grid, WG_THREADS, 0, ST(stream)>>>(d16, reinterpret_cast<const uint32_t*>(act),
                                                             splits > 1 ? workspace : dw, rows, C, K, rows_per_split);
    EGOVLP_CHECK_LAUNCH();
    if (splits > 1) {
      const long long n = (long long)C * K;
      narrow_wgrad_merge_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(workspace, dw, n, (int)grid.z);
      EGOVLP_CHECK_LAUNCH();
    }
  }
  if (db) {
    narrow_bgrad_kernel<<<(C + 7) / 8, 256, 0, ST(stream)>>>(dout, db, rows, C);
    EGOVLP_CHECK_LAUNCH();
  }
  if (dact) {
    EGOVLP_CHECK_ARG(rows <= 65535, "narrow_linear_bwd: rows=%d > 65535", rows);
    dim3 grid((K / 2 + 127) / 128, rows);
    narrow_dgrad_kernel<<<grid, 128, 0, ST(stream)>>>(d16, reinterpret_cast<const uint32_t*>(w), dact, C, K);
    EGOVLP_CHECK_LAUNCH();
  }
  return EGOVLP_OK;
}
