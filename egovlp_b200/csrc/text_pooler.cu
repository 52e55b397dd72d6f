// BERT pooler head of the text tower (transformers modeling_bert.py, BertPooler): y = tanh(W_p h_CLS + b_p), the
// `pooler_output` the reference embeds captions with for `text_params['model'] = 'bert*'` (model/model.py:117-131),
// optionally followed by the ReLU in front of txt_proj (model/model.py:73-75).  B x D x D FMAs (19 M at B = 32,
// D = 768): fp32 CUDA-core math.  Built without --use_fast_math, so tanhf is the IEEE-accurate one.
//
// Every product is a 32 x 32 output tile per CTA whose contraction runs in 32-wide chunks in a fixed order, one
// thread owning four outputs: no atomics, the results are bitwise reproducible.
#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

constexpr int PT = 32;           // output tile edge and contraction chunk
constexpr int POOL_THREADS = 256;

// acc[q] = sum_r A(r, i0 + 4 * warp + q) * Bop(r, j0 + lane), r in [0, R).  A / Bop are (r, index) -> float loaders
// returning 0 outside the operand; A_RC / B_RC say whether r is the contiguous index in memory (the loader then walks
// r across the lanes, so the loads coalesce).  colsum (optional, lanes of warp 0): colsum[lane] = sum_r A(r, i0 + lane).
template <bool A_RC, bool B_RC, class LA, class LB>
__device__ __forceinline__ void pool_tile(LA A, LB Bop, int R, int i0, int j0, float (&acc)[4], float* colsum) {
  __shared__ float As[PT][PT + 1], Bs[PT][PT + 1];       // [r][i], [r][j]
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
#pragma unroll
  for (int q = 0; q < 4; ++q) acc[q] = 0.f;
  float cs = 0.f;
  for (int r0 = 0; r0 < R; r0 += PT) {
#pragma unroll
    for (int e = t; e < PT * PT; e += POOL_THREADS) {
      const int x = e % PT, y = e / PT;
      const int ar = A_RC ? x : y, ai = A_RC ? y : x;
      const int br = B_RC ? x : y, bj = B_RC ? y : x;
      As[ar][ai] = r0 + ar < R ? A(r0 + ar, i0 + ai) : 0.f;
      Bs[br][bj] = r0 + br < R ? Bop(r0 + br, j0 + bj) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int r = 0; r < PT; ++r) {
      const float b = Bs[r][lane];
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] += As[r][4 * warp + q] * b;
    }
    if (colsum && warp == 0) {
#pragma unroll 8
      for (int r = 0; r < PT; ++r) cs += As[r][lane];
    }
    __syncthreads();
  }
  if (colsum && warp == 0) colsum[lane] = cs;
}

// grid: ceil(B / 32) x ceil(D / 32) tiles of y [B, D] (i = b, j = n), contraction over k
__global__ void __launch_bounds__(POOL_THREADS)
text_pooler_fwd_kernel(const float* __restrict__ h, long long row_stride, const float* __restrict__ w,
                       const float* __restrict__ bias, float* __restrict__ y, bf16* __restrict__ relu16, int B, int D) {
  const int nt = (D + PT - 1) / PT;
  const int i0 = (blockIdx.x / nt) * PT, j0 = (blockIdx.x % nt) * PT;
  auto A = [&](int k, int b) { return b < B ? h[(long long)b * row_stride + k] : 0.f; };
  auto W = [&](int k, int n) { return n < D ? w[(long long)n * D + k] : 0.f; };
  float acc[4];
  pool_tile<true, true>(A, W, D, i0, j0, acc, nullptr);
  const int n = j0 + (threadIdx.x & 31);
  if (n >= D) return;
  const float bn = bias[n];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int b = i0 + 4 * (threadIdx.x >> 5) + q;
    if (b < B) {
      const float v = tanhf(acc[q] + bn);
      y[(long long)b * D + n] = v;
      if (relu16) relu16[(long long)b * D + n] = __float2bfloat16(fmaxf(v, 0.f));
    }
  }
}

// dz(b, n) = g(b, n) * [y > 0 when relu] * (1 - y^2), recomputed wherever a tile loads it.
// CTAs [0, nt * nt): dW tile (i = n, j = k) over b, the j = 0 column of tiles also writes db;
// CTAs [nt * nt, nt * nt + ceil(B / 32) * nt): dh tile (i = b, j = k) over n, written to the strided CLS rows.
__global__ void __launch_bounds__(POOL_THREADS)
text_pooler_bwd_kernel(const float* __restrict__ g, const float* __restrict__ y, bool relu,
                       const float* __restrict__ h, long long row_stride, const float* __restrict__ w,
                       float* __restrict__ dw, float* __restrict__ db, float* __restrict__ dh, int B, int D) {
  __shared__ float db_tile[PT];
  const int nt = (D + PT - 1) / PT;
  auto dz = [&](int b, int n) {
    if (b >= B || n >= D) return 0.f;
    const long long o = (long long)b * D + n;
    const float v = y[o];
    return relu && !(v > 0.f) ? 0.f : g[o] * (1.f - v * v);
  };
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float acc[4];
  if (blockIdx.x < nt * nt) {
    const int i0 = (blockIdx.x / nt) * PT, j0 = (blockIdx.x % nt) * PT;
    auto A = [&](int b, int n) { return dz(b, n); };
    auto H = [&](int b, int k) { return k < D ? h[(long long)b * row_stride + k] : 0.f; };
    const bool with_db = j0 == 0;
    pool_tile<false, false>(A, H, B, i0, j0, acc, with_db ? db_tile : nullptr);
    const int k = j0 + lane;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int n = i0 + 4 * warp + q;
      if (n < D && k < D) dw[(long long)n * D + k] = acc[q];
    }
    if (with_db && warp == 0 && i0 + lane < D) db[i0 + lane] = db_tile[lane];
  } else {
    const int t = blockIdx.x - nt * nt;
    const int i0 = (t / nt) * PT, j0 = (t % nt) * PT;
    auto A = [&](int n, int b) { return dz(b, n); };
    auto W = [&](int n, int k) { return k < D ? w[(long long)n * D + k] : 0.f; };
    pool_tile<true, false>(A, W, D, i0, j0, acc, nullptr);
    const int k = j0 + lane;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int b = i0 + 4 * warp + q;
      if (b < B && k < D) dh[(long long)b * row_stride + k] = acc[q];
    }
  }
}

}  // namespace
}  // namespace egovlp

using namespace egovlp;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

static bool pooler_dims_ok(int B, int D, long long row_stride) {
  return B >= 1 && D >= 4 && D <= 1024 && D % 4 == 0 && row_stride >= D &&
         (long long)((B + PT - 1) / PT) * ((D + PT - 1) / PT) + (long long)((D + PT - 1) / PT) * ((D + PT - 1) / PT) <
             (1ll << 31);
}

extern "C" int egovlp_text_pooler_fwd(const float* h, long long row_stride, const float* weight, const float* bias,
                                      float* y, void* relu_bf16, int B, int D, void* stream) {
  EGOVLP_CHECK_ARG(h && weight && bias && y, "text_pooler_fwd: null pointer");
  EGOVLP_CHECK_ARG(pooler_dims_ok(B, D, row_stride),
                   "text_pooler_fwd: B=%d D=%d row_stride=%lld unsupported (B >= 1, 4 <= D <= 1024, D %% 4 == 0, "
                   "row_stride >= D)", B, D, row_stride);
  const int nt = (D + PT - 1) / PT, bt = (B + PT - 1) / PT;
  text_pooler_fwd_kernel<<<(unsigned)(bt * nt), POOL_THREADS, 0, ST(stream)>>>(
      h, row_stride, weight, bias, y, reinterpret_cast<bf16*>(relu_bf16), B, D);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

extern "C" int egovlp_text_pooler_bwd(const float* grad, const float* y, int relu, const float* h, long long row_stride,
                                      const float* weight, float* dweight, float* dbias, float* dh, int B, int D,
                                      void* stream) {
  EGOVLP_CHECK_ARG(grad && y && h && weight && dweight && dbias && dh, "text_pooler_bwd: null pointer");
  EGOVLP_CHECK_ARG(pooler_dims_ok(B, D, row_stride),
                   "text_pooler_bwd: B=%d D=%d row_stride=%lld unsupported (B >= 1, 4 <= D <= 1024, D %% 4 == 0, "
                   "row_stride >= D)", B, D, row_stride);
  const int nt = (D + PT - 1) / PT, bt = (B + PT - 1) / PT;
  text_pooler_bwd_kernel<<<(unsigned)(nt * nt + bt * nt), POOL_THREADS, 0, ST(stream)>>>(
      grad, y, relu != 0, h, row_stride, weight, dweight, dbias, dh, B, D);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
