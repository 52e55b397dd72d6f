// Backward of the video tower's dropped branches (model/video_transformer.py:36-52, 100-137, 163-177 with drop_rate /
// drop_path_rate > 0): the gradient reaching a branch whose output the GEMM epilogue masked (EPI_*_DROP) is
// dy * keep / (1 - p) * f(sample), produced here as the bf16 operand of that branch's dgrad, wgrad and bias sums.  The
// keep bits and factors are the epilogue's (one Philox call per four elements of the [rows, W] tensor), so nothing is
// saved between the forward and the backward.
#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

// one thread per four elements; the block's first sample factor is drawn once, a thread past a sample boundary draws
// its own
__global__ void drop_rows_kernel(const void* __restrict__ x, int x_bf16, bf16* __restrict__ y, long long n4, int w4,
                                 float p, unsigned long long seed, uint32_t site, float path_p, uint32_t path_site,
                                 int path_rows) {
  __shared__ float f_first;
  const long long g0 = (long long)blockIdx.x * blockDim.x;
  const long long g = g0 + threadIdx.x;
  const long long b_first = path_rows ? (g0 / w4) / path_rows : 0;
  if (threadIdx.x == 0) f_first = path_rows ? drop_path_factor(seed, path_site, path_p, b_first) : 1.f;
  __syncthreads();
  if (g >= n4) return;
  const long long b = path_rows ? (g / w4) / path_rows : 0;
  const float f = b == b_first ? f_first : drop_path_factor(seed, path_site, path_p, b);
  const float s = (1.f / (1.f - p)) * f;
  const uint4 r = philox4x32_10(dropout_key(seed, site), (unsigned long long)g);
  const uint32_t t = dropout_threshold(p);
  float4 v;
  if (x_bf16) {
    const uint2 u = reinterpret_cast<const uint2*>(x)[g];
    const float2 a = unpack_bf16x2(u.x), c = unpack_bf16x2(u.y);
    v = make_float4(a.x, a.y, c.x, c.y);
  } else {
    v = reinterpret_cast<const float4*>(x)[g];
  }
  v.x = __fmul_rn(v.x, r.x >= t ? s : 0.f);
  v.y = __fmul_rn(v.y, r.y >= t ? s : 0.f);
  v.z = __fmul_rn(v.z, r.z >= t ? s : 0.f);
  v.w = __fmul_rn(v.w, r.w >= t ? s : 0.f);
  reinterpret_cast<uint2*>(y)[g] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
}

}  // namespace
}  // namespace egovlp

using namespace egovlp;

extern "C" int egovlp_drop_rows_bf16(const void* x, int x_is_bf16, void* y_bf16, long long rows, int W, float p,
                                     unsigned long long seed, unsigned int site, float path_p, unsigned int path_site,
                                     int path_rows, void* stream) {
  EGOVLP_CHECK_ARG(x && y_bf16 && rows >= 0 && W > 0 && W % 4 == 0 && path_rows >= 0,
                   "drop_rows: bad args (W=%d must be a positive multiple of 4, path_rows=%d >= 0)", W, path_rows);
  EGOVLP_CHECK_ARG(p >= 0.f && p < 1.f && path_p >= 0.f && path_p < 1.f, "drop_rows: p=%f or path_p=%f outside [0, 1)",
                   p, path_p);
  EGOVLP_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y_bf16)) & (x_is_bf16 ? 7 : 15)) == 0 &&
                       (reinterpret_cast<uintptr_t>(y_bf16) & 7) == 0,
                   "drop_rows: x and y must be aligned to four elements");
  const long long n4 = rows * (W / 4);
  if (n4 == 0) return EGOVLP_OK;
  drop_rows_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, x_is_bf16, reinterpret_cast<bf16*>(y_bf16), n4, W / 4, p, seed, site, path_p, path_site, path_rows);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
