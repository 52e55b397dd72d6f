// Spatial attention of the video tower for large frames (model/video_transformer.py:109-130, space mode): the tiled
// attention of tiled_attention.cuh, forward and backward, for 1 <= N <= 1024 patches per frame.  The divided attention
// (attention.cu) holds a whole frame in one CTA and stops at N = 255; the engine calls these kernels above that.
//
// Same contract as egovlp_divided_attn_* with mode = 1: qkv bf16 [B*S, 3D] read in place (q pre-scaled), S = 1 + T*N,
// row 1 + f*N + n = patch n of frame f, row 0 = the sample's CLS token; out bf16 [B*S, D] with the heads merged, lse
// fp32 [B, H, S].  Head dim 64.
//
// A group is (b, head, frame).  Its rows are indexed r = 0 .. N: r = 0 is the CLS token, r = 1 + n patch n of the frame.
// Queries and keys share that index, so the CLS key is the extra key ahead of the frame's first 64-key tile and the CLS
// query the extra query ahead of its first 64-query tile.  Every pair (r, j) with r, j <= N is attended except the CLS
// query on the CLS key in frames f > 0: over the T groups the CLS query then sees every key of the sample once.  Every
// key tile of the group is visited; only the last one holds keys past N.
//
// The CLS rows, with no floating-point atomics (everything is bitwise reproducible run to run):
//   forward:  each group writes the CLS query's un-normalised (max, sum, acc) partial; space_cls_merge_kernel merges
//             the T partials of a (b, head) in frame order and writes out row 0 and lse[b, h, 0];
//   backward: each group writes its fp32 partial of the CLS row's dq, dk and dv; space_cls_grad_kernel sums the T
//             partials in frame order.
// In the backward P is recomputed from lse: the CLS query's lse is the merged one, over all S keys.
#include "egovlp_b200.h"
#include "tiled_attention.cuh"

namespace egovlp {
namespace {

constexpr int MAX_N = 1024;
constexpr int PART = 66;                   // CLS-query partial: acc[64], max, sum

// The layout policy of tiled_attention.cuh for a (b, head, frame) group: row r of group (b, f) is matrix row
// r ? b*S + f*N + r : b*S, and entry r ? f*N + r : 0 of the (b, head)'s [S] slice of lse / delta.
struct SpaceAttn {
  struct Args {
    float* part;   // the CLS rows' fp32 partials: [B, H, T, PART] in the forward, [B, H, T, 3, 64] in the backward
    int T, N, H;
  };
  struct Smem {};
  static constexpr bool kCls = true, kDropout = false;

  float* part;
  int b, f, h, T, H, fn, rows;
  long long bS, fN, lrow;   // b*S, b*S + f*N, (b*H + h)*S

  __device__ SpaceAttn(const Args& a, int h_, Smem&) : part(a.part), h(h_), T(a.T), H(a.H), rows(a.N + 1) {
    const int bf = blockIdx.z;
    b = bf / T;
    f = bf - b * T;
    fn = f * a.N;
    bS = (long long)b * (1 + (long long)T * a.N);
    fN = bS + (long long)f * a.N;
    lrow = ((long long)b * H + h) * (1 + T * a.N);
  }
  __device__ long long row(int r) const { return r ? fN + r : bS; }
  __device__ long long stat(int r) const { return lrow + (r ? fn + r : 0); }

  __device__ uint32_t key_tiles() const { return (1u << ((rows + TILE - 1) / TILE)) - 1; }
  __device__ bool masked(int kt) const { return kt == (rows - 1) / TILE; }   // only the last tile holds keys past N
  __device__ uint32_t key_bits(int kt, int jl, int t) const {
    const int c = kt * TILE + jl + 2 * t;
    return (uint32_t)(c < rows) | ((uint32_t)(c + 1 < rows) << 1);
  }
  __device__ bool key_ok(int j) const { return j < rows; }
  __device__ bool skips_pair00() const { return f > 0; }

  // this group's partial of its (b, head)'s CLS rows
  __device__ float* cls_part(int floats) const { return part + (((long long)b * H + h) * T + f) * floats; }
  // the CLS query's un-normalised partial, for space_cls_merge_kernel
  __device__ void cls_fwd(const float (&o)[8][4], float m, float l, int t) const {
    float* dst = cls_part(PART);
#pragma unroll
    for (int j = 0; j < 8; ++j) { dst[j * 8 + 2 * t] = o[j][0]; dst[j * 8 + 2 * t + 1] = o[j][1]; }
    if (t == 0) { dst[64] = m; dst[65] = l; }
  }
  // the CLS key's dk, dv partials, for space_cls_grad_kernel
  __device__ void cls_dkv(const float (&dk)[8][4], const float (&dv)[8][4], int t) const {
    float* dst = cls_part(3 * HD);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      dst[HD + j * 8 + 2 * t] = dk[j][0]; dst[HD + j * 8 + 2 * t + 1] = dk[j][1];
      dst[2 * HD + j * 8 + 2 * t] = dv[j][0]; dst[2 * HD + j * 8 + 2 * t + 1] = dv[j][1];
    }
  }
  // the CLS query's dq partial (q_scale applied by space_cls_grad_kernel)
  __device__ void cls_dq(const float (&dq)[8][4], int t) const {
    float* dst = cls_part(3 * HD);
#pragma unroll
    for (int j = 0; j < 8; ++j) { dst[j * 8 + 2 * t] = dq[j][0]; dst[j * 8 + 2 * t + 1] = dq[j][1]; }
  }
};

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
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(tiled_attn_fwd_kernel<SpaceAttn>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)FWD_SMEM));
  bf16* o = reinterpret_cast<bf16*>(out);
  const dim3 grid((N + 1 + TILE - 1) / TILE, H, B * T);
  tiled_attn_fwd_kernel<SpaceAttn><<<grid, NTHREADS, FWD_SMEM, ST(stream)>>>(reinterpret_cast<const bf16*>(qkv), o, lse,
                                                                            SpaceAttn::Args{workspace, T, N, H});
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
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(tiled_attn_bwd_kv_kernel<SpaceAttn>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM));
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(tiled_attn_bwd_q_kernel<SpaceAttn>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM));
  const int S = 1 + T * N;
  const bf16* q = reinterpret_cast<const bf16*>(qkv);
  const bf16* g = reinterpret_cast<const bf16*>(dout);
  bf16* dq = reinterpret_cast<bf16*>(dqkv);
  float* delta = workspace;
  float* dcls = workspace + (long long)B * H * S;
  const long long rows = (long long)B * S, nthr = rows * H * 8;
  tiled_attn_delta_kernel<<<(unsigned)((nthr + 255) / 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const bf16*>(out), g, delta, rows, S, H);
  EGOVLP_CHECK_LAUNCH();
  const dim3 grid((N + 1 + TILE - 1) / TILE, H, B * T);
  const SpaceAttn::Args a{dcls, T, N, H};
  tiled_attn_bwd_kv_kernel<SpaceAttn><<<grid, NTHREADS, BWD_SMEM, ST(stream)>>>(q, lse, delta, g, dq, a);
  EGOVLP_CHECK_LAUNCH();
  tiled_attn_bwd_q_kernel<SpaceAttn><<<grid, NTHREADS, BWD_SMEM, ST(stream)>>>(q, lse, delta, g, dq, q_scale, a);
  EGOVLP_CHECK_LAUNCH();
  const int n = B * H * 3 * HD;
  space_cls_grad_kernel<<<(n + 255) / 256, 256, 0, ST(stream)>>>(dcls, dq, B, T, H, S, q_scale);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
