// Patch-embedding front end of the video tower: im2col (+fp32->bf16) feeding the wgmma GEMM, the
// CLS / positional / temporal embedding table its epilogue adds, and the backward reductions.
// Replaces VideoPatchEmbed.forward + the embedding assembly (model/video_transformer.py:72-77, 304-321):
// Conv2d(k16,s16) == GEMM over unfolded patches; cls cat + tiled pos_embed + repeat_interleaved temporal_embed
// become one [S, D] table R added in the GEMM epilogue (row index = token % S):
//   R[0]         = cls_token + pos_embed[0] - conv_bias       (the CLS patch row is all-zero, so GEMM gives bias)
//   R[1+t*N+n]   = pos_embed[1+n] + temporal_embed[t]
#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

// video fp32 [B, T, C, H, W] -> patches bf16 [B*S, C*P*P]; row b*S + 1 + t*N + py*gw + px; col c*P*P + iy*P + ix.
__global__ void im2col_kernel(const float* __restrict__ video, bf16* __restrict__ patches, int B, int T, int C, int H,
                              int W, int P, int S) {
  const int gw = W / P, gh = H / P, N = gw * gh, K = C * P * P, P4 = P / 4;
  const long long total = (long long)B * T * N * C * P * P4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int x4 = r % P4; r /= P4;
    const int iy = r % P; r /= P;
    const int c = r % C; r /= C;
    const int n = r % N; r /= N;
    const int t = r % T;
    const int b = r / T;
    const int py = n / gw, px = n % gw;
    const float4 v = *reinterpret_cast<const float4*>(
        video + ((((long long)b * T + t) * C + c) * H + (py * P + iy)) * W + px * P + x4 * 4);
    bf16* dst = patches + ((long long)b * S + 1 + t * N + n) * K + c * P * P + iy * P + x4 * 4;
    *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
  // zero the CLS rows
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)B * K / 2;
       i += (long long)gridDim.x * blockDim.x) {
    const int b = i / (K / 2), k2 = i % (K / 2);
    reinterpret_cast<uint32_t*>(patches + (long long)b * S * K)[k2] = 0u;
  }
}

// Same from uint8 frames with the dataset normalisation fused: v = (p / 255 - mean[c]) / std[c]
// (data_loader/transforms.py:38-41 applied on the GPU; H2D traffic drops 4x -- SURVEY.md section 8f row 2).
__global__ void im2col_u8_kernel(const uint8_t* __restrict__ video, bf16* __restrict__ patches, int B, int T, int C,
                                 int H, int W, int P, int S, float3 mean, float3 inv_std) {
  const int gw = W / P, gh = H / P, N = gw * gh, K = C * P * P, P4 = P / 4;
  const long long total = (long long)B * T * N * C * P * P4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int x4 = r % P4; r /= P4;
    const int iy = r % P; r /= P;
    const int c = r % C; r /= C;
    const int n = r % N; r /= N;
    const int t = r % T;
    const int b = r / T;
    const int py = n / gw, px = n % gw;
    const uchar4 v = *reinterpret_cast<const uchar4*>(
        video + ((((long long)b * T + t) * C + c) * H + (py * P + iy)) * W + px * P + x4 * 4);
    const float m = c == 0 ? mean.x : c == 1 ? mean.y : mean.z, is = c == 0 ? inv_std.x : c == 1 ? inv_std.y : inv_std.z;
    const float k = 1.f / 255.f;
    bf16* dst = patches + ((long long)b * S + 1 + t * N + n) * K + c * P * P + iy * P + x4 * 4;
    *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16x2((v.x * k - m) * is, (v.y * k - m) * is),
                                                pack_bf16x2((v.z * k - m) * is, (v.w * k - m) * is));
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)B * K / 2;
       i += (long long)gridDim.x * blockDim.x) {
    const int b = i / (K / 2), k2 = i % (K / 2);
    reinterpret_cast<uint32_t*>(patches + (long long)b * S * K)[k2] = 0u;
  }
}

__global__ void pos_table_kernel(const float* __restrict__ cls, const float* __restrict__ pos,
                                 const float* __restrict__ temporal, const float* __restrict__ bias,
                                 float* __restrict__ R, int T, int N, int D) {
  const int S = 1 + T * N;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)S * D) return;
  const int s = i / D, d = i % D;
  if (s == 0) R[i] = cls[d] + pos[d] - bias[d];
  else {
    const int t = (s - 1) / N, n = (s - 1) % N;
    R[i] = pos[(long long)(1 + n) * D + d] + temporal[(long long)t * D + d];
  }
}

// tmp[s, d] = sum_b dx[b, s, d]
__global__ void sum_over_batch_kernel(const float* __restrict__ dx, float* __restrict__ tmp, int B, long long SD) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= SD) return;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int b = 0; b < B; ++b) {
    const float4 v = *reinterpret_cast<const float4*>(dx + (long long)b * SD + i);
    a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
  }
  *reinterpret_cast<float4*>(tmp + i) = a;
}
// dpos[1+n] += sum_t tmp[1+tN+n];  dtemporal[t] += sum_n tmp[1+tN+n];  dcls += tmp[0]; dpos[0] += tmp[0];
// dbias += sum_{s>=1} tmp[s].     blockIdx.y selects the job, thread per (index, d).
__global__ void embed_reduce_kernel(const float* __restrict__ tmp, float* __restrict__ dcls, float* __restrict__ dpos,
                                    float* __restrict__ dtemporal, float* __restrict__ dbias, int T, int N, int D,
                                    float* __restrict__ dbias_part) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.y == 0) {            // (n, d)
    if (i >= N * D) return;
    const int n = i / D, d = i % D;
    float s = 0.f;
    for (int t = 0; t < T; ++t) s += tmp[(long long)(1 + t * N + n) * D + d];
    dpos[(long long)(1 + n) * D + d] += s;
  } else if (blockIdx.y == 1) {     // (t, d)
    if (i >= T * D) return;
    const int t = i / D, d = i % D;
    float s = 0.f;
    for (int n = 0; n < N; ++n) s += tmp[(long long)(1 + t * N + n) * D + d];
    dtemporal[(long long)t * D + d] += s;
    if (dbias_part) dbias_part[(long long)t * D + d] = s;      // deterministic form: summed over t in order after
    else atomicAdd(dbias + d, s);
  } else {                          // d
    if (i >= D) return;
    dcls[i] += tmp[i];
    dpos[i] += tmp[i];
  }
}

}  // namespace
}  // namespace egovlp

using namespace egovlp;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int egovlp_patch_im2col(const float* video, void* patches_bf16, int B, int T, int C, int H, int W, int P,
                                   void* stream) {
  EGOVLP_CHECK_ARG(video && patches_bf16 && B > 0 && T > 0 && C > 0, "patch_im2col: bad args");
  EGOVLP_CHECK_ARG(P % 4 == 0 && H % P == 0 && W % P == 0 && W % 4 == 0, "patch_im2col: H=%d W=%d P=%d unsupported", H, W, P);
  const int S = 1 + T * (H / P) * (W / P);
  const long long total = (long long)B * T * (H / P) * (W / P) * C * P * (P / 4);
  const long long blocks = (total + 255) / 256;
  const int grid = (int)(blocks > (long long)num_sms() * 32 ? (long long)num_sms() * 32 : blocks);
  im2col_kernel<<<grid, 256, 0, ST(stream)>>>(video, reinterpret_cast<bf16*>(patches_bf16), B, T, C, H, W, P, S);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

extern "C" int egovlp_patch_im2col_u8(const uint8_t* video, void* patches_bf16, int B, int T, int C, int H, int W, int P,
                                      const float* host_mean3, const float* host_std3, void* stream) {
  EGOVLP_CHECK_ARG(video && patches_bf16 && host_mean3 && host_std3 && B > 0 && T > 0 && C == 3, "patch_im2col_u8: bad args");
  EGOVLP_CHECK_ARG(P % 4 == 0 && H % P == 0 && W % P == 0 && W % 4 == 0, "patch_im2col_u8: H=%d W=%d P=%d unsupported", H, W, P);
  const int S = 1 + T * (H / P) * (W / P);
  const long long total = (long long)B * T * (H / P) * (W / P) * C * P * (P / 4);
  const long long blocks = (total + 255) / 256;
  const int grid = (int)(blocks > (long long)num_sms() * 32 ? (long long)num_sms() * 32 : blocks);
  const float3 mean = make_float3(host_mean3[0], host_mean3[1], host_mean3[2]);
  const float3 inv = make_float3(1.f / host_std3[0], 1.f / host_std3[1], 1.f / host_std3[2]);
  im2col_u8_kernel<<<grid, 256, 0, ST(stream)>>>(video, reinterpret_cast<bf16*>(patches_bf16), B, T, C, H, W, P, S, mean, inv);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

extern "C" int egovlp_video_pos_table(const float* cls_token, const float* pos_embed, const float* temporal_embed,
                                      const float* conv_bias, float* table, int T, int N, int D, void* stream) {
  EGOVLP_CHECK_ARG(cls_token && pos_embed && temporal_embed && conv_bias && table && T > 0 && N > 0 && D > 0,
                   "video_pos_table: bad args");
  const long long n = (long long)(1 + T * N) * D;
  pos_table_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(cls_token, pos_embed, temporal_embed, conv_bias,
                                                                      table, T, N, D);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

static int video_embed_bwd_impl(const float* dx, float* tmp_SD, float* dcls, float* dpos, float* dtemporal,
                                float* dbias, float* dbias_part, int B, int T, int N, int D, void* stream) {
  EGOVLP_CHECK_ARG(dx && tmp_SD && dcls && dpos && dtemporal && dbias && D % 4 == 0, "video_embed_bwd: bad args");
  const long long SD = (long long)(1 + T * N) * D;
  sum_over_batch_kernel<<<(unsigned)((SD / 4 + 255) / 256), 256, 0, ST(stream)>>>(dx, tmp_SD, B, SD);
  EGOVLP_CHECK_LAUNCH();
  const int mx = max(N, T) * D;
  dim3 grid((mx + 255) / 256, 3);
  embed_reduce_kernel<<<grid, 256, 0, ST(stream)>>>(tmp_SD, dcls, dpos, dtemporal, dbias, T, N, D, dbias_part);
  EGOVLP_CHECK_LAUNCH();
  return dbias_part ? ordered_sum(dbias_part, T, D, dbias, ST(stream)) : EGOVLP_OK;
}

extern "C" int egovlp_video_embed_bwd(const float* dx, float* tmp_SD, float* dcls, float* dpos, float* dtemporal,
                                      float* dbias, int B, int T, int N, int D, void* stream) {
  return video_embed_bwd_impl(dx, tmp_SD, dcls, dpos, dtemporal, dbias, nullptr, B, T, N, D, stream);
}

extern "C" int egovlp_video_embed_bwd_det(const float* dx, float* tmp_SD, float* dcls, float* dpos, float* dtemporal,
                                          float* dbias, float* ws_TD, int B, int T, int N, int D, void* stream) {
  EGOVLP_CHECK_ARG(ws_TD, "video_embed_bwd_det: null workspace");
  return video_embed_bwd_impl(dx, tmp_SD, dcls, dpos, dtemporal, dbias, ws_TD, B, T, N, D, stream);
}
