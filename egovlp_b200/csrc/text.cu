// Text-tower specific kernels (DistilBERT, transformers modeling_distilbert.py; call sites model/model.py:117-138):
// embedding gather (+positions), key-padding-masked self-attention for short sequences (L <= 128), and the
// CLS -> ReLU gather in front of txt_proj (model/model.py:73-75,125).  The Linear / LayerNorm / GELU work of the
// tower runs on the shared wgmma GEMM and LayerNorm kernels.  <0.4% of the step's FLOPs: fp32 CUDA-core math.
#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

constexpr int HD = 64;

// out[tok, :] = word[ids[tok], :] + pos[tok % L, :]   (fp32)
__global__ void text_embed_fwd_kernel(const long long* __restrict__ ids, const float* __restrict__ word,
                                      const float* __restrict__ pos, float* __restrict__ out, int ntok, int L, int D) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= (long long)ntok * D) return;
  const int tok = i / D, d = i % D;
  const float4 w = *reinterpret_cast<const float4*>(word + ids[tok] * D + d);
  const float4 p = *reinterpret_cast<const float4*>(pos + (long long)(tok % L) * D + d);
  *reinterpret_cast<float4*>(out + i) = make_float4(w.x + p.x, w.y + p.y, w.z + p.z, w.w + p.w);
}
__global__ void text_embed_bwd_kernel(const long long* __restrict__ ids, const float* __restrict__ dsum,
                                      float* __restrict__ dword, float* __restrict__ dpos, int ntok, int L, int D) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)ntok * D) return;
  const int tok = i / D, d = i % D;
  const float g = dsum[i];
  atomicAdd(dword + ids[tok] * D + d, g);
  atomicAdd(dpos + (long long)(tok % L) * D + d, g);
}

// Deterministic form of text_embed_bwd_kernel, from the ids stably sorted (sorted[i] = ids[perm[i]], perm ascending within
// equal ids): the CTA at the first position of each run of equal ids adds that vocabulary row's token gradients in token
// order; dpos below sums each position over the batch in b order.  Every element is written by one thread.
__global__ void __launch_bounds__(256)
text_embed_bwd_word_det_kernel(const long long* __restrict__ sorted, const long long* __restrict__ perm,
                               const float* __restrict__ dsum, float* __restrict__ dword, int ntok, int D) {
  const int i = blockIdx.x;
  const long long id = sorted[i];
  if (i > 0 && sorted[i - 1] == id) return;
  int end = i + 1;
  while (end < ntok && sorted[end] == id) ++end;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = dword[id * D + d];
    for (int j = i; j < end; ++j) acc += dsum[perm[j] * D + d];
    dword[id * D + d] = acc;
  }
}
__global__ void text_embed_bwd_pos_det_kernel(const float* __restrict__ dsum, float* __restrict__ dpos, int B, int L,
                                              int D) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)L * D) return;
  float acc = dpos[i];
  for (int b = 0; b < B; ++b) acc += dsum[(long long)b * L * D + i];
  dpos[i] = acc;
}

// One CTA per (b, h).  qkv bf16 [B*L, 3*D] (q pre-scaled), mask int64 [B, L] (0 = padded key).
template <bool BWD>
__global__ void __launch_bounds__(256)
text_attn_kernel(const bf16* __restrict__ qkv, const long long* __restrict__ mask, bf16* __restrict__ out,
                 const bf16* __restrict__ dout, bf16* __restrict__ dqkv, int B, int L, int H, float q_scale,
                 float p_drop, unsigned long long seed, uint32_t site) {
  extern __shared__ float sm[];
  const int D = H * HD, b = blockIdx.x / H, h = blockIdx.x % H;
  const int LP = L + 1, RS = HD + 1;
  float* q = sm;                    // [L][65]
  float* k = q + L * RS;
  float* v = k + L * RS;
  float* dO = v + L * RS;           // bwd only
  float* P = BWD ? dO + L * RS : v + L * RS;   // [L][L+1]
  float* keyok = P + L * LP;        // [L]
  uint32_t* keep = reinterpret_cast<uint32_t*>(keyok + L);   // [L][4] bit j of row i: probability (i, j) survives dropout
  const float inv_keep = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  const uint32_t thresh = dropout_threshold(p_drop);
  const unsigned long long dkey = dropout_key(seed, site);
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < L * HD; i += blockDim.x) {
    const int r = i / HD, d = i % HD;
    const bf16* row = qkv + ((long long)(b * L + r)) * 3 * D + h * HD + d;
    q[r * RS + d] = __bfloat162float(row[0]);
    k[r * RS + d] = __bfloat162float(row[D]);
    v[r * RS + d] = __bfloat162float(row[2 * D]);
    if (BWD) dO[r * RS + d] = __bfloat162float(dout[((long long)(b * L + r)) * D + h * HD + d]);
  }
  for (int i = threadIdx.x; i < L; i += blockDim.x) keyok[i] = mask[(long long)b * L + i] != 0 ? 1.f : 0.f;
  __syncthreads();
  // P = softmax(q k^T + key mask)
  for (int i = warp; i < L; i += nw) {
    float mx = -INFINITY;
    for (int j = lane; j < L; j += 32) {
      float s = 0.f;
#pragma unroll 16
      for (int d = 0; d < HD; ++d) s += q[i * RS + d] * k[j * RS + d];
      s = keyok[j] != 0.f ? s : -INFINITY;
      P[i * LP + j] = s;
      mx = fmaxf(mx, s);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int j = lane; j < L; j += 32) {
      const float e = __expf(P[i * LP + j] - mx);
      P[i * LP + j] = e;
      sum += e;
    }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    for (int j = lane; j < L; j += 32) P[i * LP + j] *= inv;
    // attention dropout (HF DistilBERT: `weights = dropout(softmax(scores))`): one Philox draw per (b, h, i, j)
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = lane + 32 * jj;
      bool kp = true;
      if (p_drop > 0.f && j < L)
        kp = philox4x32_10(dkey, ((unsigned long long)blockIdx.x * L + i) * L + j).x >= thresh;
      const uint32_t word = __ballot_sync(0xffffffffu, kp);
      if (lane == 0) keep[i * 4 + jj] = word;
    }
  }
  __syncthreads();
#define DROPF(i, j) (((keep[(i) * 4 + ((j) >> 5)] >> ((j) & 31)) & 1u) ? inv_keep : 0.f)
  if (!BWD) {
    for (int i = warp; i < L; i += nw) {
      float o0 = 0.f, o1 = 0.f;
      for (int j = 0; j < L; ++j) {
        const float p = P[i * LP + j] * DROPF(i, j);
        o0 += p * v[j * RS + lane];
        o1 += p * v[j * RS + lane + 32];
      }
      bf16* dst = out + ((long long)(b * L + i)) * D + h * HD;
      dst[lane] = __float2bfloat16(o0);
      dst[lane + 32] = __float2bfloat16(o1);
    }
    return;
  }
  // ---- backward ----
  // dV_j = sum_i P_ij dO_i
  for (int j = warp; j < L; j += nw) {
    float a0 = 0.f, a1 = 0.f;
    for (int i = 0; i < L; ++i) {
      const float p = P[i * LP + j] * DROPF(i, j);
      a0 += p * dO[i * RS + lane];
      a1 += p * dO[i * RS + lane + 32];
    }
    bf16* dst = dqkv + ((long long)(b * L + j)) * 3 * D + 2 * D + h * HD;
    dst[lane] = __float2bfloat16(a0);
    dst[lane + 32] = __float2bfloat16(a1);
  }
  __syncthreads();
  // dS = P * (dP - delta), in place
  for (int i = warp; i < L; i += nw) {
    float delta = 0.f;
    float dp_local[4];   // L <= 128 -> at most 4 keys per lane
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = lane + jj * 32;
      float dp = 0.f;
      if (j < L) {
#pragma unroll 16
        for (int d = 0; d < HD; ++d) dp += dO[i * RS + d] * v[j * RS + d];
        dp *= DROPF(i, j);                       // d(dropped probs) -> d(softmax probs)
        delta += P[i * LP + j] * dp;
      }
      dp_local[jj] = dp;
    }
    delta = warp_sum(delta);
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = lane + jj * 32;
      if (j < L) P[i * LP + j] *= (dp_local[jj] - delta);
    }
  }
  __syncthreads();
  // dQ_i = q_scale * sum_j dS_ij K_j ;  dK_j = sum_i dS_ij Q_i
  for (int i = warp; i < L; i += nw) {
    float a0 = 0.f, a1 = 0.f;
    for (int j = 0; j < L; ++j) {
      const float s = P[i * LP + j];
      a0 += s * k[j * RS + lane];
      a1 += s * k[j * RS + lane + 32];
    }
    bf16* dst = dqkv + ((long long)(b * L + i)) * 3 * D + h * HD;
    dst[lane] = __float2bfloat16(a0 * q_scale);
    dst[lane + 32] = __float2bfloat16(a1 * q_scale);
  }
  for (int j = warp; j < L; j += nw) {
    float a0 = 0.f, a1 = 0.f;
    for (int i = 0; i < L; ++i) {
      const float s = P[i * LP + j];
      a0 += s * q[i * RS + lane];
      a1 += s * q[i * RS + lane + 32];
    }
    bf16* dst = dqkv + ((long long)(b * L + j)) * 3 * D + D + h * HD;
    dst[lane] = __float2bfloat16(a0);
    dst[lane + 32] = __float2bfloat16(a1);
  }
}

// out[r, :] = bf16(relu(x[r * row_stride, :]))
__global__ void relu_rows_fwd_kernel(const float* __restrict__ x, long long row_stride, bf16* __restrict__ out, int rows,
                                     int D) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * D) return;
  const int r = i / D, d = i % D;
  out[i] = __float2bfloat16(fmaxf(0.f, x[(long long)r * row_stride + d]));
}
// dx[r * row_stride, :] = dh[r, :] * (x > 0)    (other rows of dx untouched)
__global__ void relu_rows_bwd_kernel(const float* __restrict__ x, long long row_stride, const float* __restrict__ dh,
                                     float* __restrict__ dx, int rows, int D) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * D) return;
  const int r = i / D, d = i % D;
  const long long o = (long long)r * row_stride + d;
  dx[o] = x[o] > 0.f ? dh[i] : 0.f;
}

size_t text_attn_smem(int L, bool bwd) {
  return (size_t)((bwd ? 4 : 3) * L * (HD + 1) + L * (L + 1) + L + 4 * L) * sizeof(float);
}

// y = dropout(x) (+ add): fp32 and / or bf16 outputs; the same (seed, site) in the backward reproduces the mask
__global__ void dropout_kernel(const float* __restrict__ x, const float* __restrict__ add, float* __restrict__ y32,
                               bf16* __restrict__ y16, long long n4, float p, unsigned long long seed, uint32_t site) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n4) return;
  const uint4 r = philox4x32_10(dropout_key(seed, site), (unsigned long long)g);
  const uint32_t thresh = dropout_threshold(p);
  const float inv = 1.f / (1.f - p);
  float4 v = reinterpret_cast<const float4*>(x)[g];
  v.x = r.x >= thresh ? v.x * inv : 0.f;
  v.y = r.y >= thresh ? v.y * inv : 0.f;
  v.z = r.z >= thresh ? v.z * inv : 0.f;
  v.w = r.w >= thresh ? v.w * inv : 0.f;
  if (add) {
    const float4 a = reinterpret_cast<const float4*>(add)[g];
    v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
  }
  if (y32) reinterpret_cast<float4*>(y32)[g] = v;
  if (y16) reinterpret_cast<uint2*>(y16)[g] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
}

}  // namespace
}  // namespace egovlp

using namespace egovlp;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int egovlp_text_embed_fwd(const long long* input_ids, const float* word_emb, const float* pos_emb,
                                     float* out, int B, int L, int D, void* stream) {
  EGOVLP_CHECK_ARG(input_ids && word_emb && pos_emb && out && B > 0 && L > 0 && D % 4 == 0, "text_embed_fwd: bad args");
  const long long n = (long long)B * L * D / 4;
  text_embed_fwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(input_ids, word_emb, pos_emb, out, B * L, L, D);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_text_embed_bwd(const long long* input_ids, const float* dsum, float* dword, float* dpos, int B,
                                     int L, int D, void* stream) {
  EGOVLP_CHECK_ARG(input_ids && dsum && dword && dpos && B > 0 && L > 0, "text_embed_bwd: bad args");
  const long long n = (long long)B * L * D;
  text_embed_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(input_ids, dsum, dword, dpos, B * L, L, D);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_text_embed_bwd_det(const long long* sorted_ids, const long long* perm, const float* dsum,
                                         float* dword, float* dpos, int B, int L, int D, void* stream) {
  EGOVLP_CHECK_ARG(sorted_ids && perm && dsum && dword && dpos && B > 0 && L > 0 && D > 0, "text_embed_bwd_det: bad args");
  text_embed_bwd_word_det_kernel<<<B * L, 256, 0, ST(stream)>>>(sorted_ids, perm, dsum, dword, B * L, D);
  EGOVLP_CHECK_LAUNCH();
  const long long n = (long long)L * D;
  text_embed_bwd_pos_det_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(dsum, dpos, B, L, D);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_dropout(const float* x, const float* add, float* y32, void* y16, long long n, float p,
                              unsigned long long seed, unsigned int site, void* stream) {
  EGOVLP_CHECK_ARG(x && (y32 || y16) && n >= 0 && n % 4 == 0, "dropout: bad args (n must be a multiple of 4)");
  EGOVLP_CHECK_ARG(p >= 0.f && p < 1.f, "dropout: p=%f outside [0, 1)", p);
  // the kernel moves four elements at a time: float4 for x, add and y32, uint2 for y16
  EGOVLP_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(add) | reinterpret_cast<uintptr_t>(y32)) &
                    15) == 0 && (reinterpret_cast<uintptr_t>(y16) & 7) == 0,
                   "dropout: x, add and y32 must be 16-byte aligned, y16 8-byte aligned");
  if (n == 0) return EGOVLP_OK;
  dropout_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, ST(stream)>>>(x, add, y32, reinterpret_cast<bf16*>(y16), n / 4,
                                                                          p, seed, site);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_text_attn_fwd(const void* qkv, const long long* attention_mask, void* out, int B, int L, int H,
                                    float p_drop, unsigned long long seed, unsigned int site, void* stream) {
  EGOVLP_CHECK_ARG(qkv && attention_mask && out && B > 0 && H > 0, "text_attn_fwd: bad args");
  EGOVLP_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, "text_attn: p_drop=%f outside [0, 1)", p_drop);
  EGOVLP_CHECK_ARG(L > 0 && L <= 128, "text_attn: L=%d unsupported (1..128)", L);
  const size_t smem = text_attn_smem(L, false);
  auto kern = text_attn_kernel<false>;
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<B * H, 256, smem, ST(stream)>>>(reinterpret_cast<const bf16*>(qkv), attention_mask,
                                        reinterpret_cast<bf16*>(out), nullptr, nullptr, B, L, H, 1.f, p_drop, seed, site);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_text_attn_bwd(const void* qkv, const long long* attention_mask, const void* dout, void* dqkv,
                                    int B, int L, int H, float q_scale, float p_drop, unsigned long long seed,
                                    unsigned int site, void* stream) {
  EGOVLP_CHECK_ARG(qkv && attention_mask && dout && dqkv && B > 0 && H > 0, "text_attn_bwd: bad args");
  EGOVLP_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, "text_attn: p_drop=%f outside [0, 1)", p_drop);
  EGOVLP_CHECK_ARG(L > 0 && L <= 128, "text_attn: L=%d unsupported (1..128)", L);
  const size_t smem = text_attn_smem(L, true);
  auto kern = text_attn_kernel<true>;
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<B * H, 256, smem, ST(stream)>>>(reinterpret_cast<const bf16*>(qkv), attention_mask, nullptr,
                                        reinterpret_cast<const bf16*>(dout), reinterpret_cast<bf16*>(dqkv), B, L, H,
                                        q_scale, p_drop, seed, site);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_relu_rows_fwd(const float* x, long long row_stride, void* out_bf16, int rows, int D,
                                    void* stream) {
  EGOVLP_CHECK_ARG(x && out_bf16 && rows > 0 && D > 0, "relu_rows_fwd: bad args");
  const long long n = (long long)rows * D;
  relu_rows_fwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(x, row_stride, reinterpret_cast<bf16*>(out_bf16), rows, D);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_relu_rows_bwd(const float* x, long long row_stride, const float* dh, float* dx, int rows, int D,
                                    void* stream) {
  EGOVLP_CHECK_ARG(x && dh && dx && rows > 0 && D > 0, "relu_rows_bwd: bad args");
  const long long n = (long long)rows * D;
  relu_rows_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(x, row_stride, dh, dx, rows, D);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
