// Similarity + contrastive losses of the EgoVLP step, forward and backward, in fp32.
//
// Replaces sim_matrix (model/model.py:189-197), EgoNCE / NormSoftmaxLoss / MaxMarginRankingLoss
// (model/loss.py:13-25, 34-53, 63-90), the dual-softmax rescoring (run/test_epic.py:137-143) and the EgoMCQ
// scoring (trainer/trainer_egoclip.py:204-215 + model/metric.py:227).  The G x G problem is tiny (G = 512 at
// 8 x 64): everything stays fp32 (logits are x / 0.05, so bf16 would cost 1e-1 in the exponent) and is
// bandwidth / latency bound; the kernels are plain CUDA-core code.
//   EgoNCE = -mean_i[LSE_pos_r(i) - LSE_all_r(i)] - mean_j[LSE_pos_c(j) - LSE_all_c(j)]   over logits x/tau, with
//   positives mask(i,j) = (i == j) or (share a verb AND share a noun)  -- the same (un-transposed) mask in both
//   directions, as the reference does (model/loss.py:47-51).
#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

// an[i,:] = a[i,:] / max(||a_i||, eps); norm[i] = ||a_i||   (one warp per row)
__global__ void rownorm_fwd_kernel(const float* __restrict__ a, float* __restrict__ an, float* __restrict__ norm,
                                   int rows, int C, float eps) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) { const float v = a[(long long)r * C + c]; s += v * v; }
  const float n = sqrtf(warp_sum(s));
  const float inv = 1.f / fmaxf(n, eps);
  for (int c = lane; c < C; c += 32) an[(long long)r * C + c] = a[(long long)r * C + c] * inv;
  if (lane == 0 && norm) norm[r] = n;
}
// da = (dan - an * <an, dan>) / ||a||  if ||a|| > eps, else dan / eps
__global__ void rownorm_bwd_kernel(const float* __restrict__ dan, const float* __restrict__ an,
                                   const float* __restrict__ norm, float* __restrict__ da, int rows, int C, float eps) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float n = norm[r];
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += an[(long long)r * C + c] * dan[(long long)r * C + c];
  s = warp_sum(s);
  for (int c = lane; c < C; c += 32) {
    const float g = dan[(long long)r * C + c];
    da[(long long)r * C + c] = n > eps ? (g - an[(long long)r * C + c] * s) / n : g / eps;
  }
}

// C[m,n] = alpha * sum_k A[m*sam + k*sak] * B[n*sbn + k*sbk] + beta * C[m,n]     (32x32 tiles, fp32)
__global__ void __launch_bounds__(256)
sgemm_strided_kernel(const float* __restrict__ A, long long sam, long long sak, const float* __restrict__ B,
                     long long sbn, long long sbk, float* __restrict__ Cm, long long ldc, int M, int N, int K,
                     float alpha, float beta) {
  __shared__ float As[32][33], Bs[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  const int m0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k0 = 0; k0 < K; k0 += 32) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int rr = ty + i * 8;
      // pick the thread->element map that makes the unit-stride index the fast one
      int am, ak, bn, bk;
      if (sak == 1) { am = rr; ak = tx; } else { am = tx; ak = rr; }
      if (sbk == 1) { bn = rr; bk = tx; } else { bn = tx; bk = rr; }
      As[am][ak] = (m0 + am < M && k0 + ak < K) ? A[(long long)(m0 + am) * sam + (long long)(k0 + ak) * sak] : 0.f;
      Bs[bn][bk] = (n0 + bn < N && k0 + bk < K) ? B[(long long)(n0 + bn) * sbn + (long long)(k0 + bk) * sbk] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 32; ++k) {
      const float b = Bs[tx][k];
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] += As[ty + i * 8][k] * b;
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty + i * 8, n = n0 + tx;
    if (m < M && n < N) {
      float* c = Cm + (long long)m * ldc + n;
      *c = alpha * acc[i] + (beta != 0.f ? beta * *c : 0.f);
    }
  }
}

__global__ void pack_multihot_kernel(const float* __restrict__ v, uint32_t* __restrict__ bits, int G, int C, int W) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G * W) return;
  const int r = i / W, w = i % W;
  uint32_t m = 0;
  for (int j = 0; j < 32; ++j) {
    const int c = w * 32 + j;
    if (c < C && v[(long long)r * C + c] != 0.f) m |= 1u << j;
  }
  bits[i] = m;
}
// mode 0: identity; 1: verb & noun; 2: noun only; 3: verb only   (always OR the diagonal)
__global__ void mask_from_bits_kernel(const uint32_t* __restrict__ vb, int Wv, const uint32_t* __restrict__ nb, int Wn,
                                      uint8_t* __restrict__ mask, int G, int mode) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (j >= G) return;
  bool sv = false, sn = false;
  if (mode == 1 || mode == 3) for (int w = 0; w < Wv; ++w) sv |= (vb[i * Wv + w] & vb[j * Wv + w]) != 0;
  if (mode == 1 || mode == 2) for (int w = 0; w < Wn; ++w) sn |= (nb[i * Wn + w] & nb[j * Wn + w]) != 0;
  const bool pos = (i == j) || (mode == 1 ? (sv && sn) : mode == 2 ? sn : mode == 3 ? sv : false);
  mask[(long long)i * G + j] = pos ? 1 : 0;
}
// the reference's own formulation from float similarity matrices: (sim_v * sim_n + I) > 0  (model/loss.py:35-47)
__global__ void mask_from_sims_kernel(const float* __restrict__ sv, const float* __restrict__ sn,
                                      uint8_t* __restrict__ mask, int G, int mode) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)G * G) return;
  const int i = idx / G, j = idx % G;
  const float eye = (i == j) ? 1.f : 0.f;
  float m = eye;
  if (mode == 1) m = sv[idx] * sn[idx] + eye;
  else if (mode == 2) m = sn[idx] + eye;
  else if (mode == 3) m = sv[idx] + eye;
  mask[idx] = m > 0.f ? 1 : 0;
}

// stats[0:G] = LSE_all rows, [G:2G] = LSE_pos rows, [2G:3G] = LSE_all cols, [3G:4G] = LSE_pos cols (natural log,
// over logits x * inv_temp).  One warp per row (blockIdx.y == 0) or per column (blockIdx.y == 1).
__global__ void nce_stats_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask, int G, float inv_temp,
                                 float* __restrict__ stats) {
  const int idx = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (idx >= G) return;
  const bool col = blockIdx.y == 1;
  const long long s_fast = col ? G : 1, base = col ? idx : (long long)idx * G;
  float mx = -INFINITY;
  for (int k = lane; k < G; k += 32) mx = fmaxf(mx, x[base + k * s_fast] * inv_temp);
  mx = warp_max(mx);
  float sa = 0.f, sp = 0.f;
  for (int k = lane; k < G; k += 32) {
    const float e = __expf(x[base + k * s_fast] * inv_temp - mx);
    sa += e;
    // column j sums softmax_col_j(i) * mask[j, i]: the reference multiplies j_sm (= x^T softmax) by the
    // UN-transposed mask (model/loss.py:50), i.e. row j of the mask for column j
    if (mask[(long long)idx * G + k]) sp += e;
  }
  sa = warp_sum(sa); sp = warp_sum(sp);
  if (lane == 0) {
    stats[(col ? 2 : 0) * G + idx] = mx + logf(sa);
    stats[(col ? 3 : 1) * G + idx] = mx + logf(sp);
  }
}
__global__ void nce_loss_kernel(const float* __restrict__ stats, int G, float* __restrict__ loss) {
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < G; i += blockDim.x) s += (stats[G + i] - stats[i]) + (stats[3 * G + i] - stats[2 * G + i]);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    s = warp_sum(s);
    if (threadIdx.x == 0) *loss = -s / G;
  }
}
// dx[i,j] = gscale * (-1/G) * inv_temp * [ m_ij e^{z - lp_r[i]} - e^{z - la_r[i]} + m_ji e^{z - lp_c[j]} - e^{z - la_c[j]} ]
__global__ void nce_bwd_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask,
                               const float* __restrict__ stats, int G, float inv_temp, const float* __restrict__ gscale,
                               float* __restrict__ dx) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)G * G) return;
  const int i = idx / G, j = idx % G;
  const float z = x[idx] * inv_temp, m = mask[idx] ? 1.f : 0.f, mt = mask[(long long)j * G + i] ? 1.f : 0.f;
  const float t = m * __expf(z - stats[G + i]) - __expf(z - stats[i]) + mt * __expf(z - stats[3 * G + j]) -
                  __expf(z - stats[2 * G + j]);
  dx[idx] = -(gscale ? *gscale : 1.f) * inv_temp / G * t;
}

// MaxMarginRankingLoss: mean over (i != j if fix_norm) of relu(m_i - (x_ii - x_ij)) + relu(m_i - (x_ii - x_ji)), /2.
// m_i = margin (model/loss.py:63-90) or margin * weight[i] (AdaptiveMaxMarginRankingLoss, model/loss.py:100-133: the
// weight is expanded along the row of the anchor i in BOTH directions).
__global__ void maxmargin_fwd_kernel(const float* __restrict__ x, const float* __restrict__ weight, int G, float margin,
                                     int fix_norm, float* __restrict__ loss, float* __restrict__ part) {
  __shared__ float red[32];
  float s = 0.f;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < (long long)G * G;
       idx += (long long)gridDim.x * blockDim.x) {
    const int i = idx / G, j = idx % G;
    if (fix_norm && i == j) continue;
    const float d = x[(long long)i * G + i], m = weight ? margin * weight[i] : margin;
    s += fmaxf(0.f, m - (d - x[idx])) + fmaxf(0.f, m - (d - x[(long long)j * G + i]));
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    s = warp_sum(s);
    const float denom = fix_norm ? 2.f * G * (G - 1) : 2.f * G * G;
    if (threadIdx.x == 0) {
      if (part) part[blockIdx.x] = s / denom;      // deterministic form: merged in CTA order
      else atomicAdd(loss, s / denom);
    }
  }
}
// dx accumulated with atomics: each (i,j) term touches x_ii, x_ij, x_ji
__global__ void maxmargin_bwd_kernel(const float* __restrict__ x, const float* __restrict__ weight, int G, float margin,
                                     int fix_norm, const float* __restrict__ gscale, float* __restrict__ dx) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)G * G) return;
  const int i = idx / G, j = idx % G;
  if (fix_norm && i == j) return;
  const float denom = fix_norm ? 2.f * G * (G - 1) : 2.f * G * G;
  const float g = (gscale ? *gscale : 1.f) / denom;
  const float d = x[(long long)i * G + i], m = weight ? margin * weight[i] : margin;
  float dd = 0.f;
  if (m - (d - x[idx]) > 0.f) { atomicAdd(dx + idx, g); dd -= g; }
  if (m - (d - x[(long long)j * G + i]) > 0.f) { atomicAdd(dx + (long long)j * G + i, g); dd -= g; }
  if (dd != 0.f) atomicAdd(dx + (long long)i * G + i, dd);
}
// Gather form of maxmargin_bwd_kernel (deterministic: each element written by one thread).  Off the diagonal, dx_ij
// takes the term of anchor i (margin m_i against x_ij) and then the term of anchor j (margin m_j against its column
// entry x_ij); the diagonal sums its row's terms in j order.  A pair (i, i) contributes +g +g -2g = 0 and is skipped.
__global__ void maxmargin_bwd_gather_kernel(const float* __restrict__ x, const float* __restrict__ weight, int G,
                                            float margin, int fix_norm, const float* __restrict__ gscale,
                                            float* __restrict__ dx) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)G * G) return;
  const int i = idx / G, j = idx % G;
  const float denom = fix_norm ? 2.f * G * (G - 1) : 2.f * G * G;
  const float g = (gscale ? *gscale : 1.f) / denom;
  const float di = x[(long long)i * G + i], mi = weight ? margin * weight[i] : margin;
  float v = 0.f;
  if (i != j) {
    const float dj = x[(long long)j * G + j], mj = weight ? margin * weight[j] : margin;
    if (mi - (di - x[idx]) > 0.f) v += g;
    if (mj - (dj - x[idx]) > 0.f) v += g;
  } else {
    for (int k = 0; k < G; ++k) {
      if (k == i) continue;
      if (mi - (di - x[(long long)i * G + k]) > 0.f) v -= g;
      if (mi - (di - x[(long long)k * G + i]) > 0.f) v -= g;
    }
  }
  dx[idx] = v;
}

// dual softmax: y = softmax(s / temp, dim=1) * s ; out = softmax(y, dim=0)
__global__ void dsm_rows_kernel(const float* __restrict__ s, float* __restrict__ y, int R, int Cc, float inv_temp) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= R) return;
  float mx = -INFINITY;
  for (int c = lane; c < Cc; c += 32) mx = fmaxf(mx, s[(long long)r * Cc + c] * inv_temp);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane; c < Cc; c += 32) sum += expf(s[(long long)r * Cc + c] * inv_temp - mx);
  sum = warp_sum(sum);
  for (int c = lane; c < Cc; c += 32) {
    const float v = s[(long long)r * Cc + c];
    y[(long long)r * Cc + c] = expf(v * inv_temp - mx) / sum * v;
  }
}
__global__ void dsm_cols_kernel(float* __restrict__ y, int R, int Cc) {   // thread per column, coalesced
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= Cc) return;
  float mx = -INFINITY;
  for (int r = 0; r < R; ++r) mx = fmaxf(mx, y[(long long)r * Cc + c]);
  float sum = 0.f;
  for (int r = 0; r < R; ++r) sum += expf(y[(long long)r * Cc + c] - mx);
  const float inv = 1.f / sum;
  for (int r = 0; r < R; ++r) y[(long long)r * Cc + c] = expf(y[(long long)r * Cc + c] - mx) * inv;
}

// EgoMCQ: scores[q,k] = cos(text[q], video[q,k]); pred[q] = argmax_k (first max wins).  One warp per query.
__global__ void egomcq_kernel(const float* __restrict__ text, const float* __restrict__ video,
                              float* __restrict__ scores, long long* __restrict__ pred, int Q, int Kc, int C, float eps) {
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (q >= Q) return;
  float tn = 0.f;
  for (int c = lane; c < C; c += 32) { const float v = text[(long long)q * C + c]; tn += v * v; }
  tn = fmaxf(sqrtf(warp_sum(tn)), eps);
  float best = -INFINITY;
  int besti = 0;
  for (int k = 0; k < Kc; ++k) {
    const float* vr = video + ((long long)q * Kc + k) * C;
    float vn = 0.f;
    for (int c = lane; c < C; c += 32) { const float v = vr[c]; vn += v * v; }
    vn = fmaxf(sqrtf(warp_sum(vn)), eps);
    // normalise both sides first, then dot: same association as sim_matrix (a/|a|) @ (b/|b|)^T
    float d2 = 0.f;
    for (int c = lane; c < C; c += 32) d2 += (text[(long long)q * C + c] / tn) * (vr[c] / vn);
    d2 = warp_sum(d2);
    if (lane == 0) scores[(long long)q * Kc + k] = d2;
    if (d2 > best) { best = d2; besti = k; }
  }
  if (lane == 0) pred[q] = besti;
}

// Softmax cross-entropy (model/loss.py:135-141 = nn.CrossEntropyLoss() with its defaults: mean over the rows whose
// target is not ignore_index, no class weights, no label smoothing).  One warp per row: max-subtracted log-sum-exp,
// row loss = lse - x[target]; 0 on an ignored row, NaN for a target outside [0, C) (never used as an index).
__device__ __forceinline__ bool ce_bad_target(long long t, int C, int ignore) { return t != ignore && (t < 0 || t >= C); }

__global__ void ce_rows_kernel(const float* __restrict__ x, long long ld, const long long* __restrict__ target, int G,
                               int C, int ignore, float* __restrict__ lse, float* __restrict__ row_loss) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= G) return;
  const float* xr = x + (long long)r * ld;
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, xr[c]);
  mx = warp_max(mx);
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += expf(xr[c] - mx);
  s = warp_sum(s);
  if (lane == 0) {
    const float l = mx + logf(s);
    const long long t = target[r];
    lse[r] = l;
    row_loss[r] = t == ignore ? 0.f : ce_bad_target(t, C, ignore) ? NAN : l - xr[t];
  }
}
// out[0] = sum(row_loss) / n_valid, out[1] = n_valid (as float): ONE CTA, each thread sums a fixed stride of rows, then a
// fixed butterfly / shared-memory tree, so the loss is bitwise reproducible.  n_valid = 0 gives 0 / 0 = NaN, as torch.
__global__ void __launch_bounds__(1024)
ce_reduce_kernel(const float* __restrict__ row_loss, const long long* __restrict__ target, int G, int ignore,
                 float* __restrict__ out) {
  __shared__ float rs[32];
  __shared__ int rn[32];
  float s = 0.f;
  int n = 0;
  for (int i = threadIdx.x; i < G; i += blockDim.x) {
    s += row_loss[i];
    n += target[i] != ignore;
  }
  s = warp_sum(s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0) { rs[threadIdx.x >> 5] = s; rn[threadIdx.x >> 5] = n; }
  __syncthreads();
  if (threadIdx.x < 32) {
    const bool have = threadIdx.x < (blockDim.x >> 5);
    s = warp_sum(have ? rs[threadIdx.x] : 0.f);
    n = have ? rn[threadIdx.x] : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if (threadIdx.x == 0) {
      out[0] = s / (float)n;
      out[1] = (float)n;
    }
  }
}
// dx[r, c] = g * (softmax(x_r)_c - [c == target_r]) / n_valid; 0 on ignored rows, NaN on rows with a bad target
__global__ void ce_bwd_kernel(const float* __restrict__ x, long long ld, const long long* __restrict__ target,
                              const float* __restrict__ lse, const float* __restrict__ out, int G, int C, int ignore,
                              const float* __restrict__ gscale, float* __restrict__ dx) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)G * C) return;
  const int r = idx / C, c = idx % C;
  const long long t = target[r];
  float v;
  if (t == ignore) v = 0.f;
  else if (ce_bad_target(t, C, ignore)) v = NAN;
  else {
    const float p = expf(x[(long long)r * ld + c] - lse[r]);
    v = (gscale ? *gscale : 1.f) * (p - (c == t ? 1.f : 0.f)) / out[1];
  }
  dx[idx] = v;
}

}  // namespace
}  // namespace egovlp

using namespace egovlp;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int egovlp_rownorm_fwd(const float* a, float* an, float* norm, int rows, int C, float eps, void* stream) {
  EGOVLP_CHECK_ARG(a && an && rows >= 0 && C > 0, "rownorm_fwd: bad args");
  if (rows == 0) return EGOVLP_OK;
  rownorm_fwd_kernel<<<(rows + 7) / 8, 256, 0, ST(stream)>>>(a, an, norm, rows, C, eps);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_rownorm_bwd(const float* dan, const float* an, const float* norm, float* da, int rows, int C,
                                  float eps, void* stream) {
  EGOVLP_CHECK_ARG(dan && an && norm && da && rows >= 0 && C > 0, "rownorm_bwd: bad args");
  if (rows == 0) return EGOVLP_OK;
  rownorm_bwd_kernel<<<(rows + 7) / 8, 256, 0, ST(stream)>>>(dan, an, norm, da, rows, C, eps);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_sgemm_f32(const float* A, long long sam, long long sak, const float* B, long long sbn,
                                long long sbk, float* Cm, long long ldc, int M, int N, int K, float alpha, float beta,
                                void* stream) {
  EGOVLP_CHECK_ARG(A && B && Cm && M > 0 && N > 0 && K > 0, "sgemm: bad args");
  dim3 grid((N + 31) / 32, (M + 31) / 32);
  sgemm_strided_kernel<<<grid, 256, 0, ST(stream)>>>(A, sam, sak, B, sbn, sbk, Cm, ldc, M, N, K, alpha, beta);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_pack_multihot(const float* v, uint32_t* bits, int G, int C, void* stream) {
  EGOVLP_CHECK_ARG(v && bits && G > 0 && C > 0, "pack_multihot: bad args");
  const int W = (C + 31) / 32;
  pack_multihot_kernel<<<(G * W + 255) / 256, 256, 0, ST(stream)>>>(v, bits, G, C, W);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_mask_from_bits(const uint32_t* vbits, int n_verb, const uint32_t* nbits, int n_noun,
                                     uint8_t* mask, int G, int mode, void* stream) {
  EGOVLP_CHECK_ARG(mask && G > 0 && mode >= 0 && mode <= 3, "mask_from_bits: bad args");
  EGOVLP_CHECK_ARG(mode == 0 || ((mode == 2 || vbits) && (mode == 3 || nbits)), "mask_from_bits: missing tags");
  dim3 grid((G + 127) / 128, G);
  mask_from_bits_kernel<<<grid, 128, 0, ST(stream)>>>(vbits, (n_verb + 31) / 32, nbits, (n_noun + 31) / 32, mask, G, mode);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_mask_from_sims(const float* sim_v, const float* sim_n, uint8_t* mask, int G, int mode,
                                     void* stream) {
  EGOVLP_CHECK_ARG(mask && G > 0 && mode >= 0 && mode <= 3, "mask_from_sims: bad args");
  const long long n = (long long)G * G;
  mask_from_sims_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(sim_v, sim_n, mask, G, mode);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_nce_fwd(const float* x, const uint8_t* mask, int G, float inv_temp, float* stats, float* loss,
                              void* stream) {
  EGOVLP_CHECK_ARG(x && mask && stats && loss && G > 0, "nce_fwd: bad args");
  dim3 grid((G + 7) / 8, 2);
  nce_stats_kernel<<<grid, 256, 0, ST(stream)>>>(x, mask, G, inv_temp, stats);
  EGOVLP_CHECK_LAUNCH();
  nce_loss_kernel<<<1, 256, 0, ST(stream)>>>(stats, G, loss);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_nce_bwd(const float* x, const uint8_t* mask, const float* stats, int G, float inv_temp,
                              const float* gscale, float* dx, void* stream) {
  EGOVLP_CHECK_ARG(x && mask && stats && dx && G > 0, "nce_bwd: bad args");
  const long long n = (long long)G * G;
  nce_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(x, mask, stats, G, inv_temp, gscale, dx);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
static int maxmargin_grid(int G) {
  const long long n = (long long)G * G;
  return (int)((n + 255) / 256 > 1024 ? 1024 : (n + 255) / 256);
}
static int maxmargin_fwd_impl(const float* x, const float* row_weight, int G, float margin, int fix_norm, float* loss,
                              float* part, void* stream) {
  EGOVLP_CHECK_ARG(x && loss && G > 1, "maxmargin_fwd: bad args");
  EGOVLP_CHECK_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), ST(stream)));
  const int grid = maxmargin_grid(G);
  maxmargin_fwd_kernel<<<grid, 256, 0, ST(stream)>>>(x, row_weight, G, margin, fix_norm, loss, part);
  EGOVLP_CHECK_LAUNCH();
  return part ? ordered_sum(part, grid, 1, loss, ST(stream)) : EGOVLP_OK;
}
extern "C" int egovlp_maxmargin_fwd(const float* x, const float* row_weight, int G, float margin, int fix_norm,
                                    float* loss, void* stream) {
  return maxmargin_fwd_impl(x, row_weight, G, margin, fix_norm, loss, nullptr, stream);
}
extern "C" long long egovlp_maxmargin_det_workspace_floats(int G) { return G > 1 ? maxmargin_grid(G) : -1; }
extern "C" int egovlp_maxmargin_fwd_det(const float* x, const float* row_weight, int G, float margin, int fix_norm,
                                        float* loss, float* ws, void* stream) {
  EGOVLP_CHECK_ARG(ws, "maxmargin_fwd_det: null workspace");
  return maxmargin_fwd_impl(x, row_weight, G, margin, fix_norm, loss, ws, stream);
}
extern "C" int egovlp_maxmargin_bwd(const float* x, const float* row_weight, int G, float margin, int fix_norm,
                                    const float* gscale, float* dx, void* stream) {
  EGOVLP_CHECK_ARG(x && dx && G > 1, "maxmargin_bwd: bad args");
  const long long n = (long long)G * G;
  EGOVLP_CHECK_CUDA(cudaMemsetAsync(dx, 0, n * sizeof(float), ST(stream)));
  maxmargin_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(x, row_weight, G, margin, fix_norm, gscale, dx);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_maxmargin_bwd_det(const float* x, const float* row_weight, int G, float margin, int fix_norm,
                                        const float* gscale, float* dx, void* stream) {
  EGOVLP_CHECK_ARG(x && dx && G > 1, "maxmargin_bwd_det: bad args");
  const long long n = (long long)G * G;
  maxmargin_bwd_gather_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(x, row_weight, G, margin, fix_norm,
                                                                                 gscale, dx);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_dual_softmax(const float* sim, float* out, int rows, int cols, float temp, void* stream) {
  EGOVLP_CHECK_ARG(sim && out && rows > 0 && cols > 0 && temp > 0.f, "dual_softmax: bad args");
  dsm_rows_kernel<<<(rows + 7) / 8, 256, 0, ST(stream)>>>(sim, out, rows, cols, 1.f / temp);
  EGOVLP_CHECK_LAUNCH();
  dsm_cols_kernel<<<(cols + 127) / 128, 128, 0, ST(stream)>>>(out, rows, cols);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_egomcq_score(const float* text, const float* video, float* scores, long long* pred, int Q,
                                   int K, int C, float eps, void* stream) {
  EGOVLP_CHECK_ARG(text && video && scores && pred && Q >= 0 && K > 0 && C > 0, "egomcq_score: bad args");
  if (Q == 0) return EGOVLP_OK;
  egomcq_kernel<<<(Q + 7) / 8, 256, 0, ST(stream)>>>(text, video, scores, pred, Q, K, C, eps);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_cross_entropy_fwd(const float* logits, long long ld, const long long* target, int G, int C,
                                        int ignore_index, float* lse, float* row_loss, float* out, void* stream) {
  EGOVLP_CHECK_ARG(logits && target && lse && row_loss && out && G >= 0 && C > 0 && ld >= C, "cross_entropy_fwd: bad args");
  if (G > 0) {
    ce_rows_kernel<<<(G + 7) / 8, 256, 0, ST(stream)>>>(logits, ld, target, G, C, ignore_index, lse, row_loss);
    EGOVLP_CHECK_LAUNCH();
  }
  ce_reduce_kernel<<<1, 1024, 0, ST(stream)>>>(row_loss, target, G, ignore_index, out);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
extern "C" int egovlp_cross_entropy_bwd(const float* logits, long long ld, const long long* target, const float* lse,
                                        const float* out, int G, int C, int ignore_index, const float* gscale, float* dx,
                                        void* stream) {
  EGOVLP_CHECK_ARG(logits && target && lse && out && dx && G >= 0 && C > 0 && ld >= C, "cross_entropy_bwd: bad args");
  const long long n = (long long)G * C;
  if (n == 0) return EGOVLP_OK;
  ce_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(logits, ld, target, lse, out, G, C, ignore_index,
                                                                    gscale, dx);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
