// EgoNCE from the gathered embeddings in ONE kernel per direction (north_star iii; reference: sim_matrix,
// model/model.py:189-197, + EgoNCE.forward, model/loss.py:34-53, as called at trainer/trainer_egoclip.py:130-135).
//
// Forward (egonce_fused_fwd_kernel): reads the packed all-gather buffer in place (row-strided text | video | verb | noun
// slices, no cat / contiguous copies), normalises the rows in its prologue (norm clamped at eps), forms the [G, G] cosine
// similarities tile by tile in shared memory -- they never exist in HBM --, derives the positives from bit-packed tag
// co-occurrence (diagonal OR (shared verb AND shared noun)), reduces the masked / unmasked log-sum-exp of every row, hands
// per-column partials to the last CTA to finish (atomic ticket), which merges them and writes the loss.
// Backward (egonce_fused_bwd_kernel): recomputes the similarities of THIS RANK's rows / columns only and emits d text and
// d video for the local slice (the reference's gather keeps only the local gradient, trainer_egoclip.py:23-27).
//
// fp32 on the CUDA cores by choice: the logits are x / 0.05, so bf16 operands (3e-3 on a cosine) would move the loss by
// 1e-2 and even kind::tf32 by ~1e-3, against the 2e-5 the fp32 reference is matched to here; the whole problem is
// 2 G^2 C = 0.13 GFLOP at G = 512 (a few microseconds), i.e. latency-, not throughput-bound.
#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

constexpr int TR = 32;            // rows of the similarity matrix per CTA / columns per inner tile
constexpr int MAXG = 512, MAXC = 256;

struct FusedGeom {
  int G, C, nverb, nnoun, Wv, Wn, mode;
  long long ld_t, ld_v, ld_verb, ld_noun;
  float inv_temp, eps;
};

__device__ __forceinline__ bool positive(const uint32_t* bi, const uint32_t* bj, int i, int j, int Wv, int Wn, int mode) {
  if (i == j) return true;
  bool sv = false, sn = false;
  if (mode == 1 || mode == 3)
    for (int w = 0; w < Wv; ++w) sv |= (bi[w] & bj[w]) != 0;
  if (mode == 1 || mode == 2)
    for (int w = 0; w < Wn; ++w) sn |= (bi[Wv + w] & bj[Wv + w]) != 0;
  return mode == 1 ? (sv && sn) : mode == 2 ? sn : mode == 3 ? sv : false;
}

// rows [r0, r0 + nr) of `src` (row stride ld) -> dst[nr][pitch] = row / max(||row||, eps); norms to norm_out (optional)
__device__ __forceinline__ void load_normalised(const float* __restrict__ src, long long ld, int r0, int nr, int G, int C,
                                                float eps, float* dst, int pitch, float* norm_out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int r = warp; r < nr; r += nw) {
    const int gr = r0 + r;
    float v[MAXC / 32];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < MAXC / 32; ++k) {
      const int c = lane + 32 * k;
      v[k] = (gr < G && c < C) ? src[(long long)gr * ld + c] : 0.f;
      s += v[k] * v[k];
    }
    const float n = sqrtf(warp_sum(s));
    const float inv = 1.f / fmaxf(n, eps);
#pragma unroll
    for (int k = 0; k < MAXC / 32; ++k) {
      const int c = lane + 32 * k;
      if (c < C) dst[r * pitch + c] = v[k] * inv;
    }
    if (lane == 0 && norm_out && gr < G) norm_out[gr] = n;
  }
}

__global__ void __launch_bounds__(256)
egonce_fused_fwd_kernel(const float* __restrict__ text, const float* __restrict__ video, const float* __restrict__ verb,
                        const float* __restrict__ noun, FusedGeom g, float* __restrict__ na, float* __restrict__ nb,
                        uint32_t* __restrict__ bits_out, float* __restrict__ stats, float* __restrict__ colpart,
                        unsigned* __restrict__ ticket, float* __restrict__ loss) {
  extern __shared__ __align__(16) uint8_t fsm[];
  const int G = g.G, C = g.C, W = g.Wv + g.Wn, CP = C + 1;
  const int GP = (G + TR - 1) / TR * TR;
  uint32_t* bits = reinterpret_cast<uint32_t*>(fsm);                    // [G][W]
  float* tn = reinterpret_cast<float*>(bits + (size_t)G * W);           // [TR][C]
  float* vn = tn + TR * C;                                              // [TR][C + 1]
  float* xs = vn + TR * CP;                                             // [TR][GP]
  uint32_t* mrow = reinterpret_cast<uint32_t*>(xs + (size_t)TR * GP);   // [TR][GP / 32] positives of this row tile
  __shared__ int is_last;
  __shared__ float red[8];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r0 = blockIdx.x * TR, nr = min(TR, G - r0);

  // ---- tag bits of every row (each CTA needs all of them for its row tile's positives)
  for (int idx = tid; idx < G * W; idx += blockDim.x) {
    const int r = idx / W, w = idx % W;
    const bool is_verb = w < g.Wv;
    const float* row = is_verb ? verb + (long long)r * g.ld_verb : noun + (long long)r * g.ld_noun;
    const int c0 = (is_verb ? w : w - g.Wv) * 32, n = is_verb ? g.nverb : g.nnoun;
    uint32_t m = 0;
    for (int j = 0; j < 32; ++j)
      if (c0 + j < n && row[c0 + j] != 0.f) m |= 1u << j;
    bits[idx] = m;
    if (blockIdx.x == 0) bits_out[idx] = m;
  }
  load_normalised(text, g.ld_t, r0, nr, G, C, g.eps, tn, C, na);
  __syncthreads();

  // ---- similarities of this row tile against every column tile (fp32 FMA, x stays in shared memory)
  const int tx = tid & 31, ty = tid >> 5;
  for (int c0 = 0; c0 < G; c0 += TR) {
    load_normalised(video, g.ld_v, c0, min(TR, G - c0), G, C, g.eps, vn, CP, blockIdx.x == 0 ? nb : nullptr);
    __syncthreads();
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (c0 + tx < G) {
      for (int k = 0; k < C; ++k) {
        const float b = vn[tx * CP + k];
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] = fmaf(tn[(ty + 8 * i) * C + k], b, acc[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) xs[(ty + 8 * i) * GP + c0 + tx] = acc[i];
    __syncthreads();
  }

  // ---- positives of the tile as bit rows, then the row statistics: one warp per row
  for (int r = warp; r < nr; r += 8) {
    const int i = r0 + r;
    for (int jb = 0; jb < GP / 32; ++jb) {
      const int j = jb * 32 + lane;
      const bool pos = j < G && positive(bits + (size_t)i * W, bits + (size_t)j * W, i, j, g.Wv, g.Wn, g.mode);
      const uint32_t word = __ballot_sync(0xffffffffu, pos);
      if (lane == 0) mrow[r * (GP / 32) + jb] = word;
    }
    __syncwarp();
    float mx = -INFINITY;
    for (int j = lane; j < G; j += 32) mx = fmaxf(mx, xs[r * GP + j] * g.inv_temp);
    mx = warp_max(mx);
    float sa = 0.f, sp = 0.f;
    for (int j = lane; j < G; j += 32) {
      const float e = expf(xs[r * GP + j] * g.inv_temp - mx);
      sa += e;
      if ((mrow[r * (GP / 32) + (j >> 5)] >> (j & 31)) & 1u) sp += e;
    }
    sa = warp_sum(sa); sp = warp_sum(sp);
    if (lane == 0) {
      stats[i] = mx + logf(sa);
      stats[G + i] = mx + logf(sp);
    }
  }
  __syncthreads();
  // ---- column partials over this tile's rows.  Column j sums softmax_col_j(i) * mask[j, i] (the reference multiplies by
  // the UN-transposed mask, model/loss.py:50); the tag condition is symmetric, so mask[j, i] == mask[i, j] = mrow bit.
  for (int j = tid; j < G; j += blockDim.x) {
    float mx = -INFINITY;
    for (int r = 0; r < nr; ++r) mx = fmaxf(mx, xs[r * GP + j] * g.inv_temp);
    float sa = 0.f, sp = 0.f;
    for (int r = 0; r < nr; ++r) {
      const float e = expf(xs[r * GP + j] * g.inv_temp - mx);
      sa += e;
      if ((mrow[r * (GP / 32) + (j >> 5)] >> (j & 31)) & 1u) sp += e;
    }
    float* cp = colpart + ((size_t)blockIdx.x * G + j) * 3;
    cp[0] = mx; cp[1] = sa; cp[2] = sp;
  }
  // ---- the last CTA merges the column partials and reduces the loss
  __threadfence();
  __syncthreads();
  if (tid == 0) is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  float part = 0.f;
  for (int j = tid; j < G; j += blockDim.x) {
    float mx = -INFINITY;
    for (unsigned t = 0; t < gridDim.x; ++t) mx = fmaxf(mx, __ldcg(colpart + ((size_t)t * G + j) * 3));
    float sa = 0.f, sp = 0.f;
    for (unsigned t = 0; t < gridDim.x; ++t) {
      const float* cp = colpart + ((size_t)t * G + j) * 3;
      const float sc = expf(__ldcg(cp) - mx);
      sa += __ldcg(cp + 1) * sc;
      sp += __ldcg(cp + 2) * sc;
    }
    const float la = mx + logf(sa), lp = mx + logf(sp);
    stats[2 * G + j] = la;
    stats[3 * G + j] = lp;
    part += (lp - la) + (__ldcg(stats + G + j) - __ldcg(stats + j));
  }
  part = warp_sum(part);
  if (lane == 0) red[warp] = part;
  __syncthreads();
  if (warp == 0) {
    float s = lane < 8 ? red[lane] : 0.f;
    s = warp_sum(s);
    if (lane == 0) {
      *loss = -s / G;
      *ticket = 0;                                        // ready for the next launch
    }
  }
}

// d text / d video of the local rows [row0, row0 + nloc).  blockIdx.y = 0: text side (a = text row i, b = video rows j);
// 1: video side (a = video row j, b = text rows i).  8 "a" rows per CTA; the b side streams through smem 32 rows at a time.
__global__ void __launch_bounds__(256)
egonce_fused_bwd_kernel(const float* __restrict__ text, const float* __restrict__ video, FusedGeom g,
                        const float* __restrict__ na, const float* __restrict__ nb, const uint32_t* __restrict__ bits,
                        const float* __restrict__ stats, const float* __restrict__ gscale, int row0, int nloc,
                        float* __restrict__ d_text, float* __restrict__ d_video) {
  __shared__ float an[8][MAXC];
  __shared__ float bn[TR][MAXC + 1];
  __shared__ float dxs[8][TR];
  const int G = g.G, C = g.C, W = g.Wv + g.Wn;
  const bool vside = blockIdx.y == 1;
  const float* A = vside ? video : text;
  const float* Bm = vside ? text : video;
  const long long lda = vside ? g.ld_v : g.ld_t, ldb = vside ? g.ld_t : g.ld_v;
  const float* norm_a = vside ? nb : na;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int a0 = row0 + blockIdx.x * 8, na_rows = min(8, row0 + nloc - a0);
  if (na_rows <= 0) return;
  load_normalised(A, lda, a0, na_rows, G, C, g.eps, &an[0][0], MAXC, nullptr);
  const float coef = -(gscale ? *gscale : 1.f) * g.inv_temp / G;
  float acc[MAXC / 32];
#pragma unroll
  for (int k = 0; k < MAXC / 32; ++k) acc[k] = 0.f;
  __syncthreads();
  const int a = a0 + warp;                               // this warp's "a" row (global index), valid if warp < na_rows
  for (int b0 = 0; b0 < G; b0 += TR) {
    const int nb_rows = min(TR, G - b0);
    load_normalised(Bm, ldb, b0, nb_rows, G, C, g.eps, &bn[0][0], MAXC + 1, nullptr);
    __syncthreads();
    // phase 1: x[a, b] and dX for (warp = a row, lane = b row of the tile)
    float dxv = 0.f;
    const int b = b0 + lane;
    if (warp < na_rows && b < G) {
      float x = 0.f;
      for (int k = 0; k < C; ++k) x = fmaf(an[warp][k], bn[lane][k], x);
      const int i = vside ? b : a, j = vside ? a : b;
      const float z = x * g.inv_temp;
      const float m = positive(bits + (size_t)i * W, bits + (size_t)j * W, i, j, g.Wv, g.Wn, g.mode) ? 1.f : 0.f;
      // mask[j, i] == mask[i, j] (symmetric tag condition), see the forward
      dxv = coef * (m * expf(z - stats[G + i]) - expf(z - stats[i]) + m * expf(z - stats[3 * G + j]) - expf(z - stats[2 * G + j]));
    }
    dxs[warp][lane] = dxv;
    __syncwarp();
    // phase 2: d an[a, :] += dX[a, b] * bn[b, :], over the rows load_normalised wrote: the rest of bn is stale (left
    // uninitialised at G < 32), and fmaf(0, NaN, acc) would be NaN.  The skipped terms were fmaf(0, finite, acc) == acc.
    if (warp < na_rows) {
      for (int bl = 0; bl < nb_rows; ++bl) {
        const float d = dxs[warp][bl];
#pragma unroll
        for (int k = 0; k < MAXC / 32; ++k)
          if (lane + 32 * k < C) acc[k] = fmaf(d, bn[bl][lane + 32 * k], acc[k]);
      }
    }
    __syncthreads();
  }
  if (warp >= na_rows) return;
  // row-normalisation backward: da = (dan - an <an, dan>) / ||a||  if ||a|| > eps, else dan / eps
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < MAXC / 32; ++k)
    if (lane + 32 * k < C) s += an[warp][lane + 32 * k] * acc[k];
  s = warp_sum(s);
  const float n = norm_a[a];
  float* dst = (vside ? d_video : d_text) + (long long)(a - row0) * C;
#pragma unroll
  for (int k = 0; k < MAXC / 32; ++k) {
    const int c = lane + 32 * k;
    if (c < C) dst[c] = n > g.eps ? (acc[k] - an[warp][c] * s) / n : acc[k] / g.eps;
  }
}

// out[r, :] = [a[r, :ca] | b[r, :cb] | c[r, :cc] | d[r, :cd]]: the send buffer of the ONE packed all-gather
__global__ void pack_rows4_kernel(const float* __restrict__ a, int ca, const float* __restrict__ b, int cb,
                                  const float* __restrict__ c, int cc, const float* __restrict__ d, int cd,
                                  float* __restrict__ out, int rows) {
  const int W = ca + cb + cc + cd;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < (long long)rows * W;
       idx += (long long)gridDim.x * blockDim.x) {
    const int r = idx / W, k = idx % W;
    out[idx] = k < ca ? a[(long long)r * ca + k]
               : k < ca + cb ? b[(long long)r * cb + k - ca]
               : k < ca + cb + cc ? c[(long long)r * cc + k - ca - cb] : d[(long long)r * cd + k - ca - cb - cc];
  }
}

FusedGeom make_fused_geom(int G, int C, long long ld_t, long long ld_v, long long ld_verb, int n_verb, long long ld_noun,
                          int n_noun, float inv_temp, int mode, float eps) {
  FusedGeom g;
  g.G = G; g.C = C; g.nverb = n_verb; g.nnoun = n_noun; g.Wv = (n_verb + 31) / 32; g.Wn = (n_noun + 31) / 32; g.mode = mode;
  g.ld_t = ld_t; g.ld_v = ld_v; g.ld_verb = ld_verb; g.ld_noun = ld_noun; g.inv_temp = inv_temp; g.eps = eps;
  return g;
}

// dynamic shared memory of the forward: tag bits [G][W], tn [TR][C], vn [TR][C + 1], xs [TR][GP], mrow [TR][GP / 32]
size_t fused_fwd_smem(int G, int C, int W) {
  const int GP = (G + TR - 1) / TR * TR;
  return (size_t)G * W * 4 + (size_t)TR * C * 4 + (size_t)TR * (C + 1) * 4 + (size_t)TR * GP * 4 + (size_t)TR * (GP / 32) * 4;
}

}  // namespace
}  // namespace egovlp

using namespace egovlp;

extern "C" int egovlp_egonce_fused_max_g(void) { return MAXG; }

// 1 if the forward can take this problem on the current device: the tag bits of every row live in shared memory, so a
// wide tag vocabulary at large G can exceed the opt-in limit (about 1,500 tag columns at G = 512, C = 256 on an H100).
extern "C" int egovlp_egonce_fused_supported(int G, int C, int n_verb, int n_noun, int mode) {
  if (G <= 0 || G > MAXG || C <= 0 || C > MAXC || mode < 0 || mode > 3) return 0;
  if (mode == 0 || mode == 2) n_verb = 0;
  if (mode == 0 || mode == 3) n_noun = 0;
  int dev = 0, optin = 0;
  cudaFuncAttributes fa;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
      cudaFuncGetAttributes(&fa, egonce_fused_fwd_kernel) != cudaSuccess)
    return 0;
  return fused_fwd_smem(G, C, (n_verb + 31) / 32 + (n_noun + 31) / 32) + fa.sharedSizeBytes <= (size_t)optin;
}

extern "C" long long egovlp_egonce_fused_workspace_floats(int G) {
  const long long tiles = (G + TR - 1) / TR;
  return tiles * G * 3 + 4;              // column partials + the ticket word (must be zero before the first launch)
}

extern "C" int egovlp_egonce_fused_fwd(const float* text, long long ld_t, const float* video, long long ld_v,
                                       const float* verb, long long ld_verb, int n_verb, const float* noun,
                                       long long ld_noun, int n_noun, int G, int C, float inv_temp, int mode, float eps,
                                       float* norm_text, float* norm_video, uint32_t* tag_bits, float* stats,
                                       float* workspace, float* loss, void* stream) {
  EGOVLP_CHECK_ARG(text && video && norm_text && norm_video && tag_bits && stats && workspace && loss, "egonce_fused_fwd: null pointer");
  EGOVLP_CHECK_ARG(G > 0 && G <= MAXG && C > 0 && C <= MAXC, "egonce_fused_fwd: G=%d (<= %d) C=%d (<= %d)", G, MAXG, C, MAXC);
  EGOVLP_CHECK_ARG(mode >= 0 && mode <= 3 && ((mode != 1 && mode != 3) || verb) && ((mode != 1 && mode != 2) || noun),
                   "egonce_fused_fwd: mode %d needs its tag matrices", mode);
  if (mode == 0 || mode == 2) n_verb = 0;
  if (mode == 0 || mode == 3) n_noun = 0;
  const FusedGeom g = make_fused_geom(G, C, ld_t, ld_v, ld_verb, n_verb, ld_noun, n_noun, inv_temp, mode, eps);
  const int GP = (G + TR - 1) / TR * TR;
  const size_t smem = fused_fwd_smem(G, C, g.Wv + g.Wn);
  static size_t attr = 0;
  if (smem > attr) {
    EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(egonce_fused_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  const int tiles = GP / TR;
  unsigned* ticket = reinterpret_cast<unsigned*>(workspace + (size_t)tiles * G * 3);
  egonce_fused_fwd_kernel<<<tiles, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      text, video, verb, noun, g, norm_text, norm_video, tag_bits, stats, workspace, ticket, loss);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

extern "C" int egovlp_egonce_fused_bwd(const float* text, long long ld_t, const float* video, long long ld_v,
                                       const float* norm_text, const float* norm_video, const uint32_t* tag_bits,
                                       int n_verb, int n_noun, const float* stats, int G, int C, float inv_temp, int mode,
                                       float eps, const float* gscale, int row0, int n_local, float* d_text,
                                       float* d_video, void* stream) {
  EGOVLP_CHECK_ARG(text && video && norm_text && norm_video && tag_bits && stats && d_text && d_video, "egonce_fused_bwd: null pointer");
  EGOVLP_CHECK_ARG(G > 0 && G <= MAXG && C > 0 && C <= MAXC && row0 >= 0 && n_local > 0 && row0 + n_local <= G,
                   "egonce_fused_bwd: bad shape G=%d C=%d rows [%d, %d)", G, C, row0, row0 + n_local);
  if (mode == 0 || mode == 2) n_verb = 0;
  if (mode == 0 || mode == 3) n_noun = 0;
  const FusedGeom g = make_fused_geom(G, C, ld_t, ld_v, 0, n_verb, 0, n_noun, inv_temp, mode, eps);
  dim3 grid((n_local + 7) / 8, 2);
  egonce_fused_bwd_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      text, video, g, norm_text, norm_video, tag_bits, stats, gscale, row0, n_local, d_text, d_video);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

extern "C" int egovlp_pack_rows4(const float* a, int ca, const float* b, int cb, const float* c, int cc, const float* d,
                                 int cd, float* out, int rows, void* stream) {
  EGOVLP_CHECK_ARG(a && b && out && rows > 0 && ca > 0 && cb > 0 && cc >= 0 && cd >= 0 && (cc == 0 || c) && (cd == 0 || d),
                   "pack_rows4: bad args");
  const long long n = (long long)rows * (ca + cb + cc + cd);
  pack_rows4_kernel<<<(int)((n + 255) / 256 < 1184 ? (n + 255) / 256 : 1184), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      a, ca, b, cb, c, cc, d, cd, out, rows);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
