// Retrieval-evaluation kernels (SURVEY.md 8f row 3): per-query ranking metrics of the EPIC-Kitchens MIR evaluation,
// reference utils/nDCG.py:3-45,96-139 (calculate_DCG / calculate_k_counts / calculate_nDCG) and utils/mAP.py:4-44
// (calculate_mAP), which the reference runs as numpy argsort + fancy indexing on the host
// (model/metric.py:257-299, run/test_epic.py:137-157).
//
// One CTA ranks one query row entirely in shared memory: the row of similarities is loaded once (coalesced), sorted
// descending together with its column indices by a bitonic network, and the relevancy row is gathered through the
// sorted indices; DCG and average precision are then block reductions / one block scan in fp64.  HBM traffic is the
// algorithmic minimum (one read of the similarity row and of the relevancy row), there is no [rows, cols] index
// matrix in global memory, and nothing is copied to the host.
#include <math_constants.h>

#include "common.cuh"

namespace egovlp {
namespace {

constexpr int RANK_THREADS = 512;
constexpr int RANK_MAX_COLS = 16384;

constexpr unsigned short RANK_PAD = 0xFFFF;      // column index of the sort's padding slots (cols <= 16384)

// Strict total order of the ranking: larger similarity first; ties by column index (tie_hi: larger index first, i.e.
// a stable ascending argsort reversed as in nDCG.py:32; otherwise smaller index first, a stable argsort of -sim as in
// mAP.py:25).  NaN goes where numpy's sort puts it: after every real score (-inf included) for the argsort of -sim,
// before every real score for the reversed ascending argsort, among NaNs by the same index rule.  The padding slots
// rank after everything, so the first `cols` ranks always hold the real columns (NaN compares false both ways, and
// without its own place it would break the network's order and let padding into them).
__device__ __forceinline__ int rank_class(float k, unsigned short i, bool tie_hi) {
  return i == RANK_PAD ? 3 : isnan(k) ? (tie_hi ? 0 : 2) : 1;
}

__device__ __forceinline__ bool ranks_before(float ka, unsigned short ia, float kb, unsigned short ib, bool tie_hi) {
  const int ca = rank_class(ka, ia, tie_hi), cb = rank_class(kb, ib, tie_hi);
  if (ca != cb) return ca < cb;
  return (ca == 1 && ka > kb) || ((ca != 1 || ka == kb) && (tie_hi ? ia > ib : ia < ib));
}

__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < RANK_THREADS / 32; ++w) s += red[w];
  return s;
}

template <typename RelT>
__global__ void __launch_bounds__(RANK_THREADS)
rank_metrics_kernel(const float* __restrict__ sim, long long ld_sim, const RelT* __restrict__ rel, long long ld_rel,
                    const int* __restrict__ k_counts, int cols, int np2, int tie_hi, double* __restrict__ dcg,
                    double* __restrict__ ap) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* key = reinterpret_cast<float*>(smem);
  unsigned short* idx = reinterpret_cast<unsigned short*>(key + np2);
  double* red = reinterpret_cast<double*>(smem + (size_t)np2 * 6);      // np2 * 6 is a multiple of 8 (np2 >= 512)
  double* scan = red + RANK_THREADS / 32;
  const int row = blockIdx.x, tid = threadIdx.x;
  const float* srow = sim + (long long)row * ld_sim;
  const RelT* rrow = rel + (long long)row * ld_rel;

  int n_pos = 0;                    // relevant items of this query (k of nDCG.py:47-75 when no k_counts is given)
  for (int c = tid; c < np2; c += RANK_THREADS) {
    key[c] = c < cols ? srow[c] : -INFINITY;
    idx[c] = c < cols ? (unsigned short)c : RANK_PAD;
    if (c < cols && (double)rrow[c] > 0.0) ++n_pos;
  }
  const int k_row = (int)(block_sum((double)n_pos, red) + 0.5);
  __syncthreads();

  for (int k = 2; k <= np2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < (np2 >> 1); t += RANK_THREADS) {
        const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1)), hi = lo + j;
        const float ka = key[lo], kb = key[hi];
        const unsigned short ia = idx[lo], ib = idx[hi];
        const bool up = (lo & k) == 0;
        const bool swap = up ? ranks_before(kb, ib, ka, ia, tie_hi) : ranks_before(ka, ia, kb, ib, tie_hi);
        if (swap) { key[lo] = kb; key[hi] = ka; idx[lo] = ib; idx[hi] = ia; }
      }
      __syncthreads();
    }
  }

  // rank i (0-based) holds column idx[i].  Each thread owns `per` consecutive ranks.
  const int per = np2 / RANK_THREADS, i0 = tid * per;
  double d_part = 0.0, c_part = 0.0;
  int n_one = 0;
  for (int i = i0; i < i0 + per && i < cols; ++i) {
    const double r = (double)rrow[idx[i]];
    const double kc = k_counts ? (double)k_counts[(long long)row * cols + i] : (i < k_row ? 1.0 : 0.0);
    d_part += r * kc / log2((double)i + 2.0);
    c_part += r;
  }
  const double d_tot = block_sum(d_part, red);
  // exclusive scan of the per-thread relevancy sums -> running cumulative relevancy (mAP.py:31)
  __syncthreads();
  scan[tid] = c_part;
  __syncthreads();
  for (int o = 1; o < RANK_THREADS; o <<= 1) {
    const double v = tid >= o ? scan[tid - o] : 0.0;
    __syncthreads();
    scan[tid] += v;
    __syncthreads();
  }
  double cum = scan[tid] - c_part, a_part = 0.0;
  for (int i = i0; i < i0 + per && i < cols; ++i) {
    const double r = (double)rrow[idx[i]];
    cum += r;
    if (r == 1.0) { a_part += cum / (double)(i + 1); ++n_one; }
  }
  const double a_tot = block_sum(a_part, red);
  const double ones = block_sum((double)n_one, red);
  if (tid == 0) {
    if (dcg) dcg[row] = d_tot;
    if (ap) ap[row] = a_tot / ones;            // 0 / 0 -> NaN, as numpy (a query without relevant items)
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Ground-truth ranks of the MSR-VTT-style retrieval metrics t2v_metrics / v2t_metrics (reference model/metric.py:20-216),
// which rank by DISTANCE SUBTRACTION (np.where(sorted_dists - gt_dist == 0)), not by argsort: a candidate's 0-based
// position among the sorted distances is fully determined by how many entries of its row are strictly closer and how
// many are equal.  So no sort is needed: one CTA streams its row and counts, per candidate, the entries with a strictly
// greater similarity (= smaller distance -sim; negation is exact) and the entries with an equal one.
//   t2v (mode 0): one candidate, column row / q; ties optimistic (first match, :71-73): rank = #greater.
//   v2t (mode 1): candidates [row * c, (row + 1) * c); ties averaged (ranks.mean() over the matching run, :187):
//                 rank = #greater + (#equal - 1) / 2 (exact in fp64); the row's rank is the minimum over candidates.
//                 col_mask[j] == 0 sets entry j to distance MISSING_VAL = 1e8, i.e. similarity -1e8 in the row's type
//                 (:163-167); a candidate whose distance is then MISSING_VAL is skipped (:177-179), and so is one
//                 whose distance is infinite (inf - inf is NaN: no match, ranks.mean() = NaN never wins :188).  No
//                 candidate left gives +inf (min_rank's initial value).
// Candidates are counted GT_GROUP at a time, each thread holding one packed counter per candidate (#greater in the low
// 16 bits, #equal in the high 16 bits: a thread visits at most GT_MAX_COLS / GT_THREADS < 2^16 entries of a row).  Rows
// of up to GT_GROUP candidates (MSR-VTT has 20; 32 spills registers) are read once; more re-read the row from L2.
// status bits: 1 = NaN in a row (after masking), 2 = non-finite t2v ground truth (the reference's `cols.size` assert).
constexpr int GT_THREADS = 256;
constexpr int GT_GROUP = 24;
constexpr int GT_MAX_CAND = 64;
constexpr int GT_MAX_COLS = 65535 * GT_THREADS;

template <typename T, int NC>
__global__ void __launch_bounds__(GT_THREADS)
gt_ranks_kernel(const T* __restrict__ sims, long long ld, int cols, int per, int v2t,
                const unsigned char* __restrict__ col_mask, double* __restrict__ ranks, int* __restrict__ status) {
  __shared__ T cand[GT_MAX_CAND];
  __shared__ int live[GT_MAX_CAND], n_gt[GT_MAX_CAND], n_eq[GT_MAX_CAND];
  const int row = blockIdx.x, tid = threadIdx.x;
  const T* srow = sims + (long long)row * ld;
  const T missing = (T)-1e8;
  const int nc = v2t ? per : 1;
  const int c0 = v2t ? row * per : row / per;
  if (tid < nc) {
    const int j = c0 + tid;
    const T v = (v2t && col_mask && !col_mask[j]) ? missing : srow[j];
    cand[tid] = v;
    live[tid] = v2t ? (v != missing && isfinite(v)) : 1;
    n_gt[tid] = n_eq[tid] = 0;
  }
  __syncthreads();

  int nan_seen = 0;
  for (int k0 = 0; k0 < nc; k0 += NC) {
    unsigned cnt[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) cnt[k] = 0u;
    for (int j = tid; j < cols; j += GT_THREADS) {
      T v = srow[j];
      if (v2t && col_mask && !col_mask[j]) v = missing;
      nan_seen |= isnan(v);
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        if (k0 + k < nc) {
          const T ck = cand[k0 + k];
          cnt[k] += (unsigned)(v > ck) + ((unsigned)(v == ck) << 16);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      if (k0 + k < nc) {
        int a = (int)(cnt[k] & 0xFFFFu), b = (int)(cnt[k] >> 16);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          a += __shfl_xor_sync(0xffffffffu, a, o);
          b += __shfl_xor_sync(0xffffffffu, b, o);
        }
        if ((tid & 31) == 0) { atomicAdd(&n_gt[k0 + k], a); atomicAdd(&n_eq[k0 + k], b); }   // integer: order-free
      }
    }
  }
  nan_seen = __syncthreads_or(nan_seen);
  if (tid == 0) {
    if (nan_seen) {
      atomicOr(status, 1);
      ranks[row] = CUDART_NAN;
      return;
    }
    if (!v2t) {
      if (!isfinite(cand[0])) atomicOr(status, 2);
      ranks[row] = (double)n_gt[0];
      return;
    }
    double best = CUDART_INF;
    for (int k = 0; k < nc; ++k)
      if (live[k]) best = fmin(best, (double)n_gt[k] + 0.5 * (double)(n_eq[k] - 1));
    ranks[row] = best;
  }
}

template <typename T>
int launch_gt_ranks(const void* sims, long long ld, int rows, int cols, int per, int v2t, const unsigned char* col_mask,
                    double* ranks, int* status, cudaStream_t st) {
  const T* s = static_cast<const T*>(sims);
  if (v2t)
    gt_ranks_kernel<T, GT_GROUP><<<rows, GT_THREADS, 0, st>>>(s, ld, cols, per, 1, col_mask, ranks, status);
  else
    gt_ranks_kernel<T, 1><<<rows, GT_THREADS, 0, st>>>(s, ld, cols, per, 0, nullptr, ranks, status);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

}  // namespace
}  // namespace egovlp

using namespace egovlp;

extern "C" int egovlp_gt_ranks_max_candidates(void) { return GT_MAX_CAND; }

extern "C" int egovlp_gt_ranks(const void* sims, int is_f64, long long ld, int rows, int cols, int mode,
                               const unsigned char* col_mask, double* ranks, int* status, void* stream) {
  EGOVLP_CHECK_ARG(sims && ranks && status && rows > 0 && cols > 0 && ld >= cols && (mode == 0 || mode == 1),
                   "gt_ranks: bad args");
  EGOVLP_CHECK_ARG(mode == 1 || !col_mask, "gt_ranks: t2v takes no column mask (drop masked queries from its ranks)");
  EGOVLP_CHECK_ARG(cols <= GT_MAX_COLS, "gt_ranks: more than %d entries per row are not supported", GT_MAX_COLS);
  int per;
  if (mode == 0) {
    EGOVLP_CHECK_ARG(rows % cols == 0, "gt_ranks: t2v needs queries (%d) to be a multiple of videos (%d)", rows, cols);
    per = rows / cols;
  } else {
    per = cols / rows;               // captions per video, floor division as the reference (:156)
    EGOVLP_CHECK_ARG(per <= GT_MAX_CAND, "gt_ranks: %d candidates per row, at most %d are supported", per,
                     GT_MAX_CAND);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  EGOVLP_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  const int rc = is_f64 ? launch_gt_ranks<double>(sims, ld, rows, cols, per, mode, col_mask, ranks, status, st)
                        : launch_gt_ranks<float>(sims, ld, rows, cols, per, mode, col_mask, ranks, status, st);
  if (rc != EGOVLP_OK) return rc;
  int host_status = 0;
  EGOVLP_CHECK_CUDA(cudaMemcpyAsync(&host_status, status, sizeof(int), cudaMemcpyDeviceToHost, st));
  EGOVLP_CHECK_CUDA(cudaStreamSynchronize(st));
  EGOVLP_CHECK_ARG(host_status == 0, "gt_ranks:%s%s", (host_status & 1) ? " NaN in the similarity matrix;" : "",
                   (host_status & 2) ? " non-finite ground-truth similarity (t2v);" : "");
  return EGOVLP_OK;
}

extern "C" int egovlp_rank_metrics(const float* sim, long long ld_sim, const void* rel, int rel_is_f64, long long ld_rel,
                                   const int* k_counts, int rows, int cols, int tie_mode, double* dcg, double* ap,
                                   void* stream) {
  EGOVLP_CHECK_ARG(sim && rel && rows >= 0 && cols > 0 && (dcg || ap), "rank_metrics: bad args");
  EGOVLP_CHECK_ARG(cols <= RANK_MAX_COLS, "rank_metrics: more than 16384 gallery items per query are not supported");
  EGOVLP_CHECK_ARG(ld_sim >= cols && ld_rel >= cols, "rank_metrics: leading dimensions smaller than cols");
  if (rows == 0) return EGOVLP_OK;
  int np2 = RANK_THREADS;
  while (np2 < cols) np2 <<= 1;
  const size_t smem = (size_t)np2 * 6 + (RANK_THREADS / 32 + RANK_THREADS) * sizeof(double);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (rel_is_f64) {
    EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(rank_metrics_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rank_metrics_kernel<double><<<rows, RANK_THREADS, smem, st>>>(sim, ld_sim, static_cast<const double*>(rel), ld_rel,
                                                                   k_counts, cols, np2, tie_mode != 0, dcg, ap);
  } else {
    EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(rank_metrics_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rank_metrics_kernel<float><<<rows, RANK_THREADS, smem, st>>>(sim, ld_sim, static_cast<const float*>(rel), ld_rel,
                                                                  k_counts, cols, np2, tie_mode != 0, dcg, ap);
  }
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
