// Shared device helpers for the sm_90a kernels: mbarrier / TMA / wgmma PTX wrappers,
// warp reductions, bf16 packing.  Hand-written inline PTX (no CUTLASS templates).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define EGOVLP_OK 0
#define EGOVLP_ERR_ARG (-1)
#define EGOVLP_ERR_CUDA (-2)
#define EGOVLP_ERR_UNSUPPORTED (-3)

namespace egovlp {

typedef __nv_bfloat16 bf16;

void set_last_error(const char* fmt, ...);

#define EGOVLP_CHECK_ARG(cond, ...)                                   \
  do {                                                                \
    if (!(cond)) {                                                    \
      ::egovlp::set_last_error(__VA_ARGS__);                          \
      return EGOVLP_ERR_ARG;                                          \
    }                                                                 \
  } while (0)

#define EGOVLP_CHECK_CUDA(expr)                                                              \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      ::egovlp::set_last_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),       \
                               __FILE__, __LINE__);                                          \
      return EGOVLP_ERR_CUDA;                                                                \
    }                                                                                        \
  } while (0)

#define EGOVLP_CHECK_LAUNCH() EGOVLP_CHECK_CUDA(cudaGetLastError())

int num_sms();

// ------------------------------------------------------------------------------------------
// generic device helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// fp8 e4m3 (e4m3fn: no infinities, largest finite 448) operands with one fp32 scale per row: scale = amax / 448 (1 for
// a row without a nonzero value) and the stored values x * (448 / amax), converted round-to-nearest-even with
// saturation to +-448 (NaN stays NaN).  Both divisions are correctly rounded whatever the compile flags.
constexpr float E4M3_MAX = 448.f;
__device__ __forceinline__ void e4m3_row_scale(float amax, float& scale, float& inv) {
  if (amax > 0.f) { scale = __fdiv_rn(amax, E4M3_MAX); inv = __fdiv_rn(E4M3_MAX, amax); }
  else { scale = 1.f; inv = 1.f; }
}
// four consecutive values -> four e4m3 bytes, a first (lowest address)
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));     // first source -> upper byte
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  return (uint32_t)lo | ((uint32_t)hi << 16);
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_erf_grad(float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

// ------------------------------------------------------------------------------------------
// fp32 pairs.  Epilogues and softmax loops are written two elements at a time; sm_90 has no packed fp32x2
// instructions, so each helper is two scalar round-to-nearest operations (the _rn intrinsics keep the compiler from
// contracting a multiply and an add into an FMA, so results do not depend on how a caller's pairs are combined).
// ------------------------------------------------------------------------------------------
typedef float2 f32x2;
__device__ __forceinline__ f32x2 pk2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void up2(f32x2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

// ------------------------------------------------------------------------------------------
// Counter-based RNG for dropout: Philox4x32-10 keyed by (seed, site), counter = element group.  Stateless, so the
// backward regenerates the forward's mask from (seed, site, index) instead of storing it.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(unsigned long long key, unsigned long long ctr) {
  uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0x2B7E1516u, c3 = 0x28AED2A6u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    const uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    c0 = h1 ^ c1 ^ k0; c1 = l1; c2 = h0 ^ c3 ^ k1; c3 = l0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}
__device__ __forceinline__ unsigned long long dropout_key(unsigned long long seed, uint32_t site) {
  return seed ^ (0x9E3779B97F4A7C15ull * (unsigned long long)(site + 1));
}
// keep-threshold: an element is DROPPED iff its 32 random bits are < p * 2^32
__device__ __forceinline__ uint32_t dropout_threshold(float p) {
  const double t = (double)p * 4294967296.0;
  return t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
}
// drop-path (stochastic depth) factor of sample b: 1 / (1 - p) if word (b & 3) of
// philox4x32_10(dropout_key(seed, site), b / 4) >= dropout_threshold(p), else 0 -- what egovlp_dropout makes of a vector
// of ones at element b
__device__ __forceinline__ float drop_path_factor(unsigned long long seed, uint32_t site, float p, long long b) {
  const uint4 r = philox4x32_10(dropout_key(seed, site), (unsigned long long)(b >> 2));
  const uint32_t w = (b & 3) == 0 ? r.x : (b & 3) == 1 ? r.y : (b & 3) == 2 ? r.z : r.w;
  return w >= dropout_threshold(p) ? 1.f / (1.f - p) : 0.f;
}

// ------------------------------------------------------------------------------------------
// mma.sync m16n8k16 (bf16 in, fp32 accumulate) on 128B-swizzled [rows x 64] bf16 tiles: row r's 16-byte chunk c sits
// at chunk c ^ (r & 7) of its 128-byte row (the layout a SWIZZLE_128B TMA box of 64 bf16 columns writes).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t sw_addr(uint32_t base, int row, int chunk) {
  return base + row * 128 + ((chunk ^ (row & 7)) << 4);
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// A-operand fragment (16 rows x 16 k) of a swizzled [rows x 64] tile: rows r0.., k-step kk
__device__ __forceinline__ void load_a_frag(uint32_t tile, int r0, int kk, int lane, uint32_t (&f)[4]) {
  ldsm_x4(sw_addr(tile, r0 + (lane & 7) + ((lane >> 3) & 1) * 8, kk * 2 + (lane >> 4)), f);
}
// B-operand fragments for two 8-wide n-tiles (n = rows n0..n0+15 of the tile, k = its 64 columns), k-step kk
__device__ __forceinline__ void load_b_frag_nk(uint32_t tile, int n0, int kk, int lane, uint32_t (&f)[4]) {
  ldsm_x4(sw_addr(tile, n0 + (lane & 7) + (lane >> 4) * 8, kk * 2 + ((lane >> 3) & 1)), f);
}
// B-operand fragments with k = rows k0..k0+15 of the tile, n = columns dp*16..dp*16+15 (two n-tiles), transposed load
__device__ __forceinline__ void load_b_frag_kn(uint32_t tile, int k0, int dp, int lane, uint32_t (&f)[4]) {
  ldsm_x4_t(sw_addr(tile, k0 + (lane & 7) + ((lane >> 3) & 1) * 8, dp * 2 + (lane >> 4)), f);
}

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}
// Bounded wait: a protocol bug traps (launch failure reported to the host) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {  // ~2 s at 1.9 GHz
      printf("egovlp: mbarrier timeout block %d thread %d bar %u parity %u\n", blockIdx.x, threadIdx.x, bar, parity);
      __trap();
    }
  }
}

// Same bound without the printf call site: a call inside a wgmma pipeline makes ptxas serialise every wgmma of the
// kernel, and makes the caller's live registers spill around it.  The clock is only read every 1024 polls.
__device__ __forceinline__ void mbar_wait_nocall(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  for (;;) {
#pragma unroll 1
    for (int i = 0; i < 1024; ++i)
      if (mbar_try_wait(bar, parity)) return;
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}

// ------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
// Multicast load: the box lands at the same smem offset in every CTA of `mask` (cluster ranks) and completes
// transaction bytes on the mbarrier at the same offset in each of them.
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1,
                                                      uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// 1-D bulk copy global -> smem (16B-aligned addresses, bytes % 16 == 0), completion on an mbarrier
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
               : "memory");
}
// TMA store smem -> global (rows / columns outside the tensor are clipped), tracked by the issuing thread's bulk groups
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
// TMA reduce smem -> global: adds the box element-wise into the tensor (fp32 add in L2, like red.global.add; rows /
// columns outside the tensor are clipped), tracked by the issuing thread's bulk groups like a store
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still READ their smem source (the buffers of the others may be rewritten)
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// at most N of this thread's bulk groups are incomplete (their global writes included)
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// barrier over `count` threads (a multiple of 32) on hardware barrier `id` (0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ------------------------------------------------------------------------------------------
// thread-block clusters
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// address of the same shared-memory offset in the CTA of the given cluster rank
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t cta_rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(cta_rank));
  return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}

// ------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): issued by all 128 threads of a warpgroup, accumulators in registers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pins accumulator registers in place around wgmma issue / wait, so that the compiler neither reads them before the
// asynchronous MMA has written them nor moves other uses across the wait.
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor (sm_90 wgmma), SWIZZLE_128B.  Offsets in bytes.
// K-major tiles: 128-byte rows, 8-row core groups SBO = 1024 apart (LBO unused).  MN-major tiles: [k][64 mn] slabs of
// 128-byte rows, 8-k-row groups SBO = 1024 apart, slabs of 64 mn LBO apart.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= uint64_t((saddr >> 4) & 0x3FFF);
  d |= uint64_t((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= uint64_t((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= uint64_t(1) << 62;  // layout_type = SWIZZLE_128B
  return d;
}

// ------------------------------------------------------------------------------------------
// host: TMA descriptor encode (driver entry point fetched through the runtime; no libcuda link)
// ------------------------------------------------------------------------------------------
// 2D row-major bf16 tensor [rows, cols] with leading dimension ld (elements); box = [box_rows, box_cols];
// 128B swizzle (box_cols * 2 bytes must be 128).
int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                      uint32_t box_cols);
// the same for fp32 (box_cols * 4 bytes must be 128)
int make_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                     uint32_t box_cols);
// the same for bytes (e4m3; box_cols must be 128)
int make_tmap_2d_u8(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                    uint32_t box_cols);
// Generic N-d (<=5) bf16 map: dims/strides innermost first, strides in elements (stride[0] must be 1).
int make_tmap_nd_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                      const uint32_t* box, bool swizzle128);

}  // namespace egovlp
