// Divided space-time attention of the video tower, forward and backward, with the reference's CLS semantics.
//
// Replaces VarAttention.forward's attention core (model/video_transformer.py:104-133: the head split, q scaling,
// CLS splice, the two einops rearranges, the CLS k/v repeat + cat, attn() = softmax(q k^T) v, and the merges)
// and its autograd.  Input is the QKV GEMM's output qkv[B*S, 3*D] (bf16, q already scaled), output is
// out[B*S, D] (bf16) ready for the proj GEMM -- no rearranged copy, no materialised probabilities.
//
// One CTA per group: (b, head, frame) for space, (b, head, block of PG patches) for time.  The group's
// queries/keys/values are gathered straight from qkv by ONE 5-D TMA box each (128B-swizzled rows of one head),
// the CLS token's q/k/v row is appended as row NP.  A group's rows carry a group id (time: the patch, space: 0);
// query r may attend key c iff  gid[c] == gid[r]  or c is the CLS key; the CLS query attends every patch key
// of the CTA plus the CLS key in the first group only, and its per-group (max, sum, acc) partials are merged by
// a tiny second kernel -- so the CLS-over-all-S row (:112) costs no extra pass over K/V.
// Math: bf16 mma.sync m16n8k16 with fp32 accumulation + fp32 online softmax (exp2).  At head_dim 64 this op does
// <= 98 FLOP per byte it moves (SURVEY.md section 8d): register-resident mma.sync tiles keep S and P out of shared
// memory, and the wgmma pipeline is kept for the GEMMs that carry 96% of the FLOPs.
#include <stdlib.h>

#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {

// wgmma space-attention forward (attention_wgmma.cu), opt-in
bool space_attn_wgmma_supported(int N);
int space_attn_fwd_wgmma(const void* qkv, void* out, float* lse, float* cls_part, int B, int T, int N, int H,
                         cudaStream_t st);

namespace {

constexpr int HD = 64;            // head dim
constexpr int ROW_BYTES = 128;    // one head-row of bf16
constexpr float LOG2E = 1.4426950408889634f;

struct Geom {
  int B, H, T, N, S, D;     // D = H * 64
  int mode;                 // 0 time, 1 space
  int PG;                   // patches per group (time)
  int G;                    // groups per (b, h)
  int NP;                   // patch rows per group (space: N, time: PG*T)
  int NPAD;                 // NP + 1 rounded up to 16
  int gsize;                // rows per group id (space: N, time: T)
};

__device__ __forceinline__ uint32_t sw_addr(uint32_t base, int row, int chunk) {
  return base + row * ROW_BYTES + ((chunk ^ (row & 7)) << 4);
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

// token (0..S-1) held by smem row r of group g, or -1 for padding / out-of-range patches
__device__ __forceinline__ int row_token(const Geom& G, int g, int r) {
  if (r == G.NP) return 0;
  if (r > G.NP) return -1;
  if (G.mode == 1) return 1 + g * G.N + r;
  const int j = r / G.T, f = r - j * G.T, n = g * G.PG + j;
  return n < G.N ? 1 + f * G.N + n : -1;
}

// The same for the specialised kernels, without the integer division: RT = 1 space, RT = 2 time with T = 1 << sh.
template <int RT>
__device__ __forceinline__ int row_token_x(const Geom& G, int g, int r, int sh) {
  if (RT == 0) return row_token(G, g, r);
  if (r == G.NP) return 0;
  if (r > G.NP) return -1;
  if (RT == 1) return 1 + g * G.N + r;
  const int n = g * G.PG + (r >> sh);
  return n < G.N ? 1 + (r & ((1 << sh) - 1)) * G.N + n : -1;
}

struct Smem {
  uint32_t q, k, v, dout;  // tile base addresses (shared space)
  short* gid;              // [NPAD] group id per row; -2 = CLS, -1 = invalid
  float* lse;              // [NPAD]  (backward)
  float* delta;            // [NPAD]  (backward)
  uint32_t stage;          // per-warp staging [warps][16 x 128B]
  uint32_t bar;
};

__device__ __forceinline__ bool pair_valid(int gq, int gk, bool first_group) {
  if (gq >= 0) return gk == gq || gk == -2;
  if (gq == -2) return gk >= 0 || (gk == -2 && first_group);
  return false;
}

// Range of "other side" rows a 16-row tile starting at r0 can interact with: [lo, hi) plus the CLS row NP.
__device__ __forceinline__ void tile_window(const Geom& G, int r0, int& lo, int& hi) {
  if (r0 <= G.NP && G.NP < r0 + 16) { lo = 0; hi = G.NP; return; }   // tile holds the CLS row: everything
  if (r0 > G.NP) { lo = 0; hi = 0; return; }
  lo = (r0 / G.gsize) * G.gsize;
  hi = min(G.NP, ((r0 + 15) / G.gsize + 1) * G.gsize);
}
__device__ __forceinline__ bool span_active(const Geom& G, int lo, int hi, int c0, int width) {
  return (c0 < hi && c0 + width > lo) || (c0 <= G.NP && G.NP < c0 + width);
}

// Stage a 16 x 64 fp32 fragment tile (mma C layout, 8 n-tiles) as bf16 into the warp's staging rows, then write
// each valid row as one 128-byte line to dst[(b*S + token) * ld + col0 ...].
template <int RT = 0>
__device__ __forceinline__ void store_rows_bf16(const float (&acc)[8][4], float s0, float s1, uint32_t stage,
                                                uint8_t* stage_gen, bf16* dst, long long ld, int col0, const Geom& G,
                                                int b, int g, int r0, int lane, bool skip_cls, int sh = 0) {
  const int gq = lane >> 2, t = lane & 3;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t lo = pack_bf16x2(acc[j][0] * s0, acc[j][1] * s0), hi = pack_bf16x2(acc[j][2] * s1, acc[j][3] * s1);
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(sw_addr(stage, gq, j) + t * 4), "r"(lo));
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(sw_addr(stage, gq + 8, j) + t * 4), "r"(hi));
  }
  __syncwarp();
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int rr = p * 4 + (lane >> 3), c = lane & 7;
    const int tok = row_token_x<RT>(G, g, r0 + rr, sh);
    if (tok > 0 || (tok == 0 && !skip_cls)) {
      const uint4 v = *reinterpret_cast<const uint4*>(stage_gen + (sw_addr(stage, rr, c) - stage));
      *reinterpret_cast<uint4*>(dst + ((long long)b * G.S + tok) * ld + col0 + c * 8) = v;
    }
  }
  __syncwarp();
}

// Same, straight from the fragments (each quad writes 16 contiguous bytes of a row): used by the backward, whose
// four resident tiles leave no room for staging when two CTAs share an SM.
template <int RT = 0>
__device__ __forceinline__ void store_frag_rows_bf16(const float (&acc)[8][4], float s, bf16* dst, long long ld, int col0,
                                                     const Geom& G, int b, int g, int r0, int lane, float s_hi = -1.f,
                                                     int sh = 0) {
  const float sB = s_hi >= 0.f ? s_hi : s;   // optional separate scale for the rows g+8
  const int gq = lane >> 2, t = lane & 3;
  const int tok0 = row_token_x<RT>(G, g, r0 + gq, sh), tok1 = row_token_x<RT>(G, g, r0 + gq + 8, sh);
  bf16* p0 = dst + ((long long)b * G.S + tok0) * ld + col0 + 2 * t;
  bf16* p1 = dst + ((long long)b * G.S + tok1) * ld + col0 + 2 * t;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (tok0 > 0) *reinterpret_cast<uint32_t*>(p0 + 8 * j) = pack_bf16x2(acc[j][0] * s, acc[j][1] * s);
    if (tok1 > 0) *reinterpret_cast<uint32_t*>(p1 + 8 * j) = pack_bf16x2(acc[j][2] * sB, acc[j][3] * sB);
  }
}

// A 16-row tile is "uniform" when all its rows are valid patch rows of one group id; an 8-wide tile on the other
// side is then fully attendable (no masking, no gid lookups) iff its first and last rows carry that same id.
__device__ __forceinline__ int tile_uniform_gid(const short* gid, int r0) {
  const int a = gid[r0], b = gid[r0 + 15];
  return (a >= 0 && a == b) ? a : -1;
}

// Head index fastest: the H CTAs launched back to back read the H adjacent 128-byte head slices of the SAME token
// rows (q/k/v of one token are 3 x H x 128 B contiguous), so the scattered row reads of a group land in DRAM pages
// that are already open instead of each 128-byte granule paying its own activation.
__device__ __forceinline__ void decode_block(const Geom& G, int& b, int& h, int& g) {
  h = blockIdx.x % G.H;
  const int bg = blockIdx.x / G.H;
  g = bg % G.G;
  b = bg / G.G;
}

// Shared prologue: carve smem, gather the group's tiles (TMA) + CLS rows (manual), build the gid table.
template <bool BWD, bool STAGE = !BWD, bool WAIT = true, bool GID = true>
__device__ __forceinline__ void load_group(const Geom& G, const CUtensorMap* tm_qkv, const CUtensorMap* tm_do,
                                           const bf16* qkv, const bf16* dout, int b, int h, int g, uint8_t* smem_gen,
                                           uint32_t smem_base, Smem& sm, int nwarps) {
  const int tile_bytes = G.NPAD * ROW_BYTES;
  sm.q = smem_base;
  sm.k = sm.q + tile_bytes;
  sm.v = sm.k + tile_bytes;
  sm.dout = sm.v + tile_bytes;
  uint32_t off = (BWD ? 4 : 3) * tile_bytes;
  sm.stage = smem_base + off;
  if (STAGE) off += nwarps * 16 * ROW_BYTES;
  sm.lse = reinterpret_cast<float*>(smem_gen + off);
  off += G.NPAD * 4;
  sm.delta = reinterpret_cast<float*>(smem_gen + off);
  off += G.NPAD * 4;
  sm.gid = reinterpret_cast<short*>(smem_gen + off);
  off += ((G.NPAD * 2 + 15) / 16) * 16;
  sm.bar = smem_base + off;

  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(sm.bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  const int ntiles = BWD ? 4 : 3;
  if (tid == 0) {
    const int rows = (G.mode == 1) ? G.N : G.T * G.PG;
    mbar_expect_tx(sm.bar, (uint32_t)(ntiles * rows * ROW_BYTES));
    const int f0 = (G.mode == 1) ? g : 0, n0 = (G.mode == 1) ? 0 : g * G.PG;
    tma_load_5d(sm.q, tm_qkv, sm.bar, 0, f0, n0, 0 * G.H + h, b);
    tma_load_5d(sm.k, tm_qkv, sm.bar, 0, f0, n0, 1 * G.H + h, b);
    tma_load_5d(sm.v, tm_qkv, sm.bar, 0, f0, n0, 2 * G.H + h, b);
    if (BWD) tma_load_5d(sm.dout, tm_do, sm.bar, 0, f0, n0, h, b);
  }
  // CLS rows (row NP) + zero padding rows NP+1 .. NPAD-1, 16B chunks
  const int pad_rows = G.NPAD - G.NP;   // >= 1
  for (int i = tid; i < pad_rows * 8; i += blockDim.x) {
    const int c = i & 7, rr = i >> 3;
#pragma unroll
    for (int which = 0; which < ntiles; ++which) {
      uint4 val = make_uint4(0, 0, 0, 0);
      if (rr == 0) {
        const bf16* src = (which < 3) ? qkv + (long long)b * G.S * 3 * G.D + which * G.D + h * HD
                                      : dout + (long long)b * G.S * G.D + h * HD;
        val = *reinterpret_cast<const uint4*>(src + c * 8);
      }
      *reinterpret_cast<uint4*>(smem_gen + (sw_addr(sm.q + which * tile_bytes, G.NP + rr, c) - smem_base)) = val;
    }
  }
  if (GID) {                            // group-id table: only the generic kernels look rows up in it
    for (int r = tid; r < G.NPAD; r += blockDim.x) {
      short gid = -1;
      if (r == G.NP) gid = -2;
      else if (r < G.NP && row_token(G, g, r) > 0) gid = (short)(r / G.gsize);
      sm.gid[r] = gid;
    }
  }
  __syncthreads();
  if (WAIT) mbar_wait(sm.bar, 0);     // !WAIT: the caller overlaps its own global loads with the TMA flight time
}

// ------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------
template <int NWARPS, int MINB>
__global__ void __launch_bounds__(NWARPS * 32, MINB)
divided_attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const bf16* __restrict__ qkv,
                        bf16* __restrict__ out, float* __restrict__ lse_out, float* __restrict__ cls_part, Geom G) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  int b, h, g;
  decode_block(G, b, h, g);
  Smem sm;
  load_group<false>(G, &tm_qkv, nullptr, qkv, nullptr, b, h, g, smem_gen, smem_base, sm, NWARPS);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gq = lane >> 2, t = lane & 3;
  const bool first_group = (g == 0);
  const int NT = G.NPAD / 8;
  const uint32_t stage = sm.stage + warp * 16 * ROW_BYTES;
  uint8_t* stage_gen = smem_gen + (stage - smem_base);

  for (int rt = warp; rt * 16 <= G.NP; rt += NWARPS) {
    const int r0 = rt * 16;
    int lo, hi;
    tile_window(G, r0, lo, hi);
    uint32_t qf[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) load_a_frag(sm.q, r0, kk, lane, qf[kk]);
    const int gid0 = sm.gid[r0 + gq], gid1 = sm.gid[r0 + gq + 8];
    const int ugid = tile_uniform_gid(sm.gid, r0);
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }

    for (int c0 = 0; c0 < NT; c0 += 8) {     // chunk of 8 n-tiles = 64 keys
      if (!span_active(G, lo, hi, c0 * 8, 64)) continue;
      float s[8][4];
#pragma unroll
      for (int j = 0; j < 8; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int n0 = (c0 + 2 * p) * 8;
        if (c0 + 2 * p < NT && span_active(G, lo, hi, n0, 16)) {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            uint32_t bf[4];
            load_b_frag_nk(sm.k, n0, kk, lane, bf);
            mma_bf16(s[2 * p], qf[kk], bf[0], bf[1]);
            mma_bf16(s[2 * p + 1], qf[kk], bf[2], bf[3]);
          }
        }
      }
      // mask (skipped for tiles that are fully attendable by every row of this tile)
      float cm0 = -INFINITY, cm1 = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = (c0 + j) * 8 + 2 * t;
        const bool inb = (c0 + j) < NT;
        const bool fast = inb && ugid >= 0 && sm.gid[(c0 + j) * 8] == ugid && sm.gid[(c0 + j) * 8 + 7] == ugid;
        if (!fast) {
          const int k0 = inb ? sm.gid[col] : -1, k1 = inb ? sm.gid[col + 1] : -1;
          s[j][0] = pair_valid(gid0, k0, first_group) ? s[j][0] : -INFINITY;
          s[j][1] = pair_valid(gid0, k1, first_group) ? s[j][1] : -INFINITY;
          s[j][2] = pair_valid(gid1, k0, first_group) ? s[j][2] : -INFINITY;
          s[j][3] = pair_valid(gid1, k1, first_group) ? s[j][3] : -INFINITY;
        }
        cm0 = fmaxf(cm0, fmaxf(s[j][0], s[j][1]));
        cm1 = fmaxf(cm1, fmaxf(s[j][2], s[j][3]));
      }
      cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 1)); cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 2));
      cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 1)); cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 2));
      const float mn0 = fmaxf(m0, cm0), mn1 = fmaxf(m1, cm1);
      const float ms0 = (mn0 == -INFINITY) ? 0.f : mn0, ms1 = (mn1 == -INFINITY) ? 0.f : mn1;
      const float a0 = exp2f((m0 - ms0) * LOG2E), a1 = exp2f((m1 - ms1) * LOG2E);   // m = -inf -> 0
      m0 = mn0; m1 = mn1;
      l0 *= a0; l1 *= a1;
#pragma unroll
      for (int j = 0; j < 8; ++j) { o[j][0] *= a0; o[j][1] *= a0; o[j][2] *= a1; o[j][3] *= a1; }
      uint32_t pf[4][4];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float p0 = exp2f((s[j][0] - ms0) * LOG2E), p1 = exp2f((s[j][1] - ms0) * LOG2E);
        const float p2 = exp2f((s[j][2] - ms1) * LOG2E), p3 = exp2f((s[j][3] - ms1) * LOG2E);
        l0 += p0 + p1; l1 += p2 + p3;
        pf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0, p1);
        pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
      }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const int k0 = (c0 + 2 * kk) * 8;
        if (c0 + 2 * kk < NT && span_active(G, lo, hi, k0, 16)) {
#pragma unroll
          for (int dp = 0; dp < 4; ++dp) {
            uint32_t bf[4];
            load_b_frag_kn(sm.v, k0, dp, lane, bf);
            mma_bf16(o[2 * dp], pf[kk], bf[0], bf[1]);
            mma_bf16(o[2 * dp + 1], pf[kk], bf[2], bf[3]);
          }
        }
      }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    // CLS query row: un-normalised partial for the merge kernel
    {
      const int rc = G.NP - r0;   // local index of the CLS row in this tile, if any
      if (rc >= 0 && rc < 16 && (rc & 7) == gq) {
        const bool hi_half = rc >= 8;
        float* dst = cls_part + (((long long)(b * G.H + h)) * G.G + g) * 66;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          dst[j * 8 + 2 * t] = hi_half ? o[j][2] : o[j][0];
          dst[j * 8 + 2 * t + 1] = hi_half ? o[j][3] : o[j][1];
        }
        if (t == 0) { dst[64] = hi_half ? m1 : m0; dst[65] = hi_half ? l1 : l0; }
      }
    }
    const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
    if (t == 0) {
      const int tok0 = row_token(G, g, r0 + gq), tok1 = row_token(G, g, r0 + gq + 8);
      if (tok0 > 0) lse_out[((long long)(b * G.H + h)) * G.S + tok0] = m0 + logf(l0);
      if (tok1 > 0) lse_out[((long long)(b * G.H + h)) * G.S + tok1] = m1 + logf(l1);
    }
    store_rows_bf16(o, i0, i1, stage, stage_gen, out, G.D, h * HD, G, b, g, r0, lane, /*skip_cls=*/true);
  }
}

// merge the per-group partials of the CLS query: one warp per (b, h)
__global__ void cls_merge_kernel(const float* __restrict__ part, bf16* __restrict__ out, float* __restrict__ lse,
                                 int BH, int H, int Gn, int S, int D) {
  const int bh = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (bh >= BH) return;
  const int lane = threadIdx.x & 31;
  const float* p = part + (long long)bh * Gn * 66;
  float M = -INFINITY;
  for (int g = 0; g < Gn; ++g) M = fmaxf(M, p[g * 66 + 64]);
  float L = 0.f, o0 = 0.f, o1 = 0.f;
  for (int g = 0; g < Gn; ++g) {
    const float mg = p[g * 66 + 64];
    const float w = (mg == -INFINITY) ? 0.f : exp2f((mg - M) * LOG2E);
    L += p[g * 66 + 65] * w;
    o0 += p[g * 66 + 2 * lane] * w;
    o1 += p[g * 66 + 2 * lane + 1] * w;
  }
  const int b = bh / H, h = bh % H;
  const float inv = 1.f / L;
  *reinterpret_cast<uint32_t*>(out + (long long)b * S * D + h * HD + 2 * lane) = pack_bf16x2(o0 * inv, o1 * inv);
  if (lane == 0) lse[(long long)bh * S] = M + logf(L);
}

// ------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------
template <int NWARPS, int MINB>
__global__ void __launch_bounds__(NWARPS * 32, MINB)
divided_attn_bwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                        const bf16* __restrict__ qkv, const bf16* __restrict__ out, const bf16* __restrict__ dout,
                        const float* __restrict__ lse_in, bf16* __restrict__ dqkv, float* __restrict__ dcls,
                        float q_scale, Geom G) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  int b, h, g;
  decode_block(G, b, h, g);
  Smem sm;
  load_group<true>(G, &tm_qkv, &tm_do, qkv, dout, b, h, g, smem_gen, smem_base, sm, NWARPS);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gq = lane >> 2, t = lane & 3;
  const bool first_group = (g == 0);
  const int NT = G.NPAD / 8;

  // phase 0: lse (log2 units) and delta = rowsum(dO * O) per row
  for (int r = warp * 4 + (lane >> 3); r < G.NPAD; r += NWARPS * 4) {
    const int tok = row_token(G, g, r), c = lane & 7;
    float d = 0.f;
    if (tok >= 0) {
      const uint4 ov = *reinterpret_cast<const uint4*>(out + ((long long)b * G.S + tok) * G.D + h * HD + c * 8);
      const uint4 dv = *reinterpret_cast<const uint4*>(smem_gen + (sw_addr(sm.dout, r, c) - smem_base));
      const uint32_t ou[4] = {ov.x, ov.y, ov.z, ov.w}, du[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 a = unpack_bf16x2(ou[i]), bb = unpack_bf16x2(du[i]);
        d += a.x * bb.x + a.y * bb.y;
      }
    }
    d += __shfl_xor_sync(0xffffffffu, d, 1); d += __shfl_xor_sync(0xffffffffu, d, 2); d += __shfl_xor_sync(0xffffffffu, d, 4);
    if (c == 0) {
      sm.delta[r] = d;
      sm.lse[r] = tok >= 0 ? lse_in[((long long)(b * G.H + h)) * G.S + tok] * LOG2E : 0.f;
    }
  }
  __syncthreads();

  // phase 1: per 16 query rows -> dQ
  for (int rt = warp; rt * 16 <= G.NP; rt += NWARPS) {
    const int r0 = rt * 16;
    int lo, hi;
    tile_window(G, r0, lo, hi);
    const int gid0 = sm.gid[r0 + gq], gid1 = sm.gid[r0 + gq + 8];
    const int ugid = tile_uniform_gid(sm.gid, r0);
    const float ls0 = sm.lse[r0 + gq], ls1 = sm.lse[r0 + gq + 8], de0 = sm.delta[r0 + gq], de1 = sm.delta[r0 + gq + 8];
    float dq[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f; }
    for (int c0 = 0; c0 < NT; c0 += 4) {     // chunk of 4 n-tiles = 32 keys
      if (!span_active(G, lo, hi, c0 * 8, 32)) continue;
      float s[4][4], dp[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; dp[j][0] = dp[j][1] = dp[j][2] = dp[j][3] = 0.f; }
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int n0 = (c0 + 2 * p) * 8;
        if (c0 + 2 * p < NT && span_active(G, lo, hi, n0, 16)) {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            uint32_t af[4], bf[4];     // A fragments re-read per use: registers are what limits CTAs per SM here
            load_a_frag(sm.q, r0, kk, lane, af);
            load_b_frag_nk(sm.k, n0, kk, lane, bf);
            mma_bf16(s[2 * p], af, bf[0], bf[1]);
            mma_bf16(s[2 * p + 1], af, bf[2], bf[3]);
            load_a_frag(sm.dout, r0, kk, lane, af);
            load_b_frag_nk(sm.v, n0, kk, lane, bf);
            mma_bf16(dp[2 * p], af, bf[0], bf[1]);
            mma_bf16(dp[2 * p + 1], af, bf[2], bf[3]);
          }
        }
      }
      uint32_t dsf[2][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = (c0 + j) * 8 + 2 * t;
        const bool inb = (c0 + j) < NT;
        const bool fast = inb && ugid >= 0 && sm.gid[(c0 + j) * 8] == ugid && sm.gid[(c0 + j) * 8 + 7] == ugid;
        bool v0 = true, v1 = true, v2 = true, v3 = true;
        if (!fast) {
          const int k0 = inb ? sm.gid[col] : -1, k1 = inb ? sm.gid[col + 1] : -1;
          v0 = pair_valid(gid0, k0, first_group); v1 = pair_valid(gid0, k1, first_group);
          v2 = pair_valid(gid1, k0, first_group); v3 = pair_valid(gid1, k1, first_group);
        }
        const float p0 = v0 ? exp2f(s[j][0] * LOG2E - ls0) : 0.f;
        const float p1 = v1 ? exp2f(s[j][1] * LOG2E - ls0) : 0.f;
        const float p2 = v2 ? exp2f(s[j][2] * LOG2E - ls1) : 0.f;
        const float p3 = v3 ? exp2f(s[j][3] * LOG2E - ls1) : 0.f;
        dsf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0 * (dp[j][0] - de0), p1 * (dp[j][1] - de0));
        dsf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2 * (dp[j][2] - de1), p3 * (dp[j][3] - de1));
      }
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        const int k0 = (c0 + 2 * kk) * 8;
        if (c0 + 2 * kk < NT && span_active(G, lo, hi, k0, 16)) {
#pragma unroll
          for (int dpi = 0; dpi < 4; ++dpi) {
            uint32_t bf[4];
            load_b_frag_kn(sm.k, k0, dpi, lane, bf);
            mma_bf16(dq[2 * dpi], dsf[kk], bf[0], bf[1]);
            mma_bf16(dq[2 * dpi + 1], dsf[kk], bf[2], bf[3]);
          }
        }
      }
    }
    // CLS query row -> fp32 atomics (summed over groups); patch rows -> dqkv q-columns (scaled back)
    {
      const int rc = G.NP - r0;
      if (rc >= 0 && rc < 16 && (rc & 7) == gq) {
        const bool hi_half = rc >= 8;
        float* dst = dcls + ((long long)(b * G.H + h) * 3 + 0) * HD;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          atomicAdd(dst + j * 8 + 2 * t, hi_half ? dq[j][2] : dq[j][0]);
          atomicAdd(dst + j * 8 + 2 * t + 1, hi_half ? dq[j][3] : dq[j][1]);
        }
      }
    }
    store_frag_rows_bf16(dq, q_scale, dqkv, 3 * G.D, h * HD, G, b, g, r0, lane);
  }

  // phase 2: per 16 keys -> dK, dV
  for (int kt = warp; kt * 16 <= G.NP; kt += NWARPS) {
    const int k0r = kt * 16;
    int lo, hi;
    tile_window(G, k0r, lo, hi);
    const int gid0 = sm.gid[k0r + gq], gid1 = sm.gid[k0r + gq + 8];
    const int ugid = tile_uniform_gid(sm.gid, k0r);
    float dk[8][4], dv[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = 0.f; dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f; }
    for (int c0 = 0; c0 < NT; c0 += 4) {     // chunk of 4 n-tiles = 32 queries
      if (!span_active(G, lo, hi, c0 * 8, 32)) continue;
      float st[4][4], dpt[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { st[j][0] = st[j][1] = st[j][2] = st[j][3] = 0.f; dpt[j][0] = dpt[j][1] = dpt[j][2] = dpt[j][3] = 0.f; }
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int n0 = (c0 + 2 * p) * 8;
        if (c0 + 2 * p < NT && span_active(G, lo, hi, n0, 16)) {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            uint32_t af[4], bf[4];
            load_a_frag(sm.k, k0r, kk, lane, af);
            load_b_frag_nk(sm.q, n0, kk, lane, bf);
            mma_bf16(st[2 * p], af, bf[0], bf[1]);
            mma_bf16(st[2 * p + 1], af, bf[2], bf[3]);
            load_a_frag(sm.v, k0r, kk, lane, af);
            load_b_frag_nk(sm.dout, n0, kk, lane, bf);
            mma_bf16(dpt[2 * p], af, bf[0], bf[1]);
            mma_bf16(dpt[2 * p + 1], af, bf[2], bf[3]);
          }
        }
      }
      uint32_t pf[2][4], dsf[2][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = (c0 + j) * 8 + 2 * t;       // query index
        const bool inb = (c0 + j) < NT;
        const bool fast = inb && ugid >= 0 && sm.gid[(c0 + j) * 8] == ugid && sm.gid[(c0 + j) * 8 + 7] == ugid;
        bool v0 = true, v1 = true, v2 = true, v3 = true;
        if (!fast) {
          const int q0 = inb ? sm.gid[col] : -1, q1 = inb ? sm.gid[col + 1] : -1;
          v0 = pair_valid(q0, gid0, first_group); v1 = pair_valid(q1, gid0, first_group);
          v2 = pair_valid(q0, gid1, first_group); v3 = pair_valid(q1, gid1, first_group);
        }
        const float lq0 = inb ? sm.lse[col] : 0.f, lq1 = inb ? sm.lse[col + 1] : 0.f;
        const float dq0 = inb ? sm.delta[col] : 0.f, dq1 = inb ? sm.delta[col + 1] : 0.f;
        const float p0 = v0 ? exp2f(st[j][0] * LOG2E - lq0) : 0.f;
        const float p1 = v1 ? exp2f(st[j][1] * LOG2E - lq1) : 0.f;
        const float p2 = v2 ? exp2f(st[j][2] * LOG2E - lq0) : 0.f;
        const float p3 = v3 ? exp2f(st[j][3] * LOG2E - lq1) : 0.f;
        pf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0, p1);
        pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
        dsf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0 * (dpt[j][0] - dq0), p1 * (dpt[j][1] - dq1));
        dsf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2 * (dpt[j][2] - dq0), p3 * (dpt[j][3] - dq1));
      }
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        const int q0r = (c0 + 2 * kk) * 8;
        if (c0 + 2 * kk < NT && span_active(G, lo, hi, q0r, 16)) {
#pragma unroll
          for (int dpi = 0; dpi < 4; ++dpi) {
            uint32_t bf[4];
            load_b_frag_kn(sm.dout, q0r, dpi, lane, bf);
            mma_bf16(dv[2 * dpi], pf[kk], bf[0], bf[1]);
            mma_bf16(dv[2 * dpi + 1], pf[kk], bf[2], bf[3]);
            load_b_frag_kn(sm.q, q0r, dpi, lane, bf);
            mma_bf16(dk[2 * dpi], dsf[kk], bf[0], bf[1]);
            mma_bf16(dk[2 * dpi + 1], dsf[kk], bf[2], bf[3]);
          }
        }
      }
    }
    {
      const int rc = G.NP - k0r;
      if (rc >= 0 && rc < 16 && (rc & 7) == gq) {
        const bool hi_half = rc >= 8;
        float* dstk = dcls + ((long long)(b * G.H + h) * 3 + 1) * HD;
        float* dstv = dcls + ((long long)(b * G.H + h) * 3 + 2) * HD;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          atomicAdd(dstk + j * 8 + 2 * t, hi_half ? dk[j][2] : dk[j][0]);
          atomicAdd(dstk + j * 8 + 2 * t + 1, hi_half ? dk[j][3] : dk[j][1]);
          atomicAdd(dstv + j * 8 + 2 * t, hi_half ? dv[j][2] : dv[j][0]);
          atomicAdd(dstv + j * 8 + 2 * t + 1, hi_half ? dv[j][3] : dv[j][1]);
        }
      }
    }
    store_frag_rows_bf16(dk, 1.f, dqkv, 3 * G.D, G.D + h * HD, G, b, g, k0r, lane);
    store_frag_rows_bf16(dv, 1.f, dqkv, 3 * G.D, 2 * G.D + h * HD, G, b, g, k0r, lane);
  }
}

// dqkv[b, 0, which*D + h*64 + d] = bf16(dcls[b,h,which,d] * (which == 0 ? q_scale : 1))
__global__ void cls_grad_finalize_kernel(const float* __restrict__ dcls, bf16* __restrict__ dqkv, int B, int H, int S,
                                         int D, float q_scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H * 3 * HD) return;
  const int d = i % HD, which = (i / HD) % 3, h = (i / (3 * HD)) % H, b = i / (3 * HD * H);
  const float v = dcls[i] * (which == 0 ? q_scale : 1.f);
  dqkv[(long long)b * S * 3 * D + which * D + h * HD + d] = __float2bfloat16(v);
}

// ------------------------------------------------------------------------------------------------------------
// Specialised ("fast") kernels.  Same math and layout as the generic kernels above, but the rows a 16-row tile
// interacts with are given as CHUNKS of 1-4 sixteen-row "pairs" (pair = two 8-wide mma n-tiles) instead of a
// per-element group-id lookup; the chunk body is compiled per pair count, ldmatrix addresses are one add from
// per-thread constants, and masks are arithmetic and only evaluated for the pairs that need them:
//   space : pairs 0,16,..  in chunks of 4 (fwd) / 2 (bwd); only the tail pair(s) (last patches, CLS key, padding)
//           are masked;
//   time  (T in {4, 8, 16}; 112 patch rows per group, row = patch*T + frame):
//           a patch tile sees ONE chunk of two pairs: its own 16 rows (block-diagonal inside when T < 16) and the
//           CLS pair; the CLS row is split into NWARPS parts of 32 rows, one chunk each (its results are
//           partials / atomics anyway, so the parts need no reduction).
// ------------------------------------------------------------------------------------------------------------
struct FragOff {
  uint32_t a[4];   // A fragments (and transposed B fragments): + tile + row0 * 128
  uint32_t b[4];   // B fragments, n = rows: + tile + n0 * 128
};
__device__ __forceinline__ FragOff make_frag_off(int lane) {
  FragOff f;
  const int ra = (lane & 7) + ((lane >> 3) & 1) * 8, ca = lane >> 4;
  const int rb = (lane & 7) + (lane >> 4) * 8, cb = (lane >> 3) & 1;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    f.a[k] = ra * ROW_BYTES + (((k * 2 + ca) ^ (ra & 7)) << 4);
    f.b[k] = rb * ROW_BYTES + (((k * 2 + cb) ^ (rb & 7)) << 4);
  }
  return f;
}

struct Chunk {
  int np;          // pairs in this chunk (1..4)
  int base[4];     // first row of each pair on the other side
  uint32_t mask;   // bit p: pair p needs masking
};

struct FastCtx {
  int NP, NPAD, sh, valid_keys;
  bool first_group;
};

// may query row q attend key row k?
template <bool TIME>
__device__ __forceinline__ bool fast_valid(const FastCtx& c, int q, int k) {
  if (k < c.NP) {
    if (!TIME) return true;
    return q == c.NP ? k < c.valid_keys : (q >> c.sh) == (k >> c.sh);
  }
  return k == c.NP && (q != c.NP || c.first_group);
}

// Work items of a CTA: (r0, part).  space: 16-row tiles 0 .. NP/16.  time: NP/16 patch tiles, then NWARPS CLS parts.
template <bool TIME, int NWARPS>
__device__ __forceinline__ bool work_item(const FastCtx& c, int it, int& r0, int& part) {
  part = -1;
  if (!TIME) {
    r0 = it * 16;
    return r0 <= c.NP;
  }
  const int n_tiles = c.NP >> 4;
  if (it < n_tiles) { r0 = it * 16; return true; }
  part = it - n_tiles;
  r0 = c.NP;
  return part < NWARPS;
}
// chunk `ci` of a work item, CW = pairs per chunk in the dense (space) case; returns false when past the end
template <bool TIME, int NWARPS, int CW>
__device__ __forceinline__ bool get_chunk(const FastCtx& c, int T, int r0, int part, int ci, Chunk& ch) {
  if (TIME) {
    if (ci > 0 && (part < 0 || CW >= 2)) return false;
    if (part < 0) {                 // patch tile: own rows + the CLS pair
      ch.np = 2; ch.base[0] = r0; ch.base[1] = c.NP; ch.mask = (T < 16 ? 1u : 0u) | 2u;
      return true;
    }
    const int w = c.NPAD / NWARPS;  // CLS part: w (= 32 or 16) consecutive rows
    if (CW >= 2 && NWARPS > 4) { ch.np = 1; ch.base[0] = part * w; ch.mask = 1u; return true; }
    if (CW >= 2) { ch.np = 2; ch.base[0] = part * w; ch.base[1] = part * w + 16; ch.mask = 3u; return true; }
    if (ci >= 2) return false;
    ch.np = 1; ch.base[0] = part * w + 16 * ci; ch.mask = 1u;
    return true;
  }
  const int k0 = ci * CW * 16;
  if (k0 >= c.NPAD) return false;
  ch.np = min(CW, (c.NPAD - k0) >> 4);
  ch.mask = 0;
#pragma unroll
  for (int p = 0; p < 4; ++p) ch.base[p] = k0 + 16 * p;
  const int first_masked = c.NP & ~15;            // the pair holding the last patches, the CLS key and the padding
  if (k0 + CW * 16 > first_masked) {              // only the tail chunk(s) pay for the mask bits
#pragma unroll
    for (int p = 0; p < CW; ++p)
      if (p < ch.np && k0 + 16 * p + 16 > first_masked) ch.mask |= 1u << p;
  }
  return true;
}

// ---- forward chunk: S = Q K^T over NPR pairs, online softmax update, O += P V
template <bool TIME, int NPR>
__device__ __forceinline__ void fwd_chunk(const FastCtx& c, const Smem& sm, const FragOff& fo, const Chunk& ch,
                                          const uint32_t (&qf)[4][4], int rowA, int rowB, int t, float& m0, float& m1,
                                          float& l0, float& l1, float (&o)[8][4]) {
  float s[2 * NPR][4];
#pragma unroll
  for (int j = 0; j < 2 * NPR; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
  for (int p = 0; p < NPR; ++p) {
    const uint32_t kb = sm.k + ch.base[p] * ROW_BYTES;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t bf[4];
      ldsm_x4(kb + fo.b[kk], bf);
      mma_bf16(s[2 * p], qf[kk], bf[0], bf[1]);
      mma_bf16(s[2 * p + 1], qf[kk], bf[2], bf[3]);
    }
  }
  if (ch.mask) {
#pragma unroll
    for (int p = 0; p < NPR; ++p) {
      if (ch.mask & (1u << p)) {
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int j = 2 * p + jj, col = ch.base[p] + 8 * jj + 2 * t;
          if (TIME && ch.base[p] == c.NP && rowA < c.NP) {    // patch rows x the CLS pair: only column NP is a key
            const bool kc = jj == 0 && t == 0;
            s[j][0] = kc ? s[j][0] : -INFINITY; s[j][1] = -INFINITY;
            s[j][2] = kc ? s[j][2] : -INFINITY; s[j][3] = -INFINITY;
          } else if (TIME && rowA >= c.NP && ch.base[p] < c.NP) {   // CLS tile x patch keys: row NP sees the valid keys
            const bool cq = rowA == c.NP;
            s[j][0] = (cq && col < c.valid_keys) ? s[j][0] : -INFINITY;
            s[j][1] = (cq && col + 1 < c.valid_keys) ? s[j][1] : -INFINITY;
            s[j][2] = -INFINITY; s[j][3] = -INFINITY;
          } else {
            s[j][0] = fast_valid<TIME>(c, rowA, col) ? s[j][0] : -INFINITY;
            s[j][1] = fast_valid<TIME>(c, rowA, col + 1) ? s[j][1] : -INFINITY;
            s[j][2] = fast_valid<TIME>(c, rowB, col) ? s[j][2] : -INFINITY;
            s[j][3] = fast_valid<TIME>(c, rowB, col + 1) ? s[j][3] : -INFINITY;
          }
        }
      }
    }
  }
  float cm0 = -INFINITY, cm1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 2 * NPR; ++j) {
    cm0 = fmaxf(cm0, fmaxf(s[j][0], s[j][1]));
    cm1 = fmaxf(cm1, fmaxf(s[j][2], s[j][3]));
  }
  cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 1)); cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 2));
  cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 1)); cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 2));
  const float mn0 = fmaxf(m0, cm0), mn1 = fmaxf(m1, cm1);
  const float ms0 = (mn0 == -INFINITY) ? 0.f : mn0 * LOG2E, ms1 = (mn1 == -INFINITY) ? 0.f : mn1 * LOG2E;
  const float a0 = exp2f(m0 * LOG2E - ms0), a1 = exp2f(m1 * LOG2E - ms1);
  m0 = mn0; m1 = mn1;
  // packed fp32x2 (FFMA2 / FMUL2 / FADD2): the softmax bookkeeping is issue-bound next to the mma stream
  const f32x2 av0 = pk2(a0, a0), av1 = pk2(a1, a1);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    up2(mul2(pk2(o[j][0], o[j][1]), av0), o[j][0], o[j][1]);
    up2(mul2(pk2(o[j][2], o[j][3]), av1), o[j][2], o[j][3]);
  }
  const f32x2 sc = pk2(LOG2E, LOG2E), nm0 = pk2(-ms0, -ms0), nm1 = pk2(-ms1, -ms1);
  f32x2 la0 = pk2(l0 * a0, 0.f), la1 = pk2(l1 * a1, 0.f);
  uint32_t pf[NPR][4];
#pragma unroll
  for (int j = 0; j < 2 * NPR; ++j) {
    float e0, e1, e2, e3;
    up2(fma2(pk2(s[j][0], s[j][1]), sc, nm0), e0, e1);
    up2(fma2(pk2(s[j][2], s[j][3]), sc, nm1), e2, e3);
    const float p0 = exp2f(e0), p1 = exp2f(e1), p2 = exp2f(e2), p3 = exp2f(e3);
    la0 = add2(la0, pk2(p0, p1));
    la1 = add2(la1, pk2(p2, p3));
    pf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0, p1);
    pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
  }
  {
    float x, y;
    up2(la0, x, y); l0 = x + y;
    up2(la1, x, y); l1 = x + y;
  }
#pragma unroll
  for (int p = 0; p < NPR; ++p) {
    const uint32_t vb = sm.v + ch.base[p] * ROW_BYTES;
#pragma unroll
    for (int dp = 0; dp < 4; ++dp) {
      uint32_t bf[4];
      ldsm_x4_t(vb + fo.a[dp], bf);
      mma_bf16(o[2 * dp], pf[p], bf[0], bf[1]);
      mma_bf16(o[2 * dp + 1], pf[p], bf[2], bf[3]);
    }
  }
}

template <bool TIME, int NWARPS, int MINB>
__global__ void __launch_bounds__(NWARPS * 32, MINB)
fast_attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const bf16* __restrict__ qkv, bf16* __restrict__ out,
                     float* __restrict__ lse_out, float* __restrict__ cls_part, Geom G, int sh) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  int b, h, g;
  decode_block(G, b, h, g);
  Smem sm;
  load_group<false, !TIME, true, false>(G, &tm_qkv, nullptr, qkv, nullptr, b, h, g, smem_gen, smem_base, sm, NWARPS);
  constexpr int RT = TIME ? 2 : 1;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gq = lane >> 2, t = lane & 3;
  FastCtx c;
  c.NP = G.NP; c.NPAD = G.NPAD; c.sh = sh; c.first_group = (g == 0);
  c.valid_keys = TIME ? min(G.PG, G.N - g * G.PG) * G.T : G.NP;
  const FragOff fo = make_frag_off(lane);
  const uint32_t stage = sm.stage + warp * 16 * ROW_BYTES;
  uint8_t* stage_gen = smem_gen + (stage - smem_base);

  for (int it = warp;; it += NWARPS) {
    int r0, part;
    if (!work_item<TIME, NWARPS>(c, it, r0, part)) break;
    const int rowA = r0 + gq, rowB = rowA + 8;
    uint32_t qf[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) ldsm_x4(sm.q + r0 * ROW_BYTES + fo.a[kk], qf[kk]);
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }
    Chunk ch;
#pragma unroll 1
    for (int ci = 0; get_chunk<TIME, NWARPS, 4>(c, G.T, r0, part, ci, ch); ++ci) {
      switch (ch.np) {
        case 4: fwd_chunk<TIME, 4>(c, sm, fo, ch, qf, rowA, rowB, t, m0, m1, l0, l1, o); break;
        case 3: fwd_chunk<TIME, 3>(c, sm, fo, ch, qf, rowA, rowB, t, m0, m1, l0, l1, o); break;
        case 2: fwd_chunk<TIME, 2>(c, sm, fo, ch, qf, rowA, rowB, t, m0, m1, l0, l1, o); break;
        default: fwd_chunk<TIME, 1>(c, sm, fo, ch, qf, rowA, rowB, t, m0, m1, l0, l1, o); break;
      }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    {
      const int rc = c.NP - r0;   // local index of the CLS row in this tile, if any
      if (rc >= 0 && rc < 16 && (rc & 7) == gq) {
        const bool hi_half = rc >= 8;
        constexpr int PARTS = TIME ? NWARPS : 1;
        float* dst = cls_part + ((((long long)(b * G.H + h)) * G.G + g) * PARTS + max(part, 0)) * 66;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          dst[j * 8 + 2 * t] = hi_half ? o[j][2] : o[j][0];
          dst[j * 8 + 2 * t + 1] = hi_half ? o[j][3] : o[j][1];
        }
        if (t == 0) { dst[64] = hi_half ? m1 : m0; dst[65] = hi_half ? l1 : l0; }
      }
    }
    if (part >= 0) continue;     // a CLS part: nothing else to store
    const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
    if (t == 0) {
      const int tok0 = row_token_x<RT>(G, g, rowA, sh), tok1 = row_token_x<RT>(G, g, rowB, sh);
      if (tok0 > 0) lse_out[((long long)(b * G.H + h)) * G.S + tok0] = m0 + logf(l0);
      if (tok1 > 0) lse_out[((long long)(b * G.H + h)) * G.S + tok1] = m1 + logf(l1);
    }
    if (TIME) store_frag_rows_bf16<RT>(o, i0, out, G.D, h * HD, G, b, g, r0, lane, i1, sh);   // no staging: 4 CTAs / SM
    else store_rows_bf16<RT>(o, i0, i1, stage, stage_gen, out, G.D, h * HD, G, b, g, r0, lane, /*skip_cls=*/true, sh);
  }
}

// ---- backward, phase 1 chunk: rows = queries (tile r0), pairs = keys.  dQ += (P o (dP - delta)) K
template <bool TIME, int NPR>
__device__ __forceinline__ void bwd_q_chunk(const FastCtx& c, const Smem& sm, const FragOff& fo, const Chunk& ch, int r0,
                                            int rowA, int rowB, int t, float ls0, float ls1, float de0, float de1,
                                            float (&dq)[8][4]) {
  float s[2 * NPR][4], dp[2 * NPR][4];
#pragma unroll
  for (int j = 0; j < 2 * NPR; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; dp[j][0] = dp[j][1] = dp[j][2] = dp[j][3] = 0.f; }
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t aq[4], ad[4];          // A fragments re-read per chunk: registers limit CTAs per SM here
    ldsm_x4(sm.q + r0 * ROW_BYTES + fo.a[kk], aq);
    ldsm_x4(sm.dout + r0 * ROW_BYTES + fo.a[kk], ad);
#pragma unroll
    for (int p = 0; p < NPR; ++p) {
      uint32_t bf[4];
      ldsm_x4(sm.k + ch.base[p] * ROW_BYTES + fo.b[kk], bf);
      mma_bf16(s[2 * p], aq, bf[0], bf[1]);
      mma_bf16(s[2 * p + 1], aq, bf[2], bf[3]);
      ldsm_x4(sm.v + ch.base[p] * ROW_BYTES + fo.b[kk], bf);
      mma_bf16(dp[2 * p], ad, bf[0], bf[1]);
      mma_bf16(dp[2 * p + 1], ad, bf[2], bf[3]);
    }
  }
  uint32_t dsf[NPR][4];
  const f32x2 sc = pk2(LOG2E, LOG2E), nl0 = pk2(-ls0, -ls0), nl1 = pk2(-ls1, -ls1);
  const f32x2 nd0 = pk2(-de0, -de0), nd1 = pk2(-de1, -de1);
#pragma unroll
  for (int p = 0; p < NPR; ++p) {
    const bool masked = ch.mask & (1u << p);
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const int j = 2 * p + jj, col = ch.base[p] + 8 * jj + 2 * t;
      if (masked) {               // exp2(-inf) = 0: masked entries drop out of P and dS
        if (TIME && ch.base[p] == c.NP && r0 < c.NP) {        // patch rows x the CLS pair: only column NP is a key
          const bool kc = jj == 0 && t == 0;
          s[j][0] = kc ? s[j][0] : -INFINITY; s[j][1] = -INFINITY;
          s[j][2] = kc ? s[j][2] : -INFINITY; s[j][3] = -INFINITY;
        } else if (TIME && r0 >= c.NP && ch.base[p] < c.NP) {   // CLS tile x patch keys: row NP sees the valid keys
          const bool cq = rowA == c.NP;
          s[j][0] = (cq && col < c.valid_keys) ? s[j][0] : -INFINITY;
          s[j][1] = (cq && col + 1 < c.valid_keys) ? s[j][1] : -INFINITY;
          s[j][2] = -INFINITY; s[j][3] = -INFINITY;
        } else {
          s[j][0] = fast_valid<TIME>(c, rowA, col) ? s[j][0] : -INFINITY;
          s[j][1] = fast_valid<TIME>(c, rowA, col + 1) ? s[j][1] : -INFINITY;
          s[j][2] = fast_valid<TIME>(c, rowB, col) ? s[j][2] : -INFINITY;
          s[j][3] = fast_valid<TIME>(c, rowB, col + 1) ? s[j][3] : -INFINITY;
        }
      }
      float e0, e1, e2, e3;
      up2(fma2(pk2(s[j][0], s[j][1]), sc, nl0), e0, e1);
      up2(fma2(pk2(s[j][2], s[j][3]), sc, nl1), e2, e3);
      float d0, d1, d2, d3;
      up2(mul2(pk2(exp2f(e0), exp2f(e1)), add2(pk2(dp[j][0], dp[j][1]), nd0)), d0, d1);
      up2(mul2(pk2(exp2f(e2), exp2f(e3)), add2(pk2(dp[j][2], dp[j][3]), nd1)), d2, d3);
      dsf[p][jj * 2] = pack_bf16x2(d0, d1);
      dsf[p][jj * 2 + 1] = pack_bf16x2(d2, d3);
    }
  }
#pragma unroll
  for (int p = 0; p < NPR; ++p) {
    const uint32_t kb = sm.k + ch.base[p] * ROW_BYTES;
#pragma unroll
    for (int dpi = 0; dpi < 4; ++dpi) {
      uint32_t bf[4];
      ldsm_x4_t(kb + fo.a[dpi], bf);
      mma_bf16(dq[2 * dpi], dsf[p], bf[0], bf[1]);
      mma_bf16(dq[2 * dpi + 1], dsf[p], bf[2], bf[3]);
    }
  }
}

// ---- backward, phase 2 chunk: rows = keys (tile k0r), pairs = queries.  dV += P^T dO, dK += dS^T Q
template <bool TIME, int NPR>
__device__ __forceinline__ void bwd_k_chunk(const FastCtx& c, const Smem& sm, const FragOff& fo, const Chunk& ch, int k0r,
                                            int keyA, int keyB, int t, float (&dk)[8][4], float (&dv)[8][4]) {
  float st[2 * NPR][4], dpt[2 * NPR][4];
#pragma unroll
  for (int j = 0; j < 2 * NPR; ++j) { st[j][0] = st[j][1] = st[j][2] = st[j][3] = 0.f; dpt[j][0] = dpt[j][1] = dpt[j][2] = dpt[j][3] = 0.f; }
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t ak[4], av[4];
    ldsm_x4(sm.k + k0r * ROW_BYTES + fo.a[kk], ak);
    ldsm_x4(sm.v + k0r * ROW_BYTES + fo.a[kk], av);
#pragma unroll
    for (int p = 0; p < NPR; ++p) {
      uint32_t bf[4];
      ldsm_x4(sm.q + ch.base[p] * ROW_BYTES + fo.b[kk], bf);
      mma_bf16(st[2 * p], ak, bf[0], bf[1]);
      mma_bf16(st[2 * p + 1], ak, bf[2], bf[3]);
      ldsm_x4(sm.dout + ch.base[p] * ROW_BYTES + fo.b[kk], bf);
      mma_bf16(dpt[2 * p], av, bf[0], bf[1]);
      mma_bf16(dpt[2 * p + 1], av, bf[2], bf[3]);
    }
  }
  uint32_t pf[NPR][4], dsf[NPR][4];
  const f32x2 sc = pk2(LOG2E, LOG2E);
#pragma unroll
  for (int p = 0; p < NPR; ++p) {
    const bool masked = ch.mask & (1u << p);
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const int j = 2 * p + jj, col = ch.base[p] + 8 * jj + 2 * t;       // query index
      if (masked) {
        if (TIME && ch.base[p] == c.NP && k0r < c.NP) {       // patch keys x the CLS pair: only the CLS query (column NP)
          const bool qc = jj == 0 && t == 0;
          st[j][0] = (qc && keyA < c.valid_keys) ? st[j][0] : -INFINITY; st[j][1] = -INFINITY;
          st[j][2] = (qc && keyB < c.valid_keys) ? st[j][2] : -INFINITY; st[j][3] = -INFINITY;
        } else if (TIME && k0r >= c.NP && ch.base[p] < c.NP) {   // CLS key tile x patch queries: every patch row sees key NP
          const bool ck = keyA == c.NP;
          st[j][0] = ck ? st[j][0] : -INFINITY; st[j][1] = ck ? st[j][1] : -INFINITY;
          st[j][2] = -INFINITY; st[j][3] = -INFINITY;
        } else {
          st[j][0] = fast_valid<TIME>(c, col, keyA) ? st[j][0] : -INFINITY;
          st[j][1] = fast_valid<TIME>(c, col + 1, keyA) ? st[j][1] : -INFINITY;
          st[j][2] = fast_valid<TIME>(c, col, keyB) ? st[j][2] : -INFINITY;
          st[j][3] = fast_valid<TIME>(c, col + 1, keyB) ? st[j][3] : -INFINITY;
        }
      }
      const float2 lq = *reinterpret_cast<const float2*>(sm.lse + col);
      const float2 dq2 = *reinterpret_cast<const float2*>(sm.delta + col);
      const f32x2 nl = pk2(-lq.x, -lq.y), nd = pk2(-dq2.x, -dq2.y);
      float e0, e1, e2, e3;
      up2(fma2(pk2(st[j][0], st[j][1]), sc, nl), e0, e1);
      up2(fma2(pk2(st[j][2], st[j][3]), sc, nl), e2, e3);
      const float p0 = exp2f(e0), p1 = exp2f(e1), p2 = exp2f(e2), p3 = exp2f(e3);
      pf[p][jj * 2] = pack_bf16x2(p0, p1);
      pf[p][jj * 2 + 1] = pack_bf16x2(p2, p3);
      float d0, d1, d2, d3;
      up2(mul2(pk2(p0, p1), add2(pk2(dpt[j][0], dpt[j][1]), nd)), d0, d1);
      up2(mul2(pk2(p2, p3), add2(pk2(dpt[j][2], dpt[j][3]), nd)), d2, d3);
      dsf[p][jj * 2] = pack_bf16x2(d0, d1);
      dsf[p][jj * 2 + 1] = pack_bf16x2(d2, d3);
    }
  }
#pragma unroll
  for (int p = 0; p < NPR; ++p) {
    const uint32_t qb = sm.q + ch.base[p] * ROW_BYTES, db = sm.dout + ch.base[p] * ROW_BYTES;
#pragma unroll
    for (int dpi = 0; dpi < 4; ++dpi) {
      uint32_t bf[4];
      ldsm_x4_t(db + fo.a[dpi], bf);
      mma_bf16(dv[2 * dpi], pf[p], bf[0], bf[1]);
      mma_bf16(dv[2 * dpi + 1], pf[p], bf[2], bf[3]);
      ldsm_x4_t(qb + fo.a[dpi], bf);
      mma_bf16(dk[2 * dpi], dsf[p], bf[0], bf[1]);
      mma_bf16(dk[2 * dpi + 1], dsf[p], bf[2], bf[3]);
    }
  }
}

template <bool TIME, int NWARPS, int MINB>
__global__ void __launch_bounds__(NWARPS * 32, MINB)
fast_attn_bwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                     const bf16* __restrict__ qkv, const bf16* __restrict__ out, const bf16* __restrict__ dout,
                     const float* __restrict__ lse_in, bf16* __restrict__ dqkv, float* __restrict__ dcls, float q_scale,
                     Geom G, int sh) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  int b, h, g;
  decode_block(G, b, h, g);
  Smem sm;
  load_group<true, false, false, false>(G, &tm_qkv, &tm_do, qkv, dout, b, h, g, smem_gen, smem_base, sm, NWARPS);
  constexpr int RT = TIME ? 2 : 1;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gq = lane >> 2, t = lane & 3;
  FastCtx c;
  c.NP = G.NP; c.NPAD = G.NPAD; c.sh = sh; c.first_group = (g == 0);
  c.valid_keys = TIME ? min(G.PG, G.N - g * G.PG) * G.T : G.NP;
  const FragOff fo = make_frag_off(lane);

  // phase 0: lse (log2 units) and delta = rowsum(dO * O) per row.  The rows of O and the lse values come straight
  // from global memory: their loads are issued BEFORE waiting for the TMA tiles so that both latencies overlap.
  constexpr int P0_ROWS = NWARPS * 4;                      // rows per pass (8 lanes x 16 B per row)
  constexpr int P0_MAX = (256 + P0_ROWS - 1) / P0_ROWS;    // NPAD <= 256
  constexpr int P0_N = TIME ? 128 / P0_ROWS : P0_MAX;
  uint4 o_pre[P0_N];
  float l_pre[P0_N];
  int t_pre[P0_N];
#pragma unroll
  for (int i = 0; i < P0_N; ++i) {
    const int r = warp * 4 + (lane >> 3) + i * P0_ROWS;
    const int tok = r < G.NPAD ? row_token_x<RT>(G, g, r, sh) : -1;
    t_pre[i] = tok;
    // unconditional loads from a clamped row, nothing computed on the values here: a select or a multiply at this point
    // makes the in-order issue wait for each load before the next one goes out (8 serialised DRAM latencies per CTA --
    // 28 % of this kernel's stall samples); validity is applied where the values are used
    const int tc = max(tok, 0);
    o_pre[i] = __ldg(reinterpret_cast<const uint4*>(out + ((long long)b * G.S + tc) * G.D + h * HD + (lane & 7) * 8));
    l_pre[i] = __ldg(lse_in + ((long long)(b * G.H + h)) * G.S + tc);
  }
  mbar_wait(sm.bar, 0);
#pragma unroll
  for (int i = 0; i < P0_N; ++i) {
    const int r = warp * 4 + (lane >> 3) + i * P0_ROWS;
    if (r >= G.NPAD) break;
    const int tok = t_pre[i], cc = lane & 7;
    float d = 0.f;
    if (tok >= 0) {
      const uint4 ov = o_pre[i];
      const uint4 dv = *reinterpret_cast<const uint4*>(smem_gen + (sw_addr(sm.dout, r, cc) - smem_base));
      const uint32_t ou[4] = {ov.x, ov.y, ov.z, ov.w}, du[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 a = unpack_bf16x2(ou[i]), bb = unpack_bf16x2(du[i]);
        d += a.x * bb.x + a.y * bb.y;
      }
    }
    d += __shfl_xor_sync(0xffffffffu, d, 1); d += __shfl_xor_sync(0xffffffffu, d, 2); d += __shfl_xor_sync(0xffffffffu, d, 4);
    if (cc == 0) {
      sm.delta[r] = d;
      sm.lse[r] = tok >= 0 ? l_pre[i] * LOG2E : 0.f;
    }
  }
  __syncthreads();

  // phase 1: per 16 query rows -> dQ
  for (int it = warp;; it += NWARPS) {
    int r0, part;
    if (!work_item<TIME, NWARPS>(c, it, r0, part)) break;
    const int rowA = r0 + gq, rowB = rowA + 8;
    const float ls0 = sm.lse[rowA], ls1 = sm.lse[rowB], de0 = sm.delta[rowA], de1 = sm.delta[rowB];
    float dq[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f; }
    Chunk ch;
#pragma unroll 1
    for (int ci = 0; get_chunk<TIME, NWARPS, 2>(c, G.T, r0, part, ci, ch); ++ci) {
      if (ch.np == 2) bwd_q_chunk<TIME, 2>(c, sm, fo, ch, r0, rowA, rowB, t, ls0, ls1, de0, de1, dq);
      else bwd_q_chunk<TIME, 1>(c, sm, fo, ch, r0, rowA, rowB, t, ls0, ls1, de0, de1, dq);
    }
    {
      const int rc = c.NP - r0;
      if (rc >= 0 && rc < 16 && (rc & 7) == gq) {
        const bool hi_half = rc >= 8;
        float* dst = dcls + ((long long)(b * G.H + h) * 3 + 0) * HD;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          atomicAdd(dst + j * 8 + 2 * t, hi_half ? dq[j][2] : dq[j][0]);
          atomicAdd(dst + j * 8 + 2 * t + 1, hi_half ? dq[j][3] : dq[j][1]);
        }
      }
    }
    if (part < 0) store_frag_rows_bf16<RT>(dq, q_scale, dqkv, 3 * G.D, h * HD, G, b, g, r0, lane, -1.f, sh);
  }

  // phase 2: per 16 keys -> dK, dV   (tile rows = keys, pairs = queries)
  for (int it = warp;; it += NWARPS) {
    int k0r, part;
    if (!work_item<TIME, NWARPS>(c, it, k0r, part)) break;
    const int keyA = k0r + gq, keyB = keyA + 8;
    float dk[8][4], dv[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = 0.f; dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f; }
    Chunk ch;
#pragma unroll 1
    for (int ci = 0; get_chunk<TIME, NWARPS, 2>(c, G.T, k0r, part, ci, ch); ++ci) {
      if (ch.np == 2) bwd_k_chunk<TIME, 2>(c, sm, fo, ch, k0r, keyA, keyB, t, dk, dv);
      else bwd_k_chunk<TIME, 1>(c, sm, fo, ch, k0r, keyA, keyB, t, dk, dv);
    }
    {
      const int rc = c.NP - k0r;
      if (rc >= 0 && rc < 16 && (rc & 7) == gq) {
        const bool hi_half = rc >= 8;
        float* dstk = dcls + ((long long)(b * G.H + h) * 3 + 1) * HD;
        float* dstv = dcls + ((long long)(b * G.H + h) * 3 + 2) * HD;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          atomicAdd(dstk + j * 8 + 2 * t, hi_half ? dk[j][2] : dk[j][0]);
          atomicAdd(dstk + j * 8 + 2 * t + 1, hi_half ? dk[j][3] : dk[j][1]);
          atomicAdd(dstv + j * 8 + 2 * t, hi_half ? dv[j][2] : dv[j][0]);
          atomicAdd(dstv + j * 8 + 2 * t + 1, hi_half ? dv[j][3] : dv[j][1]);
        }
      }
    }
    if (part < 0) {
      store_frag_rows_bf16<RT>(dk, 1.f, dqkv, 3 * G.D, G.D + h * HD, G, b, g, k0r, lane, -1.f, sh);
      store_frag_rows_bf16<RT>(dv, 1.f, dqkv, 3 * G.D, 2 * G.D + h * HD, G, b, g, k0r, lane, -1.f, sh);
    }
  }
}

// EGOVLP_ATTN_GENERIC=1 routes every geometry through the generic group-id kernels (used by the tests to check
// both implementations against the oracle)
inline bool force_generic() {
  const char* e = getenv("EGOVLP_ATTN_GENERIC");
  return e && e[0] == '1';
}
// time-mode fast path: T in {4, 8, 16} with full 112-row groups
inline bool time_fast_ok(const Geom& G) { return G.mode == 0 && (G.T == 4 || G.T == 8 || G.T == 16) && G.NP == 112; }
inline int time_shift(const Geom& G) { return G.T == 16 ? 4 : G.T == 8 ? 3 : 2; }

int make_geom(Geom& G, int B, int T, int N, int H, int mode) {
  G.B = B; G.H = H; G.T = T; G.N = N; G.S = 1 + T * N; G.D = H * HD; G.mode = mode;
  if (mode == 1) {
    G.PG = N; G.G = T; G.NP = N; G.gsize = N;
  } else {
    G.PG = (T <= 16 && 16 % T == 0) ? min(N, 112 / T) : min(N, 127 / T);   // 112-row groups keep the CLS row tile-aligned
    if (G.PG < 1) return EGOVLP_ERR_UNSUPPORTED;
    G.G = (N + G.PG - 1) / G.PG; G.NP = G.PG * T; G.gsize = T;
  }
  G.NPAD = (G.NP + 1 + 15) / 16 * 16;
  if (G.NPAD > 256 || (mode == 1 ? N : max(T, G.PG)) > 256) return EGOVLP_ERR_UNSUPPORTED;
  return EGOVLP_OK;
}

// 5-D gather map over a [B*S, ncolblk*64] bf16 matrix: dims (d, f, n, colblk, b), CLS row skipped via the base.
int make_group_tmap(CUtensorMap* tm, const void* base, const Geom& G, int ncolblk) {
  const uint64_t W = (uint64_t)ncolblk * HD;
  const uint64_t dims[5] = {HD, (uint64_t)G.T, (uint64_t)G.N, (uint64_t)ncolblk, (uint64_t)G.B};
  const uint64_t strides[5] = {1, (uint64_t)G.N * W, W, HD, (uint64_t)G.S * W};
  const uint32_t box[5] = {HD, (uint32_t)(G.mode == 1 ? 1 : G.T), (uint32_t)(G.mode == 1 ? G.N : G.PG), 1, 1};
  return make_tmap_nd_bf16(tm, reinterpret_cast<const bf16*>(base) + W, 5, dims, strides, box, true);
}

size_t attn_smem_bytes(const Geom& G, bool bwd, int nwarps, bool staging = true) {
  return (size_t)(bwd ? 4 : 3) * G.NPAD * ROW_BYTES + ((bwd || !staging) ? 0 : nwarps * 16 * ROW_BYTES) + 2 * G.NPAD * 4 +
         ((G.NPAD * 2 + 15) / 16) * 16 + 16 + 1024;
}


}  // namespace
}  // namespace egovlp

using namespace egovlp;

extern "C" long long egovlp_divided_attn_workspace_floats(int B, int T, int N, int H, int mode) {
  Geom G;
  if (make_geom(G, B, T, N, H, mode)) return -1;
  return (long long)B * H * G.G * 4 * 66;    // up to 4 CLS-row partials per group
}

extern "C" int egovlp_divided_attn_fwd(const void* qkv, void* out, float* lse, float* cls_part, int B, int T, int N,
                                       int H, int mode, void* stream) {
  EGOVLP_CHECK_ARG(qkv && out && lse && cls_part, "divided_attn_fwd: null pointer");
  EGOVLP_CHECK_ARG(B > 0 && T > 0 && N > 0 && H > 0 && (mode == 0 || mode == 1), "divided_attn_fwd: bad shape");
  Geom G;
  if (make_geom(G, B, T, N, H, mode)) { set_last_error("divided_attn: unsupported geometry T=%d N=%d", T, N); return EGOVLP_ERR_UNSUPPORTED; }
  CUtensorMap tm;
  int rc = make_group_tmap(&tm, qkv, G, 3 * H);
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bf16* q = reinterpret_cast<const bf16*>(qkv);
  bf16* o = reinterpret_cast<bf16*>(out);
  const int grid = B * H * G.G;
#define LAUNCH_FWD(KERN, W, ...)                                                                              \
  do {                                                                                                        \
    const size_t smem = attn_smem_bytes(G, false, W, generic || mode == 1);                                   \
    EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(KERN, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
    KERN<<<grid, W * 32, smem, st>>>(tm, q, o, lse, cls_part, G, ##__VA_ARGS__);                              \
  } while (0)
  const bool generic = force_generic() || (mode == 0 && !time_fast_ok(G));
  if (!generic && mode == 1 && space_attn_wgmma_supported(N)) {
    rc = space_attn_fwd_wgmma(qkv, out, lse, cls_part, B, T, N, H, st);
    if (rc) return rc;
  } else if (generic) {
    if (G.NPAD > 128) LAUNCH_FWD((divided_attn_fwd_kernel<7, 2>), 7);
    else LAUNCH_FWD((divided_attn_fwd_kernel<4, 3>), 4);
  } else if (mode == 1) {     // space: 13 row tiles over 7 warps, 2 CTAs / SM at 196 patches
    if (G.NPAD > 128) LAUNCH_FWD((fast_attn_fwd_kernel<false, 7, 2>), 7, 0);
    else LAUNCH_FWD((fast_attn_fwd_kernel<false, 4, 3>), 4, 0);
  } else {                    // time: 7 patch tiles + 4 CLS parts over 4 warps, 4 CTAs / SM (no staging)
    LAUNCH_FWD((fast_attn_fwd_kernel<true, 4, 4>), 4, time_shift(G));
  }
#undef LAUNCH_FWD
  EGOVLP_CHECK_LAUNCH();
  const int BH = B * H;
  const int parts = (!generic && mode == 0) ? 4 : 1;      // fast time kernel: CLS row split over its 4 warps
  cls_merge_kernel<<<(BH + 3) / 4, 128, 0, st>>>(cls_part, o, lse, BH, H, G.G * parts, G.S, G.D);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

extern "C" int egovlp_divided_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse,
                                       void* dqkv, float* dcls_ws, int B, int T, int N, int H, int mode,
                                       float q_scale, void* stream) {
  EGOVLP_CHECK_ARG(qkv && out && dout && lse && dqkv && dcls_ws, "divided_attn_bwd: null pointer");
  EGOVLP_CHECK_ARG(B > 0 && T > 0 && N > 0 && H > 0 && (mode == 0 || mode == 1), "divided_attn_bwd: bad shape");
  Geom G;
  if (make_geom(G, B, T, N, H, mode)) { set_last_error("divided_attn: unsupported geometry T=%d N=%d", T, N); return EGOVLP_ERR_UNSUPPORTED; }
  CUtensorMap tmq, tmd;
  int rc = make_group_tmap(&tmq, qkv, G, 3 * H);
  if (rc) return rc;
  rc = make_group_tmap(&tmd, dout, G, H);
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  EGOVLP_CHECK_CUDA(cudaMemsetAsync(dcls_ws, 0, (size_t)B * H * 3 * HD * sizeof(float), st));
  const bf16* q = reinterpret_cast<const bf16*>(qkv);
  const bf16* o = reinterpret_cast<const bf16*>(out);
  const bf16* d_o = reinterpret_cast<const bf16*>(dout);
  bf16* dq = reinterpret_cast<bf16*>(dqkv);
  const int grid = B * H * G.G;
#define LAUNCH_BWD(KERN, W, ...)                                                                              \
  do {                                                                                                        \
    const size_t smem = attn_smem_bytes(G, true, W);                                                          \
    EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(KERN, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
    KERN<<<grid, W * 32, smem, st>>>(tmq, tmd, q, o, d_o, lse, dq, dcls_ws, q_scale, G, ##__VA_ARGS__);       \
  } while (0)
  const bool generic = force_generic() || (mode == 0 && !time_fast_ok(G));
  if (generic) {
    if (G.NPAD > 128) LAUNCH_BWD((divided_attn_bwd_kernel<7, 2>), 7);
    else LAUNCH_BWD((divided_attn_bwd_kernel<4, 3>), 4);
  } else if (mode == 1) {     // space: 2 CTAs / SM (4 x 26 KB tiles each, no staging)
    if (G.NPAD > 128) LAUNCH_BWD((fast_attn_bwd_kernel<false, 7, 2>), 7, 0);
    else LAUNCH_BWD((fast_attn_bwd_kernel<false, 4, 3>), 4, 0);
  } else {
    const char* we = getenv("EGOVLP_ATTN_TIME_BWD_WARPS");
    const bool w8 = we && we[0] == '8';
    if (w8) LAUNCH_BWD((fast_attn_bwd_kernel<true, 8, 2>), 8, time_shift(G));
    else LAUNCH_BWD((fast_attn_bwd_kernel<true, 4, 3>), 4, time_shift(G));
  }
#undef LAUNCH_BWD
  EGOVLP_CHECK_LAUNCH();
  const int n = B * H * 3 * HD;
  cls_grad_finalize_kernel<<<(n + 255) / 256, 256, 0, st>>>(dcls_ws, reinterpret_cast<bf16*>(dqkv), B, H, G.S, G.D, q_scale);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
