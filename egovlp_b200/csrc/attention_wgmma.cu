// Space attention forward on wgmma (the N-length attention of VarAttention, model/video_transformer.py:109-133 in
// '(b f) n d' mode).  Same inputs / outputs / CLS semantics as the mma.sync span kernels in attention.cu.
//
// One CTA per (b, head, frame) group, two math warpgroups.  Q (patch rows + the CLS row at row N, padded to 256 rows),
// K and V (N + 1 keys padded to 208 rows) arrive by TMA into 128B-swizzled tiles.  Per 64-row query tile a warpgroup
// issues S[64 x 208] = Q K^T (wgmma, both operands from smem), runs the softmax on the accumulator fragment (each row
// lives in the 4 lanes of a quad), keeps P = exp(S - max) as bf16 in registers, where it already has the layout of the
// wgmma A fragment, and issues O[64 x 64] = P V with A from registers and V read as an MN-major B operand.  Padding
// rows and keys are zero-filled and never stored.  Opt-in (EGOVLP_ATTN_TC=1); the default is the mma.sync kernel.
#include <stdlib.h>

#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {
namespace {

constexpr int HD = 64;
constexpr int ROWB = 128;                 // bytes per head row
constexpr int QROWS = 256;                // 4 query tiles of 64 rows
constexpr int KROWS = 208;                // keys padded to the wgmma N of S
constexpr int Q_BYTES = QROWS * ROWB, KV_BYTES = KROWS * ROWB;
constexpr int SMEM_BYTES = Q_BYTES + 2 * KV_BYTES + 1024 /*align*/ + 64 /*barrier*/;
constexpr float LOG2E = 1.4426950408889634f;

struct SpaceGeom {
  int H, T, N, S, D;
};

__device__ __forceinline__ void wgmma_m64n208k16_ss(float (&d)[104], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %106, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n208k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
      "%96,%97,%98,%99,%100,%101,%102,%103}, "
      "%104, %105, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// A from registers (the m16n8k16 A-fragment layout per warp), B = V read MN-major (transpose bit set)
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                  uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(scale_d));
}

__global__ void __launch_bounds__(256, 1)
space_attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tm_rows, const __grid_constant__ CUtensorMap tm_cls,
                            bf16* __restrict__ out, float* __restrict__ lse_out, float* __restrict__ cls_part, SpaceGeom G) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t sQ = base, sK = base + Q_BYTES, sV = sK + KV_BYTES, bar = sV + KV_BYTES;
  const int g = blockIdx.x;
  const int f = g % G.T, h = (g / G.T) % G.H, b = g / (G.T * G.H);
  const int NK = G.N + 1;

  // padding rows must be finite (zero) for the MMAs; TMA writes only the N + 1 real rows of each tile
  for (int i = threadIdx.x; i < (Q_BYTES + 2 * KV_BYTES) / 16; i += blockDim.x)
    *reinterpret_cast<uint4*>(gen + 16 * i) = make_uint4(0, 0, 0, 0);
  fence_proxy_async_smem();
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, 3u * (uint32_t)NK * ROWB);
#pragma unroll
    for (int w = 0; w < 3; ++w) {
      const uint32_t dst = w == 0 ? sQ : (w == 1 ? sK : sV);
      tma_load_4d(dst, &tm_rows, bar, 0, 1 + f * G.N, w * G.H + h, b);
      tma_load_4d(dst + G.N * ROWB, &tm_cls, bar, 0, 0, w * G.H + h, b);
    }
  }
  mbar_wait_nocall(bar, 0);

  const int wg = threadIdx.x >> 7, wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int gq = lane >> 2, c = lane & 3;
  for (int t = wg; t < QROWS / 64; t += 2) {
    if (t * 64 > G.N) break;                       // the tile holds no patch row and not the CLS row
    // ---- S = Q K^T for 64 query rows
    float s[KROWS / 2];
    wgmma_fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
      wgmma_m64n208k16_ss(s, make_smem_desc_sw128(sQ + t * 64 * ROWB + kk * 32, 16, 1024),
                          make_smem_desc_sw128(sK + kk * 32, 16, 1024), kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    // ---- softmax on the fragment: rows r0 (h2 = 0) and r0 + 8 (h2 = 1), columns 8 j + 2 c + {0, 1}
    const int r0 = t * 64 + wq * 16 + gq;
    float mx[2], sum[2];
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      // the CLS key (column N) is visible to every patch query, and to the CLS query in the first frame only
      const int vis = (r0 + 8 * h2 == G.N && f != 0) ? G.N : NK;
      float m = -INFINITY;
#pragma unroll
      for (int j = 0; j < KROWS / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = s[4 * j + 2 * h2 + e];
          if (8 * j + 2 * c + e >= vis) v = -INFINITY;
          m = fmaxf(m, v);
        }
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
      mx[h2] = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    }
    uint32_t p[KROWS / 4];
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      const float nms = -mx[h2] * LOG2E;
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < KROWS / 8; ++j) {
        const float e0 = exp2f(fmaf(s[4 * j + 2 * h2], LOG2E, nms));     // masked entries: exp2(-inf) = 0
        const float e1 = exp2f(fmaf(s[4 * j + 2 * h2 + 1], LOG2E, nms));
        acc += e0 + e1;
        p[2 * j + h2] = pack_bf16x2(e0, e1);
      }
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      sum[h2] = acc + __shfl_xor_sync(0xffffffffu, acc, 2);
    }
    // ---- O = P V: k-chunk kk of P is column groups 2 kk, 2 kk + 1 = registers p[4 kk .. 4 kk + 3]
    float o[HD / 2];
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KROWS / 16; ++kk)
      wgmma_m64n64k16_rs(o, p[4 * kk], p[4 * kk + 1], p[4 * kk + 2], p[4 * kk + 3],
                         make_smem_desc_sw128(sV + kk * 16 * ROWB, 8192, 1024), kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      const int row = r0 + 8 * h2;
      if (row < G.N) {
        const float inv = 1.f / sum[h2];
        const long long tok = (long long)b * G.S + 1 + f * G.N + row;
        bf16* dst = out + tok * G.D + h * HD + 2 * c;
#pragma unroll
        for (int j = 0; j < HD / 8; ++j)
          *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(o[4 * j + 2 * h2] * inv, o[4 * j + 2 * h2 + 1] * inv);
        if (c == 0) lse_out[((long long)(b * G.H + h)) * G.S + 1 + f * G.N + row] = mx[h2] + logf(sum[h2]);
      } else if (row == G.N) {                       // CLS query: its (acc, max, sum) partial for the merge kernel
        float* dst = cls_part + (((long long)(b * G.H + h)) * G.T + f) * 66;
#pragma unroll
        for (int j = 0; j < HD / 8; ++j) {
          dst[8 * j + 2 * c] = o[4 * j + 2 * h2];
          dst[8 * j + 2 * c + 1] = o[4 * j + 2 * h2 + 1];
        }
        if (c == 0) { dst[64] = mx[h2]; dst[65] = sum[h2]; }
      }
    }
  }
}

}  // namespace

// geometry the kernel covers: N + 1 keys in 129 .. 208 (N = 196 at 224^2 / p16); opt-in through EGOVLP_ATTN_TC=1
bool space_attn_wgmma_supported(int N) {
  const char* e = getenv("EGOVLP_ATTN_TC");
  if (!(e && e[0] == '1')) return false;
  return N + 1 > 128 && N + 1 <= KROWS;
}

int space_attn_fwd_wgmma(const void* qkv, void* out, float* lse, float* cls_part, int B, int T, int N, int H,
                         cudaStream_t st) {
  SpaceGeom G;
  G.H = H; G.T = T; G.N = N; G.S = 1 + T * N; G.D = H * HD;
  const uint64_t W = 3ull * G.D;
  const uint64_t dims[4] = {HD, (uint64_t)G.S, (uint64_t)(3 * H), (uint64_t)B};
  const uint64_t strides[4] = {1, W, HD, (uint64_t)G.S * W};
  const uint32_t box_rows[4] = {HD, (uint32_t)N, 1, 1};
  const uint32_t box_cls[4] = {HD, 1, 1, 1};
  CUtensorMap tm_rows, tm_cls;
  int rc = make_tmap_nd_bf16(&tm_rows, qkv, 4, dims, strides, box_rows, true);
  if (rc) return rc;
  rc = make_tmap_nd_bf16(&tm_cls, qkv, 4, dims, strides, box_cls, true);
  if (rc) return rc;
  static bool attr = false;
  if (!attr) {
    EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(space_attn_fwd_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           SMEM_BYTES));
    attr = true;
  }
  space_attn_fwd_wgmma_kernel<<<B * H * T, 256, SMEM_BYTES, st>>>(tm_rows, tm_cls, reinterpret_cast<bf16*>(out), lse,
                                                                   cls_part, G);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

}  // namespace egovlp
