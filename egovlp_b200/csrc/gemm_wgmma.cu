// Persistent warp-specialised bf16 GEMM on wgmma (sm_90a), operands staged by TMA (128B swizzle).
//
//   D[m,n] = epilogue( sum_k A[m,k] * B[n,k] )
//
// Replaces every nn.Linear / einsum-free contraction the reference reaches through cuBLAS sgemm:
//   qkv / proj  (model/video_transformer.py:88-89,103,135), Mlp.fc1/fc2 (:41-52), patch-embed conv-as-GEMM
//   (:70,76), DistilBERT q/k/v/out_lin + ffn (transformers modeling_distilbert.py), projections
//   (model/model.py:72-79) and all their backward dgrad / wgrad contractions (autograd in the reference).
//
// Layout: A and B are bf16 in HBM.  "K-major" = the contraction index is contiguous (x[M,K], W[N,K]);
// "MN-major" = the m/n index is contiguous (stored [K, M] / [K, N]) which is what dgrad (W as B) and wgrad
// (dy and x as A and B, contraction over tokens) need -- no transposed copies are ever materialised: wgmma reads
// MN-major tiles with its transpose bit.
// One CTA per SM, 128 x BLOCK_N output tile (BLOCK_N = 256 when N % 256 == 0, else 128), 64-deep k-blocks, a 4-stage
// (BLOCK_N = 256, 48 KB a stage) or 6-stage (BLOCK_N = 128) TMA -> smem ring, fp32 accumulators in registers.
// TWO = CTA pair: a cluster of 2 CTAs computes a 256 x BLOCK_N tile; each CTA loads its own 128 rows of A and HALF of
// the B tile, which TMA multicasts into both CTAs, so every B byte fetched from L2 feeds two SMs.  A stage is refilled
// only once the math warpgroups of BOTH CTAs have released it (they arrive on the empty barriers of both).
// Warp roles: warpgroup 0 = control (warp 0 lane 0 issues the TMA loads; warp 1 lane 0 loads the epilogue's inputs in
// the specialised forms; warps 2 and 3 sum the A tiles' columns in the wgrad form), warpgroups 1 and 2 = math: each
// issues m64 x BLOCK_N x k16 wgmmas for its 64 rows of the tile and then runs the epilogue on its own accumulators,
// while the producer already streams the next tile's k-blocks into the stages the math warpgroups have released.
// setmaxnreg gives the control warpgroup 40 registers and the math warpgroups 232 (BLOCK_N = 256 keeps 128 fp32
// accumulators per thread).
// The step's hot forms get compile-time specialised epilogues (EpiMode); the host picks the mode from the epilogue
// descriptor, everything else takes the generic epilogue (same arithmetic, same order: bit-identical results).  The
// specialised epilogues move their HBM bytes by TMA: the bias row and the residual / aux subtiles arrive in shared
// memory while the tile's k-blocks run, and the results leave through 128B-swizzled staging subtiles as TMA stores that
// drain while the math warpgroups already run the next tile.  The split-K weight gradients leave the same way: each
// unit's fp32 partial tile is added into dW by TMA reduce.  The generic epilogue loads and stores from registers.
// The same kernel with FP8 = true is the e4m3 inference form (egovlp_gemm_e4m3): e4m3 operands with per-row scales of
// A and per-column scales of B, applied in the staged epilogue.
// gemm_drop_wgmma_kernel runs the same body with the video tower's training dropouts in five of the staged epilogues
// (EPI_*_DROP): the Philox keep mask and the per-sample drop-path factor are applied while the tile is in registers.
#include <stdlib.h>

#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int WG_K = 16;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;
constexpr int MN_ATOM_BYTES = BLOCK_K * 128;  // one 64(mn) x BLOCK_K(k) MN-major slab
constexpr int NUM_THREADS = 384;              // control warpgroup + 2 math warpgroups

struct EpiParams {
  const float* bias;
  const float* residual;
  const bf16* aux;
  void* out;
  bf16* out2;
  long long ldr, ldaux, ldo, ldo2;
  int out_mode;  // 0 bf16 store, 1 fp32 store, 2 fp32 atomic add
  int act;       // 0 none, 1 gelu(erf), 2 multiply by gelu'(aux), 3 gelu(erf) with out2 = gelu', 4 multiply by aux,
                 // 5 multiply by gelu'(aux) with out2 = gelu(aux)
  float alpha;
  float col_scale;
  int col_scale_ncols;
  int res_row_mod;  // 0: residual row = m; else residual row = m % res_row_mod (broadcast table)
  float* colsum;    // optional fp32 [N]: accumulates the column sums of the stored values (bias gradient)
  float* colsum_a;  // optional fp32 [M], MN-major A / MN-major B (wgrad) only: accumulates sum_k A[k, m], i.e. the bias
                    // gradient of the Linear whose weight gradient this GEMM computes, from the A tiles already in smem
  // e4m3 operands only: acc[m, n] * row_scale[m] * w_scale[n] is the product, before the epilogue above
  const float* row_scale;
  const float* w_scale;
  // deterministic form (out_mode 2 and / or colsum_a): each unit stores its fp32 partial tile to det_ws [splits][Mp][N]
  // (Mp = M rounded up to the 128-row tile) and its colsum_a partial to det_cs [splits][n-blocks][Mp]; gemm_det_merge_*
  // then add them into out / colsum_a in split (and n-block) order
  float* det_ws;
  float* det_cs;
};

// The dropout forms (EPI_*_DROP) only, a kernel parameter of their own: element (m, n) of the [M, N] output is kept iff
// word n & 3 of philox4x32_10(dropout_key(seed, site), m * (N / 4) + n / 4) >= dropout_threshold(p), and scaled by
// 1 / (1 - p) x drop_path_factor(seed, path_site, path_p, m / path_rows) (path_rows = 0: no drop-path)
struct DropParams {
  unsigned long long seed;
  float p, path_p;
  uint32_t site, path_site;
  int path_rows;
};

// Specialised epilogues stage through shared memory: each math warpgroup owns EPI_BUFS subtiles of 64 rows x 128 B
// (64 bf16 or 32 fp32 columns, 128B-swizzled like the operand tiles), which TMA fills with the residual / aux and
// drains to the outputs; plus one fp32 bias row of the tile, shared by both warpgroups.
constexpr int EPI_ROWS = 64;
constexpr int EPI_SUB_BYTES = EPI_ROWS * 128;
constexpr int EPI_BUFS = 2;
constexpr int EPI_BIAS_BYTES = 256 * 4;
constexpr int EPI_SMEM_BYTES = 2 * EPI_BUFS * EPI_SUB_BYTES + EPI_BIAS_BYTES;

template <int BLOCK_N>
struct Cfg {
  static constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGES = BLOCK_N == 256 ? 4 : 6;
  static constexpr int ACC = BLOCK_N / 2;     // fp32 accumulators per math thread (m64 x BLOCK_N over 128 threads)
  static constexpr int RING_BYTES = STAGES * (A_STAGE_BYTES + B_STAGE_BYTES);
  static constexpr int SMEM_BYTES = RING_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  static constexpr int SMEM_BYTES_STAGED = SMEM_BYTES + EPI_SMEM_BYTES;
  static_assert(SMEM_BYTES_STAGED <= 232448, "shared memory per block");
};

__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// wgmma accumulator operands: m64 x 256 (128 fp32 per thread) and m64 x 128 (64 per thread)
#define WGMMA_ACC128 \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
  "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
  "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
  "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
  "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
  "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
  "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
  "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), \
  "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), \
  "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), \
  "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), \
  "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), \
  "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), \
  "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), \
  "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), \
  "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
#define WGMMA_ACC64 \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
  "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
  "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
  "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
  "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
  "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
  "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
  "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define WGMMA_REGS128 \
  "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
  "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63," \
  "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95," \
  "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
#define WGMMA_REGS64 \
  "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
  "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"

// D (+)= A[smem desc] * B[smem desc], m64 x N x k16, bf16 -> fp32; TA / TB = 1 for an MN-major operand.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{" WGMMA_REGS128 "}, "
      "%128, %129, p, 1, 1, %131, %132;\n\t}"
      : WGMMA_ACC128
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{" WGMMA_REGS64 "}, "
      "%64, %65, p, 1, 1, %67, %68;\n\t}"
      : WGMMA_ACC64
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
}
// the same for e4m3 x e4m3 -> fp32, m64 x N x k32: K-major operands only (the instruction has no transpose bits); one
// k32 step reads 32 B of each operand row, as one bf16 k16 step does
__device__ __forceinline__ void wgmma_m64n256k32_e4m3(float (&d)[128], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k32.f32.e4m3.e4m3 "
      "{" WGMMA_REGS128 "}, "
      "%128, %129, p, 1, 1;\n\t}"
      : WGMMA_ACC128
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_m64n128k32_e4m3(float (&d)[64], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{" WGMMA_REGS64 "}, "
      "%64, %65, p, 1, 1;\n\t}"
      : WGMMA_ACC64
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <int BLOCK_N, int TA, int TB, bool FP8>
__device__ __forceinline__ void wgmma_tile(float (&d)[BLOCK_N / 2], uint64_t adesc, uint64_t bdesc, int scale_d) {
  if constexpr (FP8 && BLOCK_N == 256) wgmma_m64n256k32_e4m3(d, adesc, bdesc, scale_d);
  else if constexpr (FP8) wgmma_m64n128k32_e4m3(d, adesc, bdesc, scale_d);
  else if constexpr (BLOCK_N == 256) wgmma_m64n256k16<TA, TB>(d, adesc, bdesc, scale_d);
  else wgmma_m64n128k16<TA, TB>(d, adesc, bdesc, scale_d);
}

// GELU (exact-erf form) in the epilogue.  Phi(x) = 0.5 (1 + erf(x / sqrt2)) through Abramowitz-Stegun 7.1.26
// (|err| <= 1.5e-7 on erf).  With u = k x, k = sqrt(log2(e) / 2) (so that exp(-x^2 / 2) = 2^(-u^2)),
// t = 1 / (1 + p |x| / sqrt2) and e' = c exp(-x^2 / 2) = 2^(log2 c - u^2), c = 1 / (k sqrt(2 pi)):
//     r = 0.5 erf(|x| / sqrt2) = 0.5 + e' t (b1 + t (b2 + t (b3 + t (b4 + t b5))))      (b = -a / (2 c))
//     Phi(x) = 0.5 + copysign(r, x)       GELU = x Phi       GELU' = Phi + x phi = Phi + u e'
// Two MUFU operations (rcp, ex2) per element give GELU and GELU' together.
constexpr float GELU_K = 0.84932180028801907f;          // sqrt(log2(e) / 2)
constexpr float GELU_PT = 0.27273749f;                  // 0.3275911 / sqrt2 / GELU_K
constexpr float GELU_LOG2C = -1.0901312f;               // log2(c), c = 0.39894228 / GELU_K = 0.46971865
constexpr float GELU_B1 = -0.5f * 0.254829592f / 0.46971865f, GELU_B2 = 0.5f * 0.284496736f / 0.46971865f,
                GELU_B3 = -0.5f * 1.421413741f / 0.46971865f, GELU_B4 = 0.5f * 1.453152027f / 0.46971865f,
                GELU_B5 = -0.5f * 1.061405429f / 0.46971865f;
struct GeluConsts {       // paired constants, built once per thread
  f32x2 k, nk, l2c, b1, b2, b3, b4, b5, half;
  __device__ __forceinline__ GeluConsts()
      : k(pk2(GELU_K, GELU_K)), nk(pk2(-GELU_K, -GELU_K)), l2c(pk2(GELU_LOG2C, GELU_LOG2C)), b1(pk2(GELU_B1, GELU_B1)),
        b2(pk2(GELU_B2, GELU_B2)), b3(pk2(GELU_B3, GELU_B3)), b4(pk2(GELU_B4, GELU_B4)), b5(pk2(GELU_B5, GELU_B5)),
        half(pk2(0.5f, 0.5f)) {}
};
// two elements: Phi (returned), u = k x and e' for the derivative
__device__ __forceinline__ f32x2 gelu_phi2(const GeluConsts& gc, float x0, float x1, f32x2 x, f32x2& u, f32x2& e) {
  u = mul2(x, gc.k);
  float u0, u1, a0, a1, t0, t1, e0, e1, r0, r1;
  up2(u, u0, u1);
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t0) : "f"(fmaf(fabsf(u0), GELU_PT, 1.f)));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t1) : "f"(fmaf(fabsf(u1), GELU_PT, 1.f)));
  up2(fma2(mul2(x, gc.nk), u, gc.l2c), a0, a1);          // log2 c - u^2
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(a0));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(a1));
  const f32x2 t = pk2(t0, t1);
  e = pk2(e0, e1);
  f32x2 p = fma2(t, gc.b5, gc.b4);
  p = fma2(p, t, gc.b3);
  p = fma2(p, t, gc.b2);
  p = fma2(p, t, gc.b1);
  up2(fma2(mul2(p, t), e, gc.half), r0, r1);
  return add2(pk2(copysignf(r0, x0), copysignf(r1, x1)), gc.half);
}
__device__ __forceinline__ void gelu2(const GeluConsts& gc, float& x0, float& x1) {            // in place
  const f32x2 x = pk2(x0, x1);
  f32x2 u, e;
  up2(mul2(x, gelu_phi2(gc, x0, x1, x, u, e)), x0, x1);
}
// GELU(x) and GELU'(x) of two elements from ONE evaluation of Phi, in fp32
__device__ __forceinline__ void gelu_pair2(const GeluConsts& gc, float x0, float x1, float& g0, float& g1, float& d0,
                                           float& d1) {
  const f32x2 x = pk2(x0, x1);
  f32x2 u, e;
  const f32x2 phi = gelu_phi2(gc, x0, x1, x, u, e);
  up2(mul2(x, phi), g0, g1);
  up2(fma2(u, e, phi), d0, d1);
}
// the same, packed as bf16x2 (the fc1 epilogue stores the derivative for the backward instead of the pre-activation: the
// dgrad-fc2 epilogue then only multiplies, act = 4)
__device__ __forceinline__ void gelu_and_grad2(const GeluConsts& gc, float x0, float x1, uint32_t& g_bf, uint32_t& d_bf) {
  float g0, g1, d0, d1;
  gelu_pair2(gc, x0, x1, g0, g1, d0, d1);
  g_bf = pack_bf16x2(g0, g1);
  d_bf = pack_bf16x2(d0, d1);
}
// scalar form of the derivative for the act = 2 epilogue (recompute GELU' from the stored pre-activation)
__device__ __forceinline__ float gelu_grad_fast(float x) {     // Phi(x) + x phi(x)
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(fabsf(x), 0.3275911f * 0.70710678118654752f, 1.f)));
  const float e = exp2f(x * x * -0.72134752044448170f);            // exp(-x^2 / 2)
  float p = fmaf(t, 0.5f * 1.061405429f, 0.5f * -1.453152027f);
  p = fmaf(p, t, 0.5f * 1.421413741f);
  p = fmaf(p, t, 0.5f * -0.284496736f);
  p = fmaf(p, t, 0.5f * 0.254829592f);
  const float phi_cdf = 0.5f + copysignf(fmaf(-(p * t), e, 0.5f), x);
  return fmaf(x * 0.3989422804014327f, e, phi_cdf);
}

// MODE specialises the epilogue at compile time for the step's hot forms (the generic epilogue decides everything per
// element pair from runtime fields):
enum EpiMode {
  EPI_GENERIC = 0,   // everything EpiParams can express
  EPI_BF16 = 1,      // alpha, bias, optional column scale -> bf16                      (qkv, plain dgrad)
  EPI_ACT3 = 2,      // bias -> GELU -> bf16, GELU' -> bf16 out2                         (Mlp.fc1 forward)
  EPI_MUL_AUX = 3,   // x bf16 aux -> bf16                                               (Mlp.fc2 input gradient)
  EPI_RES_F32 = 4,   // bias + fp32 residual -> fp32                                     (proj / fc2 forward)
  EPI_ACT1 = 5,      // bias -> GELU -> bf16                                             (Mlp.fc1, inference)
  // the low-memory training pair: fc1 saves the bf16 pre-activation z, the fc2 input-gradient GEMM rebuilds GELU(z)
  EPI_ACT1_Z = 6,    // bias -> GELU -> bf16, pre-activation -> bf16 out2                (Mlp.fc1 forward)
  EPI_GELU_AUX = 7,  // x GELU'(bf16 aux) -> bf16, GELU(aux) -> bf16 out2                (Mlp.fc2 input gradient)
  // the weight gradients (MN-major A and B, split-K): each unit's fp32 partial tile is added into dW by TMA reduce
  EPI_RED_F32 = 8,   // alpha -> fp32 add into out                                      (every wgrad)
  // the video tower's training dropouts, applied while the tile is in registers: s = (kept ? 1 / (1 - p) : 0) x the
  // row's drop-path factor, from the Philox stream of DropParams (the mask does not depend on tiling or batch split)
  EPI_RES_F32_DROP = 9,    // s (acc + bias) + fp32 residual -> fp32                       (proj / fc2 forward)
  EPI_ACT3_DROP = 10,      // s GELU(v) -> bf16, GELU'(v) -> bf16 out2                     (Mlp.fc1 forward)
  EPI_ACT1_Z_DROP = 11,    // s GELU(v) -> bf16, pre-activation -> bf16 out2               (Mlp.fc1 forward, low memory)
  EPI_MUL_AUX_DROP = 12,   // s v aux -> bf16                                              (Mlp.fc2 input gradient)
  EPI_GELU_AUX_DROP = 13,  // s v GELU'(aux) -> bf16, s GELU(aux) -> bf16 out2             (the same, low memory)
};
// the form a dropout form applies its mask to
__host__ __device__ constexpr int base_mode(int mode) {
  return mode == EPI_RES_F32_DROP ? EPI_RES_F32 : mode == EPI_ACT3_DROP ? EPI_ACT3 : mode == EPI_ACT1_Z_DROP ? EPI_ACT1_Z
       : mode == EPI_MUL_AUX_DROP ? EPI_MUL_AUX : mode == EPI_GELU_AUX_DROP ? EPI_GELU_AUX : mode;
}

// FP8: A and B are e4m3 (K-major both), one k-block = 128 elements = the same 128 B per row as a bf16 k-block, so the
// TMA boxes, smem descriptors, stage ring and barriers are byte-identical; each k-block runs 4 k32 steps instead of 4
// k16 steps, and the staged epilogue first multiplies the accumulators by the row and column scales.
template <int BLOCK_N, bool A_MN, bool B_MN, bool TWO, int MODE, bool FP8>
__device__ __forceinline__ void
gemm_bf16_wgmma_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmOut, const CUtensorMap& tmOut2,
                     const CUtensorMap& tmIn, int M, int N, int K, int num_m_blocks, int num_n_blocks, int kb_per_split,
                     int num_splits, const EpiParams& ep, const DropParams& dp) {
  static_assert(!(TWO && A_MN && B_MN), "the wgrad form (column sums of A) runs on single CTAs");
  static_assert(!FP8 || (!A_MN && !B_MN && !TWO && (MODE == EPI_BF16 || MODE == EPI_ACT1)),
                "e4m3: K-major operands, single CTAs, the qkv / fc1 inference epilogues");
  constexpr int KB_ELEMS = FP8 ? 2 * BLOCK_K : BLOCK_K;      // elements of one 128-byte k-block row
  using C = Cfg<BLOCK_N>;
  constexpr int TILE_M = TWO ? 2 * BLOCK_M : BLOCK_M;
  const uint32_t rank = TWO ? cluster_ctarank() : 0u;      // CTA of the pair: rows 128 rank .. of the 256-row tile
  const int worker = TWO ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int num_workers = TWO ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  constexpr int STAGES = C::STAGES;
  // TMA-staged epilogue (the specialised forms): subtile width, subtiles per tile, which forms read an input subtile
  // (the residual or aux, transformed in place) and which write two outputs.  Without an input the two outputs fill both
  // buffers of the warpgroup; EPI_GELU_AUX has both, and stores its second output from the input's buffer once the
  // first output's store has read it, so that the other buffer stays free for the next aux subtile.
  constexpr bool STAGED = MODE != EPI_GENERIC;
  constexpr int BM = base_mode(MODE);            // a dropout form runs its base form's epilogue, plus the mask
  constexpr bool DROP = BM != MODE;
  constexpr bool RED = BM == EPI_RED_F32;        // no bias row and no input: warp 1 and the bias barriers stay idle
  constexpr bool OUT_F32 = BM == EPI_RES_F32 || RED;
  constexpr bool HAS_IN = BM == EPI_RES_F32 || BM == EPI_MUL_AUX || BM == EPI_GELU_AUX;
  constexpr bool TWO_OUT = BM == EPI_ACT3 || BM == EPI_ACT1_Z || BM == EPI_GELU_AUX;
  constexpr bool BOTH_BUFS = TWO_OUT && !HAS_IN;
  constexpr int SUB_COLS = OUT_F32 ? 32 : 64;
  constexpr int NSUB = BLOCK_N / SUB_COLS;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sA = smem_base;
  const uint32_t sB = smem_base + STAGES * A_STAGE_BYTES;
  const uint32_t sEpi = sB + STAGES * C::B_STAGE_BYTES;      // STAGED only: 2 warpgroups x EPI_BUFS subtiles
  const uint32_t sBias = sEpi + 2 * EPI_BUFS * EPI_SUB_BYTES;
  const uint32_t bars = STAGED ? sBias + EPI_BIAS_BYTES : sEpi;
  const uint32_t full_bar = bars;                    // STAGES x 8B
  const uint32_t empty_bar = bars + 8 * STAGES;      // STAGES x 8B
  // STAGED: input subtile landed / subtile buffer free again ([warpgroup][buffer]), bias row landed / consumed
  const uint32_t epi_full = bars + 16 * STAGES;
  const uint32_t epi_empty = epi_full + 8 * 2 * EPI_BUFS;
  const uint32_t bias_full = epi_empty + 8 * 2 * EPI_BUFS;
  const uint32_t bias_empty = bias_full + 8;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = num_m_blocks * num_n_blocks;
  const int num_units = num_tiles * num_splits;
  const int num_kb = (K + KB_ELEMS - 1) / KB_ELEMS;
  const bool sum_a = A_MN && B_MN && ep.colsum_a != nullptr;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      // a stage is released by both math warpgroups (of both CTAs of a pair) and, when the A tiles are column-summed, by
      // the two summing warps
      mbar_init(empty_bar + 8 * s, (TWO || sum_a) ? 4 : 2);
    }
    if (STAGED) {
      tma_prefetch_desc(&tmOut);
      if (TWO_OUT) tma_prefetch_desc(&tmOut2);
      if (HAS_IN) tma_prefetch_desc(&tmIn);
      for (int i = 0; i < 2 * EPI_BUFS; ++i) {
        mbar_init(epi_full + 8 * i, 1);
        mbar_init(epi_empty + 8 * i, 1);      // the storing thread of the warpgroup, once its store has read the buffer
      }
      mbar_init(bias_full, 1);
      mbar_init(bias_empty, 2);               // one arrive per math warpgroup
    }
    fence_mbar_init();
  }
  if (STAGED && !ep.bias && threadIdx.x < BLOCK_N)      // no bias: the row stays zero and is never loaded
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(sBias + 4 * threadIdx.x), "f"(0.f) : "memory");
  if (TWO) cluster_sync_all();      // the peer's barriers are initialised before any multicast or remote arrive
  else __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0) {
      // ===================== TMA producer =====================
      if (lane == 0) {
        int stage = 0;
        uint32_t phase = 0;
        for (int unit = worker; unit < num_units; unit += num_workers) {
          const int split = unit / num_tiles, tile = unit - split * num_tiles;
          const int m_blk = tile / num_n_blocks, n_blk = tile - m_blk * num_n_blocks;
          const int kb0 = split * kb_per_split, kb1 = min(num_kb, kb0 + kb_per_split);
          const int m_row = m_blk * TILE_M + (int)rank * BLOCK_M, n_row = n_blk * BLOCK_N;
          for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait_nocall(empty_bar + 8 * stage, phase ^ 1);
            const uint32_t fb = full_bar + 8 * stage;
            mbar_expect_tx(fb, A_STAGE_BYTES + C::B_STAGE_BYTES);
            const uint32_t a_dst = sA + stage * A_STAGE_BYTES, b_dst = sB + stage * C::B_STAGE_BYTES;
            if (!A_MN) {
              tma_load_2d(a_dst, &tmA, fb, kb * KB_ELEMS, m_row);
            } else {
#pragma unroll
              for (int i = 0; i < BLOCK_M / 64; ++i)
                tma_load_2d(a_dst + i * MN_ATOM_BYTES, &tmA, fb, m_row + i * 64, kb * BLOCK_K);
            }
            if (TWO) {          // this CTA's half of B, multicast into both CTAs of the pair
              if (!B_MN) {
                tma_load_2d_multicast(b_dst + rank * (BLOCK_N / 2) * 128, &tmB, fb, kb * BLOCK_K,
                                      n_row + (int)rank * (BLOCK_N / 2), 3);
              } else {
#pragma unroll
                for (int i = 0; i < BLOCK_N / 128; ++i) {
                  const int slab = (int)rank * (BLOCK_N / 128) + i;
                  tma_load_2d_multicast(b_dst + slab * MN_ATOM_BYTES, &tmB, fb, n_row + slab * 64, kb * BLOCK_K, 3);
                }
              }
            } else if (!B_MN) {
              tma_load_2d(b_dst, &tmB, fb, kb * KB_ELEMS, n_row);
            } else {
#pragma unroll
              for (int i = 0; i < BLOCK_N / 64; ++i)
                tma_load_2d(b_dst + i * MN_ATOM_BYTES, &tmB, fb, n_row + i * 64, kb * BLOCK_K);
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    } else if ((warp == 2 || warp == 3) && sum_a) {
      // ===================== column sums of A (wgrad only): bias gradient for free =====================
      // A stage holds A as two slabs [64 k-rows][64 m-columns] (128 B rows, 16-byte chunks XOR-swizzled by row & 7).
      // Warp 2 sums slab 0, warp 3 slab 1: lane = (row & 3 group, chunk); each lane keeps 8 fp32 column sums.  The
      // units of one (k-range, m-block) -- one per n-block, all staging the same A tiles -- share the work: unit n_blk
      // sums the k-blocks with kb % num_n_blocks == n_blk, so every A tile is summed exactly once across the grid.
      const int slab = warp - 2, chunk = lane & 7, rsub = lane >> 3;
      int stage = 0;
      uint32_t phase = 0;
      for (int unit = worker; unit < num_units; unit += num_workers) {
        const int split = unit / num_tiles, tile = unit - split * num_tiles;
        const int m_blk = tile / num_n_blocks, n_blk = tile - m_blk * num_n_blocks;
        const int kb0 = split * kb_per_split, kb1 = min(num_kb, kb0 + kb_per_split);
        // the deterministic form counts the k-blocks from the split's first, so that a split's partial is the same
        // as that of a one-split GEMM over the split's rows
        const int kb_share0 = ep.det_cs ? kb0 : 0;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait_nocall(full_bar + 8 * stage, phase);
          if ((kb - kb_share0) % num_n_blocks == n_blk) {     // this unit's share of the k-blocks
            const uint32_t slab_base = sA + stage * A_STAGE_BYTES + slab * MN_ATOM_BYTES;
#pragma unroll 4
            for (int i = 0; i < 16; ++i) {
              const int r = rsub + 4 * i;
              uint32_t v0, v1, v2, v3;
              asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                           : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3)
                           : "r"(slab_base + r * 128 + ((chunk ^ (r & 7)) << 4)));
              acc[0] += __uint_as_float(v0 << 16); acc[1] += __uint_as_float(v0 & 0xffff0000u);
              acc[2] += __uint_as_float(v1 << 16); acc[3] += __uint_as_float(v1 & 0xffff0000u);
              acc[4] += __uint_as_float(v2 << 16); acc[5] += __uint_as_float(v2 & 0xffff0000u);
              acc[6] += __uint_as_float(v3 << 16); acc[7] += __uint_as_float(v3 & 0xffff0000u);
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_bar + 8 * stage);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 8);
          acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 16);
        }
        const int col = m_blk * BLOCK_M + slab * 64 + chunk * 8;
        if (lane < 8 && col < M) {            // M % 8 == 0 is checked by the host
          if (ep.det_cs) {
            float* dst = ep.det_cs + ((long long)split * num_n_blocks + n_blk) * (num_m_blocks * BLOCK_M) + col;
            *reinterpret_cast<float4*>(dst) = make_float4(acc[0], acc[1], acc[2], acc[3]);
            *reinterpret_cast<float4*>(dst + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
          } else {
            red_add_v4(ep.colsum_a + col, acc[0], acc[1], acc[2], acc[3]);
            red_add_v4(ep.colsum_a + col + 4, acc[4], acc[5], acc[6], acc[7]);
          }
        }
      }
    } else if (STAGED && !RED && warp == 1) {
      // ===================== epilogue inputs (TMA), while the math warpgroups run the tile's k-blocks =====================
      // Per tile: the bias row once the previous tile's epilogue has consumed it, then the residual / aux subtiles of
      // both warpgroups into their buffer rings as the stores of earlier subtiles free them.  Rows >= M and columns >= N
      // are zero-filled by TMA.
      if (lane == 0) {
        uint32_t it = 0, tc = 0;
        for (int unit = worker; unit < num_units; unit += num_workers, ++tc) {
          const int m_blk = unit / num_n_blocks, n_blk = unit - m_blk * num_n_blocks;      // num_splits == 1
          const int m_row = m_blk * TILE_M + (int)rank * BLOCK_M, n0 = n_blk * BLOCK_N;
          mbar_wait_nocall(bias_empty, (tc & 1) ^ 1);
          if (ep.bias) {
            const uint32_t bytes = 4u * (uint32_t)min(BLOCK_N, N - n0);
            mbar_expect_tx(bias_full, bytes);
            bulk_load_1d(sBias, ep.bias + n0, bytes, bias_full);
          } else {
            mbar_arrive(bias_full);
          }
          if (HAS_IN) {
            for (int s = 0; s < NSUB; ++s, ++it) {
              const uint32_t b = it % EPI_BUFS, ph = (it / EPI_BUFS) & 1;
#pragma unroll
              for (int w = 0; w < 2; ++w) {
                const uint32_t slot = w * EPI_BUFS + b;
                mbar_wait_nocall(epi_empty + 8 * slot, ph ^ 1);
                mbar_expect_tx(epi_full + 8 * slot, EPI_SUB_BYTES);
                tma_load_2d(sEpi + slot * EPI_SUB_BYTES, &tmIn, epi_full + 8 * slot, n0 + s * SUB_COLS,
                            m_row + w * EPI_ROWS);
              }
            }
          }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ===================== math warpgroups: wgmma main loop, then the epilogue from registers =====================
    const int mw = (threadIdx.x >> 7) - 1;         // math warpgroup: rows 64 mw .. 64 mw + 63 of the tile
    const bool leader = (threadIdx.x & 127) == 0;  // releases the stages for the warpgroup
    auto release = [&](int st) {
      const uint32_t bar = empty_bar + 8 * st;
      if (TWO) { mbar_arrive_cluster(mapa_shared(bar, 0)); mbar_arrive_cluster(mapa_shared(bar, 1)); }
      else mbar_arrive(bar);
    };
    const int wq = warp & 3;                       // warp within the warpgroup: 16 accumulator rows each
    const GeluConsts gc;

    float acc[C::ACC];
    int stage = 0;
    uint32_t phase = 0;
    uint32_t it = 0, tc = 0;                       // STAGED: subtile and tile counters (ring / bias parities)
    for (int unit = worker; unit < num_units; unit += num_workers, ++tc) {
      const int split = unit / num_tiles, tile = unit - split * num_tiles;
      const int m_blk = tile / num_n_blocks, n_blk = tile - m_blk * num_n_blocks;
      const int kb0 = split * kb_per_split, kb1 = min(num_kb, kb0 + kb_per_split);
      int prev_stage = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait_nocall(full_bar + 8 * stage, phase);
        const uint32_t a_src = sA + stage * A_STAGE_BYTES + mw * (64 * 128), b_src = sB + stage * C::B_STAGE_BYTES;
        wgmma_fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WG_K; ++k) {
          const uint64_t adesc = A_MN ? make_smem_desc_sw128(a_src + k * (WG_K * 128), MN_ATOM_BYTES, 1024)
                                      : make_smem_desc_sw128(a_src + k * (WG_K * 2), 16, 1024);
          const uint64_t bdesc = B_MN ? make_smem_desc_sw128(b_src + k * (WG_K * 128), MN_ATOM_BYTES, 1024)
                                      : make_smem_desc_sw128(b_src + k * (WG_K * 2), 16, 1024);
          wgmma_tile<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0, FP8>(acc, adesc, bdesc, (kb > kb0 || k > 0) ? 1 : 0);
        }
        wgmma_commit();
        wgmma_fence_regs(acc);
        // the previous k-block's wgmmas have finished reading their stage once at most this group is in flight
        wgmma_wait<1>();
        wgmma_fence_regs(acc);
        if (prev_stage >= 0 && leader) release(prev_stage);
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (leader) release(prev_stage);

      // ---- epilogue.  Accumulator layout of m64nN: thread (warp wq, lane) holds rows wq*16 + lane/4 (+8) and, for
      // every 8-column group j, columns 8 j + 2 (lane % 4) + {0, 1}: acc[4 j + 2 h + {0, 1}] for row half h.
      if constexpr (STAGED) {
        // Subtile by subtile (64 rows x SUB_COLS): wait for the input subtile (HAS_IN), transform it -- or fill the
        // buffer -- in place, fence to the async proxy, sync the warpgroup; then the leader stores the subtile by TMA
        // (rows >= M / columns >= N clipped) and waits only until the store has READ the buffer before it is handed
        // back to the input warp (or rewritten).  The global writes drain while the next subtile / tile runs.
        const int m_row = m_blk * TILE_M + (int)rank * BLOCK_M + mw * EPI_ROWS, n0 = n_blk * BLOCK_N;
        const int c2 = 2 * (lane & 3);
        float rs[2] = {1.f, 1.f};             // FP8: the row scales of this thread's two rows (padding rows clamped)
        if constexpr (FP8) {
#pragma unroll
          for (int h = 0; h < 2; ++h) rs[h] = __ldg(ep.row_scale + min(m_row + wq * 16 + (lane >> 2) + 8 * h, M - 1));
        }
        // DROP: kept elements of this thread's two rows are scaled by rowf = 1 / (1 - p) x the row's drop-path factor
        float rowf[2] = {1.f, 1.f};
        unsigned long long dkey = 0ull;
        uint32_t dthresh = 0u;
        if constexpr (DROP) {
          const float inv = 1.f / (1.f - dp.p);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = m_row + wq * 16 + (lane >> 2) + 8 * h;
            rowf[h] = dp.path_rows ? inv * drop_path_factor(dp.seed, dp.path_site, dp.path_p, row / dp.path_rows)
                                   : inv;
          }
          dkey = dropout_key(dp.seed, dp.site);
          dthresh = dropout_threshold(dp.p);
        }
        if (!RED) mbar_wait_nocall(bias_full, tc & 1);
#pragma unroll
        for (int s = 0; s < NSUB; ++s, ++it) {
          const uint32_t b = it % EPI_BUFS, ph = (it / EPI_BUFS) & 1;
          // two outputs fill both buffers: the previous subtile's stores must have read them (the leader waited)
          if (BOTH_BUFS) named_bar_sync(1 + mw, 128);
          const uint32_t buf = sEpi + (mw * EPI_BUFS + (BOTH_BUFS ? 0u : b)) * EPI_SUB_BYTES;
          if (HAS_IN) mbar_wait_nocall(epi_full + 8 * (mw * EPI_BUFS + b), ph);
          uint32_t second[SUB_COLS / 4];      // EPI_GELU_AUX: GELU(aux), held until the buffer is free for it
#pragma unroll
          for (int jj = 0; jj < SUB_COLS / 8; ++jj) {
            const int j = s * (SUB_COLS / 8) + jj;        // 8-column group of the tile: constant after unrolling
            float2 bq = make_float2(0.f, 0.f);
            if (!RED)
              asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(bq.x), "=f"(bq.y) : "r"(sBias + 4 * (8 * j + c2)));
            float2 ws = make_float2(1.f, 1.f);        // FP8: column scales (N % 128 == 0: every column exists)
            if constexpr (FP8) ws = __ldg(reinterpret_cast<const float2*>(ep.w_scale + n0 + 8 * j + c2));
            uint32_t keep2[2] = {3u, 3u};             // DROP: keep bits of this thread's two columns, per row half
            if constexpr (DROP) {
              // lanes 2i and 2i + 1 hold the same four columns of the same two rows: each draws the four keep bits of one
              // of the rows (one Philox call per four elements) and the pair swaps them
              const int hh = lane & 1;
              const int row = m_row + wq * 16 + (lane >> 2) + 8 * hh;
              const uint4 r = philox4x32_10(dkey, (unsigned long long)row * (unsigned long long)(N >> 2) +
                                                      (unsigned long long)((n0 + 8 * j + c2) >> 2));
              const uint32_t mine = (uint32_t)(r.x >= dthresh) | (uint32_t)(r.y >= dthresh) << 1 |
                                    (uint32_t)(r.z >= dthresh) << 2 | (uint32_t)(r.w >= dthresh) << 3;
              const uint32_t other = __shfl_xor_sync(0xffffffffu, mine, 1);
              keep2[0] = ((hh ? other : mine) >> (c2 & 2)) & 3u;
              keep2[1] = ((hh ? mine : other) >> (c2 & 2)) & 3u;
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = wq * 16 + (lane >> 2) + 8 * h;  // row of the subtile; 16-byte chunks XOR-swizzled by r & 7
              // bf16: chunk jj, 4 bytes per lane pair; fp32: chunk 2 jj + (lane % 4) / 2, 8 bytes per lane pair
              const uint32_t off = OUT_F32 ? r * 128 + (((2 * jj + ((lane & 3) >> 1)) ^ (r & 7)) << 4) + 8 * (lane & 1)
                                           : r * 128 + ((jj ^ (r & 7)) << 4) + 4 * (lane & 3);
              float a0 = acc[4 * j + 2 * h], a1 = acc[4 * j + 2 * h + 1];
              if constexpr (FP8) {
                a0 = __fmul_rn(__fmul_rn(a0, rs[h]), ws.x); a1 = __fmul_rn(__fmul_rn(a1, rs[h]), ws.y);
              }
              float v0 = __fmaf_rn(a0, ep.alpha, bq.x);
              float v1 = __fmaf_rn(a1, ep.alpha, bq.y);
              if (BM == EPI_BF16 && n0 + 8 * j + c2 < ep.col_scale_ncols) {
                v0 = __fmul_rn(v0, ep.col_scale); v1 = __fmul_rn(v1, ep.col_scale);
              }
              // DROP: the scale of each of the two elements (0 for a dropped one)
              const float s0 = (keep2[h] & 1u) ? rowf[h] : 0.f, s1 = (keep2[h] & 2u) ? rowf[h] : 0.f;
              if (BOTH_BUFS) {                  // ACT3: out = GELU(v), out2 = GELU'(v);  ACT1_Z: out = GELU(v), out2 = v
                uint32_t g, d;
                if (BM == EPI_ACT3) {
                  if constexpr (DROP) {
                    float g0, g1, d0, d1;
                    gelu_pair2(gc, v0, v1, g0, g1, d0, d1);
                    g = pack_bf16x2(__fmul_rn(g0, s0), __fmul_rn(g1, s1));
                    d = pack_bf16x2(d0, d1);
                  } else {
                    gelu_and_grad2(gc, v0, v1, g, d);
                  }
                } else {
                  d = pack_bf16x2(v0, v1);
                  gelu2(gc, v0, v1);
                  if (DROP) { v0 = __fmul_rn(v0, s0); v1 = __fmul_rn(v1, s1); }
                  g = pack_bf16x2(v0, v1);
                }
                asm volatile("st.shared.u32 [%0], %1;" ::"r"(buf + off), "r"(g) : "memory");
                asm volatile("st.shared.u32 [%0], %1;" ::"r"(buf + EPI_SUB_BYTES + off), "r"(d) : "memory");
              } else if (BM == EPI_GELU_AUX) {  // out = v GELU'(z), out2 = GELU(z), z = aux
                uint32_t a;
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(a) : "r"(buf + off) : "memory");
                const float2 z = unpack_bf16x2(a);
                float g0, g1, d0, d1;
                gelu_pair2(gc, z.x, z.y, g0, g1, d0, d1);
                float o0 = __fmul_rn(v0, d0), o1 = __fmul_rn(v1, d1);
                if (DROP) {                     // out2 is fc2's (dropped) input: the weight gradient's operand
                  o0 = __fmul_rn(o0, s0); o1 = __fmul_rn(o1, s1);
                  g0 = __fmul_rn(g0, s0); g1 = __fmul_rn(g1, s1);
                }
                asm volatile("st.shared.u32 [%0], %1;" ::"r"(buf + off), "r"(pack_bf16x2(o0, o1)) : "memory");
                second[2 * jj + h] = pack_bf16x2(g0, g1);
              } else if (RED) {
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(buf + off), "f"(v0), "f"(v1) : "memory");
              } else if (BM == EPI_RES_F32) {
                float r0, r1;
                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(r0), "=f"(r1) : "r"(buf + off) : "memory");
                if (DROP) { v0 = __fmul_rn(v0, s0); v1 = __fmul_rn(v1, s1); }
                v0 += r0; v1 += r1;
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(buf + off), "f"(v0), "f"(v1) : "memory");
              } else {
                if (BM == EPI_ACT1) gelu2(gc, v0, v1);
                if (BM == EPI_MUL_AUX) {
                  uint32_t a;
                  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(a) : "r"(buf + off) : "memory");
                  const float2 af = unpack_bf16x2(a);
                  v0 *= af.x; v1 *= af.y;
                  if (DROP) { v0 = __fmul_rn(v0, s0); v1 = __fmul_rn(v1, s1); }
                }
                asm volatile("st.shared.u32 [%0], %1;" ::"r"(buf + off), "r"(pack_bf16x2(v0, v1)) : "memory");
              }
            }
          }
          fence_proxy_async_smem();
          named_bar_sync(1 + mw, 128);
          if (leader) {
            if (RED && ep.det_ws) tma_store_2d(&tmOut, buf, n0 + s * SUB_COLS, split * num_m_blocks * TILE_M + m_row);
            else if (RED) tma_reduce_add_2d(&tmOut, buf, n0 + s * SUB_COLS, m_row);
            else tma_store_2d(&tmOut, buf, n0 + s * SUB_COLS, m_row);
            if (BOTH_BUFS) tma_store_2d(&tmOut2, buf + EPI_SUB_BYTES, n0 + s * SUB_COLS, m_row);
            bulk_commit();
            bulk_wait_read<0>();
            if (HAS_IN && !TWO_OUT) mbar_arrive(epi_empty + 8 * (mw * EPI_BUFS + b));
          }
          if constexpr (BM == EPI_GELU_AUX) {
            named_bar_sync(1 + mw, 128);      // the first output's store has read the buffer
#pragma unroll
            for (int jj = 0; jj < SUB_COLS / 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int r = wq * 16 + (lane >> 2) + 8 * h;
                asm volatile("st.shared.u32 [%0], %1;" ::"r"(buf + r * 128 + ((jj ^ (r & 7)) << 4) + 4 * (lane & 3)),
                             "r"(second[2 * jj + h]) : "memory");
              }
            fence_proxy_async_smem();
            named_bar_sync(1 + mw, 128);
            if (leader) {
              tma_store_2d(&tmOut2, buf, n0 + s * SUB_COLS, m_row);
              bulk_commit();
              bulk_wait_read<0>();
              mbar_arrive(epi_empty + 8 * (mw * EPI_BUFS + b));
            }
          }
        }
        if (!RED && leader) mbar_arrive(bias_empty);      // after the last subtile's warpgroup sync: the bias row is read
      } else {
      const int row_lo = m_blk * TILE_M + (int)rank * BLOCK_M + mw * 64 + wq * 16 + (lane >> 2);
      const int col_base = n_blk * BLOCK_N + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {   // fully unrolled: acc[] is indexed with constants only
        const int col = col_base + 8 * j;
        if (n_blk * BLOCK_N + 8 * j >= N) break;        // warp-uniform: N % 32 == 0
        float2 bq = make_float2(0.f, 0.f);
        if (ep.bias) bq = __ldg(reinterpret_cast<const float2*>(ep.bias + col));
        float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row_lo + 8 * h;
          const bool rv = row < M;
          float v0 = __fmaf_rn(acc[4 * j + 2 * h], ep.alpha, bq.x);
          float v1 = __fmaf_rn(acc[4 * j + 2 * h + 1], ep.alpha, bq.y);
          if (col < ep.col_scale_ncols) { v0 = __fmul_rn(v0, ep.col_scale); v1 = __fmul_rn(v1, ep.col_scale); }
          if (ep.act == 3) {                 // out = GELU(v), out2 = GELU'(v)
            uint32_t g, d;
            gelu_and_grad2(gc, v0, v1, g, d);
            if (rv) {
              *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(ep.out) + (long long)row * ep.ldo + col) = g;
              if (ep.out2) *reinterpret_cast<uint32_t*>(ep.out2 + (long long)row * ep.ldo2 + col) = d;
            }
            continue;
          }
          if (ep.out2 && rv && ep.act != 5)  // pre-activation (act 1) or a second copy
            *reinterpret_cast<uint32_t*>(ep.out2 + (long long)row * ep.ldo2 + col) = pack_bf16x2(v0, v1);
          if (ep.act == 1) gelu2(gc, v0, v1);
          const int grow = rv ? row : M - 1;        // clamped: operand loads of padding rows stay in bounds
          if (ep.act == 2 || ep.act == 4 || ep.act == 5) {
            const float2 a = unpack_bf16x2(__ldg(reinterpret_cast<const unsigned int*>(ep.aux + (long long)grow * ep.ldaux + col)));
            if (ep.act == 2) { v0 *= gelu_grad_fast(a.x); v1 *= gelu_grad_fast(a.y); }
            else if (ep.act == 4) { v0 *= a.x; v1 *= a.y; }
            else {                           // out = v GELU'(aux), out2 = GELU(aux)
              float g0, g1, d0, d1;
              gelu_pair2(gc, a.x, a.y, g0, g1, d0, d1);
              v0 = __fmul_rn(v0, d0); v1 = __fmul_rn(v1, d1);
              if (rv) *reinterpret_cast<uint32_t*>(ep.out2 + (long long)row * ep.ldo2 + col) = pack_bf16x2(g0, g1);
            }
          }
          if (ep.residual) {
            const int rrow = ep.res_row_mod ? grow % ep.res_row_mod : grow;
            const float2 r = __ldg(reinterpret_cast<const float2*>(ep.residual + (long long)rrow * ep.ldr + col));
            v0 += r.x; v1 += r.y;
          }
          if (!rv) continue;
          cs0 += v0; cs1 += v1;
          if (ep.out_mode == 0) {
            *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(ep.out) + (long long)row * ep.ldo + col) = pack_bf16x2(v0, v1);
          } else if (ep.out_mode == 1) {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(ep.out) + (long long)row * ep.ldo + col) = make_float2(v0, v1);
          } else if (ep.det_ws) {
            *reinterpret_cast<float2*>(ep.det_ws + ((long long)split * num_m_blocks * TILE_M + row) * N + col) =
                make_float2(v0, v1);
          } else {
            red_add_v2(reinterpret_cast<float*>(ep.out) + (long long)row * ep.ldo + col, v0, v1);
          }
        }
        if (ep.colsum) {    // lanes with the same lane % 4 hold the same two columns: fold, then one atomic pair
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            cs0 += __shfl_xor_sync(0xffffffffu, cs0, o);
            cs1 += __shfl_xor_sync(0xffffffffu, cs1, o);
          }
          if (lane < 4) red_add_v2(ep.colsum + col, cs0, cs1);
        }
      }
      }
    }
    if (STAGED && leader) bulk_wait<0>();      // this warpgroup's last stores are complete before the CTA exits
  }
  if (TWO) cluster_sync_all();      // the peer may still multicast into this CTA's smem or arrive on its barriers
}

template <int BLOCK_N, bool A_MN, bool B_MN, bool TWO, int MODE, bool FP8>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmOut2,
                       const __grid_constant__ CUtensorMap tmIn, int M, int N, int K, int num_m_blocks,
                       int num_n_blocks, int kb_per_split, int num_splits, EpiParams ep) {
  static_assert(base_mode(MODE) == MODE, "the dropout forms run as gemm_drop_wgmma_kernel");
  gemm_bf16_wgmma_body<BLOCK_N, A_MN, B_MN, TWO, MODE, FP8>(tmA, tmB, tmOut, tmOut2, tmIn, M, N, K, num_m_blocks,
                                                             num_n_blocks, kb_per_split, num_splits, ep, DropParams{});
}
// the dropout forms: the same kernel with the mask's parameters
template <int BLOCK_N, bool B_MN, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_drop_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmOut2,
                       const __grid_constant__ CUtensorMap tmIn, int M, int N, int K, int num_m_blocks,
                       int num_n_blocks, int kb_per_split, int num_splits, EpiParams ep, DropParams dp) {
  static_assert(base_mode(MODE) != MODE, "dropout forms only");
  gemm_bf16_wgmma_body<BLOCK_N, false, B_MN, false, MODE, false>(tmA, tmB, tmOut, tmOut2, tmIn, M, N, K, num_m_blocks,
                                                                  num_n_blocks, kb_per_split, num_splits, ep, dp);
}

// The deterministic form's ordered pass: out[m, n] = ((out + P_0) + P_1) + ... + P_{s-1}, P_s the partial tile of
// split s (float4 over n: N % 32 == 0); colsum_a[m] += Q_0 + Q_1 + ..., Q_s = its n-block partials summed in order.
__global__ void gemm_det_merge_out_kernel(const float* __restrict__ ws, int splits, int M, int Mp, int N,
                                          float* __restrict__ out, long long ldo) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= (long long)M * N) return;
  const int m = (int)(i / N), n = (int)(i % N);
  float4 acc = *reinterpret_cast<const float4*>(out + m * ldo + n);
  for (int sp = 0; sp < splits; ++sp) {
    const float4 p = *reinterpret_cast<const float4*>(ws + ((long long)sp * Mp + m) * N + n);
    acc.x += p.x; acc.y += p.y; acc.z += p.z; acc.w += p.w;
  }
  *reinterpret_cast<float4*>(out + m * ldo + n) = acc;
}
__global__ void gemm_det_merge_colsum_kernel(const float* __restrict__ cs, int splits, int nnb, int M, int Mp,
                                             float* __restrict__ colsum_a) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float acc = colsum_a[m];
  for (int sp = 0; sp < splits; ++sp) {
    float q = cs[(long long)sp * nnb * Mp + m];
    for (int nb = 1; nb < nnb; ++nb) q += cs[((long long)sp * nnb + nb) * Mp + m];
    acc += q;
  }
  colsum_a[m] = acc;
}

// Split count, rows of one split's slab and floats of the deterministic workspace, as launch() computes them
struct DetLayout {
  int splits, Mp, nnb;
  long long floats;
};
inline DetLayout det_layout(int M, int N, int K, int splits) {
  const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
  splits = max(1, min(splits, num_kb));
  const int kb_per_split = (num_kb + splits - 1) / splits;
  DetLayout d;
  d.splits = (num_kb + kb_per_split - 1) / kb_per_split;
  d.Mp = (M + BLOCK_M - 1) / BLOCK_M * BLOCK_M;
  d.nnb = N % 256 == 0 ? N / 256 : (N + 127) / 128;
  d.floats = (long long)d.splits * d.Mp * N + (long long)d.splits * d.nnb * d.Mp;
  return d;
}

template <int BLOCK_N, bool A_MN, bool B_MN, bool TWO, int MODE, bool FP8>
constexpr auto kernel_of() {
  if constexpr (base_mode(MODE) != MODE) {
    static_assert(!A_MN && !TWO && !FP8, "dropout forms: K-major A, single CTAs, bf16");
    return gemm_drop_wgmma_kernel<BLOCK_N, B_MN, MODE>;
  } else {
    return gemm_bf16_wgmma_kernel<BLOCK_N, A_MN, B_MN, TWO, MODE, FP8>;
  }
}

template <int BLOCK_N, bool A_MN, bool B_MN, bool TWO, int MODE = EPI_GENERIC, bool FP8 = false>
int launch(const void* A, long long lda, const void* B, long long ldb, int M, int N, int K, int splits,
           const EpiParams& ep, cudaStream_t stream, const DropParams& dp = DropParams{}) {
  using C = Cfg<BLOCK_N>;
  const bool det = ep.det_ws != nullptr || ep.det_cs != nullptr;
  if (det && TWO) { set_last_error("gemm: the deterministic form runs on single CTAs"); return EGOVLP_ERR_UNSUPPORTED; }
  CUtensorMap tmA, tmB;
  int rc;
  if (FP8) {            // e4m3 bytes: the same [rows, 128 B] boxes as the K-major bf16 maps
    rc = make_tmap_2d_u8(&tmA, A, M, K, lda, BLOCK_M, 2 * BLOCK_K);
    if (!rc) rc = make_tmap_2d_u8(&tmB, B, N, K, ldb, BLOCK_N, 2 * BLOCK_K);
    if (rc) return rc;
  } else {
    if (!A_MN) rc = make_tmap_2d_bf16(&tmA, A, M, K, lda, BLOCK_M, BLOCK_K);
    else       rc = make_tmap_2d_bf16(&tmA, A, K, M, lda, BLOCK_K, 64);
    if (rc) return rc;
    if (!B_MN) rc = make_tmap_2d_bf16(&tmB, B, N, K, ldb, TWO ? BLOCK_N / 2 : BLOCK_N, BLOCK_K);
    else       rc = make_tmap_2d_bf16(&tmB, B, K, N, ldb, BLOCK_K, 64);
    if (rc) return rc;
  }
  // epilogue subtiles of the staged forms: [64 rows, 128 B] boxes over out / out2 / residual / aux
  constexpr bool STAGED = MODE != EPI_GENERIC;
  constexpr int BM = base_mode(MODE);
  CUtensorMap tmOut = {}, tmOut2 = {}, tmIn = {};
  if (BM == EPI_RED_F32 && ep.det_ws) {        // the split slabs of the workspace, [splits * Mp, N]
    const DetLayout dl = det_layout(M, N, K, splits);
    rc = make_tmap_2d_f32(&tmOut, ep.det_ws, (uint64_t)dl.splits * dl.Mp, N, N, EPI_ROWS, 32);
  } else if (BM == EPI_RES_F32 || BM == EPI_RED_F32) {
    rc = make_tmap_2d_f32(&tmOut, ep.out, M, N, ep.ldo, EPI_ROWS, 32);
    if (!rc && BM == EPI_RES_F32) rc = make_tmap_2d_f32(&tmIn, ep.residual, M, N, ep.ldr, EPI_ROWS, 32);
  } else if (STAGED) {
    rc = make_tmap_2d_bf16(&tmOut, ep.out, M, N, ep.ldo, EPI_ROWS, 64);
    if (!rc && (BM == EPI_ACT3 || BM == EPI_ACT1_Z || BM == EPI_GELU_AUX))
      rc = make_tmap_2d_bf16(&tmOut2, ep.out2, M, N, ep.ldo2, EPI_ROWS, 64);
    if (!rc && (BM == EPI_MUL_AUX || BM == EPI_GELU_AUX))
      rc = make_tmap_2d_bf16(&tmIn, ep.aux, M, N, ep.ldaux, EPI_ROWS, 64);
  }
  if (rc) return rc;
  constexpr int SMEM_BYTES = STAGED ? C::SMEM_BYTES_STAGED : C::SMEM_BYTES;
  constexpr int TILE_M = TWO ? 2 * BLOCK_M : BLOCK_M;
  const int num_m_blocks = (M + TILE_M - 1) / TILE_M, num_n_blocks = (N + BLOCK_N - 1) / BLOCK_N;
  const int num_kb = (K + (FP8 ? 2 : 1) * BLOCK_K - 1) / ((FP8 ? 2 : 1) * BLOCK_K);
  splits = max(1, min(splits, num_kb));
  const int kb_per_split = (num_kb + splits - 1) / splits;
  splits = (num_kb + kb_per_split - 1) / kb_per_split;  // no empty splits
  const int units = num_m_blocks * num_n_blocks * splits;
  auto kern = kernel_of<BLOCK_N, A_MN, B_MN, TWO, MODE, FP8>();
  static bool attr_set = false;
  if (!attr_set) {
    EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_set = true;
  }
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = SMEM_BYTES;
  cfg.stream = stream;
  if (TWO) {
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  }
  // persistent grid: as many workers as can be resident at once.  For pairs that is the number of co-resident 2-CTA
  // clusters, which the GPC layout can hold below num_sms() / 2: a grid sized by SM count would leave a second wave
  // of clusters that the static tile schedule then waits for.
  static int resident = 0;
  if (!resident) {
    if (TWO) {
      cfg.gridDim = dim3(num_sms() & ~1);
      EGOVLP_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&resident, kern, &cfg));
      if (resident < 1) resident = 1;
    } else {
      resident = num_sms();
    }
  }
  const int workers = min(units, resident);
  cfg.gridDim = dim3(TWO ? 2 * workers : workers);
  if constexpr (BM != MODE)
    EGOVLP_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmOut, tmOut2, tmIn, M, N, K, num_m_blocks, num_n_blocks,
                                         kb_per_split, splits, ep, dp));
  else
    EGOVLP_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmOut, tmOut2, tmIn, M, N, K, num_m_blocks, num_n_blocks,
                                         kb_per_split, splits, ep));
  if (det) {
    const int Mp = num_m_blocks * TILE_M;
    if (ep.det_ws) {
      const long long n4 = (long long)M * N / 4;
      gemm_det_merge_out_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(
          ep.det_ws, splits, M, Mp, N, reinterpret_cast<float*>(ep.out), ep.ldo);
      EGOVLP_CHECK_LAUNCH();
    }
    if (ep.det_cs) {
      gemm_det_merge_colsum_kernel<<<(M + 255) / 256, 256, 0, stream>>>(ep.det_cs, splits, num_n_blocks, M, Mp,
                                                                        ep.colsum_a);
      EGOVLP_CHECK_LAUNCH();
    }
  }
  return EGOVLP_OK;
}

// MN-major A (the wgrad forms) always runs on single CTAs
template <int BLOCK_N, bool TWO, int MODE = EPI_GENERIC>
int dispatch_major(int a_mn, int b_mn, const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                   int splits, const EpiParams& ep, cudaStream_t stream) {
  if (!a_mn && !b_mn) return launch<BLOCK_N, false, false, TWO, MODE>(A, lda, B, ldb, M, N, K, splits, ep, stream);
  if (!a_mn && b_mn) return launch<BLOCK_N, false, true, TWO, MODE>(A, lda, B, ldb, M, N, K, splits, ep, stream);
  if (a_mn && b_mn) return launch<BLOCK_N, true, true, false, EPI_GENERIC>(A, lda, B, ldb, M, N, K, splits, ep, stream);
  return launch<BLOCK_N, true, false, false, EPI_GENERIC>(A, lda, B, ldb, M, N, K, splits, ep, stream);
}

// TMA's rules for a tensor the staged epilogue loads or stores: 16-byte aligned base, row stride a multiple of 16 bytes
inline bool tma_ok(const void* p, long long ld_bytes) {
  return (reinterpret_cast<uintptr_t>(p) & 15) == 0 && ld_bytes % 16 == 0;
}

// Which specialised epilogue (if any) computes exactly what `ep` asks for; EGOVLP_GEMM_GENERIC_EPI=1 keeps every call on
// the generic one (the kernel tests run both and compare).  The specialised forms move their epilogue bytes by TMA, so a
// call whose tensors TMA cannot address (see tma_ok; the bias row is a 1-D bulk copy) takes the generic epilogue.
inline int specialised_mode(const EpiParams& ep);
inline int epi_mode(const EpiParams& ep) {
  const char* g = getenv("EGOVLP_GEMM_GENERIC_EPI");
  if (g && g[0] == '1') return EPI_GENERIC;
  return specialised_mode(ep);
}
inline int specialised_mode(const EpiParams& ep) {
  if (ep.colsum || ep.res_row_mod) return EPI_GENERIC;
  if (ep.bias && (reinterpret_cast<uintptr_t>(ep.bias) & 15) != 0) return EPI_GENERIC;
  const bool no_scale = ep.col_scale_ncols == 0;
  const bool out16 = tma_ok(ep.out, ep.ldo * 2);
  if (ep.act == 0 && ep.out_mode == 0 && !ep.residual && !ep.out2 && out16) return EPI_BF16;
  if (ep.act == 3 && ep.out_mode == 0 && !ep.residual && ep.out2 && no_scale && out16 && tma_ok(ep.out2, ep.ldo2 * 2))
    return EPI_ACT3;
  if (ep.act == 4 && ep.out_mode == 0 && !ep.residual && !ep.out2 && no_scale && out16 && tma_ok(ep.aux, ep.ldaux * 2))
    return EPI_MUL_AUX;
  if (ep.act == 0 && ep.out_mode == 1 && ep.residual && !ep.out2 && no_scale && tma_ok(ep.out, ep.ldo * 4) &&
      tma_ok(ep.residual, ep.ldr * 4))
    return EPI_RES_F32;
  if (ep.act == 1 && ep.out_mode == 0 && !ep.residual && !ep.out2 && no_scale && out16) return EPI_ACT1;
  if (ep.act == 1 && ep.out_mode == 0 && !ep.residual && ep.out2 && no_scale && out16 && tma_ok(ep.out2, ep.ldo2 * 2))
    return EPI_ACT1_Z;
  if (ep.act == 5 && ep.out_mode == 0 && !ep.residual && no_scale && out16 && tma_ok(ep.out2, ep.ldo2 * 2) &&
      tma_ok(ep.aux, ep.ldaux * 2))
    return EPI_GELU_AUX;
  if (ep.act == 0 && ep.out_mode == 2 && !ep.bias && !ep.residual && !ep.out2 && no_scale && tma_ok(ep.out, ep.ldo * 4))
    return EPI_RED_F32;
  return EPI_GENERIC;
}

// EGOVLP_GEMM_PAIR=1 runs the K-major-A forms with N % 256 == 0 on CTA pairs (the tests exercise both schedules).  Not
// the default: on a 400 W H100 the headline training step ran at 95 clips/s with pairs vs 114 with single CTAs.
inline bool use_pairs() {
  const char* e = getenv("EGOVLP_GEMM_PAIR");
  return e && e[0] == '1';
}

template <int BLOCK_N, bool TWO>
int dispatch_mode(int a_mn, int b_mn, const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                  int splits, const EpiParams& ep, cudaStream_t stream) {
  if (!a_mn) {       // the step's hot forms (K-major A) get a compile-time specialised epilogue
    switch (epi_mode(ep)) {
      case EPI_BF16: return dispatch_major<BLOCK_N, TWO, EPI_BF16>(a_mn, b_mn, A, lda, B, ldb, M, N, K, splits, ep, stream);
      case EPI_ACT3: return dispatch_major<BLOCK_N, TWO, EPI_ACT3>(a_mn, b_mn, A, lda, B, ldb, M, N, K, splits, ep, stream);
      case EPI_MUL_AUX: return dispatch_major<BLOCK_N, TWO, EPI_MUL_AUX>(a_mn, b_mn, A, lda, B, ldb, M, N, K, splits, ep, stream);
      case EPI_RES_F32: return dispatch_major<BLOCK_N, TWO, EPI_RES_F32>(a_mn, b_mn, A, lda, B, ldb, M, N, K, splits, ep, stream);
      case EPI_ACT1: return dispatch_major<BLOCK_N, TWO, EPI_ACT1>(a_mn, b_mn, A, lda, B, ldb, M, N, K, splits, ep, stream);
      case EPI_ACT1_Z: return dispatch_major<BLOCK_N, TWO, EPI_ACT1_Z>(a_mn, b_mn, A, lda, B, ldb, M, N, K, splits, ep, stream);
      case EPI_GELU_AUX: return dispatch_major<BLOCK_N, TWO, EPI_GELU_AUX>(a_mn, b_mn, A, lda, B, ldb, M, N, K, splits, ep, stream);
      default: break;
    }
  } else if (b_mn && epi_mode(ep) == EPI_RED_F32) {      // the weight gradients: split-K partial tiles added by TMA
    return launch<BLOCK_N, true, true, false, EPI_RED_F32>(A, lda, B, ldb, M, N, K, splits, ep, stream);
  }
  return dispatch_major<BLOCK_N, TWO>(a_mn, b_mn, A, lda, B, ldb, M, N, K, splits, ep, stream);
}

// The dropout forms exist for the video tower's five training calls only (K-major A; B K-major in the forward, MN-major
// in the fc2 input gradient), on single CTAs.  There is no generic fallback, as the generic epilogue has no mask: any
// other descriptor with dropout is refused.
template <int BLOCK_N>
int dispatch_drop(int a_mn, int b_mn, const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                  const EpiParams& ep, const DropParams& dp, cudaStream_t stream) {
  const int m = a_mn ? EPI_GENERIC : specialised_mode(ep);
  if (!b_mn && m == EPI_RES_F32)
    return launch<BLOCK_N, false, false, false, EPI_RES_F32_DROP>(A, lda, B, ldb, M, N, K, 1, ep, stream, dp);
  if (!b_mn && m == EPI_ACT3)
    return launch<BLOCK_N, false, false, false, EPI_ACT3_DROP>(A, lda, B, ldb, M, N, K, 1, ep, stream, dp);
  if (!b_mn && m == EPI_ACT1_Z)
    return launch<BLOCK_N, false, false, false, EPI_ACT1_Z_DROP>(A, lda, B, ldb, M, N, K, 1, ep, stream, dp);
  if (b_mn && m == EPI_MUL_AUX)
    return launch<BLOCK_N, false, true, false, EPI_MUL_AUX_DROP>(A, lda, B, ldb, M, N, K, 1, ep, stream, dp);
  if (b_mn && m == EPI_GELU_AUX)
    return launch<BLOCK_N, false, true, false, EPI_GELU_AUX_DROP>(A, lda, B, ldb, M, N, K, 1, ep, stream, dp);
  set_last_error("gemm: dropout needs one of the forms bias + fp32 residual -> fp32 (act 0), GELU with out2 (act 1 / 3) "
                 "with K-major A and B, or act 4 / 5 with K-major A and MN-major B, with TMA-aligned tensors");
  return EGOVLP_ERR_UNSUPPORTED;
}

}  // namespace

}  // namespace egovlp

using namespace egovlp;

extern "C" int egovlp_gemm_bf16(const void* A, int a_mn_major, long long lda, const void* B, int b_mn_major,
                                long long ldb, int M, int N, int K, const egovlp_gemm_epilogue* e, int split_k,
                                void* stream) {
  EGOVLP_CHECK_ARG(A && B && e && e->out, "gemm: null pointer");
  EGOVLP_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm: bad shape M=%d N=%d K=%d", M, N, K);
  EGOVLP_CHECK_ARG(N % 32 == 0, "gemm: N=%d must be a multiple of 32", N);
  EGOVLP_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "gemm: leading dimensions must be multiples of 8 (16B TMA strides)");
  EGOVLP_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0,
                   "gemm: operands must be 16B aligned");
  EGOVLP_CHECK_ARG(e->out_mode >= 0 && e->out_mode <= 2 && e->act >= 0 && e->act <= 5, "gemm: bad epilogue mode");
  EGOVLP_CHECK_ARG(split_k <= 1 || e->out_mode == 2, "gemm: split_k > 1 needs out_mode=2 (fp32 atomic accumulate)");
  EGOVLP_CHECK_ARG((e->act != 2 && e->act != 4 && e->act != 5) || e->aux, "gemm: act=2/4/5 needs aux");
  EGOVLP_CHECK_ARG(e->act != 5 || e->out2, "gemm: act=5 needs out2");
  EGOVLP_CHECK_ARG(e->ldo % 8 == 0, "gemm: ldo must be a multiple of 8");
  // the generic epilogue moves bias / residual / fp32 out / colsum as float2 and aux / bf16 out / out2 as bf16x2
  const auto off = [](const void* p, uintptr_t align) { return (reinterpret_cast<uintptr_t>(p) & (align - 1)) != 0; };
  EGOVLP_CHECK_ARG(!off(e->bias, 8) && !off(e->residual, 8) && !off(e->colsum, 8) && (e->out_mode == 0 || !off(e->out, 8)),
                   "gemm: bias, residual, colsum and an fp32 out must be 8-byte aligned");
  EGOVLP_CHECK_ARG(!off(e->aux, 4) && !off(e->out2, 4) && (e->out_mode != 0 || !off(e->out, 4)),
                   "gemm: aux, out2 and a bf16 out must be 4-byte aligned");
  EGOVLP_CHECK_ARG((!e->residual || e->ldr % 2 == 0) && (!e->aux || e->ldaux % 2 == 0) && (!e->out2 || e->ldo2 % 2 == 0),
                   "gemm: ldr, ldaux and ldo2 must be even");
  EpiParams ep;
  ep.bias = e->bias; ep.residual = e->residual; ep.aux = reinterpret_cast<const bf16*>(e->aux);
  ep.out = e->out; ep.out2 = reinterpret_cast<bf16*>(e->out2);
  ep.ldr = e->ldr; ep.ldaux = e->ldaux; ep.ldo = e->ldo; ep.ldo2 = e->ldo2;
  ep.out_mode = e->out_mode; ep.act = e->act; ep.alpha = e->alpha;
  ep.col_scale = e->col_scale; ep.col_scale_ncols = e->col_scale_ncols; ep.res_row_mod = e->res_row_mod;
  ep.colsum = e->colsum;
  ep.colsum_a = e->colsum_a;
  ep.row_scale = ep.w_scale = nullptr;
  ep.det_ws = ep.det_cs = nullptr;
  if (e->det_ws) {
    // deterministic form: partials to the workspace, merged in a fixed order (see egovlp_gemm_det_workspace_floats)
    EGOVLP_CHECK_ARG(!e->colsum, "gemm: the output column sums (colsum) have no deterministic form");
    EGOVLP_CHECK_ARG((reinterpret_cast<uintptr_t>(e->det_ws) & 15) == 0, "gemm: det_ws must be 16B aligned");
    const DetLayout dl = det_layout(M, N, K, max(split_k, 1));
    if (e->out_mode == 2) ep.det_ws = e->det_ws;
    if (e->colsum_a) ep.det_cs = e->det_ws + (long long)dl.splits * dl.Mp * N;
  }
  EGOVLP_CHECK_ARG(!e->colsum_a || (a_mn_major && b_mn_major && N % 256 == 0 && M % 8 == 0 &&
                                    (reinterpret_cast<uintptr_t>(e->colsum_a) & 15) == 0),
                   "gemm: colsum_a needs the MN/MN (wgrad) form with N % 256 == 0, M % 8 == 0 and a 16B-aligned vector");
  EGOVLP_CHECK_ARG(e->drop_p >= 0.f && e->drop_p < 1.f && e->path_p >= 0.f && e->path_p < 1.f && e->path_rows >= 0,
                   "gemm: dropout rates must lie in [0, 1) (drop_p=%f path_p=%f), path_rows >= 0", e->drop_p, e->path_p);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (e->drop_p > 0.f || e->path_rows > 0) {
    EGOVLP_CHECK_ARG(split_k <= 1, "gemm: dropout with split_k > 1");
    const DropParams dp = {e->drop_seed, e->drop_p, e->path_p, e->drop_site, e->path_site, e->path_rows};
    if (N % 256 == 0) return dispatch_drop<256>(a_mn_major, b_mn_major, A, lda, B, ldb, M, N, K, ep, dp, st);
    return dispatch_drop<128>(a_mn_major, b_mn_major, A, lda, B, ldb, M, N, K, ep, dp, st);
  }
  if (N % 256 == 0 && !a_mn_major && !e->det_ws && use_pairs())
    return dispatch_mode<256, true>(a_mn_major, b_mn_major, A, lda, B, ldb, M, N, K, split_k, ep, st);
  if (N % 256 == 0) return dispatch_mode<256, false>(a_mn_major, b_mn_major, A, lda, B, ldb, M, N, K, split_k, ep, st);
  return dispatch_mode<128, false>(a_mn_major, b_mn_major, A, lda, B, ldb, M, N, K, split_k, ep, st);
}

extern "C" long long egovlp_gemm_det_workspace_floats(int M, int N, int K, int split_k) {
  if (M <= 0 || N <= 0 || K <= 0) return -1;
  return det_layout(M, N, K, max(split_k, 1)).floats;
}

extern "C" int egovlp_gemm_e4m3(const void* A8, long long lda, const void* B8, long long ldb, const float* row_scale,
                                const float* col_scale, int M, int N, int K, const egovlp_gemm_epilogue* e,
                                void* stream) {
  EGOVLP_CHECK_ARG(A8 && B8 && row_scale && col_scale && e && e->out, "gemm_e4m3: null pointer");
  EGOVLP_CHECK_ARG(M > 0 && N > 0 && K > 0 && N % 128 == 0 && K % 16 == 0,
                   "gemm_e4m3: bad shape M=%d N=%d K=%d (N %% 128 == 0 and K %% 16 == 0 needed)", M, N, K);
  EGOVLP_CHECK_ARG(lda >= K && ldb >= K && lda % 16 == 0 && ldb % 16 == 0,
                   "gemm_e4m3: leading dimensions must be >= K and multiples of 16 (16B TMA strides)");
  EGOVLP_CHECK_ARG(((reinterpret_cast<uintptr_t>(A8) | reinterpret_cast<uintptr_t>(B8) |
                     reinterpret_cast<uintptr_t>(col_scale)) & 15) == 0,
                   "gemm_e4m3: operands and column scales must be 16B aligned");
  EGOVLP_CHECK_ARG(e->out_mode == 0 && (e->act == 0 || e->act == 1) && !e->residual && !e->aux && !e->out2 &&
                       !e->colsum && !e->colsum_a && !e->res_row_mod && (e->act == 0 || e->col_scale_ncols == 0),
                   "gemm_e4m3: only the bf16 store (act 0, optional column scale) and GELU (act 1) epilogues");
  EGOVLP_CHECK_ARG(tma_ok(e->out, e->ldo * 2) && (reinterpret_cast<uintptr_t>(e->bias) & 15) == 0,
                   "gemm_e4m3: out and bias must be 16B aligned, ldo a multiple of 8");
  EpiParams ep = {};
  ep.bias = e->bias; ep.out = e->out; ep.ldo = e->ldo; ep.out_mode = 0; ep.act = e->act; ep.alpha = e->alpha;
  ep.col_scale = e->col_scale; ep.col_scale_ncols = e->col_scale_ncols;
  ep.row_scale = row_scale; ep.w_scale = col_scale;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (N % 256 == 0) {
    if (e->act == 1) return launch<256, false, false, false, EPI_ACT1, true>(A8, lda, B8, ldb, M, N, K, 1, ep, st);
    return launch<256, false, false, false, EPI_BF16, true>(A8, lda, B8, ldb, M, N, K, 1, ep, st);
  }
  if (e->act == 1) return launch<128, false, false, false, EPI_ACT1, true>(A8, lda, B8, ldb, M, N, K, 1, ep, st);
  return launch<128, false, false, false, EPI_BF16, true>(A8, lda, B8, ldb, M, N, K, 1, ep, st);
}
