// Text-tower self-attention for long captions (128 < L <= 512; any L in 1..512 is accepted): the tiled attention of
// tiled_attention.cuh with a key-padding mask and in-kernel attention dropout, forward and backward.
//
// Same contract as text_attn_* (text.cu): qkv bf16 [B*L, 3D] read in place (q pre-scaled by the QKV GEMM epilogue),
// attention_mask int64 [B, L] (0 = padded key, any 0/1 pattern), out bf16 [B*L, D] with the heads merged.  Head dim 64.
//
// A group is (sample, head): row r is matrix row b*L + r, and lse / delta are fp32 [B, H, L].  The CTA builds a bitmap
// of its sample's valid keys in the prologue and skips every 64-key tile without one -- in the forward and in both
// backward passes -- so a batch padded to 512 for one long caption costs what its valid key tiles cost.  A sample
// without any valid key gets NaN out and lse rows, as the L <= 128 kernel gives them.
//
// Dropout keep mask (HF DistilBERT: `weights = dropout(softmax(scores))`): element (b, h, i, j) is kept iff word
// (j & 3) of philox4x32_10(dropout_key(seed, site), ((b * 4096 + h) * 512 + i) * 128 + (j >> 2)) is
// >= dropout_threshold(p).  One Philox call serves four consecutive keys; the mask does not depend on B, H or L.
#include "egovlp_b200.h"
#include "tiled_attention.cuh"

namespace egovlp {
namespace {

constexpr int MAX_L = 512;

// ---- dropout ----
struct Drop {
  bool on;
  uint32_t thresh;
  float inv_keep;
  unsigned long long key;
};
__device__ __forceinline__ Drop make_drop(float p, unsigned long long seed, uint32_t site) {
  return Drop{p > 0.f, dropout_threshold(p), p > 0.f ? 1.f / (1.f - p) : 1.f, dropout_key(seed, site)};
}

// The layout policy of tiled_attention.cuh for a (sample, head) group under a key-padding mask.
struct TextAttn {
  struct Args {
    const long long* mask;
    int L, H;
    float p_drop;
    unsigned long long seed;
    uint32_t site;
  };
  struct Smem {
    uint32_t kb[MAX_L / 32];   // bit j of kb[j >> 5]: key j is valid (bits >= L are 0)
  };
  static constexpr bool kCls = false, kDropout = true;

  const long long* mask;
  uint32_t* kb;
  int b, h, H, L, rows;
  Drop drop;

  __device__ TextAttn(const Args& a, int h_, Smem& sm)
      : mask(a.mask), kb(sm.kb), b(blockIdx.z), h(h_), H(a.H), L(a.L), rows(a.L),
        drop(make_drop(a.p_drop, a.seed, a.site)) {}
  __device__ long long row(int r) const { return (long long)b * L + r; }
  __device__ long long stat(int r) const { return ((long long)b * H + h) * L + r; }

  // fills kb; the 64-key tiles with a valid key
  __device__ uint32_t key_tiles() const {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int j0 = warp * 32; j0 < MAX_L; j0 += NTHREADS) {
      const int j = j0 + lane;
      const uint32_t w = __ballot_sync(0xffffffffu, j < L && mask[(long long)b * L + j] != 0);
      if (lane == 0) kb[j0 >> 5] = w;
    }
    __syncthreads();
    uint32_t tiles = 0;
#pragma unroll
    for (int kt = 0; kt < MAX_L / TILE; ++kt)
      if (kb[2 * kt] | kb[2 * kt + 1]) tiles |= 1u << kt;
    return tiles;
  }
  __device__ bool masked(int) const { return true; }
  __device__ uint32_t key_bits(int kt, int jl, int t) const { return kb[2 * kt + (jl >> 5)] >> ((jl & 31) + 2 * t); }
  __device__ bool key_ok(int j) const { return (kb[j >> 5] >> (j & 31)) & 1u; }
  __device__ bool skips_pair00() const { return false; }

  // keep bits of keys 4*jg .. 4*jg+3 of row i (bit w = key 4*jg + w)
  __device__ uint32_t keep4(int i, int jg) const {
    const uint4 r = philox4x32_10(drop.key, (((unsigned long long)b * 4096ull + h) * 512ull + i) * 128ull + jg);
    return (uint32_t)(r.x >= drop.thresh) | ((uint32_t)(r.y >= drop.thresh) << 1) |
           ((uint32_t)(r.z >= drop.thresh) << 2) | ((uint32_t)(r.w >= drop.thresh) << 3);
  }
  // Keep bits of one m16n8 accumulator with rows = queries i0.. (16) and columns = keys j0.. (8, j0 % 8 == 0), as
  // bits 0..3 in the order of the fragment's c[0..3]: lane computes (row lane & 15, key group lane >> 4) and the quad
  // fetches its two rows' nibbles.
  __device__ uint32_t keep_qk(int i0, int j0, int lane) const {
    const uint32_t nib = keep4(i0 + (lane & 15), (j0 >> 2) + (lane >> 4));
    const int gq = lane >> 2, t = lane & 3, src = gq + 16 * (t >> 1), sh = 2 * (t & 1);
    const uint32_t n0 = __shfl_sync(0xffffffffu, nib, src), n1 = __shfl_sync(0xffffffffu, nib, src + 8);
    return ((n0 >> sh) & 3u) | (((n1 >> sh) & 3u) << 2);
  }
  // The same with rows = keys j0.. (16, j0 % 4 == 0) and columns = queries i0.. (8): lane computes (query lane & 7,
  // key group lane >> 3).
  __device__ uint32_t keep_kq(int j0, int i0, int lane) const {
    const uint32_t nib = keep4(i0 + (lane & 7), (j0 >> 2) + (lane >> 3));
    const int gq = lane >> 2, t = lane & 3, w = gq & 3, s0 = (gq >> 2) * 8 + 2 * t, s1 = s0 + 16;
    const uint32_t a = __shfl_sync(0xffffffffu, nib, s0), bb = __shfl_sync(0xffffffffu, nib, s0 + 1);
    const uint32_t c = __shfl_sync(0xffffffffu, nib, s1), e = __shfl_sync(0xffffffffu, nib, s1 + 1);
    return ((a >> w) & 1u) | (((bb >> w) & 1u) << 1) | (((c >> w) & 1u) << 2) | (((e >> w) & 1u) << 3);
  }
};

}  // namespace
}  // namespace egovlp

using namespace egovlp;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int egovlp_text_attn_long_fwd(const void* qkv, const long long* attention_mask, void* out, float* lse, int B,
                                         int L, int H, float p_drop, unsigned long long seed, unsigned int site,
                                         void* stream) {
  EGOVLP_CHECK_ARG(qkv && attention_mask && out && lse, "text_attn_long_fwd: null pointer");
  EGOVLP_CHECK_ARG(B > 0 && B <= 65535 && H > 0 && H <= 4096, "text_attn_long_fwd: B=%d H=%d unsupported", B, H);
  EGOVLP_CHECK_ARG(L > 0 && L <= MAX_L, "text_attn_long: L=%d unsupported (1..512)", L);
  EGOVLP_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, "text_attn_long: p_drop=%f outside [0, 1)", p_drop);
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(tiled_attn_fwd_kernel<TextAttn>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)FWD_SMEM));
  const dim3 grid((L + TILE - 1) / TILE, H, B);
  tiled_attn_fwd_kernel<TextAttn><<<grid, NTHREADS, FWD_SMEM, ST(stream)>>>(
      reinterpret_cast<const bf16*>(qkv), reinterpret_cast<bf16*>(out), lse,
      TextAttn::Args{attention_mask, L, H, p_drop, seed, site});
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

extern "C" int egovlp_text_attn_long_bwd(const void* qkv, const long long* attention_mask, const void* out,
                                         const float* lse, const void* dout, void* dqkv, float* workspace, int B,
                                         int L, int H, float q_scale, float p_drop, unsigned long long seed,
                                         unsigned int site, void* stream) {
  EGOVLP_CHECK_ARG(qkv && attention_mask && out && lse && dout && dqkv && workspace,
                   "text_attn_long_bwd: null pointer");
  EGOVLP_CHECK_ARG(B > 0 && B <= 65535 && H > 0 && H <= 4096, "text_attn_long_bwd: B=%d H=%d unsupported", B, H);
  EGOVLP_CHECK_ARG(L > 0 && L <= MAX_L, "text_attn_long: L=%d unsupported (1..512)", L);
  EGOVLP_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, "text_attn_long: p_drop=%f outside [0, 1)", p_drop);
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(tiled_attn_bwd_kv_kernel<TextAttn>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM));
  EGOVLP_CHECK_CUDA(cudaFuncSetAttribute(tiled_attn_bwd_q_kernel<TextAttn>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)BWD_SMEM));
  const bf16* q = reinterpret_cast<const bf16*>(qkv);
  const bf16* o = reinterpret_cast<const bf16*>(out);
  const bf16* g = reinterpret_cast<const bf16*>(dout);
  bf16* dq = reinterpret_cast<bf16*>(dqkv);
  const TextAttn::Args a{attention_mask, L, H, p_drop, seed, site};
  const long long nthr = (long long)B * L * H * 8;
  tiled_attn_delta_kernel<<<(unsigned)((nthr + 255) / 256), 256, 0, ST(stream)>>>(o, g, workspace, (long long)B * L, L,
                                                                                   H);
  EGOVLP_CHECK_LAUNCH();
  const dim3 grid((L + TILE - 1) / TILE, H, B);
  tiled_attn_bwd_kv_kernel<TextAttn><<<grid, NTHREADS, BWD_SMEM, ST(stream)>>>(q, lse, workspace, g, dq, a);
  EGOVLP_CHECK_LAUNCH();
  tiled_attn_bwd_q_kernel<TextAttn><<<grid, NTHREADS, BWD_SMEM, ST(stream)>>>(q, lse, workspace, g, dq, q_scale, a);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
