/* egovlp_b200 — C-ABI of the H100-native (sm_90a) EgoVLP hot path (libegovlp_b200.so).
 *
 * The reference (showlab/EgoVLP) has no FFI layer: its hot path is Python over torch ops
 * (SURVEY.md section 8b).  This header is the boundary a maintainer binds instead of those torch
 * ops: plain device pointers, sizes and a CUstream/cudaStream_t passed as void*.  Every entry point
 * cites the reference call site(s) it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless named host_*; the caller owns every buffer; kernels
 *     never allocate or free; work is enqueued on `stream` and the call returns immediately.
 *   - return 0 on success, <0 on error (EGOVLP_ERR_*); egovlp_last_error() gives the message
 *     (thread-local).  No global state except per-process function attributes.
 *   - bf16 = __nv_bfloat16 bit pattern (uint16_t); "row-major [R, C] ld" = element (r,c) at r*ld+c.
 *   - token layout of the video tower: x[b, s, :] with s = 0 the CLS token and s = 1 + f*N + n the
 *     patch n of frame f (frame-major), exactly the reference's (model/video_transformer.py:305-310).
 */
#ifndef EGOVLP_B200_H_
#define EGOVLP_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EGOVLP_ERR_ARG (-1)
#define EGOVLP_ERR_CUDA (-2)
#define EGOVLP_ERR_UNSUPPORTED (-3)

const char* egovlp_last_error(void);
/* ABI version of this header; bumped on any signature change. */
int egovlp_abi_version(void);

/* ------------------------------------------------------------------------------------------------
 * GEMM  D[m,n] = epi( sum_k A[m,k] * B[n,k] ),  bf16 operands, fp32 accumulation (wgmma).
 * Replaces nn.Linear forward/backward everywhere on the path: model/video_transformer.py:41-52
 * (Mlp), :88-89,103,135 (qkv/proj), :70,76 (patch-embed conv as GEMM); DistilBERT q/k/v/out_lin,
 * ffn.lin1/lin2; model/model.py:72-79 (projections); and autograd's dgrad/wgrad of each.
 *   a_mn_major = 0: A stored [M, K] (ld = lda);  1: A stored [K, M] (m contiguous)
 *   b_mn_major = 0: B stored [N, K] (ld = ldb);  1: B stored [K, N] (n contiguous)
 * Epilogue, applied in this order to v = alpha * acc:
 *   v += bias[n];  if (n < col_scale_ncols) v *= col_scale;  out2[m,n] = bf16(v) (if out2);
 *   act 1: v = gelu_erf(v)   act 2: v *= gelu_erf'(aux[m,n]);
 *   act 3: out2[m,n] = bf16(gelu_erf'(v)) (instead of v), then v = gelu_erf(v)   act 4: v *= aux[m,n]
 *          (3 + 4 = the Mlp pair, model/video_transformer.py:46-52: fc1 saves the GELU derivative, the fc2 input-gradient
 *          GEMM only multiplies by it);
 *   act 5: z = aux[m,n]: out2[m,n] = bf16(gelu_erf(z)) (instead of v), then v *= gelu_erf'(z)
 *          (1 with out2 + 5 = the low-memory Mlp pair: fc1 saves the pre-activation z, and the fc2 input-gradient GEMM
 *          also rebuilds gelu(z), the fc2 weight gradient's operand);   v += residual[m,n] (fp32);
 *   out_mode 0: out(bf16) = v;  1: out(fp32) = v;  2: atomicAdd(out(fp32), v) (needed for split_k>1)
 * Constraints: N % 32 == 0, lda/ldb/ldo % 8 == 0, ldr/ldaux/ldo2 even; A and B 16B-aligned, bias / residual / colsum /
 * an fp32 out 8B-aligned, aux / out2 / a bf16 out 4B-aligned (EGOVLP_ERR_ARG otherwise).
 * The library chooses the kernel instance itself (tile scheduler, compile-time specialised epilogue for the common
 * descriptor forms); every instance computes the arithmetic above in the same order, so the choice never changes a bit of
 * the result (tests/test_kernels_gpu.py::test_gemm_specialised_epilogues_match_the_generic_one).
 */
typedef struct egovlp_gemm_epilogue {
  const float* bias;     /* [N] fp32 or NULL */
  const float* residual; /* [M, ldr] fp32 or NULL */
  const void* aux;       /* [M, ldaux] bf16, for act == 2 / 4 / 5 */
  void* out;             /* [M, ldo] bf16 (out_mode 0) or fp32 (1, 2) */
  void* out2;            /* [M, ldo2] bf16 or NULL */
  long long ldr, ldaux, ldo, ldo2;
  int out_mode;
  int act;
  float alpha;
  float col_scale;
  int col_scale_ncols;
  int res_row_mod; /* 0: residual row = m; >0: residual row = m % res_row_mod (broadcast [res_row_mod, ldr] table) */
  float* colsum;   /* optional fp32 [N]: ACCUMULATES the column sums of the stored values (bias gradient of dy) */
  float* colsum_a; /* optional fp32 [M], only with a_mn_major && b_mn_major (the token-contraction weight gradient
                      dW = dy^T x): ACCUMULATES sum_k A[k, m] = the bias gradient of the same Linear, summed from the
                      A tiles while they sit in shared memory for the MMA (no extra pass over dy) */
  /* Dropout (the video tower's training forms), active when drop_p > 0 or path_rows > 0: the value v that would be
   * stored (act 0 + residual: the value before the residual is added; act 1 / 3: gelu_erf(v), not out2; act 4: the
   * product; act 5: both out and out2) is multiplied by keep(m, n) / (1 - drop_p) x f(m / path_rows).  keep(m, n) = 1
   * iff word (n & 3) of philox4x32_10(key(drop_seed, drop_site), m * (N / 4) + n / 4) >= drop_p * 2^32 -- the mask
   * egovlp_dropout draws over the [M, N] output, whatever the tiling; f(b) = the drop-path factor of sample b: 1 / (1 -
   * path_p) if word (b & 3) of philox4x32_10(key(drop_seed, path_site), b / 4) >= path_p * 2^32, else 0 (f = 1 when
   * path_rows = 0).  Only five forms take it: act 0 + residual + out_mode 1, act 1 / 3 with out2 (K-major A and B),
   * act 4 / 5 (K-major A, MN-major B); other descriptors return EGOVLP_ERR_UNSUPPORTED.  Rates in [0, 1).
   * The library reads every field of the struct: zero-initialise it (e.g. `egovlp_gemm_epilogue e = {0};`) so that
   * the fields a caller does not use, these included, select nothing. */
  float drop_p;
  unsigned int drop_site;
  unsigned long long drop_seed;
  float path_p;
  unsigned int path_site;
  int path_rows;
  /* Deterministic form (NULL: off), for out_mode 2 and / or colsum_a: an fp32 workspace of
   * egovlp_gemm_det_workspace_floats(M, N, K, split_k) floats, 16B aligned.  Each split s stores its partial tile P_s
   * (the products of its k-blocks, times alpha) to the workspace, and an ordered pass then computes
   * out = ((out + P_0) + P_1) + ... + P_{s-1} in fp32; colsum_a gets the same treatment, its per-split partial being
   * the sum of its n-block partials in n-block order (a split's k-blocks are shared among the n-blocks counting from
   * the split's first).  The result depends on the operands, M, N, K and split_k only: a split's partial equals the
   * output of a one-split GEMM over that split's rows of A and B.  Not with colsum (EGOVLP_ERR_ARG). */
  float* det_ws;
} egovlp_gemm_epilogue;

int egovlp_gemm_bf16(const void* A, int a_mn_major, long long lda, const void* B, int b_mn_major, long long ldb,
                     int M, int N, int K, const egovlp_gemm_epilogue* epi, int split_k, void* stream);
/* Workspace of the deterministic form: splits' * Mp * N + splits' * nb * Mp floats, splits' = the split count after
 * empty splits are dropped, Mp = M rounded up to 128, nb = N / 256 when N % 256 == 0, else ceil(N / 128). */
long long egovlp_gemm_det_workspace_floats(int M, int N, int K, int split_k);
/* e4m3 inference form of the same GEMM (the video tower's LayerNorm-fed qkv and Mlp.fc1 GEMMs, opt-in,
 * SpaceTimeTransformer.set_inference_precision("fp8")):
 *   D[m,n] = epi( (sum_k A8[m,k] * B8[n,k]) * row_scale[m] * col_scale[n] )
 * A8 [M, lda] and B8 [N, ldb] are e4m3 (e4m3fn bytes), both K-major; row_scale fp32 [M], col_scale fp32 [N] (16B
 * aligned).  fp32 accumulation in the e4m3 wgmma.  Only two epilogues: act 0 with out_mode 0 (bias, optional column
 * scale, bf16 out; the qkv form) and act 1 with out_mode 0 (bias, GELU, bf16 out; fc1).  No residual, aux, out2, column
 * sums or split-K.  Constraints: N % 128 == 0, K % 16 == 0, lda / ldb >= K and multiples of 16, 16B-aligned bases. */
int egovlp_gemm_e4m3(const void* A8, long long lda, const void* B8, long long ldb, const float* row_scale,
                     const float* col_scale, int M, int N, int K, const egovlp_gemm_epilogue* epi, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LayerNorm over the last dim (nn.LayerNorm; model/video_transformer.py:146,156,159,228,253 eps 1e-6;
 * DistilBERT sa_layer_norm/output_layer_norm/embeddings.LayerNorm eps 1e-12).
 * x fp32 [rows, D] (row stride ldx) -> y bf16 [rows, D] and/or y32 fp32 [rows, D]; mean/rstd fp32 [rows]
 * are saved for the backward.  Optional fused residual: x_eff = x + add (fp32 [rows, D]), and x_eff is
 * written to sum_out (post-LN DistilBERT: LN(sa + x)).  D % 4 == 0 and D <= 1024.
 */
int egovlp_layernorm_fwd(const float* x, long long ldx, const float* add, float* sum_out, const float* gamma,
                         const float* beta, void* y_bf16, float* y_f32, float* mean, float* rstd, int rows, int D,
                         float eps, void* stream);
/* The same forward (no fused add) that also writes the normalised row as the A operand of egovlp_gemm_e4m3:
 * y8 e4m3 [rows, D] (contiguous, 4B aligned) = y * (448 / amax) rounded to nearest with saturation, row_scale fp32
 * [rows] = amax / 448, amax = max |y| over the row of fp32 outputs (scale 1 for a row of zeros).  y_bf16 / y_f32 /
 * mean / rstd may each be NULL and are bit-identical to egovlp_layernorm_fwd's.  256 < D <= 1024. */
int egovlp_layernorm_fwd_e4m3(const float* x, long long ldx, const float* gamma, const float* beta, void* y_bf16,
                              float* y_f32, float* mean, float* rstd, uint8_t* y8, float* row_scale, int rows, int D,
                              float eps, void* stream);
/* Backward.  dx = LNbwd(dy) [+ add1] [+ add2]  (fp32 [rows, D], row stride lddx), optionally also stored as bf16
 * (dx_bf16, row stride D) for use as a GEMM operand.  add1/add2 carry the residual-stream gradients that bypass the LN
 * (SpaceTimeBlock: dsr = dy + LN2bwd, dx = dsr + dtr + LN3bwd).  dgamma/dbeta (fp32 [D]) are ACCUMULATED
 * with atomicAdd -- zero them first for a plain gradient; either may be NULL.  dy, add1 and add2 are each fp32 or
 * bf16 (the *_is_bf16 flags; add rows are dense, stride D).  colsum_dx (fp32 [D], optional) ACCUMULATES the
 * column sums of the result: the bias gradient of the Linear that produced the normalised tensor's residual. */
int egovlp_layernorm_bwd(const void* dy, int dy_is_bf16, long long lddy, const float* x, long long ldx,
                         const float* gamma, const float* mean, const float* rstd, const void* add1, int add1_is_bf16,
                         const void* add2, int add2_is_bf16, float* dx, long long lddx, void* dx_bf16, float* dgamma,
                         float* dbeta, float* colsum_dx, int rows, int D, void* stream);
/* Deterministic form of the backward: the same outputs, with each CTA's dgamma / dbeta / colsum_dx partials stored to
 * ws (egovlp_layernorm_bwd_det_workspace_floats(rows, D) floats) and added into the outputs in CTA order by a second
 * kernel.  The grid is sized for 132 SMs on every card, and the kernel (so the partition, and with it the bits of the
 * sums) is chosen from the shapes, the strides and whether dy, x, add1 and add2 are 16-byte aligned: the pipelined
 * kernel takes rows >= 4096, D % 128 == 0, dense rows and 16-byte aligned bases; anything else the other one. */
long long egovlp_layernorm_bwd_det_workspace_floats(int rows, int D);
int egovlp_layernorm_bwd_det(const void* dy, int dy_is_bf16, long long lddy, const float* x, long long ldx,
                             const float* gamma, const float* mean, const float* rstd, const void* add1, int add1_is_bf16,
                             const void* add2, int add2_is_bf16, float* dx, long long lddx, void* dx_bf16, float* dgamma,
                             float* dbeta, float* colsum_dx, int rows, int D, float* ws, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Divided space-time attention core of VarAttention.forward (model/video_transformer.py:104-133) and its
 * autograd.  Head dim must be 64 (D = 64*H).  mode 0 = time ('b (f n) d -> (b n) f d'), 1 = space ('(b f) n d').
 *   qkv   bf16 [B*S, 3*D], S = 1 + T*N, columns [q | k | v] each (head, 64); q ALREADY scaled by 64^-0.5
 *         (the QKV GEMM epilogue applies it, :106)
 *   out   bf16 [B*S, D]  = cat(cls_out, attended patches) with heads merged (:130-133), ready for proj
 *   lse   fp32 [B, H, S] log-sum-exp of every query row (saved for the backward)
 *   cls_part fp32 workspace of egovlp_divided_attn_workspace_floats() floats (CLS-query partials)
 * Semantics kept from the reference: the CLS query attends over ALL S keys (:112); every patch query attends
 * over its group's keys plus the CLS key/value (:117-124).
 * Backward: dqkv bf16 [B*S, 3*D] receives d(q_prescale), dk, dv for every token (q gradient multiplied by
 * q_scale); dcls_ws is an fp32 workspace of B*H*3*64 floats (zeroed internally).
 */
long long egovlp_divided_attn_workspace_floats(int B, int T, int N, int H, int mode);
int egovlp_divided_attn_fwd(const void* qkv, void* out, float* lse, float* cls_part, int B, int T, int N, int H,
                            int mode, void* stream);
int egovlp_divided_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                            float* dcls_ws, int B, int T, int N, int H, int mode, float q_scale, void* stream);
/* Deterministic form of the backward: every CTA stores its CLS-row dq / dk / dv into a slot of its own (dcls_ws, of
 * egovlp_divided_attn_bwd_det_workspace_floats() floats: [B, H, groups, parts, 3, 64], parts = 4 in the T in
 * {4, 8, 16} time kernel, else 1), summed in group, then part, order.  The kernel follows from the geometry alone. */
long long egovlp_divided_attn_bwd_det_workspace_floats(int B, int T, int N, int H, int mode);
int egovlp_divided_attn_bwd_det(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                                float* dcls_ws, int B, int T, int N, int H, int mode, float q_scale, void* stream);
/* Spatial attention for large frames: egovlp_divided_attn_{fwd,bwd} with mode = 1 (model/video_transformer.py:109-130,
 * space mode), for 1 <= N <= 1024 patches per frame (the divided attention stops at N = 255; the engine uses these
 * above that).  Same qkv / out / lse / dqkv layouts and semantics; tiled on the tensor cores (bf16 mma.sync, fp32
 * online softmax, 64-row tiles of a frame's rows behind the CLS row).  workspace: fp32, at least
 * egovlp_space_attn_long_workspace_floats() floats, shared by the forward and the backward (CLS-row partials; the
 * backward's delta = rowsum(dO * O)).  No floating-point atomics: out, lse and dqkv, the CLS rows included, are
 * bitwise reproducible, and a sample's results do not depend on the others in the batch.  Indexing is 64-bit.
 * Refused (EGOVLP_ERR_ARG, nothing written): a null pointer, N outside [1, 1024], B, T or H < 1, B*T or H > 65535.
 * The workspace query returns -1 for such a shape. */
long long egovlp_space_attn_long_workspace_floats(int B, int T, int N, int H);
int egovlp_space_attn_long_fwd(const void* qkv, void* out, float* lse, float* workspace, int B, int T, int N, int H,
                               void* stream);
int egovlp_space_attn_long_bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                               float* workspace, int B, int T, int N, int H, float q_scale, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Video patch-embedding front end (model/video_transformer.py:72-77, 304-321).
 *   egovlp_patch_im2col: video fp32 [B,T,C,H,W] -> patches bf16 [B*S, C*P*P] (row b*S+1+t*N+n, CLS rows zero),
 *     the A operand of the conv-as-GEMM against patch_embed.proj.weight viewed [D, C*P*P].
 *   egovlp_video_pos_table: table fp32 [S, D] added by that GEMM's epilogue (res_row_mod = S):
 *     row 0 = cls_token + pos_embed[0] - conv_bias, row 1+t*N+n = pos_embed[1+n] + temporal_embed[t].
 *   egovlp_video_embed_bwd: from dx fp32 [B,S,D] ACCUMULATE dcls[D], dpos[(1+N),D], dtemporal[T,D] (first T rows)
 *     and the conv bias gradient dbias[D]; tmp_SD is an fp32 workspace of S*D floats.
 */
int egovlp_patch_im2col(const float* video, void* patches_bf16, int B, int T, int C, int H, int W, int P, void* stream);
/* uint8 frames [B,T,3,H,W] with the dataset normalisation (data_loader/transforms.py:38-41) fused:
 * v = (p/255 - mean[c]) / std[c]; host_mean3 / host_std3 are HOST arrays of 3 floats. */
int egovlp_patch_im2col_u8(const uint8_t* video, void* patches_bf16, int B, int T, int C, int H, int W, int P,
                           const float* host_mean3, const float* host_std3, void* stream);
/* Dataset video transforms from decoded uint8 frames (replaces, per clip, the reader's `.float() / 255`
 * (base/base_dataset.py:220-243 and the EgoClip / EPIC / Charades readers), the `init_video_transform_dict` transform
 * (data_loader/transforms.py:34-61) and the zero-padded `final` copy (base/base_dataset.py:117-140)).
 *   frames: packed uint8, clip b channels-last [T_b, H_b, W_b, 3] at byte offset desc[b][0]; frames_bytes its size.
 *   desc: int64 [B, 10] rows (offset, T, H, W, mode, i, j, h, w, flip); mode 0 = train: bilinear resize (no antialias) of
 *         the crop box rows [i, i + h) x cols [j, j + w) to R x R, then flip != 0 reverses the output columns;
 *         mode 1 = eval: Resize(center_crop) (short side), CenterCrop(center_crop), Resize(R), both antialiased;
 *         (i, j, h, w, flip) unused.  T <= F, H, W <= 65535.
 *   out: fp32 [B, F, 3, R, R] = (resampled p / 255 - mean[c]) / std[c]; frames t >= T are 0.0.  R <=
 *        egovlp_video_transform_max_res(); the eval weights of one output index may span at most
 *        egovlp_video_transform_max_taps() source pixels per axis (short side up to ~7 x center_crop at 256 -> 224).
 *   host_mean / host_std: HOST arrays of 3 floats.
 * The descriptor table is not checked on the host here (it is device memory): the caller validates it.  A row that
 * would read outside `frames` is not read; its outputs become NaN. */
int egovlp_video_transform_max_taps(void);
int egovlp_video_transform_max_res(void);
int egovlp_video_transform(const uint8_t* frames, long long frames_bytes, const long long* desc, int B, int F, int R,
                           int center_crop, const float* host_mean, const float* host_std, float* out, void* stream);
int egovlp_video_pos_table(const float* cls_token, const float* pos_embed, const float* temporal_embed,
                           const float* conv_bias, float* table, int T, int N, int D, void* stream);
int egovlp_video_embed_bwd(const float* dx, float* tmp_SD, float* dcls, float* dpos, float* dtemporal, float* dbias,
                           int B, int T, int N, int D, void* stream);
/* Deterministic form: the per-frame partials of dbias go to ws_TD (fp32 [T, D]) and are added in frame order. */
int egovlp_video_embed_bwd_det(const float* dx, float* tmp_SD, float* dcls, float* dpos, float* dtemporal, float* dbias,
                               float* ws_TD, int B, int T, int N, int D, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Text tower pieces (DistilBERT; call sites model/model.py:117-138).  ids / attention_mask are int64 as the
 * HuggingFace tokenizer returns them.  Head dim 64; L <= 128 for text_attn_*, L <= 512 for text_attn_long_*.
 *   text_embed_fwd : out fp32 [B*L, D] = word_emb[ids] + pos_emb[l]   (LayerNorm follows via egovlp_layernorm_fwd;
 *                    the caller guarantees L <= rows of pos_emb)
 *   text_embed_bwd : dword[ids] += dsum, dpos[l] += dsum  (atomic accumulate)
 *   text_attn_fwd  : out bf16 [B*L, D] = softmax(q k^T + key-padding mask) v per (b, head); qkv bf16 [B*L, 3D],
 *                    q pre-scaled by 64^-0.5
 *   text_attn_bwd  : dqkv bf16 [B*L, 3D]  (dq multiplied by q_scale)
 *                    p_drop / seed / site: attention dropout on the probabilities as HuggingFace DistilBERT applies it
 *                    in train mode (transformers modeling_distilbert.py, `weights = self.dropout(weights)`), mask
 *                    drawn from a counter-based Philox4x32-10 keyed by (seed, site) and indexed by (b, head, i, j);
 *                    the backward must be given the forward's (p_drop, seed, site).  p_drop = 0 disables it.
 *   text_attn_long_fwd : the same attention for 1 <= L <= 512 (the text tower uses it above L = 128), tiled on the
 *                    tensor cores (bf16 mma.sync, fp32 online softmax); 64-key tiles without a valid key are skipped.
 *                    Also writes lse fp32 [B, H, L] (natural log of each row's softmax denominator, scores included),
 *                    which the backward needs.  A sample whose mask is all zero gets NaN rows in out and lse.
 *   text_attn_long_bwd : dqkv bf16 [B*L, 3D] (dq multiplied by q_scale; dk = dv = 0 for padded keys) from the
 *                    forward's out and lse; workspace fp32 [B*H*L].  No floating-point atomics: bitwise reproducible.
 *                    A sample whose mask is all zero gets dqkv = 0.
 *                    Dropout as for text_attn, but the keep mask is its own stream: (b, h, i, j) is kept iff word
 *                    (j & 3) of philox4x32_10(key(seed, site), ((b * 4096 + h) * 512 + i) * 128 + (j >> 2)) is
 *                    >= p_drop * 2^32 (one Philox call per four keys; independent of B, H and L).
 *                    Refused (EGOVLP_ERR_ARG, nothing written): a null pointer, L outside [1, 512], B outside
 *                    [1, 65535], H outside [1, 4096], p_drop outside [0, 1).
 *   dropout        : y = dropout_p(x) (+ add), fp32 [n] -> fp32 y32 and / or bf16 y16 (n % 4 == 0; x, add, y32 16-byte
 *                    and y16 8-byte aligned, else EGOVLP_ERR_ARG before any launch).  The embedding and
 *                    FFN-output dropouts of DistilBERT (reference model/model.py:36 puts the text model in train mode);
 *                    calling it on a gradient with the same (p, seed, site) is the backward.
 *   relu_rows      : out bf16 [rows, D] = relu(x[r*row_stride + :D]) (CLS -> ReLU of txt_proj, model/model.py:73-75)
 */
int egovlp_text_embed_fwd(const long long* input_ids, const float* word_emb, const float* pos_emb, float* out, int B,
                          int L, int D, void* stream);
int egovlp_text_embed_bwd(const long long* input_ids, const float* dsum, float* dword, float* dpos, int B, int L, int D,
                          void* stream);
/* Deterministic form, from the ids stably sorted (sorted_ids[i] = input_ids[perm[i]], int64 [B*L], perm ascending among
 * equal ids): each vocabulary row adds its tokens' gradients in token order, each position its batch's in b order. */
int egovlp_text_embed_bwd_det(const long long* sorted_ids, const long long* perm, const float* dsum, float* dword,
                              float* dpos, int B, int L, int D, void* stream);
int egovlp_text_attn_fwd(const void* qkv, const long long* attention_mask, void* out, int B, int L, int H, float p_drop,
                         unsigned long long seed, unsigned int site, void* stream);
int egovlp_text_attn_bwd(const void* qkv, const long long* attention_mask, const void* dout, void* dqkv, int B, int L,
                         int H, float q_scale, float p_drop, unsigned long long seed, unsigned int site, void* stream);
int egovlp_text_attn_long_fwd(const void* qkv, const long long* attention_mask, void* out, float* lse, int B, int L,
                              int H, float p_drop, unsigned long long seed, unsigned int site, void* stream);
int egovlp_text_attn_long_bwd(const void* qkv, const long long* attention_mask, const void* out, const float* lse,
                              const void* dout, void* dqkv, float* workspace, int B, int L, int H, float q_scale,
                              float p_drop, unsigned long long seed, unsigned int site, void* stream);
int egovlp_dropout(const float* x, const float* add, float* y32, void* y16_bf16, long long n, float p,
                   unsigned long long seed, unsigned int site, void* stream);
int egovlp_relu_rows_fwd(const float* x, long long row_stride, void* out_bf16, int rows, int D, void* stream);
int egovlp_relu_rows_bwd(const float* x, long long row_stride, const float* dh, float* dx, int rows, int D, void* stream);

/* ------------------------------------------------------------------------------------------------
 * BERT pooler (transformers modeling_bert.py BertPooler), the text embedding of the reference's `bert*` tower:
 * `self.text_model(...)['pooler_output']` (model/model.py:117-131), followed by txt_proj's ReLU (model/model.py:73-75).
 * fp32, no atomics (bitwise reproducible).  1 <= B, 4 <= D <= 1024, D % 4 == 0, row_stride >= D; otherwise
 * EGOVLP_ERR_ARG and nothing is launched.
 *   text_pooler_fwd : y fp32 [B, D] = tanh(h[b * row_stride + :D] W^T + bias), W fp32 [D, D] (nn.Linear layout);
 *                     h = the CLS rows read in place from the [B*L, D] hidden state (row_stride = L * D).
 *                     relu_bf16 (optional, bf16 [B, D]) = relu(y): the txt_proj GEMM operand.
 *   text_pooler_bwd : from grad fp32 [B, D] at relu(y) (relu != 0) or at y (relu == 0, projection=''):
 *                     dz = grad * [y > 0 if relu] * (1 - y^2); writes dweight fp32 [D, D] = dz^T h, dbias [D] = sum_b dz,
 *                     dh[b * row_stride + :D] = dz W (only the B CLS rows of dh are written).
 */
int egovlp_text_pooler_fwd(const float* h, long long row_stride, const float* weight, const float* bias, float* y,
                           void* relu_bf16, int B, int D, void* stream);
int egovlp_text_pooler_bwd(const float* grad, const float* y, int relu, const float* h, long long row_stride,
                           const float* weight, float* dweight, float* dbias, float* dh, int B, int D, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Narrow projection heads: the vid_proj / txt_proj Linear(K, C) of model/model.py:72-79 for widths C the GEMM above
 * cannot take (C % 32 != 0: the OSCC head C = 2, configs/ft/oscc.json; the PNR head C = 16, configs/ft/pnr.json).
 * CUDA-core kernels, no atomics: bitwise reproducible.  All tensors contiguous; K % 8 == 0, 16B-aligned bases.
 *   fwd: out fp32 [rows, C] = act bf16 [rows, K] . w bf16 [C, K]^T + bias fp32 [C] (bias may be NULL); K <= 2048.
 *   bwd: from dout_bf16 [rows, C] (= bf16(dout)):  dw fp32 [C, K] = dout_bf16^T . act,  dact fp32 [rows, K] =
 *        dout_bf16 . w  (rows <= 65535), and from the fp32 dout [rows, C]: db fp32 [C] = column sums of dout.  Each of
 *        dw / db / dact may be NULL.  dw needs a workspace of egovlp_narrow_linear_workspace_floats(rows, C, K) floats
 *        (0: none) for its row splits, which are merged in a fixed order.
 */
int egovlp_narrow_linear_fwd(const void* act_bf16, const void* w_bf16, const float* bias, float* out, int rows, int C,
                             int K, void* stream);
long long egovlp_narrow_linear_workspace_floats(int rows, int C, int K);
int egovlp_narrow_linear_bwd(const float* dout, const void* dout_bf16, const void* act_bf16, const void* w_bf16,
                             float* dw, float* db, float* dact, float* workspace, int rows, int C, int K, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Similarity and losses, fp32 (model/model.py:189-197 sim_matrix; model/loss.py EgoNCE :34-53,
 * NormSoftmaxLoss :13-25, MaxMarginRankingLoss :63-90; run/test_epic.py:137-143 dual softmax;
 * trainer/trainer_egoclip.py:204-215 + model/metric.py:227 EgoMCQ scoring).
 *   rownorm_fwd: an = a / max(||a||, eps) per row, norm[rows] saved;  rownorm_bwd: its backward.
 *   sgemm_f32 : C[m,n] = alpha * sum_k A[m*sam + k*sak] * B[n*sbn + k*sbk] + beta*C  (small fp32 products:
 *               sim = an bn^T, d an = dX bn, d bn = dX^T an)
 *   pack_multihot / mask_from_bits: positives mask uint8 [G,G] from multi-hot verb/noun vectors
 *               (mode 0 identity, 1 verb&noun, 2 noun, 3 verb; diagonal always set) -- equals the reference's
 *               (sim_v*sim_n + I) > 0 for 0/1 tags;  mask_from_sims: the reference's float formulation itself.
 *   nce_fwd   : stats fp32 [4G] (row/col log-sum-exp over all / over positives of x*inv_temp), loss scalar
 *   nce_bwd   : dx fp32 [G,G] = gscale[0] * dloss/dx   (gscale device pointer or NULL for 1)
 *   maxmargin_fwd/bwd : MaxMarginRankingLoss (model/loss.py:63-90); row_weight fp32 [G] or NULL -- with it the margin
 *               of anchor i is margin*row_weight[i] = AdaptiveMaxMarginRankingLoss (model/loss.py:100-133)
 *   dual_softmax (in: sim [rows, cols] -> out), egomcq_score (scores [Q,K], pred int64 [Q], ties -> lowest index).
 */
int egovlp_rownorm_fwd(const float* a, float* an, float* norm, int rows, int C, float eps, void* stream);
int egovlp_rownorm_bwd(const float* dan, const float* an, const float* norm, float* da, int rows, int C, float eps,
                       void* stream);
int egovlp_sgemm_f32(const float* A, long long sam, long long sak, const float* B, long long sbn, long long sbk,
                     float* C, long long ldc, int M, int N, int K, float alpha, float beta, void* stream);
int egovlp_pack_multihot(const float* v, uint32_t* bits, int G, int C, void* stream);
int egovlp_mask_from_bits(const uint32_t* vbits, int n_verb, const uint32_t* nbits, int n_noun, uint8_t* mask, int G,
                          int mode, void* stream);
int egovlp_mask_from_sims(const float* sim_v, const float* sim_n, uint8_t* mask, int G, int mode, void* stream);
int egovlp_nce_fwd(const float* x, const uint8_t* mask, int G, float inv_temp, float* stats, float* loss, void* stream);
int egovlp_nce_bwd(const float* x, const uint8_t* mask, const float* stats, int G, float inv_temp, const float* gscale,
                   float* dx, void* stream);
int egovlp_maxmargin_fwd(const float* x, const float* row_weight, int G, float margin, int fix_norm, float* loss,
                         void* stream);
int egovlp_maxmargin_bwd(const float* x, const float* row_weight, int G, float margin, int fix_norm,
                         const float* gscale, float* dx, void* stream);
/* Deterministic forms: the forward merges its per-CTA partials (ws: egovlp_maxmargin_det_workspace_floats(G) floats)
 * in CTA order; the backward writes each dx element from one thread (off the diagonal: anchor i's term, then anchor
 * j's; on it: the row's terms in j order). */
long long egovlp_maxmargin_det_workspace_floats(int G);
int egovlp_maxmargin_fwd_det(const float* x, const float* row_weight, int G, float margin, int fix_norm, float* loss,
                             float* ws, void* stream);
int egovlp_maxmargin_bwd_det(const float* x, const float* row_weight, int G, float margin, int fix_norm,
                             const float* gscale, float* dx, void* stream);
int egovlp_dual_softmax(const float* sim, float* out, int rows, int cols, float temp, void* stream);

/* EgoNCE from the gathered embeddings, ONE kernel per direction (trainer/trainer_egoclip.py:130-135 = sim_matrix x3 +
 * EgoNCE.forward, model/model.py:189-197 + model/loss.py:34-53).  text / video fp32 [G, C] and the multi-hot verb / noun
 * tags fp32 [G, n_verb] / [G, n_noun] are row-strided views (ld_*, in floats) -- e.g. column slices of ONE packed
 * all-gather buffer, read in place.  mode: 0 InfoNCE (diagonal positives), 1 verb AND noun, 2 noun only, 3 verb only.
 * G <= egovlp_egonce_fused_max_g(), C <= 256.  Forward outputs: norm_text / norm_video [G], tag_bits
 * [G, ceil(n_verb/32) + ceil(n_noun/32)] (only the tag sets `mode` uses are counted), stats [4 G] (row / column
 * log-sum-exps), loss [1]; `workspace`: egovlp_egonce_fused_workspace_floats(G) floats, ZERO before the first launch (the
 * kernel leaves its ticket word zero again).  Backward: d text / d video [n_local, C] of rows [row0, row0 + n_local) only
 * (the gather's backward keeps the local slice, trainer_egoclip.py:23-27); gscale = optional device scalar dL/dloss. */
/* out[rows, ca+cb+cc+cd] = [a | b | c | d] row by row: the send buffer of the ONE packed embedding / tag all-gather that
 * replaces the four AllGather_multi calls of trainer/trainer_egoclip.py:126-129. */
int egovlp_pack_rows4(const float* a, int ca, const float* b, int cb, const float* c, int cc, const float* d, int cd,
                      float* out, int rows, void* stream);
int egovlp_egonce_fused_max_g(void);
/* 1 if egovlp_egonce_fused_fwd can launch this problem on the current device, else 0: besides the G and C limits, the
 * tag bits of all G rows (the widths `mode` uses) must fit in shared memory with the similarity tile. */
int egovlp_egonce_fused_supported(int G, int C, int n_verb, int n_noun, int mode);
long long egovlp_egonce_fused_workspace_floats(int G);
int egovlp_egonce_fused_fwd(const float* text, long long ld_t, const float* video, long long ld_v, const float* verb,
                            long long ld_verb, int n_verb, const float* noun, long long ld_noun, int n_noun, int G, int C,
                            float inv_temp, int mode, float eps, float* norm_text, float* norm_video, uint32_t* tag_bits,
                            float* stats, float* workspace, float* loss, void* stream);
int egovlp_egonce_fused_bwd(const float* text, long long ld_t, const float* video, long long ld_v, const float* norm_text,
                            const float* norm_video, const uint32_t* tag_bits, int n_verb, int n_noun, const float* stats,
                            int G, int C, float inv_temp, int mode, float eps, const float* gscale, int row0, int n_local,
                            float* d_text, float* d_video, void* stream);
int egovlp_egomcq_score(const float* text, const float* video, float* scores, long long* pred, int Q, int K, int C,
                        float eps, void* stream);

/* Softmax cross-entropy, nn.CrossEntropyLoss() with its defaults (model/loss.py:135-141; the OSCC / PNR fine-tuning
 * steps, trainer/trainer_oscc.py:333-338, trainer/trainer_pnr.py:341-348).  logits fp32 [G, C] (row stride ld),
 * target int64 [G].  Forward: lse fp32 [G] (max-subtracted log-sum-exp per row), row_loss fp32 [G] (workspace),
 * out fp32 [2] = {mean of lse - logit[target] over the rows whose target != ignore_index, number of those rows}.
 * A target outside [0, C) that is not ignore_index is never used as an index: its row loss, hence the loss, is NaN
 * (torch raises a device assert instead).  No valid row gives 0 / 0 = NaN, as torch.  The reduction order is fixed:
 * the loss is bitwise reproducible.  Backward: dx fp32 [G, C] contiguous = gscale[0] * (softmax - onehot) / n_valid,
 * zero on ignored rows, NaN on rows with a bad target (gscale device pointer or NULL for 1). */
int egovlp_cross_entropy_fwd(const float* logits, long long ld, const long long* target, int G, int C, int ignore_index,
                             float* lse, float* row_loss, float* out, void* stream);
int egovlp_cross_entropy_bwd(const float* logits, long long ld, const long long* target, const float* lse,
                             const float* out, int G, int C, int ignore_index, const float* gscale, float* dx,
                             void* stream);

/* ------------------------------------------------------------------------------------------------
 * Retrieval evaluation (EPIC-Kitchens MIR; SURVEY.md 8f row 3).  Replaces the host numpy argsort + fancy indexing of
 * utils/nDCG.py:3-45 (calculate_DCG) and utils/mAP.py:4-44 (calculate_mAP) called from model/metric.py:257-299 and
 * run/test_epic.py:137-157.  One CTA ranks one query row in shared memory (bitonic sort of (similarity, column)).
 *   sim  fp32 [rows, cols] (row stride ld_sim);  rel fp32 or fp64 [rows, cols] (row stride ld_rel)
 *   k_counts int32 [rows, cols] contiguous or NULL (NULL: the first k ranks count, k = #(rel[row] > 0), which is what
 *            calculate_k_counts, nDCG.py:47-75, produces)
 *   tie_mode 0: equal similarities rank by smaller column first (stable argsort of -sim, mAP.py:25);
 *            1: by larger column first (stable ascending argsort reversed, nDCG.py:32)
 *            NaN similarities rank where numpy's sort puts them: after every real value (-inf included) in mode 0,
 *            before every real value in mode 1, among themselves by the same column rule.
 *   dcg[row] = sum_i k_i * rel[row, rank_i] / log2(i + 2);  ap[row] = sum_i [rel_i == 1] cumsum(rel)_i / (i + 1) / #(rel == 1)
 *            (NaN for a row without relevant items, as numpy).  Either output may be NULL.  cols <= 16384.
 */
int egovlp_rank_metrics(const float* sim, long long ld_sim, const void* rel, int rel_is_f64, long long ld_rel,
                        const int* k_counts, int rows, int cols, int tie_mode, double* dcg, double* ap, void* stream);

/* Ground-truth ranks of the MSR-VTT-style retrieval metrics (model/metric.py:20-216, t2v_metrics / v2t_metrics), which
 * rank by distance subtraction, so their ranks are fully determined, ties included.  One CTA counts, per candidate, the
 * entries of its row with a greater and with an equal similarity; no sort.  sims fp32 or fp64 [rows, cols] (row stride
 * ld), compared exactly in that type.  ranks fp64 [rows], 0-based.
 *   mode 0 (t2v): rows = queries, cols = videos, rows % cols == 0, q = rows / cols; row i's ground truth is column i / q;
 *                 rank = #{j : sims[i, j] > sims[i, gt]} (ties optimistic).  col_mask must be NULL.
 *   mode 1 (v2t): rows = videos, cols = captions (sims transposed), c = cols / rows (floor) <= egovlp_gt_ranks_max_candidates();
 *                 candidates of row i are columns [i c, (i + 1) c); per candidate rank = #greater + (#equal - 1) / 2
 *                 (ties averaged); the row's rank is the minimum over its candidates, +inf if none is left.  col_mask
 *                 uint8 [cols] or NULL: entries with col_mask == 0 become similarity -1e8 (the reference's distance
 *                 MISSING_VAL); candidates equal to -1e8 or non-finite are skipped.
 * status: int [1] device workspace (bits: 1 NaN in a row, 2 non-finite t2v ground truth).  The call SYNCHRONISES the
 * stream to read it and returns EGOVLP_ERR_ARG, naming every condition found, for a NaN anywhere in a row (after the
 * caption mask) or (t2v) a non-finite ground-truth similarity.  cols <= 65535 * 256. */
int egovlp_gt_ranks_max_candidates(void);
int egovlp_gt_ranks(const void* sims, int is_f64, long long ld, int rows, int cols, int mode, const uint8_t* col_mask,
                    double* ranks, int* status, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Elementwise / reduction helpers on the path.
 */
/* fp32 -> bf16 cast (weights: fp32 master -> bf16 GEMM operand). */
int egovlp_cast_f32_to_bf16(const float* src, void* dst_bf16, long long n, void* stream);
/* Per-row e4m3 quantisation of fp32 weights W [rows, K] (row stride ldw) for egovlp_gemm_e4m3: scale[r] = amax_r / 448
 * (1 for a zero row), q [rows, K] contiguous = e4m3(W[r, k] * (448 / amax_r)), round to nearest, saturating.  K % 4 == 0,
 * w 16B and q 4B aligned. */
int egovlp_quantize_rows_e4m3(const float* w, long long ldw, uint8_t* q, float* scale, int rows, int K, void* stream);
/* out[n] += sum_m dy[m, n]  (bias gradients).  dy bf16 or fp32 [M, N] row stride ld. */
int egovlp_colsum_accum(const void* dy, int dy_is_fp32, long long ld, float* out, int M, int N, void* stream);
/* Deterministic form: row-block partials (ws: egovlp_colsum_det_workspace_floats(M, N, dy_is_fp32) floats, the split
 * sized for 132 SMs on every card) added into out in row-block order. */
long long egovlp_colsum_det_workspace_floats(int M, int N, int dy_is_fp32);
int egovlp_colsum_accum_det(const void* dy, int dy_is_fp32, long long ld, float* out, int M, int N, float* ws,
                            void* stream);
/* Backward of a GEMM dropout form (egovlp_gemm_epilogue.drop_*): y bf16 [rows, W] = bf16(x[r, c] * keep(r, c) /
 * (1 - p) * f(r / path_rows)), keep and f drawn exactly as that form draws them for a [rows, W] output (f = 1 when
 * path_rows = 0): the gradient of the video tower's dropped branches (model/video_transformer.py:36-52, 135-136,
 * 171-175).  x fp32 (x_is_bf16 = 0) or bf16 [rows, W] contiguous, W % 4 == 0, both aligned to four elements; p and
 * path_p in [0, 1). */
int egovlp_drop_rows_bf16(const void* x, int x_is_bf16, void* y_bf16, long long rows, int W, float p,
                          unsigned long long seed, unsigned int site, float path_p, unsigned int path_site,
                          int path_rows, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused multi-tensor AdamW, HuggingFace transformers.AdamW semantics (run/train_egoclip.py:72-73,
 * configs/pt/egoclip.json:49-54): m,v update; p -= step_size * m / (sqrt(v) + eps) with
 * step_size = lr * sqrt(1-b2^t)/(1-b1^t) (computed by the host); then p -= lr * wd * p.
 * tensors_dev: device array of descriptors; chunk_tensor_dev / chunk_offset_dev: for every CTA the tensor index
 * and the chunk index (egovlp_adamw_chunk_elems() elements per chunk) it updates.  grad_scale_dev: optional
 * device scalar multiplied into every gradient (e.g. 1/world for a summed all-reduce), or NULL.
 */
typedef struct egovlp_adamw_tensor {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  long long numel;
  void* shadow_bf16;   /* optional: bf16 copy of the updated parameter written in the same pass (NULL: none) */
} egovlp_adamw_tensor;
int egovlp_adamw_chunk_elems(void);
int egovlp_adamw_multi(const egovlp_adamw_tensor* tensors_dev, const int* chunk_tensor_dev, const int* chunk_offset_dev,
                       int n_chunks, float lr, float beta1, float beta2, float eps, float weight_decay, float step_size,
                       const float* grad_scale_dev, void* stream);


/* fp32 -> bf16 cast of many tensors in ONE launch (the bf16 GEMM-operand copies of all fp32 master weights, refreshed at
 * the top of every training forward so that ANY optimizer -- e.g. transformers.AdamW updating through p.data, as
 * run/train_egoclip.py:72-73 configures -- is seen).  Same chunk-table scheme as egovlp_adamw_multi
 * (egovlp_adamw_chunk_elems() elements per chunk). */
typedef struct egovlp_cast_tensor {
  const float* src;
  void* dst_bf16;
  long long numel;
} egovlp_cast_tensor;
int egovlp_cast_multi_f32_to_bf16(const egovlp_cast_tensor* tensors_dev, const int* chunk_tensor_dev,
                                  const int* chunk_offset_dev, int n_chunks, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EGOVLP_B200_H_ */
