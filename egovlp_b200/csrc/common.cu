// Host-side glue: thread-local error string, SM count, TMA descriptor encoding.
#include <stdarg.h>
#include <stdio.h>

#include "common.cuh"
#include "egovlp_b200.h"

namespace egovlp {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// out_k[i] = ((out_k[i] + part_k[0][i]) + part_k[1][i]) + ... for up to three outputs (part_k = part + k * nparts * n):
// the fixed-order merge of per-CTA partials.  Eight partials are loaded before they are added, in order, so that the
// loads overlap while the order of the additions stays that of the partials.
__global__ void ordered_sum_kernel(const float* __restrict__ part, int nparts, long long n, float* __restrict__ out0,
                                   float* __restrict__ out1, float* __restrict__ out2) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int k = (int)(j / n);
  const long long i = j - (long long)k * n;
  float* out = k == 0 ? out0 : k == 1 ? out1 : out2;
  if (k > 2 || !out) return;
  const float* p = part + (long long)k * nparts * n + i;
  float acc = out[i];
  int q = 0;
  for (; q + 8 <= nparts; q += 8) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = p[(long long)(q + u) * n];
#pragma unroll
    for (int u = 0; u < 8; ++u) acc += v[u];
  }
  for (; q < nparts; ++q) acc += p[(long long)q * n];
  out[i] = acc;
}

int ordered_sum(const float* part, int nparts, long long n, float* out0, float* out1, float* out2, cudaStream_t st) {
  const int nout = out2 ? 3 : out1 ? 2 : out0 ? 1 : 0;
  if (nout == 0 || n <= 0) return EGOVLP_OK;
  const long long total = nout * n;
  ordered_sum_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(part, nparts, n, out0, out1, out2);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 148;
  }
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static int make_tmap_nd(CUtensorMap* out, CUtensorMapDataType dtype, uint64_t esize, const void* base, int rank,
                        const uint64_t* dims, const uint64_t* strides, const uint32_t* box, bool swizzle128) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable");
    return EGOVLP_ERR_CUDA;
  }
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    if (i > 0) gstr[i - 1] = strides[i] * esize;
  }
  CUresult r = fn(out, dtype, rank, const_cast<void*>(base), gdim, gstr, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: CUresult %d (rank %d dims %llu,%llu box %u,%u)", (int)r, rank,
                   (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
                   rank > 1 ? box[1] : 0);
    return EGOVLP_ERR_CUDA;
  }
  return EGOVLP_OK;
}

int make_tmap_nd_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                      const uint32_t* box, bool swizzle128) {
  return make_tmap_nd(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, rank, dims, strides, box, swizzle128);
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                      uint32_t box_cols) {
  const uint64_t dims[2] = {cols, rows};
  const uint64_t strides[2] = {1, ld};
  const uint32_t box[2] = {box_cols, box_rows};
  return make_tmap_nd_bf16(out, base, 2, dims, strides, box, true);
}

int make_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                     uint32_t box_cols) {
  const uint64_t dims[2] = {cols, rows};
  const uint64_t strides[2] = {1, ld};
  const uint32_t box[2] = {box_cols, box_rows};
  return make_tmap_nd(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, 2, dims, strides, box, true);
}

int make_tmap_2d_u8(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                    uint32_t box_cols) {
  const uint64_t dims[2] = {cols, rows};
  const uint64_t strides[2] = {1, ld};
  const uint32_t box[2] = {box_cols, box_rows};
  return make_tmap_nd(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, base, 2, dims, strides, box, true);
}

}  // namespace egovlp

extern "C" const char* egovlp_last_error(void) { return egovlp::g_err; }
extern "C" int egovlp_abi_version(void) { return 1; }
