// Dataset video transforms on the GPU (data_loader/transforms.py:34-61 + the reader tail of base/base_dataset.py:220-243
// and :117-140): decoded uint8 frames in, the normalised, zero-padded fp32 [B, F, 3, R, R] clip batch out.
//
// IEEE build (build.py IEEE_SOURCES): b / 255.f and (v - mean) / std are correctly rounded divisions, as torch's.
//
// Every output pixel is a separable weighted sum over the source frame, sum_y wy * (sum_x wx * src[y, x] / 255), with
// per-axis weights that depend only on the clip's geometry:
//   train: bilinear, align_corners=False, no antialias, on the crop box (i, j, h, w) (F.interpolate in
//          _functional_video.resized_crop), then an optional reversal of the output columns (hflip after the resize);
//   eval:  Resize(center_crop) -> CenterCrop(center_crop) -> Resize(R), both resizes torch's antialiased (PIL-style
//          triangle filter) bilinear, composed per axis into one weight row over the source.  A resize whose output
//          equals its input is the identity, as torchvision returns the image unchanged.
// The reference runs the eval resizes as two separable passes through fp32 intermediates; the composed weights sum
// the same products in another order, which moves results by fp32 rounding only.
//
// One CTA per (band of VT_ROWS output rows, frame, clip).  It builds the band's row weights and all R column weights in
// shared memory, then each thread gathers its pixels straight from the uint8 frame (through L1: neighbouring outputs
// share taps, so each source byte comes from L2 / HBM about once per CTA).  Frames t >= T_i are written as 0.0.
// No atomics: the output is bitwise reproducible.
#include "common.cuh"

namespace egovlp {
namespace {

constexpr int VT_TAPS = 32;      // source taps per output index per axis (composed eval weights need up to ~26 at 1440p)
constexpr int VT_ROWS = 8;       // output rows per CTA
constexpr int VT_THREADS = 256;
constexpr int VT_MAX_RES = 320;  // R: VT_TAPS * R column weights must fit in 48 KB of shared memory
constexpr int VT_DESC = 10;      // descriptor row: offset, T, H, W, mode, i, j, h, w, flip

__device__ __forceinline__ float tri(float x) {
  x = fabsf(x);
  return x < 1.f ? 1.f - x : 0.f;
}

// Antialiased linear resize in -> out (torch _upsample_bilinear2d_aa, align_corners=False): taps [xmin, xmin + n) of
// output o; weight k is tri((k + xmin - center + 0.5) * invscale) / total.
struct AaAxis {
  float scale, support, invscale;
  int in;
  __device__ AaAxis(int in_, int out) : in(in_) {
    scale = (float)in_ / (float)out;
    support = scale >= 1.f ? scale : 1.f;
    invscale = scale >= 1.f ? 1.f / scale : 1.f;
  }
  __device__ void taps(int o, int& xmin, int& n, float& center, float& total) const {
    center = scale * ((float)o + 0.5f);
    xmin = max((int)(center - support + 0.5f), 0);
    n = min((int)(center + support + 0.5f), in) - xmin;
    total = 0.f;
    for (int k = 0; k < n; ++k) total += tri(((float)(k + xmin) - center + 0.5f) * invscale);
  }
  __device__ float weight(int k, int xmin, float center, float total) const {
    return tri(((float)(k + xmin) - center + 0.5f) * invscale) / total;
  }
};

// Weights of output index o along one axis, written to w[k * ld] (k < VT_TAPS, pre-zeroed); returns the first source
// index in *s0 and the tap count.  Returns -1 if the weights need more than VT_TAPS taps.
__device__ int axis_weights_train(int o, int R, int off, int ext, bool flip, float* w, int ld, int* s0) {
  const int od = flip ? R - 1 - o : o;
  const float scale = (float)ext / (float)R;
  float src = __fmaf_rn(scale, (float)od + 0.5f, -0.5f);    // one rounding, as torch's CPU kernel on the reference's
                                                            // [C, T, h, w] crop view (an fma there)
  src = src < 0.f ? 0.f : src;
  const int i0 = min((int)src, ext - 1);
  const float l1 = fminf(fmaxf(src - (float)i0, 0.f), 1.f), l0 = 1.f - l1;
  *s0 = off + i0;
  if (i0 < ext - 1) {
    w[0] = l0;
    w[ld] = l1;
    return 2;
  }
  w[0] = l0 + l1;      // both taps on the last source index
  return 1;
}

// Eval axis: source extent `in` -> resize to d1 -> crop [c0, c0 + cc) -> resize to R.
__device__ int axis_weights_eval(int o, int R, int in, int d1, int c0, int cc, float* w, int ld, int* s0) {
  const bool id1 = d1 == in, id2 = cc == R;
  const AaAxis r1(in, d1), r2(cc, R);
  int u0 = o, nu = 1;
  float cu = 0.f, tu = 1.f;
  if (!id2) r2.taps(o, u0, nu, cu, tu);
  int first = -1, count = 0;
  for (int ku = 0; ku < nu; ++ku) {
    const float a = id2 ? 1.f : r2.weight(ku, u0, cu, tu);
    const int v = u0 + ku + c0;
    int x0 = v, nx = 1;
    float cx = 0.f, tx = 1.f;
    if (!id1) r1.taps(v, x0, nx, cx, tx);
    if (first < 0) first = x0;            // xmin of resize 1 is non-decreasing in v
    for (int kx = 0; kx < nx; ++kx) {
      const float b = id1 ? 1.f : r1.weight(kx, x0, cx, tx);
      const int idx = x0 + kx - first;
      if (idx >= VT_TAPS) return -1;
      w[idx * ld] += a * b;
      count = max(count, idx + 1);
    }
  }
  *s0 = first;
  return count;
}

// Python's int(round(d / 2)) for d >= 0: halves round to even.
__device__ __forceinline__ int round_half_even_half(int d) {
  const int q = d >> 1;
  return (d & 1) && (q & 1) ? q + 1 : q;
}

struct Norm3 {
  float v[3];
};

__global__ void __launch_bounds__(VT_THREADS) video_transform_kernel(
    const uint8_t* __restrict__ frames, long long frames_bytes, const long long* __restrict__ desc, int F, int R, int cc,
    Norm3 mean, Norm3 stdv, float* __restrict__ out) {
  extern __shared__ float vt_smem[];
  float* lut = vt_smem;                              // [256]  b / 255.f
  float* colw = lut + 256;                           // [VT_TAPS][R]
  float* roww = colw + VT_TAPS * R;                  // [VT_TAPS][VT_ROWS]
  int* col_s0 = reinterpret_cast<int*>(roww + VT_TAPS * VT_ROWS);   // [R]
  int* col_n = col_s0 + R;                           // [R]
  int* row_s0 = col_n + R;                           // [VT_ROWS]
  int* row_n = row_s0 + VT_ROWS;                     // [VT_ROWS]
  __shared__ int bad;

  const int y0 = blockIdx.x * VT_ROWS, t = blockIdx.y, b = blockIdx.z;
  const int rows = min(VT_ROWS, R - y0);
  const size_t plane = (size_t)R * R;
  float* ob = out + ((size_t)b * F + t) * 3 * plane + (size_t)y0 * R;

  const long long* d = desc + (size_t)b * VT_DESC;
  const long long off = d[0], T = d[1], H = d[2], W = d[3], mode = d[4];
  const long long ci = d[5], cj = d[6], ch = d[7], cw = d[8], flip = d[9];

  if (t >= T) {                                      // the reader's zero padding (`final`, base_dataset.py:138-140)
    for (int p = threadIdx.x; p < rows * R; p += VT_THREADS)
      for (int c = 0; c < 3; ++c) ob[c * plane + p] = 0.f;
    return;
  }
  // The host validates every row; a row that still fails here is reported as NaN instead of being read.
  bool ok = T >= 1 && T <= F && H >= 1 && W >= 1 && H <= 65535 && W <= 65535 && off >= 0 &&
            off + T * H * W * 3 <= frames_bytes && (mode == 0 || mode == 1);
  if (ok && mode == 0) ok = ch >= 1 && cw >= 1 && ci >= 0 && cj >= 0 && ci + ch <= H && cj + cw <= W;

  if (threadIdx.x == 0) bad = !ok;
  for (int k = threadIdx.x; k < VT_TAPS * (R + VT_ROWS); k += VT_THREADS) colw[k] = 0.f;   // colw and roww
  lut[threadIdx.x] = (float)threadIdx.x / 255.f;
  __syncthreads();
  if (ok) {
    int fail = 0;
    if (mode == 0) {
      for (int x = threadIdx.x; x < R; x += VT_THREADS) {
        col_n[x] = axis_weights_train(x, R, (int)cj, (int)cw, flip != 0, colw + x, R, col_s0 + x);
      }
      if (threadIdx.x < rows)
        row_n[threadIdx.x] = axis_weights_train(y0 + threadIdx.x, R, (int)ci, (int)ch, false, roww + threadIdx.x,
                                                VT_ROWS, row_s0 + threadIdx.x);
    } else {
      // torchvision Resize(cc): short side -> cc, long side -> int(cc * long / short); then CenterCrop(cc)
      const int h = (int)H, w = (int)W;
      const bool wshort = w <= h;
      const int shrt = wshort ? w : h, lng = wshort ? h : w;
      const int nlong = (int)(((long long)cc * lng) / shrt);
      const int dh = wshort ? nlong : cc, dw = wshort ? cc : nlong;
      const bool skip1 = dh == h && dw == w;
      const int c0y = round_half_even_half(dh - cc), c0x = round_half_even_half(dw - cc);
      for (int x = threadIdx.x; x < R; x += VT_THREADS) {
        col_n[x] = axis_weights_eval(x, R, w, skip1 ? w : dw, c0x, cc, colw + x, R, col_s0 + x);
        fail |= col_n[x] < 0;
      }
      if (threadIdx.x < rows) {
        row_n[threadIdx.x] = axis_weights_eval(y0 + threadIdx.x, R, h, skip1 ? h : dh, c0y, cc, roww + threadIdx.x,
                                               VT_ROWS, row_s0 + threadIdx.x);
        fail |= row_n[threadIdx.x] < 0;
      }
    }
    if (fail) bad = 1;
  }
  __syncthreads();

  if (bad) {
    for (int p = threadIdx.x; p < rows * R; p += VT_THREADS)
      for (int c = 0; c < 3; ++c) ob[c * plane + p] = __int_as_float(0x7fc00000);
    return;
  }
  const uint8_t* fr = frames + off + (size_t)t * H * W * 3;
  for (int p = threadIdx.x; p < rows * R; p += VT_THREADS) {
    const int yl = p / R, x = p - yl * R;
    const int ny = row_n[yl], nx = col_n[x];
    const uint8_t* src = fr + ((size_t)row_s0[yl] * W + col_s0[x]) * 3;
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f;
    for (int ky = 0; ky < ny; ++ky) {
      const float wy = roww[ky * VT_ROWS + yl];
      const uint8_t* s = src + (size_t)ky * W * 3;
      float h0 = 0.f, h1 = 0.f, h2 = 0.f;
      for (int kx = 0; kx < nx; ++kx) {
        const float wx = colw[kx * R + x];
        h0 += wx * lut[__ldg(s + 3 * kx)];
        h1 += wx * lut[__ldg(s + 3 * kx + 1)];
        h2 += wx * lut[__ldg(s + 3 * kx + 2)];
      }
      acc0 += wy * h0;
      acc1 += wy * h1;
      acc2 += wy * h2;
    }
    ob[p] = (acc0 - mean.v[0]) / stdv.v[0];
    ob[plane + p] = (acc1 - mean.v[1]) / stdv.v[1];
    ob[2 * plane + p] = (acc2 - mean.v[2]) / stdv.v[2];
  }
}

}  // namespace
}  // namespace egovlp

using namespace egovlp;

extern "C" int egovlp_video_transform_max_taps(void) { return VT_TAPS; }
extern "C" int egovlp_video_transform_max_res(void) { return VT_MAX_RES; }

extern "C" int egovlp_video_transform(const uint8_t* frames, long long frames_bytes, const long long* desc, int B, int F,
                                      int R, int center_crop, const float* host_mean, const float* host_std, float* out,
                                      void* stream) {
  EGOVLP_CHECK_ARG(frames && desc && out && host_mean && host_std && frames_bytes > 0, "video_transform: bad args");
  EGOVLP_CHECK_ARG(B >= 1 && B <= 65535 && F >= 1 && F <= 65535 && R >= 1 && R <= VT_MAX_RES && center_crop >= 1,
                   "video_transform: need 1 <= B, F <= 65535, 1 <= R <= %d, center_crop >= 1 (got B=%d F=%d R=%d "
                   "center_crop=%d)", VT_MAX_RES, B, F, R, center_crop);
  Norm3 mean, stdv;
  for (int c = 0; c < 3; ++c) {
    mean.v[c] = host_mean[c];
    stdv.v[c] = host_std[c];
  }
  const size_t smem = (256 + (size_t)VT_TAPS * (R + VT_ROWS)) * sizeof(float) + (2 * (size_t)R + 2 * VT_ROWS) * sizeof(int);
  const dim3 grid((R + VT_ROWS - 1) / VT_ROWS, F, B);
  video_transform_kernel<<<grid, VT_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      frames, frames_bytes, desc, F, R, center_crop, mean, stdv, out);
  EGOVLP_CHECK_LAUNCH();
  return EGOVLP_OK;
}
