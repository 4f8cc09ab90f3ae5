// Pillow's bicubic resize of 8-bit RGB images on the GPU (C ABI in include/gsb200.h), in its own translation unit so
// that the other kernels are compiled exactly as before.  DESIGN.md 4.21.
//
// Image.resize((W', H')) on an RGB image (libImaging Resample.c, 8 bits per channel) is two separable passes with
// integer weights: the horizontal pass (when the width changes) turns [H, W] into [H, W'] u8, the vertical pass (when
// the height changes) turns that into [H', W'] u8.  Each output channel is
//
//   clamp((2^21 + sum_k src[first + k] * coef[k]) >> 22, 0, 255)
//
// over the taps of its output index, with the tables (first, count) and coef built on the host in Pillow's fp64 order
// (resample.py).  The sums are exact int32 integers, so the order the taps are added in does not matter and every
// output byte is Pillow's.  Pillow runs the horizontal pass on the rows the vertical pass reads only; running it on all
// rows gives the same bytes.
//
//   k_resample_h  one thread per output byte of a row: grid (row chunks, H, V); reads the taps of its channel.
//   k_resample_v  one thread per output byte of a row: grid (row chunks, H', V); consecutive threads read consecutive
//                 bytes of each source row.
//
// A view's bytes depend on its own pixels only: not on V, its place in the batch or the stream.
#include <cuda_runtime.h>
#include <stdio.h>

#include "../../include/gsb200.h"

void gsb_set_error(const char* s);
void gsb_count_launch(int n);

namespace {

constexpr int kThreads = 256;
constexpr int kShift = 22;                       // Pillow's PRECISION_BITS
constexpr int kMaxDim = 65535;                   // rows and views index grid.y and grid.z

int check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return GSB_OK;
  char buf[256];
  snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  gsb_set_error(buf);
  return GSB_ERR_CUDA;
}

__device__ __forceinline__ uint8_t clip8(int acc) {
  const int v = acc >> kShift;                   // arithmetic shift, as Pillow's clip8
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// The taps of output index o, clamped to [0, n_in) and to ksize so that a malformed table cannot read outside the
// image (a table from gsb's own builder is already inside).
__device__ __forceinline__ void taps(const int32_t* bounds, int o, int ksize, int n_in, int* first, int* count) {
  int f = bounds[2 * o], n = bounds[2 * o + 1];
  f = f < 0 ? 0 : (f > n_in ? n_in : f);
  n = n < 0 ? 0 : (n > ksize ? ksize : n);
  *first = f;
  *count = n > n_in - f ? n_in - f : n;
}

// in [V, H, W, 3] -> out [V, H, Wo, 3]
__global__ void __launch_bounds__(kThreads) k_resample_h(int H, int W, int Wo, const uint8_t* __restrict__ in,
                                                         uint8_t* __restrict__ out, const int32_t* __restrict__ bounds,
                                                         const int32_t* __restrict__ coefs, int ksize) {
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j >= 3 * Wo) return;
  const int y = blockIdx.y, v = blockIdx.z;
  const int xo = j / 3, c = j - 3 * xo;
  int first, n;
  taps(bounds, xo, ksize, W, &first, &n);
  const uint8_t* src = in + ((size_t)v * H + y) * (size_t)(3 * W) + 3 * first + c;
  const int32_t* k = coefs + (size_t)xo * ksize;
  int acc = 1 << (kShift - 1);
  for (int t = 0; t < n; ++t) acc += (int)__ldg(src + 3 * t) * __ldg(k + t);
  out[((size_t)v * H + y) * (size_t)(3 * Wo) + j] = clip8(acc);
}

// in [V, H, Wr, 3] -> out [V, Ho, Wr, 3]; Wr is the width after the horizontal pass
__global__ void __launch_bounds__(kThreads) k_resample_v(int H, int Ho, int Wr, const uint8_t* __restrict__ in,
                                                         uint8_t* __restrict__ out, const int32_t* __restrict__ bounds,
                                                         const int32_t* __restrict__ coefs, int ksize) {
  const int j = blockIdx.x * kThreads + threadIdx.x;
  const int row = 3 * Wr;
  if (j >= row) return;
  const int yo = blockIdx.y, v = blockIdx.z;
  int first, n;
  taps(bounds, yo, ksize, H, &first, &n);
  const uint8_t* src = in + ((size_t)v * H + first) * (size_t)row + j;
  const int32_t* k = coefs + (size_t)yo * ksize;
  int acc = 1 << (kShift - 1);
  for (int t = 0; t < n; ++t) acc += (int)__ldg(src + (size_t)t * row) * __ldg(k + t);
  out[((size_t)v * Ho + yo) * (size_t)row + j] = clip8(acc);
}

}  // namespace

extern "C" GSB_API int gsb_resample_u8_batch(int32_t V, int32_t H, int32_t W, int32_t Ho, int32_t Wo,
                                             const uint8_t* in, uint8_t* out, const int32_t* x_bounds,
                                             const int32_t* x_coefs, int32_t x_ksize, const int32_t* y_bounds,
                                             const int32_t* y_coefs, int32_t y_ksize, void* scratch,
                                             size_t scratch_bytes, gsb_stream_t stream) {
  const bool horiz = Wo != W, vert = Ho != H;
  const int64_t max_row = (int64_t)kMaxDim * kThreads;   // bytes of one row the x grid covers
  if (V <= 0 || V > kMaxDim || H <= 0 || H > kMaxDim || Ho <= 0 || Ho > kMaxDim || W <= 0 || Wo <= 0 ||
      3 * (int64_t)W > max_row || 3 * (int64_t)Wo > max_row || !in || !out ||
      (horiz && (!x_bounds || !x_coefs || x_ksize <= 0)) || (vert && (!y_bounds || !y_coefs || y_ksize <= 0))) {
    gsb_set_error("gsb_resample_u8_batch: bad argument");
    return GSB_ERR_INVALID;
  }
  const size_t mid_bytes = (size_t)V * H * Wo * 3;
  if (horiz && vert && (!scratch || scratch_bytes < mid_bytes)) {
    gsb_set_error("gsb_resample_u8_batch: scratch smaller than V * H * Wo * 3 bytes");
    return GSB_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (!horiz && !vert)
    return check(cudaMemcpyAsync(out, in, (size_t)V * H * W * 3, cudaMemcpyDeviceToDevice, st),
                 "gsb_resample_u8_batch copy");
  gsb_count_launch((int)horiz + (int)vert);
  const uint8_t* src = in;
  if (horiz) {
    uint8_t* dst = vert ? static_cast<uint8_t*>(scratch) : out;
    const dim3 grid((unsigned)((3 * Wo + kThreads - 1) / kThreads), (unsigned)H, (unsigned)V);
    k_resample_h<<<grid, kThreads, 0, st>>>(H, W, Wo, in, dst, x_bounds, x_coefs, x_ksize);
    int rc = check(cudaGetLastError(), "k_resample_h");
    if (rc != GSB_OK) return rc;
    src = dst;
  }
  if (vert) {
    const dim3 grid((unsigned)((3 * Wo + kThreads - 1) / kThreads), (unsigned)Ho, (unsigned)V);
    k_resample_v<<<grid, kThreads, 0, st>>>(H, Ho, Wo, src, out, y_bounds, y_coefs, y_ksize);
    return check(cudaGetLastError(), "k_resample_v");
  }
  return GSB_OK;
}
