// LPIPS (VGG16, v0.1) for metrics.py (C ABI in include/gsb200.h), in its own translation unit so that the training,
// tracking and metrics kernels are compiled exactly as before.
//
// Replaces lpipsPyTorch.lpips(x, y, net_type='vgg') (lpipsPyTorch/__init__.py, modules/lpips.py, networks.py,
// utils.py) called per image by metrics.py:69.  Activations are NHWC fp32: a pixel's channels are contiguous, so the
// 3x3 gather of a conv reads whole 32-byte runs.  Every sum is taken in one fixed order (no split-K, no atomics), so
// an image's features, and so its LPIPS, do not depend on the batch it is in or on the run.
//
// Conv: implicit GEMM, M = pixels, N = Cout, K = 9 Cin, fp32 FFMA.  One CTA of 256 threads computes a 16x16 pixel
// tile of one image for 64 output channels; a thread owns 8 consecutive pixels of one row times 8 channels (64
// accumulators).  The input tile with its 1-pixel halo and the weights of CK input channels are staged in shared
// memory by cp.async, double buffered over the Cin chunks.  Per (channel, kernel row) a thread reads the 10 input
// values its 8 pixels need once and reuses them for the 3 kernel columns: 10 scalar and 6 128-bit shared loads per
// 192 FFMA.  Each output adds its K terms as chunk -> channel -> kernel row -> kernel column, then the bias.
#include <cuda_runtime.h>
#include <stdio.h>

#include "../../include/gsb200.h"

void gsb_set_error(const char* s);
void gsb_count_launch(int n);

namespace {

constexpr int kThreads = 256;
constexpr int TH = 16, TW = 16;     // output tile per CTA
constexpr int PX = 8;               // consecutive pixels of one row per thread
constexpr int CO = 8;               // output channels per thread
constexpr int BN = 64;              // output channels per CTA
constexpr int EH = TH + 2, EW = TW + 2;

// Shared-memory geometry of one pipeline stage for CK input channels per chunk.  The row stride of the staged input
// is padded (CK = 8) so that the four rows a warp reads at once fall in different banks.
template <int CK> struct Stage {
  static constexpr int RS = EW * CK + (CK == 8 ? 4 : 0);
  static constexpr int IN = EH * RS;                 // floats of the input tile
  static constexpr int WT = 9 * CK * BN;             // floats of the weight slice
  static constexpr int FLOATS = IN + WT;
  static constexpr int STAGES = CK == 8 ? 2 : 1;
  static constexpr size_t BYTES = (size_t)STAGES * FLOATS * sizeof(float);
};

__device__ __forceinline__ void cp_async16(float* dst, const float* src, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(src), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(d), "l"(src), "r"(valid ? 4 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// Stage input channels c0 .. c0 + CK of the (EH x EW) halo tile at (y0 - 1, x0 - 1) and their weights for output
// channels n0 .. n0 + BN.  Out-of-image pixels are zero-filled (the conv's zero padding).
template <int CK>
__device__ __forceinline__ void stage_chunk(float* s, const float* __restrict__ img, int H, int W, int Cin, int Cout,
                                            int y0, int x0, int c0, const float* __restrict__ wp, int n0) {
  using S = Stage<CK>;
  float* s_in = s;
  float* s_w = s + S::IN;
  if constexpr (CK == 8) {
    for (int i = threadIdx.x; i < EH * EW * 2; i += kThreads) {
      const int q = i & 1, pix = i >> 1, r = pix / EW, c = pix % EW;
      const int gy = y0 - 1 + r, gx = x0 - 1 + c;
      const bool ok = gy >= 0 && gy < H && gx >= 0 && gx < W;
      const float* src = ok ? img + ((size_t)gy * W + gx) * Cin + c0 + 4 * q : img;
      cp_async16(s_in + r * S::RS + c * CK + 4 * q, src, ok);
    }
  } else {
    for (int i = threadIdx.x; i < EH * EW * CK; i += kThreads) {
      const int k = i % CK, pix = i / CK, r = pix / EW, c = pix % EW;
      const int gy = y0 - 1 + r, gx = x0 - 1 + c;
      const bool ok = gy >= 0 && gy < H && gx >= 0 && gx < W;
      const float* src = ok ? img + ((size_t)gy * W + gx) * Cin + c0 + k : img;
      cp_async4(s_in + r * S::RS + c * CK + k, src, ok);
    }
  }
  // packed weights: row (ci * 9 + tap) of Cout floats; rows c0 * 9 .. (c0 + CK) * 9, columns n0 .. n0 + BN
  const float* wsrc = wp + (size_t)c0 * 9 * Cout + n0;
  for (int i = threadIdx.x; i < 9 * CK * (BN / 4); i += kThreads) {
    const int row = i / (BN / 4), q = i % (BN / 4);
    cp_async16(s_w + row * BN + 4 * q, wsrc + (size_t)row * Cout + 4 * q, true);
  }
}

// in [N, H, W, Cin] -> out [N, H, W, Cout] = relu(conv3x3(in, pad 1) + bias).  Grid (N * tilesY * tilesX, Cout / BN).
template <int CK>
__global__ void __launch_bounds__(kThreads, 2)
k_lpips_conv3x3_relu(int H, int W, int Cin, int Cout, int tiles_x, int tiles_per_img, const float* __restrict__ in,
                     const float* __restrict__ wp, const float* __restrict__ bias, float* __restrict__ out) {
  using S = Stage<CK>;
  extern __shared__ __align__(16) float smem[];
  const int n = blockIdx.x / tiles_per_img, t = blockIdx.x % tiles_per_img;
  const int y0 = (t / tiles_x) * TH, x0 = (t % tiles_x) * TW;
  const int n0 = blockIdx.y * BN;
  const float* img = in + (size_t)n * H * W * Cin;
  const int tc = threadIdx.x & 7;           // channels n0 + 8 tc .. + 7
  const int pg = threadIdx.x >> 3;          // 32 pixel groups: row pg % 16, columns 8 (pg / 16) .. + 7
  const int row = pg & 15, col = (pg >> 4) * PX;

  float acc[PX][CO];
#pragma unroll
  for (int p = 0; p < PX; ++p)
#pragma unroll
    for (int j = 0; j < CO; ++j) acc[p][j] = 0.f;

  const int chunks = Cin / CK;
  stage_chunk<CK>(smem, img, H, W, Cin, Cout, y0, x0, 0, wp, n0);
  cp_async_commit();
  for (int k = 0; k < chunks; ++k) {
    if (S::STAGES == 2 && k + 1 < chunks) {
      stage_chunk<CK>(smem + ((k + 1) & 1) * S::FLOATS, img, H, W, Cin, Cout, y0, x0, (k + 1) * CK, wp, n0);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* s_in = smem + (S::STAGES == 2 ? (k & 1) * S::FLOATS : 0);
    const float* s_w = s_in + S::IN;
#pragma unroll 1
    for (int ci = 0; ci < CK; ++ci) {
      // the kernel-row loop stays rolled: unrolled, its addresses push the 64 accumulators past 128 registers (spill)
#pragma unroll 1
      for (int dy = 0; dy < 3; ++dy) {
        float a[PX + 2];
        const float* src = s_in + (row + dy) * S::RS + col * CK + ci;
#pragma unroll
        for (int q = 0; q < PX + 2; ++q) a[q] = src[q * CK];
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          const float* w = s_w + (ci * 9 + dy * 3 + dx) * BN + tc * CO;
          const float4 w0 = *reinterpret_cast<const float4*>(w);
          const float4 w1 = *reinterpret_cast<const float4*>(w + 4);
          const float wv[CO] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
          for (int p = 0; p < PX; ++p)
#pragma unroll
            for (int j = 0; j < CO; ++j) acc[p][j] = fmaf(a[p + dx], wv[j], acc[p][j]);
        }
      }
    }
    __syncthreads();
  }

  const int gy = y0 + row;
  if (gy >= H) return;
  float b[CO];
#pragma unroll
  for (int j = 0; j < CO; ++j) b[j] = __ldg(bias + n0 + tc * CO + j);
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    const int gx = x0 + col + p;
    if (gx >= W) break;
    float v[CO];
#pragma unroll
    for (int j = 0; j < CO; ++j) {
      const float s = acc[p][j] + b[j];
      v[j] = s > 0.f ? s : 0.f;
    }
    float4* dst = reinterpret_cast<float4*>(out + (((size_t)n * H + gy) * W + gx) * Cout + n0 + tc * CO);
    dst[0] = make_float4(v[0], v[1], v[2], v[3]);
    dst[1] = make_float4(v[4], v[5], v[6], v[7]);
  }
}

// x, y [V, 3, H, W] (k / 255) -> out [2V, H, W, 3] NHWC, images 0..V-1 from x and V..2V-1 from y, z-scored as
// BaseNet.z_score: (v - mean) / std in fp32.  Grid (ceil(H W / 256), 2V).
__global__ void __launch_bounds__(kThreads)
k_lpips_prepare(int V, int HW, const float* __restrict__ x, const float* __restrict__ y, float* __restrict__ out) {
  const int p = blockIdx.x * kThreads + threadIdx.x;
  if (p >= HW) return;
  const int i = blockIdx.y;
  const float* src = i < V ? x + (size_t)i * 3 * HW : y + (size_t)(i - V) * 3 * HW;
  const float mean[3] = {-.030f, -.088f, -.188f}, stdv[3] = {.458f, .448f, .450f};
  float* dst = out + ((size_t)i * HW + p) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) dst[c] = (__ldg(src + (size_t)c * HW + p) - mean[c]) / stdv[c];
}

// MaxPool2d(2, 2), floor mode, NHWC: in [N, H, W, C] -> out [N, H / 2, W / 2, C], 4 channels per thread.
__global__ void __launch_bounds__(kThreads)
k_lpips_maxpool2(int64_t total4, int H, int W, int C, const float* __restrict__ in, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i >= total4) return;
  const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
  const int c4 = (int)(i % C4);
  int64_t r = i / C4;
  const int xo = (int)(r % Wo);
  r /= Wo;
  const int yo = (int)(r % Ho);
  const int64_t n = r / Ho;
  const float4* base = reinterpret_cast<const float4*>(in) + ((n * H + 2 * yo) * W + 2 * xo) * C4 + c4;
  const float4 a = __ldg(base), b = __ldg(base + C4), c = __ldg(base + (size_t)W * C4), d = __ldg(base + (size_t)W * C4 + C4);
  reinterpret_cast<float4*>(out)[i] = make_float4(fmaxf(fmaxf(a.x, b.x), fmaxf(c.x, d.x)), fmaxf(fmaxf(a.y, b.y), fmaxf(c.y, d.y)),
                                                  fmaxf(fmaxf(a.z, b.z), fmaxf(c.z, d.z)), fmaxf(fmaxf(a.w, b.w), fmaxf(c.w, d.w)));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One warp per pixel, lanes over channels c = lane + 32 k: normalize_activation of x's and y's features
// (f / (sqrt(sum_c f^2) + 1e-10)), the squared difference dotted with the lin weights.  The warp adds its pixels'
// values in fp64 in pixel order; block (b, v) writes the sum of its 8 warps to partials[v * GSB_LPIPS_HEAD_PARTS + b].
// The pixels of block b are p = 8 b + warp + 8 GSB_LPIPS_HEAD_PARTS i: a function of H and W only.
__global__ void __launch_bounds__(kThreads)
k_lpips_head(int V, int HW, int C, const float* __restrict__ feats, const float* __restrict__ lin,
             double* __restrict__ partials) {
  __shared__ double red[kThreads / 32];
  const int v = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* fx = feats + (size_t)v * HW * C;
  const float* fy = feats + (size_t)(V + v) * HW * C;
  double s = 0.0;
  for (int p = blockIdx.x * (kThreads / 32) + warp; p < HW; p += GSB_LPIPS_HEAD_PARTS * (kThreads / 32)) {
    const float* a = fx + (size_t)p * C;
    const float* b = fy + (size_t)p * C;
    float sa = 0.f, sb = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float u = __ldg(a + c), w = __ldg(b + c);
      sa = fmaf(u, u, sa);
      sb = fmaf(w, w, sb);
    }
    const float na = sqrtf(warp_sum(sa)) + 1e-10f, nb = sqrtf(warp_sum(sb)) + 1e-10f;
    float d = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float e = __ldg(a + c) / na - __ldg(b + c) / nb;
      d = fmaf(__ldg(lin + c), e * e, d);
    }
    s += (double)warp_sum(d);
  }
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];
    partials[(size_t)v * GSB_LPIPS_HEAD_PARTS + blockIdx.x] = t;
  }
}

// out[v * 5 + layer] = the sum of view v's GSB_LPIPS_HEAD_PARTS partials in a fixed tree.
__global__ void __launch_bounds__(GSB_LPIPS_HEAD_PARTS)
k_lpips_head_reduce(int layer, const double* __restrict__ partials, double* __restrict__ out) {
  __shared__ double red[GSB_LPIPS_HEAD_PARTS];
  const int v = blockIdx.x;
  red[threadIdx.x] = partials[(size_t)v * GSB_LPIPS_HEAD_PARTS + threadIdx.x];
  __syncthreads();
#pragma unroll
  for (int o = GSB_LPIPS_HEAD_PARTS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[(size_t)v * 5 + layer] = red[0];
}

int check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return GSB_OK;
  char buf[256];
  snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  gsb_set_error(buf);
  return GSB_ERR_CUDA;
}

int invalid(const char* msg) {
  gsb_set_error(msg);
  return GSB_ERR_INVALID;
}

bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

template <int CK>
int launch_conv(int N, int H, int W, int Cin, int Cout, const float* in, const float* wp, const float* bias, float* out,
                cudaStream_t st) {
  using S = Stage<CK>;
  // set on every call: the attribute belongs to the current device, and setting it is a host-side call
  int rc = check(cudaFuncSetAttribute(k_lpips_conv3x3_relu<CK>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)S::BYTES), "gsb_lpips_conv3x3_relu: shared memory");
  if (rc != GSB_OK) return rc;
  const int tiles_x = (W + TW - 1) / TW, tiles = tiles_x * ((H + TH - 1) / TH);
  dim3 grid((unsigned)((int64_t)N * tiles), (unsigned)(Cout / BN));
  gsb_count_launch(1);
  k_lpips_conv3x3_relu<CK><<<grid, kThreads, S::BYTES, st>>>(H, W, Cin, Cout, tiles_x, tiles, in, wp, bias, out);
  return check(cudaGetLastError(), "k_lpips_conv3x3_relu");
}

}  // namespace

extern "C" GSB_API size_t gsb_lpips_scratch_bytes(int32_t V, int32_t H, int32_t W) {
  if (V <= 0 || H <= 0 || W <= 0) return 0;
  return 2 * ((size_t)2 * V * H * W * 64 * sizeof(float)) + (size_t)V * GSB_LPIPS_HEAD_PARTS * sizeof(double);
}

extern "C" GSB_API int gsb_lpips_prepare(int32_t V, int32_t H, int32_t W, const float* x, const float* y, float* out,
                                         gsb_stream_t stream) {
  if (V <= 0 || V > 32767 || H <= 0 || W <= 0 || (int64_t)H * W > INT32_MAX - kThreads || !x || !y || !out)
    return invalid("gsb_lpips_prepare: bad argument");
  const int HW = H * W;
  dim3 grid((unsigned)((HW + kThreads - 1) / kThreads), (unsigned)(2 * V));
  gsb_count_launch(1);
  k_lpips_prepare<<<grid, kThreads, 0, (cudaStream_t)stream>>>(V, HW, x, y, out);
  return check(cudaGetLastError(), "k_lpips_prepare");
}

extern "C" GSB_API int gsb_lpips_conv3x3_relu(int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout,
                                              const float* in, const float* w_packed, const float* bias, float* out,
                                              gsb_stream_t stream) {
  if (N <= 0 || H <= 0 || W <= 0 || !in || !w_packed || !bias || !out || Cout <= 0 || Cout % BN != 0 ||
      Cout / BN > 65535 || (Cin != 3 && (Cin <= 0 || Cin % 8 != 0)))
    return invalid("gsb_lpips_conv3x3_relu: bad argument (Cin must be 3 or a multiple of 8, Cout a multiple of 64)");
  const int64_t tiles = (int64_t)((W + TW - 1) / TW) * ((H + TH - 1) / TH);
  if (tiles * N > INT32_MAX) return invalid("gsb_lpips_conv3x3_relu: too many tiles for one launch");
  if (!aligned16(w_packed) || !aligned16(out) || (Cin != 3 && !aligned16(in)))
    return invalid("gsb_lpips_conv3x3_relu: in (Cin > 3), w_packed and out must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  return Cin == 3 ? launch_conv<3>(N, H, W, Cin, Cout, in, w_packed, bias, out, st)
                  : launch_conv<8>(N, H, W, Cin, Cout, in, w_packed, bias, out, st);
}

extern "C" GSB_API int gsb_lpips_maxpool2(int32_t N, int32_t H, int32_t W, int32_t C, const float* in, float* out,
                                          gsb_stream_t stream) {
  if (N <= 0 || H < 2 || W < 2 || C <= 0 || C % 4 != 0 || !in || !out || !aligned16(in) || !aligned16(out))
    return invalid("gsb_lpips_maxpool2: bad argument (H, W >= 2, C a multiple of 4, 16-byte aligned buffers)");
  const int64_t total4 = (int64_t)N * (H / 2) * (W / 2) * (C / 4);
  const int64_t blocks = (total4 + kThreads - 1) / kThreads;
  if (blocks > INT32_MAX) return invalid("gsb_lpips_maxpool2: too large for one launch");
  gsb_count_launch(1);
  k_lpips_maxpool2<<<(unsigned)blocks, kThreads, 0, (cudaStream_t)stream>>>(total4, H, W, C, in, out);
  return check(cudaGetLastError(), "k_lpips_maxpool2");
}

extern "C" GSB_API int gsb_lpips_head(int32_t V, int32_t H, int32_t W, int32_t C, const float* feats,
                                      const float* lin_w, int32_t layer, double* out, double* partials,
                                      gsb_stream_t stream) {
  if (V <= 0 || V > 65535 || H <= 0 || W <= 0 || (int64_t)H * W > INT32_MAX / 2 || C <= 0 || C % 32 != 0 ||
      layer < 0 || layer >= 5 || !feats || !lin_w || !out || !partials)
    return invalid("gsb_lpips_head: bad argument (C a multiple of 32, layer 0..4)");
  cudaStream_t st = (cudaStream_t)stream;
  gsb_count_launch(2);
  k_lpips_head<<<dim3(GSB_LPIPS_HEAD_PARTS, V), kThreads, 0, st>>>(V, H * W, C, feats, lin_w, partials);
  int rc = check(cudaGetLastError(), "k_lpips_head");
  if (rc != GSB_OK) return rc;
  k_lpips_head_reduce<<<V, GSB_LPIPS_HEAD_PARTS, 0, st>>>(layer, partials, out);
  return check(cudaGetLastError(), "k_lpips_head_reduce");
}
