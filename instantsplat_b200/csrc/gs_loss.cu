// Fused SSIM / L1 loss kernels for sm_90a (C ABI in include/gsb200.h).
//
// Replaces fused_ssim.fused_ssim (train.py:39-43,172-173; an empty submodule,
// rahul-goel/fused-ssim @ a7c48d6) whose semantics are those of the reference's PyTorch fallback
// utils/loss_utils.py:55-85: 11x11 Gaussian window sigma 1.5, zero "same"
// padding, C1 = 0.01^2, C2 = 0.03^2, per-channel (depthwise), mean over all elements -- plus
// l1_loss (utils/loss_utils.py:39-40) and the combine of train.py:176.
//
// One CTA = one 32x16 output tile of one channel: the (32+10)x(16+10) halo of both images is staged
// in shared memory once and the 11-tap window is applied separably with register tiling (4 outputs
// per thread horizontally from 128-bit shared loads, 2 outputs per thread vertically), so HBM
// traffic is the compulsory read of the two images plus the three partial-derivative maps written
// for the backward.
//
// The evaluation metrics (gsb_image_metrics_batch: train.py's training_report, metrics.py) are the same forward on
// clamped or 8-bit-quantised inputs, with per-CTA partial sums and a fixed-order reduction instead of atomics.
// gsb_frames_u8_batch writes that 8-bit quantisation out as interleaved RGB frames (render.py's save_image).
#include <cuda_runtime.h>
#include <stdio.h>

#include "../../include/gsb200.h"
#include "gs_math.cuh"

using gsb::fma2;
using gsb::mul2;

void gsb_set_error(const char* s);
void gsb_count_launch(int n);
int gsb_prof_begin(int id, cudaStream_t st);
void gsb_prof_end(int slot, cudaStream_t st);

namespace {

constexpr int TW = 32, TH = 16;     // output tile per CTA
constexpr int HALO = 5;
constexpr int EH = TH + 2 * HALO;   // 26 staged rows
constexpr int EWP = 44;             // 42 staged columns padded to a multiple of 4 (128-bit shared loads)
constexpr int HS = TW + 1;          // row stride of the horizontally filtered planes (conflict-free)
constexpr float C1 = 0.01f * 0.01f;
constexpr float C2 = 0.03f * 0.03f;

// normalised 1-D window exp(-(x-5)^2 / 4.5), built like loss_utils.gaussian() (fp32 sum)
__constant__ float c_win[11];
bool g_win_ready[64] = {};     // __constant__ memory is per device

int ensure_window() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (dev >= 0 && dev < 64 && g_win_ready[dev]) return 0;
  float w[11], s = 0.f;
  for (int i = 0; i < 11; ++i) { w[i] = (float)exp(-(double)((i - 5) * (i - 5)) / 4.5); s += w[i]; }
  for (int i = 0; i < 11; ++i) w[i] /= s;
  if (cudaMemcpyToSymbol(c_win, w, sizeof(w)) != cudaSuccess) return -1;
  if (dev >= 0 && dev < 64) g_win_ready[dev] = true;
  return 0;
}

__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x < 32) {
    r = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  }
  return r;   // valid in thread 0
}

// What the forward compares: the pixel values as they are (the training loss), clamped to [0, 1] (train.py's
// training_report), or through torchvision's save_image and to_tensor (render.py -> metrics.py):
// uint8(clamp(x * 255 + 0.5, 0, 255)) / 255 in fp32, truncating, so exact ties round up.
// NaN: the clamp keeps it, as torch.clamp does, so a diverged render reports NaN metrics rather than plausible
// finite ones (fminf / fmaxf alone would return the bound); save_image's quantisation makes it 0, as png8_level does.
enum { kInRaw = 0, kInClamp = GSB_METRIC_CLAMP, kInPng8 = GSB_METRIC_PNG8 };

// save_image's 8-bit level of x as a float in {0, ..., 255}: x.mul(255).add_(0.5).clamp_(0, 255).to(uint8) with each
// operation rounded as torch rounds it (no FMA contraction), truncating, so exact ties round up.  NaN gives 0.
__device__ __forceinline__ float png8_level(float x) {
  return truncf(fminf(fmaxf(__fadd_rn(__fmul_rn(x, 255.f), 0.5f), 0.f), 255.f));
}

template <int kIn>
__device__ __forceinline__ float metric_input(float x) {
  if constexpr (kIn == kInClamp) return isnan(x) ? x : fminf(fmaxf(x, 0.f), 1.f);
  if constexpr (kIn == kInPng8) return __fdiv_rn(png8_level(x), 255.f);
  return x;
}

// Stage the (TH+10) x (TW+10) halo of TWO planes into shared memory as interleaved float2 {a, b} (zero 'same'
// padding): one warp per row, lanes along x (two coalesced accesses per row and plane).  Fully unrolled with all
// global loads issued before the first shared store, so a lane has 16 loads in flight.  kIn: metric_input applied to
// every loaded pixel (the padding stays zero).
constexpr int kRowsPerWarp = (EH + 7) / 8;   // 4
struct HaloRegs { float a[kRowsPerWarp], b[kRowsPerWarp]; };

template <int kIn = kInRaw>
__device__ __forceinline__ void halo_load(HaloRegs& h, const float* __restrict__ src, int H, int W, int x0, int y0) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int xa = x0 - HALO + lane, xb = xa + 32;
  const bool xa_in = xa >= 0 && xa < W;
  const bool xb_in = lane < TW + 2 * HALO - 32 && xb < W;
#pragma unroll
  for (int i = 0; i < kRowsPerWarp; ++i) {
    const int r = warp + 8 * i;
    const int y = y0 + r - HALO;
    const bool yin = r < EH && y >= 0 && y < H;
    const float* row = src + (size_t)(yin ? y : 0) * W;
    h.a[i] = (yin && xa_in) ? metric_input<kIn>(__ldg(row + xa)) : 0.f;
    h.b[i] = (yin && xb_in) ? metric_input<kIn>(__ldg(row + xb)) : 0.f;
  }
}
// dst[r][x] = {p.(x), q.(x)}
__device__ __forceinline__ void halo_store2(const HaloRegs& p, const HaloRegs& q, float2 (*dst)[EWP]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < kRowsPerWarp; ++i) {
    const int r = warp + 8 * i;
    if (r < EH) {
      dst[r][lane] = make_float2(p.a[i], q.a[i]);
      if (lane < EWP - 32) dst[r][32 + lane] = make_float2(p.b[i], q.b[i]);
    }
  }
}
__device__ __forceinline__ void halo_store1(const HaloRegs& p, float (*dst)[EWP]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < kRowsPerWarp; ++i) {
    const int r = warp + 8 * i;
    if (r < EH) {
      dst[r][lane] = p.a[i];
      if (lane < EWP - 32) dst[r][32 + lane] = p.b[i];
    }
  }
}
__device__ __forceinline__ float2 bcast(float w) { return make_float2(w, w); }

// Register-tiled separable 11-tap filter: the five windowed statistics are carried as {E[a], E[b]}, {E[a^2], E[b^2]}
// (two float2 accumulators) and E[ab] (scalar).  Horizontal: thread -> (row, 4 adjacent columns), inputs fetched
// with seven 128-bit shared loads.  Vertical: thread -> (column, 2 adjacent rows).
// img planes [BC][H][W].  maps (optional) [3][BC][H][W].  sums[0] += sum|a-b| (if do_l1), sums[1] += sum ssim.
// kViews: a batch of views of C planes each (BC = V * C): plane z = v * C + c of img1 is compared with plane
// gt_row[v] * C + c of img2, and view v's sums go to sums[2v], sums[2v + 1].  Every plane keeps the single-view CTA
// split, so each view's partials are those of the single-view call.
// kIn != kInRaw (evaluation metrics, needs kViews): both planes go through metric_input<kIn>, and instead of adding
// to `sums` with atomics every CTA writes its own {sum|a-b|, sum ssim, sum (a-b)^2} (CTA sums in fp32, as above) to
// sums[3 * cta], cta = (bc * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x; k_metrics_reduce adds them up.
template <bool kViews = false, int kIn = kInRaw>
__global__ void __launch_bounds__(256, 4)
k_ssim_fwd(int H, int W, const float* __restrict__ img1, const float* __restrict__ img2,
           double* __restrict__ sums, float* __restrict__ maps, size_t plane_total, int do_l1, int C = 1,
           const int32_t* __restrict__ gt_row = nullptr) {
  static_assert(kIn == kInRaw || kViews, "the metric forward is the view-batched one");
  __shared__ __align__(16) float2 sAB[EH][EWP];
  __shared__ __align__(16) float2 sH1[EH][HS];     // {E_h[a], E_h[b]}
  __shared__ __align__(16) float2 sH2[EH][HS];     // {E_h[a^2], E_h[b^2]}
  __shared__ float sH3[EH][HS];                    // E_h[ab]
  __shared__ float red[8];
  const int bc = blockIdx.z;
  const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
  size_t gt_plane = bc;
  if constexpr (kViews) {
    const int v = bc / C;
    gt_plane = (size_t)__ldg(gt_row + v) * C + (bc - v * C);
    if constexpr (kIn == kInRaw) sums += 2 * v;
    else sums += 3 * (((size_t)bc * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x);
  }
  {
    HaloRegs ha, hb;
    halo_load<kIn>(ha, img1 + (size_t)bc * H * W, H, W, x0, y0);
    halo_load<kIn>(hb, img2 + gt_plane * H * W, H, W, x0, y0);
    halo_store2(ha, hb, sAB);
  }
  __syncthreads();
  if (threadIdx.x < EH * (TW / 4)) {
    const int r = threadIdx.x >> 3, c0 = (threadIdx.x & 7) * 4;
    float2 a1[4], a2[4];
    float a3[4];
#pragma unroll
    for (int o = 0; o < 4; ++o) { a1[o] = make_float2(0.f, 0.f); a2[o] = make_float2(0.f, 0.f); a3[o] = 0.f; }
#pragma unroll
    for (int q = 0; q < 7; ++q) {
      const float4 v = *reinterpret_cast<const float4*>(&sAB[r][c0 + 2 * q]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = 2 * q + h;
        const float2 ab = h ? make_float2(v.z, v.w) : make_float2(v.x, v.y);
        const float2 sq = mul2(ab, ab);
        const float x = ab.x * ab.y;
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const int t = i - o;
          if (t >= 0 && t < 11) {
            const float w = c_win[t];
            a1[o] = fma2(bcast(w), ab, a1[o]);
            a2[o] = fma2(bcast(w), sq, a2[o]);
            a3[o] = fmaf(w, x, a3[o]);
          }
        }
      }
    }
#pragma unroll
    for (int o = 0; o < 4; ++o) { sH1[r][c0 + o] = a1[o]; sH2[r][c0 + o] = a2[o]; sH3[r][c0 + o] = a3[o]; }
  }
  __syncthreads();
  const int tx = threadIdx.x & 31, ty = (threadIdx.x >> 5) * 2;
  float2 m[2], e[2];
  float e12[2];
#pragma unroll
  for (int o = 0; o < 2; ++o) { m[o] = make_float2(0.f, 0.f); e[o] = make_float2(0.f, 0.f); e12[o] = 0.f; }
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    const float2 v1 = sH1[ty + i][tx], v2 = sH2[ty + i][tx];
    const float v3 = sH3[ty + i][tx];
#pragma unroll
    for (int o = 0; o < 2; ++o) {
      const int t = i - o;
      if (t >= 0 && t < 11) {
        const float w = c_win[t];
        m[o] = fma2(bcast(w), v1, m[o]);
        e[o] = fma2(bcast(w), v2, e[o]);
        e12[o] = fmaf(w, v3, e12[o]);
      }
    }
  }
  float ssim_v = 0.f, l1_v = 0.f, sq_v = 0.f;
#pragma unroll
  for (int o = 0; o < 2; ++o) {
    const int x = x0 + tx, y = y0 + ty + o;
    if (x < W && y < H) {
      const float mu1 = m[o].x, mu2 = m[o].y;
      float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
      float s1 = e[o].x - mu1_sq, s2 = e[o].y - mu2_sq, s12 = e12[o] - mu12;
      float A1 = 2.f * mu12 + C1, A2 = 2.f * s12 + C2, B1 = mu1_sq + mu2_sq + C1, B2 = s1 + s2 + C2;
      float inv = 1.f / (B1 * B2);
      float sv = A1 * A2 * inv;
      ssim_v += sv;
      if (maps) {
        size_t off = (size_t)bc * H * W + (size_t)y * W + x;
        maps[off] = 2.f * mu2 * (A2 - A1) * inv - sv * 2.f * mu1 * (B2 - B1) * inv;   // d/dmu1
        maps[plane_total + off] = -sv / B2;                                       // d/dE[x^2]
        maps[2 * plane_total + off] = 2.f * A1 * inv;                             // d/dE[xy]
      }
      if (do_l1) { const float2 c = sAB[ty + o + HALO][tx + HALO]; l1_v += fabsf(c.x - c.y); }
      if constexpr (kIn != kInRaw) {
        const float2 c = sAB[ty + o + HALO][tx + HALO];
        const float d = c.x - c.y;
        sq_v = fmaf(d, d, sq_v);
      }
    }
  }
  if constexpr (kIn != kInRaw) {
    const float s = block_sum(ssim_v, red);
    __syncthreads();
    const float l = block_sum(l1_v, red);
    __syncthreads();
    const float q = block_sum(sq_v, red);
    if (threadIdx.x == 0) { sums[0] = (double)l; sums[1] = (double)s; sums[2] = (double)q; }
    return;
  }
  float s = block_sum(ssim_v, red);
  if (threadIdx.x == 0) atomicAdd(sums + 1, (double)s);
  if (do_l1) {
    __syncthreads();
    float l = block_sum(l1_v, red);
    if (threadIdx.x == 0) atomicAdd(sums + 0, (double)l);
  }
}

// out = ssim_scale * (conv(m_mu) + 2 x conv(m_s1) + y conv(m_s12)) [* *dyn_scale] + l1_scale * sign(x-y)
// The first two maps travel as one float2 through both filter passes.  kViews: y from plane gt_row[v] * C + c of img2
// (as in k_ssim_fwd<true>).
template <bool kViews = false>
__global__ void __launch_bounds__(256, 5)
k_ssim_bwd(int H, int W, const float* __restrict__ img1, const float* __restrict__ img2,
           const float* __restrict__ maps, size_t plane_total, float ssim_scale,
           const float* __restrict__ dyn_scale, float l1_scale, float* __restrict__ out, int C = 1,
           const int32_t* __restrict__ gt_row = nullptr) {
  __shared__ __align__(16) float2 sM12[EH][EWP];
  __shared__ __align__(16) float sM3[EH][EWP];
  __shared__ __align__(16) float2 sH12[EH][HS];
  __shared__ float sH3[EH][HS];
  const int bc = blockIdx.z;
  const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
  const size_t pbase = (size_t)bc * H * W;
  size_t gbase = pbase;
  if constexpr (kViews) {
    const int v = bc / C;
    gbase = ((size_t)__ldg(gt_row + v) * C + (bc - v * C)) * H * W;
  }
  {
    HaloRegs h0, h1, h2;
    halo_load(h0, maps + pbase, H, W, x0, y0);
    halo_load(h1, maps + plane_total + pbase, H, W, x0, y0);
    halo_load(h2, maps + 2 * plane_total + pbase, H, W, x0, y0);
    halo_store2(h0, h1, sM12);
    halo_store1(h2, sM3);
  }
  __syncthreads();
  if (threadIdx.x < EH * (TW / 4)) {
    const int r = threadIdx.x >> 3, c0 = (threadIdx.x & 7) * 4;
    float2 a12[4];
    float a3[4];
#pragma unroll
    for (int o = 0; o < 4; ++o) { a12[o] = make_float2(0.f, 0.f); a3[o] = 0.f; }
    float m3[16];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float4 v = *reinterpret_cast<const float4*>(&sM3[r][c0 + 4 * u]);
      m3[4 * u] = v.x; m3[4 * u + 1] = v.y; m3[4 * u + 2] = v.z; m3[4 * u + 3] = v.w;
    }
#pragma unroll
    for (int q = 0; q < 7; ++q) {
      const float4 v = *reinterpret_cast<const float4*>(&sM12[r][c0 + 2 * q]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = 2 * q + h;
        const float2 p = h ? make_float2(v.z, v.w) : make_float2(v.x, v.y);
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const int t = i - o;
          if (t >= 0 && t < 11) {
            const float w = c_win[t];
            a12[o] = fma2(bcast(w), p, a12[o]);
            a3[o] = fmaf(w, m3[i], a3[o]);
          }
        }
      }
    }
#pragma unroll
    for (int o = 0; o < 4; ++o) { sH12[r][c0 + o] = a12[o]; sH3[r][c0 + o] = a3[o]; }
  }
  __syncthreads();
  const int tx = threadIdx.x & 31, ty = (threadIdx.x >> 5) * 2;
  float2 g12[2];
  float g3[2];
#pragma unroll
  for (int o = 0; o < 2; ++o) { g12[o] = make_float2(0.f, 0.f); g3[o] = 0.f; }
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    const float2 v12 = sH12[ty + i][tx];
    const float v3 = sH3[ty + i][tx];
#pragma unroll
    for (int o = 0; o < 2; ++o) {
      const int t = i - o;
      if (t >= 0 && t < 11) {
        const float w = c_win[t];
        g12[o] = fma2(bcast(w), v12, g12[o]);
        g3[o] = fmaf(w, v3, g3[o]);
      }
    }
  }
  const float sc = ssim_scale * (dyn_scale ? *dyn_scale : 1.f);
#pragma unroll
  for (int o = 0; o < 2; ++o) {
    const int x = x0 + tx, y = y0 + ty + o;
    if (x < W && y < H) {
      size_t off = pbase + (size_t)y * W + x;
      float xv = img1[off], yv = img2[gbase + (size_t)y * W + x];
      float g = sc * (g12[o].x + 2.f * xv * g12[o].y + yv * g3[o]);
      if (l1_scale != 0.f) {
        float df = xv - yv;
        g += l1_scale * (df > 0.f ? 1.f : (df < 0.f ? -1.f : 0.f));
      }
      out[off] = g;
    }
  }
}

// One CTA per view: out[v] = {sum|a-b|, sum ssim, sum (a-b)^2 of each channel} from the view's C * T CTA partials
// (T tiles per plane, laid out as k_ssim_fwd<true, kIn> writes them).  Every sum is taken in fp64 in one fixed order
// (thread t adds items t, t + 256, ...; then a fixed tree), so a view's result depends on its own partials only.
constexpr int kReduceThreads = 256;
__global__ void __launch_bounds__(kReduceThreads)
k_metrics_reduce(int C, int T, const double* __restrict__ partials, double* __restrict__ out) {
  __shared__ double red[kReduceThreads];
  const int v = blockIdx.x;
  const double* p = partials + (size_t)v * C * T * 3;
  for (int j = 0; j < 2 + C; ++j) {
    // j = 0, 1: l1 / ssim over all C * T CTAs of the view; j >= 2: squared error over the T CTAs of channel j - 2
    const int n = j < 2 ? C * T : T;
    const double* q = j < 2 ? p + j : p + (size_t)(j - 2) * T * 3 + 2;
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += kReduceThreads) s += q[(size_t)3 * i];
    red[threadIdx.x] = s;
    __syncthreads();
#pragma unroll
    for (int o = kReduceThreads / 2; o > 0; o >>= 1) {
      if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
      __syncthreads();
    }
    if (threadIdx.x == 0) out[(size_t)v * (2 + C) + j] = red[0];
    __syncthreads();
  }
}

// save_image's 8-bit frames: img [V, 3, H, W] fp32 -> out [V, H, W, 3] uint8, png8_level of every value with the three
// channels interleaved per pixel.  Grid (ceil(H W / 1024), V): thread t of view v = blockIdx.y takes the 4 pixels
// p = 4t .. 4t + 3 of that view.  kVec (H W % 4 == 0, img 16-byte and out 4-byte aligned): one float4 load per channel
// plane and the 12 interleaved bytes as three uint32 stores; 12 bytes read and 3 written per pixel, nothing else.
// Otherwise the planes of a view start at misaligned addresses: scalar loads and byte stores, stopping at the view's
// last pixel (the tail of a group of 4).
constexpr int kFrameThreads = 256;

__device__ __forceinline__ uint32_t png8_byte(float x) { return __float2uint_rz(png8_level(x)); }

template <bool kVec>
__global__ void __launch_bounds__(kFrameThreads)
k_frames_u8(int HW, const float* __restrict__ img, uint8_t* __restrict__ out) {
  const int p = 4 * (blockIdx.x * kFrameThreads + threadIdx.x);
  if (p >= HW) return;
  const size_t pix = (size_t)blockIdx.y * HW + p;            // first pixel of the group in [V, H, W]
  const float* src = img + (size_t)blockIdx.y * 3 * HW + p;   // its red value
  if constexpr (kVec) {
    const float4 r = __ldg(reinterpret_cast<const float4*>(src));
    const float4 g = __ldg(reinterpret_cast<const float4*>(src + HW));
    const float4 b = __ldg(reinterpret_cast<const float4*>(src + 2 * (size_t)HW));
    uint32_t* dst = reinterpret_cast<uint32_t*>(out + 3 * pix);   // little endian: byte k of the group is bits 8k
    dst[0] = png8_byte(r.x) | png8_byte(g.x) << 8 | png8_byte(b.x) << 16 | png8_byte(r.y) << 24;
    dst[1] = png8_byte(g.y) | png8_byte(b.y) << 8 | png8_byte(r.z) << 16 | png8_byte(g.z) << 24;
    dst[2] = png8_byte(b.z) | png8_byte(r.w) << 8 | png8_byte(g.w) << 16 | png8_byte(b.w) << 24;
  } else {
    const int n = min(4, HW - p);
    for (int k = 0; k < n; ++k) {
      uint8_t* d = out + 3 * (pix + k);
      d[0] = (uint8_t)png8_byte(__ldg(src + k));
      d[1] = (uint8_t)png8_byte(__ldg(src + HW + k));
      d[2] = (uint8_t)png8_byte(__ldg(src + 2 * (size_t)HW + k));
    }
  }
}

int check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return GSB_OK;
  char buf[256];
  snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  gsb_set_error(buf);
  return GSB_ERR_CUDA;
}

}  // namespace

extern "C" GSB_API int gsb_ssim_forward(int32_t BC, int32_t H, int32_t W, const float* img1, const float* img2,
                                double* ssim_sum2, float* maps, gsb_stream_t stream) {
  if (BC <= 0 || H <= 0 || W <= 0 || !img1 || !img2 || !ssim_sum2) { gsb_set_error("gsb_ssim_forward: bad argument"); return GSB_ERR_INVALID; }
  if (ensure_window()) return check(cudaGetLastError(), "window upload");
  dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, BC);
  gsb_count_launch(1);
  int slot = gsb_prof_begin(GSB_K_LOSS_FWD, (cudaStream_t)stream);
  k_ssim_fwd<<<grid, 256, 0, (cudaStream_t)stream>>>(H, W, img1, img2, ssim_sum2, maps, (size_t)BC * H * W, 0);
  gsb_prof_end(slot, (cudaStream_t)stream);
  return check(cudaGetLastError(), "k_ssim_fwd");
}

extern "C" GSB_API int gsb_ssim_backward(int32_t BC, int32_t H, int32_t W, const float* img1, const float* img2,
                                 const float* maps, float scale_host, const float* dL_dmean_scale,
                                 float* dL_dimg1, gsb_stream_t stream) {
  if (BC <= 0 || H <= 0 || W <= 0 || !img1 || !img2 || !maps || !dL_dimg1) { gsb_set_error("gsb_ssim_backward: bad argument"); return GSB_ERR_INVALID; }
  if (ensure_window()) return check(cudaGetLastError(), "window upload");
  dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, BC);
  gsb_count_launch(1);
  int slot = gsb_prof_begin(GSB_K_LOSS_BWD, (cudaStream_t)stream);
  k_ssim_bwd<<<grid, 256, 0, (cudaStream_t)stream>>>(H, W, img1, img2, maps, (size_t)BC * H * W, scale_host,
                                                     dL_dmean_scale, 0.f, dL_dimg1);
  gsb_prof_end(slot, (cudaStream_t)stream);
  return check(cudaGetLastError(), "k_ssim_bwd");
}

extern "C" GSB_API int gsb_loss_forward(int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                                double* sums, float* maps, gsb_stream_t stream) {
  if (C <= 0 || H <= 0 || W <= 0 || !img || !gt || !sums || !maps) { gsb_set_error("gsb_loss_forward: bad argument"); return GSB_ERR_INVALID; }
  if (ensure_window()) return check(cudaGetLastError(), "window upload");
  dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, C);
  gsb_count_launch(1);
  int slot = gsb_prof_begin(GSB_K_LOSS_FWD, (cudaStream_t)stream);
  k_ssim_fwd<<<grid, 256, 0, (cudaStream_t)stream>>>(H, W, img, gt, sums, maps, (size_t)C * H * W, 1);
  gsb_prof_end(slot, (cudaStream_t)stream);
  return check(cudaGetLastError(), "k_loss_fwd");
}

extern "C" GSB_API int gsb_loss_backward(int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                                 const float* maps, float lambda_dssim, float* dL_dimg, gsb_stream_t stream) {
  if (C <= 0 || H <= 0 || W <= 0 || !img || !gt || !maps || !dL_dimg) { gsb_set_error("gsb_loss_backward: bad argument"); return GSB_ERR_INVALID; }
  if (ensure_window()) return check(cudaGetLastError(), "window upload");
  const double N = (double)C * H * W;
  dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, C);
  gsb_count_launch(1);
  int slot = gsb_prof_begin(GSB_K_LOSS_BWD, (cudaStream_t)stream);
  k_ssim_bwd<<<grid, 256, 0, (cudaStream_t)stream>>>(H, W, img, gt, maps, (size_t)C * H * W,
                                                     (float)(-(double)lambda_dssim / N), nullptr,
                                                     (float)((1.0 - (double)lambda_dssim) / N), dL_dimg);
  gsb_prof_end(slot, (cudaStream_t)stream);
  return check(cudaGetLastError(), "k_loss_bwd");
}

// The loss of V views [V, C, H, W] in one launch each: view v against target plane block gt_row[v] of gt (device int32
// [V]), its sums at sums[2v] and sums[2v + 1], its dL/dimg scaled by the single-view 1/N (N = C H W).
extern "C" GSB_API int gsb_loss_forward_batch(int32_t V, int32_t C, int32_t H, int32_t W, const float* img,
                                              const float* gt, const int32_t* gt_row, double* sums, float* maps,
                                              gsb_stream_t stream) {
  if (V <= 0 || V > 65535 / (C > 0 ? C : 1) || C <= 0 || H <= 0 || W <= 0 || !img || !gt || !gt_row || !sums || !maps) {
    gsb_set_error("gsb_loss_forward_batch: bad argument");
    return GSB_ERR_INVALID;
  }
  if (ensure_window()) return check(cudaGetLastError(), "window upload");
  dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, V * C);
  gsb_count_launch(1);
  int slot = gsb_prof_begin(GSB_K_LOSS_FWD, (cudaStream_t)stream);
  k_ssim_fwd<true><<<grid, 256, 0, (cudaStream_t)stream>>>(H, W, img, gt, sums, maps, (size_t)V * C * H * W, 1, C,
                                                            gt_row);
  gsb_prof_end(slot, (cudaStream_t)stream);
  return check(cudaGetLastError(), "k_loss_fwd_batch");
}

extern "C" GSB_API int gsb_loss_backward_batch(int32_t V, int32_t C, int32_t H, int32_t W, const float* img,
                                               const float* gt, const int32_t* gt_row, const float* maps,
                                               float lambda_dssim, float* dL_dimg, gsb_stream_t stream) {
  if (V <= 0 || V > 65535 / (C > 0 ? C : 1) || C <= 0 || H <= 0 || W <= 0 || !img || !gt || !gt_row || !maps ||
      !dL_dimg) {
    gsb_set_error("gsb_loss_backward_batch: bad argument");
    return GSB_ERR_INVALID;
  }
  if (ensure_window()) return check(cudaGetLastError(), "window upload");
  const double N = (double)C * H * W;
  dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, V * C);
  gsb_count_launch(1);
  int slot = gsb_prof_begin(GSB_K_LOSS_BWD, (cudaStream_t)stream);
  k_ssim_bwd<true><<<grid, 256, 0, (cudaStream_t)stream>>>(H, W, img, gt, maps, (size_t)V * C * H * W,
                                                            (float)(-(double)lambda_dssim / N), nullptr,
                                                            (float)((1.0 - (double)lambda_dssim) / N), dL_dimg, C,
                                                            gt_row);
  gsb_prof_end(slot, (cudaStream_t)stream);
  return check(cudaGetLastError(), "k_loss_bwd_batch");
}

// Evaluation metrics of V views (include/gsb200.h): k_ssim_fwd<true, mode> writes one partial per CTA to `scratch`,
// k_metrics_reduce adds each view's partials in a fixed order into out[v].  No atomics, so every view's result is
// bit-identical from run to run and whatever else is in the batch.
extern "C" GSB_API size_t gsb_image_metrics_scratch_bytes(int32_t V, int32_t C, int32_t H, int32_t W) {
  if (V <= 0 || C <= 0 || H <= 0 || W <= 0) return 0;
  const size_t T = (size_t)((W + TW - 1) / TW) * ((H + TH - 1) / TH);
  return (size_t)V * C * T * 3 * sizeof(double);
}

extern "C" GSB_API int gsb_image_metrics_batch(int32_t V, int32_t C, int32_t H, int32_t W, const float* img,
                                               const float* gt, const int32_t* gt_row, int32_t mode, double* out,
                                               void* scratch, size_t scratch_bytes, gsb_stream_t stream) {
  if (V <= 0 || C <= 0 || V > 65535 / C || H <= 0 || W <= 0 || !img || !gt || !gt_row || !out || !scratch ||
      (mode != GSB_METRIC_CLAMP && mode != GSB_METRIC_PNG8)) {
    gsb_set_error("gsb_image_metrics_batch: bad argument");
    return GSB_ERR_INVALID;
  }
  if (scratch_bytes < gsb_image_metrics_scratch_bytes(V, C, H, W)) {
    gsb_set_error("gsb_image_metrics_batch: scratch smaller than gsb_image_metrics_scratch_bytes()");
    return GSB_ERR_INVALID;
  }
  if (ensure_window()) return check(cudaGetLastError(), "window upload");
  dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, V * C);
  double* part = static_cast<double*>(scratch);
  cudaStream_t st = (cudaStream_t)stream;
  gsb_count_launch(2);
  if (mode == GSB_METRIC_CLAMP)
    k_ssim_fwd<true, kInClamp><<<grid, 256, 0, st>>>(H, W, img, gt, part, nullptr, 0, 1, C, gt_row);
  else
    k_ssim_fwd<true, kInPng8><<<grid, 256, 0, st>>>(H, W, img, gt, part, nullptr, 0, 1, C, gt_row);
  int rc = check(cudaGetLastError(), "k_metrics_fwd");
  if (rc != GSB_OK) return rc;
  k_metrics_reduce<<<V, kReduceThreads, 0, st>>>(C, (int)(grid.x * grid.y), part, out);
  return check(cudaGetLastError(), "k_metrics_reduce");
}

extern "C" GSB_API int gsb_frames_u8_batch(int32_t V, int32_t H, int32_t W, const float* img, uint8_t* out,
                                           gsb_stream_t stream) {
  if (V <= 0 || V > 65535 || H <= 0 || W <= 0 || (int64_t)H * W > (int64_t)INT32_MAX - 3 || !img || !out) {
    gsb_set_error("gsb_frames_u8_batch: bad argument");
    return GSB_ERR_INVALID;
  }
  const int HW = H * W;
  const bool vec = HW % 4 == 0 && reinterpret_cast<uintptr_t>(img) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0;
  dim3 grid((unsigned)((HW + 4 * kFrameThreads - 1) / (4 * kFrameThreads)), (unsigned)V);
  cudaStream_t st = (cudaStream_t)stream;
  gsb_count_launch(1);
  if (vec)
    k_frames_u8<true><<<grid, kFrameThreads, 0, st>>>(HW, img, out);
  else
    k_frames_u8<false><<<grid, kFrameThreads, 0, st>>>(HW, img, out);
  return check(cudaGetLastError(), "k_frames_u8");
}
