// Per-tile alpha blend of the rasterizer, forward and backward (SURVEY.md Appendix A.2.10 / A.3;
// reference call site gaussian_renderer/__init__.py:126-135).
//
//   k_blend_fwd2 / k_blend_bwd2   CTA = 16x16 tile (4 warps), warp = 8x8 block, TWO pixels per lane sharing dx
//                                 (per-pair math on float2 lanes); per-warp
//                                 ballot-compacted exact sub-tile culling.  Staging, three-deep software pipeline:
//                                 the tile's sorted ID chunk arrives by a TMA bulk copy (cp.async.bulk + mbarrier)
//                                 two chunks ahead, the 48-byte splat records of those ids are GATHERED with
//                                 cp.async (LDGSTS) out of the record table (mostly L2 hits) one chunk ahead, the
//                                 current chunk is blended from shared memory.  No per-instance copy of the records
//                                 is ever written to HBM, and nothing is fetched for the part of a list that early
//                                 termination never reaches.
//   k_blend_fwd / k_blend_bwd     v1: one pixel per lane, 8 warps per tile, cooperative staging -- the first
//                                 correct version, kept as the in-library cross-check (gsb_set_option)
#include "gs_internal.cuh"
#include "gs_tma.cuh"

using namespace gsb;

namespace {

constexpr float kLn2 = 0.6931471805599453f;

#ifndef GSB_CHUNK
#define GSB_CHUNK 224
#endif
#ifndef GSB_FWD_MINB
#define GSB_FWD_MINB 8
#endif
#ifndef GSB_BWD_CHUNK
#define GSB_BWD_CHUNK 192
#endif
#ifndef GSB_BWD_MINB
#define GSB_BWD_MINB 6
#endif
constexpr int kChunk1 = 256;           // v1 blend kernels: one entry per thread
constexpr int kChunk = GSB_CHUNK;      // slab entries staged per step in the forward (and the butterfly backward)
// The batched backward (k_blend_bwd2<..., BATCH>) adds 15.2 KB of batch rows per CTA; with shorter chunks its CTA
// (35.5 KB + 1 KB reserved) fits GSB_BWD_MINB = 6 times into an SM's 228 KB, and 6 x 128 threads x 80 registers
// fit.  The butterfly instance keeps the forward's chunk and 8 CTAs / SM.
constexpr int kChunkB = GSB_BWD_CHUNK;
constexpr int kBwdMinBFly = 8;

// ------------------------------------------------------------------------------------------
// blend
// ------------------------------------------------------------------------------------------
struct PairEval { float dx, dy, power, G, alpha; };   // power is in the log2 domain (power * log2 e)

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ PairEval pair_eval(const float4& e0, const float4& e1, float fx, float fy) {
  PairEval r;
  r.dx = e0.x - fx;
  r.dy = e0.y - fy;
  r.power = e0.z * r.dx * r.dx + (e0.w * r.dx + e1.x * r.dy) * r.dy;
  r.G = ex2_approx(r.power);   // MUFU.EX2 directly (valid pairs have power >= -8)
  r.alpha = fminf(0.99f, e1.y * r.G);
  return r;
}

// cull test on a slab entry: q' = -(A'dx^2 + B'dxdy + C'dy^2) = q * log2(e)/2 against qthr' = qthr * log2(e)/2
__device__ __forceinline__ bool slab_may_contribute(const float4& e0, const float4& e1, float rx0, float ry0,
                                                    float rx1, float ry1) {
  return rect_may_contribute(e0.x, e0.y, -e0.z, -0.5f * e0.w, -e1.x, e1.z, rx0, ry0, rx1, ry1);
}

// Batches of V views: the grid is (tiles of one frame, V), so CTA (t, v) blends local tile t of view v.  Returns the
// global tile index v * ntiles + t (the view's binning lists) and moves the per-pixel buffers to the view's frame; once
// per CTA, so the per-pair work is the single-view one.
__device__ __forceinline__ int view_tile(int W, int H, float* __restrict__& color, float* __restrict__& final_T,
                                         uint32_t* __restrict__& n_contrib) {
  const size_t hw = (size_t)W * H, v = blockIdx.y;
  color += 3 * hw * v;
  final_T += hw * v;
  n_contrib += hw * v;
  return (int)(v * gridDim.x) + (int)blockIdx.x;
}
__device__ __forceinline__ int view_tile_bwd(int W, int H, const float* __restrict__& dL, const float* __restrict__& final_T,
                                             const uint32_t* __restrict__& n_contrib, const uint32_t* __restrict__& dscale) {
  const size_t hw = (size_t)W * H, v = blockIdx.y;
  dL += 3 * hw * v;
  final_T += hw * v;
  n_contrib += hw * v;
  dscale += v;
  return (int)(v * gridDim.x) + (int)blockIdx.x;
}

__global__ void __launch_bounds__(kThreads)
k_blend_fwd(const uint2* __restrict__ ranges, const uint32_t* __restrict__ ids, const float4* __restrict__ rec,
            const float* __restrict__ bg, int W, int H, int gx,
            float* __restrict__ out_color, float* __restrict__ final_T, uint32_t* __restrict__ n_contrib) {
  __shared__ float4 sm0[kChunk1], sm1[kChunk1], sm2[kChunk1];
  const int tile = view_tile(W, H, out_color, final_T, n_contrib);
  const int tx = blockIdx.x % gx, ty = blockIdx.x / gx;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sx0 = tx * kBlock + (warp & 1) * 8, sy0 = ty * kBlock + (warp >> 1) * 4;
  const int px = sx0 + (lane & 7), py = sy0 + (lane >> 3);
  const bool inside = px < W && py < H;
  const float fx = (float)px, fy = (float)py;
  const float rx0 = (float)sx0, ry0 = (float)sy0;
  const float rx1 = (float)min(sx0 + 7, W - 1), ry1 = (float)min(sy0 + 3, H - 1);
  const uint2 rg = ranges[tile];
  const int n = (int)(rg.y - rg.x);
  float T = 1.f, Cr = 0.f, Cg = 0.f, Cb = 0.f;
  uint32_t last = 0;
  bool done = !inside;
  bool wdone = !(sx0 < W && sy0 < H);
  for (int base = 0; base < n; base += kChunk1) {
    const int cnt = min(kChunk1, n - base);
    if ((int)threadIdx.x < cnt) {
      const float4* r = rec + 3 * (size_t)ids[(size_t)rg.x + base + threadIdx.x];
      sm0[threadIdx.x] = r[0];
      sm1[threadIdx.x] = r[1];
      sm2[threadIdx.x] = r[2];
    }
    __syncthreads();
    if (!wdone) {
      for (int b = 0; b < cnt; b += 32) {
        const int j = b + lane;
        bool hit = false;
        if (j < cnt) {
          float4 e0 = sm0[j], e1 = sm1[j];
          hit = slab_may_contribute(e0, e1, rx0, ry0, rx1, ry1);
        }
        unsigned mask = __ballot_sync(0xffffffffu, hit);
        while (mask) {
          const int k = __ffs(mask) - 1;
          mask &= mask - 1;
          const float4 e0 = sm0[b + k], e1 = sm1[b + k];
          PairEval pe = pair_eval(e0, e1, fx, fy);
          bool valid = !done && pe.power <= 0.f && pe.alpha >= kAlphaMin;
          float testT = T * (1.f - pe.alpha);
          if (valid && testT < kTEps) { done = true; valid = false; }
          if (valid) {
            const float4 c = sm2[b + k];
            float w = pe.alpha * T;
            Cr += c.x * w; Cg += c.y * w; Cb += c.z * w;
            T = testT;
            last = (uint32_t)(base + b + k + 1);
          }
        }
        if (__all_sync(0xffffffffu, done)) { wdone = true; break; }
      }
    }
    if (__syncthreads_and(wdone)) break;
  }
  if (inside) {
    size_t pix = (size_t)py * W + px, hw = (size_t)W * H;
    final_T[pix] = T;
    n_contrib[pix] = last;
    out_color[pix] = Cr + T * bg[0];
    out_color[hw + pix] = Cg + T * bg[1];
    out_color[2 * hw + pix] = Cb + T * bg[2];
  }
}

// *dscale = max |dL[i]| (float bits of non-negative floats order like the floats, so the integer max is exact and
// independent of the order of the atomics); grid y = view: dscale[v] over the view's n values
__global__ void __launch_bounds__(kThreads) k_abs_max(size_t n, const float* __restrict__ dL, uint32_t* __restrict__ dscale) {
  dL += n * blockIdx.y;
  dscale += blockIdx.y;
  float m = 0.f;
  for (size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x; e < n; e += (size_t)gridDim.x * kThreads)
    m = fmaxf(m, fabsf(__ldg(dL + e)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(dscale, __float_as_uint(m));
}

// Adds the warp's totals to a Gaussian's fixed-point slots.  After warp_reduce9 / warp_reduce8, lane 4i holds total i
// (i < 8) in v0 and every lane holds total 8 in v8; lane 1 adds slot 8 when `ninth`.
__device__ __forceinline__ void flush_fixed(unsigned long long* dst, float v0, float v8, float extent, float inv_m, int lane,
                                            bool ninth) {
  if ((lane & 3) == 0 || (ninth && lane == 1)) {
    const int slot = (lane & 3) ? 8 : lane >> 2;
    atomicAdd(dst + slot, fix_encode((lane & 3) ? v8 : v0, fix_scale(slot, extent, inv_m)));
  }
}

// Reduce 9 per-lane values over the warp with 14 shuffles.  On return, lane l with (l & 3) == 0
// holds the total of v[l >> 2] in v[0]; every lane holds the total of v[8] in v[8].
__device__ __forceinline__ void warp_reduce9(float* v, int lane) {
  const unsigned full = 0xffffffffu;
  float b[4], c[2], d;
  {
    const bool hi = lane & 16;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float send = hi ? v[k] : v[k + 4];
      float keep = hi ? v[k + 4] : v[k];
      b[k] = keep + __shfl_xor_sync(full, send, 16);
    }
  }
  {
    const bool hi = lane & 8;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      float send = hi ? b[k] : b[k + 2];
      float keep = hi ? b[k + 2] : b[k];
      c[k] = keep + __shfl_xor_sync(full, send, 8);
    }
  }
  {
    const bool hi = lane & 4;
    float send = hi ? c[0] : c[1];
    float keep = hi ? c[1] : c[0];
    d = keep + __shfl_xor_sync(full, send, 4);
  }
  d += __shfl_xor_sync(full, d, 2);
  d += __shfl_xor_sync(full, d, 1);
  v[0] = d;
  float e = v[8];
  e += __shfl_xor_sync(full, e, 16);
  e += __shfl_xor_sync(full, e, 8);
  e += __shfl_xor_sync(full, e, 4);
  e += __shfl_xor_sync(full, e, 2);
  e += __shfl_xor_sync(full, e, 1);
  v[8] = e;
}

// Same butterfly without the ninth value.
__device__ __forceinline__ void warp_reduce8(float* v, int lane) {
  const unsigned full = 0xffffffffu;
  float b[4], c[2], d;
  {
    const bool hi = lane & 16;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float send = hi ? v[k] : v[k + 4];
      float keep = hi ? v[k + 4] : v[k];
      b[k] = keep + __shfl_xor_sync(full, send, 16);
    }
  }
  {
    const bool hi = lane & 8;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      float send = hi ? b[k] : b[k + 2];
      float keep = hi ? b[k + 2] : b[k];
      c[k] = keep + __shfl_xor_sync(full, send, 8);
    }
  }
  {
    const bool hi = lane & 4;
    float send = hi ? c[0] : c[1];
    float keep = hi ? c[1] : c[0];
    d = keep + __shfl_xor_sync(full, send, 4);
  }
  d += __shfl_xor_sync(full, d, 2);
  d += __shfl_xor_sync(full, d, 1);
  v[0] = d;
}

__global__ void __launch_bounds__(kThreads)
k_blend_bwd(const uint2* __restrict__ ranges, const uint32_t* __restrict__ ids, const float4* __restrict__ rec,
            const float* __restrict__ bg, int W, int H, int gx,
            const float* __restrict__ final_T, const uint32_t* __restrict__ n_contrib,
            const float* __restrict__ dL_dpix, unsigned long long* __restrict__ dacc, const uint32_t* __restrict__ dscale) {
  __shared__ float4 sm0[kChunk1], sm1[kChunk1], sm2[kChunk1];
  __shared__ int s_bmax;
  const int tile = view_tile_bwd(W, H, dL_dpix, final_T, n_contrib, dscale);
  const float inv_m = fix_inv_m(dscale);
  const int tx = blockIdx.x % gx, ty = blockIdx.x / gx;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sx0 = tx * kBlock + (warp & 1) * 8, sy0 = ty * kBlock + (warp >> 1) * 4;
  const int px = sx0 + (lane & 7), py = sy0 + (lane >> 3);
  const bool inside = px < W && py < H;
  const float fx = (float)px, fy = (float)py;
  const float rx0 = (float)sx0, ry0 = (float)sy0;
  const float rx1 = (float)min(sx0 + 7, W - 1), ry1 = (float)min(sy0 + 3, H - 1);
  const uint2 rg = ranges[tile];
  const size_t pix = (size_t)py * W + px, hw = (size_t)W * H;
  const float T_final = inside ? final_T[pix] : 0.f;
  const int last_contrib = inside ? (int)n_contrib[pix] : 0;
  float dLr = 0.f, dLg = 0.f, dLb = 0.f;
  if (inside) { dLr = dL_dpix[pix]; dLg = dL_dpix[hw + pix]; dLb = dL_dpix[2 * hw + pix]; }
  const float bg_dot = bg[0] * dLr + bg[1] * dLg + bg[2] * dLb;
  int wmax = last_contrib;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
  if (threadIdx.x == 0) s_bmax = 0;
  __syncthreads();
  if (lane == 0) atomicMax(&s_bmax, wmax);
  __syncthreads();
  const int bmax = s_bmax;
  float T = T_final;
  float acc_r = 0.f, acc_g = 0.f, acc_b = 0.f, last_alpha = 0.f, last_r = 0.f, last_g = 0.f, last_b = 0.f;
  const int nchunks = (bmax + kChunk1 - 1) / kChunk1;
  for (int ch = nchunks - 1; ch >= 0; --ch) {
    const int base = ch * kChunk1;
    const int cnt = min(kChunk1, bmax - base);
    if ((int)threadIdx.x < cnt) {
      const float4* r = rec + 3 * (size_t)ids[(size_t)rg.x + base + threadIdx.x];
      sm0[threadIdx.x] = r[0];
      sm1[threadIdx.x] = r[1];
      sm2[threadIdx.x] = r[2];
    }
    __syncthreads();
    if (base < wmax) {
      for (int b = (cnt - 1) & ~31; b >= 0; b -= 32) {
        if (base + b >= wmax) continue;
        const int j = b + lane;
        bool hit = false;
        if (j < cnt && base + j < wmax) {
          float4 e0 = sm0[j], e1 = sm1[j];
          hit = slab_may_contribute(e0, e1, rx0, ry0, rx1, ry1);
        }
        unsigned mask = __ballot_sync(0xffffffffu, hit);
        while (mask) {
          const int k = 31 - __clz(mask);
          mask &= ~(1u << k);
          const int pos = base + b + k;
          const float4 e0 = sm0[b + k], e1 = sm1[b + k];
          PairEval pe = pair_eval(e0, e1, fx, fy);
          const bool valid = inside && pos < last_contrib && pe.power <= 0.f && pe.alpha >= kAlphaMin;
          if (!__any_sync(0xffffffffu, valid)) continue;
          float v[9];
#pragma unroll
          for (int u = 0; u < 9; ++u) v[u] = 0.f;
          if (valid) {
            const float4 c = sm2[b + k];
            const float inv1ma = rcp_approx(1.f - pe.alpha);      // 1-alpha in [0.01, 1]
            T = T * inv1ma;
            const float dchannel_dcolor = pe.alpha * T;
            acc_r = last_alpha * last_r + (1.f - last_alpha) * acc_r; last_r = c.x;
            acc_g = last_alpha * last_g + (1.f - last_alpha) * acc_g; last_g = c.y;
            acc_b = last_alpha * last_b + (1.f - last_alpha) * acc_b; last_b = c.z;
            float dL_dalpha = (c.x - acc_r) * dLr + (c.y - acc_g) * dLg + (c.z - acc_b) * dLb;
            dL_dalpha *= T;
            last_alpha = pe.alpha;
            dL_dalpha -= T_final * inv1ma * bg_dot;
            // raw moments of w = dL/dalpha * opacity * G (constants applied in k_preprocess_bwd, see k_blend_bwd2)
            const float w = e1.y * pe.G * dL_dalpha;
            v[0] = w * pe.dx;
            v[1] = w * pe.dy;
            v[2] = v[0] * pe.dx;
            v[3] = v[0] * pe.dy;
            v[4] = v[1] * pe.dy;
            v[5] = w;
            v[6] = dchannel_dcolor * dLr;
            v[7] = dchannel_dcolor * dLg;
            v[8] = dchannel_dcolor * dLb;
          }
          warp_reduce9(v, lane);
          flush_fixed(dacc + (size_t)__float_as_uint(e1.w) * kDaccSlots, v[0], v[8], sm2[b + k].w, inv_m, lane, true);
        }
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// blend v2: 4 warps per tile, each warp owns an 8x8 block = two 8x4 halves; every lane carries TWO
// pixels (x, y) and (x, y+4) that share dx, so the per-Gaussian loads, dx terms, cull test and
// warp reduction are shared by 64 (pixel, Gaussian) pairs.
// The sub-tile cull is evaluated per half and the loop runs over the union of the two masks.
// ------------------------------------------------------------------------------------------
constexpr int kThreads2 = 128;

// ------------------------------------------------------------------------------------------
// TMA (bulk async copy) staging of the per-tile slabs: one elected thread arms an mbarrier with the
// byte count and issues cp.async.bulk.shared.global for the three slab arrays of the NEXT chunk
// while the CTA blends the current one (double buffered).  SASS: UBLKCP + SYNCS.
// ------------------------------------------------------------------------------------------
template <int CH>
struct SlabStage {
  float4 s0[CH], s1[CH], s2[CH];                 // record rows 0..2 of the chunk's entries: x,y,A',B' | C',o,qthr',id | r,g,b,-
};
template <int CH>
constexpr int id_row() { return CH + 4; }        // id chunk + up to 3 leading entries (bulk copies start 16-byte aligned)

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// The staging pipeline of one CTA over a sequence of chunks q = 0, 1, ... (chunk q = entries [e_q, e_q + cnt_q) of the
// tile's sorted id list; the forward walks the list front to back, the backward back to front).
//   request(q)  thread 0: TMA bulk copy of the id chunk into sid[q % 3], completing on bars[q % 3]
//   gather(q)   all threads: wait for the ids, then cp.async the three record rows of every entry into stg[q & 1]
//   land(more)  wait until the oldest outstanding gather has landed (more: a younger one is in flight) + CTA barrier
// Schedule used by the kernels: request(0), request(1), gather(0); then per chunk q: gather(q+1), request(q+2), land,
// blend chunk q, CTA barrier.  Every buffer is rewritten only after the barrier that ends its last reader.
template <bool BULK, int NT, int CH>
struct Stager {
  SlabStage<CH>* stg;             // [2]
  uint32_t (*sid)[id_row<CH>()];  // [3]   (BULK only)
  uint64_t* bars;                 // [3]   (BULK only)
  const uint32_t* ids;
  const float4* rec;
  int requested, waited;          // id chunks requested / consumed so far

  __device__ __forceinline__ void init() {
    requested = waited = 0;
    if (BULK) {
      if (threadIdx.x == 0) { mbar_init(&bars[0], 1); mbar_init(&bars[1], 1); mbar_init(&bars[2], 1); mbar_fence_init(); }
      __syncthreads();
    }
  }
  __device__ __forceinline__ void request(int q, size_t e, int cnt) {
    if (BULK) {
      if (threadIdx.x == 0) {
        const size_t ea = e & ~(size_t)3;
        const uint32_t bytes = (uint32_t)(((e - ea) + (size_t)cnt + 3) & ~(size_t)3) * 4u;
        mbar_expect_tx(&bars[q % 3], bytes);
        bulk_g2s(sid[q % 3], ids + ea, bytes, &bars[q % 3]);
      }
      requested = q + 1;
    }
  }
  __device__ __forceinline__ void gather(int q, size_t e, int cnt) {
    SlabStage<CH>* st = &stg[q & 1];
    if (BULK) {
      mbar_wait(&bars[q % 3], (uint32_t)((q / 3) & 1));
      waited = q + 1;
      const uint32_t* row = sid[q % 3] + (e & 3);
      for (int k = threadIdx.x; k < cnt; k += NT) {
        const float4* r = rec + 3 * (size_t)row[k];
        cp_async16(&st->s0[k], r); cp_async16(&st->s1[k], r + 1); cp_async16(&st->s2[k], r + 2);
      }
    } else {
      for (int k = threadIdx.x; k < cnt; k += NT) {
        const float4* r = rec + 3 * (size_t)__ldg(ids + e + k);
        cp_async16(&st->s0[k], r); cp_async16(&st->s1[k], r + 1); cp_async16(&st->s2[k], r + 2);
      }
    }
    cp_async_commit();
  }
  __device__ __forceinline__ void land(bool more) {
    if (more) cp_async_wait<1>(); else cp_async_wait<0>();
    __syncthreads();
  }
  // never leave the kernel with copies in flight
  __device__ __forceinline__ void drain() {
    cp_async_wait<0>();
    if (BULK)
      for (int q = waited; q < requested; ++q) mbar_wait(&bars[q % 3], (uint32_t)((q / 3) & 1));
  }
};

__device__ __forceinline__ float2 f2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ float2 f2s(float a) { return make_float2(a, a); }

// STATS (instrumentation build of the same kernel, gsb_blend_stats): counts warp iterations (= 64 evaluated
// (pixel, Gaussian) pairs each) and contributing pairs into stats[0..1].
template <bool BULK, bool STATS = false>
__global__ void __launch_bounds__(kThreads2, GSB_FWD_MINB)
k_blend_fwd2(const uint2* __restrict__ ranges, const uint32_t* __restrict__ ids, const float4* __restrict__ rec,
             const float* __restrict__ bg, int W, int H, int gx,
             float* __restrict__ out_color, float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
             unsigned long long* __restrict__ stats = nullptr) {
  unsigned int st_iter = 0, st_valid = 0;
  __shared__ __align__(128) SlabStage<kChunk> stg[2];
  __shared__ __align__(16) uint32_t sid[BULK ? 3 : 1][id_row<kChunk>()];
  __shared__ __align__(8) uint64_t bars[3];
  Stager<BULK, kThreads2, kChunk> sg{stg, sid, bars, ids, rec, 0, 0};
  sg.init();
  const int tile = view_tile(W, H, out_color, final_T, n_contrib);
  const int tx = blockIdx.x % gx, ty = blockIdx.x / gx;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sx0 = tx * kBlock + (warp & 1) * 8, sy0 = ty * kBlock + (warp >> 1) * 8;
  const int px = sx0 + (lane & 7), pyA = sy0 + (lane >> 3), pyB = pyA + 4;
  const bool inA = px < W && pyA < H, inB = px < W && pyB < H;
  const float fx = (float)px;
  const float2 fy = f2((float)pyA, (float)pyB);
  const float rx0 = (float)sx0, rx1 = (float)min(sx0 + 7, W - 1);
  const float ryA0 = (float)sy0, ryA1 = (float)min(sy0 + 3, H - 1);
  const float ryB0 = (float)(sy0 + 4), ryB1 = (float)min(sy0 + 7, H - 1);
  const uint2 rg = ranges[tile];
  const int n = (int)(rg.y - rg.x);
  float2 T = f2(1.f, 1.f), Cr = f2(0.f, 0.f), Cg = f2(0.f, 0.f), Cb = f2(0.f, 0.f);
  uint32_t lastA = 0, lastB = 0;
  bool doneA = !inA, doneB = !inB;
  bool wdoneA = !(sx0 < W && sy0 < H), wdoneB = !(sx0 < W && sy0 + 4 < H);
  const int nch = (n + kChunk - 1) / kChunk;
  // chunk q = entries [rg.x + q*kChunk, ...) of the tile's list
  auto c_e = [&](int q) { return (size_t)rg.x + (size_t)q * kChunk; };
  auto c_n = [&](int q) { return min(kChunk, n - q * kChunk); };
  if (nch > 0) {
    sg.request(0, c_e(0), c_n(0));
    if (nch > 1) sg.request(1, c_e(1), c_n(1));
    sg.gather(0, c_e(0), c_n(0));
  }
  for (int ci = 0; ci < nch; ++ci) {
    const int base = ci * kChunk;
    const int cnt = min(kChunk, n - base);
    const SlabStage<kChunk>* cur = &stg[ci & 1];
    if (ci + 1 < nch) {          // keep the pipeline full: records of chunk ci+1, ids of chunk ci+2
      sg.gather(ci + 1, c_e(ci + 1), c_n(ci + 1));
      if (ci + 2 < nch) sg.request(ci + 2, c_e(ci + 2), c_n(ci + 2));
    }
    sg.land(ci + 1 < nch);
    const float4* sm0 = cur->s0;
    const float4* sm1 = cur->s1;
    const float4* sm2 = cur->s2;
    if (!(wdoneA && wdoneB)) {
      for (int b = 0; b < cnt; b += 32) {
        const int j = b + lane;
        // ONE conservative cull test per entry: the bounding rectangle of the halves that are still live (while both
        // are, the 8x8 block -- a superset of the two 8x4 tests; extra pairs fail the exact per-pixel test)
        bool hit = false;
        if (j < cnt) {
          const float4 e0 = sm0[j], e1 = sm1[j];
          hit = slab_may_contribute(e0, e1, rx0, wdoneA ? ryB0 : ryA0, rx1, wdoneB ? ryA1 : ryB1);
        }
        unsigned mask = __ballot_sync(0xffffffffu, hit);
        while (mask) {
          const int k = __ffs(mask) - 1;
          mask &= mask - 1;
          const float4 e0 = sm0[b + k], e1 = sm1[b + k], c = sm2[b + k];
          const float dx = e0.x - fx;
          const float2 dy = f2(e0.y - fy.x, e0.y - fy.y);
          const float c1 = e0.w * dx, c0 = e0.z * dx * dx;
          // power' = c0 + dy * (c1 + C' * dy)
          const float2 pw = fma2(dy, fma2(f2s(e1.x), dy, f2s(c1)), f2s(c0));
          const float2 G = f2(ex2_approx(pw.x), ex2_approx(pw.y));
          float2 al = mul2(f2s(e1.y), G);
          al.x = fminf(0.99f, al.x); al.y = fminf(0.99f, al.y);
          bool vA = !doneA && pw.x <= 0.f && al.x >= kAlphaMin;
          bool vB = !doneB && pw.y <= 0.f && al.y >= kAlphaMin;
          const float2 tT = mul2(T, fma2(al, f2s(-1.f), f2s(1.f)));
          if (vA && tT.x < kTEps) { doneA = true; vA = false; }
          if (vB && tT.y < kTEps) { doneB = true; vB = false; }
          float2 w = mul2(al, T);
          w.x = vA ? w.x : 0.f; w.y = vB ? w.y : 0.f;
          Cr = fma2(f2s(c.x), w, Cr);
          Cg = fma2(f2s(c.y), w, Cg);
          Cb = fma2(f2s(c.z), w, Cb);
          const uint32_t pos = (uint32_t)(base + b + k + 1);
          T.x = vA ? tT.x : T.x; T.y = vB ? tT.y : T.y;
          lastA = vA ? pos : lastA; lastB = vB ? pos : lastB;
          if (STATS) { ++st_iter; st_valid += (vA ? 1u : 0u) + (vB ? 1u : 0u); }
        }
        wdoneA = __all_sync(0xffffffffu, doneA);
        wdoneB = __all_sync(0xffffffffu, doneB);
        if (wdoneA && wdoneB) break;
      }
    }
    if (__syncthreads_and(wdoneA && wdoneB)) break;
  }
  sg.drain();
  if (STATS) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) st_valid += __shfl_xor_sync(0xffffffffu, st_valid, o);
    if (lane == 0) { atomicAdd(stats + 0, (unsigned long long)st_iter); atomicAdd(stats + 1, (unsigned long long)st_valid); }
  }
  const size_t hw = (size_t)W * H;
  const float b0 = bg[0], b1 = bg[1], b2 = bg[2];
  if (inA) {
    size_t pix = (size_t)pyA * W + px;
    final_T[pix] = T.x; n_contrib[pix] = lastA;
    out_color[pix] = Cr.x + T.x * b0; out_color[hw + pix] = Cg.x + T.x * b1; out_color[2 * hw + pix] = Cb.x + T.x * b2;
  }
  if (inB) {
    size_t pix = (size_t)pyB * W + px;
    final_T[pix] = T.y; n_contrib[pix] = lastB;
    out_color[pix] = Cr.y + T.y * b0; out_color[hw + pix] = Cg.y + T.y * b1; out_color[2 * hw + pix] = Cb.y + T.y * b2;
  }
}

// A batch row: the 32 lanes' values of one (entry, value), padded to 36 floats.  The row stores (lane L -> word
// 36 r + L) hit 32 banks; so do the reduction's LDS.128 (lane t reads row t, and the 8 lanes of a phase start at
// banks 4 t mod 32, 8 different 16-byte bank groups), and every address is a base plus an immediate.
constexpr int kBatchRow = 36;

// The sum of the 32 floats of a batch row, grouped as warp_reduce9 / warp_reduce8 group a value over the lanes: pairs
// over lane bits 4, 3, 2, 1, 0 in that order.  Float addition is commutative, so only the grouping decides the bits
// and the total equals the butterfly's bit for bit.
__device__ __forceinline__ float batch_row_sum(const float* row) {
  auto col = [&](int c) { return *reinterpret_cast<const float4*>(row + 4 * c); };
  auto add = [](float4 a, float4 b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
  };
  float4 q[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) q[c] = add(col(c), col(c + 4));       // lane bit 4: lanes 4c.. and 4c+16..
  q[0] = add(q[0], q[2]);                                            // lane bit 3
  q[1] = add(q[1], q[3]);
  q[0] = add(q[0], q[1]);                                            // lane bit 2
  return __fadd_rn(__fadd_rn(q[0].x, q[0].z), __fadd_rn(q[0].y, q[0].w));   // lane bits 1, 0
}

// Reduces a warp's batch of n entries (rows[s * NV + i] = value i of entry s, one column per lane) and adds the
// totals to the fixed-point accumulators: lane t < n * NV owns value t % NV of entry t / NV.  Lane s holds entry s's
// accumulator index in idx and its extent in ext.  The first __syncwarp orders the lanes' row stores before these
// reads, the second these reads before the next batch's stores.
template <int NV, bool STATS>
__device__ __forceinline__ void batch_flush(const float (*rows)[kBatchRow], int n, uint32_t idx, float ext,
                                            unsigned long long* dacc, float inv_m, int lane) {
  __syncwarp();
  const int s = lane / NV, slot = lane - s * NV;
  const uint32_t gi = __shfl_sync(0xffffffffu, idx, s);
  const float e = __shfl_sync(0xffffffffu, ext, s);
  if (lane < n * NV) {
    const float total = batch_row_sum(rows[lane]);
    if (!STATS) atomicAdd(dacc + (size_t)gi * kDaccSlots + slot, fix_encode(total, fix_scale(slot, e, inv_m)));
  }
  __syncwarp();
}

// POSE_ONLY (tracking mode, render.py:99-170: Gaussians frozen): dL/dopacity is not needed, so the moment S w is
// dropped and dL/db takes its slot -- eight values, no ninth reduction chain, no scalar RED; k_preprocess_bwd is
// told about the layout (dacc[5] = dL/db, dacc[8] unused).
//
// BATCH (default): instead of one butterfly per list entry, every lane stores its NV values of the entry as one
// column of the warp's batch rows (row s * NV + i = value i of the batch's entry s) and the warp walks on; when
// NB = 3 entries are stored, and at the end of the list, lane t sums row t (batch_row_sum) and adds the total with
// one fixed-point RED.  The rows need no staging memory, and the entry's accumulator index and extent are captured
// in registers when it is stored, so a batch may span a chunk barrier.  !BATCH is the per-entry butterfly
// (warp_reduce9 / warp_reduce8 + flush_fixed) with the forward's chunk and 8 CTAs / SM, selected by
// gsb_set_option("blend_bwd_batch", 0): the bit-for-bit reference of the batched reduction.
template <bool BULK, bool STATS = false, bool POSE_ONLY = false, bool BATCH = true>
__global__ void __launch_bounds__(kThreads2, BATCH ? GSB_BWD_MINB : kBwdMinBFly)
k_blend_bwd2(const uint2* __restrict__ ranges, const uint32_t* __restrict__ ids, const float4* __restrict__ rec,
             const float* __restrict__ bg, int W, int H, int gx,
             const float* __restrict__ final_T, const uint32_t* __restrict__ n_contrib,
             const float* __restrict__ dL_dpix, unsigned long long* __restrict__ dacc,
             const uint32_t* __restrict__ dscale, unsigned long long* __restrict__ stats = nullptr) {
  constexpr int CH = BATCH ? kChunkB : kChunk;
  constexpr int NV = POSE_ONLY ? 8 : 9;                 // values per entry
  constexpr int NB = 3;                                 // entries per batch: NB * NV <= 32 rows, one per lane
  unsigned int st_iter = 0, st_red = 0, st_valid = 0;
  const int tile = view_tile_bwd(W, H, dL_dpix, final_T, n_contrib, dscale);
  const float inv_m = fix_inv_m(dscale);
  __shared__ __align__(128) SlabStage<CH> stg[2];
  __shared__ __align__(16) uint32_t sid[BULK ? 3 : 1][id_row<CH>()];
  __shared__ __align__(8) uint64_t bars[3];
  __shared__ int s_bmax;
  __shared__ __align__(16) float s_batch[BATCH ? kThreads2 / 32 : 1][BATCH ? NB * NV : 1][kBatchRow];
  Stager<BULK, kThreads2, CH> sg{stg, sid, bars, ids, rec, 0, 0};
  sg.init();
  const int tx = blockIdx.x % gx, ty = blockIdx.x / gx;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sx0 = tx * kBlock + (warp & 1) * 8, sy0 = ty * kBlock + (warp >> 1) * 8;
  const int px = sx0 + (lane & 7), pyA = sy0 + (lane >> 3), pyB = pyA + 4;
  const bool inA = px < W && pyA < H, inB = px < W && pyB < H;
  const float fx = (float)px;
  const float2 fy = f2((float)pyA, (float)pyB);
  const float rx0 = (float)sx0, rx1 = (float)min(sx0 + 7, W - 1);
  const float ryA0 = (float)sy0, ryA1 = (float)min(sy0 + 3, H - 1);
  const float ryB0 = (float)(sy0 + 4), ryB1 = (float)min(sy0 + 7, H - 1);
  const uint2 rg = ranges[tile];
  const size_t hw = (size_t)W * H;
  const size_t pixA = (size_t)pyA * W + px, pixB = (size_t)pyB * W + px;
  const float2 T_final = f2(inA ? final_T[pixA] : 0.f, inB ? final_T[pixB] : 0.f);
  const int lcA = inA ? (int)n_contrib[pixA] : 0, lcB = inB ? (int)n_contrib[pixB] : 0;
  float2 dLr = f2(0.f, 0.f), dLg = f2(0.f, 0.f), dLb = f2(0.f, 0.f);
  if (inA) { dLr.x = dL_dpix[pixA]; dLg.x = dL_dpix[hw + pixA]; dLb.x = dL_dpix[2 * hw + pixA]; }
  if (inB) { dLr.y = dL_dpix[pixB]; dLg.y = dL_dpix[hw + pixB]; dLb.y = dL_dpix[2 * hw + pixB]; }
  const float b0 = bg[0], b1 = bg[1], b2 = bg[2];
  const float2 tf_bg = mul2(T_final, f2(b0 * dLr.x + b1 * dLg.x + b2 * dLb.x, b0 * dLr.y + b1 * dLg.y + b2 * dLb.y));
  int wmaxA = lcA, wmaxB = lcB;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    wmaxA = max(wmaxA, __shfl_xor_sync(0xffffffffu, wmaxA, o));
    wmaxB = max(wmaxB, __shfl_xor_sync(0xffffffffu, wmaxB, o));
  }
  const int wmax = max(wmaxA, wmaxB);
  if (threadIdx.x == 0) s_bmax = 0;
  __syncthreads();
  if (lane == 0) atomicMax(&s_bmax, wmax);
  __syncthreads();
  const int bmax = s_bmax;
  float2 T = T_final;
  float2 acc_r = f2(0.f, 0.f), acc_g = f2(0.f, 0.f), acc_b = f2(0.f, 0.f);
  int nb = 0;                                           // BATCH: entries in the warp's batch
  uint32_t b_idx = 0;                                   // BATCH: lane s < nb holds entry s's accumulator index
  float b_ext = 0.f;                                    //        and fixed-point extent
  const int nchunks = (bmax + CH - 1) / CH;
  // chunks are visited back to front; pipeline step q = 0 is the LAST chunk
  auto c_e = [&](int q) { return (size_t)rg.x + (size_t)(nchunks - 1 - q) * CH; };
  auto c_n = [&](int q) { return min(CH, bmax - (nchunks - 1 - q) * CH); };
  if (nchunks > 0) {
    sg.request(0, c_e(0), c_n(0));
    if (nchunks > 1) sg.request(1, c_e(1), c_n(1));
    sg.gather(0, c_e(0), c_n(0));
  }
  for (int it = 0; it < nchunks; ++it) {
    const int ch = nchunks - 1 - it;
    const int base = ch * CH;
    const int cnt = min(CH, bmax - base);
    const SlabStage<CH>* cur = &stg[it & 1];
    if (it + 1 < nchunks) {
      sg.gather(it + 1, c_e(it + 1), c_n(it + 1));
      if (it + 2 < nchunks) sg.request(it + 2, c_e(it + 2), c_n(it + 2));
    }
    sg.land(it + 1 < nchunks);
    const float4* sm0 = cur->s0;
    const float4* sm1 = cur->s1;
    const float4* sm2 = cur->s2;
    if (base < wmax) {
      for (int b = (cnt - 1) & ~31; b >= 0; b -= 32) {
        if (base + b >= wmax) continue;
        const int j = b + lane;
        bool hit = false;
        if (j < cnt) {
          const float4 e0 = sm0[j], e1 = sm1[j];
          const bool la = base + j < wmaxA, lb = base + j < wmaxB;        // which halves can still contain contributors
          if (la || lb) hit = slab_may_contribute(e0, e1, rx0, la ? ryA0 : ryB0, rx1, lb ? ryB1 : ryA1);
        }
        unsigned mask = __ballot_sync(0xffffffffu, hit);
        while (mask) {
          const int k = 31 - __clz(mask);
          mask &= ~(1u << k);
          const int pos = base + b + k;
          const float4 e0 = sm0[b + k], e1 = sm1[b + k];
          const float dx = e0.x - fx;
          const float2 dy = f2(e0.y - fy.x, e0.y - fy.y);
          const float c1 = e0.w * dx, c0 = e0.z * dx * dx;
          const float2 pw = fma2(dy, fma2(f2s(e1.x), dy, f2s(c1)), f2s(c0));
          const float2 G = f2(ex2_approx(pw.x), ex2_approx(pw.y));
          const float2 alu = mul2(f2s(e1.y), G);           // opacity * G (unclamped: the straight-through alpha)
          const bool vA = inA && pos < lcA && pw.x <= 0.f && alu.x >= kAlphaMin;      // min(0.99, a) >= 1/255 <=> a >= 1/255
          const bool vB = inB && pos < lcB && pw.y <= 0.f && alu.y >= kAlphaMin;
          if (STATS) { ++st_iter; st_valid += (vA ? 1u : 0u) + (vB ? 1u : 0u); }
          if (!__any_sync(0xffffffffu, vA || vB)) continue;
          if (STATS) ++st_red;
          const float4 c = sm2[b + k];
          // masked alphas: an invalid pixel behaves as alpha = 0 (T, accumulator and every moment unchanged)
          const float2 aw = f2(vA ? alu.x : 0.f, vB ? alu.y : 0.f);              // weight of the moments (unclamped)
          const float2 am = f2(fminf(0.99f, aw.x), fminf(0.99f, aw.y));          // blending alpha (clamped)
          const float2 one_m = fma2(am, f2s(-1.f), f2s(1.f));
          const float2 inv = f2(rcp_approx(one_m.x), rcp_approx(one_m.y));
          T = mul2(T, inv);
          const float2 dcol = mul2(am, T);                 // dchannel/dcolor = alpha * T
          // acc = colour composited from everything BEHIND this entry (the reference's accum_rec);
          // dL/dalpha = T * sum_ch (c - acc) dL_ch  -  T_final/(1-alpha) * bg.dL ; then acc += alpha (c - acc)
          const float2 d_r = add2(f2s(c.x), f2(-acc_r.x, -acc_r.y));
          const float2 d_g = add2(f2s(c.y), f2(-acc_g.x, -acc_g.y));
          const float2 d_b = add2(f2s(c.z), f2(-acc_b.x, -acc_b.y));
          float2 da = fma2(d_b, dLb, fma2(d_g, dLg, mul2(d_r, dLr)));
          da = mul2(da, T);
          da = fma2(f2(-tf_bg.x, -tf_bg.y), inv, da);
          acc_r = fma2(am, d_r, acc_r);
          acc_g = fma2(am, d_g, acc_g);
          acc_b = fma2(am, d_b, acc_b);
          // w = dL/dalpha * opacity * G, zero on invalid pixels through aw.  The warp accumulates the raw moments of w;
          // the per-Gaussian constants (conic, 1/opacity) are applied once in k_preprocess_bwd.
          const float2 w = mul2(aw, da);
          const float2 wy = mul2(w, dy);
          const float ws = w.x + w.y;
          float v[9];
          v[0] = ws * dx;                                        // S w dx
          v[1] = wy.x + wy.y;                                    // S w dy
          v[2] = v[0] * dx;                                      // S w dx^2
          v[3] = v[1] * dx;                                      // S w dx dy
          v[4] = wy.x * dy.x + wy.y * dy.y;                      // S w dy^2
          v[6] = dcol.x * dLr.x + dcol.y * dLr.y;
          v[7] = dcol.x * dLg.x + dcol.y * dLg.y;
          v[8] = dcol.x * dLb.x + dcol.y * dLb.y;
          v[5] = POSE_ONLY ? v[8] : ws;                          // S w (or dL/db in the 8-value layout)
          if constexpr (BATCH) {
            float* col = &s_batch[warp][nb * NV][lane];
#pragma unroll
            for (int i = 0; i < NV; ++i) col[kBatchRow * i] = v[i];
            if (lane == nb) { b_idx = __float_as_uint(e1.w); b_ext = c.w; }
            if (++nb == NB) {
              batch_flush<NV, STATS>(s_batch[warp], NB, b_idx, b_ext, dacc, inv_m, lane);
              nb = 0;
            }
          } else {
            if (POSE_ONLY) warp_reduce8(v, lane); else warp_reduce9(v, lane);
            if (!STATS)
              flush_fixed(dacc + (size_t)__float_as_uint(e1.w) * kDaccSlots, v[0], v[8], c.w, inv_m, lane, !POSE_ONLY);
          }
        }
      }
    }
    __syncthreads();
  }
  if constexpr (BATCH)
    if (nb > 0) batch_flush<NV, STATS>(s_batch[warp], nb, b_idx, b_ext, dacc, inv_m, lane);
  sg.drain();
  if (STATS) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) st_valid += __shfl_xor_sync(0xffffffffu, st_valid, o);
    if (lane == 0) {
      atomicAdd(stats + 2, (unsigned long long)st_iter);
      atomicAdd(stats + 3, (unsigned long long)st_valid);
      atomicAdd(stats + 4, (unsigned long long)st_red);
    }
  }
}


}  // namespace

int gsb_launch_blend_fwd(const GeomView& gv, const BinView& bv, const ImgView& iv, const float* bg, int W, int H, int V,
                         float* out_color, cudaStream_t st) {
  const int gx = (W + kBlock - 1) / kBlock;
  const dim3 grid(gx * ((H + kBlock - 1) / kBlock), V);
  ProfScope ps(GSB_K_BLEND_FWD, st);
  const int ver = gsb_option_blend_version(), bulk = gsb_option_stage_bulk();
  if (ver == 2 && bulk)
    k_blend_fwd2<true><<<grid, kThreads2, 0, st>>>(bv.ranges, bv.ids, gv.rec, bg, W, H, gx, out_color,
                                                   iv.final_T, iv.n_contrib);
  else if (ver == 2)
    k_blend_fwd2<false><<<grid, kThreads2, 0, st>>>(bv.ranges, bv.ids, gv.rec, bg, W, H, gx, out_color,
                                                    iv.final_T, iv.n_contrib);
  else
    k_blend_fwd<<<grid, kThreads, 0, st>>>(bv.ranges, bv.ids, gv.rec, bg, W, H, gx, out_color, iv.final_T,
                                           iv.n_contrib);
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}

int gsb_launch_blend_bwd(const GeomView& gv, const BinView& bv, const ImgView& iv, const float* bg, int W, int H, int V,
                         const float* dL_dout, bool pose_only, cudaStream_t st) {
  const int gx = (W + kBlock - 1) / kBlock;
  const dim3 grid(gx * ((H + kBlock - 1) / kBlock), V);
  ProfScope ps(GSB_K_BLEND_BWD, st, 2);
  const size_t n = (size_t)3 * W * H;
  const size_t nb = (n + kThreads - 1) / kThreads, max_blocks = 4 * (size_t)gsb_sm_count();
  k_abs_max<<<dim3((int)(nb < max_blocks ? nb : max_blocks), V), kThreads, 0, st>>>(n, dL_dout, gv.dscale);
  const int ver = gsb_option_blend_version(), bulk = gsb_option_stage_bulk();
  const bool batch = gsb_option_blend_bwd_batch();
  unsigned long long* dacc = gv.dacc;
  auto v2 = [&](auto kernel) {
    kernel<<<grid, kThreads2, 0, st>>>(bv.ranges, bv.ids, gv.rec, bg, W, H, gx, iv.final_T, iv.n_contrib, dL_dout, dacc,
                                       gv.dscale, nullptr);
  };
  if (pose_only)
    batch ? v2(k_blend_bwd2<true, false, true, true>) : v2(k_blend_bwd2<true, false, true, false>);
  else if (ver == 2 && bulk)
    batch ? v2(k_blend_bwd2<true, false, false, true>) : v2(k_blend_bwd2<true, false, false, false>);
  else if (ver == 2)
    batch ? v2(k_blend_bwd2<false, false, false, true>) : v2(k_blend_bwd2<false, false, false, false>);
  else
    k_blend_bwd<<<grid, kThreads, 0, st>>>(bv.ranges, bv.ids, gv.rec, bg, W, H, gx, iv.final_T, iv.n_contrib,
                                           dL_dout, dacc, gv.dscale);
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}

// Instrumentation (bench.py roofline block): re-runs the v2 blend kernels on the buffers of the last forward /
// backward with counters on.  stats (device, 8 x u64, zeroed here): [0] forward warp iterations (64 evaluated
// pairs each), [1] forward contributing pairs, [2] backward warp iterations, [3] backward contributing pairs,
// [4] backward warp iterations that reached the gradient reduction.  The forward pass rewrites identical outputs;
// the backward pass (run only if dL_dout != NULL) issues no atomics.
extern "C" GSB_API int gsb_blend_stats(const GsbCamera* cam, int32_t P, void* geom, void* binning, int64_t R,
                                       void* image, float* out_color, const float* dL_dout,
                                       unsigned long long* stats, gsb_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  GSB_REQUIRE(cam && geom && binning && image && out_color && stats, "null buffer");
  const int W = cam->width, H = cam->height;
  const int gx = (W + kBlock - 1) / kBlock, gy = (H + kBlock - 1) / kBlock;
  GeomView gv = geom_view(geom, P);
  BinView bv = bin_view(binning, R, W, H);
  ImgView iv = img_view(image, W, H);
  GSB_CUDA(cudaMemsetAsync(stats, 0, 8 * sizeof(unsigned long long), st));
  k_blend_fwd2<true, true><<<gx * gy, kThreads2, 0, st>>>(bv.ranges, bv.ids, gv.rec, cam->bg, W, H, gx, out_color,
                                                          iv.final_T, iv.n_contrib, stats);
  if (dL_dout)
    k_blend_bwd2<true, true><<<gx * gy, kThreads2, 0, st>>>(bv.ranges, bv.ids, gv.rec, cam->bg, W, H, gx, iv.final_T,
                                                            iv.n_contrib, dL_dout, gv.dacc, gv.dscale, stats);
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}
