// H100 (sm_90a) differentiable Gaussian rasterizer: per-Gaussian kernels + C ABI (include/gsb200.h).
//
// Pipeline (one view), every kernel hand-written for sm_90a, no library sort/scan, no host round trip:
//   k_setup_cam        camera/pose constants -> one CamConst in HBM (read by every block)
//   k_preprocess       fused pose transform + activations + EWA projection + SH->RGB, 128-bit
//                      coalesced loads staged through shared memory; writes packed splat records and
//                      counts instances per Gaussian and per tile (lossless alpha < 1/255 tile cull)
//   k_tile_scan        (gs_bin.cu) exclusive scan of the per-tile counts -> segment offsets, R on device
//   k_scatter          (gs_bin.cu) (depth | id) keys appended to the tiles' segments
//   k_tile_sort        (gs_bin.cu) per-tile shared-memory sort + gather into contiguous per-tile slabs
//   k_blend_fwd2       (gs_blend.cu) one CTA per 16x16 tile, TMA-staged slab chunks, two pixels per lane
//   k_blend_bwd2       (gs_blend.cu) back-to-front replay, 9 gradients per (warp, Gaussian) reduced in-warp
//   k_preprocess_bwd   analytic backward to the model's own tensors + in-kernel pose-gradient
//                      reduction; k_pose_finalize chains it to dL/dP[7].  <., ., true>: the gradients of a batch
//                      of views summed in view order, inputs staged once per Gaussian slice, and (<., true, true>)
//                      the densification statistics of its first views (gsb_backward_batch_stats)
//
// Reference behaviour: SURVEY.md Appendix A; call site gaussian_renderer/__init__.py:60-135.
#include <string.h>

#include "gs_internal.cuh"
#include "gs_tiles.cuh"
#include "gs_tma.cuh"

using namespace gsb;

// ------------------------------------------------------------------------------------------
// error handling
// ------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
void gsb_set_error(const char* s) { snprintf(g_err, sizeof(g_err), "%s", s); }
void gsb_set_errorf(const char* file, int line, const char* what, const char* detail) {
  snprintf(g_err, sizeof(g_err), "%s:%d %s: %s", file, line, what, detail);
}
extern "C" GSB_API const char* gsb_last_error(void) { return g_err; }

// ------------------------------------------------------------------------------------------
// optional per-kernel timing (CUDA events on the launching stream) and launch counting.
// The record list is guarded by a mutex: the backward runs on the autograd engine's thread.
// ------------------------------------------------------------------------------------------
#include <atomic>
#include <mutex>
static std::mutex g_prof_mu;
static std::atomic<bool> g_prof_on{false};
static std::atomic<unsigned long long> g_launches{0};
struct ProfRec { cudaEvent_t a, b; int id; };
static ProfRec g_prof[8192];
static int g_prof_n = 0, g_prof_cap = 0;
void gsb_count_launch(int n) { g_launches += (unsigned long long)n; }
int gsb_prof_begin(int id, cudaStream_t st) {
  if (!g_prof_on.load(std::memory_order_relaxed)) return -1;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (g_prof_n >= 8192) return -1;
  if (g_prof_n >= g_prof_cap) {
    cudaEventCreate(&g_prof[g_prof_n].a);
    cudaEventCreate(&g_prof[g_prof_n].b);
    g_prof_cap = g_prof_n + 1;
  }
  g_prof[g_prof_n].id = id;
  cudaEventRecord(g_prof[g_prof_n].a, st);
  return g_prof_n++;
}
void gsb_prof_end(int slot, cudaStream_t st) {
  if (slot < 0) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (slot < g_prof_n) cudaEventRecord(g_prof[slot].b, st);
}
extern "C" GSB_API void gsb_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_on = on != 0;
  g_prof_n = 0;
}
// ms_sum[id] += elapsed, count[id] += 1 for every recorded interval; resets the record list.
extern "C" GSB_API int gsb_profile_collect(double* ms_sum, int64_t* count, int n_ids) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (int i = 0; i < g_prof_n; ++i) {
    float ms = 0.f;
    if (cudaEventSynchronize(g_prof[i].b) != cudaSuccess) return GSB_ERR_CUDA;
    if (cudaEventElapsedTime(&ms, g_prof[i].a, g_prof[i].b) != cudaSuccess) return GSB_ERR_CUDA;
    if (g_prof[i].id >= 0 && g_prof[i].id < n_ids) { ms_sum[g_prof[i].id] += ms; count[g_prof[i].id] += 1; }
  }
  g_prof_n = 0;
  return GSB_OK;
}
extern "C" GSB_API uint64_t gsb_launch_count(void) { return g_launches.load(); }
static std::atomic<int> g_blend_version{2};
static std::atomic<int> g_stage_bulk{1};   // 1: slabs staged with cp.async.bulk (TMA) + mbarrier, 0: cooperative loads
int gsb_option_blend_version() { return g_blend_version.load(std::memory_order_relaxed); }
static std::atomic<int> g_blend_bwd_batch{1};   // 1: batched moment reduction, 0: per-entry butterfly (its reference)
int gsb_option_stage_bulk() { return g_stage_bulk.load(std::memory_order_relaxed); }
int gsb_option_blend_bwd_batch() { return g_blend_bwd_batch.load(std::memory_order_relaxed); }
// SM count of the current device, cached per device: sizes the persistent and grid-stride launches (132 on an H100 SXM)
int gsb_sm_count() {
  static std::atomic<int> sms[64];
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  n = sms[dev].load(std::memory_order_relaxed);
  if (n > 0) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
  sms[dev] = n;
  return n;
}
// option "blend_version": 1 = one pixel per lane (8 warps / tile; cross-check), 2 = two pixels per lane (default)
extern "C" GSB_API int gsb_set_option(const char* name, int value) {
  if (name && strcmp(name, "blend_version") == 0 && value >= 1 && value <= 2) { g_blend_version = value; return GSB_OK; }
  if (name && strcmp(name, "stage_bulk") == 0 && (value == 0 || value == 1)) { g_stage_bulk = value; return GSB_OK; }
  if (name && strcmp(name, "blend_bwd_batch") == 0 && (value == 0 || value == 1)) { g_blend_bwd_batch = value; return GSB_OK; }
  gsb_set_error("gsb_set_option: unknown option or bad value");
  return GSB_ERR_INVALID;
}
extern "C" GSB_API int gsb_abi_version(void) { return 2; }

constexpr float kLog2e = 1.4426950408889634f;
constexpr int kRowPad = 49;      // shared-memory SH row stride (48 + 1, conflict-free)

extern "C" GSB_API size_t gsb_geom_bytes(int32_t P) { return geom_view(nullptr, P).total; }
extern "C" GSB_API size_t gsb_binning_bytes(int64_t R, int32_t W, int32_t H) { return bin_view(nullptr, R, W, H).total; }
extern "C" GSB_API size_t gsb_image_bytes(int32_t W, int32_t H) { return img_view(nullptr, W, H).total; }
static int frame_tiles(int W, int H) { return ((W + kBlock - 1) / kBlock) * ((H + kBlock - 1) / kBlock); }
extern "C" GSB_API size_t gsb_geom_bytes_batch(int32_t P, int32_t V, int32_t W, int32_t H) {
  return geom_view(nullptr, P, V, frame_tiles(W, H)).total;
}
extern "C" GSB_API size_t gsb_binning_bytes_batch(int64_t R, int32_t W, int32_t H, int32_t V) {
  return bin_view(nullptr, R, W, H, V).total;
}
extern "C" GSB_API size_t gsb_image_bytes_batch(int32_t W, int32_t H, int32_t V) { return img_view(nullptr, W, H, V).total; }

// ------------------------------------------------------------------------------------------
// kernel parameter blocks
// ------------------------------------------------------------------------------------------
struct InPtrs {
  int P;
  const float* means;
  const float* scales;
  const float* rots;
  const float* opac;
  const float* sh_dc;
  const float* sh_rest;
  const float* colors;
  const float* cov3D;
  int sh_packed;
  int vec_ok;       // all base pointers 16-byte aligned
  int exact_cull;
  Mip mip;          // mip.on == 0: reference path; the 3D filter's f comes from filter3D[i]
  const float* filter3D;
};

// this Gaussian's filters
__device__ __forceinline__ Mip gauss_mip(const InPtrs& in, int i) {
  Mip m = in.mip;
  if (m.on3d) m.f = __ldg(in.filter3D + i);
  return m;
}

// ------------------------------------------------------------------------------------------
// k_setup_cam
// ------------------------------------------------------------------------------------------
struct CamArgs {
  const float* V; const float* Pm; const float* campos; const float* pose;
  int W, H; float tanfovx, tanfovy, scale_mod; int D, M, raw_params;
};
__device__ __forceinline__ void fill_cam(CamConst& c, const CamArgs& a) {
  const float* V = a.V; const float* Pm = a.Pm; const float* campos = a.campos; const float* pose = a.pose;
  const int W = a.W, H = a.H, D = a.D, M = a.M, raw_params = a.raw_params;
  const float tanfovx = a.tanfovx, tanfovy = a.tanfovy, scale_mod = a.scale_mod;
  for (int i = 0; i < 16; ++i) { c.V[i] = V[i]; c.Pm[i] = Pm[i]; }
  for (int i = 0; i < 3; ++i) c.campos[i] = campos[i];
  c.tanfovx = tanfovx; c.tanfovy = tanfovy;
  c.fx = W / (2.0f * tanfovx); c.fy = H / (2.0f * tanfovy);
  c.scale_mod = scale_mod; c.W = W; c.H = H;
  c.gx = (W + kBlock - 1) / kBlock; c.gy = (H + kBlock - 1) / kBlock;
  c.D = D; c.M = M; c.raw_params = raw_params; c.pose_on = 0;
  for (int i = 0; i < 9; ++i) c.Rc[i] = (i % 4 == 0) ? 1.f : 0.f;
  c.tc[0] = c.tc[1] = c.tc[2] = 0.f;
  c.qc[0] = 1.f; c.qc[1] = c.qc[2] = c.qc[3] = 0.f;
  if (pose) pose_to_const(pose, c);
}
// one CTA per view: CamConst v from pose row v of the [V, 7] pose table
__global__ void k_setup_cam(CamConst* out, CamArgs a) {
  if (threadIdx.x != 0) return;
  if (a.pose) a.pose += 7 * blockIdx.x;
  CamConst c;
  fill_cam(c, a);
  out[blockIdx.x] = c;
}

// ------------------------------------------------------------------------------------------
// staging helpers: copy `n` contiguous floats global -> shared (or back) with 128-bit accesses
// ------------------------------------------------------------------------------------------
// dst index of source element k is (k / row) * stride + col0 + (k % row)
__device__ __forceinline__ void stage_in(float* sm, const float* __restrict__ src, int n, int row,
                                         int stride, int col0, bool vec) {
  if (vec) {
    int n4 = n >> 2;
    const float4* s4 = reinterpret_cast<const float4*>(src);
    for (int k = threadIdx.x; k < n4; k += blockDim.x) {
      float4 v = __ldg(s4 + k);
      int e = 4 * k;
      int r = e / row, c = e - r * row;
      float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        sm[r * stride + col0 + c] = vv[u];
        if (++c == row) { c = 0; ++r; }
      }
    }
    for (int e = 4 * n4 + threadIdx.x; e < n; e += blockDim.x) {
      int r = e / row, c = e - r * row;
      sm[r * stride + col0 + c] = __ldg(src + e);
    }
  } else {
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
      int r = e / row, c = e - r * row;
      sm[r * stride + col0 + c] = __ldg(src + e);
    }
  }
}

__device__ __forceinline__ void stage_out(float* __restrict__ dst, const float* sm, int n, int row,
                                          int stride, int col0, bool vec) {
  if (vec) {
    int n4 = n >> 2;
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int k = threadIdx.x; k < n4; k += blockDim.x) {
      int e = 4 * k;
      int r = e / row, c = e - r * row;
      float vv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        vv[u] = sm[r * stride + col0 + c];
        if (++c == row) { c = 0; ++r; }
      }
      d4[k] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    }
    for (int e = 4 * n4 + threadIdx.x; e < n; e += blockDim.x) {
      int r = e / row, c = e - r * row;
      dst[e] = sm[r * stride + col0 + c];
    }
  } else {
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
      int r = e / row, c = e - r * row;
      dst[e] = sm[r * stride + col0 + c];
    }
  }
}

// Shared-memory layout of the two per-Gaussian kernels (dynamic, floats, N = kPT Gaussians per CTA):
//   cam | xyz[3N] | scale[3N] | quat[4N] | opacity[N] | sh[49N]
// Every array is copied CONTIGUOUSLY (128-bit global loads -> 128-bit shared stores, conflict-free);
// each thread then walks its own row with an odd word stride (3, 45; the quaternion is one LDS.128), so
// the strided accesses are conflict-free too.  Split SH layout: dc at sh[3t], rest at sh[3N + 3(M-1)t] (stride 45 at
// M = 16 and 9 at M = 4; the 24 of M = 9 is even, so its rest rows see 8-way bank conflicts).
// Packed [P,M,3] layout (generic B2 boundary): rows padded to kRowPad = 49 words.
constexpr int kSmXyz = 0, kSmSc = 3 * kPT, kSmQ = 6 * kPT, kSmOp = 10 * kPT, kSmSh = 11 * kPT;
constexpr int kSmFloats = 11 * kPT + kRowPad * kPT;
constexpr size_t kPrepSmem = sizeof(CamConst) + 16 + (size_t)kSmFloats * 4;
// The view-summing backward (k_preprocess_bwd<., false, true>) keeps the staged SH rows as inputs for every view and adds
// each view's SH gradient into a second region of the same layout behind them.
constexpr size_t kPrepSmemViews = kPrepSmem + (size_t)kRowPad * kPT * 4;

__device__ __forceinline__ void copy_in(float* sm, const float* __restrict__ src, int n, bool vec) {
  if (vec) {
    const int n4 = n >> 2;
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(sm);
    for (int k = threadIdx.x; k < n4; k += blockDim.x) d4[k] = __ldg(s4 + k);
    for (int e = 4 * n4 + threadIdx.x; e < n; e += blockDim.x) sm[e] = __ldg(src + e);
  } else {
    for (int e = threadIdx.x; e < n; e += blockDim.x) sm[e] = __ldg(src + e);
  }
}
__device__ __forceinline__ void copy_out(float* __restrict__ dst, const float* sm, int n, bool vec) {
  if (vec) {
    const int n4 = n >> 2;
    float4* d4 = reinterpret_cast<float4*>(dst);
    const float4* s4 = reinterpret_cast<const float4*>(sm);
    for (int k = threadIdx.x; k < n4; k += blockDim.x) d4[k] = s4[k];
    for (int e = 4 * n4 + threadIdx.x; e < n; e += blockDim.x) dst[e] = sm[e];
  } else {
    for (int e = threadIdx.x; e < n; e += blockDim.x) dst[e] = sm[e];
  }
}

struct ShRows { int dc_stride, rest_off, rest_stride; };   // thread t: dc at sh[dc_stride*t], rest at sh[rest_off + rest_stride*t]
__device__ __forceinline__ ShRows sh_rows(int sh_packed, int M) {
  ShRows r;
  if (sh_packed) { r.dc_stride = kRowPad; r.rest_off = 3; r.rest_stride = kRowPad; }
  else { r.dc_stride = 3; r.rest_off = 3 * kPT; r.rest_stride = 3 * (M - 1); }
  return r;
}

// Generic staging (ragged last CTA, unaligned pointers, packed SH layout, precomputed inputs); full aligned CTAs take
// the bulk-copy path below.
__device__ __forceinline__ void load_block_inputs(const InPtrs& in, int first, int nv, bool use_sh, int D, int M,
                                                  float* sm) {
  const bool vec = in.vec_ok != 0;
  copy_in(sm + kSmXyz, in.means + (size_t)3 * first, 3 * nv, vec);
  if (in.scales) copy_in(sm + kSmSc, in.scales + (size_t)3 * first, 3 * nv, vec);
  if (in.rots) copy_in(sm + kSmQ, in.rots + (size_t)4 * first, 4 * nv, vec);
  copy_in(sm + kSmOp, in.opac + first, nv, vec);
  if (use_sh) {
    if (in.sh_packed) {
      stage_in(sm + kSmSh, in.sh_dc + (size_t)3 * M * first, 3 * M * nv, 3 * M, kRowPad, 0, vec);
    } else {
      copy_in(sm + kSmSh, in.sh_dc + (size_t)3 * first, 3 * nv, vec);
      if (D > 0 && M > 1)
        copy_in(sm + kSmSh + 3 * kPT, in.sh_rest + (size_t)3 * (M - 1) * first, 3 * (M - 1) * nv, vec);
    }
  }
}

// The same full-CTA fast path with the copies done by the TMA unit: one thread arms an mbarrier with the byte count and
// issues one bulk copy per input array (cp.async.bulk.shared.global, SASS UBLKCP); nothing passes through registers or
// allocates L1 lines (with register staging, the 180 KB a resident set of CTAs keeps in flight is bounded by the L1
// carve-out, so giving shared memory the whole unified storage does not help).
// Any coefficient count M of the split layout qualifies: the CTA's rest slice is 3 (M - 1) kPT floats, a multiple of 16
// bytes in size and offset (rest_bytes).
__device__ __forceinline__ uint32_t rest_bytes(int M) { return (uint32_t)(3 * (M - 1) * kPT * 4); }
__device__ __forceinline__ bool block_inputs_bulk_ok(const InPtrs& in, int nv, bool use_sh) {
  return in.vec_ok != 0 && nv == kPT && in.scales && in.rots && (!use_sh || !in.sh_packed);
}
__device__ __forceinline__ void bulk_load_block_inputs(const InPtrs& in, int first, bool use_sh, int D, int M, float* sm,
                                                       uint64_t* bar) {
  constexpr uint32_t B3 = 3 * kPT * 4, B4 = 4 * kPT * 4, B1 = kPT * 4;
  const uint32_t BR = rest_bytes(M);
  const bool rest = use_sh && D > 0;
  mbar_expect_tx(bar, 2 * B3 + B4 + B1 + (use_sh ? B3 : 0u) + (rest ? BR : 0u));
  bulk_g2s(sm + kSmXyz, in.means + (size_t)3 * first, B3, bar);
  bulk_g2s(sm + kSmSc, in.scales + (size_t)3 * first, B3, bar);
  bulk_g2s(sm + kSmQ, in.rots + (size_t)4 * first, B4, bar);
  bulk_g2s(sm + kSmOp, in.opac + first, B1, bar);
  if (use_sh) bulk_g2s(sm + kSmSh, in.sh_dc + (size_t)3 * first, B3, bar);
  if (rest) bulk_g2s(sm + kSmSh + 3 * kPT, in.sh_rest + (size_t)3 * (M - 1) * first, BR, bar);
}
// all threads call; returns when the CTA's inputs are in shared memory
__device__ __forceinline__ void stage_block_inputs(const InPtrs& in, int first, int nv, bool use_sh, int D, int M, float* sm,
                                                   uint64_t* bar) {
  if (block_inputs_bulk_ok(in, nv, use_sh)) {
    if (threadIdx.x == 0) bulk_load_block_inputs(in, first, use_sh, D, M, sm, bar);
    mbar_wait(bar, 0u);
  } else {
    load_block_inputs(in, first, nv, use_sh, D, M, sm);
    __syncthreads();
  }
}

__device__ __forceinline__ void read_gauss(const float* sm, int t, bool has_sr, GaussIn& g) {
  g.m[0] = sm[kSmXyz + 3 * t]; g.m[1] = sm[kSmXyz + 3 * t + 1]; g.m[2] = sm[kSmXyz + 3 * t + 2];
  if (has_sr) {
    g.sc[0] = sm[kSmSc + 3 * t]; g.sc[1] = sm[kSmSc + 3 * t + 1]; g.sc[2] = sm[kSmSc + 3 * t + 2];
    const float4 q = *reinterpret_cast<const float4*>(sm + kSmQ + 4 * t);
    g.q[0] = q.x; g.q[1] = q.y; g.q[2] = q.z; g.q[3] = q.w;
  } else {
    g.sc[0] = g.sc[1] = g.sc[2] = 1.f;
    g.q[0] = 1.f; g.q[1] = g.q[2] = g.q[3] = 0.f;
  }
  g.op = sm[kSmOp + t];
}

// ------------------------------------------------------------------------------------------
// k_preprocess
// ------------------------------------------------------------------------------------------
// Grid (Gaussian CTAs, V): CTA (b, v) projects Gaussians [b * kPT, ...) in view v.  Inputs are read at the Gaussian's
// index i, outputs are written at its record id r = v * P + i, and tiles are counted in the view's slice of tcount.
template <bool kMip>
__global__ void __launch_bounds__(kPT)
k_preprocess(InPtrs in, GeomView gv, int* __restrict__ radii) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  CamConst* cam = reinterpret_cast<CamConst*>(smem_raw);
  float* sm = reinterpret_cast<float*>(smem_raw + ((sizeof(CamConst) + 15) / 16) * 16);
  {
    const uint32_t* s = reinterpret_cast<const uint32_t*>(gv.cam + blockIdx.y);
    uint32_t* d = reinterpret_cast<uint32_t*>(cam);
    for (int k = threadIdx.x; k < (int)(sizeof(CamConst) / 4); k += blockDim.x) d[k] = s[k];
  }
  __shared__ __align__(8) uint64_t s_bar;
  if (threadIdx.x == 0) { mbar_init(&s_bar, 1); mbar_fence_init(); }
  int first = blockIdx.x * kPT;
  int nv = min(kPT, in.P - first);
  bool use_sh = in.colors == nullptr;
  __syncthreads();
  stage_block_inputs(in, first, nv, use_sh, cam->D, cam->M, sm, &s_bar);
  const int t = threadIdx.x;
  const bool active = t < nv;
  const int i = first + (active ? t : 0);
  const size_t rb = (size_t)blockIdx.y * in.P;             // record ids of this view start here
  const uint32_t r = (uint32_t)(rb + i);
  uint32_t* const tcount = gv.tcount + (size_t)blockIdx.y * cam->gx * cam->gy;
  GaussIn g;
  read_gauss(sm, active ? t : 0, in.scales != nullptr, g);
  Proj p;
  if constexpr (kMip) project_geometry<true>(*cam, g, in.cov3D ? in.cov3D + (size_t)6 * i : nullptr, p, gauss_mip(in, i));
  else project_geometry(*cam, g, in.cov3D ? in.cov3D + (size_t)6 * i : nullptr, p);
  if (!active) p.visible = 0;
  float qthr = -1.f;
  uint32_t ntiles = 0, kmask = 0u;
  bool coop = false, big = false;
  SplatRect sr_;
  sr_.x = sr_.y = sr_.A = sr_.B = sr_.C = 0.f; sr_.qthr = -1.f;
  sr_.rx0 = sr_.rx1 = sr_.ry0 = sr_.ry1 = 0;
  const TileSink sink{tcount, nullptr, nullptr, nullptr, 0u};          // count mode
  const bool cull = in.exact_cull != 0;
  if (p.visible) {
    if (use_sh) {
      const ShRows sr = sh_rows(in.sh_packed, cam->M);
      project_color(*cam, sm + kSmSh + sr.dc_stride * t, sm + kSmSh + sr.rest_off + sr.rest_stride * t, p);
    } else {
      p.rgb[0] = in.colors[3 * i]; p.rgb[1] = in.colors[3 * i + 1]; p.rgb[2] = in.colors[3 * i + 2];
    }
    qthr = cull_threshold(p.opacity);
    // The tile coverage is decided on the record exactly as it is stored (conic and threshold in the log2 domain), so
    // that k_scatter -- which re-walks large rects from the stored record -- sees bit-identical inputs.
    sr_.x = p.x; sr_.y = p.y;
    sr_.A = 0.5f * kLog2e * p.A; sr_.B = 0.5f * kLog2e * p.B; sr_.C = 0.5f * kLog2e * p.C;
    sr_.qthr = qthr < 0.f ? -1.f : 0.5f * kLog2e * qthr;
    // Lossless tightening of the tile rect: alpha >= 1/255 needs q(d) <= qthr, an ellipse whose bounding box has the
    // half-extents sqrt(qthr C / det), sqrt(qthr A / det) -- for anisotropic or low-opacity Gaussians far inside the
    // reference's square 3-sigma rect (which stays what `radii` reports).  Tiles outside it would fail the per-tile test
    // anyway; not walking them keeps the count/emit loops proportional to what is kept, also for Gaussians that grow
    // large during training.  (+1 px margin; the tile range is rounded outwards.)
    if (cull && qthr >= 0.f) tighten_cull_rect(sr_.x, sr_.y, sr_.A, sr_.B, sr_.C, sr_.qthr, p.rx0, p.ry0, p.rx1, p.ry1);
    sr_.rx0 = p.rx0; sr_.rx1 = p.rx1; sr_.ry0 = p.ry0; sr_.ry1 = p.ry1;
    const int area = (p.rx1 - p.rx0) * (p.ry1 - p.ry0);
    if (cull && qthr < 0.f) ntiles = 0;
    else if (area > kBigRect) big = true;        // counted later by k_big_rects (which also fills gv.tiles[i])
    else if (area > kCoopTiles) coop = true;
    else {
      // per-tile counts: plain fire-and-forget RED.ADD per kept tile (measured faster here than warp-aggregating
      // them: nothing waits for the result, unlike the emit pass in k_scatter)
      kmask = rect_keep_mask_count(sr_, cam->W, cam->H, cam->gx, cull, tcount);
      ntiles = (uint32_t)__popc(kmask);
    }
  } else {
    p.x = p.y = p.A = p.B = p.C = 0.f; p.rgb[0] = p.rgb[1] = p.rgb[2] = 0.f;
  }
  {
    const uint32_t c = visit_tiles_coop(coop, sr_, cam->W, cam->H, cam->gx, cull, sink, 0ull);
    if (coop) ntiles = c;
  }
  // ---- outputs.  The 48-byte splat record (rows x,y,A',B' | C',o,qthr',id | r,g,b,extent; conic pre-scaled into the log2
  // domain: power*log2(e) = A' dx^2 + B' dx dy + C' dy^2) is what the blend kernels gather by id, so it is stored as an
  // array of structures -- transposed through shared memory so that the CTA's 128 x 48 B leave as one contiguous block
  // of 128-bit stores.  The binning record (depth, tile rect, keep mask) is a plain coalesced float4 array.
  __syncthreads();                                   // every thread is done with the staged inputs: reuse `sm`
  float4* sm4 = reinterpret_cast<float4*>(sm);
  if (active) {
    sm4[3 * t + 0] = make_float4(p.x, p.y, -0.5f * kLog2e * p.A, -kLog2e * p.B);
    sm4[3 * t + 1] = make_float4(-0.5f * kLog2e * p.C, p.opacity, 0.5f * kLog2e * qthr, __uint_as_float(r));
    sm4[3 * t + 2] = make_float4(p.rgb[0], p.rgb[1], p.rgb[2], fix_extent(p.radius, p.x, p.y, cam->W, cam->H));
    gv.brec[r] = make_float4(p.depth, __uint_as_float((uint32_t)p.rx0 | ((uint32_t)p.rx1 << 16)),
                             __uint_as_float((uint32_t)p.ry0 | ((uint32_t)p.ry1 << 16)), __uint_as_float(kmask));
    gv.tiles[r] = ntiles;
    if (big) gv.q_big[atomicAdd(gv.aux, 1u)] = r;      // at most once per record: the queue holds V * P entries
    gv.clamped[r] = (uint8_t)p.clamped;
    radii[r] = p.radius;
  }
  tma_store_fence();                                 // the records leave as ONE bulk store (shared -> global, 48 nv bytes)
  __syncthreads();
  if (threadIdx.x == 0) {
    bulk_s2g(gv.rec + 3 * (rb + first), sm4, (uint32_t)(48 * nv));
    bulk_commit();
    bulk_wait_read();
  }
}

// ------------------------------------------------------------------------------------------
// k_preprocess_bwd
// ------------------------------------------------------------------------------------------
struct OutPtrs {
  float* dmeans; float* dmeans2D; float* dscales; float* drots; float* dopac;
  float* dsh_dc; float* dsh_rest; float* dcolors; float* dcov3D;
};
// densification statistics (GsbDensifyStats), read only by the kStats instances
struct StatsPtrs {
  const int32_t* radii; float* accum; float* denom; float* max_r;
};

// The CTA's gradient rows (staging layout; SH rows at `sh`) -> the gradient tensors.  All threads call; returns whether
// the stores were bulk copies, which read shared memory until bulk_wait_read().  Used by views_bwd; the single-view
// instances keep the same code inline, which keeps their SASS the one measured before the view-summing instance.
__device__ __forceinline__ bool store_block_grads(const InPtrs& in, const OutPtrs& out, const float* sm, const float* sh,
                                                  int first, int nv, int M, bool use_sh, bool vec) {
  // Full CTA, aligned, split SH layout: every gradient array of the CTA leaves as one bulk store (shared -> global)
  // issued by one thread; the generic path below covers ragged / unaligned / packed cases.
  const bool bulk_out = vec && nv == kPT && !in.sh_packed;
  if (bulk_out) tma_store_fence();
  __syncthreads();
  if (bulk_out) {
    if (threadIdx.x == 0) {
      constexpr uint32_t B3 = 3 * kPT * 4, B4 = 4 * kPT * 4, B1 = kPT * 4;
      if (out.dmeans) bulk_s2g(out.dmeans + (size_t)3 * first, sm + kSmXyz, B3);
      if (out.dscales) bulk_s2g(out.dscales + (size_t)3 * first, sm + kSmSc, B3);
      if (out.drots) bulk_s2g(out.drots + (size_t)4 * first, sm + kSmQ, B4);
      if (out.dopac) bulk_s2g(out.dopac + first, sm + kSmOp, B1);
      if (use_sh && out.dsh_dc) {
        bulk_s2g(out.dsh_dc + (size_t)3 * first, sh, B3);
        if (M > 1 && out.dsh_rest) bulk_s2g(out.dsh_rest + (size_t)3 * (M - 1) * first, sh + 3 * kPT, rest_bytes(M));
      }
      bulk_commit();
    }
  } else {
    if (out.dmeans) copy_out(out.dmeans + (size_t)3 * first, sm + kSmXyz, 3 * nv, vec);
    if (out.dscales) copy_out(out.dscales + (size_t)3 * first, sm + kSmSc, 3 * nv, vec);
    if (out.drots) copy_out(out.drots + (size_t)4 * first, sm + kSmQ, 4 * nv, vec);
    if (out.dopac) copy_out(out.dopac + first, sm + kSmOp, nv, vec);
    if (use_sh && out.dsh_dc) {
      if (in.sh_packed) {
        stage_out(out.dsh_dc + (size_t)3 * M * first, sh, 3 * M * nv, 3 * M, kRowPad, 0, vec);
      } else {
        copy_out(out.dsh_dc + (size_t)3 * first, sh, 3 * nv, vec);
        if (M > 1 && out.dsh_rest)
          copy_out(out.dsh_rest + (size_t)3 * (M - 1) * first, sh + 3 * kPT, 3 * (M - 1) * nv, vec);
      }
    }
  }
  return bulk_out;
}

// The CTA's pose-gradient partials pa[16] (one set per thread): warp shuffle, then across the 8 warps; dst[16].
// All threads call (one barrier).
__device__ __forceinline__ void block_pose_partials(const float* pa, float (*s_pose)[16], float* dst) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    float v = pa[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s_pose[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kPT / 32; ++w) v += s_pose[w][threadIdx.x];
    dst[threadIdx.x] = v;
  }
}

// k_preprocess_bwd<kMip, false, true>: the per-Gaussian gradients of `nviews` views, summed.  For every Gaussian and
// gradient element the result is ((g_0 + g_1) + g_2) + ..., where g_v is what the single-view instance computes for
// view v from that view's moments (record v * P + i, fixed-point unit gv.dscale[v]) and camera constants (gv.cam[v]).
// The view-independent inputs are staged once by the caller; the running sums start at -0 (so the first view adds
// exactly its own bits) and every view adds with __fadd_rn, which is never contracted into an FMA.  A view in which
// the Gaussian has no moments adds the +0 the single-view call writes.  SH sums live in shared memory behind the
// staged rows (kPrepSmemViews); the others in registers.  View v's pose partials go to pose_part row (v, CTA), the
// layout of grid y = view, so k_pose_reduce / k_pose_finalize are unchanged.
// kStats (k_preprocess_bwd<., true, true>): the densification statistics of views 0 .. nstats-1 as well, each view
// adding what one single-view kStats call on it adds (train.py:197-199): where radii[v * P + i] > 0, its own
// |dL/dmeans2D[:2]|, one view and its radius.  The three running values are loaded once, kept in registers across the
// view loop and stored once; the norm is written out as the single-view instance compiles sqrtf(dx*dx + dy*dy) (an
// FMUL of dy, one FFMA of dx, IEEE sqrt) and added with __fadd_rn in view order, so the result is bit-identical to
// nstats single-view calls made in view order.  Nothing is counted after a binning overflow (the caller repeats the
// step).
template <bool kMip, bool kStats>
__device__ __forceinline__ void views_bwd(const InPtrs& in, const GeomView& gv, int pose_only_layout,
                                          const OutPtrs& out, const StatsPtrs& stats, int nviews, int nstats,
                                          CamConst* cam, float* sm, float (*s_pose)[16], int first, int nv,
                                          bool use_sh, bool vec) {
  const int t = threadIdx.x, i = first + t;
  const int D = cam->D, M = cam->M;
  const ShRows sr = sh_rows(in.sh_packed, M);
  const float* row_rest = sm + kSmSh + sr.rest_off + sr.rest_stride * t;
  float* const acc = sm + kSmFloats;
  float* const acc_dc = acc + sr.dc_stride * t;
  float* const acc_rest = acc + sr.rest_off + sr.rest_stride * t;
  const int nrest = 3 * (M - 1), nact = 3 * ((D + 1) * (D + 1) - 1);
  float am[3], asc[3], aq[4], aop = -0.f, a2d[2];
#pragma unroll
  for (int k = 0; k < 3; ++k) am[k] = asc[k] = -0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) aq[k] = -0.f;
  a2d[0] = a2d[1] = -0.f;
  if (t < nv) {
    acc_dc[0] = acc_dc[1] = acc_dc[2] = -0.f;
    for (int k = 0; k < nrest; ++k) acc_rest[k] = -0.f;
  }
  bool count = false;
  float s_acc = 0.f, s_den = 0.f, s_max = 0.f;
  if constexpr (kStats) {
    count = t < nv && nstats > 0 && gv.status[kStOverflow] == 0u;
    if (count) { s_acc = stats.accum[i]; s_den = stats.denom[i]; s_max = stats.max_r[i]; }
  }
  for (int v = 0; v < nviews; ++v) {
    if (v > 0) {
      __syncthreads();                                     // view v - 1's camera and pose partials are consumed
      const uint32_t* s = reinterpret_cast<const uint32_t*>(gv.cam + v);
      uint32_t* d = reinterpret_cast<uint32_t*>(cam);
      for (int k = threadIdx.x; k < (int)(sizeof(CamConst) / 4); k += blockDim.x) d[k] = s[k];
      __syncthreads();
    }
    const size_t r = (size_t)v * in.P + i;
    float pa[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) pa[k] = 0.f;
    GaussGrad gg;
    gg.dm[0] = gg.dm[1] = gg.dm[2] = 0.f; gg.dsc[0] = gg.dsc[1] = gg.dsc[2] = 0.f;
    gg.dq[0] = gg.dq[1] = gg.dq[2] = gg.dq[3] = 0.f; gg.dop = 0.f;
    gg.dmeans2D[0] = gg.dmeans2D[1] = 0.f;
    if (t < nv) {
      float ds[kDaccSlots];
#pragma unroll
      for (int k = 0; k < kDaccSlots; ++k) ds[k] = 0.f;
      if (gv.tiles[r] > 0) {
        const unsigned long long* a = gv.dacc + r * kDaccSlots;
        const float extent = gv.rec[3 * r + 2].w, inv_m = fix_inv_m(gv.dscale + v);
        const double unit[3] = {1.0 / (double)fix_scale(5, extent, inv_m), 1.0 / (double)fix_scale(0, extent, inv_m),
                                1.0 / (double)fix_scale(2, extent, inv_m)};
#pragma unroll
        for (int k = 0; k < kDaccSlots; ++k) ds[k] = fix_decode(a[k], unit[fix_exp(k) - 2]);
      }
      if (pose_only_layout) { ds[8] = ds[5]; ds[5] = 0.f; }
      bool any = false;
#pragma unroll
      for (int k = 0; k < 9; ++k) any |= (ds[k] != 0.f);
      bool has = false;
      if (any && gv.tiles[r] > 0) {
        GaussIn g;
        read_gauss(sm, t, in.scales != nullptr, g);
        Proj p;
        const Mip mf = kMip ? gauss_mip(in, i) : Mip();
        project_geometry<kMip>(*cam, g, in.cov3D ? in.cov3D + (size_t)6 * i : nullptr, p, mf);
        if (p.visible) {
          p.clamped = gv.clamped[r];
          const float sx = ds[0], sy = ds[1];                // as in the single-view instance
          ds[0] = -(p.A * sx + p.B * sy);
          ds[1] = -(p.C * sy + p.B * sx);
          ds[2] *= -0.5f;
          ds[3] = -ds[3];
          ds[4] *= -0.5f;
          ds[5] = p.opacity > 0.f ? ds[5] / p.opacity : 0.f;
          project_bwd<kMip, true>(*cam, g, p, row_rest, use_sh, in.cov3D != nullptr, ds, gg, acc_dc, acc_rest, pa, mf);
          has = use_sh;
        }
      }
      if (!has)
        for (int k = 0; k < 3; ++k) acc_dc[k] = __fadd_rn(acc_dc[k], 0.f);
      for (int k = has ? nact : 0; k < nrest; ++k) acc_rest[k] = __fadd_rn(acc_rest[k], 0.f);
#pragma unroll
      for (int k = 0; k < 3; ++k) { am[k] = __fadd_rn(am[k], gg.dm[k]); asc[k] = __fadd_rn(asc[k], gg.dsc[k]); }
#pragma unroll
      for (int k = 0; k < 4; ++k) aq[k] = __fadd_rn(aq[k], gg.dq[k]);
      aop = __fadd_rn(aop, gg.dop);
      a2d[0] = __fadd_rn(a2d[0], gg.dmeans2D[0]);
      a2d[1] = __fadd_rn(a2d[1], gg.dmeans2D[1]);
      if constexpr (kStats) {
        if (count && v < nstats) {
          const int rad = stats.radii[r];
          if (rad > 0) {
            const float dx = gg.dmeans2D[0], dy = gg.dmeans2D[1];
            s_acc = __fadd_rn(s_acc, __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy))));
            s_den = __fadd_rn(s_den, 1.f);
            s_max = fmaxf(s_max, (float)rad);
          }
        }
      }
    }
    if (cam->pose_on) block_pose_partials(pa, s_pose, gv.pose_part + ((size_t)v * gridDim.x + blockIdx.x) * 16);
  }
  if (t < nv) {
    sm[kSmXyz + 3 * t] = am[0]; sm[kSmXyz + 3 * t + 1] = am[1]; sm[kSmXyz + 3 * t + 2] = am[2];
    sm[kSmSc + 3 * t] = asc[0]; sm[kSmSc + 3 * t + 1] = asc[1]; sm[kSmSc + 3 * t + 2] = asc[2];
    *reinterpret_cast<float4*>(sm + kSmQ + 4 * t) = make_float4(aq[0], aq[1], aq[2], aq[3]);
    sm[kSmOp + t] = aop;
    if (out.dmeans2D) {
      out.dmeans2D[3 * (size_t)i] = a2d[0];
      out.dmeans2D[3 * (size_t)i + 1] = a2d[1];
      out.dmeans2D[3 * (size_t)i + 2] = 0.f;
    }
  }
  if constexpr (kStats) {
    if (count) { stats.accum[i] = s_acc; stats.denom[i] = s_den; stats.max_r[i] = s_max; }
  }
  const bool bulk_out = store_block_grads(in, out, sm, acc, first, nv, M, use_sh, vec);
  if (bulk_out && threadIdx.x == 0) bulk_wait_read();
}

#ifndef GSB_PBWD_MINB
#define GSB_PBWD_MINB 4
#endif
// kViews: one CTA per Gaussian slice for a whole batch of `nviews` views (grid y = 1) -- the gradients of every view,
// summed in view order, and (kStats) the statistics of its first `nstats` views; see views_bwd above.  The other
// instances take grid y = view and ignore nviews and nstats.
template <bool kMip, bool kStats, bool kViews = false>
__global__ void __launch_bounds__(kPT, kViews ? 3 : GSB_PBWD_MINB)
k_preprocess_bwd(InPtrs in, GeomView gv, const int pose_only_layout, OutPtrs out, StatsPtrs stats, const int nviews,
                 const int nstats) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  CamConst* cam = reinterpret_cast<CamConst*>(smem_raw);
  float* sm = reinterpret_cast<float*>(smem_raw + ((sizeof(CamConst) + 15) / 16) * 16);
  __shared__ float s_pose[kPT / 32][16];
  {
    const uint32_t* s = reinterpret_cast<const uint32_t*>(gv.cam + blockIdx.y);
    uint32_t* d = reinterpret_cast<uint32_t*>(cam);
    for (int k = threadIdx.x; k < (int)(sizeof(CamConst) / 4); k += blockDim.x) d[k] = s[k];
  }
  __shared__ __align__(8) uint64_t s_bar;
  if (threadIdx.x == 0) { mbar_init(&s_bar, 1); mbar_fence_init(); }
  const int first = blockIdx.x * kPT;
  const int nv = min(kPT, in.P - first);
  const bool use_sh = in.colors == nullptr;
  const bool vec = in.vec_ok != 0;
  __syncthreads();
  const int D = cam->D, M = cam->M;
  stage_block_inputs(in, first, nv, use_sh, D, M, sm, &s_bar);
  const int t = threadIdx.x;
  const int i = first + t;
  if constexpr (kViews) {
    views_bwd<kMip, kStats>(in, gv, pose_only_layout, out, stats, nviews, nstats, cam, sm, s_pose, first, nv, use_sh,
                            vec);
    return;
  }
  const size_t r = (size_t)blockIdx.y * in.P + i;          // record id (grid y = view, as in k_preprocess)
  float pa[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) pa[k] = 0.f;
  GaussGrad gg;
  gg.dm[0] = gg.dm[1] = gg.dm[2] = 0.f; gg.dsc[0] = gg.dsc[1] = gg.dsc[2] = 0.f;
  gg.dq[0] = gg.dq[1] = gg.dq[2] = gg.dq[3] = 0.f; gg.dop = 0.f;
  gg.dmeans2D[0] = gg.dmeans2D[1] = 0.f;
#pragma unroll
  for (int k = 0; k < 6; ++k) gg.dcov3D[k] = 0.f;
  gg.dcolor[0] = gg.dcolor[1] = gg.dcolor[2] = 0.f;
  // Every thread touches only its own shared-memory rows from here on (no barrier needed until the
  // cooperative stores): the SH gradient is written IN PLACE over the staged SH row.
  const ShRows sr = sh_rows(in.sh_packed, M);
  float* row_dc = sm + kSmSh + sr.dc_stride * t;
  float* row_rest = sm + kSmSh + sr.rest_off + sr.rest_stride * t;
  bool has = false;
  if (t < nv) {
    // the record (and its extent) is only read for Gaussians that cover a tile; the others have no moments
    float ds[kDaccSlots];
#pragma unroll
    for (int k = 0; k < kDaccSlots; ++k) ds[k] = 0.f;
    if (gv.tiles[r] > 0) {
      const unsigned long long* acc = gv.dacc + r * kDaccSlots;
      const float extent = gv.rec[3 * r + 2].w, inv_m = fix_inv_m(gv.dscale + blockIdx.y);
      const double unit[3] = {1.0 / (double)fix_scale(5, extent, inv_m), 1.0 / (double)fix_scale(0, extent, inv_m),
                              1.0 / (double)fix_scale(2, extent, inv_m)};      // exponents 2, 3, 4
#pragma unroll
      for (int k = 0; k < kDaccSlots; ++k) ds[k] = fix_decode(acc[k], unit[fix_exp(k) - 2]);
    }
    if (pose_only_layout) { ds[8] = ds[5]; ds[5] = 0.f; }     // tracking mode: dacc[5] carries dL/db, no dL/dopacity
    bool any = false;
#pragma unroll
    for (int k = 0; k < 9; ++k) any |= (ds[k] != 0.f);
    if (any && gv.tiles[r] > 0) {
      GaussIn g;
      read_gauss(sm, t, in.scales != nullptr, g);
      Proj p;
      const Mip mf = kMip ? gauss_mip(in, i) : Mip();
      project_geometry<kMip>(*cam, g, in.cov3D ? in.cov3D + (size_t)6 * i : nullptr, p, mf);
      if (p.visible) {
        p.clamped = gv.clamped[r];
        // The blend backward accumulates RAW pixel moments of w = dL/dalpha * (opacity * G) per Gaussian
        //   ds = [S w dx, S w dy, S w dx^2, S w dx dy, S w dy^2, S w, dL/dr, dL/dg, dL/db];
        // the per-Gaussian constants are applied once here instead of once per (warp, Gaussian) in the blend kernel:
        //   dL/dx = -(A Sx + B Sy), dL/dy = -(C Sy + B Sx), dL/dA = -Sxx/2, dL/dB = -Sxy, dL/dC = -Syy/2,
        //   dL/dopacity = Sw / opacity.
        {
          const float sx = ds[0], sy = ds[1];
          ds[0] = -(p.A * sx + p.B * sy);
          ds[1] = -(p.C * sy + p.B * sx);
          ds[2] *= -0.5f;
          ds[3] = -ds[3];
          ds[4] *= -0.5f;
          ds[5] = p.opacity > 0.f ? ds[5] / p.opacity : 0.f;     // contributing pairs have opacity >= 1/255
        }
        project_bwd<kMip>(*cam, g, p, row_rest, use_sh, in.cov3D != nullptr, ds, gg, row_dc, row_rest, pa, mf);
        has = use_sh;
      }
    }
    // inactive coefficients (and everything of a Gaussian that did not contribute) get zero gradient
    if (!has) { row_dc[0] = 0.f; row_dc[1] = 0.f; row_dc[2] = 0.f; }
    for (int k = has ? 3 * ((D + 1) * (D + 1) - 1) : 0; k < 3 * (M - 1); ++k) row_rest[k] = 0.f;
    sm[kSmXyz + 3 * t] = gg.dm[0]; sm[kSmXyz + 3 * t + 1] = gg.dm[1]; sm[kSmXyz + 3 * t + 2] = gg.dm[2];
    sm[kSmSc + 3 * t] = gg.dsc[0]; sm[kSmSc + 3 * t + 1] = gg.dsc[1]; sm[kSmSc + 3 * t + 2] = gg.dsc[2];
    *reinterpret_cast<float4*>(sm + kSmQ + 4 * t) = make_float4(gg.dq[0], gg.dq[1], gg.dq[2], gg.dq[3]);
    sm[kSmOp + t] = gg.dop;
    if (out.dmeans2D) {
      out.dmeans2D[3 * (size_t)i] = gg.dmeans2D[0];
      out.dmeans2D[3 * (size_t)i + 1] = gg.dmeans2D[1];
      out.dmeans2D[3 * (size_t)i + 2] = 0.f;
    }
    if (out.dcolors) {
      out.dcolors[3 * (size_t)i] = gg.dcolor[0]; out.dcolors[3 * (size_t)i + 1] = gg.dcolor[1];
      out.dcolors[3 * (size_t)i + 2] = gg.dcolor[2];
    }
    if (out.dcov3D) {
#pragma unroll
      for (int k = 0; k < 6; ++k) out.dcov3D[6 * (size_t)i + k] = gg.dcov3D[k];
    }
    // train.py:197-199: every Gaussian with radii > 0 (visibility_filter; also those that kept no tile, whose
    // dmeans2D is 0) adds |dL/dmeans2D[:2]| and one view, and raises its largest screen radius.  One writer per
    // Gaussian, no atomics.  Not after a binning overflow: the caller repeats that iteration.
    if (kStats && stats.radii[i] > 0 && gv.status[kStOverflow] == 0u) {
      const float dx = gg.dmeans2D[0], dy = gg.dmeans2D[1];
      stats.accum[i] += sqrtf(dx * dx + dy * dy);
      stats.denom[i] += 1.f;
      stats.max_r[i] = fmaxf(stats.max_r[i], (float)stats.radii[i]);
    }
  }
  // Full CTA, aligned, split SH layout: every gradient array of the CTA leaves as one bulk store (shared -> global)
  // issued by one thread; the generic path below covers ragged / unaligned / packed cases.
  const bool bulk_out = vec && nv == kPT && !in.sh_packed;
  if (bulk_out) tma_store_fence();
  __syncthreads();
  if (bulk_out) {
    if (threadIdx.x == 0) {
      constexpr uint32_t B3 = 3 * kPT * 4, B4 = 4 * kPT * 4, B1 = kPT * 4;
      if (out.dmeans) bulk_s2g(out.dmeans + (size_t)3 * first, sm + kSmXyz, B3);
      if (out.dscales) bulk_s2g(out.dscales + (size_t)3 * first, sm + kSmSc, B3);
      if (out.drots) bulk_s2g(out.drots + (size_t)4 * first, sm + kSmQ, B4);
      if (out.dopac) bulk_s2g(out.dopac + first, sm + kSmOp, B1);
      if (use_sh && out.dsh_dc) {
        bulk_s2g(out.dsh_dc + (size_t)3 * first, sm + kSmSh, B3);
        if (M > 1 && out.dsh_rest)
          bulk_s2g(out.dsh_rest + (size_t)3 * (M - 1) * first, sm + kSmSh + 3 * kPT, rest_bytes(M));
      }
      bulk_commit();
    }
  } else {
  if (out.dmeans) copy_out(out.dmeans + (size_t)3 * first, sm + kSmXyz, 3 * nv, vec);
  if (out.dscales) copy_out(out.dscales + (size_t)3 * first, sm + kSmSc, 3 * nv, vec);
  if (out.drots) copy_out(out.drots + (size_t)4 * first, sm + kSmQ, 4 * nv, vec);
  if (out.dopac) copy_out(out.dopac + first, sm + kSmOp, nv, vec);
  if (use_sh && out.dsh_dc) {
    if (in.sh_packed) {
      stage_out(out.dsh_dc + (size_t)3 * M * first, sm + kSmSh, 3 * M * nv, 3 * M, kRowPad, 0, vec);
    } else {
      copy_out(out.dsh_dc + (size_t)3 * first, sm + kSmSh, 3 * nv, vec);
      if (M > 1 && out.dsh_rest)
        copy_out(out.dsh_rest + (size_t)3 * (M - 1) * first, sm + kSmSh + 3 * kPT, 3 * (M - 1) * nv, vec);
    }
  }
  }
  // pose-gradient partials: warp shuffle, then across the 8 warps
  if (cam->pose_on) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      float v = pa[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) s_pose[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < 16) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kPT / 32; ++w) v += s_pose[w][threadIdx.x];
      gv.pose_part[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 16 + threadIdx.x] = v;
    }
  }
  if (bulk_out && threadIdx.x == 0) bulk_wait_read();   // shared memory must outlive the bulk stores reading it
}

// Pose-gradient partials [V][nblocks][16] -> 16 column sums per view (grid (16, V), one CTA per column, deterministic
// order) ...
__global__ void __launch_bounds__(256) k_pose_reduce(const float* __restrict__ part, int nblocks, float* __restrict__ acc16) {
  __shared__ float s[256];
  const int c = blockIdx.x;
  part += (size_t)blockIdx.y * nblocks * 16;
  acc16 += 16 * blockIdx.y;
  float v0 = 0.f, v1 = 0.f, v2 = 0.f, v3 = 0.f;
  int b = threadIdx.x;
  for (; b + 768 < nblocks; b += 1024) {
    v0 += part[(size_t)b * 16 + c];
    v1 += part[(size_t)(b + 256) * 16 + c];
    v2 += part[(size_t)(b + 512) * 16 + c];
    v3 += part[(size_t)(b + 768) * 16 + c];
  }
  for (; b < nblocks; b += 256) v0 += part[(size_t)b * 16 + c];
  s[threadIdx.x] = (v0 + v1) + (v2 + v3);
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) acc16[c] = s[0];
}
// ... and the chain to dL/dP[7] (utils/pose_utils.py quad2rotation + normalisation backward).
//     (one CTA per view)
__global__ void k_pose_finalize(const float* __restrict__ acc16, const float* pose, float* dpose) {
  if (threadIdx.x != 0) return;
  acc16 += 16 * blockIdx.x;
  pose += 7 * blockIdx.x;
  dpose += 7 * blockIdx.x;
  float acc[16];
  for (int c = 0; c < 16; ++c) acc[c] = acc16[c];
  float dp[7];
  pose_grad_finalize(pose, acc, dp);
  for (int c = 0; c < 7; ++c) dpose[c] = dp[c];
}

__global__ void k_mark_visible(int P, const float* means, const float* V, uint8_t* present) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  float z = means[3 * i] * V[2] + means[3 * i + 1] * V[6] + means[3 * i + 2] * V[10] + V[14];
  present[i] = z > kNear ? 1 : 0;
}
// ------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------
static int make_inptrs(const GsbCamera* cam, const GsbGaussians* g, InPtrs& in) {
  GSB_REQUIRE(cam && g, "null camera / gaussians");
  GSB_REQUIRE(g->P >= 0, "P < 0");
  GSB_REQUIRE(cam->width > 0 && cam->height > 0, "image size");
  GSB_REQUIRE((long long)((cam->width + kBlock - 1) / kBlock) * ((cam->height + kBlock - 1) / kBlock) < kMaxTiles,
              "image too large (more than 65535 tiles)");
  GSB_REQUIRE(cam->sh_degree >= 0 && cam->sh_degree <= 3, "sh_degree must be 0..3");
  GSB_REQUIRE(cam->sh_coeffs >= 1 && cam->sh_coeffs <= 16, "sh_coeffs must be 1..16");
  GSB_REQUIRE((cam->sh_degree + 1) * (cam->sh_degree + 1) <= cam->sh_coeffs || g->colors_precomp,
              "active SH degree exceeds stored coefficients");
  GSB_REQUIRE(cam->bg && cam->viewmatrix && cam->projmatrix && cam->campos, "null camera tensor");
  if (g->P > 0) {   // an empty cloud may come with null tensors
    GSB_REQUIRE(g->means3D && g->opacities, "means3D / opacities are required");
    GSB_REQUIRE((g->sh_dc != nullptr) != (g->colors_precomp != nullptr),
                "provide exactly one of SHs / precomputed colours");
    GSB_REQUIRE((g->scales != nullptr && g->rotations != nullptr) != (g->cov3D_precomp != nullptr),
                "provide exactly one of scale+rotation / precomputed 3D covariance");
    if (g->sh_dc && !g->sh_packed && cam->sh_coeffs > 1 && cam->sh_degree > 0)
      GSB_REQUIRE(g->sh_rest != nullptr, "sh_rest missing");
  }
  in.P = g->P; in.means = g->means3D; in.scales = g->scales; in.rots = g->rotations; in.opac = g->opacities;
  in.sh_dc = g->sh_dc; in.sh_rest = g->sh_rest; in.colors = g->colors_precomp; in.cov3D = g->cov3D_precomp;
  in.sh_packed = g->sh_packed; in.exact_cull = cam->exact_cull;
  uintptr_t a = (uintptr_t)g->means3D | (uintptr_t)g->scales | (uintptr_t)g->rotations |
                (uintptr_t)g->opacities | (uintptr_t)g->sh_dc | (uintptr_t)g->sh_rest;
  in.vec_ok = (a & 15) == 0;
  in.mip = Mip(); in.filter3D = nullptr;
  return GSB_OK;
}

// the Mip filters of GsbFilter (NULL: reference path)
static int apply_filter(const GsbFilter* f, const GsbGaussians* g, InPtrs& in) {
  if (!f) return GSB_OK;
  GSB_REQUIRE((f->flags & ~GSB_FILTER_MIP2D) == 0, "GsbFilter: unknown flags");
  const bool on2d = (f->flags & GSB_FILTER_MIP2D) != 0, on3d = f->filter3D != nullptr;
  if (on2d) GSB_REQUIRE(f->kernel_size >= 0.f && f->kernel_size < 1.0e30f, "GsbFilter: kernel_size must be >= 0");
  if (on3d) GSB_REQUIRE(g->raw_params && g->scales, "GsbFilter: filter3D needs raw parameters with scales");
  in.mip.on = on2d || on3d;
  in.mip.on2d = on2d; in.mip.on3d = on3d; in.mip.kappa = on2d ? f->kernel_size : 0.f;
  in.filter3D = f->filter3D;
  return GSB_OK;
}

// cudaFuncSetAttribute is per device: remember which devices have been configured
static int ensure_attrs() {
  static bool done[64] = {};
  int dev = 0;
  GSB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !done[dev]) {
    for (auto k : {k_preprocess<false>, k_preprocess<true>})
      GSB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPrepSmem));
    for (auto k : {k_preprocess_bwd<false, false>, k_preprocess_bwd<true, false>, k_preprocess_bwd<false, true>,
                   k_preprocess_bwd<true, true>})
      GSB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPrepSmem));
    for (auto k : {k_preprocess_bwd<false, false, true>, k_preprocess_bwd<true, false, true>,
                   k_preprocess_bwd<false, true, true>, k_preprocess_bwd<true, true, true>})
      GSB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPrepSmemViews));
    if (dev >= 0 && dev < 64) done[dev] = true;
  }
  return GSB_OK;
}

extern "C" GSB_API uint32_t* gsb_status_device(void* geom, int32_t P) { return geom ? geom_view(geom, P).status : nullptr; }
extern "C" GSB_API uint32_t* gsb_status_device_batch(void* geom, int32_t P, int32_t V) {
  return geom ? geom_view(geom, P, V).status : nullptr;      // the status words precede the tile arrays
}

static CamArgs cam_args(const GsbCamera* cam, const GsbGaussians* g) {
  CamArgs a;
  a.V = cam->viewmatrix; a.Pm = cam->projmatrix; a.campos = cam->campos; a.pose = g->pose;
  a.W = cam->width; a.H = cam->height; a.tanfovx = cam->tanfovx; a.tanfovy = cam->tanfovy;
  a.scale_mod = cam->scale_modifier; a.D = cam->sh_degree; a.M = cam->sh_coeffs; a.raw_params = g->raw_params;
  return a;
}

// A batch of V views shares cam (intrinsics, background) and g (the Gaussians); with V > 1 the poses come from
// g->pose as a [V, 7] table.  V = 1 is the single-view forward.
static int batch_args(int V, const GsbCamera* cam, const GsbGaussians* g) {
  GSB_REQUIRE(V >= 1 && V <= 65535, "V must be in 1..65535 (grid y)");
  GSB_REQUIRE(cam && g && g->P >= 0, "null camera / gaussians");
  GSB_REQUIRE((long long)V * g->P < 0x7fffffffLL, "V * P must be below 2^31");
  GSB_REQUIRE(cam->width > 0 && cam->height > 0 && (long long)V * frame_tiles(cam->width, cam->height) < 0x7fffffffLL,
              "V * tiles must be below 2^31");
  GSB_REQUIRE(V == 1 || (g->pose && g->raw_params), "a batch needs raw parameters and a [V, 7] pose table");
  return GSB_OK;
}

static int preprocess_views(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, int V, void* geom,
                            size_t geom_bytes, int32_t* radii, uint32_t* status_host, cudaStream_t st) {
  int rc = batch_args(V, cam, g);
  if (rc) return rc;
  InPtrs in;
  rc = make_inptrs(cam, g, in);
  if (rc) return rc;
  rc = apply_filter(filt, g, in);
  if (rc) return rc;
  GSB_REQUIRE(geom && (radii || g->P == 0), "null buffer");
  const int P = g->P;
  const int ntiles = frame_tiles(cam->width, cam->height);
  GeomView gv = geom_view(geom, P, V, ntiles);
  if (gv.total > geom_bytes) { gsb_set_error("geom buffer too small"); return GSB_ERR_CAPACITY; }
  rc = ensure_attrs();
  if (rc) return rc;
  gsb_count_launch(1);
  k_setup_cam<<<V, 32, 0, st>>>(gv.cam, cam_args(cam, g));
  // aux (the per-forward counters) sits immediately before tcount: one memset clears both
  GSB_CUDA(cudaMemsetAsync(gv.aux, 0, (size_t)((char*)gv.tcount - (char*)gv.aux) + (size_t)V * ntiles * 4, st));
  if (P > 0) {
    const int nb = (P + kPT - 1) / kPT;
    ProfScope ps(GSB_K_PREPROCESS, st, 2);
    (in.mip.on ? k_preprocess<true> : k_preprocess<false>)<<<dim3(nb, V), kPT, kPrepSmem, st>>>(in, gv, radii);
    rc = gsb_launch_big_rects(P, V, gv, nullptr, cam->width, cam->height, cam->exact_cull, 0u, st);   // count mode
    if (rc) return rc;
  }
  rc = gsb_launch_tile_scan(gv, V * ntiles, st);
  if (rc) return rc;
  if (status_host) GSB_CUDA(cudaMemcpyAsync(status_host, gv.status, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}

extern "C" GSB_API int gsb_preprocess_ex(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt,
                                         void* geom, size_t geom_bytes, int32_t* radii, uint32_t* status_host,
                                         gsb_stream_t stream) {
  return preprocess_views(cam, g, filt, 1, geom, geom_bytes, radii, status_host, (cudaStream_t)stream);
}

extern "C" GSB_API int gsb_preprocess_batch(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt,
                                            int32_t V, const float* poses7, void* geom, size_t geom_bytes,
                                            int32_t* radii, uint32_t* status_host, gsb_stream_t stream) {
  GSB_REQUIRE(g && poses7, "gsb_preprocess_batch: null gaussians / poses");
  GsbGaussians gb = *g;
  gb.pose = poses7;
  return preprocess_views(cam, &gb, filt, V, geom, geom_bytes, radii, status_host, (cudaStream_t)stream);
}

extern "C" GSB_API int gsb_preprocess(const GsbCamera* cam, const GsbGaussians* g, void* geom, size_t geom_bytes,
                                      int32_t* radii, uint32_t* status_host, gsb_stream_t stream) {
  return gsb_preprocess_ex(cam, g, nullptr, geom, geom_bytes, radii, status_host, stream);
}

// bg_table: [V, 3] backgrounds, view v's at bg_table + 3 v (NULL: cam->bg for every view)
static int render_views(const GsbCamera* cam, int32_t P, int V, void* geom, void* binning, size_t binning_bytes,
                        int64_t R, void* image, float* out_color, uint32_t* status_host, cudaStream_t st,
                        const float* bg_table = nullptr) {
  GSB_REQUIRE(cam && geom && binning && image && out_color, "null buffer");
  GSB_REQUIRE(R >= 0 && R < (int64_t)0x7fffffff, "R out of range");
  GSB_REQUIRE(V >= 1 && V <= 65535 && P >= 0 && (long long)V * P < 0x7fffffffLL, "bad V / P");
  const int W = cam->width, H = cam->height;
  GeomView gv = geom_view(geom, P, V, frame_tiles(W, H));
  BinView bv = bin_view(binning, R, W, H, V);
  if (bv.total > binning_bytes) { gsb_set_error("binning buffer too small"); return GSB_ERR_CAPACITY; }
  ImgView iv = img_view(image, W, H, V);
  int rc = gsb_launch_binning(P, V, gv, bv, W, H, cam->exact_cull, (uint32_t)R, st);
  if (rc) return rc;
  rc = gsb_launch_blend_fwd(gv, bv, iv, bg_table ? bg_table : cam->bg, bg_table ? 3 : 0, W, H, V, out_color, st);
  if (rc) return rc;
  if (status_host) GSB_CUDA(cudaMemcpyAsync(status_host, gv.status, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}

extern "C" GSB_API int gsb_render(const GsbCamera* cam, int32_t P, void* geom, void* binning, size_t binning_bytes,
                          int64_t R, void* image, float* out_color, uint32_t* status_host, gsb_stream_t stream) {
  return render_views(cam, P, 1, geom, binning, binning_bytes, R, image, out_color, status_host, (cudaStream_t)stream);
}

extern "C" GSB_API int gsb_render_batch(const GsbCamera* cam, int32_t P, int32_t V, void* geom, void* binning,
                                        size_t binning_bytes, int64_t R, void* image, float* out_color,
                                        uint32_t* status_host, gsb_stream_t stream) {
  return render_views(cam, P, V, geom, binning, binning_bytes, R, image, out_color, status_host, (cudaStream_t)stream);
}

extern "C" GSB_API int gsb_render_batch_bg(const GsbCamera* cam, int32_t P, int32_t V, const float* bg, void* geom,
                                           void* binning, size_t binning_bytes, int64_t R, void* image,
                                           float* out_color, uint32_t* status_host, gsb_stream_t stream) {
  GSB_REQUIRE(bg, "gsb_render_batch_bg: null background table");
  return render_views(cam, P, V, geom, binning, binning_bytes, R, image, out_color, status_host, (cudaStream_t)stream,
                      bg);
}

static int backward_views(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, const GsbDensifyStats* stats,
                          int V, void* geom, void* binning, int64_t R, void* image, const float* dL_dout,
                          const GsbGrads* grads, cudaStream_t st, bool sum_views = false, int n_stats = 1,
                          const float* bg_table = nullptr);

extern "C" GSB_API int gsb_backward_stats(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt,
                                          const GsbDensifyStats* stats, void* geom, void* binning, int64_t R, void* image,
                                          const float* dL_dout, const GsbGrads* grads, gsb_stream_t stream) {
  return backward_views(cam, g, filt, stats, 1, geom, binning, R, image, dL_dout, grads, (cudaStream_t)stream);
}

extern "C" GSB_API int gsb_backward_pose_batch(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt,
                                               int32_t V, const float* poses7, void* geom, void* binning, int64_t R,
                                               void* image, const float* dL_dout, float* dpose7, gsb_stream_t stream) {
  GSB_REQUIRE(g && poses7 && dpose7, "gsb_backward_pose_batch: null gaussians / poses / dpose");
  GsbGaussians gb = *g;
  gb.pose = poses7;
  GsbGrads gr;
  memset(&gr, 0, sizeof(gr));
  gr.dL_dpose = dpose7;
  return backward_views(cam, &gb, filt, nullptr, V, geom, binning, R, image, dL_dout, &gr, (cudaStream_t)stream);
}

static int backward_batch(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, int32_t V, int32_t n_stats,
                          const GsbDensifyStats* stats, const float* bg_table, const float* poses7, void* geom,
                          void* binning, int64_t R, void* image, const float* dL_dout, const GsbGrads* grads,
                          float* dpose7, gsb_stream_t stream) {
  GSB_REQUIRE(n_stats >= 0 && n_stats <= V, "gsb_backward_batch_stats: n_stats must be in 0..V");
  GSB_REQUIRE(stats || n_stats == 0, "gsb_backward_batch_stats: n_stats > 0 needs statistics");
  GSB_REQUIRE(g && poses7 && grads && dpose7, "gsb_backward_batch: null gaussians / poses / grads / dpose");
  GSB_REQUIRE(!g->colors_precomp && !g->cov3D_precomp && !grads->dL_dcolors && !grads->dL_dcov3D,
              "gsb_backward_batch: SH colours and scale / rotation only (no precomputed colours or covariances)");
  GsbGaussians gb = *g;
  gb.pose = poses7;
  GsbGrads gr = *grads;
  gr.dL_dpose = dpose7;
  return backward_views(cam, &gb, filt, stats, V, geom, binning, R, image, dL_dout, &gr, (cudaStream_t)stream, true,
                        n_stats, bg_table);
}

extern "C" GSB_API int gsb_backward_batch_stats(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt,
                                                int32_t V, int32_t n_stats, const GsbDensifyStats* stats,
                                                const float* poses7, void* geom, void* binning, int64_t R, void* image,
                                                const float* dL_dout, const GsbGrads* grads, float* dpose7,
                                                gsb_stream_t stream) {
  return backward_batch(cam, g, filt, V, n_stats, stats, nullptr, poses7, geom, binning, R, image, dL_dout, grads, dpose7,
                        stream);
}

extern "C" GSB_API int gsb_backward_batch_stats_bg(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt,
                                                   int32_t V, const float* bg, int32_t n_stats,
                                                   const GsbDensifyStats* stats, const float* poses7, void* geom,
                                                   void* binning, int64_t R, void* image, const float* dL_dout,
                                                   const GsbGrads* grads, float* dpose7, gsb_stream_t stream) {
  GSB_REQUIRE(bg, "gsb_backward_batch_stats_bg: null background table");
  return backward_batch(cam, g, filt, V, n_stats, stats, bg, poses7, geom, binning, R, image, dL_dout, grads, dpose7,
                        stream);
}

extern "C" GSB_API int gsb_backward_batch(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, int32_t V,
                                          const float* poses7, void* geom, void* binning, int64_t R, void* image,
                                          const float* dL_dout, const GsbGrads* grads, float* dpose7,
                                          gsb_stream_t stream) {
  return gsb_backward_batch_stats(cam, g, filt, V, 0, nullptr, poses7, geom, binning, R, image, dL_dout, grads, dpose7,
                                  stream);
}

// dL/dpose is computed per view.  sum_views (gsb_backward_batch_stats): the per-Gaussian gradients are those of all V
// views, summed in view order, bit-identical to V single-view calls added in that order (k_preprocess_bwd<., ., true>),
// and with stats the densification statistics of views 0 .. n_stats-1 (stats->radii: the batch's [V, P] radii).
// Otherwise a batch (V > 1) writes no per-Gaussian gradient and takes no statistics (gsb_backward_pose_batch), and a
// single view counts its statistics when stats is given.
static int backward_views(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, const GsbDensifyStats* stats,
                          int V, void* geom, void* binning, int64_t R, void* image, const float* dL_dout,
                          const GsbGrads* grads, cudaStream_t st, bool sum_views, int n_stats, const float* bg_table) {
  int rc = batch_args(V, cam, g);
  if (rc) return rc;
  InPtrs in;
  rc = make_inptrs(cam, g, in);
  if (rc) return rc;
  rc = apply_filter(filt, g, in);
  if (rc) return rc;
  GSB_REQUIRE(geom && binning && image && dL_dout && grads, "null buffer");
  if (g->pose) GSB_REQUIRE(grads->dL_dpose != nullptr, "dL_dpose required when pose is fused");
  GSB_REQUIRE(!stats || V == 1 || sum_views, "densification statistics of a batch need the view-summing backward");
  if (stats)
    GSB_REQUIRE((stats->radii && stats->grad_accum && stats->denom && stats->max_radii2D) || g->P == 0,
                "GsbDensifyStats: null buffer");
  const int P = g->P, W = cam->width, H = cam->height;
  GeomView gv = geom_view(geom, P, V, frame_tiles(W, H));
  BinView bv = bin_view(binning, R, W, H, V);
  ImgView iv = img_view(image, W, H, V);
  rc = ensure_attrs();
  if (rc) return rc;
  if (P == 0) {
    if (grads->dL_dpose) GSB_CUDA(cudaMemsetAsync(grads->dL_dpose, 0, (size_t)V * 7 * 4, st));
    return GSB_OK;
  }
  GSB_CUDA(cudaMemsetAsync(gv.dacc, 0, (size_t)V * P * kDaccSlots * 8, st));
  GSB_CUDA(cudaMemsetAsync(gv.dscale, 0, (size_t)V * 4, st));
  // tracking mode (render.py:99-170): only dL/dpose is wanted -> the blend backward reduces 8 values instead of 9.
  // Not with the 2D Mip filter: o_eff depends on Sigma2 and so on the pose, whose gradient then needs S w (slot 5).
  const bool pose_only = !in.mip.on2d && g->pose && grads->dL_dpose && !grads->dL_dmeans3D && !grads->dL_dmeans2D && !grads->dL_dscales &&
                         !grads->dL_drotations && !grads->dL_dopacities && !grads->dL_dsh_dc && !grads->dL_dsh_rest &&
                         !grads->dL_dcolors && !grads->dL_dcov3D && gsb_option_blend_version() == 2 &&
                         gsb_option_stage_bulk() == 1;
  rc = gsb_launch_blend_bwd(gv, bv, iv, bg_table ? bg_table : cam->bg, bg_table ? 3 : 0, W, H, V, dL_dout, pose_only,
                            st);
  if (rc) return rc;
  OutPtrs out;
  out.dmeans = grads->dL_dmeans3D; out.dmeans2D = grads->dL_dmeans2D; out.dscales = grads->dL_dscales;
  out.drots = grads->dL_drotations; out.dopac = grads->dL_dopacities; out.dsh_dc = grads->dL_dsh_dc;
  out.dsh_rest = grads->dL_dsh_rest; out.dcolors = grads->dL_dcolors; out.dcov3D = grads->dL_dcov3D;
  uintptr_t a = (uintptr_t)out.dmeans | (uintptr_t)out.dscales | (uintptr_t)out.drots | (uintptr_t)out.dopac |
                (uintptr_t)out.dsh_dc | (uintptr_t)out.dsh_rest;
  if (a & 15) in.vec_ok = 0;
  StatsPtrs sp;
  sp.radii = stats ? stats->radii : nullptr; sp.accum = stats ? stats->grad_accum : nullptr;
  sp.denom = stats ? stats->denom : nullptr; sp.max_r = stats ? stats->max_radii2D : nullptr;
  const int nb = (P + kPT - 1) / kPT;
  { ProfScope ps(GSB_K_PREPROCESS_BWD, st, g->pose ? 3 : 1);
    if (sum_views) {
      const bool count = stats && n_stats > 0;
      auto kern = in.mip.on ? (count ? k_preprocess_bwd<true, true, true> : k_preprocess_bwd<true, false, true>)
                            : (count ? k_preprocess_bwd<false, true, true> : k_preprocess_bwd<false, false, true>);
      kern<<<nb, kPT, kPrepSmemViews, st>>>(in, gv, pose_only ? 1 : 0, out, sp, V, count ? n_stats : 0);
    } else {
      auto kern = in.mip.on ? (stats ? k_preprocess_bwd<true, true> : k_preprocess_bwd<true, false>)
                            : (stats ? k_preprocess_bwd<false, true> : k_preprocess_bwd<false, false>);
      kern<<<dim3(nb, V), kPT, kPrepSmem, st>>>(in, gv, pose_only ? 1 : 0, out, sp, 1, 0);
    }
    if (g->pose) {
      k_pose_reduce<<<dim3(16, V), 256, 0, st>>>(gv.pose_part, nb, gv.pose_acc);
      k_pose_finalize<<<V, 32, 0, st>>>(gv.pose_acc, g->pose, grads->dL_dpose);
    } }
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}

extern "C" GSB_API int gsb_backward_ex(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, void* geom,
                                       void* binning, int64_t R, void* image, const float* dL_dout, const GsbGrads* grads,
                                       gsb_stream_t stream) {
  return gsb_backward_stats(cam, g, filt, nullptr, geom, binning, R, image, dL_dout, grads, stream);
}

extern "C" GSB_API int gsb_backward(const GsbCamera* cam, const GsbGaussians* g, void* geom, void* binning, int64_t R,
                                    void* image, const float* dL_dout, const GsbGrads* grads, gsb_stream_t stream) {
  return gsb_backward_ex(cam, g, nullptr, geom, binning, R, image, dL_dout, grads, stream);
}

extern "C" GSB_API int gsb_mark_visible(int32_t P, const float* means3D, const float* viewmatrix,
                                const float* projmatrix, uint8_t* present, gsb_stream_t stream_) {
  (void)projmatrix;
  GSB_REQUIRE(P >= 0 && means3D && viewmatrix && present, "null buffer");
  if (P > 0)
    k_mark_visible<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream_>>>(P, means3D, viewmatrix, present);
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}
