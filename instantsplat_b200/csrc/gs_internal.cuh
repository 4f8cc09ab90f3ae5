// Internal declarations shared by the translation units of libgsb200.so (not part of the C ABI):
// error handling, per-kernel timing hooks, and the layouts of the three caller-owned scratch buffers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/gsb200.h"
#include "gs_math.cuh"

// ------------------------------------------------------------------------------------------
// error handling (thread-local message, see gsb_last_error)
// ------------------------------------------------------------------------------------------
void gsb_set_error(const char* s);
void gsb_set_errorf(const char* file, int line, const char* what, const char* detail);
#define GSB_CUDA(x)                                                                       \
  do {                                                                                    \
    cudaError_t e_ = (x);                                                                 \
    if (e_ != cudaSuccess) {                                                              \
      gsb_set_errorf(__FILE__, __LINE__, #x, cudaGetErrorString(e_));                     \
      return GSB_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)
#define GSB_REQUIRE(cond, msg)                                                            \
  do {                                                                                    \
    if (!(cond)) {                                                                        \
      gsb_set_errorf(__FILE__, __LINE__, "invalid argument", msg);                        \
      return GSB_ERR_INVALID;                                                             \
    }                                                                                     \
  } while (0)

// ------------------------------------------------------------------------------------------
// optional per-kernel timing (CUDA events on the launching stream) and launch counting
// ------------------------------------------------------------------------------------------
void gsb_count_launch(int n);
int gsb_prof_begin(int id, cudaStream_t st);
void gsb_prof_end(int slot, cudaStream_t st);
struct ProfScope {
  int slot; cudaStream_t st;
  ProfScope(int id, cudaStream_t s, int launches = 1) : st(s) { gsb_count_launch(launches); slot = gsb_prof_begin(id, s); }
  ~ProfScope() { gsb_prof_end(slot, st); }
};
int gsb_option_blend_version();
int gsb_option_stage_bulk();
int gsb_option_blend_bwd_batch();
int gsb_sm_count();

namespace gsb {

static inline size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

constexpr int kThreads = 256;
constexpr int kPT = 128;           // threads (= Gaussians) per CTA in the per-Gaussian kernels
constexpr int kMaxTiles = 65536;   // tile ids are 16 bit (a 4K frame has 32400 tiles)

// status words written by the forward (device) and copied to the caller's pinned host array
enum { kStR = 0, kStOverflow = 1, kStMaxList = 2, kStHugeTiles = 3, kStNLarge = 4, kStNHuge = 5, kStSeq = 6,
       kStWords = 8 };
// tile-list size classes of the per-tile sort (gs_bin.cu): <= kSmallList entries are sorted by the one-CTA-per-tile
// kernel; longer lists are queued by k_tile_scan and drained by two persistent kernels
constexpr uint32_t kSmallList = 2048, kLargeList = 8192;

// ---- fixed-point backward accumulators ----------------------------------------------------
// The blend backward adds per-Gaussian pixel moments from many tiles.  Floating-point atomics would make each sum
// depend on the order in which the CTAs arrive, so the gradients -- and, through Adam, a whole training run -- would
// differ from run to run.  The moments are added as 64-bit integers instead; integer addition is associative, so every
// run produces the same bits.  Slot k of Gaussian i counts in units of 1 / fix_scale(k, e_i, M) with
// M = max |dL/dpixel| of the launch and e_i the Gaussian's extent (fix_extent): the smaller of its radius and the
// Chebyshev distance from its centre to the farthest pixel centre of the frame.  Every pixel it contributes to lies
// within both, so |dx|, |dy| <= ~e and the pixels covered are ~e^2: |slot k| <= c * M * (e + 1)^fix_exp(k) for a small
// constant c, and the unit 2^-50 * M * (e + 1)^fix_exp(k) leaves 13 bits of headroom above that bound and ~50 bits of
// resolution below it -- finer than the float each contribution starts from.  (With the radius alone, a Gaussian just
// in front of the near plane -- radius 1e5 px on a 256 px frame -- would lose ~35 of those bits.)
// Slots: [S w dx, S w dy, S w dx^2, S w dx dy, S w dy^2, S w (tracking: dL/db), dL/dr, dL/dg, dL/db].
constexpr int kDaccSlots = 9;
__host__ __device__ constexpr int fix_exp(int k) { return k < 2 ? 3 : (k < 5 ? 4 : 2); }
// the extent of the fixed-point unit, stored in the splat record (rec[2].w) by k_preprocess for the blend backward
// (encoder) and k_preprocess_bwd (decoder); 0 for a Gaussian that covers nothing
__host__ __device__ inline float fix_extent(int radius, float x, float y, int W, int H) {
  const float reach = fmaxf(fmaxf(fabsf(x), fabsf((float)(W - 1) - x)), fmaxf(fabsf(y), fabsf((float)(H - 1) - y)));
  return fminf((float)radius, reach);
}
#if defined(__CUDACC__)
// 2^50 / M (M floored at 1e-20 so that the scale stays a finite float)
__device__ __forceinline__ float fix_inv_m(const uint32_t* dscale) {
  return __fdiv_rn(0x1p50f, fmaxf(__uint_as_float(*dscale), 1e-20f));
}
// integer steps per unit of slot k for a Gaussian of the given extent.  Encoder and decoder evaluate the same expression
// (MUFU.RCP is deterministic), so the approximate reciprocal costs nothing in reproducibility.
__device__ __forceinline__ float fix_scale(int k, float extent, float inv_m) {
  float ri;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(ri) : "f"(extent + 1.f));
  const int e = fix_exp(k);
  float s = __fmul_rn(__fmul_rn(inv_m, ri), ri);
  if (e >= 3) s = __fmul_rn(s, ri);
  if (e >= 4) s = __fmul_rn(s, ri);
  return s;
}
__device__ __forceinline__ unsigned long long fix_encode(float x, float scale) {
  return (unsigned long long)__float2ll_rn(__fmul_rn(x, scale));
}
// unit = 1 / fix_scale(...) in double, computed once per Gaussian and exponent
__device__ __forceinline__ float fix_decode(unsigned long long a, double unit) { return (float)((double)(long long)a * unit); }
#endif

// ---- geom: P-sized scratch + per-tile counters (caller-owned, gsb_geom_bytes) -------------
struct GeomView {
  CamConst* cam;
  float4* rec;         // [3P] one 48-byte splat record per Gaussian, array of structures (the blend kernels gather it by id):
                       //   [0] x, y, A', B'      [1] C', opacity, cull threshold', id (bits)      (conic in the log2 domain:
                       //   [2] r, g, b, fix_extent                                                 power*log2e = A'dx^2+B'dxdy+C'dy^2)
  float4* brec;        // [P] binning record: depth, rect x (rx0 | rx1<<16), rect y (ry0 | ry1<<16), keep mask (bits)
  uint32_t* tiles;     // tile instances per Gaussian (after culling)
  uint8_t* clamped;
  unsigned long long* dacc;   // [kDaccSlots * P] backward accumulators, fixed point (see fix_scale)
  uint32_t* dscale;    // [V] max |dL/dpixel| of each view's current backward (float bits), the unit of the fixed point
  float* pose_part;    // [nblocks*16]
  float* pose_acc;     // [16]
  uint32_t* status;    // [kStWords]
  uint32_t* aux;       // [64] per-forward counters, zeroed together with tcount (they are adjacent): [0] = length of q_big
  uint32_t* tcount;    // [tile_slots] instances per tile (counted by k_preprocess / k_big_rects)
  uint32_t* tstart;    // [tile_slots] exclusive scan of tcount
  uint32_t* tcursor;   // [tile_slots] emission cursors (k_scatter)
  uint32_t* q_large;   // [tile_slots] tiles whose list has kSmallList < n <= kLargeList entries
  uint32_t* q_huge;    // [tile_slots] tiles with longer lists
  uint32_t* q_big;     // [V * P] records whose tile rect exceeds kBigRect tiles (walked by k_big_rects, flattened)
  size_t total;
};

// V > 1: a batch of V views of the same P Gaussians (gsb_preprocess_batch).  Record id r = v * P + i, so every
// per-record array has V * P entries; global tile index = v * ntiles + t, so the per-tile arrays hold V * ntiles
// entries (at least kMaxTiles, which makes V = 1 the single-view layout).
static inline size_t tile_slots(int V, int ntiles) {
  const size_t n = (size_t)(V > 0 ? V : 1) * (size_t)(ntiles > 0 ? ntiles : 0);
  return n > (size_t)kMaxTiles ? n : (size_t)kMaxTiles;
}
static inline GeomView geom_view(void* base, int P, int V = 1, int ntiles = 0) {
  GeomView v;
  size_t off = 0;
  char* p = (char*)base;
  size_t Pp = (size_t)(P > 0 ? P : 1);
  const size_t nv = (size_t)(V > 0 ? V : 1), VP = nv * Pp, TS = tile_slots(V, ntiles);
  auto take = [&](size_t bytes) { void* r = p ? p + off : nullptr; off += align_up(bytes); return r; };
  v.cam = (CamConst*)take(nv * sizeof(CamConst));
  v.rec = (float4*)take(VP * 48);
  v.brec = (float4*)take(VP * 16);
  v.tiles = (uint32_t*)take(VP * 4);
  v.clamped = (uint8_t*)take(VP);
  v.dacc = (unsigned long long*)take(VP * kDaccSlots * 8);
  v.dscale = (uint32_t*)take(nv * 4);
  size_t nb = (Pp + kPT - 1) / kPT;
  v.pose_part = (float*)take(nv * nb * 16 * 4);
  v.pose_acc = (float*)take(nv * 16 * 4);
  v.status = (uint32_t*)take(kStWords * 4);
  v.aux = (uint32_t*)take(64 * 4);                        // exactly 256 bytes: tcount follows immediately
  v.tcount = (uint32_t*)take(TS * 4);
  v.tstart = (uint32_t*)take(TS * 4);
  v.tcursor = (uint32_t*)take(TS * 4);
  v.q_large = (uint32_t*)take(TS * 4);
  v.q_huge = (uint32_t*)take(TS * 4);
  v.q_big = (uint32_t*)take(VP * 4);
  v.total = off;
  return v;
}

// ---- binning: capacity-sized scratch (caller-owned, gsb_binning_bytes) --------------------
struct BinView {
  unsigned long long* pairs;   // [cap] (depth bits << 32 | Gaussian id), unsorted per-tile segments
  uint32_t* ids;               // [cap + 8] Gaussian ids, per tile in (depth, id) order (what the blend kernels walk)
  uint2* ranges;               // [tiles]
  size_t total;
};

static inline BinView bin_view(void* base, int64_t cap, int W, int H, int V = 1) {
  BinView v;
  size_t off = 0;
  char* p = (char*)base;
  size_t Rp = (size_t)(cap > 0 ? cap : 1);
  int ntiles = ((W + kBlock - 1) / kBlock) * ((H + kBlock - 1) / kBlock);
  auto take = [&](size_t bytes) { void* r = p ? p + off : nullptr; off += align_up(bytes); return r; };
  v.pairs = (unsigned long long*)take(Rp * 8);
  v.ids = (uint32_t*)take((Rp + 8) * 4);       // + 8: bulk copies of id chunks are rounded to 16 bytes
  v.ranges = (uint2*)take((size_t)(V > 0 ? V : 1) * ntiles * 8);
  v.total = off;
  return v;
}

struct ImgView {
  float* final_T;
  uint32_t* n_contrib;
  size_t total;
};
static inline ImgView img_view(void* base, int W, int H, int V = 1) {
  ImgView v;
  size_t hw = (size_t)(V > 0 ? V : 1) * W * H;
  char* p = (char*)base;
  v.final_T = (float*)p;
  v.n_contrib = (uint32_t*)(p ? p + align_up(hw * 4) : nullptr);
  v.total = 2 * align_up(hw * 4);
  return v;
}

}  // namespace gsb

// ---- launchers implemented in gs_bin.cu / gs_blend.cu -----------------------------------------
// tile scan: tstart = exclusive scan(tcount), status = {R, 0, max list, 0, long-list queue lengths, serial}
int gsb_launch_tile_scan(const gsb::GeomView& gv, int ntiles, cudaStream_t st);
// P: Gaussians per view; V views (record id v * P + i, tile v * ntiles + t)
int gsb_launch_big_rects(int P, int V, const gsb::GeomView& gv, unsigned long long* pairs, int W, int H, int exact_cull,
                         uint32_t cap, cudaStream_t st);
// scatter + per-tile (depth, id) sort + slab gather + ranges; cap = instance capacity of the binning buffer
int gsb_launch_binning(int P, int V, const gsb::GeomView& gv, const gsb::BinView& bv, int W, int H, int exact_cull,
                       uint32_t cap, cudaStream_t st);
// out_color [V, 3, H, W]; view v's background is bg + v * bg_stride (0: one shared [3], 3: a [V, 3] table; v2 only)
int gsb_launch_blend_fwd(const gsb::GeomView& gv, const gsb::BinView& bv, const gsb::ImgView& iv, const float* bg,
                         int bg_stride, int W, int H, int V, float* out_color, cudaStream_t st);
// pose_only: 8-value accumulator layout (dacc[5] = dL/db, no dL/dopacity), see k_blend_bwd2
// computes max |dL_dout| into gv.dscale (zeroed by the caller, as is gv.dacc), then the blend backward into gv.dacc
// dL_dout [V, 3, H, W]; one M per view (gv.dscale[v]); bg, bg_stride as in gsb_launch_blend_fwd
int gsb_launch_blend_bwd(const gsb::GeomView& gv, const gsb::BinView& bv, const gsb::ImgView& iv, const float* bg,
                         int bg_stride, int W, int H, int V, const float* dL_dout, bool pose_only, cudaStream_t st);
