// Binning for the rasterizer: from per-Gaussian splat records to per-tile, depth-ordered slabs --
// hand-written, no library sort/scan, no host round trip.
//
// The reference pipeline (SURVEY.md section 2.3: InclusiveSum -> duplicateWithKeys -> 64-bit SortPairs ->
// identifyTileRanges, driven from gaussian_renderer/__init__.py:126-135) sorts ALL R
// (tile | depth) keys globally and needs R on the host to size its buffers.  Here the order is produced
// tile-locally instead:
//
//   k_preprocess   (gs_raster.cu) counts instances per tile with RED.ADD while it projects     -> tcount[T]
//   k_tile_scan    one CTA: exclusive scan of the T (<= 65535) tile counts                      -> tstart[T], R
//   k_scatter      one thread per Gaussian (any order): (depth bits << 32 | id) appended to its tiles' segments
//                  through per-tile atomic cursors
//   k_tile_sort    one CTA per tile: the segment is sorted by the unique 64-bit key in SHARED MEMORY
//                  (one adaptive-range bucket pass + per-bucket insertion sort; flip-bitonic fallback for
//                  skewed depth distributions) and written out as the tile's id list.  No per-instance copy of the
//                  splat records is materialised: the blend kernels stage id chunks with TMA bulk copies and gather
//                  the 48-byte records with cp.async out of the record table, only as far as they walk
//
// Result order = (tile, depth bits ascending, Gaussian index ascending): exactly the reference's stable radix
// sort of keys emitted in index order (Appendix A.2.9) -- deterministic although emission uses atomics.
// Every kernel reads R / offsets from device memory; the host only supplies a capacity.  If the true R
// exceeds it, lists are truncated memory-safely and status[kStOverflow] is raised for the caller to see.
#include "gs_internal.cuh"
#include "gs_tiles.cuh"

using namespace gsb;

namespace {

constexpr float kLog2e = 1.4426950408889634f;

// ------------------------------------------------------------------------------------------
// k_tile_scan
// ------------------------------------------------------------------------------------------
constexpr int kScanT = 1024;
__global__ void __launch_bounds__(kScanT) k_tile_scan(GeomView gv, int ntiles) {
  __shared__ unsigned long long s_warp[32];
  __shared__ uint32_t s_max[32];
  __shared__ uint32_t s_nq[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < 2) s_nq[tid] = 0u;
  const int per = (ntiles + kScanT - 1) / kScanT;
  const int lo = tid * per, hi = min(ntiles, lo + per);
  unsigned long long sum = 0;
  uint32_t mx = 0;
  // eight independent loads in flight per trip (the kernel is one CTA on the critical path: latency is everything)
  for (int t0 = lo; t0 < hi; t0 += 8) {
    uint32_t c[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) c[u] = t0 + u < hi ? gv.tcount[t0 + u] : 0u;
#pragma unroll
    for (int u = 0; u < 8; ++u) { sum += c[u]; mx = max(mx, c[u]); }
  }
  unsigned long long inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if (lane == 31) s_warp[warp] = inc;
  if (lane == 0) s_max[warp] = mx;
  __syncthreads();
  if (warp == 0) {
    unsigned long long w = s_warp[lane];
    uint32_t m = s_max[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long v = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += v;
      m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    }
    s_warp[lane] = w;
    if (lane == 0) s_max[0] = m;
  }
  __syncthreads();
  unsigned long long run = (inc - sum) + (warp ? s_warp[warp - 1] : 0ull);
  for (int t0 = lo; t0 < hi; t0 += 8) {
    uint32_t cc[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) cc[u] = t0 + u < hi ? gv.tcount[t0 + u] : 0u;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int t = t0 + u;
      if (t < hi) {
        const uint32_t c = cc[u];
        gv.tstart[t] = (uint32_t)min(run, 0xFFFFFFF0ull);     // saturating: such a tile is beyond any capacity
        run += c;
        if (c > kLargeList) gv.q_huge[atomicAdd(&s_nq[1], 1u)] = (uint32_t)t;        // rare: long lists are queued for
        else if (c > kSmallList) gv.q_large[atomicAdd(&s_nq[0], 1u)] = (uint32_t)t;  // the persistent sort kernels
      }
    }
  }
  __syncthreads();
  if (tid == kScanT - 1) {
    gv.status[kStR] = (uint32_t)min(s_warp[31], 0xFFFFFFF0ull);
    gv.status[kStOverflow] = 0u;
    gv.status[kStMaxList] = s_max[0];
    gv.status[kStHugeTiles] = 0u;
    gv.status[kStNLarge] = s_nq[0];
    gv.status[kStNHuge] = s_nq[1];
    // forward serial number: lets a host that replays this launch from a CUDA graph recognise, in the status words it
    // receives in pinned memory, which forward they belong to (word 7 is the device-resident counter)
    const uint32_t seq = gv.status[7] + 1u;
    gv.status[7] = seq;
    gv.status[kStSeq] = seq;
  }
}

// ------------------------------------------------------------------------------------------
// k_scatter: one thread per Gaussian
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_scatter(int P, GeomView gv, BinView bv, int W, int H, int gx, int exact_cull, uint32_t cap) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n = i < P ? gv.tiles[i] : 0u;
  SplatRect p;
  p.x = p.y = p.A = p.B = p.C = 0.f; p.qthr = -1.f;
  p.rx0 = p.rx1 = p.ry0 = p.ry1 = 0;
  unsigned long long key = 0ull;
  bool coop = false;
  TileSink sink{gv.tcount, gv.tstart, gv.tcursor, bv.pairs, cap};
  uint32_t mask = 0u;
  if (n) {
    const float4 r3 = gv.brec[i];                            // depth, rect x, rect y, keep mask
    const uint32_t rcx = __float_as_uint(r3.y), rcy = __float_as_uint(r3.z);
    p.rx0 = rcx & 0xFFFF; p.rx1 = rcx >> 16; p.ry0 = rcy & 0xFFFF; p.ry1 = rcy >> 16;
    key = ((unsigned long long)__float_as_uint(r3.x) << 32) | (unsigned long long)(uint32_t)i;
    const int area = (p.rx1 - p.rx0) * (p.ry1 - p.ry0);
    coop = area > kCoopTiles && area <= kBigRect;            // larger rects are emitted by k_big_rects
    if (area > kBigRect) {
      // nothing to do here
    } else if (coop) {                                              // re-walk the rect from the stored record (log2 domain)
      const float4 e0 = gv.rec[3 * (size_t)i], e1 = gv.rec[3 * (size_t)i + 1];
      p.x = e0.x; p.y = e0.y; p.A = -e0.z; p.B = -0.5f * e0.w; p.C = -e1.x; p.qthr = e1.z;
    } else {
      mask = __float_as_uint(r3.w);                          // exactly the tiles k_preprocess counted
    }
  }
  warp_sink_masks(mask, p.rx0, p.ry0, p.rx1 - p.rx0, gx, sink, key);
  visit_tiles_coop(coop, p, W, H, gx, exact_cull != 0, sink, key);
}


// ------------------------------------------------------------------------------------------
// k_big_rects: Gaussians whose tile rect exceeds kBigRect tiles, flattened into (Gaussian, trip) work items
// ------------------------------------------------------------------------------------------
// k_preprocess only queues such Gaussians (gv.q_big, length gv.aux[0]).  A warp walking one of them alone is a serial
// chain of trips -- a Gaussian that has grown over a 1080p frame is 8160 tiles = 64 trips, each an atomic round trip
// in emit mode -- and was the tail of both k_preprocess and k_scatter once training had inflated a few splats.  Here
// every CTA computes the exclusive prefix of the trip counts of the queue (redundantly, in shared memory; the queue is
// short) and the grid's warps take work items w = gw, gw + GW, ...: item -> (entry, trip) by binary search in the
// prefix.  EMIT = false: count per tile (RED) and per Gaussian (gv.tiles);  EMIT = true: reserve + write the keys.
// Both passes evaluate the tile test on the STORED record, so they see bit-identical inputs.
constexpr int kBigT = 256;
constexpr int kBigBatch = 4096;                 // queue entries per prefix batch
constexpr int kBigPer = kBigBatch / kBigT;      // entries per thread
template <bool EMIT>
__global__ void __launch_bounds__(kBigT)
k_big_rects(int P, GeomView gv, unsigned long long* pairs, int W, int H, int gx, int exact_cull, uint32_t cap) {
  __shared__ uint32_t s_pref[kBigBatch + 1];
  __shared__ uint32_t s_warp[kBigT / 32];
  const uint32_t n_all = min(gv.aux[0], (uint32_t)P);
  if (n_all == 0u) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t gw = blockIdx.x * (kBigT / 32) + warp, GW = gridDim.x * (kBigT / 32);
  const TileSink sink{gv.tcount, gv.tstart, gv.tcursor, EMIT ? pairs : nullptr, cap};
  const bool cull = exact_cull != 0;
  for (uint32_t b0 = 0; b0 < n_all; b0 += kBigBatch) {
    const uint32_t nb = min((uint32_t)kBigBatch, n_all - b0);
    uint32_t cnt[kBigPer], sum = 0u;
#pragma unroll
    for (int u = 0; u < kBigPer; ++u) {
      const uint32_t e = (uint32_t)tid * kBigPer + u;
      uint32_t c = 0u;
      if (e < nb) {
        const float4 r3 = gv.brec[gv.q_big[b0 + e]];
        const uint32_t rcx = __float_as_uint(r3.y), rcy = __float_as_uint(r3.z);
        const uint32_t area = ((rcx >> 16) - (rcx & 0xFFFF)) * ((rcy >> 16) - (rcy & 0xFFFF));
        c = (area + kTripTiles - 1) / kTripTiles;
      }
      cnt[u] = c;
      sum += c;
    }
    uint32_t inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    uint32_t base = inc - sum;
    for (int k = 0; k < warp; ++k) base += s_warp[k];
    uint32_t total = 0u;
    for (int k = 0; k < kBigT / 32; ++k) total += s_warp[k];
#pragma unroll
    for (int u = 0; u < kBigPer; ++u) {
      const uint32_t e = (uint32_t)tid * kBigPer + u;
      if (e < nb) s_pref[e] = base;
      base += cnt[u];
    }
    if (tid == 0) s_pref[nb] = total;
    __syncthreads();
    for (uint32_t w = gw; w < total; w += GW) {
      uint32_t lo = 0u, hi = nb;                         // largest e with s_pref[e] <= w (trip counts are >= 1)
      while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        if (s_pref[mid] <= w) lo = mid; else hi = mid;
      }
      const uint32_t trip = w - s_pref[lo];
      const uint32_t id = gv.q_big[b0 + lo];
      const float4 r3 = gv.brec[id], e0 = gv.rec[3 * (size_t)id], e1 = gv.rec[3 * (size_t)id + 1];
      const uint32_t rcx = __float_as_uint(r3.y), rcy = __float_as_uint(r3.z);
      SplatRect b;
      b.rx0 = rcx & 0xFFFF; b.rx1 = rcx >> 16; b.ry0 = rcy & 0xFFFF; b.ry1 = rcy >> 16;
      b.x = e0.x; b.y = e0.y; b.A = -e0.z; b.B = -0.5f * e0.w; b.C = -e1.x; b.qthr = e1.z;
      const unsigned long long key = ((unsigned long long)__float_as_uint(r3.x) << 32) | (unsigned long long)id;
      const int wd = b.rx1 - b.rx0, n = wd * (b.ry1 - b.ry0);
      const uint32_t kept = visit_trip(b, (int)(trip * kTripTiles), n, wd, W, H, gx, cull, sink, key);
      if (!EMIT && lane == 0 && kept) atomicAdd(gv.tiles + id, kept);
    }
    __syncthreads();                                     // s_pref is rebuilt for the next batch
  }
}

// ------------------------------------------------------------------------------------------
// k_tile_sort
// ------------------------------------------------------------------------------------------
// Compare-exchange network that sorts a[0..n) ascending for ANY n: the "flip" formulation of bitonic sort
// (first step of every merge pairs i with its mirror image, all exchanges ascending), so indices >= n act as
// +infinity and are simply skipped.  `a` may be shared or global memory (one CTA owns it).
template <int NT>
__device__ __forceinline__ void cta_bitonic(unsigned long long* a, uint32_t n) {
  uint32_t N = 1;
  while (N < n) N <<= 1;
  for (uint32_t k = 2; k <= N; k <<= 1) {
    for (uint32_t t = threadIdx.x; t < N / 2; t += NT) {          // flip step
      const uint32_t half = k >> 1, blk = t / half, off = t - blk * half;
      const uint32_t i = blk * k + off, p = blk * k + (k - 1 - off);
      if (p < n) {
        const unsigned long long x = a[i], y = a[p];
        if (x > y) { a[i] = y; a[p] = x; }
      }
    }
    __syncthreads();
    for (uint32_t j = k >> 2; j > 0; j >>= 1) {
      for (uint32_t t = threadIdx.x; t < N / 2; t += NT) {
        const uint32_t i = 2 * j * (t / j) + (t % j), p = i + j;
        if (p < n) {
          const unsigned long long x = a[i], y = a[p];
          if (x > y) { a[i] = y; a[p] = x; }
        }
      }
      __syncthreads();
    }
  }
}

// Write the tile's sorted id list (the blend kernels gather the splat records themselves, and only for the part of
// the list they actually walk: early termination stops most tiles after a fraction of their entries).
__device__ __forceinline__ void write_ids(const BinView& bv, const unsigned long long* sorted, uint32_t start, uint32_t n,
                                          int nthreads) {
  for (uint32_t j = threadIdx.x; j < n; j += nthreads) bv.ids[(size_t)start + j] = (uint32_t)sorted[j];
}

constexpr uint32_t kSkew = 24;     // a bucket longer than this sends the tile to the bitonic fallback

// Sorts one tile's segment and writes its id list.  NT threads, KPT keys per thread (lists of up to NT*KPT entries);
// HUGE: any length, sorted in global memory.
//
// Shared-memory sort: one bucket pass over the tile's own depth range -- bucket(d) = floor((d - dmin) * CAP /
// (dmax - dmin + 1)), monotone in the depth bits, CAP buckets for <= CAP keys -- then each thread finishes its KPT
// consecutive buckets with an insertion sort on the full 64-bit (depth, id) key.  Keys are re-read from global
// memory (L1/L2 hits) in the three passes instead of being held in registers: occupancy matters more here than
// load instructions, the kernel is barrier/latency bound.
template <int NT, int KPT, bool HUGE>
__device__ __forceinline__ void tile_sort_one(const GeomView& gv, const BinView& bv, uint32_t cap, uint32_t tile,
                                              unsigned char* smraw) {
  constexpr int CAP = NT * KPT;
  constexpr int NW = NT / 32;
  unsigned long long* sorted = reinterpret_cast<unsigned long long*>(smraw);   // [CAP]
  uint32_t* hist = reinterpret_cast<uint32_t*>(smraw + (size_t)CAP * 8);       // [CAP] buckets
  __shared__ uint32_t s_w[32];
  __shared__ uint32_t s_dmin, s_dmax;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t start = gv.tstart[tile], cnt = gv.tcount[tile], cur = gv.tcursor[tile];
  const uint32_t avail = start < cap ? cap - start : 0u;
  const uint32_t n = min(min(cnt, cur), avail);
  if (tid == 0) {
    const uint32_t s = min(start, cap);
    bv.ranges[tile] = make_uint2(s, s + n);
    if (cnt > avail) atomicOr(gv.status + kStOverflow, 1u);
    if (HUGE) atomicAdd(gv.status + kStHugeTiles, 1u);
    s_dmin = 0xFFFFFFFFu; s_dmax = 0u;
  }
  if (n == 0) return;
  const unsigned long long* seg = bv.pairs + start;
  if (HUGE) {
    cta_bitonic<NT>(const_cast<unsigned long long*>(seg), n);
    write_ids(bv, seg, start, n, NT);
    return;
  }
  __syncthreads();
  // ---- pass 1: depth range (and clear the buckets)
  uint32_t dmin = 0xFFFFFFFFu, dmax = 0u;
#pragma unroll
  for (int j = 0; j < KPT; ++j) {
    const uint32_t idx = (uint32_t)(j * NT + tid);
    if (idx < n) { const uint32_t d = (uint32_t)(__ldg(seg + idx) >> 32); dmin = min(dmin, d); dmax = max(dmax, d); }
    hist[idx] = 0u;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    dmin = min(dmin, __shfl_xor_sync(0xffffffffu, dmin, o));
    dmax = max(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
  }
  if (lane == 0) { atomicMin(&s_dmin, dmin); atomicMax(&s_dmax, dmax); }
  __syncthreads();
  dmin = s_dmin;
  // float arithmetic is monotone (conversion, multiplication by a positive constant and truncation all are), which
  // is all the bucket function has to be; the clamp covers rounding at the top end
  const float scale = (float)CAP / ((float)(s_dmax - dmin) + 1.0f);
  // ---- pass 2: histogram
#pragma unroll
  for (int j = 0; j < KPT; ++j) {
    const uint32_t idx = (uint32_t)(j * NT + tid);
    if (idx < n) {
      const uint32_t d = (uint32_t)(__ldg(seg + idx) >> 32);
      atomicAdd(hist + min((uint32_t)(CAP - 1), (uint32_t)((float)(d - dmin) * scale)), 1u);
    }
  }
  __syncthreads();
  // ---- exclusive scan of the CAP bucket counts (thread t owns buckets [t*KPT, (t+1)*KPT))
  uint32_t c[KPT], sum = 0u, big = 0u;
#pragma unroll
  for (int j = 0; j < KPT; ++j) { c[j] = hist[tid * KPT + j]; sum += c[j]; big = max(big, c[j]); }
  uint32_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) s_w[warp] = inc;
  const bool skew = __syncthreads_or(big > kSkew) != 0;
  uint32_t run = inc - sum;
#pragma unroll
  for (int w = 0; w < NW; ++w) run += (w < warp) ? s_w[w] : 0u;
  const uint32_t my_begin = run;
#pragma unroll
  for (int j = 0; j < KPT; ++j) { hist[tid * KPT + j] = run; run += c[j]; }
  __syncthreads();
  // ---- pass 3: scatter into buckets (order inside a bucket is arbitrary here)
#pragma unroll
  for (int j = 0; j < KPT; ++j) {
    const uint32_t idx = (uint32_t)(j * NT + tid);
    if (idx < n) {
      const unsigned long long k = __ldg(seg + idx);
      const uint32_t d = (uint32_t)(k >> 32);
      sorted[atomicAdd(hist + min((uint32_t)(CAP - 1), (uint32_t)((float)(d - dmin) * scale)), 1u)] = k;
    }
  }
  __syncthreads();
  if (skew) {
    cta_bitonic<NT>(sorted, n);
  } else {
    // ---- each thread finishes its own KPT consecutive buckets with an insertion sort on the full 64-bit key
    uint32_t b0 = my_begin;
#pragma unroll
    for (int j = 0; j < KPT; ++j) {
      const uint32_t b1 = b0 + c[j];
      for (uint32_t a = b0 + 1; a < b1; ++a) {
        const unsigned long long v = sorted[a];
        uint32_t q = a;
        while (q > b0 && sorted[q - 1] > v) { sorted[q] = sorted[q - 1]; --q; }
        sorted[q] = v;
      }
      b0 = b1;
    }
    __syncthreads();
  }
  write_ids(bv, sorted, start, n, NT);
}

// ---- kernels ------------------------------------------------------------------------------------------------
constexpr int kSmallNT = 256, kSmallKPT = 8;     // lists of up to 2048 entries: 24 KB shared memory
constexpr int kLargeNT = 512, kLargeKPT = 16;    // up to 8192 entries: 96 KB shared memory
static_assert(kSmallNT * kSmallKPT == (int)kSmallList && kLargeNT * kLargeKPT == (int)kLargeList, "size classes");
constexpr size_t kSmallSmem = (size_t)kSmallList * 12, kLargeSmem = (size_t)kLargeList * 12;

// one CTA per tile; tiles with longer lists were queued by k_tile_scan and are skipped here
__global__ void __launch_bounds__(kSmallNT, 5) k_tile_sort(GeomView gv, BinView bv, uint32_t cap) {
  extern __shared__ __align__(16) unsigned char smraw[];
  if (gv.tcount[blockIdx.x] > kSmallList) return;
  tile_sort_one<kSmallNT, kSmallKPT, false>(gv, bv, cap, blockIdx.x, smraw);
}

// persistent: CTA b takes queue entries b, b + grid, ...  (normally the queues are empty and this is a no-op)
__global__ void __launch_bounds__(kLargeNT) k_tile_sort_long(GeomView gv, BinView bv, uint32_t cap) {
  extern __shared__ __align__(16) unsigned char smraw[];
  const uint32_t nl = gv.status[kStNLarge], nh = gv.status[kStNHuge];
  for (uint32_t q = blockIdx.x; q < nl; q += gridDim.x) {
    tile_sort_one<kLargeNT, kLargeKPT, false>(gv, bv, cap, gv.q_large[q], smraw);
    __syncthreads();
  }
  for (uint32_t q = blockIdx.x; q < nh; q += gridDim.x) {
    tile_sort_one<kLargeNT, 1, true>(gv, bv, cap, gv.q_huge[q], smraw);
    __syncthreads();
  }
}

}  // namespace

int gsb_launch_tile_scan(const GeomView& gv, int ntiles, cudaStream_t st) {
  ProfScope ps(GSB_K_SCAN, st);
  k_tile_scan<<<1, kScanT, 0, st>>>(gv, ntiles);
  return GSB_OK;
}

// pairs == nullptr: count mode (after k_preprocess, before the tile scan); else emit mode (beside k_scatter)
int gsb_launch_big_rects(int P, const GeomView& gv, unsigned long long* pairs, int W, int H, int exact_cull, uint32_t cap,
                         cudaStream_t st) {
  const int gx = (W + kBlock - 1) / kBlock;
  const int grid = 2 * gsb_sm_count();
  if (pairs) k_big_rects<true><<<grid, kBigT, 0, st>>>(P, gv, pairs, W, H, gx, exact_cull, cap);
  else k_big_rects<false><<<grid, kBigT, 0, st>>>(P, gv, nullptr, W, H, gx, exact_cull, cap);
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}

int gsb_launch_binning(int P, const GeomView& gv, const BinView& bv, int W, int H, int exact_cull, uint32_t cap,
                       cudaStream_t st) {
  static bool attr_set[64] = {};
  int dev = 0;
  GSB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    GSB_CUDA(cudaFuncSetAttribute(k_tile_sort_long, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLargeSmem));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const int gx = (W + kBlock - 1) / kBlock, gy = (H + kBlock - 1) / kBlock;
  // the emission cursors are reset HERE (not by the scan) so that the render phase can be repeated on the same
  // preprocess result, e.g. with a larger buffer after an overflow
  GSB_CUDA(cudaMemsetAsync(gv.tcursor, 0, (size_t)gx * gy * 4, st));
  if (P > 0) {
    ProfScope ps(GSB_K_DUPLICATE, st, 2);
    k_scatter<<<(P + kThreads - 1) / kThreads, kThreads, 0, st>>>(P, gv, bv, W, H, gx, exact_cull, cap);
    const int rc = gsb_launch_big_rects(P, gv, bv.pairs, W, H, exact_cull, cap, st);                // emit mode
    if (rc) return rc;
  }
  {
    ProfScope ps(GSB_K_SORT_TILE, st, 2);
    k_tile_sort<<<gx * gy, kSmallNT, kSmallSmem, st>>>(gv, bv, cap);
    // persistent CTAs draining the long-list queues, one per SM
    k_tile_sort_long<<<gsb_sm_count(), kLargeNT, kLargeSmem, st>>>(gv, bv, cap);
  }
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}
