// Baseline JPEG decoding on the GPU (C ABI in include/gsb200.h), in its own translation unit so that the other
// kernels are compiled exactly as before.  DESIGN.md 4.24.  The per-symbol and per-block arithmetic is gs_jpeg.cuh.
//
//   k_flags / scan / k_unstuff   each entropy byte is flagged kept (not the 00 after an FF, not an RSTn) and RSTn;
//                                one exclusive scan of both counts places the kept bytes and gives every restart
//                                interval its first bit.  k_intervals checks the RSTn count and sequence.
//   scan                         every interval is cut into subseq_bits-bit subsequences.
//   k_sync                       self-synchronising decode: a subsequence starts from its predecessor's end state
//                                (or a guess: its first bit, block 0, DC next, also kept while the predecessor's
//                                decode fails) and decodes to its end; a CTA iterates
//                                through shared memory until its states agree, and the host repeats rounds, each
//                                CTA taking its predecessor's end from global memory, until no state changes.
//   scan                         the blocks each subsequence starts give its first block's index in the interval.
//   k_write                      re-decodes from the synchronised states, writing int16 coefficients and the DC
//                                differences (component-major, decode order), and checks each interval's last MCU.
//   scan by key                  the DC prefix per component and restart interval, in int64 so that int32 overflow
//                                is seen.
//   k_idct                       dequantise (outside int16: flagged) and islow IDCT into u8 component planes.
//   k_color                      upsample, convert to RGB and crop into each file's [H, W, 3] slot.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <cub/cub.cuh>
#include <vector>

#include "gs_jpeg.cuh"

void gsb_set_error(const char* s);
void gsb_count_launch(int n);

namespace {

using gsj::State;

constexpr int kThreads = 256;
constexpr int kSyncThreads = 128;                 // subsequences per CTA in k_sync

// What the kernels derive from a descriptor, built on the host.
struct Aux {
  int64_t data_offset, data_bytes;                // entropy bytes (stuffed) in data, and their unstuffed copy
  int64_t block_base;                             // first block of the file in the coefficient and DC arrays
  int64_t plane_base;                             // first byte of the file's component planes
  int64_t out_offset;
  int32_t interval_base;                          // first restart interval of the file (global index)
  int32_t n_intervals;
  int32_t mcus_x, mcus_y, bpm, ri;                // MCUs per row / column, blocks per MCU, MCUs per interval
  int32_t H, V, width, height;
  int32_t bw[3], bh[3];                           // component block grids (MCU-padded)
  int32_t cblock[3];                              // first block of each component, relative to block_base
  int64_t cplane[3];                              // first byte of each component plane, relative to plane_base
};

struct Plan {
  size_t off_files, off_aux, off_flags, off_bytes, off_ibits, off_irst, off_idone, off_iseq, off_start, off_end,
      off_count, off_coef, off_dcd, off_dc, off_key, off_planes, off_counter, off_temp, total;
  int64_t total_bytes, total_blocks, total_planes, nseq_max;
  int32_t total_intervals;
  size_t temp_bytes;
};

int fail(const char* who, const char* why) {
  char buf[256];
  snprintf(buf, sizeof(buf), "%s: %s", who, why);
  gsb_set_error(buf);
  return GSB_ERR_INVALID;
}

int check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return GSB_OK;
  char buf[256];
  snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  gsb_set_error(buf);
  return GSB_ERR_CUDA;
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// Validates the descriptors and derives the per-file layout; nullptr or the reason.
const char* derive(int32_t n, const GsbJpegFile* files, int32_t S, std::vector<Aux>& aux, Plan& P) {
  if (n < 0 || (n > 0 && !files)) return "bad file table";
  if (n > 65535) return "more than 65535 files in one call";      // k_color's grid.y
  if (S < 32 || S > (1 << 20) || (S & 7)) return "subseq_bits must be a multiple of 8 in 32..2^20";
  aux.resize(n);
  int64_t bytes = 0, blocks = 0, planes = 0, nseq = 0, intervals = 0;
  for (int i = 0; i < n; ++i) {
    const GsbJpegFile& f = files[i];
    Aux& a = aux[i];
    if (f.width < 1 || f.height < 1 || f.width > 65535 || f.height > 65535) return "a file's size is out of range";
    if (f.h < 1 || f.h > 2 || f.v < 1 || f.v > 2) return "a file's luma sampling is not 1 or 2";
    if (f.restart_interval < 0) return "a negative restart interval";
    if (f.data_offset != bytes || f.data_bytes < 0 || f.data_bytes >= (1 << 28))
      return "entropy segments must follow each other in data, each below 2^28 bytes";
    a.data_offset = f.data_offset;
    a.data_bytes = f.data_bytes;
    a.out_offset = f.out_offset;
    a.H = f.h;
    a.V = f.v;
    a.width = f.width;
    a.height = f.height;
    a.mcus_x = (f.width + 8 * f.h - 1) / (8 * f.h);
    a.mcus_y = (f.height + 8 * f.v - 1) / (8 * f.v);
    a.bpm = f.h * f.v + 2;
    const int64_t mcus = (int64_t)a.mcus_x * a.mcus_y;
    a.ri = f.restart_interval > 0 ? f.restart_interval : (int32_t)mcus;
    a.n_intervals = (int32_t)((mcus + a.ri - 1) / a.ri);
    a.interval_base = (int32_t)intervals;
    a.block_base = blocks;
    a.plane_base = planes;
    int64_t cb = 0, cp = 0;
    for (int c = 0; c < 3; ++c) {
      a.bw[c] = a.mcus_x * (c == 0 ? f.h : 1);
      a.bh[c] = a.mcus_y * (c == 0 ? f.v : 1);
      a.cblock[c] = (int32_t)cb;
      a.cplane[c] = cp;
      cb += (int64_t)a.bw[c] * a.bh[c];
      cp += (int64_t)a.bw[c] * a.bh[c] * 64;
    }
    bytes += f.data_bytes;
    blocks += cb;
    planes += cp;
    intervals += a.n_intervals;
    nseq += (f.data_bytes * 8 + S - 1) / S + a.n_intervals;
    if (intervals > (1 << 28) || blocks > ((int64_t)1 << 36)) return "batch too large";
  }
  P.total_bytes = bytes;
  P.total_blocks = blocks;
  P.total_planes = planes;
  P.total_intervals = (int32_t)intervals;
  P.nseq_max = nseq;
  if (nseq >= INT32_MAX / 2) return "batch too large";
  // cub's temporary storage: the largest of the four scans
  size_t t0 = 0, t1 = 0, t2 = 0, t3 = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, t0, (uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t)(bytes + 1));
  cub::DeviceScan::ExclusiveSum(nullptr, t1, (int32_t*)nullptr, (int32_t*)nullptr, (int)(intervals + 1));
  cub::DeviceScan::ExclusiveSum(nullptr, t2, (int32_t*)nullptr, (int32_t*)nullptr, (int)(nseq + 1));
  cub::DeviceScan::InclusiveSumByKey(nullptr, t3, (int32_t*)nullptr, (int64_t*)nullptr, (int64_t*)nullptr,
                                     (int64_t)(blocks > 0 ? blocks : 1));
  P.temp_bytes = t0 > t1 ? t0 : t1;
  P.temp_bytes = P.temp_bytes > t2 ? P.temp_bytes : t2;
  P.temp_bytes = P.temp_bytes > t3 ? P.temp_bytes : t3;
  size_t o = 0;
  auto take = [&o](size_t b) { const size_t at = o; o = align256(o + b); return at; };
  P.off_files = take(sizeof(GsbJpegFile) * (size_t)n);
  P.off_aux = take(sizeof(Aux) * (size_t)n);
  P.off_flags = take(8 * (size_t)(bytes + 1));
  P.off_bytes = take((size_t)bytes + 16);
  P.off_ibits = take(4 * (size_t)(intervals + n));
  P.off_irst = take(4 * (size_t)intervals);
  P.off_idone = take(4 * (size_t)intervals);
  P.off_iseq = take(4 * (size_t)(intervals + 1));
  P.off_start = take(8 * (size_t)nseq);
  P.off_end = take(8 * (size_t)nseq);
  P.off_count = take(4 * (size_t)(nseq + 1));
  P.off_coef = take(128 * (size_t)blocks);
  P.off_dcd = take(8 * (size_t)blocks);
  P.off_dc = take(8 * (size_t)blocks);
  P.off_key = take(4 * (size_t)blocks);
  P.off_planes = take((size_t)planes);
  P.off_counter = take(16);
  P.off_temp = take(P.temp_bytes);
  P.total = o;
  return nullptr;
}

// Largest i in [0, n) with base[i] <= x, for a nondecreasing base.
template <typename T, typename U>
__device__ __forceinline__ int upper_index(const T* base, int n, U x) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (base[mid] <= (T)x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// File of a global byte, interval or block, by binary search over the Aux array.
__device__ __forceinline__ int file_of_byte(const Aux* A, int n, int64_t j) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (A[mid].data_offset <= j) lo = mid; else hi = mid - 1;
  }
  return lo;
}
__device__ __forceinline__ int file_of_interval(const Aux* A, int n, int g) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (A[mid].interval_base <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}
__device__ __forceinline__ int file_of_block(const Aux* A, int n, int64_t b) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (A[mid].block_base <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

constexpr uint64_t kKeep = 1, kRst = 1ull << 40;  // the two counts of one scan

__global__ void k_flags(int n, const Aux* __restrict__ A, const uint8_t* __restrict__ d, int64_t total,
                        uint64_t* __restrict__ flags) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j <= total; j += (int64_t)gridDim.x * blockDim.x) {
    if (j == total) { flags[j] = 0; continue; }
    const Aux& a = A[file_of_byte(A, n, j)];
    const int64_t jl = j - a.data_offset;
    const uint32_t b = d[j], prev = jl > 0 ? d[j - 1] : 0u, next = jl + 1 < a.data_bytes ? d[j + 1] : 0u;
    const bool rst = prev == 0xFF && (b & 0xF8) == 0xD0;
    const bool stuffed = prev == 0xFF && b == 0x00;
    const bool marker = b == 0xFF && next != 0x00;       // the FF of an RSTn
    flags[j] = (rst ? kRst : 0) + ((rst || stuffed || marker) ? 0 : kKeep);
  }
}

// Scatters the kept bytes to their unstuffed place and records each RSTn's interval start (bit) and number.
__global__ void k_unstuff(int n, const Aux* __restrict__ A, const uint8_t* __restrict__ d, int64_t total,
                          const uint64_t* __restrict__ scan, uint8_t* __restrict__ out, uint32_t* __restrict__ ibits,
                          int32_t* __restrict__ irst) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < total; j += (int64_t)gridDim.x * blockDim.x) {
    const int f = file_of_byte(A, n, j);
    const Aux& a = A[f];
    const uint64_t here = scan[j], f0 = scan[a.data_offset], step = scan[j + 1] - here;
    const uint64_t kept = (here - f0) & (kRst - 1), rsts = (here - f0) >> 40;
    if (step & (kRst - 1)) out[a.data_offset + kept] = d[j];
    if (step >> 40) {
      const int64_t i = (int64_t)rsts + 1;                // the interval this RSTn starts
      if (i < a.n_intervals) {
        ibits[a.interval_base + f + i] = (uint32_t)(kept * 8);
        irst[a.interval_base + i] = d[j] & 7;
      }
    }
  }
}

// Per interval: its end bit, the RSTn count and number check, and how many subsequences it takes.
__global__ void k_intervals(int n, const Aux* __restrict__ A, int total_intervals, int S,
                            const uint64_t* __restrict__ scan, uint32_t* __restrict__ ibits,
                            const int32_t* __restrict__ irst, int32_t* __restrict__ iseq,
                            int32_t* __restrict__ status) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g == total_intervals) iseq[g] = 0;
  if (g >= total_intervals) return;
  const int f = file_of_interval(A, n, g);
  const Aux& a = A[f];
  const int i = g - a.interval_base;
  const uint64_t all = scan[a.data_offset + a.data_bytes] - scan[a.data_offset];
  const uint32_t all_bits = (uint32_t)((all & (kRst - 1)) * 8);
  if (i == 0) {
    ibits[a.interval_base + f + a.n_intervals] = all_bits;   // read by the kernels after this one
    if ((int64_t)(all >> 40) != a.n_intervals - 1) atomicOr(status + f, GSB_JPEG_RESTART);
  } else if (irst[g] != ((i - 1) & 7)) {
    atomicOr(status + f, GSB_JPEG_RESTART);
  }
  const uint32_t b0 = i == 0 ? 0u : ibits[a.interval_base + f + i];
  const uint32_t b1 = i + 1 == a.n_intervals ? all_bits : ibits[a.interval_base + f + i + 1];
  const int64_t len = b1 > b0 ? (int64_t)(b1 - b0) : 0;
  const int64_t m = (len + S - 1) / S;
  iseq[g] = (int32_t)(m > 0 ? m : 1);
}

// Where subsequence t decodes: its interval's bytes and bit range, its own range [lo, hi), and the file.
struct Seq {
  int f, g, i, local;
  uint32_t istart, iend, lo, hi;
};

__device__ __forceinline__ Seq locate(int n, const Aux* A, int total_intervals, const int32_t* iseq,
                                      const uint32_t* ibits, int S, int t) {
  Seq s;
  s.g = upper_index(iseq, total_intervals, t);
  s.f = file_of_interval(A, n, s.g);
  const Aux& a = A[s.f];
  s.i = s.g - a.interval_base;
  s.local = t - iseq[s.g];
  s.istart = ibits[a.interval_base + s.f + s.i];
  s.iend = ibits[a.interval_base + s.f + s.i + 1];
  if (s.iend < s.istart) s.iend = s.istart;
  s.lo = s.istart + (uint32_t)s.local * (uint32_t)S;
  s.hi = s.lo + (uint32_t)S < s.iend ? s.lo + (uint32_t)S : s.iend;
  return s;
}

__global__ void __launch_bounds__(kSyncThreads) k_sync(int n, const GsbJpegFile* __restrict__ files,
                                                        const Aux* __restrict__ A, int total_intervals, int S,
                                                        const int32_t* __restrict__ iseq,
                                                        const uint32_t* __restrict__ ibits,
                                                        const uint8_t* __restrict__ bytes, int round,
                                                        uint64_t* start, uint64_t* end, int32_t* __restrict__ count,
                                                        int32_t* __restrict__ changed_ctas) {
  __shared__ uint64_t s_end[kSyncThreads];
  const int tid = threadIdx.x;
  const int t = blockIdx.x * kSyncThreads + tid;
  const int nseq = iseq[total_intervals];
  const bool active = t < nseq;
  Seq q = {};
  uint64_t st = 0, en = 0;
  int32_t cnt = 0;
  const GsbJpegFile* F = nullptr;
  const uint8_t* p = nullptr;
  bool changed = false;
  // A subsequence starts where its predecessor ended; after a decode that failed (a wrong guess upstream, or a real
  // error, which the write pass flags) it keeps its own guess, so one bad guess does not stall the others.
  uint64_t guess = 0;
  auto wanted = [&](uint64_t pred) { return (pred & gsj::kInvalid) ? guess : pred; };
  if (active) {
    q = locate(n, A, total_intervals, iseq, ibits, S, t);
    F = files + q.f;
    p = bytes + A[q.f].data_offset;
    guess = gsj::pack(State{q.local == 0 ? q.istart : q.lo, 0, 0});
    if (round == 0) {
      st = guess;
      en = gsj::decode_span(st, q.hi, q.iend, p, *F, A[q.f].H, A[q.f].V, &cnt);
    } else {
      st = start[t];
      en = end[t];
      if (tid == 0 && q.local > 0) {
        const uint64_t want = wanted(*(volatile const uint64_t*)(end + t - 1));
        if (want != st) {
          st = want;
          changed = true;
          en = gsj::decode_span(st, q.hi, q.iend, p, *F, A[q.f].H, A[q.f].V, &cnt);
        }
      }
    }
  }
  bool any_change = round == 0 || __syncthreads_or(changed);
  bool wrote = changed;
  while (true) {
    s_end[tid] = en;
    __syncthreads();
    changed = false;
    if (active && tid > 0 && q.local > 0 && wanted(s_end[tid - 1]) != st) {
      st = wanted(s_end[tid - 1]);
      en = gsj::decode_span(st, q.hi, q.iend, p, *F, A[q.f].H, A[q.f].V, &cnt);
      changed = wrote = true;
    }
    if (!__syncthreads_or(changed)) break;
    any_change = true;
  }
  if (active && (round == 0 || wrote)) {
    start[t] = st;
    *(volatile uint64_t*)(end + t) = en;
    count[t] = cnt;
  }
  if (round > 0 && any_change && tid == 0) atomicAdd(changed_ctas, 1);
}

// Re-decodes each subsequence from its synchronised start, writing the coefficients, the DC differences and their
// segment keys, and checks the interval's last block.
__global__ void k_write(int n, const GsbJpegFile* __restrict__ files, const Aux* __restrict__ A, int total_intervals,
                        int S, const int32_t* __restrict__ iseq, const uint32_t* __restrict__ ibits,
                        const uint8_t* __restrict__ bytes, const uint64_t* __restrict__ start,
                        const int32_t* __restrict__ first_block, int16_t* __restrict__ coef,
                        int64_t* __restrict__ dcd, int32_t* __restrict__ key, int32_t* __restrict__ idone,
                        int32_t* __restrict__ status) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= iseq[total_intervals]) return;
  const Seq q = locate(n, A, total_intervals, iseq, ibits, S, t);
  const uint64_t st = start[t];
  if (st & gsj::kInvalid) return;                        // an error upstream, flagged there or by the interval check
  const Aux& a = A[q.f];
  const GsbJpegFile& F = files[q.f];
  const uint8_t* p = bytes + a.data_offset;
  const int hv = a.H * a.V;
  const int64_t mcus = (int64_t)a.mcus_x * a.mcus_y;
  const int64_t mcu0 = (int64_t)q.i * a.ri;
  const int64_t expected = ((mcus - mcu0 < a.ri) ? mcus - mcu0 : a.ri) * a.bpm;
  State s = gsj::unpack(st);
  // the block in progress: the one before the first block this subsequence starts
  int64_t blk = (int64_t)first_block[t] - first_block[iseq[q.g]] - 1;
  int dc, ci, cv, err = 0;
  while (s.pos < q.hi) {
    if (s.k == 0) {
      ++blk;
      if (blk >= expected) break;                        // past the interval's last MCU: padding
      if (s.c != (int)(blk % a.bpm)) { err = GSB_JPEG_UNSYNCED; break; }
    }
    if (blk < 0) { err = GSB_JPEG_UNSYNCED; break; }
    const int c = s.c, comp = c < hv ? 0 : c - hv + 1;
    const int j = comp == 0 ? c : 0, hc = comp == 0 ? a.H : 1, vc = comp == 0 ? a.V : 1;
    const int64_t mcu = mcu0 + blk / a.bpm;
    const int mx = (int)(mcu % a.mcus_x), my = (int)(mcu / a.mcus_x);
    const int64_t bx = (int64_t)mx * hc + j % hc, by = (int64_t)my * vc + j / hc;
    int16_t* bc = coef + (a.block_base + a.cblock[comp] + by * a.bw[comp] + bx) * 64;
    const bool was_dc = s.k == 0;
    const int r = gsj::step(s, &F.dc[comp], &F.ac[comp], p, q.iend >> 3, q.iend, &dc, &ci, &cv);
    if (r < 0) {
      err = r == gsj::kBadCode ? GSB_JPEG_BAD_CODE : (r == gsj::kPastEnd ? GSB_JPEG_PAST_END : GSB_JPEG_RUN_PAST_63);
      break;
    }
    if (was_dc) {
      const int64_t di = a.block_base + a.cblock[comp] + mcu * (hc * vc) + j;
      dcd[di] = dc;
      key[di] = q.g * 3 + comp;
    } else if (ci >= 0) {
      bc[ci] = (int16_t)cv;
    }
    if (r == gsj::kBlockEnd) {
      s.k = 0;
      s.c = s.c + 1 == a.bpm ? 0 : s.c + 1;
      if (blk == expected - 1) {
        idone[q.g] = 1;
        if (q.iend - s.pos >= 8) err = GSB_JPEG_TRAILING;
        break;
      }
    }
  }
  if (err) atomicOr(status + q.f, err);
}

__global__ void k_done(int n, const Aux* __restrict__ A, int total_intervals, const int32_t* __restrict__ idone,
                       int32_t* __restrict__ status) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total_intervals) return;
  if (!idone[g]) atomicOr(status + file_of_interval(A, n, g), GSB_JPEG_MCUS_LEFT);
}

// One thread per block: the DC sum, dequantisation and the islow IDCT into the component plane.
__global__ void k_idct(int n, const GsbJpegFile* __restrict__ files, const Aux* __restrict__ A, int64_t total_blocks,
                       const int16_t* __restrict__ coef, const int64_t* __restrict__ dc, uint8_t* __restrict__ planes,
                       int32_t* __restrict__ status) {
  for (int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; b < total_blocks;
       b += (int64_t)gridDim.x * blockDim.x) {
    const int f = file_of_block(A, n, b);
    const Aux& a = A[f];
    const int64_t rel = b - a.block_base;
    const int comp = rel >= a.cblock[2] ? 2 : (rel >= a.cblock[1] ? 1 : 0);
    const int64_t cb = rel - a.cblock[comp];
    const int bw = a.bw[comp];
    const int bx = (int)(cb % bw), by = (int)(cb / bw);
    const int hc = comp == 0 ? a.H : 1, vc = comp == 0 ? a.V : 1;
    const int64_t mcu = (int64_t)(by / vc) * a.mcus_x + bx / hc;
    const int64_t d = dc[a.block_base + a.cblock[comp] + mcu * (hc * vc) + (by % vc) * hc + bx % hc];
    const uint16_t* q = files[f].quant[comp];
    int32_t in[64];
    const int4* src = reinterpret_cast<const int4*>(coef + b * 64);
    bool bad = d < INT32_MIN || d > INT32_MAX;
#pragma unroll
    for (int v = 0; v < 8; ++v) {
      const int4 w = src[v];
      const int32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        in[v * 8 + h * 2] = (int16_t)(ws[h] & 0xffff);
        in[v * 8 + h * 2 + 1] = (int16_t)((uint32_t)ws[h] >> 16);
      }
    }
    in[0] = (int16_t)(int32_t)d;                          // (JCOEF) of the int32 DC prediction
#pragma unroll
    for (int k = 0; k < 64; ++k) {
      in[k] *= (int32_t)q[k];
      bad |= in[k] < -32768 || in[k] > 32767;
    }
    if (bad) atomicOr(status + f, GSB_JPEG_COEF_RANGE);
    const int ld = bw * 8;
    gsj::idct_islow(in, planes + a.plane_base + a.cplane[comp] + (int64_t)by * 8 * ld + bx * 8, ld);
  }
}

// Upsampling, colour conversion and the crop: one thread per output pixel, blockIdx.y the file.
__global__ void k_color(const Aux* __restrict__ A, const uint8_t* __restrict__ planes, uint8_t* __restrict__ out) {
  const Aux& a = A[blockIdx.y];
  const int64_t npx = (int64_t)a.width * a.height;
  const uint8_t* py = planes + a.plane_base;
  const uint8_t* pb = py + a.cplane[1];
  const uint8_t* pr = py + a.cplane[2];
  const int ldy = a.bw[0] * 8, ldc = a.bw[1] * 8;
  const int cw = (a.width + a.H - 1) / a.H, ch = (a.height + a.V - 1) / a.V;   // downsampled_width / height
  uint8_t* o = out + a.out_offset;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npx; i += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(i / a.width), x = (int)(i - (int64_t)y * a.width);
    const int Y = py[(int64_t)y * ldy + x];
    const int cb = gsj::chroma(pb, ldc, cw, ch, a.H, a.V, x, y);
    const int cr = gsj::chroma(pr, ldc, cw, ch, a.H, a.V, x, y);
    uint8_t rgb[3];
    gsj::ycc_to_rgb(Y, cb, cr, rgb);
    o[i * 3] = rgb[0];
    o[i * 3 + 1] = rgb[1];
    o[i * 3 + 2] = rgb[2];
  }
}

unsigned grid_for(int64_t items, int threads) {
  int64_t b = (items + threads - 1) / threads;
  if (b < 1) b = 1;
  return (unsigned)(b > (1 << 20) ? (1 << 20) : b);
}

}  // namespace

extern "C" GSB_API size_t gsb_jpeg_scratch_bytes(int32_t n, const GsbJpegFile* files, int32_t subseq_bits) {
  std::vector<Aux> aux;
  Plan P;
  if (derive(n, files, subseq_bits, aux, P)) return 0;
  return P.total;
}

extern "C" GSB_API int gsb_jpeg_decode_batch(int32_t n, const GsbJpegFile* files, const uint8_t* data,
                                             int32_t subseq_bits, void* scratch, size_t scratch_bytes, uint8_t* out,
                                             int32_t* status, gsb_stream_t stream) {
  const char* who = "gsb_jpeg_decode_batch";
  std::vector<Aux> aux;
  Plan P;
  if (const char* why = derive(n, files, subseq_bits, aux, P)) return fail(who, why);
  if (n == 0) return GSB_OK;
  if (!scratch || ((uintptr_t)scratch & 255)) return fail(who, "scratch is NULL or not 256-byte aligned");
  if (scratch_bytes < P.total) return fail(who, "scratch smaller than gsb_jpeg_scratch_bytes");
  if (!out || !status || (P.total_bytes > 0 && !data)) return fail(who, "NULL data, out or status");
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* base = static_cast<uint8_t*>(scratch);
  GsbJpegFile* d_files = reinterpret_cast<GsbJpegFile*>(base + P.off_files);
  Aux* d_aux = reinterpret_cast<Aux*>(base + P.off_aux);
  uint64_t* flags = reinterpret_cast<uint64_t*>(base + P.off_flags);
  uint8_t* bytes = base + P.off_bytes;
  uint32_t* ibits = reinterpret_cast<uint32_t*>(base + P.off_ibits);
  int32_t* irst = reinterpret_cast<int32_t*>(base + P.off_irst);
  int32_t* idone = reinterpret_cast<int32_t*>(base + P.off_idone);
  int32_t* iseq = reinterpret_cast<int32_t*>(base + P.off_iseq);
  uint64_t* start = reinterpret_cast<uint64_t*>(base + P.off_start);
  uint64_t* end = reinterpret_cast<uint64_t*>(base + P.off_end);
  int32_t* count = reinterpret_cast<int32_t*>(base + P.off_count);
  int16_t* coef = reinterpret_cast<int16_t*>(base + P.off_coef);
  int64_t* dcd = reinterpret_cast<int64_t*>(base + P.off_dcd);
  int64_t* dc = reinterpret_cast<int64_t*>(base + P.off_dc);
  int32_t* key = reinterpret_cast<int32_t*>(base + P.off_key);
  uint8_t* planes = base + P.off_planes;
  int32_t* counter = reinterpret_cast<int32_t*>(base + P.off_counter);
  void* temp = base + P.off_temp;
  size_t temp_bytes = P.temp_bytes;
  const int TI = P.total_intervals;
  const int S = subseq_bits;
  int rc;
#define GSJ_TRY(x, what) if ((rc = check((x), what)) != GSB_OK) return rc
  GSJ_TRY(cudaMemcpyAsync(d_files, files, sizeof(GsbJpegFile) * n, cudaMemcpyHostToDevice, s), "descriptors");
  GSJ_TRY(cudaMemcpyAsync(d_aux, aux.data(), sizeof(Aux) * n, cudaMemcpyHostToDevice, s), "layout");
  GSJ_TRY(cudaMemsetAsync(status, 0, 4 * (size_t)n, s), "status");
  GSJ_TRY(cudaMemsetAsync(ibits, 0, 4 * (size_t)(TI + n), s), "intervals");
  GSJ_TRY(cudaMemsetAsync(irst, 0xff, 4 * (size_t)TI, s), "intervals");
  GSJ_TRY(cudaMemsetAsync(idone, 0, 4 * (size_t)TI, s), "intervals");
  GSJ_TRY(cudaMemsetAsync(count, 0, 4 * (size_t)(P.nseq_max + 1), s), "counts");
  GSJ_TRY(cudaMemsetAsync(coef, 0, 128 * (size_t)P.total_blocks, s), "coefficients");
  GSJ_TRY(cudaMemsetAsync(dcd, 0, 8 * (size_t)P.total_blocks, s), "dc");
  GSJ_TRY(cudaMemsetAsync(key, 0xff, 4 * (size_t)P.total_blocks, s), "keys");
  GSJ_TRY(cudaMemsetAsync(bytes + P.total_bytes, 0, 16, s), "bytes");

  // 1. unstuff and segment
  gsb_count_launch(1);
  k_flags<<<grid_for(P.total_bytes + 1, kThreads), kThreads, 0, s>>>(n, d_aux, data, P.total_bytes, flags);
  GSJ_TRY(cudaGetLastError(), "k_flags");
  GSJ_TRY(cub::DeviceScan::ExclusiveSum(temp, temp_bytes, flags, flags, (int64_t)(P.total_bytes + 1), s), "scan");
  if (P.total_bytes > 0) {
    gsb_count_launch(1);
    k_unstuff<<<grid_for(P.total_bytes, kThreads), kThreads, 0, s>>>(n, d_aux, data, P.total_bytes, flags, bytes,
                                                                      ibits, irst);
    GSJ_TRY(cudaGetLastError(), "k_unstuff");
  }
  gsb_count_launch(1);
  k_intervals<<<grid_for(TI + 1, kThreads), kThreads, 0, s>>>(n, d_aux, TI, S, flags, ibits, irst, iseq, status);
  GSJ_TRY(cudaGetLastError(), "k_intervals");
  GSJ_TRY(cub::DeviceScan::ExclusiveSum(temp, temp_bytes, iseq, iseq, TI + 1, s), "scan");

  // 2. self-synchronising decode, in rounds until no state changes
  const unsigned sync_ctas = grid_for(P.nseq_max, kSyncThreads);
  bool synced = false;
  for (unsigned round = 0; round <= sync_ctas + 1; ++round) {
    GSJ_TRY(cudaMemsetAsync(counter, 0, 4, s), "counter");
    gsb_count_launch(1);
    k_sync<<<sync_ctas, kSyncThreads, 0, s>>>(n, d_files, d_aux, TI, S, iseq, ibits, bytes, (int)round, start, end,
                                              count, counter);
    GSJ_TRY(cudaGetLastError(), "k_sync");
    if (round == 0) continue;
    int32_t changed = 0;
    GSJ_TRY(cudaMemcpyAsync(&changed, counter, 4, cudaMemcpyDeviceToHost, s), "counter");
    GSJ_TRY(cudaStreamSynchronize(s), "k_sync");
    if (changed == 0) { synced = true; break; }
  }
  if (!synced) return fail(who, "the subsequences did not synchronise within the round bound");

  // 3. block offsets, coefficients and DC differences
  GSJ_TRY(cub::DeviceScan::ExclusiveSum(temp, temp_bytes, count, count, (int)(P.nseq_max + 1), s), "scan");
  gsb_count_launch(1);
  k_write<<<grid_for(P.nseq_max, kThreads), kThreads, 0, s>>>(n, d_files, d_aux, TI, S, iseq, ibits, bytes, start,
                                                              count, coef, dcd, key, idone, status);
  GSJ_TRY(cudaGetLastError(), "k_write");
  gsb_count_launch(1);
  k_done<<<grid_for(TI, kThreads), kThreads, 0, s>>>(n, d_aux, TI, idone, status);
  GSJ_TRY(cudaGetLastError(), "k_done");
  if (P.total_blocks > 0)
    GSJ_TRY(cub::DeviceScan::InclusiveSumByKey(temp, temp_bytes, key, dcd, dc, (int64_t)P.total_blocks,
                                               cub::Equality(), s), "scan by key");

  // 4. dequantise and IDCT; 5. upsample, convert and crop
  gsb_count_launch(1);
  k_idct<<<grid_for(P.total_blocks, kThreads), kThreads, 0, s>>>(n, d_files, d_aux, P.total_blocks, coef, dc, planes,
                                                                   status);
  GSJ_TRY(cudaGetLastError(), "k_idct");
  int64_t most = 1;
  for (const Aux& a : aux) most = (int64_t)a.width * a.height > most ? (int64_t)a.width * a.height : most;
  gsb_count_launch(1);
  k_color<<<dim3(grid_for(most, kThreads), n), kThreads, 0, s>>>(d_aux, planes, out);
  GSJ_TRY(cudaGetLastError(), "k_color");
#undef GSJ_TRY
  return GSB_OK;
}
