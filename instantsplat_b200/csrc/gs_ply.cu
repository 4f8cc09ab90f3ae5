// point_cloud.ply vertex records packed and unpacked on the GPU (C ABI in include/gsb200.h), in its own translation
// unit so that the other kernels are compiled exactly as before.  DESIGN.md 4.23.
//
// A record is R <= GSB_PLY_MAX_FLOATS 32-bit words; the segments, in record order, fill it column by column.  Both
// kernels are a tiled transpose through shared memory: a CTA owns kTile consecutive records, whose bytes are one
// contiguous run of kTile * R words in the file buffer.
//
//   k_ply_pack    stages the CTA's rows of every segment into the tile in record order (coalesced reads of each
//                 segment's contiguous slice), then writes the run with 16-byte stores.  The run starts wherever
//                 p0 * R words from the buffer's base lands: the words before the first 16-byte boundary (the head)
//                 and after the last one (the tail) are stored one by one.
//   k_ply_unpack  the reverse: 16-byte loads of the run (scalar head and tail) into the tile, then coalesced writes of
//                 each segment's slice.
//
// Words are copied as uint32, never converted, so NaN payloads, -0 and denormals survive.  Record and byte offsets are
// 64-bit.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/gsb200.h"

void gsb_set_error(const char* s);
void gsb_count_launch(int n);

namespace {

constexpr int kThreads = 256;
constexpr int kTile = 128;                       // records per CTA: at most 128 * 64 * 4 = 32 KB of shared memory

struct Layout {
  void* data[GSB_PLY_MAX_SEGMENTS];
  int32_t width[GSB_PLY_MAX_SEGMENTS];
  int32_t inner[GSB_PLY_MAX_SEGMENTS];
  int32_t col[GSB_PLY_MAX_SEGMENTS];             // the segment's first column in the record
  int32_t n;                                     // segments
  int32_t R;                                     // words per record
};

int check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return GSB_OK;
  char buf[256];
  snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  gsb_set_error(buf);
  return GSB_ERR_CUDA;
}

// Record column of word c of a segment row read as [width / inner, inner], stored transposed.
__device__ __forceinline__ int column(const Layout& L, int s, int c) {
  const int inner = L.inner[s], r = c / inner, k = c - r * inner;
  return L.col[s] + k * (L.width[s] / inner) + r;
}

// The CTA's run of words in the file buffer: [base, base + words), split at its 16-byte boundaries.
struct Run {
  int head, body, words;                         // head words, body 16-byte vectors, all words
};

__device__ __forceinline__ Run split_run(const void* base, int words) {
  Run r;
  r.words = words;
  r.head = (int)(((16 - ((uintptr_t)base & 15)) & 15) >> 2);
  r.head = r.head < words ? r.head : words;
  r.body = (words - r.head) >> 2;
  return r;
}

__global__ void __launch_bounds__(kThreads) k_ply_pack(int64_t P, const __grid_constant__ Layout L,
                                                       uint32_t* __restrict__ out) {
  extern __shared__ uint32_t tile[];             // [kTile, R] in record order
  const int64_t p0 = (int64_t)blockIdx.x * kTile;
  const int n = (int)(P - p0 < kTile ? P - p0 : kTile);
  const int R = L.R;
  for (int s = 0; s < L.n; ++s) {
    const int w = L.width[s], m = n * w;
    const uint32_t* src = static_cast<const uint32_t*>(L.data[s]);
    if (src) {
      src += p0 * w;
      for (int i = threadIdx.x; i < m; i += kThreads) {
        const int t = i / w;
        tile[t * R + column(L, s, i - t * w)] = __ldg(src + i);
      }
    } else {
      for (int i = threadIdx.x; i < m; i += kThreads) {
        const int t = i / w;
        tile[t * R + column(L, s, i - t * w)] = 0u;
      }
    }
  }
  __syncthreads();
  uint32_t* dst = out + p0 * R;
  const Run run = split_run(dst, n * R);
  for (int i = threadIdx.x; i < run.head; i += kThreads) dst[i] = tile[i];
  uint4* d4 = reinterpret_cast<uint4*>(dst + run.head);
  for (int v = threadIdx.x; v < run.body; v += kThreads) {
    const uint32_t* q = tile + run.head + 4 * v;
    d4[v] = make_uint4(q[0], q[1], q[2], q[3]);
  }
  for (int i = run.head + 4 * run.body + threadIdx.x; i < run.words; i += kThreads) dst[i] = tile[i];
}

__global__ void __launch_bounds__(kThreads) k_ply_unpack(int64_t P, const uint32_t* __restrict__ in,
                                                         const __grid_constant__ Layout L) {
  extern __shared__ uint32_t tile[];
  const int64_t p0 = (int64_t)blockIdx.x * kTile;
  const int n = (int)(P - p0 < kTile ? P - p0 : kTile);
  const int R = L.R;
  const uint32_t* src = in + p0 * R;
  const Run run = split_run(src, n * R);
  for (int i = threadIdx.x; i < run.head; i += kThreads) tile[i] = src[i];
  const uint4* s4 = reinterpret_cast<const uint4*>(src + run.head);
  for (int v = threadIdx.x; v < run.body; v += kThreads) {
    const uint4 q = s4[v];
    uint32_t* t = tile + run.head + 4 * v;
    t[0] = q.x;
    t[1] = q.y;
    t[2] = q.z;
    t[3] = q.w;
  }
  for (int i = run.head + 4 * run.body + threadIdx.x; i < run.words; i += kThreads) tile[i] = src[i];
  __syncthreads();
  for (int s = 0; s < L.n; ++s) {
    uint32_t* dst = static_cast<uint32_t*>(L.data[s]);
    if (!dst) continue;
    const int w = L.width[s], m = n * w;
    dst += p0 * w;
    for (int i = threadIdx.x; i < m; i += kThreads) {
      const int t = i / w;
      dst[i] = tile[t * R + column(L, s, i - t * w)];
    }
  }
}

// Validates the arguments and fills the kernel's layout; GSB_OK or GSB_ERR_INVALID with the reason set.
int layout(const char* who, int64_t P, int32_t n_segments, const GsbPlySegment* segments, const void* buffer,
           Layout* L) {
  char buf[256];
  const char* why = nullptr;
  if (P < 0) why = "P < 0";
  else if (n_segments < 1 || n_segments > GSB_PLY_MAX_SEGMENTS || !segments) why = "bad segment table";
  else if (!buffer || ((uintptr_t)buffer & 3)) why = "the record buffer is NULL or not 4-byte aligned";
  if (!why) {
    L->n = n_segments;
    L->R = 0;
    for (int s = 0; s < n_segments && !why; ++s) {
      const GsbPlySegment& g = segments[s];
      if (g.width < 1 || g.inner < 1 || g.width % g.inner) why = "a segment's width is not a positive multiple of inner";
      else if ((uintptr_t)g.data & 3) why = "a segment's data is not 4-byte aligned";
      else if (L->R + g.width > GSB_PLY_MAX_FLOATS) why = "the record is wider than GSB_PLY_MAX_FLOATS words";
      if (why) break;
      L->data[s] = g.data;
      L->width[s] = g.width;
      L->inner[s] = g.inner;
      L->col[s] = L->R;
      L->R += g.width;
    }
  }
  // blocks index grid.x (< 2^31), and P * R * 4 bytes must fit an int64
  if (!why && (P + kTile - 1) / kTile > INT32_MAX) why = "P too large";
  if (why) {
    snprintf(buf, sizeof(buf), "%s: %s", who, why);
    gsb_set_error(buf);
    return GSB_ERR_INVALID;
  }
  return GSB_OK;
}

}  // namespace

extern "C" GSB_API int gsb_ply_pack(int64_t P, int32_t n_segments, const GsbPlySegment* segments, void* out,
                                    gsb_stream_t stream) {
  Layout L;
  int rc = layout("gsb_ply_pack", P, n_segments, segments, out, &L);
  if (rc != GSB_OK || P == 0) return rc;
  gsb_count_launch(1);
  const unsigned blocks = (unsigned)((P + kTile - 1) / kTile);
  k_ply_pack<<<blocks, kThreads, (size_t)kTile * L.R * 4, (cudaStream_t)stream>>>(P, L, static_cast<uint32_t*>(out));
  return check(cudaGetLastError(), "k_ply_pack");
}

extern "C" GSB_API int gsb_ply_unpack(int64_t P, const void* in, int32_t n_segments, const GsbPlySegment* segments,
                                      gsb_stream_t stream) {
  Layout L;
  int rc = layout("gsb_ply_unpack", P, n_segments, segments, in, &L);
  if (rc != GSB_OK || P == 0) return rc;
  gsb_count_launch(1);
  const unsigned blocks = (unsigned)((P + kTile - 1) / kTile);
  k_ply_unpack<<<blocks, kThreads, (size_t)kTile * L.R * 4, (cudaStream_t)stream>>>(
      P, static_cast<const uint32_t*>(in), L);
  return check(cudaGetLastError(), "k_ply_unpack");
}
