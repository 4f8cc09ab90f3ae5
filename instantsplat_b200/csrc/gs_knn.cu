// simple_knn._C.distCUDA2 replacement for sm_90a (SURVEY.md section 8 row f1): mean squared distance to the
// 3 nearest neighbours of every point, used ONCE at initialisation to set the Gaussians' log-scales
// (scene/gaussian_model.py:20,156-160).  The reference's module (gitlab.inria.fr/bkerbl/simple-knn
// @ 86710c2) is an empty submodule; its published behaviour is an exact 3-NN (Morton order + box pruning).
//
// Here: uniform grid hash (cell ids sorted with cub), then one thread per point searches growing cubes of cells
// and stops as soon as the 3rd-best distance is provably final (<= distance to the boundary of the searched
// cube), so the result is EXACT for any distribution; for surface-like clouds one ring (27 cells) suffices.
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <float.h>
#include <stdio.h>
#include <string.h>

#include "../../include/gsb200.h"

void gsb_set_error(const char* s);
void gsb_count_launch(int n);
int gsb_sm_count();

namespace {

struct Grid {
  float mn[3], cs[3], inv[3];
  int n;
};

__device__ __forceinline__ unsigned int f2ord(float f) {
  unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(unsigned int u) {
  u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}

// bbox[0..2] = min (ordered-uint encoding), bbox[3..5] = max
__global__ void k_bbox(int P, const float* __restrict__ pts, unsigned int* bbox) {
  __shared__ unsigned int smn[3], smx[3];
  if (threadIdx.x < 3) { smn[threadIdx.x] = 0xffffffffu; smx[threadIdx.x] = 0u; }
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      unsigned int o = f2ord(pts[3 * (size_t)i + a]);
      atomicMin(&smn[a], o);
      atomicMax(&smx[a], o);
    }
  }
  __syncthreads();
  if (threadIdx.x < 3) { atomicMin(&bbox[threadIdx.x], smn[threadIdx.x]); atomicMax(&bbox[3 + threadIdx.x], smx[threadIdx.x]); }
}

__global__ void k_make_grid(const unsigned int* bbox, int n, Grid* g) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  g->n = n;
  for (int a = 0; a < 3; ++a) {
    float lo = ord2f(bbox[a]), hi = ord2f(bbox[3 + a]);
    float ext = fmaxf(hi - lo, 1e-20f);
    g->mn[a] = lo;
    g->cs[a] = ext / n * 1.000001f;
    g->inv[a] = 1.0f / g->cs[a];
  }
}

__device__ __forceinline__ int cell_of(const Grid& g, float v, int a) {
  int c = (int)floorf((v - g.mn[a]) * g.inv[a]);
  return c < 0 ? 0 : (c >= g.n ? g.n - 1 : c);
}

__global__ void k_cell_ids(int P, const float* __restrict__ pts, const Grid* gp, unsigned int* cid, unsigned int* idx) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const Grid g = *gp;
  int cx = cell_of(g, pts[3 * (size_t)i], 0), cy = cell_of(g, pts[3 * (size_t)i + 1], 1), cz = cell_of(g, pts[3 * (size_t)i + 2], 2);
  cid[i] = (unsigned int)((cz * g.n + cy) * g.n + cx);
  idx[i] = (unsigned int)i;
}

__global__ void k_cell_ranges(int P, const unsigned int* __restrict__ cid_s, unsigned int* cstart, unsigned int* cend) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  unsigned int c = cid_s[j];
  if (j == 0 || cid_s[j - 1] != c) cstart[c] = j;
  if (j == P - 1 || cid_s[j + 1] != c) cend[c] = j + 1;
}

__global__ void k_gather_pts(int P, const float* __restrict__ pts, const unsigned int* __restrict__ idx_s, float4* sorted) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  unsigned int i = idx_s[j];
  sorted[j] = make_float4(pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2], __uint_as_float(i));
}

__global__ void __launch_bounds__(128)
k_knn3(int P, const float4* __restrict__ sorted, const Grid* gp, const unsigned int* __restrict__ cstart,
       const unsigned int* __restrict__ cend, float* __restrict__ out) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  const Grid g = *gp;
  const float4 me = sorted[j];
  const int c[3] = {cell_of(g, me.x, 0), cell_of(g, me.y, 1), cell_of(g, me.z, 2)};
  const float p[3] = {me.x, me.y, me.z};
  float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;
  for (int r = 1; r <= g.n; ++r) {
    b0 = b1 = b2 = FLT_MAX;
    int lo[3], hi[3];
    float bound = FLT_MAX;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      lo[a] = max(0, c[a] - r);
      hi[a] = min(g.n - 1, c[a] + r);
      // distance from the point to the faces of the searched cube (infinite where the grid itself ends)
      if (c[a] - r >= 0) bound = fminf(bound, p[a] - (g.mn[a] + lo[a] * g.cs[a]));
      if (c[a] + r <= g.n - 1) bound = fminf(bound, (g.mn[a] + (hi[a] + 1) * g.cs[a]) - p[a]);
    }
    for (int z = lo[2]; z <= hi[2]; ++z)
      for (int y = lo[1]; y <= hi[1]; ++y) {
        const unsigned int rowc = (unsigned int)((z * g.n + y) * g.n);
        for (int x = lo[0]; x <= hi[0]; ++x) {
          const unsigned int s = cstart[rowc + x], e = cend[rowc + x];
          for (unsigned int k = s; k < e; ++k) {
            if ((int)k == j) continue;
            const float4 q = sorted[k];
            const float dx = q.x - p[0], dy = q.y - p[1], dz = q.z - p[2];
            const float d = dx * dx + dy * dy + dz * dz;
            if (d < b2) {
              if (d < b1) {
                b2 = b1;
                if (d < b0) { b1 = b0; b0 = d; } else b1 = d;
              } else b2 = d;
            }
          }
        }
      }
    const bool whole = lo[0] == 0 && lo[1] == 0 && lo[2] == 0 && hi[0] == g.n - 1 && hi[1] == g.n - 1 && hi[2] == g.n - 1;
    if (whole) break;
    if (b2 < FLT_MAX && bound > 0.f && b2 <= bound * bound) break;
  }
  // fewer than 3 other points (P <= 3): the missing neighbours count as distance 0
  float sum = 0.f;
  if (b0 < FLT_MAX) sum += b0;
  if (b1 < FLT_MAX) sum += b1;
  if (b2 < FLT_MAX) sum += b2;
  out[__float_as_uint(me.w)] = sum / 3.0f;
}

int grid_dim(int P) {
  int n = (int)cbrt((double)P / 2.0);
  if (n < 1) n = 1;
  if (n > 512) n = 512;
  return n;
}

struct Scratch {
  unsigned int *bbox, *cid, *cid_s, *idx, *idx_s, *cstart, *cend;
  float4* sorted;
  Grid* grid;
  void* cub_tmp;
  size_t cub_bytes, total;
};

size_t al(size_t v) { return (v + 255) / 256 * 256; }

Scratch view(void* base, int P) {
  Scratch s;
  size_t off = 0;
  char* p = (char*)base;
  size_t Pp = P > 0 ? P : 1;
  int n = grid_dim(P);
  size_t cells = (size_t)n * n * n;
  auto take = [&](size_t b) { void* r = p ? p + off : nullptr; off += al(b); return r; };
  s.bbox = (unsigned int*)take(6 * 4);
  s.grid = (Grid*)take(sizeof(Grid));
  s.cid = (unsigned int*)take(Pp * 4);
  s.cid_s = (unsigned int*)take(Pp * 4);
  s.idx = (unsigned int*)take(Pp * 4);
  s.idx_s = (unsigned int*)take(Pp * 4);
  s.cstart = (unsigned int*)take(cells * 4);
  s.cend = (unsigned int*)take(cells * 4);
  s.sorted = (float4*)take(Pp * 16);
  size_t tb = 0;
  unsigned int* k = nullptr;
  cub::DeviceRadixSort::SortPairs(nullptr, tb, k, k, k, k, (int)Pp, 0, 32);
  s.cub_bytes = tb + 256;
  s.cub_tmp = take(s.cub_bytes);
  s.total = off;
  return s;
}

}  // namespace

extern "C" GSB_API size_t gsb_knn_scratch_bytes(int32_t P) { return view(nullptr, P).total; }

extern "C" GSB_API int gsb_knn_mean_dist2(int32_t P, const float* points, float* out, void* scratch, size_t scratch_bytes,
                                          gsb_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  if (P < 0 || (P > 0 && (!points || !out || !scratch))) { gsb_set_error("gsb_knn_mean_dist2: bad argument"); return GSB_ERR_INVALID; }
  if (P == 0) return GSB_OK;
  Scratch s = view(scratch, P);
  if (s.total > scratch_bytes) { gsb_set_error("gsb_knn_mean_dist2: scratch too small"); return GSB_ERR_CAPACITY; }
  const int n = grid_dim(P);
  const size_t cells = (size_t)n * n * n;
  const unsigned int init[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
  cudaError_t e = cudaMemcpyAsync(s.bbox, init, sizeof(init), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(s.cstart, 0, cells * 4, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(s.cend, 0, cells * 4, st);
  if (e == cudaSuccess) {
    const int nb = (P + 255) / 256;
    gsb_count_launch(6);
    const int max_blocks = 8 * gsb_sm_count();
    k_bbox<<<nb < max_blocks ? nb : max_blocks, 256, 0, st>>>(P, points, s.bbox);
    k_make_grid<<<1, 32, 0, st>>>(s.bbox, n, s.grid);
    k_cell_ids<<<nb, 256, 0, st>>>(P, points, s.grid, s.cid, s.idx);
    int bits = 1;
    while (((size_t)1 << bits) < cells) ++bits;
    size_t tb = s.cub_bytes;
    e = cub::DeviceRadixSort::SortPairs(s.cub_tmp, tb, s.cid, s.cid_s, s.idx, s.idx_s, P, 0, bits, st);
    if (e == cudaSuccess) {
      k_cell_ranges<<<nb, 256, 0, st>>>(P, s.cid_s, s.cstart, s.cend);
      k_gather_pts<<<nb, 256, 0, st>>>(P, points, s.idx_s, s.sorted);
      k_knn3<<<(P + 127) / 128, 128, 0, st>>>(P, s.sorted, s.grid, s.cstart, s.cend, out);
      e = cudaGetLastError();
    }
  }
  if (e != cudaSuccess) {
    char buf[256];
    snprintf(buf, sizeof(buf), "gsb_knn_mean_dist2: %s", cudaGetErrorString(e));
    gsb_set_error(buf);
    return GSB_ERR_CUDA;
  }
  return GSB_OK;
}
