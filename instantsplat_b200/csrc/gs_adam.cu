// Fused per-point Adam for sm_90a: all parameter tensors of the Gaussian model (and the pose
// table) in ONE launch, no host synchronisation.
//
// Semantics are those of scene/per_point_adam.py:34-98:
//   * whole-tensor gate  mask = grad.norm() > 0  (:66-67): moments are updated only when the
//     gradient tensor is not identically zero; evaluated on the device by k_adam_gate
//   * old-style bias correction folded into step_size = lr*sqrt(1-b2^t)/(1-b1^t) (:76-81),
//     denom = sqrt(v) + eps (eps NOT divided by sqrt(bc2))
//   * optional per-row learning-rate multiplier per_point_lr [rows,1,..] (:84-95)
//   * the parameter is updated even when the gate is false (stale momentum)
// HBM traffic per element: read p,g,m,v + write p,m,v = 28 B (the roofline of this kernel).
#include <cuda_runtime.h>
#include <stdio.h>

#include "../../include/gsb200.h"

void gsb_set_error(const char* s);
void gsb_count_launch(int n);
int gsb_prof_begin(int id, cudaStream_t st);
void gsb_prof_end(int slot, cudaStream_t st);

namespace {

struct AdamT {
  float* p; const float* g; float* m; float* v; const float* ppl;
  long long numel; int row_len;
  float step, b1, omb1, b2, omb2, eps, wd, gscale;
  unsigned int first_block, nblocks;
};
struct AdamArgs { int n; const float* step_dev; AdamT t[GSB_ADAM_MAX_TENSORS]; };

constexpr int kAT = 256;
constexpr int kPerThread = 8;                     // 2 x float4
constexpr int kPerBlock = kAT * kPerThread;       // 2048 elements

__device__ __forceinline__ int find_tensor(const AdamArgs& a, unsigned int b) {
  int k = 0;
#pragma unroll
  for (int i = 1; i < GSB_ADAM_MAX_TENSORS; ++i)
    if (i < a.n && b >= a.t[i].first_block) k = i;
  return k;
}

// flags[k] = 1 when tensor k's (scaled, decayed) gradient has any element with g*g > 0.
// Grid = n_tensors x kGateSlots CTAs: CTA (k, j) scans chunks j, j+kGateSlots, ... of tensor k and re-reads
// the flag before every chunk after its first, so in the usual case (some gradient is non-zero) each CTA
// touches one chunk and the whole gate costs a few microseconds; an all-zero tensor is scanned completely.
constexpr int kGateSlots = 84;
__global__ void __launch_bounds__(kAT) k_adam_gate(AdamArgs a, unsigned int* flags) {
  const int k = blockIdx.x / kGateSlots;
  const unsigned int slot = blockIdx.x - k * kGateSlots;
  const AdamT& t = a.t[k];
  __shared__ unsigned int s_set;
  for (unsigned int vb = slot; vb < t.nblocks; vb += kGateSlots) {
    if (vb != slot) {
      __syncthreads();
      if (threadIdx.x == 0) s_set = *((volatile unsigned int*)(flags + k));
      __syncthreads();
      if (s_set) return;
    }
    const long long base = (long long)vb * kPerBlock;
    bool any = false;
#pragma unroll
    for (int u = 0; u < kPerThread; ++u) {
      const long long e = base + (long long)u * kAT + threadIdx.x;
      if (e < t.numel) {
        float g = t.g[e] * t.gscale;
        if (t.wd != 0.f) g += t.wd * t.p[e];
        any |= (g * g > 0.f);
      }
    }
    if (__syncthreads_or(any)) {
      if (threadIdx.x == 0) atomicOr(flags + k, 1u);
      return;
    }
  }
}

__device__ __forceinline__ void adam_elem(const AdamT& t, float step, bool gate, float lr_mul, float& p, float g,
                                          float& m, float& v) {
  g *= t.gscale;
  if (t.wd != 0.f) g = __fmaf_rn(t.wd, p, g);
  if (gate) {
    m = __fadd_rn(__fmul_rn(m, t.b1), __fmul_rn(g, t.omb1));
    v = __fadd_rn(__fmul_rn(v, t.b2), __fmul_rn(__fmul_rn(t.omb2, g), g));
  }
  float denom = __fadd_rn(__fsqrt_rn(v), t.eps);
  float upd = __fdiv_rn(m, denom);
  p = __fadd_rn(p, __fmul_rn(-(step * lr_mul), upd));
}

__global__ void __launch_bounds__(kAT) k_adam(AdamArgs a, const unsigned int* __restrict__ flags,
                                              const unsigned int* __restrict__ skip) {
  if (skip && *skip) return;     // e.g. the forward's overflow word: the caller redoes the step with larger buffers
  const int k = find_tensor(a, blockIdx.x);
  const AdamT& t = a.t[k];
  const bool gate = flags[k] != 0;
  // step size = lr * sqrt(1-b2^t)/(1-b1^t): a launch argument, or (CUDA-graph replay: arguments are frozen) read from
  // a device array the host refreshes before every replay
  const float step = a.step_dev ? a.step_dev[k] : t.step;
  const long long base = (long long)(blockIdx.x - t.first_block) * kPerBlock;
  const bool vec = ((((uintptr_t)t.p | (uintptr_t)t.g | (uintptr_t)t.m | (uintptr_t)t.v) & 15) == 0);
  if (vec && base + kPerBlock <= t.numel) {
#pragma unroll
    for (int u = 0; u < kPerThread / 4; ++u) {
      long long e = base + ((long long)u * kAT + threadIdx.x) * 4;
      float4 p = *reinterpret_cast<float4*>(t.p + e);
      float4 g = __ldg(reinterpret_cast<const float4*>(t.g + e));
      float4 m = *reinterpret_cast<float4*>(t.m + e);
      float4 v = *reinterpret_cast<float4*>(t.v + e);
      float l0 = 1.f, l1 = 1.f, l2 = 1.f, l3 = 1.f;
      if (t.ppl) {
        l0 = __ldg(t.ppl + e / t.row_len); l1 = __ldg(t.ppl + (e + 1) / t.row_len);
        l2 = __ldg(t.ppl + (e + 2) / t.row_len); l3 = __ldg(t.ppl + (e + 3) / t.row_len);
      }
      adam_elem(t, step, gate, l0, p.x, g.x, m.x, v.x);
      adam_elem(t, step, gate, l1, p.y, g.y, m.y, v.y);
      adam_elem(t, step, gate, l2, p.z, g.z, m.z, v.z);
      adam_elem(t, step, gate, l3, p.w, g.w, m.w, v.w);
      *reinterpret_cast<float4*>(t.p + e) = p;
      *reinterpret_cast<float4*>(t.m + e) = m;
      *reinterpret_cast<float4*>(t.v + e) = v;
    }
  } else {
    for (int u = 0; u < kPerThread; ++u) {
      long long e = base + (long long)u * kAT + threadIdx.x;
      if (e < t.numel) {
        float p = t.p[e], m = t.m[e], v = t.v[e];
        float l = t.ppl ? t.ppl[e / t.row_len] : 1.f;
        adam_elem(t, step, gate, l, p, t.g[e], m, v);
        t.p[e] = p; t.m[e] = m; t.v[e] = v;
      }
    }
  }
}

}  // namespace

static int build_args(int32_t n, const GsbAdamTensor* ts, AdamArgs& a, unsigned int& nb) {
  a.n = n;
  a.step_dev = nullptr;
  nb = 0;
  for (int i = 0; i < n; ++i) {
    const GsbAdamTensor& s = ts[i];
    if (!s.param || !s.grad || !s.exp_avg || !s.exp_avg_sq || s.numel < 0 || s.row_len <= 0) {
      gsb_set_error("gsb_adam: null tensor / bad shape");
      return GSB_ERR_INVALID;
    }
    AdamT& t = a.t[i];
    t.p = s.param; t.g = s.grad; t.m = s.exp_avg; t.v = s.exp_avg_sq; t.ppl = s.per_point_lr;
    t.numel = s.numel; t.row_len = s.row_len;
    t.step = (float)s.step_size;
    t.b1 = (float)s.beta1; t.omb1 = (float)(1.0 - s.beta1);
    t.b2 = (float)s.beta2; t.omb2 = (float)(1.0 - s.beta2);
    t.eps = (float)s.eps; t.wd = (float)s.weight_decay; t.gscale = s.grad_scale;
    t.first_block = nb;
    t.nblocks = (unsigned int)((s.numel + kPerBlock - 1) / kPerBlock);
    nb += t.nblocks;
  }
  for (int i = n; i < GSB_ADAM_MAX_TENSORS; ++i) { a.t[i] = a.t[0]; a.t[i].first_block = 0xffffffffu; a.t[i].nblocks = 0; }
  return GSB_OK;
}

static int finish(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return GSB_OK;
  char buf[256];
  snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  gsb_set_error(buf);
  return GSB_ERR_CUDA;
}

extern "C" GSB_API int gsb_adam_gate(int32_t n, const GsbAdamTensor* ts, uint32_t* flags, gsb_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  if (n < 0 || n > GSB_ADAM_MAX_TENSORS || (n > 0 && (!ts || !flags))) {
    gsb_set_error("gsb_adam_gate: bad argument");
    return GSB_ERR_INVALID;
  }
  if (n == 0) return GSB_OK;
  AdamArgs a;
  unsigned int nb;
  int rc = build_args(n, ts, a, nb);
  if (rc) return rc;
  cudaError_t e = cudaMemsetAsync(flags, 0, sizeof(uint32_t) * n, st);
  if (e == cudaSuccess && nb > 0) {
    gsb_count_launch(1);
    k_adam_gate<<<n * kGateSlots, kAT, 0, st>>>(a, flags);
    e = cudaGetLastError();
  }
  return finish(e, "gsb_adam_gate");
}

extern "C" GSB_API int gsb_adam_step_ex(int32_t n, const GsbAdamTensor* ts, uint32_t* flags,
                                        const uint32_t* skip_if_nonzero, const float* step_sizes_dev,
                                        gsb_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  if (n < 0 || n > GSB_ADAM_MAX_TENSORS || (n > 0 && (!ts || !flags))) {
    gsb_set_error("gsb_adam_step: bad argument");
    return GSB_ERR_INVALID;
  }
  if (n == 0) return GSB_OK;
  AdamArgs a;
  unsigned int nb;
  int rc = build_args(n, ts, a, nb);
  if (rc) return rc;
  a.step_dev = step_sizes_dev;
  cudaError_t e = cudaMemsetAsync(flags, 0, sizeof(uint32_t) * n, st);
  if (e == cudaSuccess && nb > 0) {
    gsb_count_launch(2);
    int slot = gsb_prof_begin(GSB_K_ADAM, st);
    k_adam_gate<<<n * kGateSlots, kAT, 0, st>>>(a, flags);
    k_adam<<<nb, kAT, 0, st>>>(a, flags, skip_if_nonzero);
    gsb_prof_end(slot, st);
    e = cudaGetLastError();
  }
  return finish(e, "gsb_adam_step");
}

extern "C" GSB_API int gsb_adam_step_gated(int32_t n, const GsbAdamTensor* ts, uint32_t* flags,
                                           const uint32_t* skip_if_nonzero, gsb_stream_t stream) {
  return gsb_adam_step_ex(n, ts, flags, skip_if_nonzero, nullptr, stream);
}

extern "C" GSB_API int gsb_adam_step(int32_t n, const GsbAdamTensor* ts, uint32_t* flags, gsb_stream_t stream) {
  return gsb_adam_step_ex(n, ts, flags, nullptr, nullptr, stream);
}
