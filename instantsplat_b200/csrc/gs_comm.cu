// Fused reduce-scatter -> per-point Adam -> all-gather over NVLink peer memory (sm_90a).
//
// Multi-GPU exchange of the view-sharded optimisation loop (SURVEY.md section 8e / 5.8): every rank
// holds a full replica of the flat parameter buffer and has just written its view's gradients into
// its flat gradient buffer.  Rank r owns the r-th contiguous shard of the flat index space.  ONE
// kernel per rank then, for each 128-bit group of its shard:
//     g   = sum over ranks of peer_grads[rank][i]          (P2P loads over NVLink, fixed order)
//     m,v = Adam moment update (local, shard-sized)         (scene/per_point_adam.py:66-73; gate: gsb_adam_gate)
//     p   = p - step * lr_i * m / (sqrt(v) + eps)           (:76-98)
//     peer_params[rank][i] = p   for every rank             (P2P stores over NVLink)
// i.e. the reduce-scatter, the optimizer and the all-gather of the "NCCL all-reduce + Adam"
// baseline in one pass: gradients cross the links once, parameters once, Adam touches 1/G of the
// elements per GPU, and the NCCL ring/tree launch latencies disappear.  The caller brackets it with
// two tiny NCCL collectives (flag/pose-gradient all-reduce before, a barrier after) that double as
// the cross-GPU barriers.
//
// Buffers that peers touch are allocated here with cudaMalloc and shared with CUDA IPC
// (cudaIpcGetMemHandle / cudaIpcOpenMemHandle) because each GPU is driven by its own process.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include "../../include/gsb200.h"

void gsb_set_error(const char* s);
void gsb_count_launch(int n);
int gsb_prof_begin(int id, cudaStream_t st);
void gsb_prof_end(int slot, cudaStream_t st);

namespace {

constexpr int kMaxWorld = 8;
constexpr int kMaxPieces = 12;

struct Piece {
  long long begin, end, seg_begin;   // flat-buffer element indices; begin/end multiples of 4
  const float* ppl;
  int row_len, flag_index;
  float step, b1, omb1, b2, omb2, eps;
  unsigned int first_block, nblocks;
};
struct FusedArgs {
  const float* step_dev;     // optional [GSB_ADAM_MAX_TENSORS]: step size per flag_index (CUDA-graph replay)
  int world, rank, n_pieces;
  long long shard_begin;
  float gscale;
  const float* grads[kMaxWorld];
  float* params[kMaxWorld];
  float* m;
  float* v;
  Piece pc[kMaxPieces];
};

constexpr int kFT = 256;
constexpr int kVecPerThread = 2;
constexpr int kElemsPerBlock = kFT * kVecPerThread * 4;   // 2048

__device__ __forceinline__ float4 ld_peer(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_peer(float* p, const float4& v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w) : "memory");
}

__device__ __forceinline__ void adam1(const Piece& t, float step, bool gate, float lr_mul, float& p, float g, float& m,
                                      float& v) {
  if (gate) {
    m = __fadd_rn(__fmul_rn(m, t.b1), __fmul_rn(g, t.omb1));
    v = __fadd_rn(__fmul_rn(v, t.b2), __fmul_rn(__fmul_rn(t.omb2, g), g));
  }
  float denom = __fadd_rn(__fsqrt_rn(v), t.eps);
  p = __fadd_rn(p, __fmul_rn(-(step * lr_mul), __fdiv_rn(m, denom)));
}

template <int WORLD>
__global__ void __launch_bounds__(kFT) k_fused_rs_adam_ag(FusedArgs a, const unsigned int* __restrict__ flags,
                                                          const unsigned int* __restrict__ skip) {
  if (skip && *skip) return;      // some rank's forward overflowed its binning buffer: nobody updates
  int k = 0;
#pragma unroll
  for (int i = 1; i < kMaxPieces; ++i)
    if (i < a.n_pieces && blockIdx.x >= a.pc[i].first_block) k = i;
  const Piece& t = a.pc[k];
  // the per-rank gate flags summed over the ranks: some rank saw a non-zero element and none saw a NaN (gsb200.h)
  const unsigned int flag = flags[t.flag_index];
  const bool gate = flag >= GSB_ADAM_FLAG_NONZERO && flag < GSB_ADAM_FLAG_NAN;
  const float step = a.step_dev ? a.step_dev[t.flag_index] : t.step;
  const long long base = t.begin + (long long)(blockIdx.x - t.first_block) * kElemsPerBlock;
#pragma unroll
  for (int u = 0; u < kVecPerThread; ++u) {
    const long long e = base + ((long long)u * kFT + threadIdx.x) * 4;
    if (e >= t.end) continue;
    float4 g[WORLD];
#pragma unroll
    for (int r = 0; r < WORLD; ++r) g[r] = ld_peer(a.grads[r] + e);      // all loads in flight together
    float4 s = g[0];
#pragma unroll
    for (int r = 1; r < WORLD; ++r) { s.x += g[r].x; s.y += g[r].y; s.z += g[r].z; s.w += g[r].w; }
    s.x *= a.gscale; s.y *= a.gscale; s.z *= a.gscale; s.w *= a.gscale;
    const long long le = e - a.shard_begin;
    float4 p = *reinterpret_cast<const float4*>(a.params[a.rank] + e);
    float4 m = *reinterpret_cast<float4*>(a.m + le);
    float4 v = *reinterpret_cast<float4*>(a.v + le);
    float l0 = 1.f, l1 = 1.f, l2 = 1.f, l3 = 1.f;
    if (t.ppl) {
      const long long q = e - t.seg_begin;
      l0 = __ldg(t.ppl + q / t.row_len); l1 = __ldg(t.ppl + (q + 1) / t.row_len);
      l2 = __ldg(t.ppl + (q + 2) / t.row_len); l3 = __ldg(t.ppl + (q + 3) / t.row_len);
    }
    adam1(t, step, gate, l0, p.x, s.x, m.x, v.x);
    adam1(t, step, gate, l1, p.y, s.y, m.y, v.y);
    adam1(t, step, gate, l2, p.z, s.z, m.z, v.z);
    adam1(t, step, gate, l3, p.w, s.w, m.w, v.w);
    *reinterpret_cast<float4*>(a.m + le) = m;
    *reinterpret_cast<float4*>(a.v + le) = v;
#pragma unroll
    for (int r = 0; r < WORLD; ++r) st_peer(a.params[r] + e, p);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Flag barriers and the small exchange (gate flags, binning-overflow word, pose-gradient table) over the same peer
// memory -- they replace the two tiny NCCL collectives that used to bracket the fused kernel (each cost a ring
// latency plus a launch at 8 ranks; these are one NVLink round trip).
//
// Signal buffer of every rank (uint32 words, peer-visible, zero-initialised):
//   [parity 2][channel 2][world]            epoch flags   (word  p*16 + c*8 + src)
//   word 60                                 local error word (1 = a wait timed out)
//   [parity 2][world][kXchMax] floats       exchange slots (from word 64)
// A rank stores its contribution into slot [parity][rank] of EVERY peer, fences, then stores the step's epoch into
// flag [parity][channel][rank] of every peer with release semantics, and finally waits (acquire) until all `world`
// flags in its OWN buffer carry the epoch.  Parity = epoch & 1, so a slot is rewritten only two steps later, by
// which time every rank has passed a later barrier and therefore finished reading it.
constexpr int kXchMax = 256;
constexpr int kSigWords = 64 + 2 * kMaxWorld * kXchMax;
constexpr long long kSpinLimit = 6000000000LL;     // ~3 s at 2 GHz: never hang the GPU on a dead peer

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys_f32(float* p, float v) {
  asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

struct SigArgs { int world, rank; unsigned int epoch; int channel; unsigned int* sig[kMaxWorld]; };

// epoch == 0 in the arguments means "device-resident epoch": word 61 of the local signal buffer, advanced by every
// k_peer_exchange (once per optimizer step on every rank, so the ranks stay in lockstep) and re-used by the
// k_peer_barrier of the same step.  That makes both launches replayable from a CUDA graph (frozen arguments).
__device__ __forceinline__ unsigned int resolve_epoch(const SigArgs& a, bool advance) {
  __shared__ unsigned int s_epoch;
  if (a.epoch != 0u) return a.epoch;
  if (threadIdx.x == 0) {
    unsigned int e = a.sig[a.rank][61];
    if (advance) { e += 1u; if (e == 0u) e = 1u; a.sig[a.rank][61] = e; }
    s_epoch = e;
  }
  __syncthreads();
  return s_epoch;
}

// all threads of the (single) CTA call this; returns after every rank has signalled `epoch` on `channel`
__device__ __forceinline__ void signal_and_wait(const SigArgs& a0, unsigned int epoch) {
  SigArgs a = a0;
  a.epoch = epoch;
  const int par = (int)(a.epoch & 1u);
  __syncthreads();
  if ((int)threadIdx.x < a.world) {
    __threadfence_system();
    st_release_sys(a.sig[threadIdx.x] + par * 16 + a.channel * 8 + a.rank, a.epoch);
    const unsigned int* mine = a.sig[a.rank] + par * 16 + a.channel * 8 + threadIdx.x;
    const long long t0 = clock64();
    while (ld_acquire_sys(mine) != a.epoch) {
      if (clock64() - t0 > kSpinLimit) { a.sig[a.rank][60] = 1u; break; }
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256) k_peer_barrier(SigArgs a) { signal_and_wait(a, resolve_epoch(a, false)); }

// flags [8] uint32 (this rank's gate flags; slot 7 is overwritten with *ovf), pose_grad [n_pose] floats: every rank
// ends up with the SUM over ranks of both, in place, accumulated in rank order (identical on all ranks).
__global__ void __launch_bounds__(256) k_peer_exchange(SigArgs a, unsigned int* flags, const unsigned int* ovf,
                                                       float* pose_grad, int n_pose) {
  const int n = 8 + n_pose;
  const unsigned int epoch = resolve_epoch(a, true);
  const int par = (int)(epoch & 1u);
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    float v;
    if (t < 7) v = (float)flags[t];
    else if (t == 7) v = ovf ? (float)(*ovf != 0u) : 0.f;
    else v = pose_grad[t - 8];
    for (int p = 0; p < a.world; ++p)
      st_relaxed_sys_f32(reinterpret_cast<float*>(a.sig[p] + 64) + ((size_t)par * kMaxWorld + a.rank) * kXchMax + t, v);
  }
  signal_and_wait(a, epoch);
  const float* mine = reinterpret_cast<const float*>(a.sig[a.rank] + 64) + (size_t)par * kMaxWorld * kXchMax;
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < a.world; ++p) s += *((volatile const float*)(mine + (size_t)p * kXchMax + t));
    if (t < 8) flags[t] = (unsigned int)(s + 0.5f);
    else pose_grad[t - 8] = s;
  }
}

int fail(cudaError_t e, const char* what) {
  char buf[256];
  snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  gsb_set_error(buf);
  return GSB_ERR_CUDA;
}

}  // namespace

extern "C" GSB_API int gsb_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64) {
  if (!dev_ptr || !handle64 || bytes == 0) { gsb_set_error("gsb_ipc_alloc: bad argument"); return GSB_ERR_INVALID; }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaError_t e = cudaMalloc(dev_ptr, bytes);
  if (e != cudaSuccess) return fail(e, "cudaMalloc");
  e = cudaMemset(*dev_ptr, 0, bytes);
  if (e != cudaSuccess) return fail(e, "cudaMemset");
  cudaIpcMemHandle_t h;
  e = cudaIpcGetMemHandle(&h, *dev_ptr);
  if (e != cudaSuccess) return fail(e, "cudaIpcGetMemHandle");
  memcpy(handle64, &h, 64);
  return GSB_OK;
}

extern "C" GSB_API int gsb_ipc_open(const unsigned char* handle64, void** dev_ptr) {
  if (!dev_ptr || !handle64) { gsb_set_error("gsb_ipc_open: bad argument"); return GSB_ERR_INVALID; }
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  cudaError_t e = cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return fail(e, "cudaIpcOpenMemHandle");
  return GSB_OK;
}

extern "C" GSB_API int gsb_ipc_close(void* dev_ptr) {
  cudaError_t e = cudaIpcCloseMemHandle(dev_ptr);
  return e == cudaSuccess ? GSB_OK : fail(e, "cudaIpcCloseMemHandle");
}

extern "C" GSB_API int gsb_ipc_free(void* dev_ptr) {
  cudaError_t e = cudaFree(dev_ptr);
  return e == cudaSuccess ? GSB_OK : fail(e, "cudaFree");
}

extern "C" GSB_API int gsb_fused_rs_adam_ag(int32_t world, int32_t rank, const float* const* peer_grads,
                                            float* const* peer_params, float* exp_avg_shard, float* exp_avg_sq_shard,
                                            int64_t shard_begin, int32_t n_pieces, const GsbShardPiece* pieces,
                                            const uint32_t* flags, const uint32_t* skip_if_nonzero, float grad_scale,
                                            const float* step_sizes_dev, gsb_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  if (world < 2 || world > kMaxWorld || rank < 0 || rank >= world || !peer_grads || !peer_params || !exp_avg_shard ||
      !exp_avg_sq_shard || n_pieces < 0 || n_pieces > kMaxPieces || (n_pieces > 0 && !pieces) || !flags ||
      (shard_begin & 3)) {
    gsb_set_error("gsb_fused_rs_adam_ag: bad argument");
    return GSB_ERR_INVALID;
  }
  FusedArgs a;
  memset(&a, 0, sizeof(a));
  a.world = world; a.rank = rank; a.n_pieces = n_pieces; a.shard_begin = shard_begin; a.gscale = grad_scale;
  a.step_dev = step_sizes_dev;
  a.m = exp_avg_shard; a.v = exp_avg_sq_shard;
  for (int r = 0; r < world; ++r) {
    if (!peer_grads[r] || !peer_params[r] || (((uintptr_t)peer_grads[r] | (uintptr_t)peer_params[r]) & 15)) {
      gsb_set_error("gsb_fused_rs_adam_ag: null / misaligned peer pointer");
      return GSB_ERR_INVALID;
    }
    a.grads[r] = peer_grads[r]; a.params[r] = peer_params[r];
  }
  unsigned int nb = 0;
  for (int i = 0; i < n_pieces; ++i) {
    const GsbShardPiece& s = pieces[i];
    if (s.begin < shard_begin || s.end < s.begin || (s.begin & 3) || (s.end & 3) || s.row_len <= 0 ||
        s.flag_index < 0 || s.flag_index >= GSB_ADAM_MAX_TENSORS) {
      gsb_set_error("gsb_fused_rs_adam_ag: bad piece (ranges must be 4-float aligned)");
      return GSB_ERR_INVALID;
    }
    Piece& t = a.pc[i];
    t.begin = s.begin; t.end = s.end; t.seg_begin = s.seg_begin; t.ppl = s.per_point_lr;
    t.row_len = s.row_len; t.flag_index = s.flag_index;
    t.step = (float)s.step_size; t.b1 = (float)s.beta1; t.omb1 = (float)(1.0 - s.beta1);
    t.b2 = (float)s.beta2; t.omb2 = (float)(1.0 - s.beta2); t.eps = (float)s.eps;
    t.first_block = nb;
    t.nblocks = (unsigned int)((s.end - s.begin + kElemsPerBlock - 1) / kElemsPerBlock);
    nb += t.nblocks;
  }
  for (int i = n_pieces; i < kMaxPieces; ++i) a.pc[i].first_block = 0xffffffffu;
  if (nb == 0) return GSB_OK;
  gsb_count_launch(1);
  int slot = gsb_prof_begin(GSB_K_ADAM, st);
  switch (world) {
    case 2: k_fused_rs_adam_ag<2><<<nb, kFT, 0, st>>>(a, flags, skip_if_nonzero); break;
    case 3: k_fused_rs_adam_ag<3><<<nb, kFT, 0, st>>>(a, flags, skip_if_nonzero); break;
    case 4: k_fused_rs_adam_ag<4><<<nb, kFT, 0, st>>>(a, flags, skip_if_nonzero); break;
    case 5: k_fused_rs_adam_ag<5><<<nb, kFT, 0, st>>>(a, flags, skip_if_nonzero); break;
    case 6: k_fused_rs_adam_ag<6><<<nb, kFT, 0, st>>>(a, flags, skip_if_nonzero); break;
    case 7: k_fused_rs_adam_ag<7><<<nb, kFT, 0, st>>>(a, flags, skip_if_nonzero); break;
    default: k_fused_rs_adam_ag<8><<<nb, kFT, 0, st>>>(a, flags, skip_if_nonzero); break;
  }
  gsb_prof_end(slot, st);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? GSB_OK : fail(e, "k_fused_rs_adam_ag");
}

static int make_sig(int32_t world, int32_t rank, void* const* sig, uint32_t epoch, int channel, SigArgs& a) {
  if (world < 2 || world > kMaxWorld || rank < 0 || rank >= world || !sig || channel < 0 || channel > 1) {
    gsb_set_error("gsb_peer_*: bad argument");
    return GSB_ERR_INVALID;
  }
  a.world = world; a.rank = rank; a.epoch = epoch; a.channel = channel;
  for (int r = 0; r < kMaxWorld; ++r) a.sig[r] = r < world ? (unsigned int*)sig[r] : nullptr;
  for (int r = 0; r < world; ++r)
    if (!a.sig[r]) { gsb_set_error("gsb_peer_*: null signal buffer"); return GSB_ERR_INVALID; }
  return GSB_OK;
}

extern "C" GSB_API size_t gsb_peer_signal_bytes(void) { return (size_t)kSigWords * 4; }

extern "C" GSB_API int gsb_peer_barrier(int32_t world, int32_t rank, void* const* peer_signal, uint32_t epoch,
                                        int32_t channel, gsb_stream_t stream_) {
  SigArgs a;
  int rc = make_sig(world, rank, peer_signal, epoch, channel, a);
  if (rc) return rc;
  gsb_count_launch(1);
  k_peer_barrier<<<1, 32, 0, (cudaStream_t)stream_>>>(a);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? GSB_OK : fail(e, "k_peer_barrier");
}

extern "C" GSB_API int gsb_peer_exchange(int32_t world, int32_t rank, void* const* peer_signal, uint32_t epoch,
                                         uint32_t* flags8, const uint32_t* overflow_word, float* pose_grad,
                                         int32_t n_pose, gsb_stream_t stream_) {
  SigArgs a;
  int rc = make_sig(world, rank, peer_signal, epoch, 0, a);
  if (rc) return rc;
  if (!flags8 || n_pose < 0 || 8 + n_pose > kXchMax || (n_pose > 0 && !pose_grad)) {
    gsb_set_error("gsb_peer_exchange: bad argument (at most 248 pose-gradient floats)");
    return GSB_ERR_INVALID;
  }
  gsb_count_launch(1);
  k_peer_exchange<<<1, 256, 0, (cudaStream_t)stream_>>>(a, flags8, overflow_word, pose_grad, n_pose);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? GSB_OK : fail(e, "k_peer_exchange");
}
