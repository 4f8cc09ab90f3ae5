// Pose-only "tracking" mode (SURVEY.md section 8 row f2): the test-view pose optimisation of
// render.py:99-170 -- Gaussians frozen, 500 Adam iterations on the 7 pose parameters of one view
// under a masked L1 loss -- as device-resident steps, so that the whole loop runs without a single host sync:
//
//   gsb_l1_mask_fwd_bwd   loss and dL/dimage of utils/loss_utils.py:17-23 (l1_loss_mask) with the mask of
//                         render.py:137-138 (mask = rendering > threshold, per element, constant w.r.t. autograd)
//   gsb_track_step        torch.optim.Adam (two parameter groups: quaternion, translation; L2 weight decay) on the
//                         pose, the loss normalisation 1/sum(mask), and the "best candidate" bookkeeping of
//                         render.py:146-151 -- all by one thread, from device-resident inputs
#include "gs_internal.cuh"

using namespace gsb;

namespace {

constexpr int kLT = 256;

// sums[0] += sum |img - gt| * mask, sums[1] += sum mask;  dL_dimg = sign(img - gt) * mask (unnormalised)
// Grid y = view: view v reads img, gt and writes dL at v * n and adds into sums[2v..2v+1].  Thread k always takes the
// elements in groups of four (4k..4k+3, then the n % 4 tail), whatever the alignment of the pointers: the split into
// blocks and threads -- and so the float partial sums -- depends only on n and the grid, so a view of a batch, a slice
// of a caller's tensor and a fresh copy of it give the same bits.  Alignment only selects 128-bit or scalar accesses.
__global__ void __launch_bounds__(kLT) k_l1_mask(size_t n, const float* __restrict__ img, const float* __restrict__ gt,
                                                 float thr, double* __restrict__ sums, float* __restrict__ dL) {
  __shared__ float red[2][kLT / 32];
  float s_abs = 0.f, s_m = 0.f;
  const size_t n4 = n >> 2;
  img += n * blockIdx.y; gt += n * blockIdx.y; dL += n * blockIdx.y; sums += 2 * blockIdx.y;
  const bool vec = ((((uintptr_t)img | (uintptr_t)gt | (uintptr_t)dL) & 15) == 0);
  for (size_t k = (size_t)blockIdx.x * kLT + threadIdx.x; k < n4; k += (size_t)gridDim.x * kLT) {
    float av[4], bv[4];
    if (vec) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(img) + k), b = __ldg(reinterpret_cast<const float4*>(gt) + k);
      av[0] = a.x; av[1] = a.y; av[2] = a.z; av[3] = a.w; bv[0] = b.x; bv[1] = b.y; bv[2] = b.z; bv[3] = b.w;
    } else {
#pragma unroll
      for (int u = 0; u < 4; ++u) { av[u] = __ldg(img + 4 * k + u); bv[u] = __ldg(gt + 4 * k + u); }
    }
    float g[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float m = av[u] > thr ? 1.f : 0.f, d = av[u] - bv[u];
      s_abs += fabsf(d) * m;
      s_m += m;
      g[u] = m * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
    }
    if (vec) {
      reinterpret_cast<float4*>(dL)[k] = make_float4(g[0], g[1], g[2], g[3]);
    } else {
#pragma unroll
      for (int u = 0; u < 4; ++u) dL[4 * k + u] = g[u];
    }
  }
  for (size_t e = 4 * n4 + (size_t)blockIdx.x * kLT + threadIdx.x; e < n; e += (size_t)gridDim.x * kLT) {
    const float m = img[e] > thr ? 1.f : 0.f, d = img[e] - gt[e];
    s_abs += fabsf(d) * m;
    s_m += m;
    dL[e] = m * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s_abs += __shfl_xor_sync(0xffffffffu, s_abs, o);
    s_m += __shfl_xor_sync(0xffffffffu, s_m, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red[0][warp] = s_abs; red[1][warp] = s_m; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, m = 0.0;
    for (int w = 0; w < kLT / 32; ++w) { a += red[0][w]; m += red[1][w]; }
    atomicAdd(sums + 0, a);
    atomicAdd(sums + 1, m);
  }
}

struct TrackArgs {
  float* pose; const float* dpose_raw; const double* sums; float* m; float* v; float* best; float* loss_out;
  int64_t loss_stride;
  float lr_q, lr_T, b1, b2, eps, wd, bc1, bc2_sqrt;
};

// one CTA per view: view w steps pose[7w..], keeps its candidate in best[8w..] and writes its loss at loss_out[w * stride]
__global__ void k_track_step(TrackArgs a) {
  if (threadIdx.x != 0) return;
  const int w = blockIdx.x;
  a.pose += 7 * w; a.dpose_raw += 7 * w; a.sums += 2 * w; a.m += 7 * w; a.v += 7 * w; a.best += 8 * w;
  if (a.loss_out) a.loss_out += a.loss_stride * w;
  const double cnt = a.sums[1];
  const float inv = cnt > 0.0 ? (float)(1.0 / cnt) : 0.f;
  const float loss = cnt > 0.0 ? (float)(a.sums[0] / cnt) : 0.f;
  float p[7];
  for (int k = 0; k < 7; ++k) {
    float g = a.dpose_raw[k] * inv;
    float pk = a.pose[k];
    g = fmaf(a.wd, pk, g);                                    // torch.optim.Adam: L2 weight decay added to the gradient
    const float m = a.b1 * a.m[k] + (1.f - a.b1) * g;
    const float v = a.b2 * a.v[k] + (1.f - a.b2) * g * g;
    a.m[k] = m; a.v[k] = v;
    const float denom = sqrtf(v) / a.bc2_sqrt + a.eps;
    const float lr = k < 4 ? a.lr_q : a.lr_T;
    pk -= (lr / a.bc1) * (m / denom);
    a.pose[k] = pk;
    p[k] = pk;
  }
  if (a.loss_out) *a.loss_out = loss;
  // render.py:146-151: the candidate is taken AFTER the optimizer step, keyed on the loss measured BEFORE it
  if (loss < a.best[0]) {
    a.best[0] = loss;
    for (int k = 0; k < 7; ++k) a.best[1 + k] = p[k];
  }
}

// ---- size of the 3D smoothing filter (DESIGN.md section 4.7) -------------------------------------------------------
// Pass 1: one thread per Gaussian, the views staged in shared memory kMV at a time as (R row-major, t):
// out[i] = smallest p_z over the views that count, -1 when none does.
constexpr int kMV = 256;
__global__ void __launch_bounds__(kLT) k_mip_depth(int P, const float* __restrict__ xyz, int V,
                                                   const float* __restrict__ poses7, float fx, float fy, int W, int H,
                                                   float* __restrict__ out) {
  __shared__ float s_v[kMV][12];
  const int i = blockIdx.x * kLT + threadIdx.x;
  float x[3] = {0.f, 0.f, 0.f};
  if (i < P) { x[0] = xyz[3 * (size_t)i]; x[1] = xyz[3 * (size_t)i + 1]; x[2] = xyz[3 * (size_t)i + 2]; }
  float d = 3.0e38f;
  for (int v0 = 0; v0 < V; v0 += kMV) {
    const int nv = min(kMV, V - v0);
    __syncthreads();
    for (int v = threadIdx.x; v < nv; v += kLT) {
      const float* q = poses7 + 7 * (size_t)(v0 + v);
      const float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
      quat_to_R(q[0] / n, q[1] / n, q[2] / n, q[3] / n, s_v[v]);
      s_v[v][9] = q[4]; s_v[v][10] = q[5]; s_v[v][11] = q[6];
    }
    __syncthreads();
    for (int v = 0; v < nv; ++v) {
      const float z = mip_view_depth(s_v[v], s_v[v] + 9, x, fx, fy, W, H);
      if (z >= 0.f) d = fminf(d, z);
    }
  }
  if (i < P) out[i] = d < 3.0e38f ? d : -1.f;
}

// Pass 2 (one CTA; a max is exact in any order, so the result is deterministic): Gaussians no view counts for take the
// largest depth found, then f = d / fx * sqrt(0.2).  When no Gaussian is seen at all, f = 0 (no filter).
constexpr int kMF = 1024;
__global__ void __launch_bounds__(kMF) k_mip_finish(int P, float fx, float* __restrict__ out) {
  __shared__ float red[kMF / 32];
  float m = -1.f;
  for (int i = threadIdx.x; i < P; i += kMF) m = fmaxf(m, out[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < kMF / 32; ++w) m = fmaxf(m, red[w]);
  for (int i = threadIdx.x; i < P; i += kMF) {
    const float d = out[i] >= 0.f ? out[i] : m;
    out[i] = d >= 0.f ? d / fx * kMipSqrtVar : 0.f;
  }
}

}  // namespace

extern "C" GSB_API int gsb_mip_filter3d(int32_t P, const float* xyz, int32_t n_views, const float* poses7,
                                        int32_t width, int32_t height, float tanfovx, float tanfovy, float* out,
                                        gsb_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  GSB_REQUIRE(P >= 0 && n_views >= 0 && width > 0 && height > 0 && tanfovx > 0.f && tanfovy > 0.f,
              "gsb_mip_filter3d: bad argument");
  if (P == 0) return GSB_OK;
  GSB_REQUIRE(xyz && out && (poses7 || n_views == 0), "gsb_mip_filter3d: null buffer");
  const float fx = width / (2.0f * tanfovx), fy = height / (2.0f * tanfovy);
  gsb_count_launch(2);
  k_mip_depth<<<(P + kLT - 1) / kLT, kLT, 0, st>>>(P, xyz, n_views, poses7, fx, fy, width, height, out);
  k_mip_finish<<<1, kMF, 0, st>>>(P, fx, out);
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}

extern "C" GSB_API int gsb_l1_mask_fwd_bwd_batch(int32_t V, int32_t C, int32_t H, int32_t W, const float* img,
                                                 const float* gt, float threshold, double* sums, float* dL_dimg,
                                                 gsb_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  GSB_REQUIRE(V >= 1 && V <= 65535 && C > 0 && H > 0 && W > 0 && img && gt && sums && dL_dimg,
              "gsb_l1_mask_fwd_bwd: bad argument");
  const size_t n = (size_t)C * H * W;
  const int max_blocks = 8 * gsb_sm_count();
  const int blocks = (int)((n / 4 + kLT - 1) / kLT < (size_t)max_blocks ? (n / 4 + kLT - 1) / kLT + 1 : max_blocks);
  ProfScope ps(GSB_K_LOSS_FWD, st);
  k_l1_mask<<<dim3(blocks, V), kLT, 0, st>>>(n, img, gt, threshold, sums, dL_dimg);
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}

extern "C" GSB_API int gsb_l1_mask_fwd_bwd(int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                                           float threshold, double* sums, float* dL_dimg, gsb_stream_t stream) {
  return gsb_l1_mask_fwd_bwd_batch(1, C, H, W, img, gt, threshold, sums, dL_dimg, stream);
}

extern "C" GSB_API int gsb_track_step_batch(int32_t V, float* pose7, const float* dpose7_raw, const double* sums2,
                                            float* exp_avg7, float* exp_avg_sq7, float* best8, float* loss_out,
                                            int64_t loss_stride, int32_t step, float lr_q, float lr_T, float beta1,
                                            float beta2, float eps, float weight_decay, gsb_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  GSB_REQUIRE(V >= 1 && V <= 65535 && pose7 && dpose7_raw && sums2 && exp_avg7 && exp_avg_sq7 && best8 && step >= 1,
              "gsb_track_step: bad argument");
  TrackArgs a;
  a.pose = pose7; a.dpose_raw = dpose7_raw; a.sums = sums2; a.m = exp_avg7; a.v = exp_avg_sq7; a.best = best8;
  a.loss_out = loss_out; a.loss_stride = loss_stride;
  a.lr_q = lr_q; a.lr_T = lr_T; a.b1 = beta1; a.b2 = beta2; a.eps = eps; a.wd = weight_decay;
  a.bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  a.bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  ProfScope ps(GSB_K_ADAM, st);
  k_track_step<<<V, 32, 0, st>>>(a);
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}

extern "C" GSB_API int gsb_track_step(float* pose7, const float* dpose7_raw, const double* sums2, float* exp_avg7,
                                      float* exp_avg_sq7, float* best8, float* loss_out, int32_t step, float lr_q,
                                      float lr_T, float beta1, float beta2, float eps, float weight_decay,
                                      gsb_stream_t stream) {
  return gsb_track_step_batch(1, pose7, dpose7_raw, sums2, exp_avg7, exp_avg_sq7, best8, loss_out, 0, step, lr_q, lr_T,
                              beta1, beta2, eps, weight_decay, stream);
}
