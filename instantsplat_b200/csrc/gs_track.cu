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

namespace {

constexpr int kLT = 256;

// sums[0] += sum |img - gt| * mask, sums[1] += sum mask;  dL_dimg = sign(img - gt) * mask (unnormalised)
__global__ void __launch_bounds__(kLT) k_l1_mask(size_t n, const float* __restrict__ img, const float* __restrict__ gt,
                                                 float thr, double* __restrict__ sums, float* __restrict__ dL) {
  __shared__ float red[2][kLT / 32];
  float s_abs = 0.f, s_m = 0.f;
  const size_t n4 = n >> 2;
  const bool vec = ((((uintptr_t)img | (uintptr_t)gt | (uintptr_t)dL) & 15) == 0);
  for (size_t k = (size_t)blockIdx.x * kLT + threadIdx.x; k < (vec ? n4 : 0); k += (size_t)gridDim.x * kLT) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(img) + k), b = __ldg(reinterpret_cast<const float4*>(gt) + k);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
    float g[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float m = av[u] > thr ? 1.f : 0.f, d = av[u] - bv[u];
      s_abs += fabsf(d) * m;
      s_m += m;
      g[u] = m * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
    }
    reinterpret_cast<float4*>(dL)[k] = make_float4(g[0], g[1], g[2], g[3]);
  }
  for (size_t e = (vec ? 4 * n4 : 0) + (size_t)blockIdx.x * kLT + threadIdx.x; e < n; e += (size_t)gridDim.x * kLT) {
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
  float lr_q, lr_T, b1, b2, eps, wd, bc1, bc2_sqrt;
};

__global__ void k_track_step(TrackArgs a) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
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

}  // namespace

extern "C" GSB_API int gsb_l1_mask_fwd_bwd(int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                                           float threshold, double* sums, float* dL_dimg, gsb_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  GSB_REQUIRE(C > 0 && H > 0 && W > 0 && img && gt && sums && dL_dimg, "gsb_l1_mask_fwd_bwd: bad argument");
  const size_t n = (size_t)C * H * W;
  const int max_blocks = 8 * gsb_sm_count();
  const int blocks = (int)((n / 4 + kLT - 1) / kLT < (size_t)max_blocks ? (n / 4 + kLT - 1) / kLT + 1 : max_blocks);
  ProfScope ps(GSB_K_LOSS_FWD, st);
  k_l1_mask<<<blocks, kLT, 0, st>>>(n, img, gt, threshold, sums, dL_dimg);
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}

extern "C" GSB_API int gsb_track_step(float* pose7, const float* dpose7_raw, const double* sums2, float* exp_avg7,
                                      float* exp_avg_sq7, float* best8, float* loss_out, int32_t step, float lr_q,
                                      float lr_T, float beta1, float beta2, float eps, float weight_decay,
                                      gsb_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  GSB_REQUIRE(pose7 && dpose7_raw && sums2 && exp_avg7 && exp_avg_sq7 && best8 && step >= 1, "gsb_track_step: bad argument");
  TrackArgs a;
  a.pose = pose7; a.dpose_raw = dpose7_raw; a.sums = sums2; a.m = exp_avg7; a.v = exp_avg_sq7; a.best = best8;
  a.loss_out = loss_out;
  a.lr_q = lr_q; a.lr_T = lr_T; a.b1 = beta1; a.b2 = beta2; a.eps = eps; a.wd = weight_decay;
  a.bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  a.bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  ProfScope ps(GSB_K_ADAM, st);
  k_track_step<<<1, 32, 0, st>>>(a);
  GSB_CUDA(cudaGetLastError());
  return GSB_OK;
}
