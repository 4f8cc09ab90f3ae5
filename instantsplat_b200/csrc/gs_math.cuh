// Per-Gaussian and per-pair arithmetic of the rasterizer, written once as
// __host__ __device__ inline functions so the same code runs inside the sm_90a kernels
// (gs_raster.cu) and inside the CPU math harness tests compile with g++ (tests/host_math.cpp).
//
// Behaviour follows SURVEY.md Appendix A (the published algorithm of
// graphdeco-inria/diff-gaussian-rasterization @ 59f5f77, an empty submodule in the reference checkout),
// anchored on the reference call site gaussian_renderer/__init__.py:60-135.
// The InstantSplat pose pre-transform (gaussian_renderer/__init__.py:81-89,
// utils/pose_utils.py:10-55,86-104) and the parameter activations
// (scene/gaussian_model.py:101-121) are fused in.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define GS_HD __host__ __device__ __forceinline__
#else
#define GS_HD inline
#endif

namespace gsb {

constexpr int   kBlock     = 16;            // tile edge (pixels)
constexpr float kAlphaMin  = 1.0f / 255.0f;
constexpr float kTEps      = 1e-4f;
constexpr float kNear      = 0.2f;

constexpr float SH_C0 = 0.28209479177387814f;
constexpr float SH_C1 = 0.4886025119029199f;
constexpr float SH_C2_0 = 1.0925484305920792f, SH_C2_1 = -1.0925484305920792f,
                SH_C2_2 = 0.31539156525252005f, SH_C2_3 = -1.0925484305920792f,
                SH_C2_4 = 0.5462742152960396f;
constexpr float SH_C3_0 = -0.5900435899266435f, SH_C3_1 = 2.890611442640554f,
                SH_C3_2 = -0.4570457994644658f, SH_C3_3 = 0.3731763325901154f,
                SH_C3_4 = -0.4570457994644658f, SH_C3_5 = 1.445305721320277f,
                SH_C3_6 = -0.5900435899266435f;

// Camera constants shared by every Gaussian of a launch (lives in shared memory on device).
struct CamConst {
  float V[16];       // viewmatrix, row-vector convention: p_view = [p,1] @ V
  float Pm[16];      // projmatrix, same convention
  float campos[3];
  float tanfovx, tanfovy, fx, fy, scale_mod;
  int W, H, gx, gy;
  int D;             // active SH degree
  int M;             // SH coefficients stored per Gaussian
  // fused InstantSplat pose (identity when pose_on == 0)
  int pose_on;
  float Rc[9];       // rotation of the normalised pose quaternion
  float tc[3];
  float qc[4];       // RAW pose quaternion (quadmultiply uses it un-normalised)
  int raw_params;    // scales are log-scales, opacities are logits
};

GS_HD void quat_to_R(float r, float x, float y, float z, float* R) {
  R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - r * z); R[2] = 2.f * (x * z + r * y);
  R[3] = 2.f * (x * y + r * z); R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - r * x);
  R[6] = 2.f * (x * z - r * y); R[7] = 2.f * (y * z + r * x); R[8] = 1.f - 2.f * (x * x + y * y);
}

// dL/dq (raw) from dL/dR for R = quat_to_R(q)
GS_HD void quat_to_R_bwd(float r, float x, float y, float z, const float* dR, float* dq) {
  dq[0] = 2.f * (-z * dR[1] + y * dR[2] + z * dR[3] - x * dR[5] - y * dR[6] + x * dR[7]);
  dq[1] = 2.f * (y * dR[1] + z * dR[2] + y * dR[3] - 2.f * x * dR[4] - r * dR[5] + z * dR[6] +
                 r * dR[7] - 2.f * x * dR[8]);
  dq[2] = 2.f * (-2.f * y * dR[0] + x * dR[1] + r * dR[2] + x * dR[3] + z * dR[5] - r * dR[6] +
                 z * dR[7] - 2.f * y * dR[8]);
  dq[3] = 2.f * (-2.f * z * dR[0] - r * dR[1] + x * dR[2] + r * dR[3] - 2.f * z * dR[4] +
                 y * dR[5] + x * dR[6] + y * dR[7]);
}

// Fill the pose part of CamConst from pose = [qw,qx,qy,qz,tx,ty,tz]
// (utils/pose_utils.py:34-55 normalises; quadmultiply :86-104 does not).
GS_HD void pose_to_const(const float* pose, CamConst& c) {
  float n = sqrtf(pose[0] * pose[0] + pose[1] * pose[1] + pose[2] * pose[2] + pose[3] * pose[3]);
  quat_to_R(pose[0] / n, pose[1] / n, pose[2] / n, pose[3] / n, c.Rc);
  c.tc[0] = pose[4]; c.tc[1] = pose[5]; c.tc[2] = pose[6];
  c.qc[0] = pose[0]; c.qc[1] = pose[1]; c.qc[2] = pose[2]; c.qc[3] = pose[3];
  c.pose_on = 1;
}

// Final chain for the pose gradient: acc = [dqc_raw(4), dt(3), dRc(9)] summed over Gaussians.
GS_HD void pose_grad_finalize(const float* pose, const float* acc, float* dpose) {
  float n = sqrtf(pose[0] * pose[0] + pose[1] * pose[1] + pose[2] * pose[2] + pose[3] * pose[3]);
  float qn[4] = {pose[0] / n, pose[1] / n, pose[2] / n, pose[3] / n};
  float dqn[4];
  quat_to_R_bwd(qn[0], qn[1], qn[2], qn[3], acc + 7, dqn);
  float dot = qn[0] * dqn[0] + qn[1] * dqn[1] + qn[2] * dqn[2] + qn[3] * dqn[3];
  for (int i = 0; i < 4; ++i) dpose[i] = acc[i] + (dqn[i] - qn[i] * dot) / n;
  dpose[4] = acc[4]; dpose[5] = acc[5]; dpose[6] = acc[6];
}

// Mip-Splatting filters (DESIGN.md section 4.7).  on2d: the 2D Mip filter, kappa * I replaces the 0.3 px^2 dilation and
// the opacity is compensated by h2 = sqrt(max(kMipH2Min, det(Sigma2) / det(Sigma2 + kappa I))).  on3d: the 3D
// smoothing filter of size f (world units, raw parameters only): s~ = sqrt(s^2 + f^2), opacity * prod_k s_k / s~_k;
// f = 0: no 3D filter for that Gaussian.
// Mip() (on == 0) is the reference path, operation for operation.
constexpr float kMipH2Min = 2.5e-5f;
struct Mip {
  int on = 0, on2d = 0, on3d = 0;
  float kappa = 0.f, f = 0.f;
};

// Everything the forward produces for one Gaussian, plus what the backward re-derives from.
struct Proj {
  int visible;
  float x, y;              // pixel-centre coordinates
  float A, B, C;           // conic
  float opacity;           // activated; with a Mip filter the record opacity o_eff = o3 * h2
  float sig;               // activated opacity before the filters (filters on only)
  float o3, h2, h3;        // o3 = sig * h3; h2, h3 the 2D / 3D compensations (1 when off)
  float a0, c0, det0;      // undilated cov2D diagonal and determinant (2D filter)
  int h2clamp;             // 1: h2 sits at its floor, no gradient through it
  float depth;             // view-space z
  float rgb[3];
  unsigned clamped;        // bit c set: channel c was clamped at 0
  int radius;
  int rx0, ry0, rx1, ry1;  // tile rect [min, max)
  // intermediates kept for the backward
  float mc[3];             // mean handed to the rasterizer (camera frame when pose fused)
  float q[4];              // composed raw quaternion
  float s[3];              // activated scale * scale_modifier
  float Sig[6];            // cov3D (xx,xy,xz,yy,yz,zz)
  float t[3];              // view-space mean with the frustum clamp applied to x,y
  int clx, cly;
  float T[6];              // 2x3  T = J * Wr
  float a, b, c, det;
  float hom[4];
  float p_w;
};

struct GaussIn {
  float m[3];        // means3D input (world xyz when pose fused)
  float sc[3];       // scales input (log-scale when raw_params)
  float q[4];        // rotation input (raw)
  float op;          // opacity input (logit when raw_params)
};

GS_HD float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }

// SH -> RGB.  sh_dc: 3 floats; sh_rest: (M-1)*3 floats coefficient-major. dir must be unit.
GS_HD void sh_to_rgb(int D, const float* sh_dc, const float* sh_rest, float x, float y, float z,
                     float* rgb) {
  for (int ch = 0; ch < 3; ++ch) {
    float r = SH_C0 * sh_dc[ch];
    if (D > 0) {
      const float* s = sh_rest + ch;   // s[3*(k-1)] is coefficient k
      r = r - SH_C1 * y * s[0] + SH_C1 * z * s[3] - SH_C1 * x * s[6];
      if (D > 1) {
        float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
        r = r + SH_C2_0 * xy * s[9] + SH_C2_1 * yz * s[12] + SH_C2_2 * (2.f * zz - xx - yy) * s[15] +
            SH_C2_3 * xz * s[18] + SH_C2_4 * (xx - yy) * s[21];
        if (D > 2) {
          r = r + SH_C3_0 * y * (3.f * xx - yy) * s[24] + SH_C3_1 * xy * z * s[27] +
              SH_C3_2 * y * (4.f * zz - xx - yy) * s[30] +
              SH_C3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy) * s[33] +
              SH_C3_4 * x * (4.f * zz - xx - yy) * s[36] + SH_C3_5 * z * (xx - yy) * s[39] +
              SH_C3_6 * x * (xx - 3.f * yy) * s[42];
        }
      }
    }
    rgb[ch] = r;
  }
}

// d/dsh store of sh_to_rgb_bwd: kAcc adds the value to what is there, rounded once (never contracted into an FMA), so
// that a sum over views is the sum of the single-view values
template <bool kAcc>
GS_HD void sh_put(float& o, float v) {
  if constexpr (kAcc) {
#if defined(__CUDA_ARCH__)
    o = __fadd_rn(o, v);
#else
    o = o + v;
#endif
  } else {
    o = v;
  }
}

// Backward of sh_to_rgb: writes d/dsh (dc: 3, rest: 3*(K-1) for the K active coeffs; inactive
// ones are left untouched) and returns dL/ddir.  ALIAS-SAFE: d_rest may be the same memory as
// sh_rest (each channel's coefficients are read into registers before that channel is written).
// kAcc: add d/dsh to d_dc / d_rest instead (which must then not alias sh_rest).
template <bool kAcc = false>
GS_HD void sh_to_rgb_bwd(int D, const float* sh_rest, float x, float y, float z, const float* dL,
                         float* d_dc, float* d_rest, float* ddir) {
  float gx = 0.f, gy = 0.f, gz = 0.f;
  float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
  for (int ch = 0; ch < 3; ++ch) {
    float g = dL[ch];
    sh_put<kAcc>(d_dc[ch], SH_C0 * g);
    if (D > 0) {
      const float* s = sh_rest + ch;
      float* o = d_rest + ch;
      float c1 = s[0], c2 = s[3], c3 = s[6];
      float dx = -SH_C1 * c3, dy = -SH_C1 * c1, dz = SH_C1 * c2;
      if (D > 1) {
        float c4 = s[9], c5 = s[12], c6 = s[15], c7 = s[18], c8 = s[21];
        dx += SH_C2_0 * y * c4 + SH_C2_2 * (-2.f * x) * c6 + SH_C2_3 * z * c7 + SH_C2_4 * 2.f * x * c8;
        dy += SH_C2_0 * x * c4 + SH_C2_1 * z * c5 + SH_C2_2 * (-2.f * y) * c6 + SH_C2_4 * (-2.f * y) * c8;
        dz += SH_C2_1 * y * c5 + SH_C2_2 * 4.f * z * c6 + SH_C2_3 * x * c7;
        if (D > 2) {
          float c9 = s[24], c10 = s[27], c11 = s[30], c12 = s[33], c13 = s[36], c14 = s[39], c15 = s[42];
          dx += SH_C3_0 * c9 * 6.f * xy + SH_C3_1 * c10 * yz + SH_C3_2 * c11 * (-2.f * xy) +
                SH_C3_3 * c12 * (-6.f * xz) + SH_C3_4 * c13 * (4.f * zz - 3.f * xx - yy) +
                SH_C3_5 * c14 * 2.f * xz + SH_C3_6 * c15 * (3.f * xx - 3.f * yy);
          dy += SH_C3_0 * c9 * (3.f * xx - 3.f * yy) + SH_C3_1 * c10 * xz +
                SH_C3_2 * c11 * (4.f * zz - xx - 3.f * yy) + SH_C3_3 * c12 * (-6.f * yz) +
                SH_C3_4 * c13 * (-2.f * xy) + SH_C3_5 * c14 * (-2.f * yz) + SH_C3_6 * c15 * (-6.f * xy);
          dz += SH_C3_1 * c10 * xy + SH_C3_2 * c11 * 8.f * yz +
                SH_C3_3 * c12 * (6.f * zz - 3.f * xx - 3.f * yy) + SH_C3_4 * c13 * 8.f * xz +
                SH_C3_5 * c14 * (xx - yy);
          sh_put<kAcc>(o[24], SH_C3_0 * y * (3.f * xx - yy) * g); sh_put<kAcc>(o[27], SH_C3_1 * xy * z * g);
          sh_put<kAcc>(o[30], SH_C3_2 * y * (4.f * zz - xx - yy) * g);
          sh_put<kAcc>(o[33], SH_C3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy) * g);
          sh_put<kAcc>(o[36], SH_C3_4 * x * (4.f * zz - xx - yy) * g); sh_put<kAcc>(o[39], SH_C3_5 * z * (xx - yy) * g);
          sh_put<kAcc>(o[42], SH_C3_6 * x * (xx - 3.f * yy) * g);
        }
        sh_put<kAcc>(o[9], SH_C2_0 * xy * g); sh_put<kAcc>(o[12], SH_C2_1 * yz * g);
        sh_put<kAcc>(o[15], SH_C2_2 * (2.f * zz - xx - yy) * g);
        sh_put<kAcc>(o[18], SH_C2_3 * xz * g); sh_put<kAcc>(o[21], SH_C2_4 * (xx - yy) * g);
      }
      sh_put<kAcc>(o[0], -SH_C1 * y * g); sh_put<kAcc>(o[3], SH_C1 * z * g); sh_put<kAcc>(o[6], -SH_C1 * x * g);
      gx += dx * g; gy += dy * g; gz += dz * g;
    }
  }
  ddir[0] = gx; ddir[1] = gy; ddir[2] = gz;
}

// Geometry part of the forward (Appendix A.2 steps 1-7).  cov3D_pre: 6 floats or nullptr; mf: the Mip filters, read
// only by the kMip instantiation (kMip == false compiles the reference arithmetic and nothing else).
template <bool kMip = false>
GS_HD void project_geometry(const CamConst& c, const GaussIn& in, const float* cov3D_pre, Proj& o,
                            const Mip mf = Mip()) {
  o.visible = 0; o.radius = 0; o.rx0 = o.ry0 = o.rx1 = o.ry1 = 0; o.clamped = 0;
  if constexpr (kMip) { o.h2 = o.h3 = 1.f; o.h2clamp = 0; }
  // ---- fused pose pre-transform + activations
  if (c.pose_on) {
    o.mc[0] = c.Rc[0] * in.m[0] + c.Rc[1] * in.m[1] + c.Rc[2] * in.m[2] + c.tc[0];
    o.mc[1] = c.Rc[3] * in.m[0] + c.Rc[4] * in.m[1] + c.Rc[5] * in.m[2] + c.tc[1];
    o.mc[2] = c.Rc[6] * in.m[0] + c.Rc[7] * in.m[1] + c.Rc[8] * in.m[2] + c.tc[2];
    float w1 = c.qc[0], x1 = c.qc[1], y1 = c.qc[2], z1 = c.qc[3];
    float w2 = in.q[0], x2 = in.q[1], y2 = in.q[2], z2 = in.q[3];
    o.q[0] = w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2;
    o.q[1] = w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2;
    o.q[2] = w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2;
    o.q[3] = w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2;
  } else {
    o.mc[0] = in.m[0]; o.mc[1] = in.m[1]; o.mc[2] = in.m[2];
    o.q[0] = in.q[0]; o.q[1] = in.q[1]; o.q[2] = in.q[2]; o.q[3] = in.q[3];
  }
  // f == 0 is no 3D filter for this Gaussian: the unfiltered arithmetic, not (s*s)/(s*s), which is 0/0 once s*s
  // underflows (log-scale <= -52)
  const bool f3d = kMip && c.raw_params && mf.on3d && mf.f != 0.f;   // kMip == false: folded away at compile time
  if (f3d) {
    const float f2 = mf.f * mf.f;
    float r = 1.f;                                 // prod_k s_k^2 / (s_k^2 + f^2), one bounded factor at a time
    for (int k = 0; k < 3; ++k) {
      const float s = expf(in.sc[k]), v = s * s + f2;
      o.s[k] = c.scale_mod * sqrtf(v);
      r *= (s * s) / v;
    }
    o.sig = sigmoidf_(in.op);
    o.h3 = sqrtf(r);
    o.opacity = o.sig * o.h3;
  } else if (c.raw_params) {
    o.s[0] = c.scale_mod * expf(in.sc[0]); o.s[1] = c.scale_mod * expf(in.sc[1]);
    o.s[2] = c.scale_mod * expf(in.sc[2]);
    o.opacity = sigmoidf_(in.op);
  } else {
    o.s[0] = c.scale_mod * in.sc[0]; o.s[1] = c.scale_mod * in.sc[1]; o.s[2] = c.scale_mod * in.sc[2];
    o.opacity = in.op;
  }
  if (kMip && mf.on) { if (!f3d) o.sig = o.opacity; o.o3 = o.opacity; }
  const float* m = o.mc;
  // ---- view / clip transforms
  float tx = m[0] * c.V[0] + m[1] * c.V[4] + m[2] * c.V[8] + c.V[12];
  float ty = m[0] * c.V[1] + m[1] * c.V[5] + m[2] * c.V[9] + c.V[13];
  float tz = m[0] * c.V[2] + m[1] * c.V[6] + m[2] * c.V[10] + c.V[14];
  o.depth = tz;
  for (int j = 0; j < 4; ++j)
    o.hom[j] = m[0] * c.Pm[j] + m[1] * c.Pm[4 + j] + m[2] * c.Pm[8 + j] + c.Pm[12 + j];
  o.p_w = 1.0f / (o.hom[3] + 0.0000001f);
  if (!(tz > kNear)) return;                                      // A.2.1
  // ---- cov3D
  if (cov3D_pre) {
    for (int i = 0; i < 6; ++i) o.Sig[i] = cov3D_pre[i];
  } else {
    float R[9];
    quat_to_R(o.q[0], o.q[1], o.q[2], o.q[3], R);
    float Mx[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Mx[3 * i + j] = R[3 * i + j] * o.s[j];
    o.Sig[0] = Mx[0] * Mx[0] + Mx[1] * Mx[1] + Mx[2] * Mx[2];
    o.Sig[1] = Mx[0] * Mx[3] + Mx[1] * Mx[4] + Mx[2] * Mx[5];
    o.Sig[2] = Mx[0] * Mx[6] + Mx[1] * Mx[7] + Mx[2] * Mx[8];
    o.Sig[3] = Mx[3] * Mx[3] + Mx[4] * Mx[4] + Mx[5] * Mx[5];
    o.Sig[4] = Mx[3] * Mx[6] + Mx[4] * Mx[7] + Mx[5] * Mx[8];
    o.Sig[5] = Mx[6] * Mx[6] + Mx[7] * Mx[7] + Mx[8] * Mx[8];
  }
  // ---- EWA (A.2.3)
  float limx = 1.3f * c.tanfovx, limy = 1.3f * c.tanfovy;
  float txtz = tx / tz, tytz = ty / tz;
  o.clx = (txtz < -limx) || (txtz > limx);
  o.cly = (tytz < -limy) || (tytz > limy);
  float txc = fminf(limx, fmaxf(-limx, txtz)) * tz;
  float tyc = fminf(limy, fmaxf(-limy, tytz)) * tz;
  o.t[0] = txc; o.t[1] = tyc; o.t[2] = tz;
  float J00 = c.fx / tz, J02 = -(c.fx * txc) / (tz * tz);
  float J11 = c.fy / tz, J12 = -(c.fy * tyc) / (tz * tz);
  // T[r][i] = sum_j J[r][j] * Wr[j][i],  Wr[j][i] = V[4*i + j]
  for (int i = 0; i < 3; ++i) {
    o.T[i]     = J00 * c.V[4 * i + 0] + J02 * c.V[4 * i + 2];
    o.T[3 + i] = J11 * c.V[4 * i + 1] + J12 * c.V[4 * i + 2];
  }
  const float* S = o.Sig;
  float* T = o.T;
  // u_r = Sigma * T_r
  float u0[3] = {S[0] * T[0] + S[1] * T[1] + S[2] * T[2], S[1] * T[0] + S[3] * T[1] + S[4] * T[2],
                 S[2] * T[0] + S[4] * T[1] + S[5] * T[2]};
  float u1[3] = {S[0] * T[3] + S[1] * T[4] + S[2] * T[5], S[1] * T[3] + S[3] * T[4] + S[4] * T[5],
                 S[2] * T[3] + S[4] * T[4] + S[5] * T[5]};
  const bool mip2d = kMip && mf.on2d;
  if (mip2d) {
    o.a0 = T[0] * u0[0] + T[1] * u0[1] + T[2] * u0[2];
    o.b = T[0] * u1[0] + T[1] * u1[1] + T[2] * u1[2];
    o.c0 = T[3] * u1[0] + T[4] * u1[1] + T[5] * u1[2];
    o.a = o.a0 + mf.kappa;
    o.c = o.c0 + mf.kappa;
  } else {
    o.a = T[0] * u0[0] + T[1] * u0[1] + T[2] * u0[2] + 0.3f;
    o.b = T[0] * u1[0] + T[1] * u1[1] + T[2] * u1[2];
    o.c = T[3] * u1[0] + T[4] * u1[1] + T[5] * u1[2] + 0.3f;
  }
  o.det = o.a * o.c - o.b * o.b;
  if (o.det == 0.0f) return;                                      // A.2.4
  if (mip2d) {
    o.det0 = o.a0 * o.c0 - o.b * o.b;
    const float r = o.det0 / o.det;
    o.h2clamp = !(r > kMipH2Min);
    o.h2 = sqrtf(fmaxf(kMipH2Min, r));
    o.opacity = o.o3 * o.h2;
  }
  float det_inv = 1.f / o.det;
  o.A = o.c * det_inv; o.B = -o.b * det_inv; o.C = o.a * det_inv;
  float mid = 0.5f * (o.a + o.c);
  float lam = mid + sqrtf(fmaxf(0.1f, mid * mid - o.det));
  float rad = ceilf(3.f * sqrtf(lam));                            // A.2.5
  o.x = ((o.hom[0] * o.p_w + 1.0f) * c.W - 1.0f) * 0.5f;          // A.2.6
  o.y = ((o.hom[1] * o.p_w + 1.0f) * c.H - 1.0f) * 0.5f;
  // A.2.7 (C int truncation; clamp first so huge values stay defined)
  float lim = 1.0e8f;
  int rx0 = (int)fminf(lim, fmaxf(-lim, (o.x - rad) / kBlock));
  int ry0 = (int)fminf(lim, fmaxf(-lim, (o.y - rad) / kBlock));
  int rx1 = (int)fminf(lim, fmaxf(-lim, (o.x + rad + kBlock - 1) / kBlock));
  int ry1 = (int)fminf(lim, fmaxf(-lim, (o.y + rad + kBlock - 1) / kBlock));
  o.rx0 = rx0 < 0 ? 0 : (rx0 > c.gx ? c.gx : rx0);
  o.ry0 = ry0 < 0 ? 0 : (ry0 > c.gy ? c.gy : ry0);
  o.rx1 = rx1 < 0 ? 0 : (rx1 > c.gx ? c.gx : rx1);
  o.ry1 = ry1 < 0 ? 0 : (ry1 > c.gy ? c.gy : ry1);
  if ((o.rx1 - o.rx0) * (o.ry1 - o.ry0) == 0) return;
  o.radius = (int)rad;
  o.visible = 1;
}

// Size of the 3D smoothing filter (DESIGN.md section 4.7): f = d / fx_max * sqrt(0.2), d the smallest depth over the
// training views that count for the Gaussian.  A view (rotation R row-major, translation t: p = R x + t, the transform the
// fused preprocess applies to a pose row) counts when p_z > 0.2 and the projection lies in the frame widened by 15 %.
constexpr float kMipMargin = 0.15f;
constexpr float kMipSqrtVar = 0.44721359549995794f;   // sqrt(0.2)
// p_z when the view counts for world point x, else -1
GS_HD float mip_view_depth(const float* R, const float* t, const float* x, float fx, float fy, int W, int H) {
  const float pz = R[6] * x[0] + R[7] * x[1] + R[8] * x[2] + t[2];
  if (!(pz > kNear)) return -1.f;
  const float px = R[0] * x[0] + R[1] * x[1] + R[2] * x[2] + t[0];
  const float py = R[3] * x[0] + R[4] * x[1] + R[5] * x[2] + t[1];
  const float u = px / pz * fx + 0.5f * W, v = py / pz * fy + 0.5f * H;
  const bool in = u >= -kMipMargin * W && u <= (1.f + kMipMargin) * W && v >= -kMipMargin * H &&
                  v <= (1.f + kMipMargin) * H;
  return in ? pz : -1.f;
}

// Colour part (A.2.8).  Uses the mean handed to the rasterizer and campos.
GS_HD void project_color(const CamConst& c, const float* sh_dc, const float* sh_rest, Proj& o) {
  float dx = o.mc[0] - c.campos[0], dy = o.mc[1] - c.campos[1], dz = o.mc[2] - c.campos[2];
  float inv = 1.f / sqrtf(dx * dx + dy * dy + dz * dz);
  float raw[3];
  sh_to_rgb(c.D, sh_dc, sh_rest, dx * inv, dy * inv, dz * inv, raw);
  o.clamped = 0;
  for (int ch = 0; ch < 3; ++ch) {
    float v = raw[ch] + 0.5f;
    if (v < 0.f) { o.clamped |= (1u << ch); v = 0.f; }
    o.rgb[ch] = v;
  }
}

// ------------------------------------------------------------------------------------------
// Lossless culling.  A pair (Gaussian, pixel) contributes only if alpha = o*exp(-q/2) >= 1/255
// (A.2.10), i.e. q = A dx^2 + 2B dx dy + C dy^2 <= 2 ln(255 o) =: qthr.  A rectangle of pixel
// centres can therefore be skipped when min q over it exceeds qthr (with a safety margin, so
// pairs near the threshold are always evaluated by the exact per-pair rule).
// ------------------------------------------------------------------------------------------
GS_HD float gs_fdiv(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdividef(a, b);
#else
  return a / b;
#endif
}

GS_HD float cull_threshold(float opacity) {
  // returns < 0 when the Gaussian can never reach alpha >= 1/255
  if (!(opacity * 255.0f >= 0.999f)) return -1.0f;
  float q = 2.0f * logf(opacity * 255.0f);
  return q * 1.0005f + 0.01f;
}

GS_HD bool rect_may_contribute(float x, float y, float A, float B, float C, float qthr,
                               float rx0, float ry0, float rx1, float ry1) {
  if (qthr < 0.f) return false;
  float dx0 = rx0 - x, dx1 = rx1 - x, dy0 = ry0 - y, dy1 = ry1 - y;
  bool inx = (dx0 <= 0.f) && (dx1 >= 0.f);
  bool iny = (dy0 <= 0.f) && (dy1 >= 0.f);
  if (inx && iny) return true;
  // The 1-D minimiser along an edge only has to be approximately right: q evaluated at any point of the
  // edge is >= the true minimum, an error delta in the minimiser costs C*delta^2 (~1e-12 relative), far inside
  // the safety margin of cull_threshold().  So the fast (MUFU.RCP based) division is enough on the device.
  float qmin = 3.0e38f;
  if (!inx) {
    float ex = dx0 > 0.f ? dx0 : dx1;
    float dy = fminf(dy1, fmaxf(dy0, gs_fdiv(-B * ex, C)));
    qmin = A * ex * ex + 2.f * B * ex * dy + C * dy * dy;
  }
  if (!iny) {
    float ey = dy0 > 0.f ? dy0 : dy1;
    float dx = fminf(dx1, fmaxf(dx0, gs_fdiv(-B * ey, A)));
    float q = A * dx * dx + 2.f * B * dx * ey + C * ey * ey;
    qmin = fminf(qmin, q);
  }
  return !(qmin > qthr);       // NaN -> keep
}

// The same predicate for a whole tile ROW at once.  The kept tiles of a row are those whose pixel-centre span
// [16 tx, 16 tx + 15] meets the x-extent of (ellipse q <= qthr) intersected with the row's band of pixel centres -- in
// exact arithmetic precisely the tiles for which the minimum of q over the tile's rectangle of pixel centres is <= qthr
// (the ellipse cut by the band is convex, so its x-projection is an interval).  The extent of the cut is the ellipse's
// own extreme point (dx = +-hx at dy = -+B hx / C) when that lies inside the band, else the outer root of
// q(dx, dy_end) = qthr at one of the band's two ends: two square roots per row instead of one rectangle test per tile.
// The interval is widened by kRowEps pixels: a false positive only costs a list entry (the blend applies the exact
// per-pair rule), a false negative would lose a contribution.  ok == false (degenerate conic): use the per-tile test.
constexpr float kRowEps = 0.02f;
struct RowCull { float x, y, B, det, aq, invA, hx, hy, dyR; bool ok; };
GS_HD RowCull row_cull_setup(float x, float y, float A, float B, float C, float qthr) {
  RowCull r;
  r.x = x; r.y = y; r.B = B;
  r.det = A * C - B * B;
  r.ok = (r.det > 0.f) && (A > 0.f) && (C > 0.f) && (qthr >= 0.f);
  const float rdet = 1.0f / r.det;
  r.hx = sqrtf(qthr * C * rdet);
  r.hy = sqrtf(qthr * A * rdet) + kRowEps;
  r.dyR = -B * r.hx / C;                                  // dy of the rightmost point (the leftmost one is at -dyR)
  r.invA = 1.0f / A;
  r.aq = A * qthr;
  return r;
}
// tiles [ta, tb] of row ty (clipped to [rx0, rx1)) are kept; returns false when the row keeps nothing
GS_HD bool row_keep_range(const RowCull& r, int ty, int H, int rx0, int rx1, int& ta, int& tb) {
  const float y0 = (float)(ty * kBlock), y1 = fminf(y0 + (float)(kBlock - 1), (float)(H - 1));
  const float lo = fmaxf(y0 - r.y, -r.hy), hi = fminf(y1 - r.y, r.hy);
  if (lo > hi) return false;                              // the band misses the ellipse
  const float slo = sqrtf(fmaxf(0.f, r.aq - r.det * lo * lo)), shi = sqrtf(fmaxf(0.f, r.aq - r.det * hi * hi));
  const float blo = -r.B * lo, bhi = -r.B * hi;
  const float xr = (r.dyR >= lo && r.dyR <= hi) ? r.hx : fmaxf(blo + slo, bhi + shi) * r.invA;
  const float xl = (-r.dyR >= lo && -r.dyR <= hi) ? -r.hx : fminf(blo - slo, bhi - shi) * r.invA;
  const float XL = r.x + xl - kRowEps, XR = r.x + xr + kRowEps;
  // tile tx meets [XL, XR]  <=>  16 tx <= XR  and  16 tx + 15 >= XL
  const float fa = ceilf((XL - (float)(kBlock - 1)) * (1.0f / kBlock)), fb = floorf(XR * (1.0f / kBlock));
  ta = fa > (float)rx0 ? (int)fminf(fa, 1.0e6f) : rx0;
  tb = fb < (float)(rx1 - 1) ? (int)fmaxf(fb, -1.0e6f) : rx1 - 1;
  return tb >= ta;
}

// ------------------------------------------------------------------------------------------
// Per-Gaussian backward (Appendix A.3).  dsplat = accumulated over pixels:
//   [0,1] dL/d(pixel x,y)   [2,3,4] dL/dA, dL/dB (full), dL/dC   [5] dL/dopacity(activated)
//   [6,7,8] dL/drgb
// Outputs are gradients w.r.t. the kernel INPUTS (world xyz / raw quaternion / log-scale / logit
// when the fused modes are on).  pose_acc (16 floats) receives this Gaussian's contribution to
// [dqc_raw(4), dt(3), dRc(9)].
// ------------------------------------------------------------------------------------------
struct GaussGrad {
  float dm[3], dsc[3], dq[4], dop;
  float dmeans2D[2];    // dL/d(ndc)
  float dcov3D[6];      // only meaningful with cov3D_precomp
  float dcolor[3];      // dL/drgb after the clamp mask (colors_precomp path)
};

// kAcc: the SH gradient is added to d_sh_dc / d_sh_rest (sh_to_rgb_bwd<true>); everything else is unchanged
template <bool kMip = false, bool kAcc = false>
GS_HD void project_bwd(const CamConst& c, const GaussIn& in, const Proj& p, const float* sh_rest,
                       bool use_sh, bool cov_pre, const float* ds, GaussGrad& g, float* d_sh_dc,
                       float* d_sh_rest, float* pose_acc, const Mip mf = Mip()) {
  float dmc[3] = {0.f, 0.f, 0.f};
  // ---- colour
  float dL[3] = {ds[6], ds[7], ds[8]};
  for (int ch = 0; ch < 3; ++ch)
    if (p.clamped & (1u << ch)) dL[ch] = 0.f;
  g.dcolor[0] = dL[0]; g.dcolor[1] = dL[1]; g.dcolor[2] = dL[2];
  if (use_sh) {
    float vx = p.mc[0] - c.campos[0], vy = p.mc[1] - c.campos[1], vz = p.mc[2] - c.campos[2];
    float inv = 1.f / sqrtf(vx * vx + vy * vy + vz * vz);
    float dx = vx * inv, dy = vy * inv, dz = vz * inv;
    float ddir[3];
    sh_to_rgb_bwd<kAcc>(c.D, sh_rest, dx, dy, dz, dL, d_sh_dc, d_sh_rest, ddir);
    float dot = dx * ddir[0] + dy * ddir[1] + dz * ddir[2];
    dmc[0] += (ddir[0] - dx * dot) * inv;
    dmc[1] += (ddir[1] - dy * dot) * inv;
    dmc[2] += (ddir[2] - dz * dot) * inv;
  }
  // ---- conic -> cov2D
  float a = p.a, b = p.b, cc = p.c, det = p.det;
  float d2i = 1.0f / (det * det + 0.0000001f);
  float dA = ds[2], dB = ds[3], dC = ds[4];
  float dL_da = d2i * (-cc * cc * dA + b * cc * dB - b * b * dC);
  float dL_dc = d2i * (-a * a * dC + a * b * dB - b * b * dA);
  float dL_db = d2i * (2.f * b * cc * dA - (det + 2.f * b * b) * dB + 2.f * a * b * dC);
  if (kMip && mf.on2d && !p.h2clamp) {
    // o_eff = o3 h2, h2 = sqrt(r), r = det0 / det: dL/dr = dL/do_eff * o3 / (2 h2), chained to (a0, b, c0)
    const float dr = ds[5] * p.o3 * 0.5f / p.h2, i2 = dr / (det * det);
    dL_da += (p.c0 * det - p.det0 * cc) * i2;
    dL_dc += (p.a0 * det - p.det0 * a) * i2;
    dL_db += -2.f * b * (det - p.det0) * i2;
  }
  // ---- cov2D = T Sigma T^T
  const float* T = p.T;
  const float* S = p.Sig;
  float hb = 0.5f * dL_db;
  // dSigma (full symmetric matrix gradient) = T^T G T
  float dS[6];
  dS[0] = T[0] * T[0] * dL_da + 2.f * T[0] * T[3] * hb + T[3] * T[3] * dL_dc;
  dS[3] = T[1] * T[1] * dL_da + 2.f * T[1] * T[4] * hb + T[4] * T[4] * dL_dc;
  dS[5] = T[2] * T[2] * dL_da + 2.f * T[2] * T[5] * hb + T[5] * T[5] * dL_dc;
  dS[1] = T[0] * T[1] * dL_da + (T[0] * T[4] + T[3] * T[1]) * hb + T[3] * T[4] * dL_dc;
  dS[2] = T[0] * T[2] * dL_da + (T[0] * T[5] + T[3] * T[2]) * hb + T[3] * T[5] * dL_dc;
  dS[4] = T[1] * T[2] * dL_da + (T[1] * T[5] + T[4] * T[2]) * hb + T[4] * T[5] * dL_dc;
  g.dcov3D[0] = dS[0]; g.dcov3D[1] = 2.f * dS[1]; g.dcov3D[2] = 2.f * dS[2];
  g.dcov3D[3] = dS[3]; g.dcov3D[4] = 2.f * dS[4]; g.dcov3D[5] = dS[5];
  // dT = 2 G T Sigma  (2x3);  u_r = Sigma T_r
  float u0[3] = {S[0] * T[0] + S[1] * T[1] + S[2] * T[2], S[1] * T[0] + S[3] * T[1] + S[4] * T[2],
                 S[2] * T[0] + S[4] * T[1] + S[5] * T[2]};
  float u1[3] = {S[0] * T[3] + S[1] * T[4] + S[2] * T[5], S[1] * T[3] + S[3] * T[4] + S[4] * T[5],
                 S[2] * T[3] + S[4] * T[4] + S[5] * T[5]};
  float dT[6];
  for (int i = 0; i < 3; ++i) {
    dT[i]     = 2.f * (dL_da * u0[i] + hb * u1[i]);
    dT[3 + i] = 2.f * (hb * u0[i] + dL_dc * u1[i]);
  }
  // dJ[r][j] = sum_i dT[r][i] * Wr[j][i] = sum_i dT[r][i] * V[4*i + j]
  float dJ00 = dT[0] * c.V[0] + dT[1] * c.V[4] + dT[2] * c.V[8];
  float dJ02 = dT[0] * c.V[2] + dT[1] * c.V[6] + dT[2] * c.V[10];
  float dJ11 = dT[3] * c.V[1] + dT[4] * c.V[5] + dT[5] * c.V[9];
  float dJ12 = dT[3] * c.V[2] + dT[4] * c.V[6] + dT[5] * c.V[10];
  float tz = p.t[2], tz2 = 1.f / (tz * tz), tz3 = tz2 / tz;
  float dtx = p.clx ? 0.f : -c.fx * tz2 * dJ02;
  float dty = p.cly ? 0.f : -c.fy * tz2 * dJ12;
  float dtz = -c.fx * tz2 * dJ00 - c.fy * tz2 * dJ11 + 2.f * c.fx * p.t[0] * tz3 * dJ02 +
              2.f * c.fy * p.t[1] * tz3 * dJ12;
  // view transform transpose: dm_i += sum_j V[4*i + j] * dt_j
  for (int i = 0; i < 3; ++i)
    dmc[i] += c.V[4 * i + 0] * dtx + c.V[4 * i + 1] * dty + c.V[4 * i + 2] * dtz;
  // ---- pixel position
  float dnx = ds[0] * 0.5f * c.W, dny = ds[1] * 0.5f * c.H;
  g.dmeans2D[0] = dnx; g.dmeans2D[1] = dny;
  float dhx = dnx * p.p_w, dhy = dny * p.p_w;
  float dhw = -(dnx * p.hom[0] + dny * p.hom[1]) * p.p_w * p.p_w;
  for (int i = 0; i < 3; ++i)
    dmc[i] += c.Pm[4 * i + 0] * dhx + c.Pm[4 * i + 1] * dhy + c.Pm[4 * i + 3] * dhw;
  // ---- cov3D -> scale, quaternion
  float dq[4] = {0.f, 0.f, 0.f, 0.f};
  float dsc[3] = {0.f, 0.f, 0.f};
  if (!cov_pre) {
    float R[9];
    quat_to_R(p.q[0], p.q[1], p.q[2], p.q[3], R);
    // dM = 2 dSigma M,  M[i][j] = R[i][j] s[j]
    float dSf[9] = {dS[0], dS[1], dS[2], dS[1], dS[3], dS[4], dS[2], dS[4], dS[5]};
    float dR[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        float dM = 2.f * (dSf[3 * i + 0] * R[0 + j] * p.s[j] + dSf[3 * i + 1] * R[3 + j] * p.s[j] +
                          dSf[3 * i + 2] * R[6 + j] * p.s[j]);
        dsc[j] += dM * R[3 * i + j];
        dR[3 * i + j] = dM * p.s[j];
      }
    quat_to_R_bwd(p.q[0], p.q[1], p.q[2], p.q[3], dR, dq);
  }
  // ---- activations
  float dop = ds[5];
  if (kMip && mf.on) {
    // o_eff = sig * h3 * h2 (h3 = prod_k s_k / s~_k with the 3D filter, else 1); neither filter's f or kappa is trained
    const float dsig = dop * p.h2 * p.h3;
    if (c.raw_params && mf.on3d && mf.f != 0.f) {
      // o.s = mod * s~, s~^2 = s^2 + f^2, s = exp(sc):  d(mod s~)/dsc = o.s * s^2 / s~^2,  dh3/dsc = h3 f^2 / s~^2
      const float f2 = mf.f * mf.f, dh3 = dop * p.h2 * p.sig * p.h3;
      for (int k = 0; k < 3; ++k) {
        const float s = expf(in.sc[k]), v = s * s + f2;
        g.dsc[k] = dsc[k] * p.s[k] * ((s * s) / v) + dh3 * (f2 / v);
      }
    } else if (c.raw_params) {
      g.dsc[0] = dsc[0] * p.s[0]; g.dsc[1] = dsc[1] * p.s[1]; g.dsc[2] = dsc[2] * p.s[2];
    } else {
      g.dsc[0] = dsc[0] * c.scale_mod; g.dsc[1] = dsc[1] * c.scale_mod; g.dsc[2] = dsc[2] * c.scale_mod;
    }
    g.dop = c.raw_params ? dsig * p.sig * (1.f - p.sig) : dsig;
  } else if (c.raw_params) {
    // s = mod * exp(sc): ds/dsc = s ; (dsc[] currently holds dL/ds)
    g.dsc[0] = dsc[0] * p.s[0]; g.dsc[1] = dsc[1] * p.s[1]; g.dsc[2] = dsc[2] * p.s[2];
    g.dop = dop * p.opacity * (1.f - p.opacity);
  } else {
    g.dsc[0] = dsc[0] * c.scale_mod; g.dsc[1] = dsc[1] * c.scale_mod; g.dsc[2] = dsc[2] * c.scale_mod;
    g.dop = dop;
  }
  // ---- pose pre-transform
  if (c.pose_on) {
    for (int i = 0; i < 3; ++i)
      g.dm[i] = c.Rc[0 + i] * dmc[0] + c.Rc[3 + i] * dmc[1] + c.Rc[6 + i] * dmc[2];
    float w1 = c.qc[0], x1 = c.qc[1], y1 = c.qc[2], z1 = c.qc[3];
    float w2 = in.q[0], x2 = in.q[1], y2 = in.q[2], z2 = in.q[3];
    g.dq[0] = w1 * dq[0] + x1 * dq[1] + y1 * dq[2] + z1 * dq[3];
    g.dq[1] = -x1 * dq[0] + w1 * dq[1] + z1 * dq[2] - y1 * dq[3];
    g.dq[2] = -y1 * dq[0] - z1 * dq[1] + w1 * dq[2] + x1 * dq[3];
    g.dq[3] = -z1 * dq[0] + y1 * dq[1] - x1 * dq[2] + w1 * dq[3];
    pose_acc[0] = w2 * dq[0] + x2 * dq[1] + y2 * dq[2] + z2 * dq[3];
    pose_acc[1] = -x2 * dq[0] + w2 * dq[1] - z2 * dq[2] + y2 * dq[3];
    pose_acc[2] = -y2 * dq[0] + z2 * dq[1] + w2 * dq[2] - x2 * dq[3];
    pose_acc[3] = -z2 * dq[0] - y2 * dq[1] + x2 * dq[2] + w2 * dq[3];
    pose_acc[4] = dmc[0]; pose_acc[5] = dmc[1]; pose_acc[6] = dmc[2];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) pose_acc[7 + 3 * i + j] = dmc[i] * in.m[j];
  } else {
    g.dm[0] = dmc[0]; g.dm[1] = dmc[1]; g.dm[2] = dmc[2];
    g.dq[0] = dq[0]; g.dq[1] = dq[1]; g.dq[2] = dq[2]; g.dq[3] = dq[3];
  }
}

#if defined(__CUDACC__)
// Lane-wise float2 arithmetic, rounded like the scalar __f*_rn intrinsics (never contracted), used where the blend and
// loss kernels carry two pixels or two statistics per register pair.  sm_90 has no packed FP32x2 instructions, so each
// call issues two FFMA / FMUL / FADD.
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
#endif

}  // namespace gsb
