// CPU harness for the Mip-Splatting arithmetic of instantsplat_b200/csrc/gs_math.cuh (the kMip instantiations of
// project_geometry / project_bwd and mip_view_depth), compiled for the host by g++ in tests/test_mip_cpu.py.  It builds on
// the camera helper of tests/host_math.cpp.  Test utility only.
#include "host_math.cpp"

extern "C" {

static Mip host_mip(int on2d, float kappa, const float* f3d, int i) {
  Mip m;
  m.on2d = on2d; m.kappa = kappa; m.on3d = f3d != nullptr; m.f = f3d ? f3d[i] : 0.f;
  m.on = m.on2d || m.on3d;
  return m;
}

static GaussIn host_in(const float* means, const float* scales, const float* rots, const float* opac, int i) {
  GaussIn in;
  for (int k = 0; k < 3; ++k) { in.m[k] = means[3 * i + k]; in.sc[k] = scales[3 * i + k]; }
  for (int k = 0; k < 4; ++k) in.q[k] = rots[4 * i + k];
  in.op = opac[i];
  return in;
}

// out_geom [P,12] as host_project; out_h2 [P,2]: h2, clamp flag
void host_project_mip(const HostCam* h, int P, const float* means, const float* scales, const float* rots,
                      const float* opac, const float* sh_dc, const float* sh_rest, int on2d, float kappa,
                      const float* f3d, float* out_geom, float* out_h2) {
  CamConst c; fill(h, c);
  for (int i = 0; i < P; ++i) {
    GaussIn in = host_in(means, scales, rots, opac, i);
    Proj p;
    std::memset(&p, 0, sizeof(p));
    project_geometry<true>(c, in, nullptr, p, host_mip(on2d, kappa, f3d, i));
    if (p.visible) project_color(c, sh_dc + 3 * i, sh_rest + (size_t)3 * (c.M - 1) * i, p);
    float* o = out_geom + 12 * i;
    o[0] = p.x; o[1] = p.y; o[2] = p.A; o[3] = p.B; o[4] = p.C; o[5] = p.opacity; o[6] = p.depth;
    o[7] = p.rgb[0]; o[8] = p.rgb[1]; o[9] = p.rgb[2]; o[10] = (float)p.radius; o[11] = (float)p.visible;
    out_h2[2 * i] = p.h2; out_h2[2 * i + 1] = (float)p.h2clamp;
  }
}

// dsplat [P,9] -> dm [P,3], dsc [P,3], dq [P,4], dop [P], dpose [7]
void host_project_bwd_mip(const HostCam* h, int P, const float* means, const float* scales, const float* rots,
                          const float* opac, const float* sh_dc, const float* sh_rest, int on2d, float kappa,
                          const float* f3d, const float* dsplat, float* dm, float* dsc, float* dq, float* dop,
                          float* dpose) {
  CamConst c; fill(h, c);
  double acc[16] = {0};
  for (int i = 0; i < P; ++i) {
    GaussIn in = host_in(means, scales, rots, opac, i);
    const Mip mf = host_mip(on2d, kappa, f3d, i);
    Proj p;
    std::memset(&p, 0, sizeof(p));
    project_geometry<true>(c, in, nullptr, p, mf);
    for (int k = 0; k < 3; ++k) { dm[3 * i + k] = 0.f; dsc[3 * i + k] = 0.f; }
    for (int k = 0; k < 4; ++k) dq[4 * i + k] = 0.f;
    dop[i] = 0.f;
    if (!p.visible) continue;
    const float* rest_in = sh_rest + (size_t)3 * (c.M - 1) * i;
    project_color(c, sh_dc + 3 * i, rest_in, p);
    GaussGrad g;
    float pa[16] = {0}, ddc[3], drest[45];
    for (int k = 0; k < 45; ++k) drest[k] = 0.f;
    project_bwd<true>(c, in, p, rest_in, true, false, dsplat + 9 * i, g, ddc, drest, pa, mf);
    for (int k = 0; k < 3; ++k) { dm[3 * i + k] = g.dm[k]; dsc[3 * i + k] = g.dsc[k]; }
    for (int k = 0; k < 4; ++k) dq[4 * i + k] = g.dq[k];
    dop[i] = g.dop;
    for (int k = 0; k < 16; ++k) acc[k] += pa[k];
  }
  float accf[16];
  for (int k = 0; k < 16; ++k) accf[k] = (float)acc[k];
  pose_grad_finalize(h->pose, accf, dpose);
}

// poses [V,7]: out [P] = smallest mip_view_depth over the views (-1: none counts)
void host_mip_depth(int P, const float* xyz, int V, const float* poses, float fx, float fy, int W, int H, float* out) {
  for (int i = 0; i < P; ++i) {
    float d = 3.0e38f;
    for (int v = 0; v < V; ++v) {
      const float* q = poses + 7 * v;
      const float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
      float R[9];
      quat_to_R(q[0] / n, q[1] / n, q[2] / n, q[3] / n, R);
      const float z = mip_view_depth(R, q + 4, xyz + 3 * i, fx, fy, W, H);
      if (z >= 0.f) d = fminf(d, z);
    }
    out[i] = d < 3.0e38f ? d : -1.f;
  }
}
}
