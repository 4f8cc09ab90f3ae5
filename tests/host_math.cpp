// CPU harness around instantsplat_b200/csrc/gs_math.cuh: runs the SAME per-Gaussian forward /
// backward arithmetic the sm_90a kernels inline, on the host, so the algebra can be checked
// against the oracle without a GPU (tests/test_host_math.py).  Test utility only -- it is not
// part of the product library and is never loaded by instantsplat_b200.
#include <cstring>
#include <vector>

#include "../instantsplat_b200/csrc/gs_math.cuh"

using namespace gsb;

extern "C" {

struct HostCam {
  int W, H, D, M, pose_on, raw_params;
  float tanfovx, tanfovy, scale_mod;
  float V[16], Pm[16], campos[3], pose[7];
};

static void fill(const HostCam* h, CamConst& c) {
  std::memcpy(c.V, h->V, sizeof(c.V));
  std::memcpy(c.Pm, h->Pm, sizeof(c.Pm));
  std::memcpy(c.campos, h->campos, sizeof(c.campos));
  c.tanfovx = h->tanfovx; c.tanfovy = h->tanfovy;
  c.W = h->W; c.H = h->H;
  c.fx = h->W / (2.0f * h->tanfovx); c.fy = h->H / (2.0f * h->tanfovy);
  c.scale_mod = h->scale_mod;
  c.gx = (h->W + kBlock - 1) / kBlock; c.gy = (h->H + kBlock - 1) / kBlock;
  c.D = h->D; c.M = h->M; c.raw_params = h->raw_params; c.pose_on = 0;
  if (h->pose_on) pose_to_const(h->pose, c);
}

// out_geom [P,12]: x,y,A,B,C,opacity,depth,r,g,b,radius,visible ; out_rect [P,4] ; clamped [P]
void host_project(const HostCam* h, int P, const float* means, const float* scales,
                  const float* rots, const float* opac, const float* sh_dc, const float* sh_rest,
                  float* out_geom, int* out_rect, int* out_clamped) {
  CamConst c; fill(h, c);
  for (int i = 0; i < P; ++i) {
    GaussIn in;
    for (int k = 0; k < 3; ++k) { in.m[k] = means[3 * i + k]; in.sc[k] = scales[3 * i + k]; }
    for (int k = 0; k < 4; ++k) in.q[k] = rots[4 * i + k];
    in.op = opac[i];
    Proj p;
    std::memset(&p, 0, sizeof(p));
    project_geometry(c, in, nullptr, p);
    if (p.visible) project_color(c, sh_dc + 3 * i, sh_rest + (size_t)3 * (c.M - 1) * i, p);
    float* o = out_geom + 12 * i;
    o[0] = p.x; o[1] = p.y; o[2] = p.A; o[3] = p.B; o[4] = p.C; o[5] = p.opacity; o[6] = p.depth;
    o[7] = p.rgb[0]; o[8] = p.rgb[1]; o[9] = p.rgb[2]; o[10] = (float)p.radius; o[11] = (float)p.visible;
    out_rect[4 * i] = p.rx0; out_rect[4 * i + 1] = p.ry0; out_rect[4 * i + 2] = p.rx1; out_rect[4 * i + 3] = p.ry1;
    out_clamped[i] = (int)p.clamped;
  }
}

// dsplat [P,9] -> grads: dm [P,3], dsc [P,3], dq [P,4], dop [P], dsh_dc [P,3], dsh_rest [P,M-1,3],
// dmeans2D [P,2], dpose [7]
void host_project_bwd(const HostCam* h, int P, const float* means, const float* scales,
                      const float* rots, const float* opac, const float* sh_dc, const float* sh_rest,
                      const float* dsplat, float* dm, float* dsc, float* dq, float* dop,
                      float* dsh_dc, float* dsh_rest, float* dmeans2D, float* dpose) {
  CamConst c; fill(h, c);
  double acc[16] = {0};
  int K = (c.D + 1) * (c.D + 1);
  for (int i = 0; i < P; ++i) {
    GaussIn in;
    for (int k = 0; k < 3; ++k) { in.m[k] = means[3 * i + k]; in.sc[k] = scales[3 * i + k]; }
    for (int k = 0; k < 4; ++k) in.q[k] = rots[4 * i + k];
    in.op = opac[i];
    Proj p;
    std::memset(&p, 0, sizeof(p));
    project_geometry(c, in, nullptr, p);
    float* rest_out = dsh_rest + (size_t)3 * (c.M - 1) * i;
    for (int k = 0; k < 3 * (c.M - 1); ++k) rest_out[k] = 0.f;
    if (!p.visible) {
      for (int k = 0; k < 3; ++k) { dm[3 * i + k] = 0; dsc[3 * i + k] = 0; dsh_dc[3 * i + k] = 0; }
      for (int k = 0; k < 4; ++k) dq[4 * i + k] = 0;
      dop[i] = 0; dmeans2D[2 * i] = dmeans2D[2 * i + 1] = 0;
      continue;
    }
    const float* rest_in = sh_rest + (size_t)3 * (c.M - 1) * i;
    project_color(c, sh_dc + 3 * i, rest_in, p);
    GaussGrad g;
    float pa[16] = {0};
    float drest[45];
    for (int k = 0; k < 45; ++k) drest[k] = 0.f;
    project_bwd(c, in, p, rest_in, true, false, dsplat + 9 * i, g, dsh_dc + 3 * i, drest, pa);
    for (int k = 0; k < 3 * (K - 1); ++k) rest_out[k] = drest[k];
    for (int k = 0; k < 3; ++k) { dm[3 * i + k] = g.dm[k]; dsc[3 * i + k] = g.dsc[k]; }
    for (int k = 0; k < 4; ++k) dq[4 * i + k] = g.dq[k];
    dop[i] = g.dop; dmeans2D[2 * i] = g.dmeans2D[0]; dmeans2D[2 * i + 1] = g.dmeans2D[1];
    for (int k = 0; k < 16; ++k) acc[k] += pa[k];
  }
  if (c.pose_on) {
    float accf[16];
    for (int k = 0; k < 16; ++k) accf[k] = (float)acc[k];
    pose_grad_finalize(h->pose, accf, dpose);
  }
}

// pose_grad_finalize alone: acc [16] = [dqc_raw(4), dt(3), dRc(9)] -> dpose [7]
void host_pose_grad_finalize(const float* pose, const float* acc, float* dpose) { pose_grad_finalize(pose, acc, dpose); }

// rect_may_contribute brute-force check helper: returns 1 if the predicate says "may contribute"
int host_rect_may_contribute(float x, float y, float A, float B, float C, float opacity, float rx0,
                             float ry0, float rx1, float ry1) {
  return rect_may_contribute(x, y, A, B, C, cull_threshold(opacity), rx0, ry0, rx1, ry1) ? 1 : 0;
}

// Row form of the same predicate (row_keep_range): kept[(ty - ry0) * (rx1 - rx0) + (tx - rx0)] = 1 for the kept tiles
// of the tile rect [rx0, rx1) x [ry0, ry1) on an image of height H.  Returns 0 if the conic is degenerate.
int host_row_keep(float x, float y, float A, float B, float C, float opacity, int H, int rx0, int ry0, int rx1, int ry1,
                  int* kept) {
  const RowCull rc = row_cull_setup(x, y, A, B, C, cull_threshold(opacity));
  for (int k = 0; k < (rx1 - rx0) * (ry1 - ry0); ++k) kept[k] = 0;
  if (!rc.ok) return 0;
  for (int ty = ry0; ty < ry1; ++ty) {
    int ta, tb;
    if (!row_keep_range(rc, ty, H, rx0, rx1, ta, tb)) continue;
    for (int tx = ta; tx <= tb; ++tx) kept[(ty - ry0) * (rx1 - rx0) + (tx - rx0)] = 1;
  }
  return 1;
}

// The culls as the kernels call them, on a conic and threshold already in the log2 domain (k_preprocess's SplatRect,
// the blend's slab entry).  cull_threshold alone:
float host_cull_threshold(float opacity) { return cull_threshold(opacity); }

// rect_may_contribute over n pixel-centre rectangles rects[4 k .. 4 k + 3] = x0, y0, x1, y1 -> keep[k]
void host_rect_keep_many(float x, float y, float A, float B, float C, float qthr, int n, const float* rects,
                         int* keep) {
  for (int k = 0; k < n; ++k) {
    const float* r = rects + 4 * k;
    keep[k] = rect_may_contribute(x, y, A, B, C, qthr, r[0], r[1], r[2], r[3]) ? 1 : 0;
  }
}

// tighten_cull_rect on the tile rect rect[4] = rx0, ry0, rx1, ry1 (in place)
void host_tighten_cull_rect(float x, float y, float A, float B, float C, float qthr, int* rect) {
  tighten_cull_rect(x, y, A, B, C, qthr, rect[0], rect[1], rect[2], rect[3]);
}

// row_keep_range for tile rows ry0 .. ry1 - 1 of the tile rect [rx0, rx1): row ry0 + k keeps tiles ta[k] .. tb[k]
// (ta > tb: none).  Returns 0 when row_cull_setup falls back to the per-tile test (nothing is written then).
int host_row_ranges(float x, float y, float A, float B, float C, float qthr, int H, int rx0, int ry0, int rx1, int ry1,
                    int* ta, int* tb) {
  const RowCull rc = row_cull_setup(x, y, A, B, C, qthr);
  if (!rc.ok) return 0;
  for (int ty = ry0; ty < ry1; ++ty) {
    int a, b;
    if (!row_keep_range(rc, ty, H, rx0, rx1, a, b)) { a = 1; b = 0; }
    ta[ty - ry0] = a;
    tb[ty - ry0] = b;
  }
  return 1;
}
}
