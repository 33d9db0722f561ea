// Point geometry shared by both MLP engines: camera transform, projection into a source view,
// bilinear tap selection (grid_sample align_corners=True / border) and the 42 geometric input
// channels.  Written with explicit round-to-nearest intrinsics (no FMA contraction) so that
// every translation unit produces the same bits as the reference's op-by-op torch code
// (src/model/models.py:158-212, src/model/code.py:30-42, src/model/encoder.py:96-108).
#pragma once
#include <math.h>

#include "pnr_common.cuh"

namespace pnr {

struct PointGeom {
  float q[3];    // R x            (z_feature input, normalize_z: models.py:171)
  float dcam[3]; // R dir          (models.py:188-193)
  float w_nw, w_ne, w_sw, w_se;
  int x0, y0, x1, y1;
};

__device__ __forceinline__ void load_point(const PointSource& src, int64_t g, float x[3], float d[3]) {
  if (src.mode == 0) {
    for (int i = 0; i < 3; ++i) {
      x[i] = src.xyz[g * 3 + i];
      d[i] = src.dirs ? src.dirs[g * 3 + i] : 0.f;
    }
  } else {
    int64_t ray = g / src.K;
    int k = (int)(g - ray * src.K);
    const float* rr = src.rays + ray * 8;
    float zz = src.z[ray * src.K + k];
    for (int i = 0; i < 3; ++i) {
      d[i] = rr[3 + i];
      x[i] = __fadd_rn(rr[i], __fmul_rn(zz, d[i]));  // nerf.py:185
    }
  }
}

__device__ __forceinline__ PointGeom point_geometry(const PnrScene& sc, int sb, int v, const float x[3],
                                                    const float d[3]) {
  PointGeom g;
  const float* M = sc.poses + (size_t)(sb * sc.NS + v) * 12;
  float p[3];
  for (int i = 0; i < 3; ++i) {
    g.q[i] = __fadd_rn(__fadd_rn(__fmul_rn(M[i * 4 + 0], x[0]), __fmul_rn(M[i * 4 + 1], x[1])), __fmul_rn(M[i * 4 + 2], x[2]));
    p[i] = __fadd_rn(g.q[i], M[i * 4 + 3]);
    g.dcam[i] = __fadd_rn(__fadd_rn(__fmul_rn(M[i * 4 + 0], d[0]), __fmul_rn(M[i * 4 + 1], d[1])), __fmul_rn(M[i * 4 + 2], d[2]));
  }
  const float* fo = sc.focal + (sc.n_focal > 1 ? sb * 2 : 0);
  const float* cc = sc.c + (sc.n_c > 1 ? sb * 2 : 0);
  float u = __fadd_rn(__fmul_rn(__fdiv_rn(-p[0], p[2]), fo[0]), cc[0]);   // models.py:206-212
  float w = __fadd_rn(__fmul_rn(__fdiv_rn(-p[1], p[2]), fo[1]), cc[1]);
  // encoder.py:96-99: uv * (latent_scaling / image_size) - 1
  float gx = __fsub_rn(__fmul_rn(u, __fdiv_rn(sc.scale_x, sc.image_w)), 1.0f);
  float gy = __fsub_rn(__fmul_rn(w, __fdiv_rn(sc.scale_y, sc.image_h)), 1.0f);
  // grid_sample(align_corners=True): ((g + 1) / 2) * (size - 1), then border clip
  float ix = __fmul_rn(__fdiv_rn(__fadd_rn(gx, 1.0f), 2.0f), (float)(sc.Wl - 1));
  float iy = __fmul_rn(__fdiv_rn(__fadd_rn(gy, 1.0f), 2.0f), (float)(sc.Hl - 1));
  ix = fminf((float)(sc.Wl - 1), fmaxf(ix, 0.f));
  iy = fminf((float)(sc.Hl - 1), fmaxf(iy, 0.f));
  // NaN coordinates (point exactly on a camera plane) clip to 0 like ATen's clip_coordinates
  if (!(ix == ix)) ix = 0.f;
  if (!(iy == iy)) iy = 0.f;
  float x0 = floorf(ix), y0 = floorf(iy);
  float x1 = x0 + 1.0f, y1 = y0 + 1.0f;
  g.w_nw = __fmul_rn(x1 - ix, y1 - iy);
  g.w_ne = __fmul_rn(ix - x0, y1 - iy);
  g.w_sw = __fmul_rn(x1 - ix, iy - y0);
  g.w_se = __fmul_rn(ix - x0, iy - y0);
  g.x0 = (int)x0;
  g.y0 = (int)y0;
  g.x1 = min((int)x1, sc.Wl - 1);  // out-of-range taps carry weight 0
  g.y1 = min((int)y1, sc.Hl - 1);
  if ((int)x1 > sc.Wl - 1) { g.w_ne = 0.f; g.w_se = 0.f; }
  if ((int)y1 > sc.Hl - 1) { g.w_sw = 0.f; g.w_se = 0.f; }
  return g;
}

// The bilinear taps of point x in view v of object sb as k_geom_bwd (pnr_field_bwd.cu) computes them, with the
// backward's contractible arithmetic rather than point_geometry's; the fixed-point latent scatter of pnr_determ.cu
// uses them.  k_geom_bwd keeps its own inline copy, so the default path's code is unchanged.
struct BwdTaps {
  bool vx1, vy1;                   // the second tap of x / y lies inside the map (taps outside carry nothing)
  float w_nw, w_ne, w_sw, w_se;
  size_t o_nw, o_ne, o_sw, o_se;   // channels-last offsets of the four taps into the latent
};

__device__ __forceinline__ BwdTaps bwd_taps(const PnrScene& sc, int sb, int v, const float x[3]) {
  const float* M = sc.poses + (size_t)(sb * sc.NS + v) * 12;
  float q[3], p[3];
  for (int i = 0; i < 3; ++i) {
    q[i] = M[i * 4 + 0] * x[0] + M[i * 4 + 1] * x[1] + M[i * 4 + 2] * x[2];
    p[i] = q[i] + M[i * 4 + 3];
  }
  const float* fo = sc.focal + (sc.n_focal > 1 ? sb * 2 : 0);
  const float* cc = sc.c + (sc.n_c > 1 ? sb * 2 : 0);
  const float u = (-p[0] / p[2]) * fo[0] + cc[0];
  const float w = (-p[1] / p[2]) * fo[1] + cc[1];
  const int C = sc.C, Wl = sc.Wl, Hl = sc.Hl;
  const float kx = sc.scale_x / sc.image_w, ky = sc.scale_y / sc.image_h;
  const float ix_u = ((u * kx - 1.0f) + 1.0f) * 0.5f * (float)(Wl - 1);
  const float iy_u = ((w * ky - 1.0f) + 1.0f) * 0.5f * (float)(Hl - 1);
  float ix = fminf((float)(Wl - 1), fmaxf(ix_u, 0.f));
  float iy = fminf((float)(Hl - 1), fmaxf(iy_u, 0.f));
  if (!(ix == ix)) ix = 0.f;
  if (!(iy == iy)) iy = 0.f;
  const float x0f = floorf(ix), y0f = floorf(iy);
  const int x0 = (int)x0f, y0 = (int)y0f;
  BwdTaps t;
  t.vx1 = (x0 + 1 <= Wl - 1);
  t.vy1 = (y0 + 1 <= Hl - 1);
  const int x1 = t.vx1 ? x0 + 1 : x0, y1 = t.vy1 ? y0 + 1 : y0;
  const float wx0 = (x0f + 1.0f) - ix, wx1 = ix - x0f, wy0 = (y0f + 1.0f) - iy, wy1 = iy - y0f;
  const size_t vbase = (size_t)(sb * sc.NS + v) * Hl * Wl * C;
  t.o_nw = vbase + ((size_t)y0 * Wl + x0) * C;
  t.o_ne = vbase + ((size_t)y0 * Wl + x1) * C;
  t.o_sw = vbase + ((size_t)y1 * Wl + x0) * C;
  t.o_se = vbase + ((size_t)y1 * Wl + x1) * C;
  t.w_nw = wx0 * wy0;
  t.w_ne = t.vx1 ? wx1 * wy0 : 0.f;
  t.w_sw = t.vy1 ? wx0 * wy1 : 0.f;
  t.w_se = (t.vx1 && t.vy1) ? wx1 * wy1 : 0.f;
  return t;
}

__device__ __forceinline__ float feat_channel(const PointGeom& g, int ch) {
  // [q(3) | for k<6: sin(q f_k)(3), sin(q f_k + pi/2)(3) | R dir (3)], f_k = 1.5 * 2^k
  if (ch < 3) return g.q[ch];
  if (ch < 39) {
    int j = (ch - 3) / 3, c = (ch - 3) % 3;
    float f = 1.5f * (float)(1 << (j >> 1));
    float ph = (j & 1) ? 1.57079637050628662109375f : 0.f;  // fp32(pi/2), code.py:27
    return sinf(__fadd_rn(ph, __fmul_rn(g.q[c], f)));      // addcmul(phases, x, freqs)
  }
  if (ch < 42) return g.dcam[ch - 39];
  return 0.f;
}

}  // namespace pnr
