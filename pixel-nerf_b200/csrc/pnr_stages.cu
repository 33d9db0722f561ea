// Per-ray / per-point stage kernels of the render path: latent re-layout, stratified and
// importance sampling, point feature construction (camera transform, positional code,
// projection, bilinear border gather) and alpha compositing.
//
// This file is compiled with -fmad=false: the reference evaluates these stages as separate
// elementwise torch ops (one rounding per op), and reproducing that rounding keeps the
// stochastic fine sampler (searchsorted bin edges) aligned with it.
#include <math.h>

#include "pnr_common.cuh"
#include "pnr_geom.cuh"
#include "pnr_ray_ops.cuh"

namespace pnr {

// ----------------------------------------------------------------------------------------
// NCHW -> NHWC (reference keeps NCHW and pays a strided gather: encoder.py:102, models.py:219)
// ----------------------------------------------------------------------------------------
__global__ void k_pack_latent(const float* __restrict__ src, float* __restrict__ dst, int C, int HW) {
  __shared__ float tile[32][33];
  const int v = blockIdx.z;
  const int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  const float* s = src + (size_t)v * C * HW;
  float* d = dst + (size_t)v * C * HW;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && p < HW) ? s[(size_t)c * HW + p] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    if (c < C && p < HW) d[(size_t)p * C + c] = tile[threadIdx.x][i];
  }
}

int launch_pack_latent(const float* nchw, float* nhwc, int V, int C, int Hl, int Wl, cudaStream_t s) {
  int HW = Hl * Wl;
  dim3 grid((HW + 31) / 32, (C + 31) / 32, V), block(32, 8);
  k_pack_latent<<<grid, block, 0, s>>>(nchw, nhwc, C, HW);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// ----------------------------------------------------------------------------------------
// sample_coarse (src/render/nerf.py:98-113)
// ----------------------------------------------------------------------------------------
__global__ void k_sample_coarse(const float* __restrict__ rays, const float* __restrict__ lin,
                                const float* __restrict__ u, float* __restrict__ z, int64_t R, int Kc) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * Kc) return;
  int64_t r = i / Kc;
  int k = (int)(i - r * Kc);
  z[i] = coarse_sample(rays[r * 8 + 6], rays[r * 8 + 7], lin ? lin[k] : lin_step_value(k, Kc), u[i], Kc);
}

int launch_sample_coarse(const float* rays, const float* lin, const float* u, float* z, int64_t R, int Kc,
                         cudaStream_t s) {
  int64_t n = R * Kc;
  if (n == 0) return PNR_OK;
  k_sample_coarse<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(rays, lin, u, z, R, Kc);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// ----------------------------------------------------------------------------------------
// compositing (src/render/nerf.py:178-182, 222-249).  One thread per ray; K is small.
// ----------------------------------------------------------------------------------------
__global__ void k_composite(const float* __restrict__ rays, const float* __restrict__ z,
                            const float* __restrict__ field, int white, float* __restrict__ w_out,
                            float* __restrict__ rgb_out, float* __restrict__ depth_out, int64_t R, int K) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  composite_ray(z + r * K, reinterpret_cast<const float4*>(field) + r * K, rays[r * 8 + 7], K, white,
                w_out ? w_out + r * K : nullptr, rgb_out + r * 3, depth_out + r, LdPlain(), LdPlain4());
}

int launch_composite(const float* rays, const float* z, const float* field, int white, float* w,
                     float* rgb, float* depth, int64_t R, int K, cudaStream_t s) {
  if (R == 0) return PNR_OK;
  k_composite<<<(unsigned)((R + 127) / 128), 128, 0, s>>>(rays, z, field, white, w, rgb, depth, R, K);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// ----------------------------------------------------------------------------------------
// sample_fine + sample_fine_depth + cat + sort (src/render/nerf.py:120-161, 285-295)
// One warp per ray.  cdf is accumulated sequentially (torch.cumsum order on CPU).
// ----------------------------------------------------------------------------------------
constexpr int kMaxK = 512;  // Kc + Kf upper bound for the shared-memory sorter

__global__ void k_sample_fine(const float* __restrict__ rays, const float* __restrict__ zc,
                              const float* __restrict__ wc, const float* __restrict__ dc,
                              const float* __restrict__ u, const float* __restrict__ uj,
                              const float* __restrict__ nd, float depth_std, float* __restrict__ zout,
                              int64_t R, int Kc, int Kf, int Kfd) {
  extern __shared__ float sm[];
  const int warps = blockDim.x / 32;
  const int wid = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int K = Kc + Kf, Ku = Kf - Kfd;
  float* scratch = sm + (size_t)wid * (Kc + 1 + K);
  int64_t r = (int64_t)blockIdx.x * warps + wid;
  if (r >= R) return;
  sample_fine_ray(rays[r * 8 + 6], rays[r * 8 + 7], zc + r * Kc, wc ? wc + r * Kc : nullptr, (Kfd > 0) ? dc[r] : 0.f,
                  u ? u + r * Ku : nullptr, uj ? uj + r * Ku : nullptr, nd ? nd + r * Kfd : nullptr, depth_std,
                  zout + r * K, Kc, Kf, Kfd, scratch, lane, LdPlain());
}

int launch_sample_fine(const float* rays, const float* zc, const float* wc, const float* dc,
                       const float* u, const float* uj, const float* nd, float depth_std, float* zout,
                       int64_t R, int Kc, int Kf, int Kfd, cudaStream_t s) {
  if (R == 0) return PNR_OK;
  const int warps = 4;
  size_t smem = (size_t)warps * (Kc + 1 + Kc + Kf) * sizeof(float);
  if (Kc + Kf > kMaxK) {
    set_error("n_coarse + n_fine = %d exceeds %d", Kc + Kf, kMaxK);
    return PNR_ERR_INVALID;
  }
  k_sample_fine<<<(unsigned)((R + warps - 1) / warps), warps * 32, smem, s>>>(
      rays, zc, wc, dc, u, uj, nd, depth_std, zout, R, Kc, Kf, Kfd);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// ----------------------------------------------------------------------------------------
// Point rows: camera transform, positional code, projection, bilinear border gather
// (src/model/models.py:158-227, src/model/code.py:30-42, src/model/encoder.py:80-109)
// ----------------------------------------------------------------------------------------
__global__ void k_build_rows(PnrScene sc, PointSource src, int64_t g0, int64_t n_pts,
                             float* __restrict__ feat, float* __restrict__ lat) {
  const int lane = threadIdx.x % 32;
  int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  if (row >= n_pts * sc.NS) return;
  int64_t lp = row / sc.NS;
  int v = (int)(row - lp * sc.NS);
  int64_t g = g0 + lp;
  int sb = (int)(g / src.P);
  float x[3], d[3];
  load_point(src, g, x, d);
  PointGeom pg = point_geometry(sc, sb, v, x, d);
  for (int ch = lane; ch < 48; ch += 32) feat[row * 48 + ch] = feat_channel(pg, ch);
  const float* L = sc.latent_nhwc + (size_t)(sb * sc.NS + v) * sc.Hl * sc.Wl * sc.C;
  const float4* t00 = reinterpret_cast<const float4*>(L + ((size_t)pg.y0 * sc.Wl + pg.x0) * sc.C);
  const float4* t01 = reinterpret_cast<const float4*>(L + ((size_t)pg.y0 * sc.Wl + pg.x1) * sc.C);
  const float4* t10 = reinterpret_cast<const float4*>(L + ((size_t)pg.y1 * sc.Wl + pg.x0) * sc.C);
  const float4* t11 = reinterpret_cast<const float4*>(L + ((size_t)pg.y1 * sc.Wl + pg.x1) * sc.C);
  float4* o = reinterpret_cast<float4*>(lat + row * sc.C);
  for (int c4 = lane; c4 < sc.C / 4; c4 += 32) {
    float4 a = __ldg(t00 + c4), b = __ldg(t01 + c4), c = __ldg(t10 + c4), e = __ldg(t11 + c4);
    float4 r;
    r.x = ((a.x * pg.w_nw + b.x * pg.w_ne) + c.x * pg.w_sw) + e.x * pg.w_se;
    r.y = ((a.y * pg.w_nw + b.y * pg.w_ne) + c.y * pg.w_sw) + e.y * pg.w_se;
    r.z = ((a.z * pg.w_nw + b.z * pg.w_ne) + c.z * pg.w_sw) + e.z * pg.w_se;
    r.w = ((a.w * pg.w_nw + b.w * pg.w_ne) + c.w * pg.w_sw) + e.w * pg.w_se;
    o[c4] = r;
  }
}

int launch_build_rows(const PnrScene& sc, const PointSource& src, int64_t g0, int64_t n_pts, float* feat,
                      float* lat, cudaStream_t s) {
  int64_t rows = n_pts * sc.NS;
  if (rows == 0) return PNR_OK;
  const int warps = 8;
  k_build_rows<<<(unsigned)((rows + warps - 1) / warps), warps * 32, 0, s>>>(sc, src, g0, n_pts, feat, lat);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// ----------------------------------------------------------------------------------------
// ray generation (src/util/util.py:238-276 gen_rays, :113-143 unproj_map).  Ray i of the flattened
// (NV, H, W) pixel grid, i in [first, first+count): [origin(3), unit dir(3), near, far].  One thread
// computes one ray; a warp then writes its 32 rays (1 KB) with two fully coalesced float4 stores.
// ----------------------------------------------------------------------------------------
__global__ void k_gen_rays(const float* __restrict__ poses, int W, int H, float fx, float fy, float cx, float cy,
                           float z_near, float z_far, int64_t first, int64_t count, float* __restrict__ rays) {
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t warp_base = t - lane;
  float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (t < count) {
    const int64_t i = first + t, hw = (int64_t)W * H;
    const int64_t v = i / hw;
    const int rem = (int)(i - v * hw);
    const int y = rem / W, x = rem - y * W;
    const float* P = poses + v * 16;                 // camera-to-world, row-major 4x4
    const float X = ((float)x - cx) / fx;            // unproj_map: (arange - c) / f
    const float Y = ((float)y - cy) / fy;
    float dx = X, dy = -Y, dz = -1.0f;
    const float n = sqrtf((dx * dx + dy * dy) + dz * dz);
    dx = dx / n; dy = dy / n; dz = dz / n;
    o[0] = P[3]; o[1] = P[7]; o[2] = P[11];
    o[3] = (P[0] * dx + P[1] * dy) + P[2] * dz;
    o[4] = (P[4] * dx + P[5] * dy) + P[6] * dz;
    o[5] = (P[8] * dx + P[9] * dy) + P[10] * dz;
    o[6] = z_near; o[7] = z_far;
  }
  float4* dst = reinterpret_cast<float4*>(rays) + warp_base * 2;
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int q = s * 32 + lane, src = q >> 1, half = q & 1;   // float4 q of the warp's 64
    float4 lo, hi;
    lo.x = __shfl_sync(0xffffffffu, o[0], src); lo.y = __shfl_sync(0xffffffffu, o[1], src);
    lo.z = __shfl_sync(0xffffffffu, o[2], src); lo.w = __shfl_sync(0xffffffffu, o[3], src);
    hi.x = __shfl_sync(0xffffffffu, o[4], src); hi.y = __shfl_sync(0xffffffffu, o[5], src);
    hi.z = __shfl_sync(0xffffffffu, o[6], src); hi.w = __shfl_sync(0xffffffffu, o[7], src);
    if (warp_base + src < count) dst[q] = half ? hi : lo;
  }
}

int launch_gen_rays(const float* poses, int W, int H, float fx, float fy, float cx, float cy, float z_near,
                    float z_far, int64_t first, int64_t count, float* rays, cudaStream_t s) {
  if (count == 0) return PNR_OK;
  k_gen_rays<<<(unsigned)((count + 255) / 256), 256, 0, s>>>(poses, W, H, fx, fy, cx, cy, z_near, z_far, first,
                                                              count, rays);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// ----------------------------------------------------------------------------------------
// frame assembly (eval/gen_video.py:213-222, 236): (rgb * 255).astype(uint8), i.e. one fp32 multiply and a
// truncating cast; four values per thread (coalesced 16 B loads, 4 B stores).
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int to_u8(float x) { return (unsigned int)__float2int_rz(x * 255.0f) & 255u; }

__global__ void k_frames_u8(const float* __restrict__ rgb, int64_t n, uint8_t* __restrict__ out) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t i = q * 4;
  if (i + 3 < n) {
    const float4 v = __ldcs(reinterpret_cast<const float4*>(rgb) + q);
    const unsigned int w = to_u8(v.x) | (to_u8(v.y) << 8) | (to_u8(v.z) << 16) | (to_u8(v.w) << 24);
    reinterpret_cast<unsigned int*>(out)[q] = w;
  } else {
    for (int64_t k = i; k < n; ++k) out[k] = (uint8_t)to_u8(rgb[k]);
  }
}

int launch_frames_u8(const float* rgb, int64_t n, uint8_t* out, cudaStream_t s) {
  if (n == 0) return PNR_OK;
  const int64_t quads = (n + 3) / 4;
  k_frames_u8<<<(unsigned)((quads + 255) / 256), 256, 0, s>>>(rgb, n, out);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// ----------------------------------------------------------------------------------------
// Backward of the renderer's own arithmetic (oracle/pnr_aux_backward.py::composite_backward / render_backward, which
// extend oracle/pnr_backward.py's rgb-only formulas).  One thread per ray; two sweeps over the K samples and no
// per-sample state beyond the outputs.  With t_k = (1 - a_k) + 1e-10 and T_k = prod_{j<k} t_j, the alpha gradient is
//   d_a_k = g_k T_k - sum_{m>k} g_m w_m / t_k = T_k (g_k - U_k),   U_k = sum_{m>k} g_m a_m prod_{k<j<m} t_j,
// and U follows U_{K-1} = 0, U_{k-1} = g_k a_k + t_k U_k.  Sweep 1 runs back to front and parks U_k in d_z[k] (which
// sweep 2 overwrites); sweep 2 runs front to back with T.  No suffix is formed as a difference and nothing is divided
// by t: behind a near-opaque sample t is 1e-4 .. 1e-10, and (total - prefix) / t there loses every bit to cancellation.
// The per-sample weight gradient is g_k = d_rgb . c_k + d_depth z_k (- sum d_rgb on a white background) + d_weights_k;
// any of the three upstream gradients may be NULL (zero).  Without d_weights the arithmetic is that of the rgb/depth-only
// kernel bit for bit (the add is skipped, not done with 0).
// ----------------------------------------------------------------------------------------
__global__ void k_composite_bwd(const float* __restrict__ rays, const float* __restrict__ z,
                                const float* __restrict__ field, const float* __restrict__ d_rgb,
                                const float* __restrict__ d_depth, const float* __restrict__ d_weights, int white,
                                float* __restrict__ d_field, float* __restrict__ d_z, float* __restrict__ d_far,
                                int64_t R, int K) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float far = rays[r * 8 + 7];
  const float* zr = z + r * K;
  float* dzr = d_z + r * K;
  const float4* fr = reinterpret_cast<const float4*>(field) + r * K;
  const float* dwr = d_weights ? d_weights + r * K : nullptr;
  const float gr = d_rgb ? d_rgb[r * 3 + 0] : 0.f, gg = d_rgb ? d_rgb[r * 3 + 1] : 0.f,
              gb = d_rgb ? d_rgb[r * 3 + 2] : 0.f;
  const float gd = d_depth ? d_depth[r] : 0.f;
  const float gbg = white ? (gr + gg + gb) : 0.f;   // rgb += 1 - sum w  (nerf.py:241-244)
  {
    float U = 0.f, znext = far;
    for (int k = K - 1; k >= 0; --k) {
      dzr[k] = U;
      const float zk = zr[k];
      const float4 f = fr[k];
      const float alpha = 1.0f - expf(-(znext - zk) * fmaxf(f.w, 0.f));    // sweep 2's e and alpha, same roundings
      float gw = ((gr * f.x + gg * f.y) + gb * f.z) + gd * zk - gbg;
      if (dwr) gw += dwr[k];
      U = gw * alpha + ((1.0f - alpha) + 1e-10f) * U;
      znext = zk;
    }
  }
  float T = 1.0f, zk = zr[0], carry = 0.f;
  float4* dfr = reinterpret_cast<float4*>(d_field) + r * K;
  for (int k = 0; k < K; ++k) {
    const float znext = (k + 1 < K) ? zr[k + 1] : far;
    const float delta = znext - zk;
    const float4 f = fr[k];
    const float sg = fmaxf(f.w, 0.f);
    const float e = expf(-delta * sg);
    const float alpha = 1.0f - e;
    const float t = (1.0f - alpha) + 1e-10f;
    const float w = alpha * T;
    float gw = ((gr * f.x + gg * f.y) + gb * f.z) + gd * zk - gbg;
    if (dwr) gw += dwr[k];
    const float d_a = T * (gw - dzr[k]);              // dzr[k] = U_k from sweep 1
    const float d_delta = d_a * e * sg;
    float4 o;
    o.x = w * gr; o.y = w * gg; o.z = w * gb;
    o.w = (f.w > 0.f) ? d_a * e * delta : 0.f;
    dfr[k] = o;
    dzr[k] = (w * gd - d_delta) + carry;               // delta_{k-1} = z_k - z_{k-1} gives +d_delta_{k-1}
    carry = d_delta;
    T = T * t;
    zk = znext;
  }
  if (d_far) d_far[r] = carry;                        // delta_{K-1} = far - z_{K-1} (nerf.py:181): d_far += d_delta
}

int launch_composite_bwd(const float* rays, const float* z, const float* field, const float* d_rgb,
                         const float* d_depth, const float* d_weights, int white, float* d_field, float* d_z,
                         float* d_far, int64_t R, int K, cudaStream_t s) {
  if (R == 0) return PNR_OK;
  k_composite_bwd<<<(unsigned)((R + 127) / 128), 128, 0, s>>>(rays, z, field, d_rgb, d_depth, d_weights, white,
                                                              d_field, d_z, d_far, R, K);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// d_z[ray][k] += d_xyz[ray][k] . dir[ray]      (points = o + z d, nerf.py:185)
__global__ void k_dz_from_dxyz(float* __restrict__ d_z, const float* __restrict__ d_xyz,
                               const float* __restrict__ rays, int64_t R, int K) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * K) return;
  const float* rr = rays + (i / K) * 8;
  d_z[i] += (d_xyz[i * 3 + 0] * rr[3] + d_xyz[i * 3 + 1] * rr[4]) + d_xyz[i * 3 + 2] * rr[5];
}

// Slot of depth sample j in the sorted merged row zs [K] (the forward's rank rule: smaller values first, ties by original
// index, the depth samples being the last index group); v = its clamped value.  k_depth_grad and k_ray_grad both route
// a depth sample's d_z through this one function, so they agree slot for slot.
__device__ __forceinline__ int depth_slot(const float* zs, int K, const float* ndr, int Kfd, int j, float d, float std_,
                                          float near, float far, float v) {
  int lo = 0, hi = K;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (zs[mid] < v) lo = mid + 1; else hi = mid;
  }
  int ub = lo;
  while (ub < K && zs[ub] == v) ++ub;
  int n_eq_depth = 0, n_eq_before = 0;
  for (int q = 0; q < Kfd; ++q) {
    const float zq = fmaxf(fminf(d + ndr[q] * std_, far), near);
    if (zq == v) { ++n_eq_depth; if (q < j) ++n_eq_before; }
  }
  return lo + ((ub - lo) - n_eq_depth) + n_eq_before;
}

// Gradient of the coarse depth through the depth-centred fine samples (nerf.py:150-161, 289-295): each sample
// z_j = clamp(depth + n_j * std, near, far) sits somewhere in the sorted merged row; its slot is recomputed with the
// forward's rank rule (smaller values first, ties by original index, the depth samples being the last index group).
// d_depth = d_depth_up (the caller's gradient of the coarse depth output; NULL = zero) + that contribution.
__global__ void k_depth_grad(const float* __restrict__ rays, const float* __restrict__ z_sorted,
                             const float* __restrict__ depth, const float* __restrict__ nd, float depth_std,
                             const float* __restrict__ d_z, const float* __restrict__ d_depth_up,
                             float* __restrict__ d_depth, int64_t R, int K, int Kfd) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float near = rays[r * 8 + 6], far = rays[r * 8 + 7], d = depth[r];
  const float* zs = z_sorted + r * K;
  float acc = 0.f;
  for (int j = 0; j < Kfd; ++j) {
    const float zz = d + nd[r * Kfd + j] * depth_std;
    if (!(zz >= near && zz <= far)) continue;            // clamped: no gradient
    const float v = fmaxf(fminf(zz, far), near);
    const int pos = depth_slot(zs, K, nd + r * Kfd, Kfd, j, d, depth_std, near, far, v);
    if (pos >= 0 && pos < K) acc += d_z[r * K + pos];
  }
  d_depth[r] = d_depth_up ? d_depth_up[r] + acc : acc;
}

// Ray gradient of one pass (nerf.py:98-118, 120-161, 178-204): d_rays[r] = [d_origin, d_dir, d_near, d_far], written
// (accum = 0) or added (accum = 1).  points = o + z d and viewdirs = d give d_o = sum_k d_x, d_d = sum_k z_k d_x + d_vd;
// the sample depths' gradient d_z (+ d_x . d unless d_z already holds it) goes to near / far through
// z = near (1 - s) + far s, s = (z - near) / (far - near), for the stratified and importance samples; a depth-centred
// sample z = max(min(depth + n std, far), near) sends it to far or near when clamped (k_depth_grad carries the unclamped
// ones to the coarse depth); the last interval far - z_{K-1} adds d_far_last.
__global__ void k_ray_grad(const float* __restrict__ rays, const float* __restrict__ z, const float* __restrict__ d_z,
                           const float* __restrict__ d_xyz, const float* __restrict__ d_vd,
                           const float* __restrict__ d_far_last, int dz_has_pos, const float* __restrict__ depth,
                           const float* __restrict__ nd, float depth_std, int Kfd, int accum,
                           float* __restrict__ d_rays, int64_t R, int K) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* rr = rays + r * 8;
  const float near = rr[6], far = rr[7], dir[3] = {rr[3], rr[4], rr[5]};
  const float* zr = z + r * K;
  const float* dzr = d_z + r * K;
  const float* dxr = d_xyz + r * K * 3;
  const float* dvr = d_vd + r * K * 3;
  auto dz_total = [&](int k) {
    const float* dx = dxr + k * 3;
    return dz_has_pos ? dzr[k] : dzr[k] + ((dx[0] * dir[0] + dx[1] * dir[1]) + dx[2] * dir[2]);
  };
  uint32_t is_depth[kMaxK / 32];
  for (int i = 0; i < kMaxK / 32; ++i) is_depth[i] = 0u;
  float g_near = 0.f, g_far = d_far_last[r];
  if (Kfd > 0) {
    const float d = depth[r];
    const float* ndr = nd + r * Kfd;
    for (int j = 0; j < Kfd; ++j) {
      const float zz = d + ndr[j] * depth_std;
      const float v = fmaxf(fminf(zz, far), near);
      const int pos = depth_slot(zr, K, ndr, Kfd, j, d, depth_std, near, far, v);
      if (pos < 0 || pos >= K) continue;
      is_depth[pos >> 5] |= 1u << (pos & 31);
      // torch.min chose far / torch.max chose near; at zz == far or zz == near exactly torch splits the gradient in
      // halves, here (as in k_depth_grad) all of it goes to the depth -- a tie of measure zero
      if (zz > far) g_far += dz_total(pos);
      else if (zz < near) g_near += dz_total(pos);
    }
  }
  float go[3] = {0.f, 0.f, 0.f}, gd[3] = {0.f, 0.f, 0.f};
  const float span = far - near;
  for (int k = 0; k < K; ++k) {
    const float* dx = dxr + k * 3;
    const float* dv = dvr + k * 3;
    const float zk = zr[k];
    for (int i = 0; i < 3; ++i) {
      go[i] += dx[i];
      gd[i] += zk * dx[i] + dv[i];
    }
    if (is_depth[k >> 5] & (1u << (k & 31))) continue;
    const float s = (zk - near) / span, g = dz_total(k);
    g_near += g * (1.0f - s);
    g_far += g * s;
  }
  float* o = d_rays + r * 8;
  const float vals[8] = {go[0], go[1], go[2], gd[0], gd[1], gd[2], g_near, g_far};
  for (int i = 0; i < 8; ++i) o[i] = accum ? o[i] + vals[i] : vals[i];
}

int launch_ray_grad(const float* rays, const float* z, const float* d_z, const float* d_xyz, const float* d_vd,
                    const float* d_far_last, bool dz_has_pos, const float* depth, const float* nd, float depth_std,
                    int Kfd, bool accum, float* d_rays, int64_t R, int K, cudaStream_t s) {
  if (R == 0) return PNR_OK;
  if (K > kMaxK) {
    set_error("n_coarse + n_fine = %d exceeds %d", K, kMaxK);
    return PNR_ERR_INVALID;
  }
  k_ray_grad<<<(unsigned)((R + 127) / 128), 128, 0, s>>>(rays, z, d_z, d_xyz, d_vd, d_far_last, dz_has_pos ? 1 : 0,
                                                         depth, nd, depth_std, Kfd, accum ? 1 : 0, d_rays, R, K);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// Backward of k_gen_rays (util.py:238-276): origin = P[:3, 3], dir = P[:3, :3] unproj (unit), so
// d_P[:3, 3] += sum_pixels d_origin and d_P[:3, :3] += sum_pixels d_dir unproj^T.  One block per camera of the range
// sums its pixels in a fixed order (thread-strided partial sums, then a shared-memory tree); one writer per pose.
constexpr int kGenBwdThreads = 256;
__global__ void __launch_bounds__(kGenBwdThreads) k_gen_rays_bwd(const float* __restrict__ d_rays, int W, int H,
                                                                 float fx, float fy, float cx, float cy, int64_t first,
                                                                 int64_t count, float* __restrict__ d_poses) {
  __shared__ float red[12][kGenBwdThreads];
  const int64_t hw = (int64_t)W * H;
  const int64_t v = first / hw + blockIdx.x;
  const int t = threadIdx.x;
  int64_t a = v * hw, b = (v + 1) * hw;
  if (a < first) a = first;
  if (b > first + count) b = first + count;
  float s[12];
  for (int j = 0; j < 12; ++j) s[j] = 0.f;
  for (int64_t i = a + t; i < b; i += kGenBwdThreads) {
    const int rem = (int)(i - v * hw);
    const int y = rem / W, x = rem - y * W;
    const float X = ((float)x - cx) / fx;
    const float Y = ((float)y - cy) / fy;
    float dx = X, dy = -Y, dz = -1.0f;
    const float n = sqrtf((dx * dx + dy * dy) + dz * dz);
    const float u[3] = {dx / n, dy / n, dz / n};
    const float* g = d_rays + (i - first) * 8;
    for (int row = 0; row < 3; ++row) {
      for (int col = 0; col < 3; ++col) s[row * 4 + col] += g[3 + row] * u[col];
      s[row * 4 + 3] += g[row];
    }
  }
  for (int j = 0; j < 12; ++j) red[j][t] = s[j];
  __syncthreads();
  for (int w = kGenBwdThreads / 2; w > 0; w >>= 1) {
    if (t < w)
      for (int j = 0; j < 12; ++j) red[j][t] += red[j][t + w];
    __syncthreads();
  }
  if (t < 12) d_poses[v * 16 + t] += red[t][0];
}

int launch_gen_rays_bwd(const float* d_rays, int W, int H, float fx, float fy, float cx, float cy, int64_t first,
                        int64_t count, float* d_poses, cudaStream_t s) {
  if (count == 0) return PNR_OK;
  const int64_t hw = (int64_t)W * H;
  const int64_t nv = (first + count - 1) / hw - first / hw + 1;
  k_gen_rays_bwd<<<(unsigned)nv, kGenBwdThreads, 0, s>>>(d_rays, W, H, fx, fy, cx, cy, first, count, d_poses);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

int launch_depth_grad(const float* rays, const float* z_sorted, const float* depth, const float* nd,
                      float depth_std, float* d_z, const float* d_xyz, const float* d_depth_up, float* d_depth,
                      int64_t R, int K, int Kfd, cudaStream_t s) {
  if (R == 0) return PNR_OK;
  k_dz_from_dxyz<<<(unsigned)((R * K + 255) / 256), 256, 0, s>>>(d_z, d_xyz, rays, R, K);
  PNR_LAUNCH_CHECK();
  k_depth_grad<<<(unsigned)((R + 127) / 128), 128, 0, s>>>(rays, z_sorted, depth, nd, depth_std, d_z, d_depth_up, d_depth, R,
                                                           K, Kfd);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

}  // namespace pnr
