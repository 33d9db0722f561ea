// Backward of the conditioned field (SURVEY 8f-1), first path: fp32 SIMT, recompute-in-backward.
//
// Arithmetic = oracle/pnr_backward.py::field_backward (checked on the CPU against autograd and against gradients
// produced by the reference itself).  Per chunk of points the forward is run again with the block inputs and fc_0
// outputs kept (the ReLU masks and the operands of the weight gradients), then the layers are walked in reverse:
//   dX = dY W        : the NT SGEMM of the forward engine on a transposed copy of W
//   dW += dY^T X     : the same SGEMM on transposed, zero-padded copies of dY and X (K = rows)
//   db += colsum(dY) : row sums of the transposed dY
// followed by one warp per point for pos-enc, projection and the 4-tap gather (latent scatter + d uv).
// Row order inside a chunk is the forward SIMT engine's: row = local_point * NS + view.
//
// The GEMMs run on the tensor cores by default (split-bf16 wgmma GEMM, pnr_gemm_tc.cu); PNR_BWD_GEMM=simt selects
// the fp32 FFMA SGEMM instead (the first, reference implementation of this path).
// Validated on H100 against the oracle's formulas, the composed-torch path and the reference's own gradients
// (tests/test_gpu_backward.py), compute-sanitizer memcheck clean.
#include <stdlib.h>

#include "pnr_geom.cuh"

namespace pnr {

int sgemm(const float* A, int lda, const float* W, const float* bias, float* C, int ldc, int M, int N, int K,
          bool relu_a, bool accum, cudaStream_t s);
int gemm_bf16x3(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc, int M, int N,
                int K, bool relu_a, bool accum, cudaStream_t s);   // pnr_gemm_tc.cu
int gemm_bf16x3_masked(const float* A, int lda, const float* W, int ldw, float* C, int ldc, int M, int N, int K, bool accum,
                       const float* mask, cudaStream_t s);
__global__ void k_pad_rows(const float* __restrict__ src, float* __restrict__ dst, int rows, int k_src, int k_dst);
__global__ void k_view_mean(const float* __restrict__ X, float* __restrict__ Y, int64_t n_pts, int NS, int d);
// pnr_determ.cu (deterministic mode).  Weak, so that a build without that unit (the host emulator of the SIMT units)
// still links; there deterministic mode reports itself unavailable.
int latent_scatter_fixed(const PnrScene& sc, const PointSource& src, int64_t g0, int64_t n, const float* d_lat,
                         float* d_latent, long long* acc, unsigned* m_bits, cudaStream_t s) __attribute__((weak));

namespace bwd {

static inline int pad16(int x) { return (x + 15) / 16 * 16; }

// C (+)= act(A) W^T + bias on the tensor cores (default) or the fp32 SIMT SGEMM (PNR_BWD_GEMM=simt)
static bool use_tc_gemm() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("PNR_BWD_GEMM");
    v = (e && e[0] == 's') ? 0 : 1;
  }
  return v == 1;
}
static int gemm(const float* A, int lda, const float* W, const float* bias, float* C, int ldc, int M, int N, int K,
                bool relu_a, bool accum, cudaStream_t s) {
  if (use_tc_gemm()) return gemm_bf16x3(A, lda, W, K, bias, C, ldc, M, N, K, relu_a, accum, s);
  return sgemm(A, lda, W, bias, C, ldc, M, N, K, relu_a, accum, s);
}
// The forward recomputed per chunk runs on the same engine, or on the fp32 SIMT SGEMM with PNR_BWD_RECOMPUTE=simt while
// the backward's GEMMs stay on the tensor cores: a test hook that keeps the split-bf16 rounding of the recomputed
// activations (which the gradients inherit, ~1e-4 at width 512) out of a check of the backward's own GEMMs.
static bool recompute_on_simt() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("PNR_BWD_RECOMPUTE");
    v = (e && e[0] == 's') ? 1 : 0;
  }
  return v == 1;
}
static int fwd_gemm(const float* A, int lda, const float* W, const float* bias, float* C, int ldc, int M, int N, int K,
                    bool relu_a, bool accum, cudaStream_t s) {
  if (recompute_on_simt()) return sgemm(A, lda, W, bias, C, ldc, M, N, K, relu_a, accum, s);
  return gemm(A, lda, W, bias, C, ldc, M, N, K, relu_a, accum, s);
}

// dst[c][m] = f(src[m][c]) for m < M (f = identity or ReLU), 0 for M <= m < Mpad.   32x32 tiles.
template <bool RELU>
__global__ void k_transpose_pad(const float* __restrict__ src, int ld, int M, int C, float* __restrict__ dst, int Mpad) {
  __shared__ float tile[32][33];
  const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int m = m0 + j, c = c0 + threadIdx.x;
    float v = (m < M && c < C) ? src[(size_t)m * ld + c] : 0.f;
    if (RELU) v = fmaxf(v, 0.f);
    tile[j][threadIdx.x] = v;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int c = c0 + j, m = m0 + threadIdx.x;
    if (c < C && m < Mpad) dst[(size_t)c * Mpad + m] = tile[threadIdx.x][j];
  }
}

template <bool RELU>
static int transpose_pad(const float* src, int ld, int M, int C, float* dst, int Mpad, cudaStream_t s) {
  dim3 grid((Mpad + 31) / 32, (C + 31) / 32), block(32, 8);
  k_transpose_pad<RELU><<<grid, block, 0, s>>>(src, ld, M, C, dst, Mpad);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// T *= (ref > 0)
__global__ void k_mask(float* __restrict__ T, const float* __restrict__ ref, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) T[i] = (ref[i] > 0.f) ? T[i] : 0.f;
}

// D += T * (ref > 0)
__global__ void k_mask_add(float* __restrict__ D, const float* __restrict__ T, const float* __restrict__ ref, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && ref[i] > 0.f) D[i] += T[i];
}

// out[r] += sum_m src[r][m]   (one block per row: the rows are few (d <= 512) and long (a chunk's points))
__global__ void k_rowsum_acc(const float* __restrict__ src, int ld, int n_rows, float* __restrict__ out) {
  __shared__ float part[8];
  const int r = blockIdx.x, lane = threadIdx.x % 32, wid = threadIdx.x / 32;
  if (r >= n_rows) return;
  float s = 0.f;
  const float* row = src + (size_t)r * ld;
  for (int m = threadIdx.x; m < ld; m += blockDim.x) s += row[m];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) part[wid] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x / 32); ++i) t += part[i];
    out[r] += t;
  }
}

static int rowsum_acc(const float* src, int ld, int n_rows, float* out, cudaStream_t s) {
  k_rowsum_acc<<<n_rows, 256, 0, s>>>(src, ld, n_rows, out);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// dV[(p*NS + v)][c] = dM[p][c] / NS      (backward of util.combine_interleaved(average), util.py:461-471)
__global__ void k_view_mean_bwd(const float* __restrict__ dM, float* __restrict__ dV, int64_t n_pts, int NS, int d) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pts * NS * d) return;
  const int c = (int)(i % d);
  const int64_t p = i / d / NS;
  dV[i] = dM[p * d + c] / (float)NS;
}

// dst[r][0..k_dst) += src[r][0..k_dst)   (src rows are k_src wide)
__global__ void k_add_cols(float* __restrict__ dst, const float* __restrict__ src, int rows, int k_dst, int k_src) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * k_dst) return;
  const int r = i / k_dst, k = i % k_dst;
  dst[i] += src[r * k_src + k];
}

// lin_out + activations backward (resnetfc.py:183, models.py:260-264).  One warp per point:
// o4 = W relu(h) + b;  d_o4 = [d_rgb * s(1-s), d_sigma * (o4_3 > 0)];  d_h = (W^T d_o4) * (h > 0)
__global__ void k_lin_out_bwd(const float* __restrict__ H, const float* __restrict__ W, const float* __restrict__ b,
                              const float* __restrict__ d_out, float* __restrict__ d_o4, float* __restrict__ d_h,
                              int64_t n_pts, int d) {
  const int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (p >= n_pts) return;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  for (int k = lane; k < d; k += 32) {
    const float x = fmaxf(H[p * d + k], 0.f);
    a0 = fmaf(x, W[0 * d + k], a0);
    a1 = fmaf(x, W[1 * d + k], a1);
    a2 = fmaf(x, W[2 * d + k], a2);
    a3 = fmaf(x, W[3 * d + k], a3);
  }
  for (int o = 16; o > 0; o >>= 1) {
    a0 += __shfl_xor_sync(0xffffffffu, a0, o);
    a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    a2 += __shfl_xor_sync(0xffffffffu, a2, o);
    a3 += __shfl_xor_sync(0xffffffffu, a3, o);
  }
  const float4 g = reinterpret_cast<const float4*>(d_out)[p];
  const float s0 = 1.0f / (1.0f + expf(-(a0 + b[0])));
  const float s1 = 1.0f / (1.0f + expf(-(a1 + b[1])));
  const float s2 = 1.0f / (1.0f + expf(-(a2 + b[2])));
  float4 q;
  q.x = g.x * s0 * (1.0f - s0);
  q.y = g.y * s1 * (1.0f - s1);
  q.z = g.z * s2 * (1.0f - s2);
  q.w = (a3 + b[3] > 0.f) ? g.w : 0.f;
  if (lane == 0) reinterpret_cast<float4*>(d_o4)[p] = q;
  for (int k = lane; k < d; k += 32) {
    const float v = q.x * W[0 * d + k] + q.y * W[1 * d + k] + q.z * W[2 * d + k] + q.w * W[3 * d + k];
    d_h[p * d + k] = (H[p * d + k] > 0.f) ? v : 0.f;
  }
}

// Geometry backward, one warp per point over its NS views (rows lp*NS + v of the chunk):
//   d_lat row (C) -> atomic scatter into d_latent (channels-last) over the 4 taps, and d(ix, iy)
//   d_feat row (48) -> pos-enc derivative; projection; rotate back; sum over views -> d_xyz[point]
//   optional: d_dirs[point] = sum over views of R^T d(R dir) (models.py:188-193), and per row the 16 camera partials
//   cam_part[row] = [dR (3x3) | dt (3) in the [3][4] pose layout | d_focal (2) | d_c (2)] (models.py:161-212), which
//   k_cam_reduce sums per view in a fixed order (no same-address atomics)
__global__ void k_geom_bwd(PnrScene sc, PointSource src, int64_t g0, int64_t n_pts, const float* __restrict__ d_feat,
                           const float* __restrict__ d_lat, float* __restrict__ d_latent, float* __restrict__ d_xyz,
                           float* __restrict__ d_dirs, float* __restrict__ cam_part) {
  const int64_t lp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (lp >= n_pts) return;
  const int64_t g = g0 + lp;
  const int sb = (int)(g / src.P);
  float x[3], dir[3];
  load_point(src, g, x, dir);
  float dx[3] = {0.f, 0.f, 0.f}, dd[3] = {0.f, 0.f, 0.f};
  const int C = sc.C, Wl = sc.Wl, Hl = sc.Hl;
  for (int v = 0; v < sc.NS; ++v) {
    const int64_t row = lp * sc.NS + v;
    // the tap arithmetic below (to w_se) is restated by bwd_taps (pnr_geom.cuh) for deterministic mode's scatter:
    // change both together
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
    const float kx = sc.scale_x / sc.image_w, ky = sc.scale_y / sc.image_h;
    const float ix_u = ((u * kx - 1.0f) + 1.0f) * 0.5f * (float)(Wl - 1);
    const float iy_u = ((w * ky - 1.0f) + 1.0f) * 0.5f * (float)(Hl - 1);
    const bool in_x = (ix_u >= 0.f) && (ix_u <= (float)(Wl - 1));     // false for NaN, like the clamp's zero gradient
    const bool in_y = (iy_u >= 0.f) && (iy_u <= (float)(Hl - 1));
    float ix = fminf((float)(Wl - 1), fmaxf(ix_u, 0.f));
    float iy = fminf((float)(Hl - 1), fmaxf(iy_u, 0.f));
    if (!(ix == ix)) ix = 0.f;
    if (!(iy == iy)) iy = 0.f;
    const float x0f = floorf(ix), y0f = floorf(iy);
    const int x0 = (int)x0f, y0 = (int)y0f;
    const bool vx1 = (x0 + 1 <= Wl - 1), vy1 = (y0 + 1 <= Hl - 1);     // taps outside the map carry nothing
    const int x1 = vx1 ? x0 + 1 : x0, y1 = vy1 ? y0 + 1 : y0;
    const float wx0 = (x0f + 1.0f) - ix, wx1 = ix - x0f, wy0 = (y0f + 1.0f) - iy, wy1 = iy - y0f;
    const size_t vbase = (size_t)(sb * sc.NS + v) * Hl * Wl * C;
    const size_t o_nw = vbase + ((size_t)y0 * Wl + x0) * C, o_ne = vbase + ((size_t)y0 * Wl + x1) * C;
    const size_t o_sw = vbase + ((size_t)y1 * Wl + x0) * C, o_se = vbase + ((size_t)y1 * Wl + x1) * C;
    const float w_nw = wx0 * wy0, w_ne = vx1 ? wx1 * wy0 : 0.f, w_sw = vy1 ? wx0 * wy1 : 0.f,
                w_se = (vx1 && vy1) ? wx1 * wy1 : 0.f;
    float dnw = 0.f, dne = 0.f, dsw = 0.f, dse = 0.f;
    const float* dl = d_lat ? d_lat + row * C : nullptr;   // NULL: only d_dirs is wanted, which does not read it
    for (int c = lane; dl && c < C; c += 32) {
      const float gdl = dl[c];
      dnw = fmaf(gdl, sc.latent_nhwc[o_nw + c], dnw);
      dne = fmaf(gdl, sc.latent_nhwc[o_ne + c], dne);
      dsw = fmaf(gdl, sc.latent_nhwc[o_sw + c], dsw);
      dse = fmaf(gdl, sc.latent_nhwc[o_se + c], dse);
      if (d_latent) {
        atomicAdd(d_latent + o_nw + c, gdl * w_nw);
        if (vx1) atomicAdd(d_latent + o_ne + c, gdl * w_ne);
        if (vy1) atomicAdd(d_latent + o_sw + c, gdl * w_sw);
        if (vx1 && vy1) atomicAdd(d_latent + o_se + c, gdl * w_se);
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      dnw += __shfl_xor_sync(0xffffffffu, dnw, o);
      dne += __shfl_xor_sync(0xffffffffu, dne, o);
      dsw += __shfl_xor_sync(0xffffffffu, dsw, o);
      dse += __shfl_xor_sync(0xffffffffu, dse, o);
    }
    if (!vx1) { dne = 0.f; dse = 0.f; }
    if (!vy1) { dsw = 0.f; dse = 0.f; }
    float d_ix = wy0 * (dne - dnw) + wy1 * (dse - dsw);
    float d_iy = wx0 * (dsw - dnw) + wx1 * (dse - dne);
    if (!in_x) d_ix = 0.f;
    if (!in_y) d_iy = 0.f;
    const float d_u = d_ix * kx * 0.5f * (float)(Wl - 1);
    const float d_w = d_iy * ky * 0.5f * (float)(Hl - 1);
    // pos-enc (code.py:30-42): channels [q(3) | sin(q f_j + ph_j)(3) for j < 12 | R dir(3)]
    const float* df = d_feat + row * 48;
    float dq[3];
    for (int c = 0; c < 3; ++c) {
      float acc = df[c];
      for (int j = 0; j < 12; ++j) {
        const float f = 1.5f * (float)(1 << (j >> 1));
        const float ph = (j & 1) ? 1.57079637050628662109375f : 0.f;
        acc = fmaf(df[3 + 3 * j + c] * f, cosf(q[c] * f + ph), acc);
      }
      dq[c] = acc;
    }
    // projection (models.py:206-212): uv = -p.xy / p.z * focal + c
    const float gz0 = d_u * fo[0], gz1 = d_w * fo[1];
    const float dp[3] = {-gz0 / p[2], -gz1 / p[2], (gz0 * p[0] + gz1 * p[1]) / (p[2] * p[2])};
    dq[0] += dp[0];
    dq[1] += dp[1];
    dq[2] += dp[2];
    for (int i = 0; i < 3; ++i) dx[i] += M[0 * 4 + i] * dq[0] + M[1 * 4 + i] * dq[1] + M[2 * 4 + i] * dq[2];   // R^T dq
    const float* dv = df + 39;                                                     // d(R dir)
    if (d_dirs)
      for (int i = 0; i < 3; ++i) dd[i] += M[0 * 4 + i] * dv[0] + M[1 * 4 + i] * dv[1] + M[2 * 4 + i] * dv[2];
    if (cam_part && lane == 0) {   // q = R x, p = q + t, dir_cam = R dir, uv = -p.xy / p.z * focal + c
      float* cp = cam_part + row * 16;
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) cp[i * 4 + j] = dq[i] * x[j] + dv[i] * dir[j];
        cp[i * 4 + 3] = dp[i];
      }
      cp[12] = d_u * (-p[0] / p[2]);
      cp[13] = d_w * (-p[1] / p[2]);
      cp[14] = d_u;
      cp[15] = d_w;
    }
  }
  if (d_xyz && lane == 0) {
    d_xyz[g * 3 + 0] = dx[0];
    d_xyz[g * 3 + 1] = dx[1];
    d_xyz[g * 3 + 2] = dx[2];
  }
  if (d_dirs && lane == 0) {
    d_dirs[g * 3 + 0] = dd[0];
    d_dirs[g * 3 + 1] = dd[1];
    d_dirs[g * 3 + 2] = dd[2];
  }
}

// Camera partials of one chunk, summed per source view: block vi = sb*NS + v adds, over the chunk's points of object
// sb in a fixed order (thread-strided partial sums, then a shared-memory tree), its 16 partials into acc[vi][16].
// One writer per address and chunks in stream order, so the result does not depend on scheduling.
constexpr int kCamThreads = 256;
__global__ void __launch_bounds__(kCamThreads) k_cam_reduce(const float* __restrict__ cam_part, int64_t g0,
                                                            int64_t n_pts, int64_t P, int NS, float* __restrict__ acc) {
  __shared__ float red[16][kCamThreads];
  const int vi = blockIdx.x, sb = vi / NS, v = vi - sb * NS, t = threadIdx.x;
  int64_t a = (int64_t)sb * P - g0, b = (int64_t)(sb + 1) * P - g0;   // local points of object sb
  if (a < 0) a = 0;
  if (b > n_pts) b = n_pts;
  float s[16];
  for (int j = 0; j < 16; ++j) s[j] = 0.f;
  for (int64_t lp = a + t; lp < b; lp += kCamThreads) {
    const float* cp = cam_part + (lp * NS + v) * 16;
    for (int j = 0; j < 16; ++j) s[j] += cp[j];
  }
  for (int j = 0; j < 16; ++j) red[j][t] = s[j];
  __syncthreads();
  for (int w = kCamThreads / 2; w > 0; w >>= 1) {
    if (t < w)
      for (int j = 0; j < 16; ++j) red[j][t] += red[j][t + w];
    __syncthreads();
  }
  if (t < 16 && b > a) acc[vi * 16 + t] += red[t][0];
}

// acc [V][16] -> d_poses [V][3][4] (+=), d_focal [n_focal][2] (+=) and d_c [n_c][2] (+=); a shared focal / c row sums
// the views of every object, in view order.
__global__ void k_cam_finish(const float* __restrict__ acc, int V, int NS, int n_focal, int n_c,
                             float* __restrict__ d_poses, float* __restrict__ d_focal, float* __restrict__ d_c) {
  const int t = threadIdx.x;
  if (d_poses)
    for (int i = t; i < V * 12; i += blockDim.x) d_poses[i] += acc[(i / 12) * 16 + i % 12];
  if (t < 4) {
    float* dst = t < 2 ? d_focal : d_c;
    const int rows = t < 2 ? n_focal : n_c, k = t & 1, col = 12 + t;
    if (dst)
      for (int r = 0; r < rows; ++r) {
        const int v0 = rows > 1 ? r * NS : 0, v1 = rows > 1 ? (r + 1) * NS : V;
        float sum = 0.f;
        for (int vi = v0; vi < v1; ++vi) sum += acc[vi * 16 + col];
        dst[r * 2 + k] += sum;
      }
  }
}

static int64_t chunk_points(const PnrScene& sc, int64_t total_points) {
  int64_t rows = 32768;       // rows per chunk
  if (const char* e = getenv("PNR_BWD_CHUNK_ROWS")) {   // test hook: force several chunks on small inputs
    const long v = atol(e);
    if (v >= sc.NS) rows = v;
  }
  int64_t c = rows / sc.NS;
  if (c > total_points) c = total_points;
  return c < 1 ? 1 : c;
}

struct Bufs {
  float *feat, *lat, *latT, *featT, *hpre[PNR_MAX_BLOCKS], *nbuf[PNR_MAX_BLOCKS], *xv, *hlast, *dh, *dhv, *T, *T2, *tA, *tB,
      *dlat, *dfeat, *do4, *w_in, *w_inT, *tmp_win, *w0T[PNR_MAX_BLOCKS], *w1T[PNR_MAX_BLOCKS], *wzT[PNR_MAX_BLOCKS],
      *cam_acc, *splitk;
  long long* lat_fixed;
  unsigned* m_bits;
  size_t splitk_bytes;
};

// Deterministic mode's split-K partials: a split GEMM covers splits * tiles <= 2 * SMs + tiles - 1 < 3 * SMs output
// tiles of 128 x 128, and never has more splits than K / 256.  Sized for the 132 SMs of an H100 SXM (a GPU with more
// splits less) and for this call's shapes.
static size_t splitk_budget(int64_t R, int d, int L) {
  const int64_t w = d > L ? (d > 48 ? d : 48) : (L > 48 ? L : 48);
  const int64_t dw = (pad16((int)R) / 256) * w * w, dx = (w / 256) * R * w, cap = (int64_t)3 * 132 * 128 * 128;
  int64_t e = dw > dx ? dw : dx;
  if (e > cap) e = cap;
  return (size_t)e * sizeof(float);
}

static size_t carve(Arena& ar, Bufs& b, const PnrScene& sc, const PnrMlp& mlp, int64_t cp, bool det) {
  const size_t R = (size_t)cp * sc.NS, d = mlp.d_hidden, L = mlp.d_latent, Rp = pad16((int)R);
  b.feat = ar.take<float>(R * 48);
  b.lat = ar.take<float>(R * L);
  b.latT = ar.take<float>(L * Rp);
  b.featT = ar.take<float>(48 * Rp);
  for (int i = 0; i < mlp.n_blocks; ++i) {
    b.hpre[i] = ar.take<float>(R * d);
    b.nbuf[i] = ar.take<float>(R * d);
    b.w0T[i] = ar.take<float>(d * d);
    b.w1T[i] = ar.take<float>(d * d);
    b.wzT[i] = ar.take<float>(L * d);
  }
  b.xv = ar.take<float>(R * d);
  b.hlast = ar.take<float>(R * d);
  b.dh = ar.take<float>(R * d);
  b.dhv = ar.take<float>(R * d);
  b.T = ar.take<float>(R * d);
  b.T2 = ar.take<float>(R * d);
  b.tA = ar.take<float>((d > L ? d : L) * Rp);
  b.tB = ar.take<float>((d > L ? d : L) * Rp);
  b.dlat = ar.take<float>(R * L);
  b.dfeat = ar.take<float>(R * 48);
  b.do4 = ar.take<float>((size_t)pad16((int)cp) * 4);
  b.w_in = ar.take<float>(d * 48);
  b.w_inT = ar.take<float>(48 * d);
  b.tmp_win = ar.take<float>(d * 48);
  b.cam_acc = ar.take<float>((size_t)sc.SB * sc.NS * 16);
  b.splitk_bytes = det ? splitk_budget((int64_t)R, (int)d, (int)L) : 0;
  b.splitk = det ? ar.take<float>(b.splitk_bytes / sizeof(float)) : nullptr;
  b.lat_fixed = det ? ar.take<long long>((size_t)sc.SB * sc.NS * sc.Hl * sc.Wl * sc.C) : nullptr;
  b.m_bits = det ? ar.take<unsigned>(1) : nullptr;
  return ar.off;
}

}  // namespace bwd

size_t field_backward_workspace_bytes(const PnrScene& sc, const PnrMlp& mlp, int64_t total_points) {
  Arena ar(nullptr, (size_t)-1);
  bwd::Bufs b;
  return bwd::carve(ar, b, sc, mlp, bwd::chunk_points(sc, total_points), deterministic()) + 4096;
}

#define BW(expr)                \
  do {                          \
    int _rc = (expr);           \
    if (_rc) return _rc;        \
  } while (0)

int field_backward(const PnrScene& sc, const PnrMlp& mlp, const PointSource& src, int64_t total_points,
                   const float* d_out, const PnrMlp& grad, float* d_latent, float* d_xyz, float* d_dirs,
                   const PnrCameraGrad* cam, void* ws, size_t ws_bytes, cudaStream_t s, bool sel) {
  using namespace bwd;
  PNR_CHECK_ARG(mlp.d_in == 42 && mlp.d_out == 4, "backward expects d_in == 42, d_out == 4");
  PNR_CHECK_ARG(mlp.d_hidden % 16 == 0 && mlp.d_latent % 16 == 0, "d_hidden and d_latent must be multiples of 16");
  PNR_CHECK_ARG(mlp.d_latent == sc.C, "latent channel mismatch");
  PNR_CHECK_ARG(mlp.n_blocks <= PNR_MAX_BLOCKS, "too many blocks");
  const int d = mlp.d_hidden, L = mlp.d_latent, NS = sc.NS, nb = mlp.n_blocks;
  const int comb = mlp.combine_layer < nb ? mlp.combine_layer : nb;
  if (mlp.combine_layer >= nb && NS > 1) {
    set_error("combine_layer >= n_blocks with NS > 1 is not supported");
    return PNR_ERR_UNSUPPORTED;
  }
  if (ws_bytes < field_backward_workspace_bytes(sc, mlp, total_points)) {
    set_error("workspace too small: %zu < %zu", ws_bytes, field_backward_workspace_bytes(sc, mlp, total_points));
    return PNR_ERR_WORKSPACE;
  }
  const bool det = deterministic();
  if (det && d_latent && !latent_scatter_fixed) {
    set_error("deterministic mode is not available in this build");
    return PNR_ERR_UNSUPPORTED;
  }
  const int64_t cp = chunk_points(sc, total_points);
  Arena ar(ws, ws_bytes);
  Bufs b;
  carve(ar, b, sc, mlp, cp, det);
  SplitKScope splitk(b.splitk, b.splitk_bytes);
  const bool want_cam = cam && (cam->d_poses || cam->d_focal || cam->d_c);
  const int V = sc.SB * NS;

  // The plan of a selective call (sel: the _sel entry points): which of the backward's steps its wanted gradients need
  // (a NULL member of grad is frozen).  The input-gradient chain runs top down through the stages fc_1, fc_0, lin_z of
  // each block, then lin_in; stage(blk, j) numbers them in that order.  It has to deliver dY to the lowest stage with a
  // wanted tensor, and all the way down when an input gradient is wanted.  Other calls run every step.
  auto stage = [&](int blk, int j) { return (nb - 1 - blk) * 3 + j; };
  const int lin_in_stage = nb * 3;
  const bool want_dlat = !sel || d_latent || d_xyz || want_cam;     // k_geom_bwd reads dlat for the scatter and d uv
  const bool want_geom = want_dlat || d_dirs;
  const bool want_lin_out = grad.lin_out_w || grad.lin_out_b;
  int reach = want_geom || grad.lin_in_w || grad.lin_in_b ? lin_in_stage : -1;
  for (int blk = 0; blk < nb; ++blk) {
    if (grad.fc1_w[blk] || grad.fc1_b[blk]) reach = reach > stage(blk, 0) ? reach : stage(blk, 0);
    if (grad.fc0_w[blk] || grad.fc0_b[blk]) reach = reach > stage(blk, 1) ? reach : stage(blk, 1);
    if (blk < comb && (grad.lin_z_w[blk] || grad.lin_z_b[blk])) reach = reach > stage(blk, 2) ? reach : stage(blk, 2);
  }
  if (!want_lin_out && reach < 0) return PNR_OK;             // nothing wanted: no recompute either
  if (want_cam) PNR_CUDA(cudaMemsetAsync(b.cam_acc, 0, (size_t)V * 16 * sizeof(float), s));

  // transposed weights, once per call: W [out][in] -> W^T [in][out]; only those of the dX steps the chain runs
  k_pad_rows<<<(d * 48 + 255) / 256, 256, 0, s>>>(mlp.lin_in_w, b.w_in, d, mlp.d_in, 48);
  PNR_LAUNCH_CHECK();
  if (want_geom) BW(transpose_pad<false>(b.w_in, 48, d, 48, b.w_inT, d, s));
  for (int i = 0; i < nb; ++i) {
    if (reach >= stage(i, 2)) BW(transpose_pad<false>(mlp.fc0_w[i], d, d, d, b.w0T[i], d, s));
    if (reach >= stage(i, 1)) BW(transpose_pad<false>(mlp.fc1_w[i], d, d, d, b.w1T[i], d, s));
    if (i < comb && want_dlat) BW(transpose_pad<false>(mlp.lin_z_w[i], L, d, L, b.wzT[i], d, s));
  }

  for (int64_t g0 = 0; g0 < total_points; g0 += cp) {
    const int64_t n = (total_points - g0 < cp) ? (total_points - g0) : cp;
    const int R = (int)(n * NS), Rp = pad16(R);
    // ---------------- forward again, keeping block inputs (hpre) and fc_0 outputs (nbuf) ----------------
    BW(launch_build_rows(sc, src, g0, n, b.feat, b.lat, s));
    auto dst_of = [&](int blk) -> float* {
      if (blk == nb) return b.hlast;
      if (blk == comb && NS > 1 && comb < nb) return b.xv;
      return b.hpre[blk];
    };
    float* cur = dst_of(0);
    int rows_cur = R;
    BW(fwd_gemm(b.feat, 48, b.w_in, mlp.lin_in_b, cur, d, R, d, 48, false, false, s));
    for (int blk = 0; blk < nb; ++blk) {
      if (blk == comb && comb < nb) {
        if (NS > 1) {
          k_view_mean<<<(unsigned)((n * d + 255) / 256), 256, 0, s>>>(b.xv, b.hpre[blk], n, NS, d);
          PNR_LAUNCH_CHECK();
          cur = b.hpre[blk];
        }
        rows_cur = (int)n;
      }
      if (blk < comb) BW(fwd_gemm(b.lat, L, mlp.lin_z_w[blk], mlp.lin_z_b[blk], cur, d, rows_cur, d, L, false, true, s));
      BW(fwd_gemm(cur, d, mlp.fc0_w[blk], mlp.fc0_b[blk], b.nbuf[blk], d, rows_cur, d, d, true, false, s));
      float* nxt = dst_of(blk + 1);
      PNR_CUDA(cudaMemcpyAsync(nxt, cur, (size_t)rows_cur * d * sizeof(float), cudaMemcpyDeviceToDevice, s));
      BW(fwd_gemm(b.nbuf[blk], d, mlp.fc1_w[blk], mlp.fc1_b[blk], nxt, d, rows_cur, d, d, true, true, s));
      cur = nxt;
    }
    // ---------------- backward ----------------
    const int rows_last = rows_cur, rlp = pad16(rows_last);
    k_lin_out_bwd<<<(unsigned)(((int64_t)rows_last * 32 + 255) / 256), 256, 0, s>>>(
        b.hlast, mlp.lin_out_w, mlp.lin_out_b, d_out + g0 * 4, b.do4, b.dh, rows_last, d);
    PNR_LAUNCH_CHECK();
    if (want_lin_out) BW(transpose_pad<false>(b.do4, 4, rows_last, 4, b.tA, rlp, s));
    if (grad.lin_out_w) {
      BW(transpose_pad<true>(b.hlast, d, rows_last, d, b.tB, rlp, s));
      BW(gemm(b.tA, rlp, b.tB, nullptr, const_cast<float*>(grad.lin_out_w), d, 4, d, rlp, false, true, s));
    }
    if (grad.lin_out_b) BW(rowsum_acc(b.tA, rlp, 4, const_cast<float*>(grad.lin_out_b), s));
    if (want_dlat) PNR_CUDA(cudaMemsetAsync(b.dlat, 0, (size_t)R * L * sizeof(float), s));
    bool lat_transposed = false;
    float* dh = b.dh;
    float* dh_other = b.dhv;
    for (int blk = nb - 1; blk >= 0 && reach >= stage(blk, 0); --blk) {
      const int rows_b = (blk >= comb && comb < nb) ? (int)n : R;
      const int Mp = pad16(rows_b);
      const int64_t cnt = (int64_t)rows_b * d;
      const unsigned eg = (unsigned)((cnt + 255) / 256);
      // fc_1: dW1 += dh^T relu(n), db1 += colsum(dh); dn = (dh W1) * (n > 0)
      if (grad.fc1_w[blk] || grad.fc1_b[blk]) BW(transpose_pad<false>(dh, d, rows_b, d, b.tA, Mp, s));
      if (grad.fc1_w[blk]) {
        BW(transpose_pad<true>(b.nbuf[blk], d, rows_b, d, b.tB, Mp, s));
        BW(gemm(b.tA, Mp, b.tB, nullptr, const_cast<float*>(grad.fc1_w[blk]), d, d, d, Mp, false, true, s));
      }
      if (grad.fc1_b[blk]) BW(rowsum_acc(b.tA, Mp, d, const_cast<float*>(grad.fc1_b[blk]), s));
      if (reach < stage(blk, 1)) break;
      if (use_tc_gemm()) {   // the ReLU mask rides in the GEMM's epilogue
        BW(gemm_bf16x3_masked(dh, d, b.w1T[blk], d, b.T, d, rows_b, d, d, false, b.nbuf[blk], s));
      } else {
        BW(gemm(dh, d, b.w1T[blk], nullptr, b.T, d, rows_b, d, d, false, false, s));
        k_mask<<<eg, 256, 0, s>>>(b.T, b.nbuf[blk], cnt);
        PNR_LAUNCH_CHECK();
      }
      // fc_0: dW0 += dn^T relu(hpre), db0 += colsum(dn); dh += (dn W0) * (hpre > 0)
      if (grad.fc0_w[blk] || grad.fc0_b[blk]) BW(transpose_pad<false>(b.T, d, rows_b, d, b.tA, Mp, s));
      if (grad.fc0_w[blk]) {
        BW(transpose_pad<true>(b.hpre[blk], d, rows_b, d, b.tB, Mp, s));
        BW(gemm(b.tA, Mp, b.tB, nullptr, const_cast<float*>(grad.fc0_w[blk]), d, d, d, Mp, false, true, s));
      }
      if (grad.fc0_b[blk]) BW(rowsum_acc(b.tA, Mp, d, const_cast<float*>(grad.fc0_b[blk]), s));
      if (reach < stage(blk, 2)) break;
      if (use_tc_gemm()) {
        BW(gemm_bf16x3_masked(b.T, d, b.w0T[blk], d, dh, d, rows_b, d, d, true, b.hpre[blk], s));
      } else {
        BW(gemm(b.T, d, b.w0T[blk], nullptr, b.T2, d, rows_b, d, d, false, false, s));
        k_mask_add<<<eg, 256, 0, s>>>(dh, b.T2, b.hpre[blk], cnt);
        PNR_LAUNCH_CHECK();
      }
      if (blk < comb) {   // x = x + lin_z[blk](latent): dWz += dh^T lat, dbz += colsum(dh), dlat += dh Wz
        if (grad.lin_z_w[blk] && !lat_transposed) {
          BW(transpose_pad<false>(b.lat, L, R, L, b.latT, Rp, s));
          lat_transposed = true;
        }
        if (grad.lin_z_w[blk] || grad.lin_z_b[blk]) BW(transpose_pad<false>(dh, d, R, d, b.tA, Rp, s));
        if (grad.lin_z_w[blk])
          BW(gemm(b.tA, Rp, b.latT, nullptr, const_cast<float*>(grad.lin_z_w[blk]), L, d, L, Rp, false, true, s));
        if (grad.lin_z_b[blk]) BW(rowsum_acc(b.tA, Rp, d, const_cast<float*>(grad.lin_z_b[blk]), s));
        if (want_dlat) BW(gemm(dh, d, b.wzT[blk], nullptr, b.dlat, L, R, L, d, false, true, s));
      }
      if (blk == comb && comb < nb && NS > 1 && reach > stage(blk, 2)) {   // the block's input was the mean over views
        k_view_mean_bwd<<<(unsigned)(((int64_t)R * d + 255) / 256), 256, 0, s>>>(dh, dh_other, n, NS, d);
        PNR_LAUNCH_CHECK();
        float* t = dh; dh = dh_other; dh_other = t;
      }
    }
    // lin_in: dW += dh^T feat (42 of the 48 padded columns), db += colsum(dh), dfeat = dh W_in
    if (grad.lin_in_w || grad.lin_in_b) BW(transpose_pad<false>(dh, d, R, d, b.tA, Rp, s));
    if (grad.lin_in_w) {
      BW(transpose_pad<false>(b.feat, 48, R, 48, b.featT, Rp, s));
      BW(gemm(b.tA, Rp, b.featT, nullptr, b.tmp_win, 48, d, 48, Rp, false, false, s));
      k_add_cols<<<(d * mlp.d_in + 255) / 256, 256, 0, s>>>(const_cast<float*>(grad.lin_in_w), b.tmp_win, d, mlp.d_in,
                                                            48);
      PNR_LAUNCH_CHECK();
    }
    if (grad.lin_in_b) BW(rowsum_acc(b.tA, Rp, d, const_cast<float*>(grad.lin_in_b), s));
    if (!want_geom) continue;
    BW(gemm(dh, d, b.w_inT, nullptr, b.dfeat, 48, R, 48, d, false, false, s));
    float* cam_part = want_cam ? b.T : nullptr;    // [R][16]; T (R x d, d >= 16) is free again here
    k_geom_bwd<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(sc, src, g0, n, b.dfeat, want_dlat ? b.dlat : nullptr,
                                                               det ? nullptr : d_latent, d_xyz, d_dirs, cam_part);
    PNR_LAUNCH_CHECK();
    if (det && d_latent) BW(latent_scatter_fixed(sc, src, g0, n, b.dlat, d_latent, b.lat_fixed, b.m_bits, s));
    if (want_cam) {
      k_cam_reduce<<<V, kCamThreads, 0, s>>>(cam_part, g0, n, src.P, NS, b.cam_acc);
      PNR_LAUNCH_CHECK();
    }
  }
  if (want_cam) {
    k_cam_finish<<<1, 256, 0, s>>>(b.cam_acc, V, NS, sc.n_focal, sc.n_c, cam->d_poses, cam->d_focal, cam->d_c);
    PNR_LAUNCH_CHECK();
  }
  return PNR_OK;
}

}  // namespace pnr
