// Fixed-order variants of deterministic mode (pnr_set_deterministic, include/pnr.h):
//
//  * the latent gradient of a field-backward chunk, added in 64-bit fixed point instead of with float atomics.
//    Arithmetic (restated by oracle/pnr_determinism.py):
//      m     = max |d_lat| over the chunk's finite entries        (integer atomicMax on the fp32 bits: exact, order-free)
//      e     = 62 - ceil(log2(n_max)) - E,  m = f 2^E, f in [0.5, 1),  n_max = 4 * rows of the chunk
//      term  = d_lat[row][c] * w_tap                              (the fp32 product k_geom_bwd adds)
//      acc  += round_half_even((double)term * 2^e)                 (int64 atomicAdd: exact, so order-free)
//      d_latent += (float)((double)acc * 2^-e)                     (per chunk, in stream order)
//    |term| <= m (w_tap <= 1) and one texel takes at most n_max terms, so |acc| <= n_max 2^(62 - ceil log2 n_max)
//    <= 2^62: no overflow, also when every point clamps onto one border texel.  Each term is rounded once at 2^-e,
//    i.e. by at most m 2^(ceil log2 n_max - 63) (2^-45 m at 32 k rows).
//    A non-finite term instead stores NaN into every d_latent element it reaches (plain stores of one value, so the
//    result is the same whatever the order), and the later conversion adds to NaN.
//  * the backward of align_corners=True bilinear upsampling (the encoder's F.interpolate) as a gather.
//
// Integer atomics and the rounding intrinsics are the only device-specific operations; the host emulator of
// tests/determ_emu.py supplies them.
#include <math.h>

#include "pnr_geom.cuh"

namespace pnr {

namespace determ {

// out = max over finite x of the bits of |x| (the order of non-negative floats is that of their bits); a warp
// reduces its elements first, so there is one atomic per warp
__global__ void k_finite_absmax(const float* __restrict__ x, int64_t n, unsigned* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned b = i < n ? __float_as_uint(x[i]) & 0x7fffffffu : 0u;
  if (b >= 0x7f800000u) b = 0u;
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned t = __shfl_xor_sync(0xffffffffu, b, o);
    b = t > b ? t : b;
  }
  if ((threadIdx.x & 31) == 0 && b != 0u) atomicMax(out, b);
}

// 2^e of a chunk whose finite |d_lat| <= m: n_max m 2^e < 2^62 with n_max <= 2^log2_nmax
__device__ __forceinline__ int fixed_exponent(unsigned m_bits, int log2_nmax) {
  int E = 0;
  frexpf(__uint_as_float(m_bits), &E);
  return 62 - log2_nmax - E;
}

__device__ __forceinline__ void add_tap(long long* acc, float* d_latent, size_t o, float term, double scale) {
  if (isfinite(term)) {
    atomicAdd(reinterpret_cast<unsigned long long*>(acc + o), (unsigned long long)__double2ll_rn((double)term * scale));
  } else {
    d_latent[o] = __int_as_float(0x7fffffff);
  }
}

// One warp per point, the taps of k_geom_bwd; row = local_point * NS + view
__global__ void k_latent_scatter_fixed(PnrScene sc, PointSource src, int64_t g0, int64_t n_pts,
                                       const float* __restrict__ d_lat, const unsigned* __restrict__ m_bits,
                                       int log2_nmax, long long* __restrict__ acc, float* __restrict__ d_latent) {
  const int64_t lp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (lp >= n_pts) return;
  const int64_t g = g0 + lp;
  const int sb = (int)(g / src.P);
  float x[3], dir[3];
  load_point(src, g, x, dir);
  const double scale = ldexp(1.0, fixed_exponent(*m_bits, log2_nmax));
  for (int v = 0; v < sc.NS; ++v) {
    const BwdTaps t = bwd_taps(sc, sb, v, x);
    const float* dl = d_lat + (lp * sc.NS + v) * sc.C;
    for (int c = lane; c < sc.C; c += 32) {
      const float gdl = dl[c];
      add_tap(acc, d_latent, t.o_nw + c, gdl * t.w_nw, scale);
      if (t.vx1) add_tap(acc, d_latent, t.o_ne + c, gdl * t.w_ne, scale);
      if (t.vy1) add_tap(acc, d_latent, t.o_sw + c, gdl * t.w_sw, scale);
      if (t.vx1 && t.vy1) add_tap(acc, d_latent, t.o_se + c, gdl * t.w_se, scale);
    }
  }
}

// d_latent += acc 2^-e  (int64 -> double and double -> float round to nearest even; the scaling is exact)
__global__ void k_fixed_to_float(const long long* __restrict__ acc, const unsigned* __restrict__ m_bits, int log2_nmax,
                                 int64_t n, float* __restrict__ d_latent) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long a = acc[i];
  if (a == 0) return;
  const double inv = ldexp(1.0, -fixed_exponent(*m_bits, log2_nmax));
  d_latent[i] += __double2float_rn(__ll2double_rn(a) * inv);
}

// d_in[n][c][hi][wi] = sum over output pixels (oh, ow) ascending, then over their taps (h-tap major) that land on
// (hi, wi), of (h_lambda * w_lambda) * d_out[n][c][oh][ow], with torch's source index and lambdas
// (UpSampleBilinear2d.cu: scale = (in - 1) / (out - 1) in fp32, or 0 for out == 1; src = scale * dst).
struct Axis {
  int in, out;
  float scale;
};

__device__ __forceinline__ void axis_tap(const Axis& a, int o, int& i0, int& step, float& l0, float& l1) {
  const float r = __fmul_rn(a.scale, (float)o);
  i0 = (int)r;
  step = (i0 < a.in - 1) ? 1 : 0;
  l1 = __fsub_rn(r, (float)i0);
  l0 = __fsub_rn(1.0f, l1);
}

// output indices whose taps may reach input index i (a superset; the caller tests each)
__device__ __forceinline__ void axis_range(const Axis& a, int i, int& lo, int& hi) {
  if (a.in == 1 || a.out == 1) {
    lo = 0;
    hi = a.out - 1;
    return;
  }
  lo = (int)(((int64_t)(i - 1) * (a.out - 1)) / (a.in - 1)) - 1;
  hi = (int)(((int64_t)(i + 1) * (a.out - 1) + a.in - 2) / (a.in - 1)) + 1;
  lo = lo < 0 ? 0 : lo;
  hi = hi > a.out - 1 ? a.out - 1 : hi;
}

__global__ void k_upsample_ac_bwd(const float* __restrict__ d_out, int64_t planes, Axis ay, Axis ax,
                                  float* __restrict__ d_in) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t per = (int64_t)ay.in * ax.in;
  if (idx >= planes * per) return;
  const int64_t pl = idx / per;
  const int hi = (int)((idx - pl * per) / ax.in), wi = (int)((idx - pl * per) % ax.in);
  const float* src = d_out + pl * ay.out * ax.out;
  if (ay.in == ay.out && ax.in == ax.out) {
    d_in[idx] = src[(int64_t)hi * ax.out + wi];
    return;
  }
  int oh0, oh1, ow0, ow1;
  axis_range(ay, hi, oh0, oh1);
  axis_range(ax, wi, ow0, ow1);
  float s = 0.f;
  for (int oh = oh0; oh <= oh1; ++oh) {
    int h0, hs;
    float hl[2];
    axis_tap(ay, oh, h0, hs, hl[0], hl[1]);
    if (h0 != hi && h0 + hs != hi) continue;
    for (int ow = ow0; ow <= ow1; ++ow) {
      int w0, ws;
      float wl[2];
      axis_tap(ax, ow, w0, ws, wl[0], wl[1]);
      if (w0 != wi && w0 + ws != wi) continue;
      const float g = src[(int64_t)oh * ax.out + ow];
      for (int a = 0; a < 2; ++a) {
        if (h0 + a * hs != hi) continue;
        for (int b = 0; b < 2; ++b)
          if (w0 + b * ws == wi) s = __fadd_rn(s, __fmul_rn(__fmul_rn(hl[a], wl[b]), g));
      }
    }
  }
  d_in[idx] = s;
}

static int ceil_log2(int64_t n) {
  int k = 0;
  while (((int64_t)1 << k) < n) ++k;
  return k;
}

}  // namespace determ

// The latent gradient of one chunk (n points from g0, rows d_lat [n * NS][C]) added into d_latent in fixed point.
// acc: [V][Hl][Wl][C] int64 scratch, m_bits: one word of scratch.
int latent_scatter_fixed(const PnrScene& sc, const PointSource& src, int64_t g0, int64_t n, const float* d_lat,
                         float* d_latent, long long* acc, unsigned* m_bits, cudaStream_t s) {
  using namespace determ;
  const int64_t rows = n * sc.NS, cells = (int64_t)sc.SB * sc.NS * sc.Hl * sc.Wl * sc.C;
  const int log2_nmax = ceil_log2(4 * rows);
  PNR_CUDA(cudaMemsetAsync(acc, 0, (size_t)cells * sizeof(long long), s));
  PNR_CUDA(cudaMemsetAsync(m_bits, 0, sizeof(unsigned), s));
  const int64_t nl = rows * sc.C;
  k_finite_absmax<<<(unsigned)((nl + 255) / 256), 256, 0, s>>>(d_lat, nl, m_bits);
  PNR_LAUNCH_CHECK();
  k_latent_scatter_fixed<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(sc, src, g0, n, d_lat, m_bits, log2_nmax,
                                                                          acc, d_latent);
  PNR_LAUNCH_CHECK();
  k_fixed_to_float<<<(unsigned)((cells + 255) / 256), 256, 0, s>>>(acc, m_bits, log2_nmax, cells, d_latent);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

}  // namespace pnr

using namespace pnr;

extern "C" int pnr_upsample_bilinear_ac_backward(const float* d_out, int64_t N, int32_t C, int32_t h_in, int32_t w_in,
                                                 int32_t h_out, int32_t w_out, float* d_in, void* stream) {
  PNR_CHECK_ARG(N >= 0 && C >= 0 && h_in >= 1 && w_in >= 1 && h_out >= 1 && w_out >= 1, "bad sizes");
  const int64_t n = N * C * h_in * w_in;
  if (n == 0) return PNR_OK;
  PNR_CHECK_ARG(d_out && d_in, "NULL pointer");
  const determ::Axis ay{h_in, h_out, h_out > 1 ? (float)(h_in - 1) / (float)(h_out - 1) : 0.f};
  const determ::Axis ax{w_in, w_out, w_out > 1 ? (float)(w_in - 1) / (float)(w_out - 1) : 0.f};
  determ::k_upsample_ac_bwd<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_out, N * C, ay, ax,
                                                                                          d_in);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}
