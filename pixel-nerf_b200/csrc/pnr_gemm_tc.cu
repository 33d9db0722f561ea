// Split-bf16 tensor-core GEMM for the training step's backward (SURVEY 8f-1):
//     C[M][N] (+)= act(A[M][lda]) * W[N][K]^T (+ bias),   fp32 in, fp32 out, fp32 accumulate
// i.e. the signature of the SIMT `sgemm` (pnr_field_simt.cu) it replaces inside field_backward: the recomputed forward
// layers, dX = dY W (on W^T) and dW += dY^T X (on transposed panels, K = rows, split-K).
//
// wgmma (sm_90a warpgroup MMA, m64n128k16 with BF16 operands), accumulators in registers.  Each fp32 operand
// is split on the fly into an error-compensated bf16 pair x = hi + lo (16 mantissa bits; bf16 keeps fp32's exponent
// range, so the tiny values of a backward pass need no scaling) and D += Ahi*Bhi + Alo*Bhi + Ahi*Blo: 3 tensor
// passes per GEMM, measured worst relative gradient error 1.4e-5 (scripts/precision_study_backward.py), two orders
// below the 1e-3 the gradient tests allow.
//
// CTA = 2 warpgroups, one 128x128 output tile over a K range; every thread loads, splits and consumes:
//   load     : coalesced LDG.128 of the fp32 operands -> (ReLU) -> bf16 hi/lo -> st.shared into K-major
//              128B-swizzled tiles (the layout pnr_field_tc.cu uses), 3-stage ring
//   MMA      : each warpgroup issues 12 wgmma per 64-wide k-step for its 64 rows and keeps one k-step in flight
//              while the next one is loaded
//   epilogue : registers -> (+ bias) -> store / read-add-store / red.global.add (split-K); in deterministic mode a
//              split stores its partial tile and k_splitk_sum adds the partials in split order
// Roofline: tensor-bound for large K, but both operands arrive as fp32 through L2 (8 B per bf16-pair element), so
// the practical bound is L2->SM bandwidth: 64 KB of operands per 1 M MAC k-step.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "pnr_common.cuh"
#include "pnr_tc_ptx.cuh"

namespace pnr {

namespace gemmtc {

using namespace tcptx;

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int STAGES = 3;
constexpr int TILE_BYTES = 128 * 128;          // 128 rows x 64 bf16
constexpr int STAGE_BYTES = 4 * TILE_BYTES;    // A hi, A lo, B hi, B lo
constexpr int NTHREADS = 256;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES;

struct Params {
  const float* A;
  const float* W;
  const float* bias;
  float* C;
  int lda, ldw, ldc, M, N, K;
  int k_per_split;   // multiple of BK
  int relu_a, mode;  // mode 0: store, 1: C += (single split), 2: atomic add (split-K), 3: store into part (split-K)
  const float* mask; // optional [M][ldc]: the product is zeroed where mask <= 0 (ReLU backward) before store / add
  float* part;       // mode 3: [splits][M][N] partial tiles
};

// 8 fp32 values -> error-compensated 16-bit pairs x = hi + lo.  BF16: 8 + 8 mantissa bits with fp32's exponent range
// (gradient-sized values need no scaling).  F16: 11 + 11 bits for values inside fp16's range (|x| < 65504; low parts
// below 6e-5 go subnormal, i.e. an ABSOLUTE error floor of 3e-8): the per-encode projection of the latent.
template <bool BF16>
__device__ __forceinline__ void split8(const float4 a, const float4 b, bool relu, uint4& hi, uint4& lo) {
  float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float x0 = x[2 * i], x1 = x[2 * i + 1];
    if (relu) {
      x0 = fmaxf(x0, 0.f);
      x1 = fmaxf(x1, 0.f);
    }
    if (BF16) {
      asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h[i]) : "f"(x1), "f"(x0));
      const float r0 = x0 - __uint_as_float(h[i] << 16);
      const float r1 = x1 - __uint_as_float(h[i] & 0xFFFF0000u);
      asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(l[i]) : "f"(r1), "f"(r0));
    } else {
      asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h[i]) : "f"(x1), "f"(x0));
      const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&h[i]));
      asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(l[i]) : "f"(x1 - hf.y), "f"(x0 - hf.x));
    }
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

template <bool BF16>
__global__ void __launch_bounds__(NTHREADS, 1) k_gemm_split3(const __grid_constant__ Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int t = threadIdx.x, wg = t >> 7, warp = t >> 5, lane = t & 31;
  const uint32_t smem_u = smem_u32(smem);
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int k_begin = blockIdx.z * p.k_per_split;
  const int k_end = min(p.K, k_begin + p.k_per_split);
  const int nk = (k_end - k_begin + BK - 1) / BK;
  if (nk <= 0) return;   // (cannot happen with the host's split computation; uniform over the CTA)

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  const uint64_t desc0 = make_desc(0);
  for (int it = 0; it < nk; ++it) {
    const int st = it % STAGES;
    const int k0 = k_begin + it * BK;
    // all 16 loads in flight before the first use
    float4 va[4][2], vb[4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int id = t + 256 * i, row = id >> 3, u = id & 7;
      const int k = k0 + u * 8;
      const bool ka = k < k_end;
      const int m = m0 + row, n = n0 + row;
      if (ka && m < p.M) {
        const float4* src = reinterpret_cast<const float4*>(p.A + (size_t)m * p.lda + k);
        va[i][0] = __ldg(src);
        va[i][1] = __ldg(src + 1);
      } else {
        va[i][0] = va[i][1] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (ka && n < p.N) {
        const float4* src = reinterpret_cast<const float4*>(p.W + (size_t)n * p.ldw + k);
        vb[i][0] = __ldg(src);
        vb[i][1] = __ldg(src + 1);
      } else {
        vb[i][0] = vb[i][1] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    // stage `st` was last read by the wgmma of step it - STAGES, which both warpgroups waited for (wait_group 1 at
    // the end of step it - STAGES + 1) before the barrier of step it - 1
    const uint32_t sbase = smem_u + st * STAGE_BYTES;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int id = t + 256 * i, row = id >> 3, u = id & 7;
      const uint32_t off = (uint32_t)(row * 128 + ((u ^ (row & 7)) * 16));
      uint4 hi, lo;
      split8<BF16>(va[i][0], va[i][1], p.relu_a != 0, hi, lo);
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sbase + off), "r"(hi.x), "r"(hi.y), "r"(hi.z), "r"(hi.w) : "memory");
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sbase + TILE_BYTES + off), "r"(lo.x), "r"(lo.y), "r"(lo.z), "r"(lo.w) : "memory");
      split8<BF16>(vb[i][0], vb[i][1], false, hi, lo);
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sbase + 2 * TILE_BYTES + off), "r"(hi.x), "r"(hi.y), "r"(hi.z), "r"(hi.w) : "memory");
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sbase + 3 * TILE_BYTES + off), "r"(lo.x), "r"(lo.y), "r"(lo.z), "r"(lo.w) : "memory");
    }
    fence_proxy_async();
    __syncthreads();
    // warpgroup wg: rows [64 wg, 64 wg + 64) of the A tile against all 128 rows of the B tile
    const uint64_t a_hi = desc0 + ((sbase + wg * (TILE_BYTES / 2)) >> 4), a_lo = a_hi + (TILE_BYTES >> 4);
    const uint64_t b_hi = desc0 + ((sbase + 2 * TILE_BYTES) >> 4), b_lo = b_hi + (TILE_BYTES >> 4);
    fence_acc<64>(acc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      if (BF16) {
        wgmma_m64n128_bf16(acc, a_hi + 2 * kk, b_hi + 2 * kk, (it | kk) ? 1u : 0u);
        wgmma_m64n128_bf16(acc, a_lo + 2 * kk, b_hi + 2 * kk, 1u);
        wgmma_m64n128_bf16(acc, a_hi + 2 * kk, b_lo + 2 * kk, 1u);
      } else {
        wgmma_m64n128_f16(acc, a_hi + 2 * kk, b_hi + 2 * kk, (it | kk) ? 1u : 0u);
        wgmma_m64n128_f16(acc, a_lo + 2 * kk, b_hi + 2 * kk, 1u);
        wgmma_m64n128_f16(acc, a_hi + 2 * kk, b_lo + 2 * kk, 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();
    fence_acc<64>(acc);
  }
  wgmma_wait<0>();
  fence_acc<64>(acc);

  // ------------------------------ epilogue ------------------------------
  const bool add_bias = p.bias != nullptr && blockIdx.z == 0;
  const int rbase = m0 + wg * 64 + 16 * (warp & 3) + (lane >> 2);
  const int cbase = n0 + 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int m = rbase + 8 * ((i >> 1) & 1);
    const int n = cbase + 8 * (i >> 2) + (i & 1);
    if (m >= p.M || n >= p.N) continue;
    float o = acc[i];
    if (p.mask && !(p.mask[(size_t)m * p.ldc + n] > 0.f)) o = 0.f;
    if (add_bias) o += __ldg(p.bias + n);
    if (p.mode == 3) {
      p.part[((size_t)blockIdx.z * p.M + m) * p.N + n] = o;
      continue;
    }
    float* dst = p.C + (size_t)m * p.ldc + n;
    if (p.mode == 2) atomicAdd(dst, o);
    else if (p.mode == 1) *dst += o;
    else *dst = o;
  }
}

// C (+)= ((P0 + P1) + P2) + ...: the partial tiles of an ordered split-K, summed in split order
__global__ void k_splitk_sum(const float* __restrict__ part, int splits, int M, int N, float* __restrict__ C, int ldc,
                             int accum) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t mn = (int64_t)M * N;
  if (i >= mn) return;
  float s = part[i];
  for (int z = 1; z < splits; ++z) s += part[z * mn + i];
  float* dst = C + (i / N) * ldc + i % N;
  if (accum) *dst += s;
  else *dst = s;
}

}  // namespace gemmtc

static int gemm_split3(bool bf16, const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc,
                       int M, int N, int K, bool relu_a, bool accum, const float* mask, cudaStream_t s) {
  using namespace gemmtc;
  if (M == 0 || N == 0) return PNR_OK;
  if (K % 16 != 0 || lda % 4 != 0 || ldw % 4 != 0 || ((uintptr_t)A & 15) || ((uintptr_t)W & 15)) {
    set_error("tensor-core gemm: K must be a multiple of 16 and the operands 16-byte aligned");
    return PNR_ERR_INVALID;
  }
  Params p;
  p.A = A; p.W = W; p.bias = bias; p.C = C;
  p.lda = lda; p.ldw = ldw; p.ldc = ldc; p.M = M; p.N = N; p.K = K;
  p.relu_a = relu_a ? 1 : 0;
  p.mask = mask;
  if (mask && bias) {
    set_error("tensor-core gemm: mask and bias together are not supported");
    return PNR_ERR_INVALID;
  }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
  const int ksteps = (K + BK - 1) / BK;
  // split K when the output has too few tiles to fill the GPU (the weight-gradient GEMMs: 512 x 512 over K = rows)
  int splits = 1;
  if (tiles < sms && ksteps >= 8) {
    splits = (2 * sms + tiles - 1) / tiles;
    if (splits > ksteps / 4) splits = ksteps / 4;
    if (splits < 1) splits = 1;
  }
  // deterministic mode: the partials go to the installed scratch and are summed in order; never more splits than it
  // holds (none installed: no split)
  const bool ordered = splits > 1 && deterministic();
  if (ordered) {
    const size_t fit = splitk_scratch().bytes / ((size_t)M * N * sizeof(float));
    if ((size_t)splits > fit) splits = fit > 1 ? (int)fit : 1;
  }
  const int steps_per = (ksteps + splits - 1) / splits;
  splits = (ksteps + steps_per - 1) / steps_per;
  p.k_per_split = steps_per * BK;
  p.mode = splits > 1 ? (ordered ? 3 : 2) : (accum ? 1 : 0);
  p.part = p.mode == 3 ? splitk_scratch().p : nullptr;
  if (p.mode == 2 && !accum) PNR_CUDA(cudaMemset2DAsync(C, (size_t)ldc * 4, 0, (size_t)N * 4, (size_t)M, s));
  static bool attr_set[64] = {false};
  if (dev >= 0 && dev < 64 && !attr_set[dev]) {
    PNR_CUDA(cudaFuncSetAttribute(k_gemm_split3<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    PNR_CUDA(cudaFuncSetAttribute(k_gemm_split3<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_set[dev] = true;
  }
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM, splits);
  prof_before(s);
  if (bf16) k_gemm_split3<true><<<grid, NTHREADS, SMEM_BYTES, s>>>(p);
  else k_gemm_split3<false><<<grid, NTHREADS, SMEM_BYTES, s>>>(p);
  prof_after(s);
  PNR_LAUNCH_CHECK();
  if (p.mode == 3) {
    const int64_t mn = (int64_t)M * N;
    k_splitk_sum<<<(unsigned)((mn + 255) / 256), 256, 0, s>>>(p.part, splits, M, N, C, ldc, accum ? 1 : 0);
    PNR_LAUNCH_CHECK();
  }
  return PNR_OK;
}

// Same contract as sgemm() (pnr_field_simt.cu) plus `ldw` (row stride of W).  K % 16 == 0, 16-byte aligned rows.
int gemm_bf16x3(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc, int M, int N,
                int K, bool relu_a, bool accum, cudaStream_t s) {
  return gemm_split3(true, A, lda, W, ldw, bias, C, ldc, M, N, K, relu_a, accum, nullptr, s);
}
// ... with the ReLU-backward mask fused into the epilogue: C (+)= (A W^T) * (mask > 0), mask laid out like C
int gemm_bf16x3_masked(const float* A, int lda, const float* W, int ldw, float* C, int ldc, int M, int N, int K, bool accum,
                       const float* mask, cudaStream_t s) {
  return gemm_split3(true, A, lda, W, ldw, nullptr, C, ldc, M, N, K, false, accum, mask, s);
}
// fp16 hi/lo operands (22 mantissa bits inside fp16's range): the per-encode projection of the latent
int gemm_f16x3(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc, int M, int N, int K,
               cudaStream_t s) {
  return gemm_split3(false, A, lda, W, ldw, bias, C, ldc, M, N, K, false, false, nullptr, s);
}

}  // namespace pnr
