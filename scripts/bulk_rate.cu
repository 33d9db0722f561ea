// Micro-benchmark: L2 -> shared-memory cp.async.bulk streaming (16 KB copies) with all 132 SMs reading the SAME
// 10 MB weight image (as the tensor engine does), N slots in flight per SM.  Reports cycles per copy.
#include <cstdio>
#include <cuda_runtime.h>
#include "pnr_tc_ptx.cuh"
using namespace pnr::tcptx;

template <int N>
__global__ void __launch_bounds__(64, 1) k_stream(const uint8_t* src, size_t src_bytes, int copies, long long* out, int stagger) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(8) unsigned long long bars[N];
  if (threadIdx.x == 0) {
    for (int i = 0; i < N; ++i) mbar_init(smem_u32(&bars[i]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int st = 0;
    const size_t nslots = src_bytes / 16384;
    size_t idx = stagger ? (size_t)blockIdx.x * 37 % nslots : 0;
    const long long t0 = clock64();
    for (int i = 0; i < copies + N; ++i) {
      const int sl = i % N;
      if (i >= N) mbar_wait(smem_u32(&bars[sl]), ((i / N) - 1) & 1, &st, 1);   // previous copy into this slot landed
      if (i < copies) {
        mbar_expect_tx(smem_u32(&bars[sl]), 16384);
        bulk_g2s(smem_u32(smem) + sl * 16384, src + idx * 16384, 16384, smem_u32(&bars[sl]));
        idx = (idx + 1) % nslots;
      }
    }
    const long long t1 = clock64();
    if (blockIdx.x == 0) out[0] = t1 - t0;
  }
}

template <int N>
void run(const uint8_t* src, size_t bytes, int stagger, int grid = 132) {
  long long* d; cudaMalloc(&d, 8);
  auto kern = k_stream<N>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, N * 16384);
  const int copies = 4000;
  for (int rep = 0; rep < 2; ++rep) kern<<<grid, 64, N * 16384>>>(src, bytes, copies, d, stagger);
  cudaError_t e = cudaDeviceSynchronize();
  long long c = 0; cudaMemcpy(&c, d, 8, cudaMemcpyDeviceToHost);
  double per = (double)c / copies;
  printf("grid %3d slots %2d stagger %d: %8.1f cycles per 16 KB copy -> %6.1f B/cycle/SM (%s)\n", grid, N, stagger, per, 16384.0 / per, cudaGetErrorString(e));
  cudaFree(d);
}

int main() {
  const size_t bytes = 10u << 20;
  uint8_t* src; cudaMalloc(&src, bytes); cudaMemset(src, 1, bytes);
  run<1>(src, bytes, 0); run<2>(src, bytes, 0); run<4>(src, bytes, 0); run<6>(src, bytes, 0); run<8>(src, bytes, 0); run<12>(src, bytes, 0);
  run<1>(src, bytes, 1); run<6>(src, bytes, 1); run<12>(src, bytes, 1);
  run<6>(src, bytes, 1, 8); run<6>(src, bytes, 1, 32); run<6>(src, bytes, 1, 74); run<12>(src, bytes, 1, 8); run<12>(src, bytes, 1, 37);
  return 0;
}
