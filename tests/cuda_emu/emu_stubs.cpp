// TEST INFRASTRUCTURE: the tensor-engine entry points are not emulated (wgmma has no host meaning); the emulated
// library reports the tensor engine as unavailable so that every call takes the SIMT path.
#include <vector>

#include "pnr_common.cuh"

namespace pnr {
bool tc_supported(const PnrScene&, const PnrMlp&) { return false; }
size_t tc_workspace_bytes(const PnrScene&, const PnrMlp&, int64_t) { return 0; }
int tc_field_eval(const PnrScene&, const PnrMlp&, const float*, const PointSource&, int64_t, float*, void*, size_t,
                  cudaStream_t) {
  set_error("tensor engine is not available in the emulator build");
  return PNR_ERR_UNSUPPORTED;
}
size_t tc_render_workspace_bytes(const PnrScene&, int64_t, int, int) { return 0; }
int tc_render(const PnrScene&, const PnrMlp&, const PnrMlp&, const float*, const float*, const PnrRenderCfg&, const float*,
              const PnrNoise&, float*, float*, float*, const PnrRenderOut&, int64_t, void*, size_t, cudaStream_t) {
  set_error("tensor engine is not available in the emulator build");
  return PNR_ERR_UNSUPPORTED;
}
// the backward's GEMMs run on the fp32 SIMT SGEMM in the emulator (the wgmma GEMM has no host meaning)
int sgemm(const float* A, int lda, const float* W, const float* bias, float* C, int ldc, int M, int N, int K, bool relu_a,
          bool accum, cudaStream_t s);
int gemm_bf16x3(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc, int M, int N, int K,
                bool relu_a, bool accum, cudaStream_t s) {
  if (ldw != K) {
    set_error("emulator gemm: ldw must equal K");
    return PNR_ERR_INVALID;
  }
  return sgemm(A, lda, W, bias, C, ldc, M, N, K, relu_a, accum, s);
}
int gemm_f16x3(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc, int M, int N, int K,
               cudaStream_t s) {
  return gemm_bf16x3(A, lda, W, ldw, bias, C, ldc, M, N, K, false, false, s);
}
// C (+)= (A W^T) * (mask > 0): emulated launches run synchronously on host memory, so a host temporary does
int gemm_bf16x3_masked(const float* A, int lda, const float* W, int ldw, float* C, int ldc, int M, int N, int K, bool accum,
                       const float* mask, cudaStream_t s) {
  std::vector<float> tmp((size_t)M * N);
  int rc = gemm_bf16x3(A, lda, W, ldw, nullptr, tmp.data(), N, M, N, K, false, false, s);
  if (rc) return rc;
  for (int m = 0; m < M; ++m)
    for (int n = 0; n < N; ++n) {
      const float v = mask[(size_t)m * ldc + n] > 0.f ? tmp[(size_t)m * N + n] : 0.f;
      float& c = C[(size_t)m * ldc + n];
      c = accum ? c + v : v;
    }
  return PNR_OK;
}
}  // namespace pnr

extern "C" {
size_t pnr_pack_mlp_bytes(const PnrMlp*) { return 0; }
int pnr_pack_mlp(const PnrMlp*, void*, size_t, void*) { return PNR_ERR_UNSUPPORTED; }
size_t pnr_project_latent_bytes(const PnrScene*, const PnrMlp*) { return 0; }
int pnr_project_latent(const PnrScene*, const PnrMlp*, float*, size_t, void*, size_t, void*) { return PNR_ERR_UNSUPPORTED; }
int pnr_tc_status(int*) { return 0; }
int pnr_tc_counters(unsigned long long* out8) {
  for (int i = 0; i < 8; ++i) out8[i] = 0;
  return 0;
}
}
