// C-ABI entry points of libpnr_sm90.so (see include/pnr.h).  Thin: argument checks, engine
// selection, workspace carving, and the coarse -> fine orchestration of NeRFRenderer.forward
// (src/render/nerf.py:251-303).  No CPU fallback: everything below launches CUDA kernels.
#include <atomic>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "pnr_common.cuh"

namespace pnr {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sgemm(const float* A, int lda, const float* W, const float* bias, float* C, int ldc, int M, int N, int K,
          bool relu_a, bool accum, cudaStream_t s);                 // pnr_field_simt.cu
int gemm_bf16x3(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc, int M, int N,
                int K, bool relu_a, bool accum, cudaStream_t s);    // pnr_gemm_tc.cu
int gemm_f16x3(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc, int M, int N, int K,
               cudaStream_t s);

// ---- dominant-kernel profiling ----------------------------------------------------------
static bool g_prof_on = false;
static std::vector<cudaEvent_t> g_prof_ev;  // pairs (start, stop)
static std::vector<cudaEvent_t> g_prof_pool;
static cudaEvent_t prof_event() {
  cudaEvent_t e;
  if (!g_prof_pool.empty()) { e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
  cudaEventCreate(&e);
  return e;
}
void prof_before(cudaStream_t s) {
  if (!g_prof_on) return;
  cudaEvent_t e = prof_event();
  cudaEventRecord(e, s);
  g_prof_ev.push_back(e);
}
void prof_after(cudaStream_t s) {
  if (!g_prof_on) return;
  cudaEvent_t e = prof_event();
  cudaEventRecord(e, s);
  g_prof_ev.push_back(e);
}

static int check_scene(const PnrScene* sc) {
  PNR_CHECK_ARG(sc != nullptr, "scene is NULL");
  PNR_CHECK_ARG(sc->latent_nhwc && sc->poses && sc->focal && sc->c, "scene pointers must not be NULL");
  PNR_CHECK_ARG(sc->SB >= 1 && sc->NS >= 1, "SB and NS must be >= 1");
  PNR_CHECK_ARG(sc->Hl >= 2 && sc->Wl >= 2, "latent must be at least 2x2");
  PNR_CHECK_ARG(sc->C % 4 == 0, "latent channels must be a multiple of 4");
  PNR_CHECK_ARG(sc->n_focal == 1 || sc->n_focal == sc->SB, "n_focal must be 1 or SB");
  PNR_CHECK_ARG(sc->n_c == 1 || sc->n_c == sc->SB, "n_c must be 1 or SB");
  return PNR_OK;
}

static int check_mlp(const PnrMlp* m) {
  PNR_CHECK_ARG(m != nullptr, "mlp is NULL");
  PNR_CHECK_ARG(m->n_blocks >= 1 && m->n_blocks <= PNR_MAX_BLOCKS, "n_blocks out of range");
  PNR_CHECK_ARG(m->lin_in_w && m->lin_in_b && m->lin_out_w && m->lin_out_b, "lin_in/lin_out weights are NULL");
  for (int i = 0; i < m->n_blocks; ++i) {
    PNR_CHECK_ARG(m->fc0_w[i] && m->fc0_b[i] && m->fc1_w[i] && m->fc1_b[i], "block weights are NULL");
    if (i < m->combine_layer) PNR_CHECK_ARG(m->lin_z_w[i] && m->lin_z_b[i], "lin_z weights are NULL");
  }
  return PNR_OK;
}

// engine actually used for (scene, mlp): AUTO prefers the tensor engine when it applies.
static int resolve_engine(const PnrScene& sc, const PnrMlp& mlp, const float* proj, int engine) {
  bool tc_ok = tc_supported(sc, mlp) && mlp.packed != nullptr && proj != nullptr;
  if (engine == PNR_ENGINE_TC) {
    if (!tc_ok) {
      set_error("tensor engine unavailable for this call (needs d_hidden=512, d_latent=512, 5 blocks, "
                "combine_layer=3, packed weights and projected latent)");
      return PNR_ERR_UNSUPPORTED;
    }
    return PNR_ENGINE_TC;
  }
  if (engine == PNR_ENGINE_SIMT) return PNR_ENGINE_SIMT;
  if (engine == PNR_ENGINE_AUTO) return tc_ok ? PNR_ENGINE_TC : PNR_ENGINE_SIMT;
  set_error("unknown engine %d", engine);
  return PNR_ERR_INVALID;
}

static size_t field_ws(const PnrScene& sc, const PnrMlp& mlp, int64_t total_points, int engine) {
  size_t a = simt_workspace_bytes(sc, mlp, total_points);
  if (engine == PNR_ENGINE_SIMT) return a;
  size_t b = tc_supported(sc, mlp) ? tc_workspace_bytes(sc, mlp, total_points) : 0;
  if (engine == PNR_ENGINE_TC) return b;
  return a > b ? a : b;
}

static int field_dispatch(const PnrScene& sc, const PnrMlp& mlp, const float* proj, const PointSource& src,
                          int64_t total_points, float* out, int engine, void* ws, size_t ws_bytes,
                          cudaStream_t s) {
  int e = resolve_engine(sc, mlp, proj, engine);
  if (e < 0) return e;
  if (e == PNR_ENGINE_TC) return tc_field_eval(sc, mlp, proj, src, total_points, out, ws, ws_bytes, s);
  return simt_field_eval(sc, mlp, src, total_points, out, ws, ws_bytes, s);
}

}  // namespace pnr

using namespace pnr;

extern "C" {

int pnr_abi_version(void) { return PNR_ABI_VERSION; }
const char* pnr_last_error(void) { return g_err; }
int64_t pnr_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int pnr_profile_begin(void) {
  for (cudaEvent_t e : g_prof_ev) g_prof_pool.push_back(e);
  g_prof_ev.clear();
  g_prof_on = true;
  return PNR_OK;
}

int pnr_profile_end(double* total_ms, int64_t* launches) {
  g_prof_on = false;
  double tot = 0.0;
  int64_t n = 0;
  for (size_t i = 0; i + 1 < g_prof_ev.size(); i += 2) {
    PNR_CUDA(cudaEventSynchronize(g_prof_ev[i + 1]));
    float ms = 0.f;
    PNR_CUDA(cudaEventElapsedTime(&ms, g_prof_ev[i], g_prof_ev[i + 1]));
    tot += ms;
    ++n;
  }
  for (cudaEvent_t e : g_prof_ev) g_prof_pool.push_back(e);
  g_prof_ev.clear();
  if (total_ms) *total_ms = tot;
  if (launches) *launches = n;
  return PNR_OK;
}

int pnr_pack_latent(const float* latent_nchw, float* latent_nhwc, int32_t V, int32_t C, int32_t Hl, int32_t Wl,
                    void* stream) {
  PNR_CHECK_ARG(latent_nchw && latent_nhwc, "latent pointers are NULL");
  PNR_CHECK_ARG(V >= 1 && C >= 1 && Hl >= 1 && Wl >= 1, "bad latent shape");
  return launch_pack_latent(latent_nchw, latent_nhwc, V, C, Hl, Wl, (cudaStream_t)stream);
}

int pnr_sample_coarse(const float* rays, const float* lin_steps, const float* u_coarse, float* z, int64_t R,
                      int32_t Kc, void* stream) {
  PNR_CHECK_ARG(R >= 0 && Kc >= 1, "bad sizes");
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(rays && u_coarse && z, "NULL pointer");
  return launch_sample_coarse(rays, lin_steps, u_coarse, z, R, Kc, (cudaStream_t)stream);
}

int pnr_gen_rays(const float* poses_c2w, int64_t NV, int32_t W, int32_t H, float fx, float fy, float cx, float cy,
                 float z_near, float z_far, int64_t first, int64_t count, float* rays, void* stream) {
  PNR_CHECK_ARG(NV >= 0 && W >= 1 && H >= 1, "bad sizes");
  PNR_CHECK_ARG(first >= 0 && count >= 0 && first + count <= NV * (int64_t)W * H, "ray range outside the pixel grid");
  if (count == 0) return PNR_OK;
  PNR_CHECK_ARG(poses_c2w && rays, "NULL pointer");
  PNR_CHECK_ARG(fx != 0.f && fy != 0.f, "zero focal length");
  PNR_CHECK_ARG((reinterpret_cast<uintptr_t>(rays) & 15) == 0, "rays must be 16-byte aligned");
  return launch_gen_rays(poses_c2w, W, H, fx, fy, cx, cy, z_near, z_far, first, count, rays, (cudaStream_t)stream);
}

int pnr_frames_u8(const float* rgb, int64_t n, uint8_t* out, void* stream) {
  PNR_CHECK_ARG(n >= 0, "bad size");
  if (n == 0) return PNR_OK;
  PNR_CHECK_ARG(rgb && out, "NULL pointer");
  PNR_CHECK_ARG((reinterpret_cast<uintptr_t>(rgb) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0,
                "rgb must be 16-byte and out 4-byte aligned");
  return launch_frames_u8(rgb, n, out, (cudaStream_t)stream);
}

int pnr_composite(const float* rays, const float* z, const float* field, int32_t white_bkgd, float* weights,
                  float* rgb, float* depth, int64_t R, int32_t K, void* stream) {
  PNR_CHECK_ARG(R >= 0 && K >= 1, "bad sizes");
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(rays && z && field && rgb && depth, "NULL pointer");
  return launch_composite(rays, z, field, white_bkgd, weights, rgb, depth, R, K, (cudaStream_t)stream);
}

int pnr_sample_fine(const float* rays, const float* z_coarse, const float* weights_coarse,
                    const float* depth_coarse, const float* u_fine, const float* u_fine_jit,
                    const float* n_depth, float depth_std, float* z_out, int64_t R, int32_t Kc, int32_t Kf,
                    int32_t Kfd, void* stream) {
  PNR_CHECK_ARG(R >= 0 && Kc >= 1 && Kf >= 1 && Kfd >= 0 && Kfd <= Kf, "bad sizes");
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(rays && z_coarse && z_out, "NULL pointer");
  if (Kf - Kfd > 0) PNR_CHECK_ARG(weights_coarse && u_fine && u_fine_jit, "importance-sampling inputs are NULL");
  if (Kfd > 0) PNR_CHECK_ARG(depth_coarse && n_depth, "depth-sampling inputs are NULL");
  return launch_sample_fine(rays, z_coarse, weights_coarse, depth_coarse, u_fine, u_fine_jit, n_depth, depth_std,
                            z_out, R, Kc, Kf, Kfd, (cudaStream_t)stream);
}

size_t pnr_field_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp, int64_t P, int32_t engine) {
  if (!scene || !mlp || P < 0) return 0;
  return field_ws(*scene, *mlp, P * scene->SB, engine);
}

int pnr_field_eval(const PnrScene* scene, const PnrMlp* mlp, const float* xyz, const float* viewdirs, float* out,
                   int64_t P, int32_t engine, void* workspace, size_t workspace_bytes, void* stream) {
  int rc;
  if ((rc = check_scene(scene))) return rc;
  if ((rc = check_mlp(mlp))) return rc;
  PNR_CHECK_ARG(P >= 0, "P must be >= 0");
  if (P == 0) return PNR_OK;
  PNR_CHECK_ARG(xyz && viewdirs && out && workspace, "NULL pointer");
  PointSource src{};
  src.mode = 0;
  src.xyz = xyz;
  src.dirs = viewdirs;
  src.P = P;
  src.K = 1;
  return field_dispatch(*scene, *mlp, scene->proj_coarse, src, P * scene->SB, out, engine, workspace,
                        workspace_bytes, (cudaStream_t)stream);
}

int pnr_gemm_nt(const float* A, int32_t lda, const float* W, const float* bias, float* C, int32_t ldc, int32_t M,
                int32_t N, int32_t K, int32_t relu_a, int32_t accum, int32_t engine, void* stream) {
  PNR_CHECK_ARG(M >= 0 && N >= 0 && K >= 16 && K % 16 == 0, "bad sizes (K must be a positive multiple of 16)");
  if (M == 0 || N == 0) return PNR_OK;
  PNR_CHECK_ARG(A && W && C, "NULL pointer");
  PNR_CHECK_ARG(lda >= K && ldc >= N && lda % 4 == 0, "bad leading dimensions");
  if (engine == PNR_ENGINE_SIMT) return sgemm(A, lda, W, bias, C, ldc, M, N, K, relu_a != 0, accum != 0, (cudaStream_t)stream);
  if (engine == PNR_GEMM_F16X3) {
    PNR_CHECK_ARG(!relu_a && !accum, "the fp16-split engine is store-only without activation");
    return gemm_f16x3(A, lda, W, K, bias, C, ldc, M, N, K, (cudaStream_t)stream);
  }
  return gemm_bf16x3(A, lda, W, K, bias, C, ldc, M, N, K, relu_a != 0, accum != 0, (cudaStream_t)stream);
}

size_t pnr_field_backward_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp, int64_t P) {
  if (!scene || !mlp || P < 0) return 0;
  return field_backward_workspace_bytes(*scene, *mlp, P * scene->SB);
}

int pnr_field_backward(const PnrScene* scene, const PnrMlp* mlp, const float* xyz, const float* viewdirs,
                       const float* d_out, const PnrMlp* grad, float* d_latent_nhwc, float* d_xyz, int64_t P,
                       void* workspace, size_t workspace_bytes, void* stream) {
  int rc;
  if ((rc = check_scene(scene))) return rc;
  if ((rc = check_mlp(mlp))) return rc;
  if ((rc = check_mlp(grad))) return rc;
  PNR_CHECK_ARG(grad->d_hidden == mlp->d_hidden && grad->n_blocks == mlp->n_blocks && grad->d_in == mlp->d_in &&
                    grad->d_latent == mlp->d_latent && grad->combine_layer == mlp->combine_layer,
                "grad must have the shape of mlp");
  PNR_CHECK_ARG(P >= 0, "P must be >= 0");
  if (P == 0) return PNR_OK;
  PNR_CHECK_ARG(xyz && viewdirs && d_out && workspace, "NULL pointer");
  PointSource src{};
  src.mode = 0;
  src.xyz = xyz;
  src.dirs = viewdirs;
  src.P = P;
  src.K = 1;
  return field_backward(*scene, *mlp, src, P * scene->SB, d_out, *grad, d_latent_nhwc, d_xyz, workspace,
                        workspace_bytes, (cudaStream_t)stream);
}

static size_t render_bwd_field_ws(const PnrScene& sc, const PnrMlp& m, int64_t pts) {
  size_t a = field_ws(sc, m, pts, PNR_ENGINE_AUTO), b = field_backward_workspace_bytes(sc, m, pts);
  return a > b ? a : b;
}

size_t pnr_render_backward_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp_coarse, const PnrMlp* mlp_fine,
                                           const PnrRenderCfg* cfg, int64_t B) {
  if (!scene || !mlp_coarse || !cfg || B < 0) return 0;
  const int64_t R = B * scene->SB;
  const int K = cfg->n_coarse + cfg->n_fine;
  size_t b = 0;
  b += align_up((size_t)R * K * 4 * 4, 256) * 2;   // field, d_field
  b += align_up((size_t)R * K * 4, 256);           // d_z
  b += align_up((size_t)R * K * 3 * 4, 256);       // d_xyz
  b += align_up((size_t)R * 4, 256);               // d_depth
  size_t f = render_bwd_field_ws(*scene, *mlp_coarse, R * K);
  if (mlp_fine) {
    size_t f2 = render_bwd_field_ws(*scene, *mlp_fine, R * K);
    if (f2 > f) f = f2;
  }
  return b + f + 4096;
}

int pnr_render_backward(const PnrScene* scene, const PnrMlp* mlp_coarse, const PnrMlp* mlp_fine,
                        const PnrRenderCfg* cfg, const float* rays, const PnrNoise* noise, const PnrRenderOut* fwd,
                        const float* d_rgb_coarse, const float* d_rgb_fine, const PnrMlp* grad_coarse,
                        const PnrMlp* grad_fine, float* d_latent_nhwc, int64_t B, void* workspace,
                        size_t workspace_bytes, void* stream) {
  int rc;
  if ((rc = check_scene(scene))) return rc;
  if ((rc = check_mlp(mlp_coarse))) return rc;
  if ((rc = check_mlp(grad_coarse))) return rc;
  if (mlp_fine && (rc = check_mlp(mlp_fine))) return rc;
  if (mlp_fine && (rc = check_mlp(grad_fine))) return rc;
  PNR_CHECK_ARG(cfg && noise && fwd, "cfg / noise / fwd is NULL");
  PNR_CHECK_ARG(cfg->n_coarse >= 1 && cfg->n_fine >= 0 && cfg->n_fine_depth >= 0 &&
                    cfg->n_fine_depth <= cfg->n_fine,
                "bad sample counts");
  PNR_CHECK_ARG(B >= 0, "B must be >= 0");
  const int64_t R = B * scene->SB;
  if (R == 0) return PNR_OK;
  const int Kc = cfg->n_coarse, Kf = cfg->n_fine, Kfd = cfg->n_fine_depth, K = Kc + Kf;
  PNR_CHECK_ARG(rays && workspace && d_rgb_coarse && fwd->z_coarse, "NULL pointer (rays, workspace, d_rgb_coarse, z_coarse)");
  if (Kf > 0) PNR_CHECK_ARG(d_rgb_fine && fwd->z_fine, "fine pass needs d_rgb_fine and the forward's z_fine");
  if (Kf > 0 && Kfd > 0) PNR_CHECK_ARG(fwd->depth_coarse && noise->n_depth, "depth samples need depth_coarse and n_depth");
  if (workspace_bytes < pnr_render_backward_workspace_bytes(scene, mlp_coarse, mlp_fine, cfg, B)) {
    set_error("workspace too small: %zu < %zu", workspace_bytes,
              pnr_render_backward_workspace_bytes(scene, mlp_coarse, mlp_fine, cfg, B));
    return PNR_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  Arena ar(workspace, workspace_bytes);
  float* field = ar.take<float>((size_t)R * K * 4);
  float* d_field = ar.take<float>((size_t)R * K * 4);
  float* d_z = ar.take<float>((size_t)R * K);
  float* d_xyz = ar.take<float>((size_t)R * K * 3);
  float* d_depth = ar.take<float>((size_t)R);
  char* rest = ar.base + align_up(ar.off, 256);
  const size_t rest_bytes = workspace_bytes - align_up(ar.off, 256);
  const bool depth_path = Kf > 0 && Kfd > 0;
  PointSource src{};
  src.mode = 1;
  src.rays = rays;
  if (Kf > 0) {   // fine pass first: it feeds d(depth_coarse) into the coarse pass (nerf.py:289-291)
    const PnrMlp* m = mlp_fine ? mlp_fine : mlp_coarse;
    const PnrMlp* g = mlp_fine ? grad_fine : grad_coarse;
    src.z = fwd->z_fine;
    src.K = K;
    src.P = B * K;
    const float* pj = mlp_fine ? scene->proj_fine : scene->proj_coarse;
    if ((rc = field_dispatch(*scene, *m, pj, src, R * K, field, cfg->engine, rest, rest_bytes, s))) return rc;
    if ((rc = launch_composite_bwd(rays, fwd->z_fine, field, d_rgb_fine, nullptr, cfg->white_bkgd, d_field, d_z, R, K, s)))
      return rc;
    if ((rc = field_backward(*scene, *m, src, R * K, d_field, *g, d_latent_nhwc, depth_path ? d_xyz : nullptr, rest,
                             rest_bytes, s)))
      return rc;
    if (depth_path &&
        (rc = launch_depth_grad(rays, fwd->z_fine, fwd->depth_coarse, noise->n_depth, cfg->depth_std, d_z, d_xyz,
                                d_depth, R, K, Kfd, s)))
      return rc;
  }
  src.z = fwd->z_coarse;
  src.K = Kc;
  src.P = B * Kc;
  if ((rc = field_dispatch(*scene, *mlp_coarse, scene->proj_coarse, src, R * Kc, field, cfg->engine, rest, rest_bytes, s)))
    return rc;
  if ((rc = launch_composite_bwd(rays, fwd->z_coarse, field, d_rgb_coarse, depth_path ? d_depth : nullptr,
                                 cfg->white_bkgd, d_field, d_z, R, Kc, s)))
    return rc;
  return field_backward(*scene, *mlp_coarse, src, R * Kc, d_field, *grad_coarse, d_latent_nhwc, nullptr, rest, rest_bytes, s);
}

size_t pnr_render_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp_coarse, const PnrMlp* mlp_fine,
                                  const PnrRenderCfg* cfg, int64_t B) {
  if (!scene || !mlp_coarse || !cfg || B < 0) return 0;
  const int64_t R = B * scene->SB;
  const int Kc = cfg->n_coarse, K = cfg->n_coarse + cfg->n_fine;
  size_t b = 0;
  b += align_up((size_t)R * K * 4 * 4, 256);   // field values of the larger pass
  b += align_up((size_t)R * Kc * 4, 256) * 2;  // z_coarse, weights_coarse
  b += align_up((size_t)R * K * 4, 256);       // z_fine
  b += align_up((size_t)R * 4 * 4, 256) * 2;   // rgb/depth scratch when the caller passes NULL
  size_t f = field_ws(*scene, *mlp_coarse, R * K, cfg->engine);
  if (mlp_fine) {
    size_t f2 = field_ws(*scene, *mlp_fine, R * K, cfg->engine);
    if (f2 > f) f = f2;
  }
  if (cfg->engine != PNR_ENGINE_SIMT && tc_supported(*scene, *mlp_coarse)) {
    size_t f3 = tc_render_workspace_bytes(*scene, R, cfg->n_coarse, cfg->n_fine);
    if (f3 > f) f = f3;
  }
  return b + f + 4096;
}

// PNR_RENDER_FUSED=0 keeps the tensor engine on the stage-by-stage orchestration (six launches); default: one launch.
static bool fused_render_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("PNR_RENDER_FUSED");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}

int pnr_render(const PnrScene* scene, const PnrMlp* mlp_coarse, const PnrMlp* mlp_fine, const PnrRenderCfg* cfg,
               const float* rays, const PnrNoise* noise, const PnrRenderOut* out, int64_t B, void* workspace,
               size_t workspace_bytes, void* stream) {
  int rc;
  if ((rc = check_scene(scene))) return rc;
  if ((rc = check_mlp(mlp_coarse))) return rc;
  if (mlp_fine && (rc = check_mlp(mlp_fine))) return rc;
  PNR_CHECK_ARG(cfg && noise && out, "cfg / noise / out is NULL");
  PNR_CHECK_ARG(cfg->n_coarse >= 1 && cfg->n_fine >= 0 && cfg->n_fine_depth >= 0 &&
                    cfg->n_fine_depth <= cfg->n_fine,
                "bad sample counts");
  PNR_CHECK_ARG(B >= 0, "B must be >= 0");
  const int64_t R = B * scene->SB;
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(rays && workspace, "NULL pointer");
  PNR_CHECK_ARG(noise->u_coarse, "u_coarse is NULL");
  PNR_CHECK_ARG(out->rgb_coarse && out->depth_coarse, "coarse rgb/depth outputs are required");
  const int Kc = cfg->n_coarse, Kf = cfg->n_fine, Kfd = cfg->n_fine_depth, K = Kc + Kf;
  if (Kf > 0) PNR_CHECK_ARG(out->rgb_fine && out->depth_fine, "fine rgb/depth outputs are required");
  if (workspace_bytes < pnr_render_workspace_bytes(scene, mlp_coarse, mlp_fine, cfg, B)) {
    set_error("workspace too small: %zu < %zu", workspace_bytes,
              pnr_render_workspace_bytes(scene, mlp_coarse, mlp_fine, cfg, B));
    return PNR_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  Arena ar(workspace, workspace_bytes);
  float* field = ar.take<float>((size_t)R * K * 4);
  float* zc = out->z_coarse ? out->z_coarse : ar.take<float>((size_t)R * Kc);
  float* wc = out->weights_coarse ? out->weights_coarse : ar.take<float>((size_t)R * Kc);
  float* zf = nullptr;
  if (Kf > 0) zf = out->z_fine ? out->z_fine : ar.take<float>((size_t)R * K);
  char* rest = ar.base + align_up(ar.off, 256);
  size_t rest_bytes = workspace_bytes - align_up(ar.off, 256);

  if (Kf - Kfd > 0) PNR_CHECK_ARG(noise->u_fine && noise->u_fine_jit, "u_fine / u_fine_jit is NULL");
  if (Kf > 0 && Kfd > 0) PNR_CHECK_ARG(noise->n_depth, "n_depth is NULL");
  {
    // ---- tensor engine: the whole call is ONE launch (sampling, both field passes, compositing, resampling) ----
    const PnrMlp* mf = mlp_fine ? mlp_fine : mlp_coarse;                       // models.py:242
    const float* pf = mlp_fine ? scene->proj_fine : scene->proj_coarse;
    int ec = resolve_engine(*scene, *mlp_coarse, scene->proj_coarse, cfg->engine);
    if (ec < 0) return ec;
    int ef = Kf > 0 ? resolve_engine(*scene, *mf, pf, cfg->engine) : ec;
    if (ef < 0) return ef;
    if (ec == PNR_ENGINE_TC && ef == PNR_ENGINE_TC && fused_render_enabled())
      return tc_render(*scene, *mlp_coarse, *mf, scene->proj_coarse, pf, *cfg, rays, *noise, zc, wc, zf, *out, B, rest,
                       rest_bytes, s);
  }

  // ---- coarse pass (nerf.py:273-276) ----
  if ((rc = launch_sample_coarse(rays, noise->lin_steps, noise->u_coarse, zc, R, Kc, s))) return rc;
  PointSource src{};
  src.mode = 1;
  src.rays = rays;
  src.z = zc;
  src.K = Kc;
  src.P = B * Kc;
  if ((rc = field_dispatch(*scene, *mlp_coarse, scene->proj_coarse, src, R * Kc, field, cfg->engine, rest,
                           rest_bytes, s)))
    return rc;
  if ((rc = launch_composite(rays, zc, field, cfg->white_bkgd, wc, out->rgb_coarse, out->depth_coarse, R, Kc, s)))
    return rc;
  if (Kf == 0) return PNR_OK;

  // ---- fine pass (nerf.py:284-301) ----
  if ((rc = launch_sample_fine(rays, zc, wc, out->depth_coarse, noise->u_fine, noise->u_fine_jit, noise->n_depth,
                               cfg->depth_std, zf, R, Kc, Kf, Kfd, s)))
    return rc;
  const PnrMlp* mf = mlp_fine ? mlp_fine : mlp_coarse;  // models.py:242
  const float* pf = mlp_fine ? scene->proj_fine : scene->proj_coarse;
  src.z = zf;
  src.K = K;
  src.P = B * K;
  if ((rc = field_dispatch(*scene, *mf, pf, src, R * K, field, cfg->engine, rest, rest_bytes, s))) return rc;
  return launch_composite(rays, zf, field, cfg->white_bkgd, out->weights_fine, out->rgb_fine, out->depth_fine, R, K,
                          s);
}

}  // extern "C"
