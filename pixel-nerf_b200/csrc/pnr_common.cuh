// Internal helpers shared by the libpnr_sm90 translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/pnr.h"

namespace pnr {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define PNR_CHECK_ARG(cond, msg)                      \
  do {                                                \
    if (!(cond)) {                                    \
      pnr::set_error("invalid argument: %s", msg);    \
      return PNR_ERR_INVALID;                         \
    }                                                 \
  } while (0)

#define PNR_CUDA(expr)                                                                  \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      pnr::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return PNR_ERR_CUDA;                                                              \
    }                                                                                   \
  } while (0)

#define PNR_LAUNCH_CHECK()                                                             \
  do {                                                                                 \
    cudaError_t _e = cudaGetLastError();                                               \
    if (_e != cudaSuccess) {                                                           \
      pnr::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return PNR_ERR_CUDA;                                                             \
    }                                                                                  \
    pnr::count_launch();                                                               \
  } while (0)

// dominant-kernel profiling (pnr_profile_begin/end): bracket a launch with events
void prof_before(cudaStream_t s);
void prof_after(cudaStream_t s);

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- deterministic mode (pnr_set_deterministic; pnr_api.cu) -----------------------------
// The calling thread's flag.  When set, the training path uses its fixed-order variants: ordered split-K in the
// tensor-core GEMM and the fixed-point latent scatter of the field backward.
bool deterministic();
// Partial tiles of the ordered split-K, carved from the caller's workspace by the entry point that runs the GEMMs and
// installed for the duration of its call (SplitKScope).  A GEMM in deterministic mode splits K no further than this
// buffer holds; with none installed it does not split.
struct SplitKScratch {
  float* p;
  size_t bytes;
};
SplitKScratch& splitk_scratch();
struct SplitKScope {
  SplitKScratch saved;
  SplitKScope(float* p, size_t bytes) : saved(splitk_scratch()) { splitk_scratch() = SplitKScratch{p, bytes}; }
  ~SplitKScope() { splitk_scratch() = saved; }
};

// Bump allocator over the caller's workspace.
struct Arena {
  char* base;
  size_t cap;
  size_t off;
  Arena(void* p, size_t n) : base(static_cast<char*>(p)), cap(n), off(0) {}
  template <typename T>
  T* take(size_t count) {
    off = align_up(off, 256);
    T* r = reinterpret_cast<T*>(base + off);
    off += count * sizeof(T);
    return r;
  }
  bool ok() const { return off <= cap; }
};

// Where the points of a field evaluation come from.
//   mode 0: explicit xyz / viewdirs arrays [SB][P][3]            (PixelNeRFNet.forward callers)
//   mode 1: rays [SB*B][8] and z [SB*B][K]; point (sb, p): ray = sb*B + p / K, sample = p % K
//           (NeRFRenderer.composite, src/render/nerf.py:185-211)
struct PointSource {
  int mode;
  const float* xyz;
  const float* dirs;
  const float* rays;
  const float* z;
  int K;          // samples per ray (mode 1)
  int64_t P;      // points per object
};

// ---- stage launchers (pnr_stages.cu, compiled with -fmad=false) -------------------------
int launch_pack_latent(const float* nchw, float* nhwc, int V, int C, int Hl, int Wl, cudaStream_t s);
int launch_sample_coarse(const float* rays, const float* lin, const float* u, float* z, int64_t R, int Kc,
                         cudaStream_t s);
int launch_composite(const float* rays, const float* z, const float* field, int white, float* w,
                     float* rgb, float* depth, int64_t R, int K, cudaStream_t s);
int launch_sample_fine(const float* rays, const float* zc, const float* wc, const float* dc,
                       const float* u, const float* uj, const float* nd, float depth_std, float* zout,
                       int64_t R, int Kc, int Kf, int Kfd, cudaStream_t s);
// rows of a point chunk: feat [rows][48] (42 used) and gathered latent lat [rows][C];
// row = local_point * NS + view.  g0 = first global point (sb*P + p), n_pts points.
int launch_build_rows(const PnrScene& sc, const PointSource& src, int64_t g0, int64_t n_pts, float* feat,
                      float* lat, cudaStream_t s);

// rays of pixels [first, first+count) of the flattened (NV,H,W) grid; rgb floats -> uint8 frame bytes
int launch_gen_rays(const float* poses, int W, int H, float fx, float fy, float cx, float cy, float z_near,
                    float z_far, int64_t first, int64_t count, float* rays, cudaStream_t s);
int launch_frames_u8(const float* rgb, int64_t n, uint8_t* out, cudaStream_t s);

// ---- SIMT engine (pnr_field_simt.cu) ---------------------------------------------------
size_t simt_workspace_bytes(const PnrScene& sc, const PnrMlp& mlp, int64_t total_points);
int simt_field_eval(const PnrScene& sc, const PnrMlp& mlp, const PointSource& src, int64_t total_points,
                    float* out, void* ws, size_t ws_bytes, cudaStream_t s);

// renderer backward pieces (pnr_stages.cu): compositing, z from positions, coarse depth through the depth samples.
// d_rgb [R][3], d_depth [R], d_weights [R][K], d_depth_up [R] may each be NULL (zero).
int launch_composite_bwd(const float* rays, const float* z, const float* field, const float* d_rgb,
                         const float* d_depth, const float* d_weights, int white, float* d_field, float* d_z,
                         float* d_far, int64_t R, int K, cudaStream_t s);   // d_far [R]: d(last interval), may be NULL
int launch_depth_grad(const float* rays, const float* z_sorted, const float* depth, const float* nd,
                      float depth_std, float* d_z, const float* d_xyz, const float* d_depth_up, float* d_depth,
                      int64_t R, int K, int Kfd, cudaStream_t s);
// ray gradient of one pass from its per-sample d_z / d_xyz / d_vd (written, or added when accum); Kfd > 0: the pass
// holds the depth-centred samples of depth / nd (the fine pass)
int launch_ray_grad(const float* rays, const float* z, const float* d_z, const float* d_xyz, const float* d_vd,
                    const float* d_far_last, bool dz_has_pos, const float* depth, const float* nd, float depth_std,
                    int Kfd, bool accum, float* d_rays, int64_t R, int K, cudaStream_t s);
// backward of launch_gen_rays: d_rays [count][8] -> d_poses [NV][4][4] (+=)
int launch_gen_rays_bwd(const float* d_rays, int W, int H, float fx, float fy, float cx, float cy, int64_t first,
                        int64_t count, float* d_poses, cudaStream_t s);

// PNR_ERR_INVALID (with the message) for an engine the backward entry points refuse: PNR_ENGINE_TC_FAST (pnr_api.cu)
int check_backward_engine(int engine);

// ---- field backward, SIMT first path (pnr_field_bwd.cu) --------------------------------
size_t field_backward_workspace_bytes(const PnrScene& sc, const PnrMlp& mlp, int64_t total_points);
int field_backward(const PnrScene& sc, const PnrMlp& mlp, const PointSource& src, int64_t total_points,
                   const float* d_out, const PnrMlp& grad, float* d_latent, float* d_xyz, float* d_dirs,
                   const PnrCameraGrad* cam, void* ws, size_t ws_bytes, cudaStream_t s, bool sel = false);

// ---- tensor engine (pnr_field_tc.cu) ---------------------------------------------------
bool tc_supported(const PnrScene& sc, const PnrMlp& mlp);
size_t tc_workspace_bytes(const PnrScene& sc, const PnrMlp& mlp, int64_t total_points);
int tc_field_eval(const PnrScene& sc, const PnrMlp& mlp, const float* proj, const PointSource& src,
                  int64_t total_points, float* out, void* ws, size_t ws_bytes, cudaStream_t s);
// tc_field_eval on the single-pass kernel (PNR_ENGINE_TC_FAST).  Weak: the host-emulator build has no tensor engine
// (tc_supported is false there, so this is never reached) and still links without it.
int tc_field_eval_fast(const PnrScene& sc, const PnrMlp& mlp, const float* proj, const PointSource& src,
                       int64_t total_points, float* out, void* ws, size_t ws_bytes, cudaStream_t s)
    __attribute__((weak));
// NeRFRenderer.forward in one launch (coarse + fine field passes with compositing / resampling in the ray-completion
// epilogue); zc, wc [R][Kc] and zf [R][Kc+Kf] are caller or workspace buffers that also serve as outputs.  The kernel is
// the single-pass one when cfg.engine is PNR_ENGINE_TC_FAST.
size_t tc_render_workspace_bytes(const PnrScene& sc, int64_t R, int Kc, int Kf);
int tc_render(const PnrScene& sc, const PnrMlp& mlp_coarse, const PnrMlp& mlp_fine, const float* proj_coarse,
              const float* proj_fine, const PnrRenderCfg& cfg, const float* rays, const PnrNoise& noise, float* zc,
              float* wc, float* zf, const PnrRenderOut& out, int64_t B, void* ws, size_t ws_bytes, cudaStream_t s);

// ---- exclusive scan of the mesh-extraction kernels (pnr_recon.cu), shared with the mesh components (pnr_mesh.cu) -----
// out[i] = in[0] + ... + in[i - 1] and *total = the sum (int64, device), in three launches on s; n >= 1.  sums:
// scan_tile_count(n) int64 of scratch.  Reduce-then-scan, no atomics.
int64_t scan_tile_count(int64_t n);
int exclusive_scan(const uint8_t* in, int64_t n, int64_t* sums, int64_t* out, int64_t* total, cudaStream_t s);

}  // namespace pnr
