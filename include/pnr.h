/*
 * pnr.h -- C ABI of libpnr_sm90.so, the H100-native (sm_90a) replacement for pixelNeRF's
 * volume-rendering hot path.
 *
 * The reference (sxyu/pixel-nerf) is 100 % Python/PyTorch and has no FFI of its own, so
 * every entry point below cites the reference FUNCTION it replaces (paths relative to the
 * reference root).  INTEGRATION.md shows the ctypes binding a maintainer would add.
 *
 * Conventions
 *   - plain C types only; every pointer is a DEVICE pointer unless marked "host".
 *   - all tensors are dense fp32, row-major, laid out exactly as the reference's tensors.
 *   - the caller (PyTorch) owns all memory, including the scratch `workspace`; the library
 *     allocates nothing that outlives a call.
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*), performs no
 *     device synchronisation, and is re-entrant per (device, stream).
 *   - return value 0 = success, negative = error; text via pnr_last_error() (thread local).
 *   - there is NO CPU fallback anywhere behind this ABI.
 */
#ifndef PNR_H_
#define PNR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PNR_ABI_VERSION 2
#define PNR_MAX_BLOCKS 8

enum {
  PNR_OK = 0,
  PNR_ERR_INVALID = -1,      /* bad argument / unsupported configuration           */
  PNR_ERR_WORKSPACE = -2,    /* workspace too small                                 */
  PNR_ERR_CUDA = -3,         /* CUDA runtime error (launch, attribute, ...)         */
  PNR_ERR_UNSUPPORTED = -4   /* engine cannot run this shape (e.g. tensor engine, d != 512) */
};

/* Which implementation evaluates the conditioned MLP. */
enum {
  PNR_ENGINE_AUTO = 0,   /* tensor engine when the shape allows it, else SIMT            */
  PNR_ENGINE_SIMT = 1,   /* fp32 FFMA kernels, any shape (bring-up / small-d engine)      */
  PNR_ENGINE_TC = 2,     /* wgmma split-fp16 (3 products, fp32 accumulate) fused kernel: rgb within 1e-4 of fp32 */
  /* 3 is PNR_GEMM_F16X3 (pnr_gemm_nt only).
   * Single-pass tensor engine, inference only: the same fused kernel with ONE fp16 product per GEMM
   * (D += Ahi*Whi, fp32 accumulate) for lin_in, fc_0 and fc_1; lin_z, geometry, the view mean, lin_out, compositing and
   * resampling stay as in PNR_ENGINE_TC.  Expect rgb errors against fp32 of a few 1e-4 on real scenes and up to
   * about one uint8 step (a few 1e-3), and more importance-sampling bin flips; DESIGN.md 3.1 has the measured
   * figures.  Never chosen by AUTO; the shape requirements of PNR_ENGINE_TC (PNR_ERR_UNSUPPORTED otherwise, no
   * fallback).  The render backward entry points (pnr_render_backward*, pnr_mgpu_render_backward*) refuse it with
   * PNR_ERR_INVALID: their recompute could not reproduce this forward.  pnr_field_backward* take no engine and
   * always recompute on the exact arithmetic, so a caller must not pair them with a forward of this engine. */
  PNR_ENGINE_TC_FAST = 4
};

/* State left behind by PixelNeRFNet.encode (src/model/models.py:89-144) and
 * SpatialEncoder.forward (src/model/encoder.py:111-164). */
typedef struct PnrScene {
  const float* latent_nhwc; /* [V][Hl][Wl][C] channels-last copy of encoder.latent (pnr_pack_latent) */
  const float* poses;       /* [V][3][4] world->camera, models.py:112-114                    */
  const float* focal;       /* [n_focal][2] (fx, -fy), models.py:119-130                     */
  const float* c;           /* [n_c][2] principal point, models.py:132-141                   */
  int32_t n_focal;          /* 1 or SB (per object, models.py:207-209)                        */
  int32_t n_c;              /* 1 or SB                                                        */
  int32_t SB;               /* objects                                                        */
  int32_t NS;               /* source views per object; V = SB*NS                             */
  int32_t Hl, Wl, C;        /* latent height, width, channels (C == mlp.d_latent)             */
  float image_w, image_h;   /* image_shape, models.py:116-117                                 */
  float scale_x, scale_y;   /* encoder.latent_scaling, encoder.py:161-163                     */
  /* tensor engine only (NULL for SIMT): per-view maps of lin_z[i](latent) built by
   * pnr_project_latent, [3][V][Hl][Wl][d_hidden]; one set per MLP (coarse, fine).            */
  const float* proj_coarse;
  const float* proj_fine;
} PnrScene;

/* One ResnetFC (src/model/resnetfc.py:66-130).  Weights are nn.Linear layout [out][in]. */
typedef struct PnrMlp {
  int32_t d_in;          /* 42 for the shipped configs (models.py:48-60)  */
  int32_t d_latent;      /* 512                                           */
  int32_t d_hidden;
  int32_t d_out;         /* 4                                             */
  int32_t n_blocks;      /* <= PNR_MAX_BLOCKS                             */
  int32_t combine_layer; /* views are averaged before this block (resnetfc.py:152,170) */
  const float* lin_in_w;
  const float* lin_in_b;
  const float* lin_out_w;
  const float* lin_out_b;
  const float* lin_z_w[PNR_MAX_BLOCKS];
  const float* lin_z_b[PNR_MAX_BLOCKS];
  const float* fc0_w[PNR_MAX_BLOCKS];
  const float* fc0_b[PNR_MAX_BLOCKS];
  const float* fc1_w[PNR_MAX_BLOCKS];
  const float* fc1_b[PNR_MAX_BLOCKS];
  /* tensor engine only: fp16 hi/lo split, wgmma-tiled weights from pnr_pack_mlp (else NULL) */
  const void* packed;
  size_t packed_bytes;
} PnrMlp;

/* NeRFRenderer attributes read at call time (src/render/nerf.py:62-96). */
typedef struct PnrRenderCfg {
  int32_t n_coarse;
  int32_t n_fine;        /* total fine samples incl. depth samples; 0 = coarse only */
  int32_t n_fine_depth;
  float depth_std;
  int32_t white_bkgd;
  int32_t engine;        /* PNR_ENGINE_* */
} PnrRenderCfg;

/* The random draws NeRFRenderer.forward makes, in its order (nerf.py:111,135,141,158),
 * made by the caller with torch so that results replay the reference's RNG exactly. */
typedef struct PnrNoise {
  const float* lin_steps;  /* [Kc] torch.linspace(0, 1-1/Kc, Kc) (nerf.py:107); NULL = computed */
  const float* u_coarse;   /* [R][Kc]      U[0,1)                     */
  const float* u_fine;     /* [R][Kf-Kfd]  U[0,1)   (NULL if Kf-Kfd==0) */
  const float* u_fine_jit; /* [R][Kf-Kfd]  U[0,1)                      */
  const float* n_depth;    /* [R][Kfd]     N(0,1)   (NULL if Kfd==0)    */
} PnrNoise;

/* Outputs of NeRFRenderer.forward (nerf.py:251-316); R = SB*B rays.  Any pointer may be
 * NULL when the caller does not need that tensor (weights/z are optional extras). */
typedef struct PnrRenderOut {
  float* rgb_coarse;     /* [R][3]      */
  float* depth_coarse;   /* [R]         */
  float* weights_coarse; /* [R][Kc]     */
  float* z_coarse;       /* [R][Kc]     */
  float* rgb_fine;       /* [R][3]      */
  float* depth_fine;     /* [R]         */
  float* weights_fine;   /* [R][Kc+Kf]  */
  float* z_fine;         /* [R][Kc+Kf]  sorted merged samples (nerf.py:294-295) */
} PnrRenderOut;

/* Upstream gradients of a loss w.r.t. the six differentiable outputs of NeRFRenderer.forward (nerf.py:251-316), shapes
 * as in PnrRenderOut.  Any pointer may be NULL, meaning a zero gradient (the loss does not use that output). */
typedef struct PnrRenderGrad {
  const float* d_rgb_coarse;     /* [R][3]      */
  const float* d_depth_coarse;   /* [R]         */
  const float* d_weights_coarse; /* [R][Kc]     */
  const float* d_rgb_fine;       /* [R][3]      */
  const float* d_depth_fine;     /* [R]         */
  const float* d_weights_fine;   /* [R][Kc+Kf]  */
} PnrRenderGrad;

/* Gradients w.r.t. the source cameras that PixelNeRFNet.encode leaves in PnrScene (models.py:112-141), for a loss on
 * what the field / renderer computed from them (models.py:161-212).  Each is accumulated (+=); any pointer may be NULL
 * (not wanted).  The world->camera poses' gradient reaches encode()'s camera->world poses through the caller's
 * autograd (rot = R^T, t = -R^T T). */
typedef struct PnrCameraGrad {
  float* d_poses;  /* [V][3][4] as PnrScene.poses          */
  float* d_focal;  /* [n_focal][2] as PnrScene.focal (fx, -fy) */
  float* d_c;      /* [n_c][2] as PnrScene.c                */
} PnrCameraGrad;

int pnr_abi_version(void);
const char* pnr_last_error(void);

/* Deterministic mode, a flag of the calling thread (like pnr_last_error), 0 by default.  pnr_set_deterministic sets
 * it (nonzero = on) and returns the previous value.  With it on, the calls of this thread give the same bits run to
 * run on the same device and inputs:
 *   - the tensor-core GEMMs (field backward, pnr_project_latent) sum split-K partial tiles in split order from a
 *     partial buffer in the caller's workspace, instead of adding them with float atomics;
 *   - the field backward adds the latent gradient per chunk in 64-bit fixed point (integer atomics, exact and
 *     order-free) and converts it into d_latent_nhwc once per chunk.  A non-finite term makes every d_latent element
 *     it reaches NaN.
 * pnr_field_backward_workspace_bytes and pnr_render_backward_workspace_bytes report the extra space when the calling
 * thread's flag is set, so set it before the size query.  With the flag off every call is unchanged. */
int pnr_set_deterministic(int on);
int pnr_get_deterministic(void);

/* Backward of bilinear upsampling with align_corners=True (torch.nn.functional.interpolate):
 * d_out [N][C][h_out][w_out] -> d_in [N][C][h_in][w_in] (overwritten), contiguous fp32.  A gather: each input pixel
 * sums, in output order, the terms (tap weight products as torch computes them) of the output pixels that read it,
 * so the result does not depend on scheduling.  Same-size maps copy. */
int pnr_upsample_bilinear_ac_backward(const float* d_out, int64_t N, int32_t C, int32_t h_in, int32_t w_in,
                                      int32_t h_out, int32_t w_out, float* d_in, void* stream);

/* NCHW -> channels-last copy of the encoder latent (replaces the strided gather +
 * transpose of encoder.py:102-108 / models.py:219).  src [V][C][Hl][Wl] -> dst [V][Hl][Wl][C]. */
int pnr_pack_latent(const float* latent_nchw, float* latent_nhwc, int32_t V, int32_t C, int32_t Hl,
                    int32_t Wl, void* stream);

/* NeRFRenderer.sample_coarse (nerf.py:98-118, lindisp=False).  rays [R][8] -> z [R][Kc]. */
int pnr_sample_coarse(const float* rays, const float* lin_steps, const float* u_coarse, float* z,
                      int64_t R, int32_t Kc, void* stream);

/* util.gen_rays with unproj_map (src/util/util.py:238-276, :113-143; ndc=False): rays of pixels
 * [first, first+count) of the flattened (NV, H, W) grid of NV camera-to-world poses [NV][4][4] ->
 * rays [count][8] = [origin, unit dir, z_near, z_far].  The caller's split loop
 * (eval/gen_video.py:209-212) can so generate each ray batch in place instead of holding (NV,H,W,8). */
int pnr_gen_rays(const float* poses_c2w, int64_t NV, int32_t W, int32_t H, float fx, float fy, float cx,
                 float cy, float z_near, float z_far, int64_t first, int64_t count, float* rays,
                 void* stream);

/* Backward of pnr_gen_rays w.r.t. the poses (util.py:251-254: origins = poses[:, :3, 3], dirs = poses[:, :3, :3]
 * unproj): d_rays [count][8] of pixels [first, first+count) -> d_poses_c2w [NV][4][4], accumulated (+=):
 * d_t += sum_pixels d_origin, d_R += sum_pixels d_dir unproj^T.  Rows 3 and the near / far columns get nothing (near
 * and far are constants there).  Each pose's pixels are summed by one block in a fixed order (no atomics), so repeated
 * calls give the same bits; one block per camera means a single large view is summed by one SM (not the training
 * path's cost: a training step's rays are a few thousand pixels).  Intrinsics are host floats, as in pnr_gen_rays: not
 * differentiated. */
int pnr_gen_rays_backward(const float* d_rays, const float* poses_c2w, int64_t NV, int32_t W, int32_t H, float fx,
                          float fy, float cx, float cy, int64_t first, int64_t count, float* d_poses_c2w,
                          void* stream);

/* Frame assembly of eval/gen_video.py:213-222 + :236: out[i] = (uint8)(rgb[i] * 255), truncating
 * (numpy astype); n = number of float values (rays * 3).  Values outside [0, 256/255) wrap like the
 * x86 cast (low 8 bits of the truncated int32). */
int pnr_frames_u8(const float* rgb, int64_t n, uint8_t* out, void* stream);

/* Compositing tail of NeRFRenderer.composite (nerf.py:178-182, 222-249) given the field
 * values field [R][K][4] = (sigmoid rgb, relu sigma).  weights may be NULL. */
int pnr_composite(const float* rays, const float* z, const float* field, int32_t white_bkgd,
                  float* weights, float* rgb, float* depth, int64_t R, int32_t K, void* stream);

/* sample_fine + sample_fine_depth + cat + sort (nerf.py:120-161, 285-295).
 * z_out [R][Kc+Kf] ascending. */
int pnr_sample_fine(const float* rays, const float* z_coarse, const float* weights_coarse,
                    const float* depth_coarse, const float* u_fine, const float* u_fine_jit,
                    const float* n_depth, float depth_std, float* z_out, int64_t R, int32_t Kc,
                    int32_t Kf, int32_t Kfd, void* stream);

/* PixelNeRFNet.forward (models.py:146-266): xyz, viewdirs [SB][P][3] -> out [SB][P][4]. */
size_t pnr_field_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp, int64_t P, int32_t engine);
int pnr_field_eval(const PnrScene* scene, const PnrMlp* mlp, const float* xyz, const float* viewdirs,
                   float* out, int64_t P, int32_t engine, void* workspace, size_t workspace_bytes,
                   void* stream);

/* Backward of pnr_field_eval (what autograd does for PixelNeRFNet.forward in the reference's training step,
 * train/train.py:199-215): d_out [SB][P][4] w.r.t. (sigmoid rgb, relu sigma) ->
 *   grad          : a PnrMlp whose weight pointers are WRITABLE gradient buffers of the same shapes; accumulated (+=)
 *   d_latent_nhwc : [V][Hl][Wl][C] channels-last gradient of the latent; accumulated (+=); may be NULL
 *   d_xyz         : [SB][P][3] gradient of the sample positions (overwritten); may be NULL
 * Recompute-in-backward (arithmetic = oracle/pnr_backward.py); the GEMMs run on the tensor cores (split-bf16 wgmma,
 * PNR_BWD_GEMM=simt selects the fp32 FFMA SGEMM).  This is what PixelNeRFNet.forward's autograd node calls on CUDA. */
size_t pnr_field_backward_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp, int64_t P);
int pnr_field_backward(const PnrScene* scene, const PnrMlp* mlp, const float* xyz, const float* viewdirs,
                       const float* d_out, const PnrMlp* grad, float* d_latent_nhwc, float* d_xyz, int64_t P,
                       void* workspace, size_t workspace_bytes, void* stream);
/* pnr_field_backward plus the gradients of the view directions and the cameras (models.py:161-212):
 *   d_viewdirs : [SB][P][3] = sum over views of R^T d(R dir) (overwritten); may be NULL
 *   cam        : camera gradients (+=), see PnrCameraGrad; may be NULL.  With q = R x, p = q + t, uv = -p.xy/p.z f + c:
 *                d_R += dq (x) x + d(R dir) (x) dir, d_t += d_p (projection part), d_f += d_uv * (-p.xy/p.z),
 *                d_c += d_uv; per-(point, view) partials are reduced per view in a fixed order (no atomics).
 * Same workspace as pnr_field_backward; with d_viewdirs and cam NULL it is pnr_field_backward. */
int pnr_field_backward_cam(const PnrScene* scene, const PnrMlp* mlp, const float* xyz, const float* viewdirs,
                           const float* d_out, const PnrMlp* grad, float* d_latent_nhwc, float* d_xyz,
                           float* d_viewdirs, const PnrCameraGrad* cam, int64_t P, void* workspace,
                           size_t workspace_bytes, void* stream);
/* pnr_field_backward_cam for a partly frozen network: computes only the gradients that are wanted, each bit-equal to
 * what pnr_field_backward_cam gives for it.  NULL means frozen:
 *   grad       : may be NULL (the whole MLP frozen), and so may any of its weight / bias members.  A NULL weight skips
 *                its weight-gradient GEMM and the two transposes that feed it; a NULL bias skips its row sum.
 *   d_latent_nhwc, d_xyz, d_viewdirs, cam : as in pnr_field_backward_cam.
 * The input-gradient chain stops below the lowest layer with a wanted tensor unless d_latent_nhwc, d_xyz, d_viewdirs
 * or cam is wanted, and the transposed weight copies of layers it does not reach are not made.  dlat = dh Wz runs only
 * for d_latent_nhwc, d_xyz or cam; the lin_in input GEMM and the geometry backward only for an input gradient.  With
 * nothing wanted the call returns before the forward recompute.  Same workspace as pnr_field_backward. */
int pnr_field_backward_sel(const PnrScene* scene, const PnrMlp* mlp, const float* xyz, const float* viewdirs,
                           const float* d_out, const PnrMlp* grad, float* d_latent_nhwc, float* d_xyz,
                           float* d_viewdirs, const PnrCameraGrad* cam, int64_t P, void* workspace,
                           size_t workspace_bytes, void* stream);

/* Backward of the compositing tail (pnr_composite; oracle/pnr_aux_backward.py::composite_backward): upstream gradients
 * d_rgb [R][3], d_depth [R], d_weights [R][K] (each may be NULL = zero) ->
 *   d_field [R][K][4] w.r.t. (sigmoid rgb, relu sigma), d_z [R][K] w.r.t. the sample depths (both overwritten).
 * d_z is the compositing's own term only (deltas and depth); the positions' share (points = o + z d) is not in it. */
int pnr_composite_backward(const float* rays, const float* z, const float* field, int32_t white_bkgd,
                           const float* d_rgb, const float* d_depth, const float* d_weights, float* d_field,
                           float* d_z, int64_t R, int32_t K, void* stream);

/* Backward of pnr_render for a loss on any of its outputs, i.e. what loss.backward() does below
 * `render_par(all_rays, want_weights=True)` (train/train.py:199-215, plus e.g. the alpha loss of model/loss.py on
 * fine.weights.sum(-1), or a depth loss):
 *   fwd          : the forward call's outputs that the backward needs: z_coarse, z_fine (sorted), depth_coarse
 *   up           : upstream gradients of the six outputs (NULL = all zero); a pass whose three gradients are all
 *                  NULL is skipped
 *   grad_*       : writable PnrMlp-shaped gradient buffers, accumulated (+=); grad_fine NULL when mlp_fine is NULL
 *   d_latent_nhwc: [V][Hl][Wl][C], accumulated (+=); may be NULL
 * The coarse weights are detached for importance sampling but the coarse depth is not (nerf.py:286-291), so the fine
 * outputs' gradients also reach the coarse MLP: d(depth_coarse) = up->d_depth_coarse + the depth-centred samples' share.
 * Arithmetic = oracle/pnr_aux_backward.py::render_backward.  Same workspace as pnr_render_backward.
 * This is the backward of the default CUDA training path (NeRFRenderer.forward in grad mode). */
size_t pnr_render_backward_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp_coarse,
                                           const PnrMlp* mlp_fine, const PnrRenderCfg* cfg, int64_t B);
int pnr_render_backward_ex(const PnrScene* scene, const PnrMlp* mlp_coarse, const PnrMlp* mlp_fine,
                           const PnrRenderCfg* cfg, const float* rays, const PnrNoise* noise,
                           const PnrRenderOut* fwd, const PnrRenderGrad* up, const PnrMlp* grad_coarse,
                           const PnrMlp* grad_fine, float* d_latent_nhwc, int64_t B, void* workspace,
                           size_t workspace_bytes, void* stream);

/* pnr_render_backward_ex plus the gradients of the rays and the source cameras (nerf.py:98-204, models.py:161-212):
 *   d_rays : [SB][B][8] = d(origin, direction, near, far), overwritten; NULL = not wanted.  points = o + z d and
 *            viewdirs = d (nerf.py:185, 204); the sample depths send their gradient to near / far through
 *            z = near (1 - s) + far s (stratified and importance samples of both passes, nerf.py:111-113, 146-147), the
 *            depth-centred samples z = max(min(depth + n std, far), near) (nerf.py:160) to the coarse depth, far or
 *            near as torch's min / max route it, and the last interval far - z_{K-1} (nerf.py:181) to far.
 *   cam    : camera gradients of both passes (+=), see PnrCameraGrad and pnr_field_backward_cam; NULL = none.
 * With both NULL this is pnr_render_backward_ex (same kernels, same bits); otherwise the coarse pass's positions
 * gradient is computed as well.  Not differentiated: image_shape and latent_scaling (buffers, as in the reference).
 * Same workspace as pnr_render_backward_ex. */
int pnr_render_backward_cam(const PnrScene* scene, const PnrMlp* mlp_coarse, const PnrMlp* mlp_fine,
                            const PnrRenderCfg* cfg, const float* rays, const PnrNoise* noise,
                            const PnrRenderOut* fwd, const PnrRenderGrad* up, const PnrMlp* grad_coarse,
                            const PnrMlp* grad_fine, float* d_latent_nhwc, float* d_rays, const PnrCameraGrad* cam,
                            int64_t B, void* workspace, size_t workspace_bytes, void* stream);
/* pnr_render_backward_cam for a partly frozen network (pnr_field_backward_sel's NULL rules): grad_coarse / grad_fine
 * may be NULL (that MLP frozen), and so may any of their members; wanted gradients are bit-equal to
 * pnr_render_backward_cam's.  A pass runs (field recompute, compositing backward, field backward) only when it has an
 * upstream gradient and its MLP has a wanted tensor or d_latent_nhwc, d_rays or cam is wanted.  The fine pass also runs
 * when depth-centred samples carry d(depth_coarse) to a coarse pass that runs; it then only computes the positions'
 * gradient for that.  Same workspace as pnr_render_backward_ex. */
int pnr_render_backward_sel(const PnrScene* scene, const PnrMlp* mlp_coarse, const PnrMlp* mlp_fine,
                            const PnrRenderCfg* cfg, const float* rays, const PnrNoise* noise,
                            const PnrRenderOut* fwd, const PnrRenderGrad* up, const PnrMlp* grad_coarse,
                            const PnrMlp* grad_fine, float* d_latent_nhwc, float* d_rays, const PnrCameraGrad* cam,
                            int64_t B, void* workspace, size_t workspace_bytes, void* stream);

/* pnr_render_backward_ex for a loss on the two rgb outputs only (train/train.py:199-215: MSE coarse + MSE fine):
 *   d_rgb_*      : [SB*B][3] upstream gradients, required (d_rgb_fine NULL when n_fine == 0)
 * Gradients w.r.t. the depth / weights outputs are not supported by this entry point; use pnr_render_backward_ex.
 * Arithmetic = oracle/pnr_backward.py::train_loss_backward; validated on H100 against the reference's own gradients. */
int pnr_render_backward(const PnrScene* scene, const PnrMlp* mlp_coarse, const PnrMlp* mlp_fine,
                        const PnrRenderCfg* cfg, const float* rays, const PnrNoise* noise,
                        const PnrRenderOut* fwd, const float* d_rgb_coarse, const float* d_rgb_fine,
                        const PnrMlp* grad_coarse, const PnrMlp* grad_fine, float* d_latent_nhwc, int64_t B,
                        void* workspace, size_t workspace_bytes, void* stream);

/* NeRFRenderer.forward (nerf.py:251-303) with the model call inlined:
 * sample_coarse -> composite(coarse) -> sample_fine(+depth) -> sort -> composite(fine).
 * rays [SB][B][8]; mlp_fine may be NULL (then mlp_coarse is used, models.py:242). */
size_t pnr_render_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp_coarse,
                                  const PnrMlp* mlp_fine, const PnrRenderCfg* cfg, int64_t B);
int pnr_render(const PnrScene* scene, const PnrMlp* mlp_coarse, const PnrMlp* mlp_fine,
               const PnrRenderCfg* cfg, const float* rays, const PnrNoise* noise,
               const PnrRenderOut* out, int64_t B, void* workspace, size_t workspace_bytes,
               void* stream);

/* Tensor-engine preparation (once per weight version / per encode()):
 *  - pnr_pack_mlp: fp32 nn.Linear weights -> fp16 hi/lo split, K-major 128B-swizzled wgmma tiles
 *    (128 output rows x 64 k, in the order the fused kernel consumes them).
 *  - pnr_project_latent: proj[i][v][y][x][:] = lin_z[i](latent[v,:,y,x]) (+ bias), so that the
 *    per-sample lin_z GEMMs (resnetfc.py:175) become a bilinear gather of the projected map
 *    (bilinear interpolation commutes with a linear layer).  In deterministic mode the workspace beyond its first
 *    3 * d_hidden floats (+ 256 B) holds the GEMM's split-K partials; 64 MiB more covers every shipped shape. */
size_t pnr_pack_mlp_bytes(const PnrMlp* mlp);
int pnr_pack_mlp(const PnrMlp* mlp, void* packed, size_t packed_bytes, void* stream);
size_t pnr_project_latent_bytes(const PnrScene* scene, const PnrMlp* mlp);
int pnr_project_latent(const PnrScene* scene, const PnrMlp* mlp, float* proj, size_t proj_bytes,
                       void* workspace, size_t workspace_bytes, void* stream);

/* ---- single-process multi-GPU driver: replaces nn.DataParallel(_RenderWrapper, gpus, dim=1), nerf.py:354-371 ----
 * One host thread, n devices of one node.  The read-only scene state is sent once per change (pnr_mgpu_broadcast, peer
 * copies over NVLink); a render call shards the rays along B with torch.chunk bounds (ceil(B/n) per device, in device
 * order -- the order DataParallel gathers in), runs ONE pnr_render per device and returns the pixels to device 0.  For a
 * single object (SB = 1) the final rgb / depth are stored by the kernels directly into the caller's tensors on
 * device 0 through peer memory; other outputs / SB > 1 come back as strided peer copies.  Asynchronous: the caller's
 * stream on device 0 waits for the shards.  Errors: as everywhere (negative code + pnr_last_error). */
typedef struct PnrMgpu PnrMgpu;   /* opaque: device list, events, fallback streams */

typedef struct PnrShard {         /* everything device i needs for its piece of a render call (pointers on device i) */
  const PnrScene* scene;          /* replica of the scene state on device i (host struct, device pointers)            */
  const PnrMlp* mlp_coarse;
  const PnrMlp* mlp_fine;         /* NULL: the coarse MLP serves both passes                                           */
  const PnrNoise* noise;          /* draws for the shard's SB * B_i rays (device i's generator, as under DataParallel)  */
  void* workspace;                /* >= pnr_render_workspace_bytes(scene, mlp_coarse, mlp_fine, cfg, B_i)              */
  size_t workspace_bytes;
  float* rays_stage;              /* [SB][B_i][8] on device i (unused for shard 0 when SB == 1)                        */
  PnrRenderOut stage;             /* local outputs [SB*B_i][...]: rgb / depth of both passes required, rest optional  */
  void* stream;                   /* stream on device i to enqueue on (NULL: the handle's own stream)                  */
} PnrShard;

/* Gradient mode (train/train.py with several --gpu_id): pnr_mgpu_render_backward is the backward of one pnr_mgpu_render
 * call.  Each shard runs pnr_render_backward_ex on its own device from the samples its forward left there; shard 0
 * accumulates into the caller's gradient buffers on device 0, every other shard into a zeroed gradient arena on its
 * device, and one kernel on device 0 then adds the arenas into device 0's, in shard order: grad0 += g_1 + ... + g_{n-1}
 * (read over NVLink where device 0 can address device i, else first copied into a device-0 staging buffer).
 * Shards on the same device run one after another on one stream, in the forward and the backward alike: the tensor
 * engine's fused launch needs the whole device. */
typedef struct PnrShardGrad {     /* everything device i needs for its piece of a backward call (pointers on device i) */
  const float* rays;              /* [SB][B_i][8] the rays the shard's forward rendered (rays_stage, or device 0's)   */
  const float* z_coarse;          /* [SB*B_i][Kc] the forward's samples: pnr_mgpu_render keeps stage.z_coarse /      */
  const float* z_fine;            /* [SB*B_i][Kc+Kf]  stage.z_fine / stage.depth_coarse on device i even when out0     */
  const float* depth_coarse;      /* [SB*B_i]         does not ask for them (z_fine NULL when n_fine == 0)            */
  float* up_stage;                /* SB*B_i*(8+2*Kc+Kf) floats: the shard's slices of up0 (unused: shard 0, SB == 1)   */
  const PnrMlp* grad_coarse;      /* shards i > 0: writable gradient buffers inside `arena` (shard 0: grad_coarse0)   */
  const PnrMlp* grad_fine;        /* NULL when mlp_fine is NULL                                                       */
  float* d_latent_nhwc;           /* [V][Hl][Wl][C] inside `arena`; NULL when d_latent0_nhwc is NULL                  */
  float* arena;                   /* i > 0: [arena_count] holding the three above, zeroed by the driver; i == 0: the  */
  int64_t arena_count;            /*   device-0 arena holding grad_coarse0 / grad_fine0 / d_latent0, same offsets     */
  float* arena_stage0;            /* [arena_count] on DEVICE 0, needed where pnr_mgpu_peer_load(h, i) == 0             */
  void* workspace;                /* >= pnr_render_backward_workspace_bytes(scene, mlp_coarse, mlp_fine, cfg, B_i)    */
  size_t workspace_bytes;
  void* stream;                   /* stream on device i (NULL: the handle's own stream)                               */
} PnrShardGrad;

/* Ray and camera gradients of a sharded step (pnr_render_backward_cam on every shard): one per shard, on device i. */
typedef struct PnrShardCam {
  PnrCameraGrad cam;              /* shards i > 0: buffers inside the shard's `arena`, at the offsets cam0 has in device */
                                  /*   0's arena, so the reduction sums them in shard order (shard 0: cam0 is used)      */
  float* d_rays;                  /* [SB][B_i][8] staging on device i, copied into rows [a, b) of d_rays0 (unused for   */
                                  /*   shard 0 of one object, which writes d_rays0 in place)                            */
} PnrShardCam;

int pnr_mgpu_create(const int32_t* device_ids, int32_t n, PnrMgpu** out);   /* enables peer access towards device_ids[0] */
int pnr_mgpu_destroy(PnrMgpu* h);
int32_t pnr_mgpu_size(const PnrMgpu* h);
int32_t pnr_mgpu_peer_store(const PnrMgpu* h, int32_t i);   /* 1 if device i can store into device 0's memory */
int32_t pnr_mgpu_peer_load(const PnrMgpu* h, int32_t i);    /* 1 if device 0 can read device i's memory (i > 0) */
/* dst[i] on device i  <-  src on device 0 (dst[0] ignored, NULL entries skipped); ordered after streams[0] (device 0)
 * and enqueued on streams[i] (NULL array / entry: the handle's own streams). */
int pnr_mgpu_broadcast(PnrMgpu* h, const void* src, void* const* dst, size_t bytes, void* const* streams);
/* rays0 [SB][B][8] and out0 (tensors [SB*B][...], NULL = not wanted) on device 0; shards[n]. */
int pnr_mgpu_render(PnrMgpu* h, const PnrShard* shards, const PnrRenderCfg* cfg, const float* rays0,
                    const PnrRenderOut* out0, int64_t B, void* stream0);
/* Backward of the pnr_mgpu_render call made with the same shards, cfg and B.  up0: upstream gradients on device 0,
 * [SB*B][...] as out0 (NULL / NULL entries = zero); grad_coarse0, grad_fine0, d_latent0_nhwc: device 0's buffers,
 * accumulated (+=) as in pnr_render_backward_ex.  On return every shard's stream is ordered after the reduction, so
 * the caller may release the shard buffers; the caller's stream0 is ordered after everything. */
int pnr_mgpu_render_backward(PnrMgpu* h, const PnrShard* shards, const PnrShardGrad* shard_grads,
                             const PnrRenderCfg* cfg, const PnrRenderGrad* up0, const PnrMlp* grad_coarse0,
                             const PnrMlp* grad_fine0, float* d_latent0_nhwc, int64_t B, void* stream0);
/* pnr_mgpu_render_backward plus the gradients of the rays and the source cameras (pnr_render_backward_cam):
 *   d_rays0     : [SB][B][8] on device 0, overwritten; NULL = not wanted.  Each shard's rows come back as the reverse
 *                 of the forward's strided ray staging.
 *   cam0        : device 0's camera gradients (+=), inside shard 0's arena when there are several shards; NULL = none.
 *   shard_cams  : [n] per-shard buffers (PnrShardCam); may be NULL when d_rays0 and cam0 are.
 * Camera gradients of every shard are summed onto cam0 by the same reduction as the weights, in shard order.  With
 * d_rays0 and cam0 NULL this is pnr_mgpu_render_backward. */
int pnr_mgpu_render_backward_cam(PnrMgpu* h, const PnrShard* shards, const PnrShardGrad* shard_grads,
                                 const PnrShardCam* shard_cams, const PnrRenderCfg* cfg, const PnrRenderGrad* up0,
                                 const PnrMlp* grad_coarse0, const PnrMlp* grad_fine0, float* d_latent0_nhwc,
                                 float* d_rays0, const PnrCameraGrad* cam0, int64_t B, void* stream0);
/* pnr_mgpu_render_backward_cam over pnr_render_backward_sel on every shard: grad_coarse0 / grad_fine0 and their members
 * may be NULL (frozen), and each shard's structs must be NULL in the same places.  The arenas then hold only the wanted
 * tensors, so the reduction adds fewer floats; an arena_count of 0 (nothing but ray gradients wanted) skips it. */
int pnr_mgpu_render_backward_sel(PnrMgpu* h, const PnrShard* shards, const PnrShardGrad* shard_grads,
                                 const PnrShardCam* shard_cams, const PnrRenderCfg* cfg, const PnrRenderGrad* up0,
                                 const PnrMlp* grad_coarse0, const PnrMlp* grad_fine0, float* d_latent0_nhwc,
                                 float* d_rays0, const PnrCameraGrad* cam0, int64_t B, void* stream0);
/* The reduction step on its own: dst[j] += src[0][j] + src[1][j] + ... + src[n-1][j], added left to right, for
 * j < count.  src: host array of n <= 63 device pointers readable from the current device. */
int pnr_sum_into(float* dst, const float* const* src, int32_t n, int64_t count, void* stream);

/* Sharded field evaluation for mesh extraction (util/recon.py marching_cubes with several GPUs): the field of ONE object
 * (scene SB == 1) at points [0, count) of a point set that every device generates itself, channels
 * [channel, channel + n_channels) of each point's output stored into out0 [count][n_channels] on device 0.
 * The points are cut into chunks of `chunk` points starting at 0 (the chunks a one-GPU loop of pnr_field_eval calls
 * evaluates), and shard i takes torch.chunk piece i of the chunk indices: a contiguous run of whole chunks, so every
 * point is evaluated in the same chunk, at the same offset, as in the one-GPU loop, and the result is bit-equal to it
 * with every engine.  Shards past the last chunk do nothing.  Per chunk, on device i: the points and view directions
 * into the shard's workspace (pnr_grid_points / pnr_band_lattice_points / pnr_band_points, or a peer copy of the
 * chunk's rows of a LIST), one pnr_field_eval, then one small kernel that stores the wanted channels into out0 -- through
 * peer memory where pnr_mgpu_peer_store(h, i), else into a staging slice of the workspace that is peer-copied to out0.
 * Shards on the same device run one after another on one stream (as in pnr_mgpu_render); stream0 (device 0) is
 * ordered after every shard.  Asynchronous, no host synchronisation.
 * Errors (PNR_ERR_INVALID): an unknown kind, bad reso / block / apron, count outside the grid or lattice, count !=
 * n_points for BAND, NULL LIST rows or BAND plan, chunk < 1, a channel range outside [0, d_out), a scene with SB != 1;
 * PNR_ERR_WORKSPACE: a shard workspace below pnr_mgpu_field_workspace_bytes.  Every shard with chunks is checked before
 * anything is enqueued. */
enum { PNR_POINTS_GRID = 1, PNR_POINTS_LATTICE = 2, PNR_POINTS_BAND = 3, PNR_POINTS_LIST = 4 };

typedef struct PnrPointSource {   /* which points; host struct                                                           */
  int32_t kind;                   /* PNR_POINTS_*                                                                        */
  double lo[3], hi[3];            /* GRID / LATTICE / BAND: the bounds pnr_grid_points / pnr_band_*_points take           */
  int32_t reso[3];                /* GRID / LATTICE / BAND                                                               */
  int32_t block, apron;           /* LATTICE (block) / BAND (block, apron): as pnr_band_lattice_points / pnr_band_points */
  int64_t n_points;               /* BAND: the plan's refinement point count (must equal count)                          */
  const float* xyz0;              /* LIST: [count][3] points on DEVICE 0                                                 */
  const float* viewdirs0;         /* LIST: [count][3] view directions on DEVICE 0                                        */
} PnrPointSource;

typedef struct PnrFieldShard {    /* device i's piece (pointers on device i)                                             */
  const PnrScene* scene;          /* the scene on device i (shard 0: device 0's own); SB == 1                            */
  const PnrMlp* mlp;              /* evaluated with scene->proj_coarse, as pnr_field_eval does                           */
  const void* plan;               /* BAND: the pnr_band_plan buffer on device i                                          */
  size_t plan_bytes;
  void* workspace;                /* >= pnr_mgpu_field_workspace_bytes(scene, mlp, chunk, engine)                        */
  size_t workspace_bytes;
  void* stream;                   /* stream on device i (NULL: the handle's own; shard 0 always runs on stream0)         */
} PnrFieldShard;

size_t pnr_mgpu_field_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp, int64_t chunk, int32_t engine);
int pnr_mgpu_field_eval(PnrMgpu* h, const PnrFieldShard* shards, const PnrPointSource* src, int64_t count,
                        int64_t chunk, int32_t engine, int32_t channel, int32_t n_channels, float* out0,
                        void* stream0);

/* ---- mesh extraction: util/recon.py marching_cubes (src/util/recon.py:12-78) ------------------------------------ */

/* The evaluation grid of recon.py:43, util.gen_grid(*zip(lo, hi, reso), ij_indexing=True) (src/util/util.py:93-110):
 * points [first, first+count) of the nx*ny*nz grid in ij order (x slowest) -> xyz [count][3].  Each axis is
 * np.linspace(lo, hi, n, dtype=float32): computed in float64 with the last point set to hi, then rounded, so the
 * points are bit-equal to the reference's.  viewdirs (may be NULL) [count][3] = -p / |p| in fp32 (recon.py:54, with
 * |p| = sqrt((x*x + y*y) + z*z) as torch's CPU norm sums it there, so the bits agree too); a grid point at the origin
 * gets NaN there, as in the reference.
 * lo, hi (double[3]) and reso (int32[3], each >= 1) are HOST arrays. */
int pnr_grid_points(const double* lo, const double* hi, const int32_t* reso, int64_t first, int64_t count, float* xyz,
                    float* viewdirs, void* stream);

/* Marching cubes over a dense fp32 volume vol [nx][ny][nz] (what recon.py:68 `sigmas.view(*reso)` is), in two phases
 * so that the caller can size the outputs exactly:
 *   pnr_mc_count: counts_out[0] = vertices, counts_out[1] = triangles (int64, DEVICE memory); leaves in the workspace
 *                 the edge flags, vertex ids, cell configurations and triangle offsets that pnr_mc_emit reads.
 *   pnr_mc_emit : same vol / dims / iso / workspace, after pnr_mc_count on the same stream ->
 *                 verts [n_verts][3] float64, tris [n_tris][3] int64 vertex ids (n_* = the counted values).
 * A corner is inside when it is finite and sigma > iso.  One vertex per grid edge whose corners differ, numbered in
 * (grid point, axis) order and shared by every cell touching the edge (the mesh is welded), at the lower corner's grid
 * index plus t = (iso - s_a) / (s_b - s_a) along the edge in float64 (0.5 when the outside corner is NaN or infinite).  Triangles
 * come from generated tables (oracle/make_mc_tables.py), cells in linear order, counter-clockwise seen from outside
 * the inside region (normals toward decreasing sigma; pnr_mc_vertex_attrs gives per-vertex ones); every face is resolved from its own four corners, so the
 * surface is watertight.  Offsets are exclusive scans (no atomics): repeated calls give the same bits.
 * A dimension below 2 gives no cells, vertices or triangles.  Errors: dimensions < 1 or above 2^36 points, negative
 * sizes, NULL pointers -> PNR_ERR_INVALID; workspace < pnr_mc_workspace_bytes -> PNR_ERR_WORKSPACE. */
size_t pnr_mc_workspace_bytes(int32_t nx, int32_t ny, int32_t nz);
int pnr_mc_count(const float* vol, int32_t nx, int32_t ny, int32_t nz, double iso, int64_t* counts_out,
                 void* workspace, size_t workspace_bytes, void* stream);
int pnr_mc_emit(const float* vol, int32_t nx, int32_t ny, int32_t nz, double iso, double* verts, int64_t* tris,
                int64_t n_verts, int64_t n_tris, void* workspace, size_t workspace_bytes, void* stream);

/* Per-vertex attributes of the mesh pnr_mc_emit writes (call it after pnr_mc_count on the same stream, with the same
 * vol / dims / iso / workspace); attribute i belongs to vertex i.  lo, hi: HOST double[3], the bounds the grid spans
 * (pnr_grid_points' lo / hi), h_k = (hi_k - lo_k) / (n_k - 1).  All in float64 with round-to-nearest intrinsics, no
 * atomics: repeated calls give the same bits.
 *   normals  [n_verts][3] float64: -G / |G|, toward decreasing sigma (the side the winding faces).  G is the grid
 *            gradient of sigma at the edge's corners a, b, interpolated as (1 - t) g(a) + t g(b) with the vertex's t,
 *            then divided by h_k.  Per axis at a grid point, g is the central difference where both neighbours exist
 *            and are finite, else the forward, else the backward difference where the point and that neighbour are
 *            finite, else 0, so a non-finite sigma never spreads into its neighbours.  |G|^2 = (Gx^2 + Gy^2) + Gz^2;
 *            where |G| is 0 or not finite, the unit vector along the edge from its inside corner to its outside one.
 *   xyz      [n_verts][3] fp32: the vertex's world position lo + v h (v its index coordinate), with pnr_grid_points'
 *            bits on grid indices.  This is where the surface is, unlike recon.py's returned vertices, which keep the
 *            reference's (c2 - c1) / reso scale.
 *   viewdirs [n_verts][3] fp32: -normal, a camera facing the surface head-on from outside.
 * Any output may be NULL.  A dimension below 2 returns PNR_OK without writing.  Errors: dimensions < 1 or above 2^36
 * points, negative n_verts, NULL vol / lo / hi -> PNR_ERR_INVALID; workspace < pnr_mc_workspace_bytes ->
 * PNR_ERR_WORKSPACE. */
int pnr_mc_vertex_attrs(const float* vol, int32_t nx, int32_t ny, int32_t nz, double iso, const double* lo,
                        const double* hi, double* normals, float* xyz, float* viewdirs, int64_t n_verts,
                        void* workspace, size_t workspace_bytes, void* stream);

/* Narrow-band marching cubes: the mesh of the entry points above with every cell outside the active blocks treated as
 * empty and the vertices no remaining triangle uses dropped (the order stays the dense one: vertex ids by (grid
 * point, axis), triangles by cell, then table order).  Only the blocks the surface crosses, seen on a coarse lattice,
 * are refined, so sigma is evaluated and workspace taken for the band around the surface instead of the whole grid.
 * reso: HOST int32[3] as pnr_grid_points takes it; block: b cells per side, 2 <= b <= 256; apron: 0 or 1.
 *   blocks       block i of an axis covers the cells [i b, min((i + 1) b, n - 1)); nb = ceil((n - 1) / b) per axis.
 *   lattice      the grid indices min(j b, n - 1), j = 0 .. nb, per axis: (nb0 + 1)(nb1 + 1)(nb2 + 1) grid points in
 *                ij order, so block i's corners are lattice points i and i + 1.
 *   seeded       a block whose 8 corners are not all in the same state (inside = finite and sigma > iso);
 *   active       a block that is seeded or has a seeded one among its 26 neighbours.
 *   refinement   the grid points of the active blocks' closed cells ([i b, min((i + 1) b, n - 1)] per axis), with
 *                apron = 1 widened by one point on each side (the neighbours the vertex normals read), in ij order
 *                (x slowest), as the grid orders them.
 * Where every non-empty cell of the dense extraction lies in an active block the mesh is the dense one, bit for bit;
 * otherwise pieces are missing (a feature smaller than a block that no lattice point sees) and the mesh can be open
 * where the surface leaves the band.
 *
 *   pnr_band_plan_bytes     the plan buffer for reso / block / apron (0 when they are invalid); it grows with the
 *                           block grid (a few bytes per block and per run of points: 2 or 3 runs per block per axis).
 *   pnr_band_lattice_points lattice points [first, first+count) -> xyz / viewdirs, bit-equal to pnr_grid_points' at
 *                           the same grid index.
 *   pnr_band_plan           coarse [nb0 + 1][nb1 + 1][nb2 + 1] fp32 sigma of the lattice -> the plan (active blocks and
 *                           the offsets that index the refinement set, and a header recording reso, block, apron and
 *                           the point count); counts_out (int64[2], DEVICE) = active blocks, refinement points.
 *   pnr_band_points         refinement points [first, first+count) -> xyz / viewdirs, as pnr_band_lattice_points.
 *                           n_points must be the plan's count; no point past it is written.
 *   pnr_band_mc_workspace_bytes  the marching-cubes workspace for n_points refinement points (37 bytes per point).
 *   pnr_band_mc_count / pnr_band_mc_emit / pnr_band_mc_vertex_attrs  pnr_mc_count / pnr_mc_emit /
 *                           pnr_mc_vertex_attrs over sigma [n_points], the field at the refinement points in their
 *                           order, with the same plan and workspace on the same stream; the same arithmetic, exclusive
 *                           scans and no atomics, so repeated calls give the same bits.  Each reads the plan's header
 *                           back (one synchronise of the stream) and refuses a plan made for another reso / block /
 *                           apron or another n_points; vertex attributes need apron = 1.
 * Errors: dimensions < 1 or above 2^36 points, block outside [2, 256], apron not 0 / 1, ranges outside the lattice or
 * the refinement set, a plan that does not match the call, negative sizes, NULL pointers -> PNR_ERR_INVALID; a plan
 * buffer below pnr_band_plan_bytes or a workspace below pnr_band_mc_workspace_bytes -> PNR_ERR_WORKSPACE. */
size_t pnr_band_plan_bytes(const int32_t* reso, int32_t block, int32_t apron);
int pnr_band_lattice_points(const double* lo, const double* hi, const int32_t* reso, int32_t block, int64_t first,
                            int64_t count, float* xyz, float* viewdirs, void* stream);
int pnr_band_plan(const float* coarse, const int32_t* reso, int32_t block, double iso, int32_t apron,
                  int64_t* counts_out, void* plan, size_t plan_bytes, void* stream);
int pnr_band_points(const double* lo, const double* hi, const int32_t* reso, int32_t block, int32_t apron,
                    const void* plan, size_t plan_bytes, int64_t n_points, int64_t first, int64_t count, float* xyz,
                    float* viewdirs, void* stream);
size_t pnr_band_mc_workspace_bytes(int64_t n_points);
int pnr_band_mc_count(const float* sigma, int64_t n_points, const int32_t* reso, int32_t block, int32_t apron,
                      double iso, const void* plan, size_t plan_bytes, int64_t* counts_out, void* workspace,
                      size_t workspace_bytes, void* stream);
int pnr_band_mc_emit(const float* sigma, int64_t n_points, const int32_t* reso, int32_t block, int32_t apron,
                     double iso, const void* plan, size_t plan_bytes, double* verts, int64_t* tris, int64_t n_verts,
                     int64_t n_tris, void* workspace, size_t workspace_bytes, void* stream);
int pnr_band_mc_vertex_attrs(const float* sigma, int64_t n_points, const int32_t* reso, int32_t block, int32_t apron,
                             double iso, const double* lo, const double* hi, const void* plan, size_t plan_bytes,
                             double* normals, float* xyz, float* viewdirs, int64_t n_verts, void* workspace,
                             size_t workspace_bytes, void* stream);

/* TSDF fusion of rendered depth maps (no counterpart in the reference; util/recon.py fuse_views): a truncated signed
 * distance volume tsdf [nx][ny][nz] fp32 (DEVICE) from V views' depth and opacity maps depth / opacity [V][H][W] fp32
 * (DEVICE: the renderer's depth sum(w z) and weights.sum(-1) of each pixel, the pixel order of pnr_gen_rays) and their
 * camera-to-world poses_c2w [V][4][4] fp32 (DEVICE, as pnr_gen_rays takes them).  fx, fy, cx, cy: HOST floats, as
 * pnr_gen_rays; lo, hi (double[3]) and reso (int32[3]): HOST, as pnr_grid_points.  One thread per voxel, the views in
 * order, no atomics: repeated calls give the same bits.  All in float64 with round-to-nearest intrinsics.  Voxel x is
 * pnr_grid_points' point (lo + i (hi - lo) / (n - 1) rounded to fp32).  Per view v, with R = pose[:3, :3], t =
 * pose[:3, 3]:
 *   q = R^T (x - t), each component (R0j d0 + R1j d1) + R2j d2.  q_z >= 0: v does not see the voxel.
 *   px = cx + fx q_x / (-q_z), py = cy + fy q_y / q_z (the inverse of pnr_gen_rays: -z forward, +y up, pixel centres on
 *   integers), rounded to the nearest pixel as floor(p + 0.5) (ties round up).  Outside [0, W-1] x [0, H-1]: v does
 *   not see the voxel.
 *   a = opacity of that pixel.  a < min_opacity (or NaN): the pixel saw background, s = +1 (free space).  Otherwise
 *   s = (depth / a - d) / trunc with d = sqrt((q_x^2 + q_y^2) + q_z^2) (the rays are unit-norm, so depth is a distance
 *   along the ray); s < -1 (or NaN): occluded, no observation; else s = min(s, 1).
 * tsdf = the mean of the observations' s (summed in view order).  A voxel with no observation gets -1 (inside) when some
 * view saw it in front of the camera and inside its image, and +1 (outside) when none did, so every voxel has a value
 * and pnr_mc_count / pnr_mc_emit mesh -tsdf at iso 0 (positive inside) as they are.
 * Errors (before any CUDA call): NULL pointers, V, W or H < 1, reso outside [1, 2^36 points], trunc not positive and
 * finite, min_opacity outside (0, 1] -> PNR_ERR_INVALID. */
int pnr_tsdf_fuse(const float* depth, const float* opacity, int32_t V, int32_t W, int32_t H, const float* poses_c2w,
                  float fx, float fy, float cx, float cy, const double* lo, const double* hi, const int32_t* reso,
                  double trunc, double min_opacity, float* tsdf, void* stream);

/* Vertex colours from rendered views (no counterpart in the reference; util/recon.py fuse_views(colors="views")): each
 * vertex gets the weighted mean of the rendered pixels of the views that see it, under pnr_tsdf_fuse's visibility.
 * xyz, normals [n][3] float64 (DEVICE: world-space vertices and their unit outward normals); rgb [V][H][W][3], depth
 * and opacity [V][H][W] fp32 (DEVICE: the renderer's rgb, sum(w z) and weights.sum(-1) of each pixel, the pixel order
 * of pnr_gen_rays); poses_c2w [V][4][4] fp32 (DEVICE); fx, fy, cx, cy: HOST floats, as pnr_tsdf_fuse.  One thread per
 * vertex, the views in order, no atomics: repeated calls give the same bits.  All in float64 with round-to-nearest
 * intrinsics.  Per view v, with R = pose[:3, :3], t = pose[:3, 3], vertex x and normal n:
 *   q, px, py and the pixel as pnr_tsdf_fuse (the same device code); q_z >= 0 or outside the image: skip v.
 *   a = opacity of that pixel.  a < min_opacity (or NaN): the pixel saw background, which has no surface colour;
 *   skip v.
 *   s = (depth / a - d) / trunc with d = sqrt((q_x^2 + q_y^2) + q_z^2).  |s| > 1 (or NaN): v sees another surface
 *   (occluded) or this one elsewhere; skip v.
 *   cos = ((n_0 e_0 + n_1 e_1) + n_2 e_2) / d with e = t - x.  cos <= 0 (or NaN): v faces the back of the surface;
 *   skip v.
 *   c_k = (rgb_k - background (1 - a)) / a per channel, then clamped to [0, 1] (NaN -> 0): the renderer composites
 *   sum(w c) + background (1 - sum(w)), so this is the ray's mean surface colour sum(w c) / sum(w).
 *   sum_c += cos c, sum_w += cos (in view order).
 * rgb_out [n][3] fp32 (DEVICE) = sum_c / sum_w rounded to fp32, NaN where no view painted the vertex; weight_out [n]
 * float64 (DEVICE) = sum_w, 0 where no view painted it.  background: 1 for a white_bkgd renderer, else 0.
 * Errors (before any CUDA call): NULL pointers, n < 0, V, W or H < 1, trunc not positive and finite, min_opacity
 * outside (0, 1], background not finite -> PNR_ERR_INVALID.  n = 0 launches nothing. */
int pnr_paint_vertices(const double* xyz, const double* normals, int64_t n, const float* rgb, const float* depth,
                       const float* opacity, int32_t V, int32_t W, int32_t H, const float* poses_c2w, float fx,
                       float fy, float cx, float cy, double trunc, double min_opacity, double background,
                       float* rgb_out, double* weight_out, void* stream);

/* Connected components of a triangle mesh (no counterpart in the reference; util/recon.py keep_components), in two
 * steps that share one workspace of pnr_mesh_workspace_bytes(n_verts, n_tris) bytes on one stream.  tris [n_tris][3]
 * int64 vertex ids (DEVICE).  Two vertices are connected when some triangle uses both; a component is a maximal
 * connected set of vertices with its triangles.  The meshes of pnr_mc_emit are welded, so this is their connectivity.
 *   pnr_mesh_components  label [n_verts] int64 (DEVICE) = the smallest vertex id of each vertex's component (a vertex
 *                        no triangle uses is its own component); tri_count [n_verts] int64 (DEVICE) = at a component's
 *                        label, its number of triangles, 0 at every other index; *counts_out (HOST int64) = the number
 *                        of components with at least one triangle.  Lock-free union-find over the edges (a, b), (a, c)
 *                        of each triangle: a root is only ever hooked under a smaller root (64-bit atomicCAS), so every
 *                        root is its component's minimum whatever the order the threads run in, then one full path
 *                        compression and integer atomicAdd counts.  The result is one function of the input:
 *                        repeated calls give the same bits.  Synchronises the stream once, to download the count and
 *                        the device-side check of the ids.
 *   pnr_mesh_compact_count  keep_root [n_verts] uint8 (DEVICE), read at the labels: a vertex is kept when
 *                        keep_root[label[v]] != 0, a triangle when its first vertex is.  counts_out (int64[2], DEVICE) =
 *                        kept vertices, kept triangles (exclusive scans of the flags, no atomics); leaves in the
 *                        workspace the flags and new ids pnr_mesh_compact_emit reads.
 *   pnr_mesh_compact_emit  after pnr_mesh_compact_count with the same tris / label / keep_root / workspace ->
 *                        vert_ids [n_keep_verts] int64: the kept vertices' old ids, ascending (new id i is old id
 *                        vert_ids[i]); tris_out [n_keep_tris][3] int64: the kept triangles in their order, through the
 *                        new ids (n_keep_* = the counted values).
 * Errors: n_verts or n_tris negative, NULL pointers where a size is non-zero -> PNR_ERR_INVALID; a vertex id outside
 * [0, n_verts) -> PNR_ERR_INVALID from pnr_mesh_components (found on the device, reported after its synchronise;
 * label and tri_count are then unspecified).  The compact steps take the tris pnr_mesh_components accepted and the
 * label it wrote (a triangle with an id out of range is never kept).  A workspace below pnr_mesh_workspace_bytes ->
 * PNR_ERR_WORKSPACE.  n_tris = 0 or n_verts = 0 launch no union-find. */
size_t pnr_mesh_workspace_bytes(int64_t n_verts, int64_t n_tris);
int pnr_mesh_components(const int64_t* tris, int64_t n_tris, int64_t n_verts, int64_t* label, int64_t* tri_count,
                        int64_t* counts_out, void* workspace, size_t workspace_bytes, void* stream);
int pnr_mesh_compact_count(const int64_t* tris, int64_t n_tris, int64_t n_verts, const int64_t* label,
                           const uint8_t* keep_root, int64_t* counts_out, void* workspace, size_t workspace_bytes,
                           void* stream);
int pnr_mesh_compact_emit(const int64_t* tris, int64_t n_tris, int64_t n_verts, int64_t* vert_ids, int64_t* tris_out,
                          int64_t n_keep_verts, int64_t n_keep_tris, void* workspace, size_t workspace_bytes,
                          void* stream);

/* Decimation of a triangle mesh (no counterpart in the reference; util/recon.py decimate, oracle/pnr_recon_decimate.py):
 * rounds of independent half-edge collapses with Garland-Heckbert quadrics, on one stream, with one workspace of
 * pnr_decimate_workspace_bytes(n_verts, n_tris) bytes for the initial sizes (it fits every later, smaller round).
 * xyz [n_verts][3] float64, tris [n_tris][3] int64, quadrics [n_verts][10] float64 (a00 a01 a02 a11 a12 a22 b0 b1 b2 c
 * of Q(p) = p'Ap + 2b'p + c), all DEVICE.  Every float64 operation rounds to nearest in the order the oracle writes.
 *   Quadrics  a triangle (p0, p1, p2) has n = (p1 - p0) x (p2 - p0); when |n|^2 > 0 it contributes area * (u u', u d,
 *             d^2) with u = n / |n|, d = -u.p0, area = |n| / 2, else nothing.  A vertex's quadric is the sum over its
 *             incident triangles in ascending id (once per corner), starting from 0; a collapse c -> d sets Q_d += Q_c.
 *             A vertex with more than 64 corners at the start is frozen for the whole call: it is never removed and
 *             never a d (so its quadric, written as 0, is never read), even after collapses around it take corners
 *             away.  Cone tips and the poles of UV spheres are such vertices.
 *   Error     of c -> d: Q = Q_c + Q_d at p_d, err = sqrt(max(Q(p_d), 0) / trace(A)), 0 when trace(A) = 0.
 *   Vertices  v's corners are its incident triangles, each rotated to (v, x, y); its neighbours are the other ids;
 *             valence = their number.  A vertex with more than 64 corners in a round is not examined in it:
 *             valence +inf, no flags.  A frozen vertex has no flags.
 *             Fan: no incident triangle repeats an id, every neighbour is the x of at most one corner and the y of at
 *             most one, and the link edges x -> y form one path or one cycle.  Removable: a fan whose link is a cycle
 *             (closed: every incident edge has two triangles) with 3 to 32 neighbours.
 *   Valid     c -> d: c removable; d a fan; valence(c) + valence(d) - 4 <= 32; with (c, d, o1) and (c, o2, d) the
 *             corners of c at d, valence(o1), valence(o2) >= 4 and c, d share no neighbour but o1, o2; no triangle of c
 *             without d flips (n0 != 0 and n0.n1 <= 0, n1 with c replaced by d); err <= max_error.
 *   Edge      {a, b} takes its cheaper valid direction, on a tie removing the larger id; key (err, min id, max id).
 *             best(v) = the smallest key at v, (+inf, INT64_MAX, INT64_MAX) without one.  An edge is selected when it
 *             is best(a) and best(b) and its key is below best(w) for every other neighbour w of a or b: no two
 *             selected edges touch or neighbour each other, so a round equals its collapses applied in any order.
 *   pnr_decimate_init    checks the ids (one synchronise; PNR_ERR_INVALID for an id outside [0, n_verts)) and writes
 *                        the initial quadrics and frozen [n_verts] uint8 (DEVICE, 1 = frozen), which select reads.
 *   pnr_decimate_select  -> c_out, d_out [n_verts / 2] int64 and err_out [n_verts / 2] float64 (DEVICE): the selected
 *                        collapses in ascending c; counts_out (HOST int64[2]) = their number, and 1 when some collapse
 *                        was valid but for max_error (pass +inf for no bound).  Synchronises once.
 *   pnr_decimate_apply   the collapses (c[i], d[i]) of one selection (any subset of it): Q_d += Q_c, each c rewritten
 *                        to its d, each edge cd's two triangles dropped, the rest compacted in order into tris_out
 *                        [n_tris][3] (not tris); *count_out (HOST) = their number.  Synchronises once.
 * Errors: negative sizes, NULL pointers where a size is non-zero, a negative or NaN max_error, n_collapses outside
 * [0, n_verts / 2] -> PNR_ERR_INVALID; a workspace below pnr_decimate_workspace_bytes -> PNR_ERR_WORKSPACE. */
size_t pnr_decimate_workspace_bytes(int64_t n_verts, int64_t n_tris);
int pnr_decimate_init(const double* xyz, int64_t n_verts, const int64_t* tris, int64_t n_tris, double* quadrics,
                      uint8_t* frozen, void* workspace, size_t workspace_bytes, void* stream);
int pnr_decimate_select(const double* xyz, int64_t n_verts, const int64_t* tris, int64_t n_tris,
                        const double* quadrics, const uint8_t* frozen, double max_error, int64_t* c_out,
                        int64_t* d_out, double* err_out, int64_t* counts_out, void* workspace,
                        size_t workspace_bytes, void* stream);
int pnr_decimate_apply(const int64_t* tris, int64_t n_tris, int64_t n_verts, const int64_t* c, const int64_t* d,
                       int64_t n_collapses, double* quadrics, int64_t* tris_out, int64_t* count_out, void* workspace,
                       size_t workspace_bytes, void* stream);

/* Test hook for the dense contraction the backward path is built from (nn.Linear forward / input gradient / weight
 * gradient are all this "NT" product): C[M][N] (+)= act(A[M][lda]) * W[N][K]^T (+ bias[N]), fp32 in and out.
 * engine = PNR_ENGINE_SIMT: fp32 FFMA SGEMM; PNR_ENGINE_TC (or AUTO): split-bf16 wgmma GEMM (3 products, fp32
 * accumulate, split-K with atomics when the output has few tiles) -- the backward's engine; PNR_GEMM_F16X3: the same
 * kernel with fp16 hi/lo operands (22 mantissa bits inside fp16's range) -- pnr_project_latent's engine.
 * K % 16 == 0, rows 16-byte aligned. */
#define PNR_GEMM_F16X3 3
int pnr_gemm_nt(const float* A, int32_t lda, const float* W, const float* bias, float* C, int32_t ldc, int32_t M,
                int32_t N, int32_t K, int32_t relu_a, int32_t accum, int32_t engine, void* stream);

/* How many kernels this library has launched in this process (bench.py "gpu_launches"). */
int64_t pnr_launch_count(void);

/* Device-time profile of the DOMINANT kernel (the MLP contraction: the fused wgmma kernel of
 * the tensor engine, or the SGEMM of the SIMT engine).  Between begin and end every launch of
 * that kernel is bracketed by cudaEvents on its own stream; end synchronises those events and
 * returns the summed device milliseconds and the number of launches.  Off by default. */
int pnr_profile_begin(void);
int pnr_profile_end(double* total_ms, int64_t* launches);

/* Debug / test hook for the tensor engine: synchronises the current device and returns its
 * status word (0 = ok, otherwise the tag of the first barrier wait that timed out), then clears it. */
int pnr_tc_status(int* status);
/* Debug: per-role stall-cycle counters of the tensor engine (8 values, documented at pnr_tc_counters in
 * csrc/pnr_field_tc.cu); synchronises the device and clears them. */
int pnr_tc_counters(unsigned long long* out8);

#ifdef __cplusplus
}
#endif
#endif /* PNR_H_ */
