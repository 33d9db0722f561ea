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
  PNR_ENGINE_TC = 2      /* wgmma split-fp16 (3 products, fp32 accumulate) fused kernel */
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

int pnr_abi_version(void);
const char* pnr_last_error(void);

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

/* Backward of pnr_render for a loss on the two rgb outputs (train/train.py:199-215: MSE coarse + MSE fine), i.e. what
 * loss.backward() does below `render_par(all_rays, want_weights=True)`:
 *   fwd          : the forward call's outputs that the backward needs: z_coarse, z_fine (sorted), depth_coarse
 *   d_rgb_*      : [SB*B][3] upstream gradients (d_rgb_fine NULL when n_fine == 0)
 *   grad_*       : writable PnrMlp-shaped gradient buffers, accumulated (+=); grad_fine NULL when mlp_fine is NULL
 *   d_latent_nhwc: [V][Hl][Wl][C], accumulated (+=); may be NULL
 * The coarse weights are detached for importance sampling but the coarse depth is not (nerf.py:286-291), so the fine
 * loss also reaches the coarse MLP.  Gradients w.r.t. the depth / weights outputs are not supported.
 * Arithmetic = oracle/pnr_backward.py::train_loss_backward; validated on H100 against the reference's own gradients.
 * This is the backward of the default CUDA training path (NeRFRenderer.forward in grad mode). */
size_t pnr_render_backward_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp_coarse,
                                           const PnrMlp* mlp_fine, const PnrRenderCfg* cfg, int64_t B);
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
 *    (bilinear interpolation commutes with a linear layer). */
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

int pnr_mgpu_create(const int32_t* device_ids, int32_t n, PnrMgpu** out);   /* enables peer access towards device_ids[0] */
int pnr_mgpu_destroy(PnrMgpu* h);
int32_t pnr_mgpu_size(const PnrMgpu* h);
int32_t pnr_mgpu_peer_store(const PnrMgpu* h, int32_t i);   /* 1 if device i can store into device 0's memory */
/* dst[i] on device i  <-  src on device 0 (dst[0] ignored, NULL entries skipped); ordered after streams[0] (device 0)
 * and enqueued on streams[i] (NULL array / entry: the handle's own streams). */
int pnr_mgpu_broadcast(PnrMgpu* h, const void* src, void* const* dst, size_t bytes, void* const* streams);
/* rays0 [SB][B][8] and out0 (tensors [SB*B][...], NULL = not wanted) on device 0; shards[n]. */
int pnr_mgpu_render(PnrMgpu* h, const PnrShard* shards, const PnrRenderCfg* cfg, const float* rays0,
                    const PnrRenderOut* out0, int64_t B, void* stream0);

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
