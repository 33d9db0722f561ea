// Single-process multi-GPU driver of the ray-sharded render (C ABI: pnr_mgpu_*, include/pnr.h).
//
// Replaces `torch.nn.DataParallel(_RenderWrapper, gpus, dim=1)` (reference src/render/nerf.py:354-371), which on EVERY
// forward call re-broadcasts the whole module (~113 MB + latents) from gpus[0], scatters the rays, runs one Python
// thread per GPU and gathers the outputs.  Here:
//   * the read-only scene state (packed weights, projected maps, cameras) is sent ONCE per change with
//     pnr_mgpu_broadcast: peer copies over NVLink / NVSwitch on per-device streams;
//   * a render call enqueues, from one host thread, per shard: a peer copy of the shard's rays (32 B/ray), ONE fused
//     render launch on that device, and the return of its pixels.  For a single object (SB = 1, every eval script) the
//     final rgb / depth are not copied at all: the kernel's compositing epilogue on GPU i stores them straight into
//     the caller's output tensor on gpus[0] through peer memory (the exchange is 16 B/ray against ~2 GFLOP/ray, so
//     the "collective" is fused away as the epilogue's store target); other outputs and SB > 1 use strided peer copies.
// Shards are torch.chunk pieces of the ray axis, so the gathered ray order equals DataParallel's.  Everything is
// asynchronous; the caller's stream on gpus[0] waits on per-shard events.  No NCCL: inside one process peer access
// is the whole transport (bench.py's one-process-per-GPU launcher uses NCCL through torch.distributed instead).
#include <stdint.h>
#include <stdlib.h>

#include <vector>

#include "pnr_mgpu.cuh"

namespace pnr {

// dst[j] += src[0][j] + ... + src[n-1][j], left to right; float4 body when every pointer is 16-byte aligned
struct SumSources {
  const float* p[PNR_MGPU_MAX_SOURCES];
};

__global__ void k_sum_into(float* dst, SumSources src, int n, int64_t count, int vec) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n4 = vec ? count / 4 : 0;
  for (int64_t v = t; v < n4; v += stride) {
    float4 a = reinterpret_cast<const float4*>(dst)[v];
    for (int k = 0; k < n; ++k) {
      const float4 b = reinterpret_cast<const float4*>(src.p[k])[v];
      a.x += b.x;
      a.y += b.y;
      a.z += b.z;
      a.w += b.w;
    }
    reinterpret_cast<float4*>(dst)[v] = a;
  }
  for (int64_t j = n4 * 4 + t; j < count; j += stride) {
    float a = dst[j];
    for (int k = 0; k < n; ++k) a += src.p[k][j];
    dst[j] = a;
  }
}

static int launch_sum_into(float* dst, const float* const* src, int n, int64_t count, cudaStream_t s) {
  if (count == 0 || n == 0) return PNR_OK;
  SumSources ss{};
  bool vec = ((uintptr_t)dst & 15) == 0;
  for (int k = 0; k < n; ++k) {
    ss.p[k] = src[k];
    vec = vec && ((uintptr_t)src[k] & 15) == 0;
  }
  const int64_t items = vec ? count / 4 : count;  // (the <= 3 floats of a float4 tail go to the first threads)
  const int threads = 256;
  int64_t blocks = (items + threads - 1) / threads;
  if (blocks < 1) blocks = 1;
  if (blocks > 132 * 8) blocks = 132 * 8;        // grid-stride beyond 8 blocks per H100 SM
  k_sum_into<<<(unsigned)blocks, threads, 0, s>>>(dst, ss, n, count, vec ? 1 : 0);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

// Pointer p (into arena a) and q (into arena b) sit at the same offset inside the first `count` floats, or are both NULL.
static bool same_offset(const void* p, const float* a, const void* q, const float* b, int64_t count) {
  if (!p || !q) return !p && !q;
  const intptr_t op = ((intptr_t)p - (intptr_t)a), oq = ((intptr_t)q - (intptr_t)b);
  return op == oq && op >= 0 && op % 4 == 0 && op / 4 < count;
}

// Every gradient buffer of the two PnrMlp sits at the same offset in its arena.
static bool same_layout(const PnrMlp* x, const float* a, const PnrMlp* y, const float* b, int64_t count) {
  if (!x || !y) return !x && !y;
  if (x->n_blocks != y->n_blocks || x->combine_layer != y->combine_layer) return false;
  bool ok = same_offset(x->lin_in_w, a, y->lin_in_w, b, count) && same_offset(x->lin_in_b, a, y->lin_in_b, b, count) &&
            same_offset(x->lin_out_w, a, y->lin_out_w, b, count) && same_offset(x->lin_out_b, a, y->lin_out_b, b, count);
  const int nb = x->n_blocks < PNR_MAX_BLOCKS ? x->n_blocks : PNR_MAX_BLOCKS;
  for (int k = 0; k < nb && ok; ++k)
    ok = same_offset(x->fc0_w[k], a, y->fc0_w[k], b, count) && same_offset(x->fc0_b[k], a, y->fc0_b[k], b, count) &&
         same_offset(x->fc1_w[k], a, y->fc1_w[k], b, count) && same_offset(x->fc1_b[k], a, y->fc1_b[k], b, count);
  for (int k = 0; k < nb && k < x->combine_layer && ok; ++k)
    ok = same_offset(x->lin_z_w[k], a, y->lin_z_w[k], b, count) && same_offset(x->lin_z_b[k], a, y->lin_z_b[k], b, count);
  return ok;
}

}  // namespace pnr

using namespace pnr;

extern "C" {

int pnr_mgpu_create(const int32_t* device_ids, int32_t n, PnrMgpu** out) {
  PNR_CHECK_ARG(device_ids && out && n >= 1 && n <= 64, "bad device list");
  DevGuard guard;
  PnrMgpu* h = new PnrMgpu();
  h->dev.assign(device_ids, device_ids + n);
  h->stream.assign(n, nullptr);
  h->done.assign(n, nullptr);
  h->peer_to_0.assign(n, 0);
  h->peer_from_0.assign(n, 0);
  for (int i = 0; i < n; ++i) {
    if (cudaSetDevice(h->dev[i]) != cudaSuccess) {
      set_error("pnr_mgpu_create: cannot select device %d", h->dev[i]);
      delete h;
      return PNR_ERR_CUDA;
    }
    if (i > 0) cudaStreamCreateWithFlags(&h->stream[i], cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&h->done[i], cudaEventDisableTiming);
    if (i > 0) {
      int can = 0;
      cudaDeviceCanAccessPeer(&can, h->dev[i], h->dev[0]);
      if (can) {
        cudaError_t e = cudaDeviceEnablePeerAccess(h->dev[0], 0);
        if (e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled) h->peer_to_0[i] = 1;
        cudaGetLastError();
      }
    }
  }
  cudaSetDevice(h->dev[0]);
  for (int i = 1; i < n; ++i) {
    int can = 0;
    cudaDeviceCanAccessPeer(&can, h->dev[0], h->dev[i]);
    if (can) {
      cudaError_t e = cudaDeviceEnablePeerAccess(h->dev[i], 0);
      if (e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled) h->peer_from_0[i] = 1;
      cudaGetLastError();
    }
  }
  cudaEventCreateWithFlags(&h->start, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&h->reduced, cudaEventDisableTiming);
  *out = h;
  return PNR_OK;
}

int pnr_mgpu_destroy(PnrMgpu* h) {
  if (!h) return PNR_OK;
  DevGuard guard;
  for (size_t i = 0; i < h->dev.size(); ++i) {
    cudaSetDevice(h->dev[i]);
    if (h->stream[i]) {
      cudaStreamSynchronize(h->stream[i]);
      cudaStreamDestroy(h->stream[i]);
    }
    if (h->done[i]) cudaEventDestroy(h->done[i]);
  }
  cudaSetDevice(h->dev[0]);
  cudaEventDestroy(h->start);
  cudaEventDestroy(h->reduced);
  delete h;
  return PNR_OK;
}

int32_t pnr_mgpu_size(const PnrMgpu* h) { return h ? (int32_t)h->dev.size() : 0; }

int32_t pnr_mgpu_peer_store(const PnrMgpu* h, int32_t i) {
  return (h && i >= 0 && i < (int32_t)h->dev.size()) ? (i == 0 ? 1 : h->peer_to_0[i]) : 0;
}

int32_t pnr_mgpu_peer_load(const PnrMgpu* h, int32_t i) {
  return (h && i >= 0 && i < (int32_t)h->dev.size()) ? (i == 0 ? 1 : h->peer_from_0[i]) : 0;
}

int pnr_mgpu_broadcast(PnrMgpu* h, const void* src, void* const* dst, size_t bytes, void* const* streams) {
  PNR_CHECK_ARG(h && src && dst, "NULL argument");
  if (bytes == 0) return PNR_OK;
  DevGuard guard;
  const int n = (int)h->dev.size();
  PNR_CUDA(cudaSetDevice(h->dev[0]));
  PNR_CUDA(cudaEventRecord(h->start, streams ? (cudaStream_t)streams[0] : (cudaStream_t)0));      // the source is ready
  for (int i = 1; i < n; ++i) {
    if (!dst[i]) continue;                                  // this device does not take part
    cudaStream_t s = (streams && streams[i]) ? (cudaStream_t)streams[i] : h->stream[i];
    PNR_CUDA(cudaSetDevice(h->dev[i]));
    PNR_CUDA(cudaStreamWaitEvent(s, h->start, 0));
    PNR_CUDA(cudaMemcpyPeerAsync(dst[i], h->dev[i], src, h->dev[0], bytes, s));
    // (renders on device i are enqueued on the same stream, so they are ordered after the copy)
  }
  return PNR_OK;
}

// strided copy of a per-ray tensor: rows = objects, row payload = rays of the shard x `width` floats
static int copy_rows(float* dst, int64_t dst_pitch_f, const float* src, int64_t src_pitch_f, int64_t width_f, int64_t rows,
                     cudaStream_t s) {
  if (!dst || !src || width_f == 0 || rows == 0) return PNR_OK;
  PNR_CUDA(cudaMemcpy2DAsync(dst, (size_t)dst_pitch_f * 4, src, (size_t)src_pitch_f * 4, (size_t)width_f * 4, (size_t)rows,
                             cudaMemcpyDefault, s));
  return PNR_OK;
}

int pnr_mgpu_render(PnrMgpu* h, const PnrShard* shards, const PnrRenderCfg* cfg, const float* rays0,
                    const PnrRenderOut* out0, int64_t B, void* stream0) {
  PNR_CHECK_ARG(h && shards && cfg && rays0 && out0, "NULL argument");
  PNR_CHECK_ARG(B >= 0, "B must be >= 0");
  DevGuard guard;
  const int n = (int)h->dev.size();
  const int SB = shards[0].scene ? shards[0].scene->SB : 0;
  PNR_CHECK_ARG(SB >= 1, "shard 0 has no scene");
  const int Kc = cfg->n_coarse, K = cfg->n_coarse + cfg->n_fine;
  const bool fine = cfg->n_fine > 0;
  const std::vector<cudaStream_t> streams = shard_streams(h, (cudaStream_t)stream0, [&](int i) { return shards[i].stream; });
  PNR_CUDA(cudaSetDevice(h->dev[0]));
  PNR_CUDA(cudaEventRecord(h->start, (cudaStream_t)stream0));
  int rc = PNR_OK;
  int used = 0;
  for (int i = 0; i < n && rc == PNR_OK; ++i) {
    int64_t a, b;
    chunk_bounds(B, n, i, &a, &b);
    const int64_t Bi = b - a;
    if (Bi <= 0) continue;
    const PnrShard& sh = shards[i];
    PNR_CHECK_ARG(sh.scene && sh.mlp_coarse && sh.noise && sh.workspace, "incomplete shard");
    PNR_CHECK_ARG(sh.scene->SB == SB, "all shards must hold the same objects");
    cudaStream_t s = streams[i];
    PNR_CUDA(cudaSetDevice(h->dev[i]));
    if (i > 0) PNR_CUDA(cudaStreamWaitEvent(s, h->start, 0));
    // rays of the shard: in place on device 0 for one object, else a (strided) peer copy into the shard's stage
    const float* rays_i = rays0 + a * 8;
    if (i > 0 || SB > 1) {
      PNR_CHECK_ARG(sh.rays_stage, "shard needs a ray staging buffer");
      if ((rc = copy_rows(sh.rays_stage, Bi * 8, rays0 + a * 8, B * 8, Bi * 8, SB, s))) break;
      rays_i = sh.rays_stage;
    }
    // outputs: final rgb / depth of a single object go straight into the caller's tensors (peer stores from the
    // kernel's epilogue); everything else is rendered locally and copied back with the object stride
    const bool direct = SB == 1 && (i == 0 || h->peer_to_0[i]);
    PnrRenderOut o = sh.stage;
    float* best_rgb0 = fine ? out0->rgb_fine : out0->rgb_coarse;
    float* best_dep0 = fine ? out0->depth_fine : out0->depth_coarse;
    if (direct) {
      if (fine) {
        if (best_rgb0) o.rgb_fine = best_rgb0 + a * 3;
        if (best_dep0) o.depth_fine = best_dep0 + a;
      } else {
        if (best_rgb0) o.rgb_coarse = best_rgb0 + a * 3;
        if (best_dep0) o.depth_coarse = best_dep0 + a;
      }
    }
    // the samples stay in the stage when it has room for them, wanted by out0 or not: the backward reads them there
    if (!out0->weights_coarse) o.weights_coarse = nullptr;
    if (!out0->weights_fine) o.weights_fine = nullptr;
    rc = pnr_render(sh.scene, sh.mlp_coarse, sh.mlp_fine, cfg, rays_i, sh.noise, &o, Bi, sh.workspace, sh.workspace_bytes, s);
    if (rc) break;
    struct Item { float* dst; const float* src; int64_t w; };
    const Item items[] = {
        {out0->rgb_coarse, o.rgb_coarse, 3}, {out0->depth_coarse, o.depth_coarse, 1},
        {out0->weights_coarse, o.weights_coarse, Kc}, {out0->z_coarse, o.z_coarse, Kc},
        {fine ? out0->rgb_fine : nullptr, o.rgb_fine, 3}, {fine ? out0->depth_fine : nullptr, o.depth_fine, 1},
        {fine ? out0->weights_fine : nullptr, o.weights_fine, K}, {fine ? out0->z_fine : nullptr, o.z_fine, K}};
    for (const Item& it : items) {
      if (!it.dst || !it.src) continue;
      if (it.src == it.dst + a * it.w) continue;   // written in place by the kernel
      if ((rc = copy_rows(it.dst + a * it.w, B * it.w, it.src, Bi * it.w, Bi * it.w, SB, s))) break;
    }
    if (rc) break;
    if (i > 0) PNR_CUDA(cudaEventRecord(h->done[i], s));
    used = i + 1;
  }
  PNR_CUDA(cudaSetDevice(h->dev[0]));
  for (int i = 1; i < used; ++i) PNR_CUDA(cudaStreamWaitEvent((cudaStream_t)stream0, h->done[i], 0));
  return rc;
}

int pnr_sum_into(float* dst, const float* const* src, int32_t n, int64_t count, void* stream) {
  PNR_CHECK_ARG(n >= 0 && n <= PNR_MGPU_MAX_SOURCES && count >= 0, "bad sizes");
  if (n == 0 || count == 0) return PNR_OK;
  PNR_CHECK_ARG(dst && src, "NULL argument");
  for (int k = 0; k < n; ++k) PNR_CHECK_ARG(src[k], "NULL source");
  return launch_sum_into(dst, src, n, count, (cudaStream_t)stream);
}

int pnr_mgpu_render_backward(PnrMgpu* h, const PnrShard* shards, const PnrShardGrad* shard_grads,
                             const PnrRenderCfg* cfg, const PnrRenderGrad* up0, const PnrMlp* grad_coarse0,
                             const PnrMlp* grad_fine0, float* d_latent0_nhwc, int64_t B, void* stream0) {
  return pnr_mgpu_render_backward_cam(h, shards, shard_grads, nullptr, cfg, up0, grad_coarse0, grad_fine0,
                                      d_latent0_nhwc, nullptr, nullptr, B, stream0);
}

// pnr_mgpu_render_backward_cam (sel = false) and pnr_mgpu_render_backward_sel (sel = true: NULL gradient structs /
// members are frozen, NULL in the same places on every shard; the arenas hold only the wanted tensors, and may be empty)
static int mgpu_render_backward(PnrMgpu* h, const PnrShard* shards, const PnrShardGrad* shard_grads,
                                const PnrShardCam* shard_cams, const PnrRenderCfg* cfg, const PnrRenderGrad* up0,
                                const PnrMlp* grad_coarse0, const PnrMlp* grad_fine0, float* d_latent0_nhwc,
                                float* d_rays0, const PnrCameraGrad* cam0, int64_t B, void* stream0, bool sel) {
  PNR_CHECK_ARG(h && shards && shard_grads && cfg && (sel || grad_coarse0), "NULL argument");
  const PnrCameraGrad c0 = cam0 ? *cam0 : PnrCameraGrad{};
  const bool want_cam = c0.d_poses || c0.d_focal || c0.d_c;
  // shard i's camera buffers: those of cam0 that are wanted, at the same arena offsets on device i
  auto shard_cam = [&](int i) {
    if (i == 0) return c0;
    PnrCameraGrad ci = shard_cams[i].cam;
    if (!c0.d_poses) ci.d_poses = nullptr;
    if (!c0.d_focal) ci.d_focal = nullptr;
    if (!c0.d_c) ci.d_c = nullptr;
    return ci;
  };
  PNR_CHECK_ARG(B >= 0, "B must be >= 0");
  PNR_CHECK_ARG(cfg->n_coarse >= 1 && cfg->n_fine >= 0, "bad sample counts");
  if (int rc = check_backward_engine(cfg->engine)) return rc;
  DevGuard guard;
  const int n = (int)h->dev.size();
  const int SB = shards[0].scene ? shards[0].scene->SB : 0;
  PNR_CHECK_ARG(SB >= 1, "shard 0 has no scene");
  const int Kc = cfg->n_coarse, K = cfg->n_coarse + cfg->n_fine;
  const bool fine = cfg->n_fine > 0;
  // the six upstream gradients of up0 and their widths; a NULL one stays NULL (zero) on every shard
  const PnrRenderGrad g0 = up0 ? *up0 : PnrRenderGrad{};
  const float* PnrRenderGrad::*const fields[6] = {&PnrRenderGrad::d_rgb_coarse, &PnrRenderGrad::d_depth_coarse,
                                                 &PnrRenderGrad::d_weights_coarse, &PnrRenderGrad::d_rgb_fine,
                                                 &PnrRenderGrad::d_depth_fine, &PnrRenderGrad::d_weights_fine};
  const int64_t widths[6] = {3, 1, Kc, 3, 1, K};
  bool any_up = false;
  for (int k = 0; k < 6; ++k) any_up = any_up || ((k < 3 || fine) && g0.*fields[k]);
  // check every shard before anything is enqueued
  const PnrShardGrad& sg0 = shard_grads[0];
  int used = 0;
  for (int i = 0; i < n; ++i) {
    int64_t a, b;
    chunk_bounds(B, n, i, &a, &b);
    if (b - a <= 0) continue;
    const PnrShard& sh = shards[i];
    const PnrShardGrad& sg = shard_grads[i];
    PNR_CHECK_ARG(sh.scene && sh.mlp_coarse && sh.noise, "incomplete shard");
    PNR_CHECK_ARG(sh.scene->SB == SB, "all shards must hold the same objects");
    PNR_CHECK_ARG(sg.rays && sg.z_coarse && sg.workspace, "incomplete shard gradient (rays, z_coarse, workspace)");
    if (any_up && (i > 0 || SB > 1)) PNR_CHECK_ARG(sg.up_stage, "shard gradient needs an upstream staging buffer");
    if (i > 0) {
      PNR_CHECK_ARG((sg0.arena && sg0.arena_count > 0) || (sel && sg0.arena_count == 0),
                    "shard gradient 0 needs device 0's gradient arena");
      PNR_CHECK_ARG((sg.arena || sg0.arena_count == 0) && sg.arena_count == sg0.arena_count,
                    "shard gradient needs an arena of device 0's size");
      if (sel)
        PNR_CHECK_ARG(!sg.grad_coarse == !grad_coarse0 && (!sh.mlp_fine || !sg.grad_fine == !grad_fine0),
                      "shard gradient structs must be NULL where device 0's are");
      else
        PNR_CHECK_ARG(sg.grad_coarse && (!sh.mlp_fine || sg.grad_fine),
                      "incomplete shard gradient (grad_coarse / grad_fine)");
      PNR_CHECK_ARG(same_layout(sg.grad_coarse, sg.arena, grad_coarse0, sg0.arena, sg0.arena_count) &&
                        same_layout(sh.mlp_fine ? sg.grad_fine : nullptr, sg.arena,
                                    sh.mlp_fine ? grad_fine0 : nullptr, sg0.arena, sg0.arena_count) &&
                        same_offset(sg.d_latent_nhwc, sg.arena, d_latent0_nhwc, sg0.arena, sg0.arena_count),
                    "shard gradient arena must have device 0's layout");
      PNR_CHECK_ARG(h->peer_from_0[i] || sg.arena_stage0 || sg0.arena_count == 0, "shard gradient needs a device-0 staging arena (no peer access)");
      if (want_cam) {
        PNR_CHECK_ARG(shard_cams, "camera gradients need the per-shard camera buffers");
        const PnrCameraGrad ci = shard_cam(i);
        PNR_CHECK_ARG(same_offset(ci.d_poses, sg.arena, c0.d_poses, sg0.arena, sg0.arena_count) &&
                          same_offset(ci.d_focal, sg.arena, c0.d_focal, sg0.arena, sg0.arena_count) &&
                          same_offset(ci.d_c, sg.arena, c0.d_c, sg0.arena, sg0.arena_count),
                      "shard camera gradients must sit in the arena at device 0's offsets");
      }
    }
    if (d_rays0 && (i > 0 || SB > 1))
      PNR_CHECK_ARG(shard_cams && shard_cams[i].d_rays, "ray gradients need a per-shard staging buffer");
    used = i + 1;
  }
  if (used == 0) return PNR_OK;
  PNR_CHECK_ARG(used - 1 <= PNR_MGPU_MAX_SOURCES, "too many shards");
  const std::vector<cudaStream_t> streams =
      shard_streams(h, (cudaStream_t)stream0, [&](int i) { return shard_grads[i].stream; });
  PNR_CUDA(cudaSetDevice(h->dev[0]));
  PNR_CUDA(cudaEventRecord(h->start, (cudaStream_t)stream0));     // up0 is ready
  for (int i = 0; i < used; ++i) {
    int64_t a, b;
    chunk_bounds(B, n, i, &a, &b);
    const int64_t Bi = b - a;
    if (Bi <= 0) continue;
    const PnrShard& sh = shards[i];
    const PnrShardGrad& sg = shard_grads[i];
    cudaStream_t s = streams[i];
    PNR_CUDA(cudaSetDevice(h->dev[i]));
    if (i > 0) PNR_CUDA(cudaStreamWaitEvent(s, h->start, 0));
    // the shard's slice of each upstream gradient: in place for shard 0 of one object, else a strided copy
    PnrRenderGrad gi{};
    float* stage = sg.up_stage;
    for (int k = 0; k < 6; ++k) {
      const float* src = (k < 3 || fine) ? g0.*fields[k] : nullptr;
      if (!src) continue;
      const int64_t w = widths[k];
      if (i == 0 && SB == 1) {
        gi.*fields[k] = src + a * w;
        continue;
      }
      int rc = copy_rows(stage, Bi * w, src + a * w, B * w, Bi * w, SB, s);
      if (rc) return rc;
      gi.*fields[k] = stage;
      stage += SB * Bi * w;
    }
    if (i > 0 && sg.arena_count > 0) PNR_CUDA(cudaMemsetAsync(sg.arena, 0, (size_t)sg.arena_count * 4, s));
    PnrRenderOut fwd{};
    fwd.z_coarse = const_cast<float*>(sg.z_coarse);
    fwd.z_fine = const_cast<float*>(sg.z_fine);
    fwd.depth_coarse = const_cast<float*>(sg.depth_coarse);
    // ray gradients: shard 0 of one object writes device 0's rows in place, the others a staging buffer
    const bool in_place = i == 0 && SB == 1;
    float* dr = d_rays0 ? (in_place ? d_rays0 : shard_cams[i].d_rays) : nullptr;
    const PnrCameraGrad ci = want_cam ? shard_cam(i) : PnrCameraGrad{};
    int rc = (sel ? pnr_render_backward_sel : pnr_render_backward_cam)(
        sh.scene, sh.mlp_coarse, sh.mlp_fine, cfg, sg.rays, sh.noise, &fwd, &gi, i == 0 ? grad_coarse0 : sg.grad_coarse,
        i == 0 ? grad_fine0 : sg.grad_fine, i == 0 ? d_latent0_nhwc : sg.d_latent_nhwc, dr, want_cam ? &ci : nullptr, Bi,
        sg.workspace, sg.workspace_bytes, s);
    if (rc) return rc;
    // the reverse of the forward's ray staging: [SB][B_i][8] -> rows [a, b) of each object in d_rays0 [SB][B][8]
    if (dr && !in_place && (rc = copy_rows(d_rays0 + a * 8, B * 8, dr, Bi * 8, Bi * 8, SB, s))) return rc;
    if (i > 0) PNR_CUDA(cudaEventRecord(h->done[i], s));
  }
  // device 0: grad0 += g_1 + ... + g_{used-1}, one launch over the arenas, shards in order
  PNR_CUDA(cudaSetDevice(h->dev[0]));
  cudaStream_t s0 = (cudaStream_t)stream0;
  std::vector<const float*> src;
  for (int i = 1; i < used; ++i) {
    int64_t a, b;
    chunk_bounds(B, n, i, &a, &b);
    if (b - a <= 0) continue;
    const PnrShardGrad& sg = shard_grads[i];
    PNR_CUDA(cudaStreamWaitEvent(s0, h->done[i], 0));
    if (sg.arena_count == 0) continue;                           // nothing in the arenas (e.g. ray gradients only)
    if (h->peer_from_0[i]) {
      src.push_back(sg.arena);                                   // read over NVLink by the reduction kernel
    } else {
      PNR_CUDA(cudaMemcpyPeerAsync(sg.arena_stage0, h->dev[0], sg.arena, h->dev[i], (size_t)sg.arena_count * 4, s0));
      src.push_back(sg.arena_stage0);
    }
  }
  if (src.empty()) return PNR_OK;
  int rc = launch_sum_into(sg0.arena, src.data(), (int)src.size(), sg0.arena_count, s0);
  if (rc) return rc;
  // later work on the shards' streams waits for the reduction, so their arenas can be released once this returns
  PNR_CUDA(cudaEventRecord(h->reduced, s0));
  for (int i = 1; i < used; ++i) {
    if (streams[i] == s0) continue;
    PNR_CUDA(cudaSetDevice(h->dev[i]));
    PNR_CUDA(cudaStreamWaitEvent(streams[i], h->reduced, 0));
  }
  return PNR_OK;
}

int pnr_mgpu_render_backward_cam(PnrMgpu* h, const PnrShard* shards, const PnrShardGrad* shard_grads,
                                 const PnrShardCam* shard_cams, const PnrRenderCfg* cfg, const PnrRenderGrad* up0,
                                 const PnrMlp* grad_coarse0, const PnrMlp* grad_fine0, float* d_latent0_nhwc,
                                 float* d_rays0, const PnrCameraGrad* cam0, int64_t B, void* stream0) {
  return mgpu_render_backward(h, shards, shard_grads, shard_cams, cfg, up0, grad_coarse0, grad_fine0, d_latent0_nhwc,
                              d_rays0, cam0, B, stream0, false);
}

int pnr_mgpu_render_backward_sel(PnrMgpu* h, const PnrShard* shards, const PnrShardGrad* shard_grads,
                                 const PnrShardCam* shard_cams, const PnrRenderCfg* cfg, const PnrRenderGrad* up0,
                                 const PnrMlp* grad_coarse0, const PnrMlp* grad_fine0, float* d_latent0_nhwc,
                                 float* d_rays0, const PnrCameraGrad* cam0, int64_t B, void* stream0) {
  return mgpu_render_backward(h, shards, shard_grads, shard_cams, cfg, up0, grad_coarse0, grad_fine0, d_latent0_nhwc,
                              d_rays0, cam0, B, stream0, true);
}

}  // extern "C"
