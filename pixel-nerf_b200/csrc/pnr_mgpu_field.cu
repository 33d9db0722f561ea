// Sharded field evaluation for mesh extraction (C ABI: pnr_mgpu_field_*, include/pnr.h): util/recon.py's field passes
// over the devices of a pnr_mgpu handle.  The point range is cut into the chunks a one-GPU loop evaluates and every
// device takes a contiguous run of whole chunks, so each point is evaluated exactly as on one GPU.  Every device
// generates its own points (grid, band lattice, band refinement set) or copies its rows of a point list from device 0
// (24 B per point); only the wanted output channels (4 or 12 B per point) travel back, stored by a small kernel straight
// into device 0's tensor through peer memory, or staged and peer-copied where the device cannot address device 0.
#include <stdint.h>

#include <vector>

#include "pnr_mgpu.cuh"

namespace pnr {

// dst[r][k] = field[r][channel + k], k < nc: the wanted channels of a chunk's field values, one thread per row
__global__ void k_store_channels(const float* field, int d_out, int channel, int nc, int64_t n, float* dst) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  for (int k = 0; k < nc; ++k) dst[r * nc + k] = field[r * d_out + channel + k];
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// A field shard's workspace: the chunk's points, view directions, field values and staged channels, then
// pnr_field_eval's own workspace.  Returns the bytes needed; with base != NULL also the pointers.
struct FieldShardWs {
  float *xyz, *viewdirs, *field, *stage;
  void* eval;
  size_t eval_bytes;
};

static size_t field_shard_carve(const PnrScene* sc, const PnrMlp* mlp, int64_t chunk, int32_t engine, void* base,
                                size_t cap, FieldShardWs* w) {
  const size_t pts = align256((size_t)chunk * 3 * 4), vals = align256((size_t)chunk * mlp->d_out * 4);
  const size_t head = 2 * pts + 2 * vals;
  const size_t eval = pnr_field_workspace_bytes(sc, mlp, chunk, engine);
  if (base) {
    const uintptr_t b = (uintptr_t)base;
    w->xyz = (float*)b;
    w->viewdirs = (float*)(b + pts);
    w->field = (float*)(b + 2 * pts);
    w->stage = (float*)(b + 2 * pts + vals);
    w->eval = (void*)(b + head);
    w->eval_bytes = cap > head ? cap - head : 0;
  }
  return head + eval;
}

// The source's points [first, first + n) into xyz / viewdirs on the current device (LIST: a peer copy of device 0's
// rows, or the rows themselves on device 0)
static int source_points(const PnrPointSource& src, const PnrFieldShard& sh, int dev, int dev0, int64_t first, int64_t n,
                         float* xyz, float* viewdirs, const float** xyz_out, const float** vd_out, cudaStream_t s) {
  *xyz_out = xyz;
  *vd_out = viewdirs;
  switch (src.kind) {
    case PNR_POINTS_GRID:
      return pnr_grid_points(src.lo, src.hi, src.reso, first, n, xyz, viewdirs, s);
    case PNR_POINTS_LATTICE:
      return pnr_band_lattice_points(src.lo, src.hi, src.reso, src.block, first, n, xyz, viewdirs, s);
    case PNR_POINTS_BAND:
      return pnr_band_points(src.lo, src.hi, src.reso, src.block, src.apron, sh.plan, sh.plan_bytes, src.n_points,
                             first, n, xyz, viewdirs, s);
    default:                                             // PNR_POINTS_LIST
      if (dev == dev0) {
        *xyz_out = src.xyz0 + first * 3;
        *vd_out = src.viewdirs0 + first * 3;
        return PNR_OK;
      }
      PNR_CUDA(cudaMemcpyPeerAsync(xyz, dev, src.xyz0 + first * 3, dev0, (size_t)n * 12, s));
      PNR_CUDA(cudaMemcpyPeerAsync(viewdirs, dev, src.viewdirs0 + first * 3, dev0, (size_t)n * 12, s));
      return PNR_OK;
  }
}

// The source is well formed for `count` points (the point entry points' own checks, run on an empty range at the end)
static int check_source(const PnrPointSource& src, int64_t count) {
  switch (src.kind) {
    case PNR_POINTS_GRID:
      return pnr_grid_points(src.lo, src.hi, src.reso, count, 0, nullptr, nullptr, nullptr);
    case PNR_POINTS_LATTICE:
      return pnr_band_lattice_points(src.lo, src.hi, src.reso, src.block, count, 0, nullptr, nullptr, nullptr);
    case PNR_POINTS_BAND:
      PNR_CHECK_ARG(src.apron == 0 || src.apron == 1, "apron must be 0 or 1");
      PNR_CHECK_ARG(src.n_points == count, "a BAND source's count must be its n_points");
      return PNR_OK;                                     // reso / block / plan: per shard, with its plan
    case PNR_POINTS_LIST:
      PNR_CHECK_ARG(count == 0 || (src.xyz0 && src.viewdirs0), "a LIST source needs xyz0 and viewdirs0");
      return PNR_OK;
    default:
      set_error("invalid argument: unknown point source kind %d", src.kind);
      return PNR_ERR_INVALID;
  }
}

}  // namespace pnr

using namespace pnr;

extern "C" {

size_t pnr_mgpu_field_workspace_bytes(const PnrScene* scene, const PnrMlp* mlp, int64_t chunk, int32_t engine) {
  if (!scene || !mlp || chunk < 1 || mlp->d_out < 1) return 0;
  return field_shard_carve(scene, mlp, chunk, engine, nullptr, 0, nullptr);
}

int pnr_mgpu_field_eval(PnrMgpu* h, const PnrFieldShard* shards, const PnrPointSource* src, int64_t count,
                        int64_t chunk, int32_t engine, int32_t channel, int32_t n_channels, float* out0,
                        void* stream0) {
  PNR_CHECK_ARG(h && shards && src, "NULL argument");
  PNR_CHECK_ARG(count >= 0, "count must be >= 0");
  PNR_CHECK_ARG(chunk >= 1, "chunk must be >= 1");
  PNR_CHECK_ARG(channel >= 0 && n_channels >= 1, "channel range outside the field's outputs");
  if (int rc = check_source(*src, count)) return rc;
  const int n = (int)h->dev.size();
  const int64_t n_chunks = (count + chunk - 1) / chunk;
  // check every shard with chunks before anything is enqueued
  int used = 0;
  for (int i = 0; i < n; ++i) {
    int64_t ca, cb;
    chunk_bounds(n_chunks, n, i, &ca, &cb);
    if (cb - ca <= 0) continue;
    const PnrFieldShard& sh = shards[i];
    PNR_CHECK_ARG(sh.scene && sh.mlp, "incomplete field shard (scene, mlp)");
    PNR_CHECK_ARG(sh.scene->SB == 1, "the sharded field evaluation takes a scene of one object");
    PNR_CHECK_ARG(channel + n_channels <= sh.mlp->d_out, "channel range outside the field's outputs");
    PNR_CHECK_ARG(out0, "NULL out0");
    if (src->kind == PNR_POINTS_BAND) {
      PNR_CHECK_ARG(sh.plan, "a BAND source needs each shard's plan");
      if (int rc = pnr_band_points(src->lo, src->hi, src->reso, src->block, src->apron, sh.plan, sh.plan_bytes,
                                   src->n_points, count, 0, nullptr, nullptr, nullptr))
        return rc;
    }
    const size_t need = field_shard_carve(sh.scene, sh.mlp, chunk, engine, nullptr, 0, nullptr);
    if (!sh.workspace || sh.workspace_bytes < need) {
      set_error("field shard %d: workspace too small: %zu < %zu", i, sh.workspace_bytes, need);
      return PNR_ERR_WORKSPACE;
    }
    used = i + 1;
  }
  if (used == 0) return PNR_OK;
  DevGuard guard;
  const std::vector<cudaStream_t> streams = shard_streams(h, (cudaStream_t)stream0, [&](int i) { return shards[i].stream; });
  const int dev0 = h->dev[0];
  PNR_CUDA(cudaSetDevice(dev0));
  PNR_CUDA(cudaEventRecord(h->start, (cudaStream_t)stream0));      // out0 (and a LIST's rows) are ready
  int rc = PNR_OK;
  int last = 0;
  for (int i = 0; i < used && rc == PNR_OK; ++i) {
    int64_t ca, cb;
    chunk_bounds(n_chunks, n, i, &ca, &cb);
    if (cb - ca <= 0) continue;
    const PnrFieldShard& sh = shards[i];
    const int dev = h->dev[i];
    cudaStream_t s = streams[i];
    PNR_CUDA(cudaSetDevice(dev));
    if (i > 0) PNR_CUDA(cudaStreamWaitEvent(s, h->start, 0));
    FieldShardWs w;
    field_shard_carve(sh.scene, sh.mlp, chunk, engine, sh.workspace, sh.workspace_bytes, &w);
    // the channels go straight into out0 where device i can store there, else through the staging slice (reused by
    // the next chunk only after its copy, which is ahead on stream s)
    const bool direct = pnr_mgpu_peer_store(h, i) != 0;
    for (int64_t c = ca; c < cb && rc == PNR_OK; ++c) {
      const int64_t first = c * chunk, m = count - first < chunk ? count - first : chunk;
      const float *xyz, *vd;
      if ((rc = source_points(*src, sh, dev, dev0, first, m, w.xyz, w.viewdirs, &xyz, &vd, s))) break;
      if ((rc = pnr_field_eval(sh.scene, sh.mlp, xyz, vd, w.field, m, engine, w.eval, w.eval_bytes, s))) break;
      float* dst = direct ? out0 + first * n_channels : w.stage;
      k_store_channels<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(w.field, sh.mlp->d_out, channel, n_channels, m, dst);
      PNR_LAUNCH_CHECK();
      if (!direct)
        PNR_CUDA(cudaMemcpyPeerAsync(out0 + first * n_channels, dev0, w.stage, dev, (size_t)m * n_channels * 4, s));
    }
    if (rc) break;
    if (i > 0) PNR_CUDA(cudaEventRecord(h->done[i], s));
    last = i + 1;
  }
  PNR_CUDA(cudaSetDevice(dev0));
  for (int i = 1; i < last; ++i) {
    int64_t ca, cb;
    chunk_bounds(n_chunks, n, i, &ca, &cb);
    if (cb - ca > 0) PNR_CUDA(cudaStreamWaitEvent((cudaStream_t)stream0, h->done[i], 0));
  }
  return rc;
}

}  // extern "C"
