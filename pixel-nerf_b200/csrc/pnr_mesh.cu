// Connected components of a triangle mesh (include/pnr.h pnr_mesh_components, pnr_mesh_compact_count / _emit;
// util/recon.py keep_components), restated in oracle/pnr_recon_components.py.  The labelling is the one place in mesh
// extraction with atomics: integer ones only, whose result does not depend on the order they land in, so two runs give
// the same bits.  The compaction numbers the kept vertices and triangles with the exclusive scan of pnr_recon.cu.
#include "pnr_common.cuh"

namespace pnr {

namespace {
constexpr int kPtThreads = 256;
unsigned grid_for(int64_t n) { return (unsigned)((n + kPtThreads - 1) / kPtThreads); }
}  // namespace

// Lock-free union-find in the style of ECL-CC over the parent array `par` (the label output).  Invariant: par[v] <= v,
// and every write stores an ancestor of v: hooking (atomicCAS) only replaces a root r by a smaller root, and path
// halving only stores a grandparent.  So a root is the minimum of its tree, and once every edge has been united the
// roots are the components' minima whatever order the threads ran in.  Integer atomics give one result for any order,
// which is the property the rest of this file keeps by avoiding atomics on floats.
typedef unsigned long long ull;

// par[x], never served stale from L1: other threads rewrite it
__device__ __forceinline__ int64_t ld_parent(const int64_t* par, int64_t x) {
  return *((const volatile int64_t*)par + x);
}

__device__ __forceinline__ int64_t cc_find(int64_t* par, int64_t x) {
  int64_t cur = ld_parent(par, x);
  if (cur == x) return x;
  int64_t prev = x, next;
  while (cur > (next = ld_parent(par, cur))) {          // path halving: prev skips to its grandparent
    *((volatile int64_t*)par + prev) = next;
    prev = cur;
    cur = next;
  }
  return cur;
}

__device__ __forceinline__ void cc_unite(int64_t* par, int64_t a, int64_t b) {
  int64_t ra = cc_find(par, a), rb = cc_find(par, b);
  while (ra != rb) {
    const int64_t lo = ra < rb ? ra : rb, hi = ra < rb ? rb : ra;
    const int64_t old = (int64_t)atomicCAS((ull*)(par + hi), (ull)hi, (ull)lo);
    if (old == hi) return;                               // hooked: hi's tree is now under lo
    // hi stopped being a root; its new parent is smaller, so carry on from that root
    ra = cc_find(par, old);
    rb = lo;
  }
}

__device__ __forceinline__ bool tri_ids_ok(const int64_t* __restrict__ tris, int64_t t, int64_t n_verts) {
  const int64_t a = tris[3 * t], b = tris[3 * t + 1], c = tris[3 * t + 2];
  return a >= 0 && a < n_verts && b >= 0 && b < n_verts && c >= 0 && c < n_verts;
}

__global__ void k_cc_init(int64_t n_verts, int64_t* __restrict__ label, int64_t* __restrict__ tri_count) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_verts) return;
  label[v] = v;
  tri_count[v] = 0;
}

// one thread per triangle: unite (a, b) and (a, c); an id out of range raises status[0] and unites nothing
__global__ void k_cc_hook(const int64_t* __restrict__ tris, int64_t n_tris, int64_t n_verts, int64_t* label,
                          int64_t* __restrict__ status) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tris) return;
  if (!tri_ids_ok(tris, t, n_verts)) {
    status[0] = 1;
    return;
  }
  const int64_t a = tris[3 * t];
  cc_unite(label, a, tris[3 * t + 1]);
  cc_unite(label, a, tris[3 * t + 2]);
}

// full path compression: label[v] = v's root.  A concurrent reader sees v's old parent or its root, both ancestors.
__global__ void k_cc_compress(int64_t n_verts, int64_t* label) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_verts) return;
  int64_t r = ld_parent(label, v);
  if (r == v) return;
  for (int64_t p; (p = ld_parent(label, r)) != r;) r = p;
  label[v] = r;
}

// triangles per root; status[1] = the roots that got their first triangle
__global__ void k_cc_count(const int64_t* __restrict__ tris, int64_t n_tris, int64_t n_verts,
                           const int64_t* __restrict__ label, int64_t* __restrict__ tri_count,
                           int64_t* __restrict__ status) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tris || !tri_ids_ok(tris, t, n_verts)) return;
  if (atomicAdd((ull*)(tri_count + label[tris[3 * t]]), 1ull) == 0ull) atomicAdd((ull*)(status + 1), 1ull);
}

__global__ void k_cc_flag_verts(int64_t n_verts, const int64_t* __restrict__ label,
                                const uint8_t* __restrict__ keep_root, uint8_t* __restrict__ vflag) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_verts) return;
  vflag[v] = keep_root[label[v]] != 0;
}

__global__ void k_cc_flag_tris(const int64_t* __restrict__ tris, int64_t n_tris, int64_t n_verts,
                               const int64_t* __restrict__ label, const uint8_t* __restrict__ keep_root,
                               uint8_t* __restrict__ tflag) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tris) return;
  tflag[t] = tri_ids_ok(tris, t, n_verts) && keep_root[label[tris[3 * t]]] != 0;
}

__global__ void k_cc_emit_verts(int64_t n_verts, const uint8_t* __restrict__ vflag, const int64_t* __restrict__ vnew,
                                int64_t n_keep, int64_t* __restrict__ vert_ids) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_verts || !vflag[v] || vnew[v] >= n_keep) return;
  vert_ids[vnew[v]] = v;
}

__global__ void k_cc_emit_tris(const int64_t* __restrict__ tris, int64_t n_tris, const uint8_t* __restrict__ tflag,
                               const int64_t* __restrict__ tnew, const int64_t* __restrict__ vnew, int64_t n_keep,
                               int64_t* __restrict__ tris_out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tris || !tflag[t]) return;
  const int64_t o = tnew[t];
  if (o >= n_keep) return;
  for (int k = 0; k < 3; ++k) tris_out[3 * o + k] = vnew[tris[3 * t + k]];
}

// workspace: status [2] i64 (bad id, components), vertex flags [N] u8, triangle flags [M] u8, new vertex ids [N] i64,
// new triangle ids [M] i64, tile sums of both scans
struct MeshWs {
  int64_t* status;
  uint8_t* vflag;
  uint8_t* tflag;
  int64_t* vnew;
  int64_t* tnew;
  int64_t* sums_v;
  int64_t* sums_t;
};

static size_t mesh_carve(int64_t N, int64_t M, void* base, size_t cap, MeshWs* w) {
  Arena a(base, cap);
  w->status = a.take<int64_t>(2);
  w->vflag = a.take<uint8_t>(N);
  w->tflag = a.take<uint8_t>(M);
  w->vnew = a.take<int64_t>(N);
  w->tnew = a.take<int64_t>(M);
  w->sums_v = a.take<int64_t>(scan_tile_count(N));
  w->sums_t = a.take<int64_t>(scan_tile_count(M));
  return a.off;
}

static int mesh_setup(const int64_t* tris, int64_t n_tris, int64_t n_verts, void* workspace, size_t workspace_bytes,
                      MeshWs* w) {
  PNR_CHECK_ARG(n_verts >= 0 && n_tris >= 0, "negative n_verts or n_tris");
  PNR_CHECK_ARG(tris != nullptr || n_tris == 0, "NULL tris");
  const size_t need = mesh_carve(n_verts, n_tris, workspace, workspace_bytes, w);
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("workspace too small: %zu < %zu", workspace_bytes, need);
    return PNR_ERR_WORKSPACE;
  }
  return PNR_OK;
}

}  // namespace pnr

using namespace pnr;

extern "C" {

size_t pnr_mesh_workspace_bytes(int64_t n_verts, int64_t n_tris) {
  if (n_verts < 0 || n_tris < 0) return 0;
  MeshWs w;
  return mesh_carve(n_verts, n_tris, nullptr, 0, &w);
}

int pnr_mesh_components(const int64_t* tris, int64_t n_tris, int64_t n_verts, int64_t* label, int64_t* tri_count,
                        int64_t* counts_out, void* workspace, size_t workspace_bytes, void* stream) {
  MeshWs w;
  int rc = mesh_setup(tris, n_tris, n_verts, workspace, workspace_bytes, &w);
  if (rc) return rc;
  PNR_CHECK_ARG(counts_out != nullptr, "NULL counts_out");
  PNR_CHECK_ARG((label != nullptr && tri_count != nullptr) || n_verts == 0, "NULL label or tri_count");
  cudaStream_t s = (cudaStream_t)stream;
  PNR_CUDA(cudaMemsetAsync(w.status, 0, 2 * sizeof(int64_t), s));
  if (n_verts > 0) {
    k_cc_init<<<grid_for(n_verts), kPtThreads, 0, s>>>(n_verts, label, tri_count);
    PNR_LAUNCH_CHECK();
  }
  if (n_tris > 0) {
    k_cc_hook<<<grid_for(n_tris), kPtThreads, 0, s>>>(tris, n_tris, n_verts, label, w.status);
    PNR_LAUNCH_CHECK();
  }
  if (n_tris > 0 && n_verts > 0) {
    k_cc_compress<<<grid_for(n_verts), kPtThreads, 0, s>>>(n_verts, label);
    PNR_LAUNCH_CHECK();
    k_cc_count<<<grid_for(n_tris), kPtThreads, 0, s>>>(tris, n_tris, n_verts, label, tri_count, w.status);
    PNR_LAUNCH_CHECK();
  }
  int64_t st[2];
  PNR_CUDA(cudaMemcpyAsync(st, w.status, sizeof(st), (cudaMemcpyKind)cudaMemcpyDefault, s));   // (unified addressing)
  PNR_CUDA(cudaStreamSynchronize(s));
  PNR_CHECK_ARG(st[0] == 0, "a triangle's vertex id is outside [0, n_verts)");
  *counts_out = st[1];
  return PNR_OK;
}

int pnr_mesh_compact_count(const int64_t* tris, int64_t n_tris, int64_t n_verts, const int64_t* label,
                           const uint8_t* keep_root, int64_t* counts_out, void* workspace, size_t workspace_bytes,
                           void* stream) {
  MeshWs w;
  int rc = mesh_setup(tris, n_tris, n_verts, workspace, workspace_bytes, &w);
  if (rc) return rc;
  PNR_CHECK_ARG(counts_out != nullptr, "NULL counts_out");
  PNR_CHECK_ARG((label != nullptr && keep_root != nullptr) || n_verts == 0, "NULL label or keep_root");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_verts == 0) {                              // no vertex: any triangle's ids are out of range, none is kept
    PNR_CUDA(cudaMemsetAsync(counts_out, 0, 2 * sizeof(int64_t), s));
    if (n_tris > 0) PNR_CUDA(cudaMemsetAsync(w.tflag, 0, (size_t)n_tris, s));
    return PNR_OK;
  }
  k_cc_flag_verts<<<grid_for(n_verts), kPtThreads, 0, s>>>(n_verts, label, keep_root, w.vflag);
  PNR_LAUNCH_CHECK();
  rc = exclusive_scan(w.vflag, n_verts, w.sums_v, w.vnew, counts_out, s);
  if (rc) return rc;
  if (n_tris == 0) {
    PNR_CUDA(cudaMemsetAsync(counts_out + 1, 0, sizeof(int64_t), s));
    return PNR_OK;
  }
  k_cc_flag_tris<<<grid_for(n_tris), kPtThreads, 0, s>>>(tris, n_tris, n_verts, label, keep_root, w.tflag);
  PNR_LAUNCH_CHECK();
  return exclusive_scan(w.tflag, n_tris, w.sums_t, w.tnew, counts_out + 1, s);
}

int pnr_mesh_compact_emit(const int64_t* tris, int64_t n_tris, int64_t n_verts, int64_t* vert_ids, int64_t* tris_out,
                          int64_t n_keep_verts, int64_t n_keep_tris, void* workspace, size_t workspace_bytes,
                          void* stream) {
  MeshWs w;
  int rc = mesh_setup(tris, n_tris, n_verts, workspace, workspace_bytes, &w);
  if (rc) return rc;
  PNR_CHECK_ARG(n_keep_verts >= 0 && n_keep_tris >= 0, "negative output sizes");
  PNR_CHECK_ARG(vert_ids != nullptr || n_keep_verts == 0, "NULL vert_ids");
  PNR_CHECK_ARG(tris_out != nullptr || n_keep_tris == 0, "NULL tris_out");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_keep_verts > 0 && n_verts > 0) {
    k_cc_emit_verts<<<grid_for(n_verts), kPtThreads, 0, s>>>(n_verts, w.vflag, w.vnew, n_keep_verts, vert_ids);
    PNR_LAUNCH_CHECK();
  }
  if (n_keep_tris > 0 && n_tris > 0) {
    k_cc_emit_tris<<<grid_for(n_tris), kPtThreads, 0, s>>>(tris, n_tris, w.tflag, w.tnew, w.vnew, n_keep_tris,
                                                           tris_out);
    PNR_LAUNCH_CHECK();
  }
  return PNR_OK;
}

}  // extern "C"
