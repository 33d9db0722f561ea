// Mesh extraction (src/util/recon.py of the reference, restated in oracle/pnr_recon.py): the evaluation grid of
// util.gen_grid and marching cubes over a dense sigma volume.  Everything is deterministic: vertex ids and triangle
// offsets come from exclusive scans (reduce-then-scan, no atomics), so two runs give the same bits, and the
// arithmetic uses explicit round-to-nearest intrinsics so that numpy reproduces it exactly.
#include "pnr_common.cuh"
#include "pnr_mc_tables.cuh"

namespace pnr {

constexpr int kPtThreads = 256;
constexpr int kScanThreads = 256;
constexpr int kScanItems = 16;
constexpr int64_t kScanTile = (int64_t)kScanThreads * kScanItems;
constexpr int64_t kMaxGridPoints = (int64_t)1 << 36;

// ---- grid points -------------------------------------------------------------------------------------------------
// np.linspace(lo, hi, n, dtype=float32): y_i = i * ((hi - lo) / (n - 1)) + lo in float64, the last point set to hi,
// then rounded to float32.
__device__ __forceinline__ float linspace_f32(double lo, double hi, int n, int i) {
  if (n > 1 && i == n - 1) return __double2float_rn(hi);
  if (n <= 1) return __double2float_rn(lo);
  const double step = __ddiv_rn(__dsub_rn(hi, lo), (double)(n - 1));
  return __double2float_rn(__dadd_rn(__dmul_rn((double)i, step), lo));
}

__global__ void k_grid_points(double lo0, double lo1, double lo2, double hi0, double hi1, double hi2, int nx, int ny,
                              int nz, int64_t first, int64_t count, float* __restrict__ xyz,
                              float* __restrict__ viewdirs) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  const int64_t i = first + t;
  const int iz = (int)(i % nz);
  const int64_t r = i / nz;
  const int iy = (int)(r % ny);
  const int ix = (int)(r / ny);
  const float x = linspace_f32(lo0, hi0, nx, ix), y = linspace_f32(lo1, hi1, ny, iy), z = linspace_f32(lo2, hi2, nz, iz);
  xyz[t * 3 + 0] = x;
  xyz[t * 3 + 1] = y;
  xyz[t * 3 + 2] = z;
  if (viewdirs) {
    // recon.py:54 -grid / torch.norm(grid, dim=-1): on gen_grid's transposed (non-contiguous) grid torch's CPU norm
    // sums (x*x + y*y) + z*z, one rounding per operation; 0 / 0 = NaN at the origin, as there
    const float n = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    viewdirs[t * 3 + 0] = __fdiv_rn(-x, n);
    viewdirs[t * 3 + 1] = __fdiv_rn(-y, n);
    viewdirs[t * 3 + 2] = __fdiv_rn(-z, n);
  }
}

// ---- marching cubes ------------------------------------------------------------------------------------------------
// A corner is inside when its value is finite and above iso (NaN and +-inf are outside).
__device__ __forceinline__ bool mc_inside(float v, double iso) {
  return fabsf(v) <= 3.402823466e38f && (double)v > iso;
}

// edge slots are (grid point, axis), point-major: slot = 3 * point + axis.  flags[slot] = 1 when the edge exists and
// its two corners differ in state.
__global__ void k_mc_edges(const float* __restrict__ vol, int nx, int ny, int nz, double iso,
                           uint8_t* __restrict__ flags) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t N = (int64_t)nx * ny * nz;
  if (p >= N) return;
  const int z = (int)(p % nz);
  const int y = (int)((p / nz) % ny);
  const int x = (int)(p / ((int64_t)ny * nz));
  const bool a = mc_inside(vol[p], iso);
  flags[p * 3 + 0] = x + 1 < nx && mc_inside(vol[p + (int64_t)ny * nz], iso) != a;
  flags[p * 3 + 1] = y + 1 < ny && mc_inside(vol[p + nz], iso) != a;
  flags[p * 3 + 2] = z + 1 < nz && mc_inside(vol[p + 1], iso) != a;
}

// cell = its lower corner's point index; cells on the upper faces of the grid do not exist (count 0).
__global__ void k_mc_cells(const float* __restrict__ vol, int nx, int ny, int nz, double iso,
                           uint8_t* __restrict__ cube, uint8_t* __restrict__ tcount) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t N = (int64_t)nx * ny * nz;
  if (p >= N) return;
  const int z = (int)(p % nz);
  const int y = (int)((p / nz) % ny);
  const int x = (int)(p / ((int64_t)ny * nz));
  int c = 0;
  if (x + 1 < nx && y + 1 < ny && z + 1 < nz) {
    const int64_t sx = (int64_t)ny * nz, sy = nz;
#pragma unroll
    for (int k = 0; k < 8; ++k)
      c |= (int)mc_inside(vol[p + (k & 1) * sx + ((k >> 1) & 1) * sy + ((k >> 2) & 1)], iso) << k;
  }
  cube[p] = (uint8_t)c;
  tcount[p] = (uint8_t)kMcTriCount[c];
}

// Block-wide inclusive scan of one int64 per thread (Hillis-Steele in shared memory; blockDim.x == kScanThreads).
__device__ __forceinline__ int64_t block_incl_scan(int64_t v, int64_t* buf) {
  const int t = threadIdx.x;
  buf[t] = v;
  __syncthreads();
  for (int off = 1; off < kScanThreads; off <<= 1) {
    const int64_t a = t >= off ? buf[t - off] : 0;
    __syncthreads();
    buf[t] += a;
    __syncthreads();
  }
  const int64_t r = buf[t];
  __syncthreads();
  return r;
}

// pass 1: sum of each kScanTile-element tile
__global__ void __launch_bounds__(kScanThreads) k_scan_reduce(const uint8_t* __restrict__ in, int64_t n,
                                                              int64_t* __restrict__ sums) {
  __shared__ int64_t red[kScanThreads];
  const int t = threadIdx.x;
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
  int64_t s = 0;
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t i = base + (int64_t)k * kScanThreads + t;
    if (i < n) s += in[i];
  }
  red[t] = s;
  __syncthreads();
  for (int w = kScanThreads / 2; w > 0; w >>= 1) {
    if (t < w) red[t] += red[t + w];
    __syncthreads();
  }
  if (t == 0) sums[blockIdx.x] = red[0];
}

// pass 2 (one block): exclusive scan of the tile sums in place; *total = their sum
__global__ void __launch_bounds__(kScanThreads) k_scan_tiles(int64_t* __restrict__ sums, int64_t nb,
                                                             int64_t* __restrict__ total) {
  __shared__ int64_t buf[kScanThreads];
  const int t = threadIdx.x;
  int64_t carry = 0;
  for (int64_t base = 0; base < nb; base += kScanThreads) {
    const int64_t i = base + t;
    const int64_t v = i < nb ? sums[i] : 0;
    const int64_t incl = block_incl_scan(v, buf);
    if (i < nb) sums[i] = carry + incl - v;
    // every thread adds the chunk's total (the last thread's inclusive value), passed through shared memory
    if (t == kScanThreads - 1) buf[0] = incl;
    __syncthreads();
    carry += buf[0];
    __syncthreads();
  }
  if (t == 0) *total = carry;
}

// pass 3: out[i] = exclusive prefix of in[i], from the tile offsets of pass 2
__global__ void __launch_bounds__(kScanThreads) k_scan_apply(const uint8_t* __restrict__ in, int64_t n,
                                                             const int64_t* __restrict__ tile_off,
                                                             int64_t* __restrict__ out) {
  __shared__ uint8_t tile[kScanTile];
  __shared__ int64_t buf[kScanThreads];
  const int t = threadIdx.x;
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t i = base + (int64_t)k * kScanThreads + t;
    tile[k * kScanThreads + t] = i < n ? in[i] : 0;
  }
  __syncthreads();
  int64_t s = 0;
  for (int k = 0; k < kScanItems; ++k) s += tile[t * kScanItems + k];
  int64_t run = tile_off[blockIdx.x] + block_incl_scan(s, buf) - s;
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t i = base + (int64_t)t * kScanItems + k;
    if (i < n) out[i] = run;
    run += tile[t * kScanItems + k];
  }
}

// one vertex per crossed edge, at its exclusive-scan id: lower corner + t along the axis, t in float64
__global__ void k_mc_verts(const float* __restrict__ vol, int nx, int ny, int nz, double iso,
                           const uint8_t* __restrict__ flags, const int64_t* __restrict__ vid, int64_t n_verts,
                           double* __restrict__ verts) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t N = (int64_t)nx * ny * nz;
  if (p >= N) return;
  const int z = (int)(p % nz);
  const int y = (int)((p / nz) % ny);
  const int x = (int)(p / ((int64_t)ny * nz));
  const int64_t step[3] = {(int64_t)ny * nz, (int64_t)nz, 1};
  for (int a = 0; a < 3; ++a) {
    if (!flags[p * 3 + a]) continue;
    const int64_t id = vid[p * 3 + a];
    if (id >= n_verts) continue;
    const float sa = vol[p], sb = vol[p + step[a]];
    double t = 0.5;                       // the outside corner is NaN or +-inf: the edge's midpoint
    if (fabsf(sa) <= 3.402823466e38f && fabsf(sb) <= 3.402823466e38f)
      t = __ddiv_rn(__dsub_rn(iso, (double)sa), __dsub_rn((double)sb, (double)sa));
    double c[3] = {(double)x, (double)y, (double)z};
    c[a] = __dadd_rn(c[a], t);
    verts[id * 3 + 0] = c[0];
    verts[id * 3 + 1] = c[1];
    verts[id * 3 + 2] = c[2];
  }
}

// ---- vertex attributes ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool finite_f32(float v) { return fabsf(v) <= 3.402823466e38f; }

// axis k of the sigma gradient at grid point p (index i of n along the axis), in index units: the central difference
// where both neighbours exist and are finite, else a one-sided difference with a finite centre, else 0.  A NaN (the
// grid origin, whose fake view direction is 0 / 0) or an infinity never reaches a neighbour's gradient.
__device__ __forceinline__ double grid_grad(const float* __restrict__ vol, int64_t p, int i, int n, int64_t step) {
  const bool up = i + 1 < n, dn = i > 0;
  const float c = vol[p], su = up ? vol[p + step] : 0.0f, sd = dn ? vol[p - step] : 0.0f;
  if (up && dn && finite_f32(su) && finite_f32(sd)) return __ddiv_rn(__dsub_rn((double)su, (double)sd), 2.0);
  if (up && finite_f32(c) && finite_f32(su)) return __dsub_rn((double)su, (double)c);
  if (dn && finite_f32(c) && finite_f32(sd)) return __dsub_rn((double)c, (double)sd);
  return 0.0;
}

// lo + v * h for an index coordinate v of an axis of n >= 2 points; on a grid index the bits of linspace_f32
__device__ __forceinline__ float index_to_world_f32(double lo, double hi, int n, double v) {
  const int i = (int)v;
  if ((double)i == v) return linspace_f32(lo, hi, n, i);
  const double h = __ddiv_rn(__dsub_rn(hi, lo), (double)(n - 1));
  return __double2float_rn(__dadd_rn(__dmul_rn(v, h), lo));
}

// per vertex of k_mc_verts (same edges, same ids, same t): the unit normal -G/|G| from the grid gradient interpolated
// along the edge, G in world units (toward decreasing sigma; along the edge from its inside corner to its outside
// corner where |G| is 0 or not finite), the vertex's world position, and the view direction -normal
__global__ void k_mc_vertex_attrs(const float* __restrict__ vol, int nx, int ny, int nz, double iso, double lo0,
                                  double lo1, double lo2, double hi0, double hi1, double hi2,
                                  const uint8_t* __restrict__ flags, const int64_t* __restrict__ vid, int64_t n_verts,
                                  double* __restrict__ normals, float* __restrict__ xyz,
                                  float* __restrict__ viewdirs) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t N = (int64_t)nx * ny * nz;
  if (p >= N) return;
  const int z = (int)(p % nz);
  const int y = (int)((p / nz) % ny);
  const int x = (int)(p / ((int64_t)ny * nz));
  const int64_t step[3] = {(int64_t)ny * nz, (int64_t)nz, 1};
  const int dim[3] = {nx, ny, nz};
  const double lo[3] = {lo0, lo1, lo2}, hi[3] = {hi0, hi1, hi2};
  double ga[3];
  bool have_ga = false;
  for (int a = 0; a < 3; ++a) {
    if (!flags[p * 3 + a]) continue;
    const int64_t id = vid[p * 3 + a];
    if (id >= n_verts) continue;
    const float sa = vol[p], sb = vol[p + step[a]];
    double t = 0.5;                       // as k_mc_verts computes it
    if (finite_f32(sa) && finite_f32(sb))
      t = __ddiv_rn(__dsub_rn(iso, (double)sa), __dsub_rn((double)sb, (double)sa));
    int ia[3] = {x, y, z}, ib[3] = {x, y, z};
    ib[a] += 1;
    if (!have_ga) {
      for (int k = 0; k < 3; ++k) ga[k] = grid_grad(vol, p, ia[k], dim[k], step[k]);
      have_ga = true;
    }
    double G[3], h[3];
    for (int k = 0; k < 3; ++k) {
      const double gb = grid_grad(vol, p + step[a], ib[k], dim[k], step[k]);
      h[k] = __ddiv_rn(__dsub_rn(hi[k], lo[k]), (double)(dim[k] - 1));
      G[k] = __ddiv_rn(__dadd_rn(__dmul_rn(__dsub_rn(1.0, t), ga[k]), __dmul_rn(t, gb)), h[k]);
    }
    // the double-precision sqrt is IEEE round-to-nearest on the GPU (as __dsqrt_rn) and in numpy
    const double len =
        sqrt(__dadd_rn(__dadd_rn(__dmul_rn(G[0], G[0]), __dmul_rn(G[1], G[1])), __dmul_rn(G[2], G[2])));
    double nrm[3] = {0.0, 0.0, 0.0};
    if (len > 0.0 && len <= 1.7976931348623157e308) {
      for (int k = 0; k < 3; ++k) nrm[k] = __ddiv_rn(-G[k], len);
    } else {
      nrm[a] = (mc_inside(sa, iso) != (h[a] < 0.0)) ? 1.0 : -1.0;
    }
    double v[3] = {(double)x, (double)y, (double)z};     // the vertex of k_mc_verts, in index units
    v[a] = __dadd_rn(v[a], t);
    for (int k = 0; k < 3; ++k) {
      if (normals) normals[id * 3 + k] = nrm[k];
      if (xyz) xyz[id * 3 + k] = index_to_world_f32(lo[k], hi[k], dim[k], v[k]);
      if (viewdirs) viewdirs[id * 3 + k] = __double2float_rn(-nrm[k]);
    }
  }
}

// the triangles of each cell in table order at the cell's scanned offset, as vertex ids of their edges
__global__ void k_mc_tris(int nx, int ny, int nz, const uint8_t* __restrict__ cube,
                          const int64_t* __restrict__ toff, const int64_t* __restrict__ vid, int64_t n_tris,
                          int64_t* __restrict__ tris) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t N = (int64_t)nx * ny * nz;
  if (p >= N) return;
  const int c = cube[p];
  const int cnt = kMcTriCount[c];
  if (cnt == 0) return;
  const int64_t sx = (int64_t)ny * nz, sy = nz;
  const int64_t o = toff[p];
  for (int j = 0; j < cnt; ++j) {
    if (o + j >= n_tris) return;
    for (int k = 0; k < 3; ++k) {
      const int e = kMcTris[c][j * 3 + k];
      const int q = kMcEdgeCorner[e];
      const int64_t pt = p + (q & 1) * sx + ((q >> 1) & 1) * sy + ((q >> 2) & 1);
      tris[(o + j) * 3 + k] = vid[pt * 3 + kMcEdgeAxis[e]];
    }
  }
}

// workspace: edge flags [3N] u8, vertex ids [3N] i64, cube index [N] u8, triangle counts [N] u8, triangle offsets
// [N] i64, tile sums of both scans
struct McWs {
  uint8_t* flags;
  int64_t* vid;
  uint8_t* cube;
  uint8_t* tcount;
  int64_t* toff;
  int64_t* sums_e;
  int64_t* sums_c;
};

static size_t mc_carve(int64_t N, void* base, size_t cap, McWs* w) {
  Arena a(base, cap);
  const int64_t nbe = (3 * N + kScanTile - 1) / kScanTile, nbc = (N + kScanTile - 1) / kScanTile;
  w->flags = a.take<uint8_t>(3 * N);
  w->vid = a.take<int64_t>(3 * N);
  w->cube = a.take<uint8_t>(N);
  w->tcount = a.take<uint8_t>(N);
  w->toff = a.take<int64_t>(N);
  w->sums_e = a.take<int64_t>(nbe);
  w->sums_c = a.take<int64_t>(nbc);
  return a.off;
}

static int exclusive_scan(const uint8_t* in, int64_t n, int64_t* sums, int64_t* out, int64_t* total, cudaStream_t s) {
  const int64_t nb = (n + kScanTile - 1) / kScanTile;
  k_scan_reduce<<<(unsigned)nb, kScanThreads, 0, s>>>(in, n, sums);
  PNR_LAUNCH_CHECK();
  k_scan_tiles<<<1, kScanThreads, 0, s>>>(sums, nb, total);
  PNR_LAUNCH_CHECK();
  k_scan_apply<<<(unsigned)nb, kScanThreads, 0, s>>>(in, n, sums, out);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

static int check_dims(int32_t nx, int32_t ny, int32_t nz) {
  PNR_CHECK_ARG(nx >= 1 && ny >= 1 && nz >= 1, "grid dimensions must be >= 1");
  PNR_CHECK_ARG((int64_t)nx * ny * nz <= kMaxGridPoints, "grid has more than 2^36 points");
  return PNR_OK;
}

}  // namespace pnr

using namespace pnr;

extern "C" {

int pnr_grid_points(const double* lo, const double* hi, const int32_t* reso, int64_t first, int64_t count, float* xyz,
                    float* viewdirs, void* stream) {
  PNR_CHECK_ARG(lo && hi && reso, "NULL bounds");
  int rc = check_dims(reso[0], reso[1], reso[2]);
  if (rc) return rc;
  const int64_t N = (int64_t)reso[0] * reso[1] * reso[2];
  PNR_CHECK_ARG(first >= 0 && count >= 0 && first + count <= N, "point range outside the grid");
  if (count == 0) return PNR_OK;
  PNR_CHECK_ARG(xyz != nullptr, "NULL xyz");
  k_grid_points<<<(unsigned)((count + kPtThreads - 1) / kPtThreads), kPtThreads, 0, (cudaStream_t)stream>>>(
      lo[0], lo[1], lo[2], hi[0], hi[1], hi[2], reso[0], reso[1], reso[2], first, count, xyz, viewdirs);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

size_t pnr_mc_workspace_bytes(int32_t nx, int32_t ny, int32_t nz) {
  if (nx < 2 || ny < 2 || nz < 2 || (int64_t)nx * ny * nz > kMaxGridPoints) return 0;
  McWs w;
  return mc_carve((int64_t)nx * ny * nz, nullptr, 0, &w);
}

int pnr_mc_count(const float* vol, int32_t nx, int32_t ny, int32_t nz, double iso, int64_t* counts_out,
                 void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_dims(nx, ny, nz);
  if (rc) return rc;
  PNR_CHECK_ARG(counts_out != nullptr, "NULL counts_out");
  cudaStream_t s = (cudaStream_t)stream;
  if (nx < 2 || ny < 2 || nz < 2) {                // no cells: no vertices, no triangles
    PNR_CUDA(cudaMemsetAsync(counts_out, 0, 2 * sizeof(int64_t), s));
    return PNR_OK;
  }
  PNR_CHECK_ARG(vol != nullptr, "NULL volume");
  const int64_t N = (int64_t)nx * ny * nz;
  McWs w;
  const size_t need = mc_carve(N, workspace, workspace_bytes, &w);
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("workspace too small: %zu < %zu", workspace_bytes, need);
    return PNR_ERR_WORKSPACE;
  }
  const unsigned blocks = (unsigned)((N + kPtThreads - 1) / kPtThreads);
  k_mc_edges<<<blocks, kPtThreads, 0, s>>>(vol, nx, ny, nz, iso, w.flags);
  PNR_LAUNCH_CHECK();
  k_mc_cells<<<blocks, kPtThreads, 0, s>>>(vol, nx, ny, nz, iso, w.cube, w.tcount);
  PNR_LAUNCH_CHECK();
  rc = exclusive_scan(w.flags, 3 * N, w.sums_e, w.vid, counts_out, s);
  if (rc) return rc;
  return exclusive_scan(w.tcount, N, w.sums_c, w.toff, counts_out + 1, s);
}

int pnr_mc_emit(const float* vol, int32_t nx, int32_t ny, int32_t nz, double iso, double* verts, int64_t* tris,
                int64_t n_verts, int64_t n_tris, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_dims(nx, ny, nz);
  if (rc) return rc;
  PNR_CHECK_ARG(n_verts >= 0 && n_tris >= 0, "negative output sizes");
  if (nx < 2 || ny < 2 || nz < 2) return PNR_OK;
  PNR_CHECK_ARG(vol != nullptr, "NULL volume");
  PNR_CHECK_ARG(verts != nullptr || n_verts == 0, "NULL verts");
  PNR_CHECK_ARG(tris != nullptr || n_tris == 0, "NULL tris");
  const int64_t N = (int64_t)nx * ny * nz;
  McWs w;
  const size_t need = mc_carve(N, workspace, workspace_bytes, &w);
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("workspace too small: %zu < %zu", workspace_bytes, need);
    return PNR_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)((N + kPtThreads - 1) / kPtThreads);
  if (n_verts > 0) {
    k_mc_verts<<<blocks, kPtThreads, 0, s>>>(vol, nx, ny, nz, iso, w.flags, w.vid, n_verts, verts);
    PNR_LAUNCH_CHECK();
  }
  if (n_tris > 0) {
    k_mc_tris<<<blocks, kPtThreads, 0, s>>>(nx, ny, nz, w.cube, w.toff, w.vid, n_tris, tris);
    PNR_LAUNCH_CHECK();
  }
  return PNR_OK;
}

int pnr_mc_vertex_attrs(const float* vol, int32_t nx, int32_t ny, int32_t nz, double iso, const double* lo,
                        const double* hi, double* normals, float* xyz, float* viewdirs, int64_t n_verts,
                        void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_dims(nx, ny, nz);
  if (rc) return rc;
  PNR_CHECK_ARG(n_verts >= 0, "negative n_verts");
  PNR_CHECK_ARG(lo && hi, "NULL bounds");
  if (nx < 2 || ny < 2 || nz < 2) return PNR_OK;
  PNR_CHECK_ARG(vol != nullptr, "NULL volume");
  const int64_t N = (int64_t)nx * ny * nz;
  McWs w;
  const size_t need = mc_carve(N, workspace, workspace_bytes, &w);
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("workspace too small: %zu < %zu", workspace_bytes, need);
    return PNR_ERR_WORKSPACE;
  }
  if (n_verts == 0 || (!normals && !xyz && !viewdirs)) return PNR_OK;
  k_mc_vertex_attrs<<<(unsigned)((N + kPtThreads - 1) / kPtThreads), kPtThreads, 0, (cudaStream_t)stream>>>(
      vol, nx, ny, nz, iso, lo[0], lo[1], lo[2], hi[0], hi[1], hi[2], w.flags, w.vid, n_verts, normals, xyz, viewdirs);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

}  // extern "C"
