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

// grid point (ix, iy, iz) into row t of xyz (and of viewdirs when it is not NULL)
__device__ __forceinline__ void put_grid_point(double lo0, double lo1, double lo2, double hi0, double hi1, double hi2,
                                               int nx, int ny, int nz, int ix, int iy, int iz, int64_t t,
                                               float* __restrict__ xyz, float* __restrict__ viewdirs) {
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
  put_grid_point(lo0, lo1, lo2, hi0, hi1, hi2, nx, ny, nz, ix, iy, iz, t, xyz, viewdirs);
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

// where the isosurface crosses an edge whose corners differ in state, as a fraction of the edge from its lower corner
// (0.5 when the outside corner is NaN or +-inf: the edge's midpoint)
__device__ __forceinline__ double edge_t(float sa, float sb, double iso) {
  if (fabsf(sa) <= 3.402823466e38f && fabsf(sb) <= 3.402823466e38f)
    return __ddiv_rn(__dsub_rn(iso, (double)sa), __dsub_rn((double)sb, (double)sa));
  return 0.5;
}

// vertex id of the edge (x, y, z) + t along axis a, in index units
__device__ __forceinline__ void put_vertex(int x, int y, int z, int a, double t, int64_t id, double* __restrict__ verts) {
  double c[3] = {(double)x, (double)y, (double)z};
  c[a] = __dadd_rn(c[a], t);
  verts[id * 3 + 0] = c[0];
  verts[id * 3 + 1] = c[1];
  verts[id * 3 + 2] = c[2];
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
    put_vertex(x, y, z, a, edge_t(vol[p], vol[p + step[a]], iso), id, verts);
  }
}

// ---- vertex attributes ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool finite_f32(float v) { return fabsf(v) <= 3.402823466e38f; }

// axis k of the sigma gradient at grid point p (index i of n along the axis), in index units: the central difference
// where both neighbours exist and are finite, else a one-sided difference with a finite centre, else 0.  A NaN (the
// grid origin, whose fake view direction is 0 / 0) or an infinity never reaches a neighbour's gradient.
// (c: sigma at the point, su / sd: at its upper / lower neighbour, up / dn: whether that neighbour exists)
__device__ __forceinline__ double grad_of(float c, float su, float sd, bool up, bool dn) {
  if (up && dn && finite_f32(su) && finite_f32(sd)) return __ddiv_rn(__dsub_rn((double)su, (double)sd), 2.0);
  if (up && finite_f32(c) && finite_f32(su)) return __dsub_rn((double)su, (double)c);
  if (dn && finite_f32(c) && finite_f32(sd)) return __dsub_rn((double)c, (double)sd);
  return 0.0;
}

__device__ __forceinline__ double grid_grad(const float* __restrict__ vol, int64_t p, int i, int n, int64_t step) {
  const bool up = i + 1 < n, dn = i > 0;
  return grad_of(vol[p], up ? vol[p + step] : 0.0f, dn ? vol[p - step] : 0.0f, up, dn);
}

// lo + v * h for an index coordinate v of an axis of n >= 2 points; on a grid index the bits of linspace_f32
__device__ __forceinline__ float index_to_world_f32(double lo, double hi, int n, double v) {
  const int i = (int)v;
  if ((double)i == v) return linspace_f32(lo, hi, n, i);
  const double h = __ddiv_rn(__dsub_rn(hi, lo), (double)(n - 1));
  return __double2float_rn(__dadd_rn(__dmul_rn(v, h), lo));
}

// the attributes of the vertex on edge (c, axis a) at t, whose lower corner is inside when a_in, from the grid gradients
// ga, gb at the edge's corners, into row id of each non-NULL output
__device__ __forceinline__ void put_vertex_attrs(const int c[3], int a, double t, bool a_in, const double ga[3],
                                                 const double gb[3], const int dim[3], const double lo[3],
                                                 const double hi[3], int64_t id, double* __restrict__ normals,
                                                 float* __restrict__ xyz, float* __restrict__ viewdirs) {
  double G[3], h[3];
  for (int k = 0; k < 3; ++k) {
    h[k] = __ddiv_rn(__dsub_rn(hi[k], lo[k]), (double)(dim[k] - 1));
    G[k] = __ddiv_rn(__dadd_rn(__dmul_rn(__dsub_rn(1.0, t), ga[k]), __dmul_rn(t, gb[k])), h[k]);
  }
  // the double-precision sqrt is IEEE round-to-nearest on the GPU (as __dsqrt_rn) and in numpy
  const double len =
      sqrt(__dadd_rn(__dadd_rn(__dmul_rn(G[0], G[0]), __dmul_rn(G[1], G[1])), __dmul_rn(G[2], G[2])));
  double nrm[3] = {0.0, 0.0, 0.0};
  if (len > 0.0 && len <= 1.7976931348623157e308) {
    for (int k = 0; k < 3; ++k) nrm[k] = __ddiv_rn(-G[k], len);
  } else {
    nrm[a] = (a_in != (h[a] < 0.0)) ? 1.0 : -1.0;
  }
  double v[3] = {(double)c[0], (double)c[1], (double)c[2]};     // the vertex of put_vertex, in index units
  v[a] = __dadd_rn(v[a], t);
  for (int k = 0; k < 3; ++k) {
    if (normals) normals[id * 3 + k] = nrm[k];
    if (xyz) xyz[id * 3 + k] = index_to_world_f32(lo[k], hi[k], dim[k], v[k]);
    if (viewdirs) viewdirs[id * 3 + k] = __double2float_rn(-nrm[k]);
  }
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
  const int ia[3] = {x, y, z};
  double ga[3];
  bool have_ga = false;
  for (int a = 0; a < 3; ++a) {
    if (!flags[p * 3 + a]) continue;
    const int64_t id = vid[p * 3 + a];
    if (id >= n_verts) continue;
    const float sa = vol[p];
    const double t = edge_t(sa, vol[p + step[a]], iso);   // as k_mc_verts computes it
    int ib[3] = {x, y, z};
    ib[a] += 1;
    if (!have_ga) {
      for (int k = 0; k < 3; ++k) ga[k] = grid_grad(vol, p, ia[k], dim[k], step[k]);
      have_ga = true;
    }
    double gb[3];
    for (int k = 0; k < 3; ++k) gb[k] = grid_grad(vol, p + step[a], ib[k], dim[k], step[k]);
    put_vertex_attrs(ia, a, t, mc_inside(sa, iso), ga, gb, dim, lo, hi, id, normals, xyz, viewdirs);
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

int64_t scan_tile_count(int64_t n) { return (n + kScanTile - 1) / kScanTile; }

int exclusive_scan(const uint8_t* in, int64_t n, int64_t* sums, int64_t* out, int64_t* total, cudaStream_t s) {
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


// ---- narrow band ---------------------------------------------------------------------------------------------------
// Blocks of b cells per side; block i of an axis covers the cells [i b, min((i + 1) b, n - 1)), nb = ceil((n - 1) / b)
// of them.  The coarse lattice is the grid indices min(j b, n - 1), j = 0 .. nb, so block i's corners are lattice
// points i and i + 1.  A block is seeded when its 8 corners differ in state and active when it or one of its 26
// neighbours is seeded.  The refinement set is the grid points of the active blocks' closed cells, widened by an
// apron of a = 0 or 1 points per side: point x of an axis is covered by the blocks C with C b - a <= x <=
// min((C + 1) b, n - 1) + a, a range [lo(x), hi(x)], and a grid point is refined when some active block covers it on
// all three axes.  Consecutive points with the same range form a run (2 or 3 per block), so the set is a union of
// run boxes, each whole or absent.  It is stored in grid (x, y, z) order, so that scans over it run in the global
// edge-slot and cell order of the dense extraction.
constexpr int kMaxBandBlock = 256;
constexpr int64_t kBandMagic = 0x706e7262616e6431;   // "pnrband1"

struct BandGeom {
  int n[3], b, a, nb[3], R[3];                 // R: runs per axis
};

// the plan, carved from one buffer:
//   hdr      magic, reso, block, apron, refinement points: what pnr_band_plan made, checked by the later calls
//   seeded / active flags per block
//   per axis: rof[x] the run of grid index x, rstart[r] (r <= R) the first index of run r, rlo / rhi[r] its blocks
//   the offsets that locate a refined point, (X, Y, Z) its runs:
//     index(x, y, z) = xoff[X] + (x - rstart[X]) plane[X] + yoff[X][Y] + (y - rstart[Y]) rowpts[X][Y] + zoff[X][Y][Z]
//                      + (z - rstart[Z])
//   plane[X] points per x plane of run slab X, rowpts[X][Y] per z row of run row (X, Y), and zoff / yoff / xoff running
//   sums of the refined widths along z, y and x.
struct BandPlan {
  int64_t* hdr;
  uint8_t* seeded;
  uint8_t* active;
  int32_t* rof[3];
  int32_t* rstart[3];
  int32_t* rlo[3];
  int32_t* rhi[3];
  int32_t* zoff;
  int64_t* rowpts;
  int64_t* yoff;
  int64_t* plane;
  int64_t* xoff;
  int64_t* sums;
};
constexpr int kBandHdr = 8;

// the blocks [lo, hi] covering grid index x of an axis with nb >= 1 blocks, apron a
__host__ __device__ __forceinline__ void axis_cover(int x, int b, int a, int nb, int* lo, int* hi) {
  const int v = x - a;                                   // C >= ceil((x - a) / b) - 1
  *lo = max(0, (v <= 0 ? 0 : (v + b - 1) / b) - 1);
  *hi = min(nb - 1, (x + a) / b);                        // C <= floor((x + a) / b)
}

static int count_runs(int n, int b, int a, int nb) {
  if (nb == 0) return 0;
  int runs = 0, plo = -1, phi = -1;
  for (int x = 0; x < n; ++x) {
    int lo, hi;
    axis_cover(x, b, a, nb, &lo, &hi);
    if (lo != plo || hi != phi) ++runs;
    plo = lo;
    phi = hi;
  }
  return runs;
}

static BandGeom band_geom(const int32_t* reso, int b, int a) {
  BandGeom g;
  g.b = b;
  g.a = a;
  for (int k = 0; k < 3; ++k) {
    g.n[k] = reso[k];
    g.nb[k] = (reso[k] - 1 + b - 1) / b;
  }
  const bool cells = g.nb[0] > 0 && g.nb[1] > 0 && g.nb[2] > 0;
  for (int k = 0; k < 3; ++k) g.R[k] = cells ? count_runs(g.n[k], b, a, g.nb[k]) : 0;
  return g;
}

__host__ __device__ __forceinline__ int64_t band_blocks(const BandGeom& g) {
  return (int64_t)g.nb[0] * g.nb[1] * g.nb[2];
}
static int64_t band_lattice(const BandGeom& g) { return (int64_t)(g.nb[0] + 1) * (g.nb[1] + 1) * (g.nb[2] + 1); }

static size_t band_carve(const BandGeom& g, void* base, size_t cap, BandPlan* p) {
  Arena a(base, cap);
  const int64_t NB = band_blocks(g), NR = (int64_t)g.R[0] * g.R[1];
  p->hdr = a.take<int64_t>(kBandHdr);
  p->seeded = a.take<uint8_t>(NB);
  p->active = a.take<uint8_t>(NB);
  for (int k = 0; k < 3; ++k) {
    p->rof[k] = a.take<int32_t>(g.R[k] ? g.n[k] : 0);
    p->rstart[k] = a.take<int32_t>(g.R[k] + 1);
    p->rlo[k] = a.take<int32_t>(g.R[k]);
    p->rhi[k] = a.take<int32_t>(g.R[k]);
  }
  p->zoff = a.take<int32_t>(NR * g.R[2]);
  p->rowpts = a.take<int64_t>(NR);
  p->yoff = a.take<int64_t>(NR);
  p->plane = a.take<int64_t>(g.R[0]);
  p->xoff = a.take<int64_t>(g.R[0] + 1);
  p->sums = a.take<int64_t>((NB + kScanTile - 1) / kScanTile);
  return a.off;
}

__device__ __forceinline__ int run_width(const BandPlan& p, int k, int r) { return p.rstart[k][r + 1] - p.rstart[k][r]; }

__device__ __forceinline__ int64_t band_index(const BandGeom& g, const BandPlan& p, int x, int y, int z) {
  const int X = p.rof[0][x], Y = p.rof[1][y], Z = p.rof[2][z];
  const int64_t xy = (int64_t)X * g.R[1] + Y;
  return p.xoff[X] + (int64_t)(x - p.rstart[0][X]) * p.plane[X] + p.yoff[xy] +
         (int64_t)(y - p.rstart[1][Y]) * p.rowpts[xy] + p.zoff[xy * g.R[2] + Z] + (z - p.rstart[2][Z]);
}

// the largest i < n with a[i] <= v (a non-decreasing, a[0] <= v)
template <typename T>
__device__ __forceinline__ int last_le(const T* __restrict__ a, int n, int64_t v) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if ((int64_t)a[mid] <= v) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// grid point of refinement index s < the refinement points (band_index's inverse); the run found is never empty,
// since the next one starts after s
__device__ __forceinline__ void band_point(const BandGeom& g, const BandPlan& p, int64_t s, int c[3]) {
  const int X = last_le(p.xoff, g.R[0], s);
  int64_t r = s - p.xoff[X];
  c[0] = p.rstart[0][X] + (int)(r / p.plane[X]);
  r %= p.plane[X];
  const int64_t* yo = p.yoff + (int64_t)X * g.R[1];
  const int Y = last_le(yo, g.R[1], r);
  r -= yo[Y];
  const int64_t xy = (int64_t)X * g.R[1] + Y;
  c[1] = p.rstart[1][Y] + (int)(r / p.rowpts[xy]);
  r %= p.rowpts[xy];
  const int32_t* zo = p.zoff + xy * g.R[2];
  const int Z = last_le(zo, g.R[2], r);
  c[2] = p.rstart[2][Z] + (int)(r - zo[Z]);
}

__device__ __forceinline__ int64_t block_id(const BandGeom& g, int i, int j, int k) {
  return ((int64_t)i * g.nb[1] + j) * g.nb[2] + k;
}

__global__ void k_band_lattice(double lo0, double lo1, double lo2, double hi0, double hi1, double hi2, BandGeom g,
                               int64_t first, int64_t count, float* __restrict__ xyz, float* __restrict__ viewdirs) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  const int64_t i = first + t;
  const int m1 = g.nb[1] + 1, m2 = g.nb[2] + 1;
  const int jz = (int)(i % m2), jy = (int)((i / m2) % m1), jx = (int)(i / ((int64_t)m1 * m2));
  put_grid_point(lo0, lo1, lo2, hi0, hi1, hi2, g.n[0], g.n[1], g.n[2], min(jx * g.b, g.n[0] - 1),
                 min(jy * g.b, g.n[1] - 1), min(jz * g.b, g.n[2] - 1), t, xyz, viewdirs);
}

// seeded[block] from the coarse sigma [nb0 + 1][nb1 + 1][nb2 + 1] at its 8 corners
__global__ void k_band_seed(const float* __restrict__ coarse, BandGeom g, double iso, uint8_t* __restrict__ seeded) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= band_blocks(g)) return;
  const int k = (int)(t % g.nb[2]), j = (int)((t / g.nb[2]) % g.nb[1]), i = (int)(t / ((int64_t)g.nb[1] * g.nb[2]));
  const int64_t sx = (int64_t)(g.nb[1] + 1) * (g.nb[2] + 1), sy = g.nb[2] + 1;
  const int64_t c0 = i * sx + j * sy + k;
  const bool first = mc_inside(coarse[c0], iso);
  bool mixed = false;
  for (int q = 1; q < 8; ++q)
    mixed |= mc_inside(coarse[c0 + (q & 1) * sx + ((q >> 1) & 1) * sy + ((q >> 2) & 1)], iso) != first;
  seeded[t] = mixed;
}

__global__ void k_band_dilate(const uint8_t* __restrict__ seeded, BandGeom g, uint8_t* __restrict__ active) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= band_blocks(g)) return;
  const int k = (int)(t % g.nb[2]), j = (int)((t / g.nb[2]) % g.nb[1]), i = (int)(t / ((int64_t)g.nb[1] * g.nb[2]));
  bool on = false;
  for (int a = max(i - 1, 0); a <= min(i + 1, g.nb[0] - 1); ++a)
    for (int b = max(j - 1, 0); b <= min(j + 1, g.nb[1] - 1); ++b)
      for (int c = max(k - 1, 0); c <= min(k + 1, g.nb[2] - 1); ++c) on |= seeded[block_id(g, a, b, c)] != 0;
  active[t] = on;
}

// one thread per axis: the runs of the axis (rof, rstart, rlo, rhi)
__global__ void k_band_runs(BandGeom g, BandPlan p) {
  const int k = threadIdx.x;
  if (blockIdx.x != 0 || k >= 3) return;
  int r = -1, plo = -1, phi = -1;
  for (int x = 0; x < g.n[k]; ++x) {
    int lo, hi;
    axis_cover(x, g.b, g.a, g.nb[k], &lo, &hi);
    if (lo != plo || hi != phi) {
      ++r;
      p.rstart[k][r] = x;
      p.rlo[k][r] = lo;
      p.rhi[k][r] = hi;
    }
    p.rof[k][x] = r;
    plo = lo;
    phi = hi;
  }
  p.rstart[k][g.R[k]] = g.n[k];
}

// per run row (X, Y): zoff along z and rowpts; run box (X, Y, Z) is refined when an active block covers it
__global__ void k_band_rows(BandGeom g, BandPlan p) {
  const int64_t xy = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (xy >= (int64_t)g.R[0] * g.R[1]) return;
  const int X = (int)(xy / g.R[1]), Y = (int)(xy % g.R[1]);
  int32_t run = 0;
  for (int Z = 0; Z < g.R[2]; ++Z) {
    p.zoff[xy * g.R[2] + Z] = run;
    bool on = false;
    for (int i = p.rlo[0][X]; i <= p.rhi[0][X] && !on; ++i)
      for (int j = p.rlo[1][Y]; j <= p.rhi[1][Y] && !on; ++j)
        for (int k = p.rlo[2][Z]; k <= p.rhi[2][Z] && !on; ++k) on = p.active[block_id(g, i, j, k)] != 0;
    if (on) run += run_width(p, 2, Z);
  }
  p.rowpts[xy] = run;
}

// per run slab X: yoff along y and plane
__global__ void k_band_slabs(BandGeom g, BandPlan p) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x;
  if (X >= g.R[0]) return;
  int64_t run = 0;
  for (int Y = 0; Y < g.R[1]; ++Y) {
    p.yoff[(int64_t)X * g.R[1] + Y] = run;
    run += p.rowpts[(int64_t)X * g.R[1] + Y] * run_width(p, 1, Y);
  }
  p.plane[X] = run;
}

// one thread: xoff along x; *total = the refinement points
__global__ void k_band_total(BandGeom g, BandPlan p, int64_t* __restrict__ total) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  int64_t run = 0;
  for (int X = 0; X < g.R[0]; ++X) {
    p.xoff[X] = run;
    run += p.plane[X] * run_width(p, 0, X);
  }
  p.xoff[g.R[0]] = run;
  *total = run;
}

// the plan's header, from the counts pnr_band_plan returns
__global__ void k_band_header(BandGeom g, int64_t* __restrict__ hdr, const int64_t* __restrict__ counts) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  hdr[0] = kBandMagic;
  hdr[1] = g.n[0];
  hdr[2] = g.n[1];
  hdr[3] = g.n[2];
  hdr[4] = g.b;
  hdr[5] = g.a;
  hdr[6] = counts[1];
  hdr[7] = 0;
}

__global__ void k_band_points(double lo0, double lo1, double lo2, double hi0, double hi1, double hi2, BandGeom g,
                              BandPlan p, int64_t first, int64_t count, float* __restrict__ xyz,
                              float* __restrict__ viewdirs) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count || first + t >= p.xoff[g.R[0]]) return;      // (nothing past the refinement set)
  int c[3];
  band_point(g, p, first + t, c);
  put_grid_point(lo0, lo1, lo2, hi0, hi1, hi2, g.n[0], g.n[1], g.n[2], c[0], c[1], c[2], t, xyz, viewdirs);
}

// whether the cell with lower corner c exists and lies in an active block
__device__ __forceinline__ bool band_cell_active(const BandGeom& g, const BandPlan& p, int x, int y, int z) {
  if (x < 0 || y < 0 || z < 0 || x + 1 >= g.n[0] || y + 1 >= g.n[1] || z + 1 >= g.n[2]) return false;
  return p.active[block_id(g, x / g.b, y / g.b, z / g.b)] != 0;
}

// k_mc_edges and k_mc_cells over the refinement points: an edge counts when its corners differ in state and one of the
// (up to 4) cells around it is active; a cell outside the active blocks is empty.  Every corner read is stored.
__global__ void k_band_classify(const float* __restrict__ sigma, int64_t M, BandGeom g, BandPlan p, double iso,
                                uint8_t* __restrict__ flags, uint8_t* __restrict__ cube,
                                uint8_t* __restrict__ tcount) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= M) return;
  int c[3];
  band_point(g, p, s, c);
  const bool in = mc_inside(sigma[s], iso);
  for (int a = 0; a < 3; ++a) {
    bool f = false;
    if (c[a] + 1 < g.n[a]) {
      const int u = (a + 1) % 3, v = (a + 2) % 3;
      bool near = false;
      for (int q = 0; q < 4; ++q) {
        int d[3] = {c[0], c[1], c[2]};
        d[u] -= q & 1;
        d[v] -= q >> 1;
        near |= band_cell_active(g, p, d[0], d[1], d[2]);
      }
      if (near) {
        int e[3] = {c[0], c[1], c[2]};
        e[a] += 1;
        f = mc_inside(sigma[band_index(g, p, e[0], e[1], e[2])], iso) != in;
      }
    }
    flags[s * 3 + a] = f;
  }
  int cfg = 0;
  if (band_cell_active(g, p, c[0], c[1], c[2])) {
#pragma unroll
    for (int k = 0; k < 8; ++k)
      cfg |= (int)mc_inside(sigma[band_index(g, p, c[0] + (k & 1), c[1] + ((k >> 1) & 1), c[2] + ((k >> 2) & 1))],
                            iso) << k;
  }
  cube[s] = (uint8_t)cfg;
  tcount[s] = (uint8_t)kMcTriCount[cfg];
}

__global__ void k_band_verts(const float* __restrict__ sigma, int64_t M, BandGeom g, BandPlan p, double iso,
                             const uint8_t* __restrict__ flags, const int64_t* __restrict__ vid, int64_t n_verts,
                             double* __restrict__ verts) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= M) return;
  int c[3];
  bool have_c = false;
  for (int a = 0; a < 3; ++a) {
    if (!flags[s * 3 + a]) continue;
    const int64_t id = vid[s * 3 + a];
    if (id >= n_verts) continue;
    if (!have_c) {
      band_point(g, p, s, c);
      have_c = true;
    }
    int e[3] = {c[0], c[1], c[2]};
    e[a] += 1;
    put_vertex(c[0], c[1], c[2], a, edge_t(sigma[s], sigma[band_index(g, p, e[0], e[1], e[2])], iso), id, verts);
  }
}

__global__ void k_band_tris(int64_t M, BandGeom g, BandPlan p, const uint8_t* __restrict__ cube,
                            const int64_t* __restrict__ toff, const int64_t* __restrict__ vid, int64_t n_tris,
                            int64_t* __restrict__ tris) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= M) return;
  const int cf = cube[s];
  const int cnt = kMcTriCount[cf];
  if (cnt == 0) return;
  int c[3];
  band_point(g, p, s, c);
  const int64_t o = toff[s];
  for (int j = 0; j < cnt; ++j) {
    if (o + j >= n_tris) return;
    for (int k = 0; k < 3; ++k) {
      const int e = kMcTris[cf][j * 3 + k];
      const int q = kMcEdgeCorner[e];
      const int64_t pt = band_index(g, p, c[0] + (q & 1), c[1] + ((q >> 1) & 1), c[2] + ((q >> 2) & 1));
      tris[(o + j) * 3 + k] = vid[pt * 3 + kMcEdgeAxis[e]];
    }
  }
}

// grid_grad at grid point c along axis k, from the refinement storage (the apron holds every neighbour it reads)
__device__ __forceinline__ double band_grad(const float* __restrict__ sigma, const BandGeom& g, const BandPlan& p,
                                            const int c[3], int k) {
  const bool up = c[k] + 1 < g.n[k], dn = c[k] > 0;
  int u[3] = {c[0], c[1], c[2]}, d[3] = {c[0], c[1], c[2]};
  u[k] += 1;
  d[k] -= 1;
  return grad_of(sigma[band_index(g, p, c[0], c[1], c[2])], up ? sigma[band_index(g, p, u[0], u[1], u[2])] : 0.0f,
                 dn ? sigma[band_index(g, p, d[0], d[1], d[2])] : 0.0f, up, dn);
}

__global__ void k_band_vertex_attrs(const float* __restrict__ sigma, int64_t M, BandGeom g, BandPlan p, double iso,
                                    double lo0, double lo1, double lo2, double hi0, double hi1, double hi2,
                                    const uint8_t* __restrict__ flags, const int64_t* __restrict__ vid,
                                    int64_t n_verts, double* __restrict__ normals, float* __restrict__ xyz,
                                    float* __restrict__ viewdirs) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= M) return;
  const double lo[3] = {lo0, lo1, lo2}, hi[3] = {hi0, hi1, hi2};
  int c[3];
  double ga[3];
  bool have_ga = false;
  for (int a = 0; a < 3; ++a) {
    if (!flags[s * 3 + a]) continue;
    const int64_t id = vid[s * 3 + a];
    if (id >= n_verts) continue;
    if (!have_ga) {
      band_point(g, p, s, c);
      for (int k = 0; k < 3; ++k) ga[k] = band_grad(sigma, g, p, c, k);
      have_ga = true;
    }
    const float sa = sigma[s];
    int e[3] = {c[0], c[1], c[2]};
    e[a] += 1;
    const double t = edge_t(sa, sigma[band_index(g, p, e[0], e[1], e[2])], iso);
    double gb[3];
    for (int k = 0; k < 3; ++k) gb[k] = band_grad(sigma, g, p, e, k);
    put_vertex_attrs(c, a, t, mc_inside(sa, iso), ga, gb, g.n, lo, hi, id, normals, xyz, viewdirs);
  }
}

static int check_band(const int32_t* reso, int32_t block, int32_t apron) {
  PNR_CHECK_ARG(reso != nullptr, "NULL reso");
  const int rc = check_dims(reso[0], reso[1], reso[2]);
  if (rc) return rc;
  PNR_CHECK_ARG(block >= 2 && block <= kMaxBandBlock, "block must be in [2, 256]");
  PNR_CHECK_ARG(apron == 0 || apron == 1, "apron must be 0 or 1");
  return PNR_OK;
}

// the plan's buffer, checked against its size
static int band_plan_of(const BandGeom& g, const void* plan, size_t plan_bytes, BandPlan* p) {
  const size_t need = band_carve(g, const_cast<void*>(plan), plan_bytes, p);
  if (plan == nullptr || plan_bytes < need) {
    set_error("plan buffer too small: %zu < %zu", plan_bytes, need);
    return PNR_ERR_WORKSPACE;
  }
  return PNR_OK;
}

// a plan pnr_band_plan made for these reso / block / apron, with n_points refinement points: its header, read back
// (one synchronise of the stream, which the caller's count download makes anyway)
static int band_check_header(const BandGeom& g, const BandPlan& p, int64_t n_points, cudaStream_t s) {
  int64_t h[kBandHdr];
  PNR_CUDA(cudaMemcpyAsync(h, p.hdr, sizeof(h), (cudaMemcpyKind)cudaMemcpyDefault, s));   // (unified addressing)
  PNR_CUDA(cudaStreamSynchronize(s));
  PNR_CHECK_ARG(h[0] == kBandMagic, "plan not made by pnr_band_plan");
  PNR_CHECK_ARG(h[1] == g.n[0] && h[2] == g.n[1] && h[3] == g.n[2] && h[4] == g.b && h[5] == g.a,
                "plan made for another reso / block / apron");
  PNR_CHECK_ARG(h[6] == n_points, "n_points is not the plan's refinement point count");
  return PNR_OK;
}

// the band's marching-cubes workspace (mc_carve over the refinement points) and plan, checked
static int band_mc_setup(const int32_t* reso, int32_t block, int32_t apron, const void* plan, size_t plan_bytes,
                         int64_t M, void* workspace, size_t workspace_bytes, cudaStream_t s, BandGeom* g,
                         BandPlan* p, McWs* w) {
  int rc = check_band(reso, block, apron);
  if (rc) return rc;
  PNR_CHECK_ARG(M >= 0, "negative n_points");
  *g = band_geom(reso, block, apron);
  rc = band_plan_of(*g, plan, plan_bytes, p);
  if (rc) return rc;
  const size_t need = mc_carve(M, workspace, workspace_bytes, w);
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("workspace too small: %zu < %zu", workspace_bytes, need);
    return PNR_ERR_WORKSPACE;
  }
  return band_check_header(*g, *p, M, s);
}

static unsigned grid_for(int64_t n) { return (unsigned)((n + kPtThreads - 1) / kPtThreads); }

// ---- TSDF fusion ---------------------------------------------------------------------------------------------------
// The pixel of the camera-to-world pose P (row-major 4x4: R = P[:3, :3], t = P[:3, 3]) that the world point x projects
// to, by the rule of include/pnr.h pnr_tsdf_fuse: d = x - t, q = R^T d, the inverse of pnr_gen_rays, rounded to the
// nearest pixel with ties up.  -> false when x is behind the camera (or on its plane) or outside the image; else
// *pix = the pixel's index within the view.  pnr_tsdf_fuse and pnr_paint_vertices share it, so they agree on what
// every view sees.
__device__ __forceinline__ bool project_pixel(const float* P, const double x[3], double fx, double fy, double cx,
                                              double cy, int W, int H, double d[3], double q[3], int64_t* pix) {
  for (int j = 0; j < 3; ++j) d[j] = __dsub_rn(x[j], (double)P[4 * j + 3]);
  for (int j = 0; j < 3; ++j)
    q[j] = __dadd_rn(__dadd_rn(__dmul_rn((double)P[j], d[0]), __dmul_rn((double)P[4 + j], d[1])),
                     __dmul_rn((double)P[8 + j], d[2]));
  if (!(q[2] < 0.0)) return false;
  const double px = __dadd_rn(cx, __ddiv_rn(__dmul_rn(fx, q[0]), -q[2]));
  const double py = __dadd_rn(cy, __ddiv_rn(__dmul_rn(fy, q[1]), q[2]));
  const double rx = floor(__dadd_rn(px, 0.5)), ry = floor(__dadd_rn(py, 0.5));    // ties round up
  if (!(rx >= 0.0 && rx <= (double)(W - 1) && ry >= 0.0 && ry <= (double)(H - 1))) return false;
  *pix = (int64_t)(int)ry * W + (int)rx;
  return true;
}

// |q| as both rules sum it: (q_x^2 + q_y^2) + q_z^2
__device__ __forceinline__ double ray_distance(const double q[3]) {
  return sqrt(__dadd_rn(__dadd_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])));
}

// One thread per voxel (pnr_grid_points' point, in float64), the views in order, the rule of include/pnr.h
// pnr_tsdf_fuse.  Every operation is one float64 round-to-nearest step, so oracle/pnr_recon_fuse.py gets the same bits.
__global__ void k_tsdf_fuse(const float* __restrict__ depth, const float* __restrict__ opacity, int V, int W, int H,
                            const float* __restrict__ poses, double fx, double fy, double cx, double cy, double lo0,
                            double lo1, double lo2, double hi0, double hi1, double hi2, int nx, int ny, int nz,
                            double trunc, double min_opacity, float* __restrict__ tsdf) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (int64_t)nx * ny * nz) return;
  const int iz = (int)(p % nz);
  const int iy = (int)((p / nz) % ny);
  const int ix = (int)(p / ((int64_t)ny * nz));
  const double x[3] = {(double)linspace_f32(lo0, hi0, nx, ix), (double)linspace_f32(lo1, hi1, ny, iy),
                       (double)linspace_f32(lo2, hi2, nz, iz)};
  double sum = 0.0;
  int n = 0;
  bool seen = false;
  for (int v = 0; v < V; ++v) {
    double d[3], q[3];
    int64_t pix;
    if (!project_pixel(poses + (int64_t)v * 16, x, fx, fy, cx, cy, W, H, d, q, &pix)) continue;
    seen = true;
    pix += (int64_t)v * H * W;
    const double a = (double)opacity[pix];
    double s = 1.0;                                    // background: free space
    if (a >= min_opacity) {
      s = __ddiv_rn(__dsub_rn(__ddiv_rn((double)depth[pix], a), ray_distance(q)), trunc);
      if (!(s >= -1.0)) continue;                      // occluded (or NaN): no observation
      if (s > 1.0) s = 1.0;
    }
    sum = __dadd_rn(sum, s);
    ++n;
  }
  tsdf[p] = n > 0 ? __double2float_rn(__ddiv_rn(sum, (double)n)) : (seen ? -1.0f : 1.0f);
}

// ---- vertex colours from the rendered views -------------------------------------------------------------------------
// One thread per vertex, the views in order, the rule of include/pnr.h pnr_paint_vertices.  Every operation is one
// float64 round-to-nearest step, so oracle/pnr_recon_paint.py gets the same bits.
__global__ void k_paint_vertices(const double* __restrict__ xyz, const double* __restrict__ normals, int64_t n_verts,
                                 const float* __restrict__ rgb, const float* __restrict__ depth,
                                 const float* __restrict__ opacity, int V, int W, int H,
                                 const float* __restrict__ poses, double fx, double fy, double cx, double cy,
                                 double trunc, double min_opacity, double background, float* __restrict__ rgb_out,
                                 double* __restrict__ weight_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_verts) return;
  const double x[3] = {xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
  const double nrm[3] = {normals[3 * i], normals[3 * i + 1], normals[3 * i + 2]};
  double sum_c[3] = {0.0, 0.0, 0.0}, sum_w = 0.0;
  for (int v = 0; v < V; ++v) {
    double d[3], q[3];
    int64_t pix;
    if (!project_pixel(poses + (int64_t)v * 16, x, fx, fy, cx, cy, W, H, d, q, &pix)) continue;
    pix += (int64_t)v * H * W;
    const double a = (double)opacity[pix];
    if (!(a >= min_opacity)) continue;                 // background (or NaN): no surface colour
    const double dist = ray_distance(q);
    const double s = __ddiv_rn(__dsub_rn(__ddiv_rn((double)depth[pix], a), dist), trunc);
    if (!(s >= -1.0 && s <= 1.0)) continue;            // occluded, or this view's surface is elsewhere (or NaN)
    // cos = n . (t - x) / |q|, with t - x = -d exactly
    const double cosv = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(nrm[0], -d[0]), __dmul_rn(nrm[1], -d[1])),
                                            __dmul_rn(nrm[2], -d[2])), dist);
    if (!(cosv > 0.0)) continue;                       // the back of the surface (or NaN)
    const double bg = __dmul_rn(background, __dsub_rn(1.0, a));
    for (int k = 0; k < 3; ++k) {
      double c = __ddiv_rn(__dsub_rn((double)rgb[3 * pix + k], bg), a);    // un-mix the background
      if (!(c > 0.0)) c = 0.0;                         // (NaN -> 0)
      if (c > 1.0) c = 1.0;
      sum_c[k] = __dadd_rn(sum_c[k], __dmul_rn(cosv, c));
    }
    sum_w = __dadd_rn(sum_w, cosv);
  }
  for (int k = 0; k < 3; ++k) rgb_out[3 * i + k] = sum_w > 0.0 ? __double2float_rn(__ddiv_rn(sum_c[k], sum_w)) : NAN;
  weight_out[i] = sum_w;
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


size_t pnr_band_plan_bytes(const int32_t* reso, int32_t block, int32_t apron) {
  if (!reso || reso[0] < 1 || reso[1] < 1 || reso[2] < 1 || block < 2 || block > kMaxBandBlock ||
      (apron != 0 && apron != 1) || (int64_t)reso[0] * reso[1] * reso[2] > kMaxGridPoints)
    return 0;
  BandPlan p;
  return band_carve(band_geom(reso, block, apron), nullptr, 0, &p);
}

int pnr_band_lattice_points(const double* lo, const double* hi, const int32_t* reso, int32_t block, int64_t first,
                            int64_t count, float* xyz, float* viewdirs, void* stream) {
  PNR_CHECK_ARG(lo && hi, "NULL bounds");
  int rc = check_band(reso, block, 0);
  if (rc) return rc;
  BandGeom g;
  g.b = block;
  for (int k = 0; k < 3; ++k) {
    g.n[k] = reso[k];
    g.nb[k] = (reso[k] - 1 + block - 1) / block;
  }
  PNR_CHECK_ARG(first >= 0 && count >= 0 && first + count <= band_lattice(g), "point range outside the lattice");
  if (count == 0) return PNR_OK;
  PNR_CHECK_ARG(xyz != nullptr, "NULL xyz");
  k_band_lattice<<<grid_for(count), kPtThreads, 0, (cudaStream_t)stream>>>(lo[0], lo[1], lo[2], hi[0], hi[1], hi[2],
                                                                            g, first, count, xyz, viewdirs);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

int pnr_band_plan(const float* coarse, const int32_t* reso, int32_t block, double iso, int32_t apron,
                  int64_t* counts_out, void* plan, size_t plan_bytes, void* stream) {
  int rc = check_band(reso, block, apron);
  if (rc) return rc;
  PNR_CHECK_ARG(counts_out != nullptr, "NULL counts_out");
  const BandGeom g = band_geom(reso, block, apron);
  BandPlan p;
  rc = band_plan_of(g, plan, plan_bytes, &p);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t NB = band_blocks(g);
  if (NB == 0) {                                   // a dimension below 2: no cells, nothing to refine
    PNR_CUDA(cudaMemsetAsync(counts_out, 0, 2 * sizeof(int64_t), s));
  } else {
    PNR_CHECK_ARG(coarse != nullptr, "NULL coarse sigma");
    const int64_t NR = (int64_t)g.R[0] * g.R[1];
    k_band_seed<<<grid_for(NB), kPtThreads, 0, s>>>(coarse, g, iso, p.seeded);
    PNR_LAUNCH_CHECK();
    k_band_dilate<<<grid_for(NB), kPtThreads, 0, s>>>(p.seeded, g, p.active);
    PNR_LAUNCH_CHECK();
    const int64_t nbt = (NB + kScanTile - 1) / kScanTile;    // the active-block count: the scan's reduce passes
    k_scan_reduce<<<(unsigned)nbt, kScanThreads, 0, s>>>(p.active, NB, p.sums);
    PNR_LAUNCH_CHECK();
    k_scan_tiles<<<1, kScanThreads, 0, s>>>(p.sums, nbt, counts_out);
    PNR_LAUNCH_CHECK();
    k_band_runs<<<1, 32, 0, s>>>(g, p);
    PNR_LAUNCH_CHECK();
    k_band_rows<<<grid_for(NR), kPtThreads, 0, s>>>(g, p);
    PNR_LAUNCH_CHECK();
    k_band_slabs<<<grid_for(g.R[0]), kPtThreads, 0, s>>>(g, p);
    PNR_LAUNCH_CHECK();
    k_band_total<<<1, 1, 0, s>>>(g, p, counts_out + 1);
    PNR_LAUNCH_CHECK();
  }
  k_band_header<<<1, 1, 0, s>>>(g, p.hdr, counts_out);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

int pnr_band_points(const double* lo, const double* hi, const int32_t* reso, int32_t block, int32_t apron,
                    const void* plan, size_t plan_bytes, int64_t n_points, int64_t first, int64_t count, float* xyz,
                    float* viewdirs, void* stream) {
  PNR_CHECK_ARG(lo && hi, "NULL bounds");
  int rc = check_band(reso, block, apron);
  if (rc) return rc;
  PNR_CHECK_ARG(first >= 0 && count >= 0 && first + count <= n_points, "point range outside the refinement set");
  const BandGeom g = band_geom(reso, block, apron);
  BandPlan p;
  rc = band_plan_of(g, plan, plan_bytes, &p);
  if (rc) return rc;
  if (count == 0 || band_blocks(g) == 0) return PNR_OK;
  PNR_CHECK_ARG(xyz != nullptr, "NULL xyz");
  k_band_points<<<grid_for(count), kPtThreads, 0, (cudaStream_t)stream>>>(lo[0], lo[1], lo[2], hi[0], hi[1], hi[2], g,
                                                                           p, first, count, xyz, viewdirs);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

size_t pnr_band_mc_workspace_bytes(int64_t n_points) {
  if (n_points < 0 || n_points > kMaxGridPoints) return 0;
  McWs w;
  return mc_carve(n_points, nullptr, 0, &w);
}

int pnr_band_mc_count(const float* sigma, int64_t n_points, const int32_t* reso, int32_t block, int32_t apron,
                      double iso, const void* plan, size_t plan_bytes, int64_t* counts_out, void* workspace,
                      size_t workspace_bytes, void* stream) {
  PNR_CHECK_ARG(counts_out != nullptr, "NULL counts_out");
  cudaStream_t s = (cudaStream_t)stream;
  BandGeom g;
  BandPlan p;
  McWs w;
  int rc = band_mc_setup(reso, block, apron, plan, plan_bytes, n_points, workspace, workspace_bytes, s, &g, &p, &w);
  if (rc) return rc;
  if (n_points == 0) {
    PNR_CUDA(cudaMemsetAsync(counts_out, 0, 2 * sizeof(int64_t), s));
    return PNR_OK;
  }
  PNR_CHECK_ARG(sigma != nullptr, "NULL sigma");
  k_band_classify<<<grid_for(n_points), kPtThreads, 0, s>>>(sigma, n_points, g, p, iso, w.flags, w.cube, w.tcount);
  PNR_LAUNCH_CHECK();
  rc = exclusive_scan(w.flags, 3 * n_points, w.sums_e, w.vid, counts_out, s);
  if (rc) return rc;
  return exclusive_scan(w.tcount, n_points, w.sums_c, w.toff, counts_out + 1, s);
}

int pnr_band_mc_emit(const float* sigma, int64_t n_points, const int32_t* reso, int32_t block, int32_t apron,
                     double iso, const void* plan, size_t plan_bytes, double* verts, int64_t* tris, int64_t n_verts,
                     int64_t n_tris, void* workspace, size_t workspace_bytes, void* stream) {
  PNR_CHECK_ARG(n_verts >= 0 && n_tris >= 0, "negative output sizes");
  cudaStream_t s = (cudaStream_t)stream;
  BandGeom g;
  BandPlan p;
  McWs w;
  int rc = band_mc_setup(reso, block, apron, plan, plan_bytes, n_points, workspace, workspace_bytes, s, &g, &p, &w);
  if (rc) return rc;
  if (n_points == 0) return PNR_OK;
  PNR_CHECK_ARG(sigma != nullptr, "NULL sigma");
  PNR_CHECK_ARG(verts != nullptr || n_verts == 0, "NULL verts");
  PNR_CHECK_ARG(tris != nullptr || n_tris == 0, "NULL tris");
  if (n_verts > 0) {
    k_band_verts<<<grid_for(n_points), kPtThreads, 0, s>>>(sigma, n_points, g, p, iso, w.flags, w.vid, n_verts,
                                                            verts);
    PNR_LAUNCH_CHECK();
  }
  if (n_tris > 0) {
    k_band_tris<<<grid_for(n_points), kPtThreads, 0, s>>>(n_points, g, p, w.cube, w.toff, w.vid, n_tris, tris);
    PNR_LAUNCH_CHECK();
  }
  return PNR_OK;
}

int pnr_band_mc_vertex_attrs(const float* sigma, int64_t n_points, const int32_t* reso, int32_t block, int32_t apron,
                             double iso, const double* lo, const double* hi, const void* plan, size_t plan_bytes,
                             double* normals, float* xyz, float* viewdirs, int64_t n_verts, void* workspace,
                             size_t workspace_bytes, void* stream) {
  PNR_CHECK_ARG(n_verts >= 0, "negative n_verts");
  PNR_CHECK_ARG(lo && hi, "NULL bounds");
  PNR_CHECK_ARG(apron == 1, "vertex attributes need a plan made with apron = 1");
  cudaStream_t s = (cudaStream_t)stream;
  BandGeom g;
  BandPlan p;
  McWs w;
  int rc = band_mc_setup(reso, block, apron, plan, plan_bytes, n_points, workspace, workspace_bytes, s, &g, &p, &w);
  if (rc) return rc;
  if (n_points == 0) return PNR_OK;
  PNR_CHECK_ARG(sigma != nullptr, "NULL sigma");
  if (n_verts == 0 || (!normals && !xyz && !viewdirs)) return PNR_OK;
  k_band_vertex_attrs<<<grid_for(n_points), kPtThreads, 0, s>>>(sigma, n_points, g, p, iso, lo[0], lo[1], lo[2], hi[0],
                                                                 hi[1], hi[2], w.flags, w.vid, n_verts, normals, xyz,
                                                                 viewdirs);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

int pnr_tsdf_fuse(const float* depth, const float* opacity, int32_t V, int32_t W, int32_t H, const float* poses_c2w,
                  float fx, float fy, float cx, float cy, const double* lo, const double* hi, const int32_t* reso,
                  double trunc, double min_opacity, float* tsdf, void* stream) {
  PNR_CHECK_ARG(depth && opacity && poses_c2w && tsdf, "NULL pointer");
  PNR_CHECK_ARG(lo && hi && reso, "NULL bounds");
  PNR_CHECK_ARG(V >= 1 && W >= 1 && H >= 1, "V, W and H must be >= 1");
  const int rc = check_dims(reso[0], reso[1], reso[2]);
  if (rc) return rc;
  PNR_CHECK_ARG(trunc > 0.0 && trunc <= 1.7976931348623157e308, "trunc must be positive and finite");
  PNR_CHECK_ARG(min_opacity > 0.0 && min_opacity <= 1.0, "min_opacity must be in (0, 1]");
  const int64_t N = (int64_t)reso[0] * reso[1] * reso[2];
  k_tsdf_fuse<<<grid_for(N), kPtThreads, 0, (cudaStream_t)stream>>>(
      depth, opacity, V, W, H, poses_c2w, (double)fx, (double)fy, (double)cx, (double)cy, lo[0], lo[1], lo[2], hi[0],
      hi[1], hi[2], reso[0], reso[1], reso[2], trunc, min_opacity, tsdf);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

int pnr_paint_vertices(const double* xyz, const double* normals, int64_t n, const float* rgb, const float* depth,
                       const float* opacity, int32_t V, int32_t W, int32_t H, const float* poses_c2w, float fx,
                       float fy, float cx, float cy, double trunc, double min_opacity, double background,
                       float* rgb_out, double* weight_out, void* stream) {
  PNR_CHECK_ARG(xyz && normals && rgb && depth && opacity && poses_c2w && rgb_out && weight_out, "NULL pointer");
  PNR_CHECK_ARG(n >= 0, "negative vertex count");
  PNR_CHECK_ARG(V >= 1 && W >= 1 && H >= 1, "V, W and H must be >= 1");
  PNR_CHECK_ARG(trunc > 0.0 && trunc <= 1.7976931348623157e308, "trunc must be positive and finite");
  PNR_CHECK_ARG(min_opacity > 0.0 && min_opacity <= 1.0, "min_opacity must be in (0, 1]");
  PNR_CHECK_ARG(background >= -1.7976931348623157e308 && background <= 1.7976931348623157e308,
                "background must be finite");
  if (n == 0) return PNR_OK;
  k_paint_vertices<<<grid_for(n), kPtThreads, 0, (cudaStream_t)stream>>>(
      xyz, normals, n, rgb, depth, opacity, V, W, H, poses_c2w, (double)fx, (double)fy, (double)cx, (double)cy, trunc,
      min_opacity, background, rgb_out, weight_out);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

}  // extern "C"
