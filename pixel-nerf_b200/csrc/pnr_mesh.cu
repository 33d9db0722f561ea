// Connected components of a triangle mesh (include/pnr.h pnr_mesh_components, pnr_mesh_compact_count / _emit;
// util/recon.py keep_components), restated in oracle/pnr_recon_components.py, and decimation (pnr_decimate_*; util/
// recon.py decimate; oracle/pnr_recon_decimate.py) at the end of the file.  The labelling is the one place in mesh
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

// ---- decimation: rounds of independent half-edge collapses with Garland-Heckbert quadrics ----------------------------
// The rule is include/pnr.h's (pnr_decimate_*), restated in oracle/pnr_recon_decimate.py.  Every float64 operation is
// an explicit round-to-nearest intrinsic in the order written there (no FMA contraction), and sqrt of a double is
// IEEE-rounded on the device and the host alike, so the quadrics and errors match the oracle bit for bit.  The only
// atomics are integer ones that build per-vertex incidence lists; what is computed from those lists (sets, minima,
// the boolean flip test) does not depend on their order, and the one order-dependent sum, the initial quadrics, walks
// each vertex's list after sorting it by triangle id.
constexpr int kDecValenceCap = 32;        // a removed vertex has at most this many neighbours, as has d after a collapse
constexpr int kDecIncCap = 64;            // vertices with more incident triangles (corners) are not examined; those
                                          // with more at the start are frozen for the whole call (never c, never d)
constexpr int kDecValInf = 1 << 30;       // their valence: larger than every cap
constexpr int64_t kNone = INT64_MAX;      // best(v) when v has no valid edge: key (+inf, kNone, kNone)
constexpr uint8_t kRemovable = 1, kFan = 2;

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }

// n = (p1 - p0) x (p2 - p0), unnormalised
__device__ __forceinline__ void tri_normal(const double* p0, const double* p1, const double* p2, double* n) {
  const double e1x = dsub(p1[0], p0[0]), e1y = dsub(p1[1], p0[1]), e1z = dsub(p1[2], p0[2]);
  const double e2x = dsub(p2[0], p0[0]), e2y = dsub(p2[1], p0[1]), e2z = dsub(p2[2], p0[2]);
  n[0] = dsub(dmul(e1y, e2z), dmul(e1z, e2y));
  n[1] = dsub(dmul(e1z, e2x), dmul(e1x, e2z));
  n[2] = dsub(dmul(e1x, e2y), dmul(e1y, e2x));
}

// the area-weighted plane quadric of triangle t, added to q (q[k] + Q_t[k]); a zero-area triangle adds nothing
__device__ void add_tri_quadric(const double* __restrict__ xyz, const int64_t* __restrict__ tris, int64_t t,
                                double* q) {
  const double* p0 = xyz + 3 * tris[3 * t];
  double n[3];
  tri_normal(p0, xyz + 3 * tris[3 * t + 1], xyz + 3 * tris[3 * t + 2], n);
  const double len2 = dadd(dadd(dmul(n[0], n[0]), dmul(n[1], n[1])), dmul(n[2], n[2]));
  if (!(len2 > 0.0)) return;
  const double s = sqrt(len2), a = dmul(0.5, s);
  const double ux = __ddiv_rn(n[0], s), uy = __ddiv_rn(n[1], s), uz = __ddiv_rn(n[2], s);
  const double d = -dadd(dadd(dmul(ux, p0[0]), dmul(uy, p0[1])), dmul(uz, p0[2]));
  const double e[10] = {dmul(ux, ux), dmul(ux, uy), dmul(ux, uz), dmul(uy, uy), dmul(uy, uz),
                        dmul(uz, uz), dmul(ux, d),  dmul(uy, d),  dmul(uz, d),  dmul(d, d)};
  for (int k = 0; k < 10; ++k) q[k] = dadd(q[k], dmul(a, e[k]));
}

// err of Q = Qc + Qd at p: sqrt(max(Q(p), 0) / trace(A)), 0 when the trace is 0
__device__ double collapse_error(const double* qc, const double* qd, const double* p) {
  double q[10];
  for (int k = 0; k < 10; ++k) q[k] = dadd(qc[k], qd[k]);
  const double x = p[0], y = p[1], z = p[2];
  const double r0 = dadd(dadd(dadd(dmul(q[0], x), dmul(q[1], y)), dmul(q[2], z)), q[6]);
  const double r1 = dadd(dadd(dadd(dmul(q[1], x), dmul(q[3], y)), dmul(q[4], z)), q[7]);
  const double r2 = dadd(dadd(dadd(dmul(q[2], x), dmul(q[4], y)), dmul(q[5], z)), q[8]);
  const double cost = dadd(dadd(dadd(dadd(dmul(r0, x), dmul(r1, y)), dmul(r2, z)),
                                dadd(dadd(dmul(q[6], x), dmul(q[7], y)), dmul(q[8], z))),
                           q[9]);
  const double tr = dadd(dadd(q[0], q[3]), q[5]);
  if (!(tr > 0.0)) return 0.0;
  return sqrt(__ddiv_rn(cost > 0.0 ? cost : 0.0, tr));
}

// one incident triangle of v, rotated so that v comes first: (v, x, y) at v's first corner; rep = an id repeats
struct Corner {
  int64_t t, x, y;
  bool rep;
};

__device__ __forceinline__ Corner corner_of(const int64_t* __restrict__ tris, int64_t t, int64_t v) {
  const int64_t a = tris[3 * t], b = tris[3 * t + 1], c = tris[3 * t + 2];
  Corner r;
  r.t = t;
  r.rep = a == b || b == c || a == c;
  if (a == v) { r.x = b; r.y = c; }
  else if (b == v) { r.x = c; r.y = a; }
  else { r.x = a; r.y = b; }
  return r;
}

// v's incident triangles: inc[off[v] .. off[v] + cnt[v]) (cnt = 0 for the unexamined)
struct Incidence {
  const int64_t* off;
  const uint8_t* cnt;
  const int64_t* inc;
};

// is w a neighbour of v (some incident triangle of v uses w, w != v)
__device__ bool is_neighbour(const int64_t* __restrict__ tris, const Incidence& I, int64_t v, int64_t w) {
  const int64_t o = I.off[v];
  for (int j = 0; j < I.cnt[v]; ++j) {
    const Corner k = corner_of(tris, I.inc[o + j], v);
    if (k.x == w || k.y == w) return true;
  }
  return false;
}

// Is c -> d valid (include/pnr.h, conditions 1-7) and at what error.  *over_bound = valid but for max_error.
__device__ bool collapse_valid(const double* __restrict__ xyz, const int64_t* __restrict__ tris, const Incidence& I,
                               const int32_t* __restrict__ val, const uint8_t* __restrict__ vflag,
                               const double* __restrict__ quad, double max_error, int64_t c, int64_t d, double* err,
                               bool* over_bound) {
  if (!(vflag[c] & kRemovable) || !(vflag[d] & kFan)) return false;
  if (val[c] + val[d] - 4 > kDecValenceCap) return false;
  const int64_t oc = I.off[c];
  const int nc = I.cnt[c];
  int64_t o1 = -1, o2 = -1;
  for (int j = 0; j < nc; ++j) {
    const Corner k = corner_of(tris, I.inc[oc + j], c);
    if (k.x == d) o1 = k.y;
    if (k.y == d) o2 = k.x;
  }
  if (o1 < 0 || o2 < 0 || val[o1] < 4 || val[o2] < 4) return false;
  // link condition: the neighbours of c (each the x of exactly one corner of c's closed fan) shared with d are o1, o2
  int common = 0;
  for (int j = 0; j < nc; ++j) {
    const Corner k = corner_of(tris, I.inc[oc + j], c);
    if (k.x != d && is_neighbour(tris, I, d, k.x) && ++common > 2) return false;
  }
  if (common != 2) return false;
  // no surviving triangle of c flips
  const double* pd = xyz + 3 * d;
  for (int j = 0; j < nc; ++j) {
    const int64_t t = I.inc[oc + j];
    const int64_t* v = tris + 3 * t;
    if (v[0] == d || v[1] == d || v[2] == d) continue;
    const double* p[3];
    const double* q[3];
    for (int i = 0; i < 3; ++i) {
      p[i] = xyz + 3 * v[i];
      q[i] = v[i] == c ? pd : p[i];
    }
    double n0[3], n1[3];
    tri_normal(p[0], p[1], p[2], n0);
    tri_normal(q[0], q[1], q[2], n1);
    const double dot = dadd(dadd(dmul(n0[0], n1[0]), dmul(n0[1], n1[1])), dmul(n0[2], n1[2]));
    if ((n0[0] != 0.0 || n0[1] != 0.0 || n0[2] != 0.0) && dot <= 0.0) return false;
  }
  *err = collapse_error(quad + 10 * c, quad + 10 * d, pd);
  if (!(*err <= max_error)) {
    *over_bound = true;
    return false;
  }
  return true;
}

__device__ __forceinline__ bool key_less(double e1, int64_t l1, int64_t h1, double e2, int64_t l2, int64_t h2) {
  return e1 < e2 || (e1 == e2 && (l1 < l2 || (l1 == l2 && h1 < h2)));
}

__global__ void k_dec_check_ids(const int64_t* __restrict__ tris, int64_t n_tris, int64_t n_verts,
                                int64_t* __restrict__ status) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n_tris && !tri_ids_ok(tris, t, n_verts)) status[0] = 1;
}

__global__ void k_dec_count(const int64_t* __restrict__ tris, int64_t n_corners, int64_t* __restrict__ deg) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_corners) atomicAdd((ull*)(deg + tris[i]), 1ull);
}

__global__ void k_dec_cap(int64_t n_verts, const int64_t* __restrict__ deg, uint8_t* __restrict__ cnt) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n_verts) cnt[v] = deg[v] <= kDecIncCap ? (uint8_t)deg[v] : 0;
}

// inc[off[v] + slot] = t for each corner of v; the slot comes from counting deg[v] down, so after this deg[v] is 0
// for every examined vertex and still above kDecIncCap for the others
__global__ void k_dec_fill(const int64_t* __restrict__ tris, int64_t n_corners, const uint8_t* __restrict__ cnt,
                           const int64_t* __restrict__ off, int64_t* __restrict__ deg, int64_t* __restrict__ inc) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_corners) return;
  const int64_t v = tris[i];
  if (cnt[v] == 0) return;
  const int64_t slot = (int64_t)atomicAdd((ull*)(deg + v), ~0ull) - 1;
  inc[off[v] + slot] = i / 3;
}

// initial quadrics: each vertex's incident triangles in ascending id (insertion sort of its list, then the sum).  A
// vertex with more than kDecIncCap corners (deg[v] still non-zero after k_dec_fill) is frozen, and its quadric, 0, is
// never read: it is never removed and never receives a collapse, however many corners it loses later.
__global__ void k_dec_quadrics(const double* __restrict__ xyz, const int64_t* __restrict__ tris, int64_t n_verts,
                               Incidence I, const int64_t* __restrict__ deg, int64_t* __restrict__ inc,
                               double* __restrict__ quad, uint8_t* __restrict__ frozen) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_verts) return;
  frozen[v] = deg[v] != 0;
  int64_t* l = inc + I.off[v];
  const int n = I.cnt[v];
  for (int i = 1; i < n; ++i) {
    const int64_t t = l[i];
    int j = i - 1;
    for (; j >= 0 && l[j] > t; --j) l[j + 1] = l[j];
    l[j + 1] = t;
  }
  double q[10] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int i = 0; i < n; ++i) add_tri_quadric(xyz, tris, l[i], q);
  for (int k = 0; k < 10; ++k) quad[10 * v + k] = q[k];
}

// valence and the two flags of include/pnr.h (none for a frozen vertex)
__global__ void k_dec_classify(const int64_t* __restrict__ tris, int64_t n_verts, Incidence I,
                               const int64_t* __restrict__ deg, const uint8_t* __restrict__ frozen,
                               int32_t* __restrict__ val, uint8_t* __restrict__ vflag) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_verts) return;
  if (deg[v] != 0) {                                    // more than kDecIncCap corners: not examined
    val[v] = kDecValInf;
    vflag[v] = 0;
    return;
  }
  const int64_t o = I.off[v];
  const int n = I.cnt[v];
  int64_t nb[2 * kDecIncCap];
  int nn = 0;
  bool rep = false;
  for (int j = 0; j < n; ++j) {
    const Corner k = corner_of(tris, I.inc[o + j], v);
    rep |= k.rep;
    const int64_t ends[2] = {k.x, k.y};
    for (int e = 0; e < 2; ++e) {
      const int64_t w = ends[e];
      if (w == v) continue;
      bool seen = false;
      for (int i = 0; i < nn && !seen; ++i) seen = nb[i] == w;
      if (!seen) nb[nn++] = w;
    }
  }
  val[v] = nn;
  uint8_t f = 0;
  if (!rep && n >= 1) {
    // link edges x -> y, one per triangle: each neighbour is the tail of at most one and the head of at most one
    bool ok = true;
    int64_t start = -1;
    for (int i = 0; i < nn && ok; ++i) {
      int outs = 0, ins = 0;
      for (int j = 0; j < n; ++j) {
        const Corner k = corner_of(tris, I.inc[o + j], v);
        outs += k.x == nb[i];
        ins += k.y == nb[i];
      }
      ok = outs <= 1 && ins <= 1;
      if (ins == 0 && start < 0) start = nb[i];
    }
    if (ok) {
      const bool closed = n == nn;                     // as many link edges as nodes: cycles only
      if (closed) start = nb[0];
      // walk the link from start; one fan when the walk visits every neighbour
      int visited = 1;
      for (int64_t cur = start;;) {
        int64_t next = -1;
        for (int j = 0; j < n; ++j) {
          const Corner k = corner_of(tris, I.inc[o + j], v);
          if (k.x == cur) next = k.y;
        }
        if (next < 0 || next == start) break;
        cur = next;
        ++visited;
      }
      if (visited == nn) f = kFan | (closed && nn >= 3 && nn <= kDecValenceCap ? kRemovable : 0);
    }
  }
  vflag[v] = frozen[v] ? 0 : f;
}

// best(v): the smallest key of the valid edges at v; best_c = the vertex that edge removes
__global__ void k_dec_best(const double* __restrict__ xyz, const int64_t* __restrict__ tris, int64_t n_verts,
                           Incidence I, const int32_t* __restrict__ val, const uint8_t* __restrict__ vflag,
                           const double* __restrict__ quad, double max_error, double* __restrict__ best_err,
                           int64_t* __restrict__ best_lo, int64_t* __restrict__ best_hi, int64_t* __restrict__ best_c,
                           int64_t* __restrict__ status) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_verts) return;
  double be = (double)INFINITY;
  int64_t bl = kNone, bh = kNone, bc = -1;
  bool over = false;
  if (vflag[v] != 0 && val[v] <= kDecValenceCap + 1) {
    const int64_t o = I.off[v];
    const int n = I.cnt[v];
    for (int j = 0; j < n; ++j) {
      const Corner k = corner_of(tris, I.inc[o + j], v);
      const int64_t ends[2] = {k.x, k.y};
      for (int e = 0; e < 2; ++e) {
        const int64_t x = ends[e];
        double e1 = 0.0, e2 = 0.0;
        const bool vx = collapse_valid(xyz, tris, I, val, vflag, quad, max_error, v, x, &e1, &over);
        const bool xv = collapse_valid(xyz, tris, I, val, vflag, quad, max_error, x, v, &e2, &over);
        if (!vx && !xv) continue;
        // the cheaper valid direction; on a tie the larger id goes
        const bool remove_v = vx && (!xv || e1 < e2 || (e1 == e2 && v > x));
        const double err = remove_v ? e1 : e2;
        const int64_t lo = v < x ? v : x, hi = v < x ? x : v;
        if (key_less(err, lo, hi, be, bl, bh)) {
          be = err;
          bl = lo;
          bh = hi;
          bc = remove_v ? v : x;
        }
      }
    }
  }
  best_err[v] = be;
  best_lo[v] = bl;
  best_hi[v] = bh;
  best_c[v] = bc;
  if (over) status[1] = 1;
}

// is key smaller than best(w) for every neighbour w of a other than skip
__device__ bool beats_neighbours(const int64_t* __restrict__ tris, const Incidence& I, int64_t a, int64_t skip,
                                 double e, int64_t lo, int64_t hi, const double* __restrict__ best_err,
                                 const int64_t* __restrict__ best_lo, const int64_t* __restrict__ best_hi) {
  const int64_t o = I.off[a];
  for (int j = 0; j < I.cnt[a]; ++j) {
    const Corner k = corner_of(tris, I.inc[o + j], a);
    const int64_t ends[2] = {k.x, k.y};
    for (int s = 0; s < 2; ++s) {
      const int64_t w = ends[s];
      if (w == skip || w == a) continue;
      if (!key_less(e, lo, hi, best_err[w], best_lo[w], best_hi[w])) return false;
    }
  }
  return true;
}

// sel[c] = 1 when c's best edge removes c, is the best edge of its other end d, and beats best(w) for every other
// neighbour w of c or d
__global__ void k_dec_mark(const int64_t* __restrict__ tris, int64_t n_verts, Incidence I,
                           const double* __restrict__ best_err, const int64_t* __restrict__ best_lo,
                           const int64_t* __restrict__ best_hi, const int64_t* __restrict__ best_c,
                           uint8_t* __restrict__ sel) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_verts) return;
  bool s = false;
  if (best_c[c] == c) {
    const double e = best_err[c];
    const int64_t lo = best_lo[c], hi = best_hi[c], d = lo == c ? hi : lo;
    s = best_err[d] == e && best_lo[d] == lo && best_hi[d] == hi &&
        beats_neighbours(tris, I, c, d, e, lo, hi, best_err, best_lo, best_hi) &&
        beats_neighbours(tris, I, d, c, e, lo, hi, best_err, best_lo, best_hi);
  }
  sel[c] = s;
}

__global__ void k_dec_emit(int64_t n_verts, const uint8_t* __restrict__ sel, const int64_t* __restrict__ pos,
                           const double* __restrict__ best_err, const int64_t* __restrict__ best_lo,
                           const int64_t* __restrict__ best_hi, int64_t* __restrict__ c_out,
                           int64_t* __restrict__ d_out, double* __restrict__ err_out) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_verts || !sel[c]) return;
  const int64_t i = pos[c];
  c_out[i] = c;
  d_out[i] = best_lo[c] == c ? best_hi[c] : best_lo[c];
  err_out[i] = best_err[c];
}

__global__ void k_dec_identity(int64_t n_verts, int64_t* __restrict__ to) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n_verts) to[v] = v;
}

// to[c] = d and Q_d <- Q_d + Q_c; the d of one round are distinct and never a c of it
__global__ void k_dec_merge(const int64_t* __restrict__ cs, const int64_t* __restrict__ ds, int64_t k,
                            int64_t* __restrict__ to, double* __restrict__ quad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  const int64_t c = cs[i], d = ds[i];
  to[c] = d;
  for (int j = 0; j < 10; ++j) quad[10 * d + j] = dadd(quad[10 * d + j], quad[10 * c + j]);
}

// a triangle is dropped when it held a collapsed c and, rewritten, repeats an id: it held the edge cd
__global__ void k_dec_flag_tris(const int64_t* __restrict__ tris, int64_t n_tris, const int64_t* __restrict__ to,
                                uint8_t* __restrict__ tflag) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tris) return;
  const int64_t a = tris[3 * t], b = tris[3 * t + 1], c = tris[3 * t + 2];
  const int64_t ra = to[a], rb = to[b], rc = to[c];
  const bool moved = ra != a || rb != b || rc != c;
  tflag[t] = !(moved && (ra == rb || rb == rc || ra == rc));
}

__global__ void k_dec_emit_tris(const int64_t* __restrict__ tris, int64_t n_tris, const uint8_t* __restrict__ tflag,
                                const int64_t* __restrict__ tnew, const int64_t* __restrict__ to,
                                int64_t* __restrict__ tris_out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tris || !tflag[t]) return;
  const int64_t o = tnew[t];
  for (int k = 0; k < 3; ++k) tris_out[3 * o + k] = to[tris[3 * t + k]];
}

// workspace: status [4] i64, per vertex deg / off / best_* / selection positions / to (i64), cnt / flags / selection
// (u8), valence (i32), per corner the incidence list (i64), per triangle a keep flag (u8) and new ids (i64), and the
// tile sums of the scans
struct DecWs {
  int64_t *status, *deg, *off, *sums_v, *inc, *best_lo, *best_hi, *best_c, *pos, *to, *tnew, *sums_t;
  uint8_t *cnt, *vflag, *sel, *tflag;
  int32_t* val;
  double* best_err;
};

static size_t dec_carve(int64_t N, int64_t M, void* base, size_t cap, DecWs* w) {
  Arena a(base, cap);
  w->status = a.take<int64_t>(4);
  w->deg = a.take<int64_t>(N);
  w->cnt = a.take<uint8_t>(N);
  w->off = a.take<int64_t>(N);
  w->sums_v = a.take<int64_t>(scan_tile_count(N));
  w->inc = a.take<int64_t>(3 * M);
  w->val = a.take<int32_t>(N);
  w->vflag = a.take<uint8_t>(N);
  w->best_err = a.take<double>(N);
  w->best_lo = a.take<int64_t>(N);
  w->best_hi = a.take<int64_t>(N);
  w->best_c = a.take<int64_t>(N);
  w->sel = a.take<uint8_t>(N);
  w->pos = a.take<int64_t>(N);
  w->to = a.take<int64_t>(N);
  w->tflag = a.take<uint8_t>(M);
  w->tnew = a.take<int64_t>(M);
  w->sums_t = a.take<int64_t>(scan_tile_count(M));
  return a.off;
}

static int dec_setup(int64_t n_verts, const int64_t* tris, int64_t n_tris, void* workspace, size_t workspace_bytes,
                     DecWs* w) {
  PNR_CHECK_ARG(n_verts >= 0 && n_tris >= 0, "negative n_verts or n_tris");
  PNR_CHECK_ARG(tris != nullptr || n_tris == 0, "NULL tris");
  const size_t need = dec_carve(n_verts, n_tris, workspace, workspace_bytes, w);
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("workspace too small: %zu < %zu", workspace_bytes, need);
    return PNR_ERR_WORKSPACE;
  }
  return PNR_OK;
}

// the incidence lists of the vertices with at most kDecIncCap corners (any order within a list)
static int dec_incidence(const int64_t* tris, int64_t n_tris, int64_t n_verts, const DecWs& w, cudaStream_t s) {
  PNR_CUDA(cudaMemsetAsync(w.deg, 0, (size_t)n_verts * sizeof(int64_t), s));
  if (n_tris > 0) {
    k_dec_count<<<grid_for(3 * n_tris), kPtThreads, 0, s>>>(tris, 3 * n_tris, w.deg);
    PNR_LAUNCH_CHECK();
  }
  k_dec_cap<<<grid_for(n_verts), kPtThreads, 0, s>>>(n_verts, w.deg, w.cnt);
  PNR_LAUNCH_CHECK();
  int rc = exclusive_scan(w.cnt, n_verts, w.sums_v, w.off, w.status + 2, s);
  if (rc) return rc;
  if (n_tris > 0) {
    k_dec_fill<<<grid_for(3 * n_tris), kPtThreads, 0, s>>>(tris, 3 * n_tris, w.cnt, w.off, w.deg, w.inc);
    PNR_LAUNCH_CHECK();
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

size_t pnr_decimate_workspace_bytes(int64_t n_verts, int64_t n_tris) {
  if (n_verts < 0 || n_tris < 0) return 0;
  DecWs w;
  return dec_carve(n_verts, n_tris, nullptr, 0, &w);
}

int pnr_decimate_init(const double* xyz, int64_t n_verts, const int64_t* tris, int64_t n_tris, double* quadrics,
                      uint8_t* frozen, void* workspace, size_t workspace_bytes, void* stream) {
  DecWs w;
  int rc = dec_setup(n_verts, tris, n_tris, workspace, workspace_bytes, &w);
  if (rc) return rc;
  PNR_CHECK_ARG((xyz != nullptr && quadrics != nullptr && frozen != nullptr) || n_verts == 0,
                "NULL xyz, quadrics or frozen");
  cudaStream_t s = (cudaStream_t)stream;
  PNR_CUDA(cudaMemsetAsync(w.status, 0, sizeof(int64_t), s));
  if (n_tris > 0) {
    k_dec_check_ids<<<grid_for(n_tris), kPtThreads, 0, s>>>(tris, n_tris, n_verts, w.status);
    PNR_LAUNCH_CHECK();
  }
  int64_t bad = 0;
  PNR_CUDA(cudaMemcpyAsync(&bad, w.status, sizeof(bad), (cudaMemcpyKind)cudaMemcpyDefault, s));
  PNR_CUDA(cudaStreamSynchronize(s));
  PNR_CHECK_ARG(bad == 0, "a triangle's vertex id is outside [0, n_verts)");
  if (n_verts == 0) return PNR_OK;
  rc = dec_incidence(tris, n_tris, n_verts, w, s);
  if (rc) return rc;
  Incidence I{w.off, w.cnt, w.inc};
  k_dec_quadrics<<<grid_for(n_verts), kPtThreads, 0, s>>>(xyz, tris, n_verts, I, w.deg, w.inc, quadrics, frozen);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

int pnr_decimate_select(const double* xyz, int64_t n_verts, const int64_t* tris, int64_t n_tris,
                        const double* quadrics, const uint8_t* frozen, double max_error, int64_t* c_out,
                        int64_t* d_out, double* err_out, int64_t* counts_out, void* workspace, size_t workspace_bytes,
                        void* stream) {
  DecWs w;
  int rc = dec_setup(n_verts, tris, n_tris, workspace, workspace_bytes, &w);
  if (rc) return rc;
  PNR_CHECK_ARG(counts_out != nullptr, "NULL counts_out");
  PNR_CHECK_ARG((xyz != nullptr && quadrics != nullptr && frozen != nullptr && c_out != nullptr && d_out != nullptr &&
                 err_out != nullptr) || n_verts == 0, "NULL xyz, quadrics, frozen or outputs");
  PNR_CHECK_ARG(!(max_error < 0.0) && max_error == max_error, "max_error must be >= 0 (+inf for none)");
  counts_out[0] = counts_out[1] = 0;
  if (n_verts == 0 || n_tris == 0) return PNR_OK;
  cudaStream_t s = (cudaStream_t)stream;
  PNR_CUDA(cudaMemsetAsync(w.status, 0, 2 * sizeof(int64_t), s));
  rc = dec_incidence(tris, n_tris, n_verts, w, s);
  if (rc) return rc;
  Incidence I{w.off, w.cnt, w.inc};
  const unsigned gv = grid_for(n_verts);
  k_dec_classify<<<gv, kPtThreads, 0, s>>>(tris, n_verts, I, w.deg, frozen, w.val, w.vflag);
  PNR_LAUNCH_CHECK();
  k_dec_best<<<gv, kPtThreads, 0, s>>>(xyz, tris, n_verts, I, w.val, w.vflag, quadrics, max_error, w.best_err,
                                       w.best_lo, w.best_hi, w.best_c, w.status);
  PNR_LAUNCH_CHECK();
  k_dec_mark<<<gv, kPtThreads, 0, s>>>(tris, n_verts, I, w.best_err, w.best_lo, w.best_hi, w.best_c, w.sel);
  PNR_LAUNCH_CHECK();
  rc = exclusive_scan(w.sel, n_verts, w.sums_v, w.pos, w.status, s);
  if (rc) return rc;
  k_dec_emit<<<gv, kPtThreads, 0, s>>>(n_verts, w.sel, w.pos, w.best_err, w.best_lo, w.best_hi, c_out, d_out,
                                       err_out);
  PNR_LAUNCH_CHECK();
  PNR_CUDA(cudaMemcpyAsync(counts_out, w.status, 2 * sizeof(int64_t), (cudaMemcpyKind)cudaMemcpyDefault, s));
  PNR_CUDA(cudaStreamSynchronize(s));
  return PNR_OK;
}

int pnr_decimate_apply(const int64_t* tris, int64_t n_tris, int64_t n_verts, const int64_t* c, const int64_t* d,
                       int64_t n_collapses, double* quadrics, int64_t* tris_out, int64_t* count_out, void* workspace,
                       size_t workspace_bytes, void* stream) {
  DecWs w;
  int rc = dec_setup(n_verts, tris, n_tris, workspace, workspace_bytes, &w);
  if (rc) return rc;
  PNR_CHECK_ARG(n_collapses >= 0 && 2 * n_collapses <= n_verts, "n_collapses outside [0, n_verts / 2]");
  PNR_CHECK_ARG((c != nullptr && d != nullptr) || n_collapses == 0, "NULL c or d");
  PNR_CHECK_ARG(quadrics != nullptr || n_verts == 0, "NULL quadrics");
  PNR_CHECK_ARG(tris_out != nullptr || n_tris == 0, "NULL tris_out");
  PNR_CHECK_ARG(count_out != nullptr, "NULL count_out");
  *count_out = 0;
  if (n_tris == 0) return PNR_OK;
  cudaStream_t s = (cudaStream_t)stream;
  k_dec_identity<<<grid_for(n_verts), kPtThreads, 0, s>>>(n_verts, w.to);
  PNR_LAUNCH_CHECK();
  if (n_collapses > 0) {
    k_dec_merge<<<grid_for(n_collapses), kPtThreads, 0, s>>>(c, d, n_collapses, w.to, quadrics);
    PNR_LAUNCH_CHECK();
  }
  k_dec_flag_tris<<<grid_for(n_tris), kPtThreads, 0, s>>>(tris, n_tris, w.to, w.tflag);
  PNR_LAUNCH_CHECK();
  rc = exclusive_scan(w.tflag, n_tris, w.sums_t, w.tnew, w.status + 3, s);
  if (rc) return rc;
  k_dec_emit_tris<<<grid_for(n_tris), kPtThreads, 0, s>>>(tris, n_tris, w.tflag, w.tnew, w.to, tris_out);
  PNR_LAUNCH_CHECK();
  PNR_CUDA(cudaMemcpyAsync(count_out, w.status + 3, sizeof(int64_t), (cudaMemcpyKind)cudaMemcpyDefault, s));
  PNR_CUDA(cudaStreamSynchronize(s));
  return PNR_OK;
}

}  // extern "C"
