// Tensor engine: the conditioned MLP of pixelNeRF (ResnetFC d=512, 5 blocks, views averaged
// before block 3; src/model/resnetfc.py:132-184) fused with point geometry, the latent gather,
// the multi-view mean and the output activations (src/model/models.py:158-265) in ONE
// persistent sm_90a kernel.  No [rows x 512] activation ever leaves the SM.
//
// Design (DESIGN.md "tensor engine"):
//  * A CTA owns 64 points of a 128-point tile (two CTAs per tile index).  Per view it runs lin_in + 3 ResNet blocks
//    on the (point, view) rows, sums the views through a per-thread-private scratch line, then runs blocks 3-4 and
//    lin_out on the averaged rows.
//  * Two consumer warpgroups issue wgmma (m64n64k16, fp32 accumulators in registers).  Warpgroup g keeps features
//    128q + 64g + [0, 64), q = 0..3, of the residual stream X in 128 registers per thread for the whole tile.  relu(X)
//    is the A operand of fc_0 and lives in shared memory (64 x 512, fp16 hi/lo, 128 KB).  The hidden layer is never
//    held in full: fc_0 and fc_1 are interleaved over 4 chunks of 128 hidden features, H_c = relu(X) W0_c^T (each
//    warpgroup 64 features, 32 registers), relu(H_c) -> shared memory, X += relu(H_c) W1[:, c]^T.  Every weight tile
//    holds 128 output rows; warpgroup g multiplies its rows [64g, 64g+64), so both warpgroups run the same steps.
//  * Operands are error-compensated fp16 pairs: A = Ahi + Alo, W = Whi + Wlo (both splits exact
//    to ~2^-22), D += Ahi*Whi + Alo*Whi + Ahi*Wlo with fp32 accumulation -- 3 tensor passes per
//    algorithmic GEMM, the cheapest split that meets the 1e-4 RGB tolerance (SURVEY.md fact 8).
//    Weights are pre-scaled by a power of two (exact) so their low parts stay normal in fp16.
//  * lin_z[i](latent) is NOT a per-sample GEMM: bilinear interpolation commutes with a linear
//    layer, so pnr_project_latent builds P_i = lin_z[i](latent) (+ biases) once per encode()
//    and the epilogue gathers 4 taps of P_i and adds them to the residual stream.
//  * 384 threads = two consumer warpgroups (geometry, wgmma, epilogues, ray finishing) and one producer warpgroup.
//    setmaxnreg moves the producer down to 40 registers per thread and the consumers up to 232: the 160 accumulator
//    registers plus addressing fit, and each step's 9 or 12 wgmma issue back to back as one commit group.  Each
//    consumer warpgroup has its own 4-slot ring of the 8 KB halves of the pre-swizzled 16 KB weight tiles that it
//    multiplies; its warps only release a step's slots, and one lane of the producer warpgroup per ring refills them
//    (cp.async.bulk in consumption order onto FULL mbarriers; struct Ring, produce()), so the warps that issue wgmma
//    never stop to refill.  tests/test_tc_codegen.py and tests/test_tc_producer.py guard the register budget.
//  * k_field_tc_fast (PNR_ENGINE_TC_FAST) is the same body with FAST = true: one tensor pass per step, D += Ahi*Whi
//    with fp32 accumulation.  It loads only the W_hi tile of each step (the W_lo slot of the ring stays idle) and never
//    writes the fp16 lo halves of its A operands.  The projected-latent gather (lin_z stays exact), geometry, the view
//    mean, lin_out, compositing, resampling and the flush are the same code.  tests/test_tc_fast_codegen.py.
#include <cuda_fp16.h>
#include <stdlib.h>

#include "pnr_common.cuh"
#include "pnr_geom.cuh"
#include "pnr_ray_ops.cuh"
#include "pnr_tc_ptx.cuh"

namespace pnr {

int sgemm(const float* A, int lda, const float* W, const float* bias, float* C, int ldc, int M, int N, int K,
          bool relu_a, bool accum, cudaStream_t s);  // pnr_field_simt.cu
int gemm_f16x3(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc, int M, int N, int K,
               cudaStream_t s);                      // pnr_gemm_tc.cu

namespace tc {

constexpr int D = 512;
constexpr int ROWS = 64;                 // rows (points) per CTA
constexpr int TILE_POINTS = 128;         // per tile index (two CTAs)
constexpr int NCONSUMER_WARPS = 8;       // two warpgroups
constexpr int NCONSUMERS = NCONSUMER_WARPS * 32;
constexpr int NTHREADS = NCONSUMERS + 128;   // + the producer warpgroup, which issues the weight-slot loads
// setmaxnreg budgets: the launch gives every thread 65536 / 384 -> 168 registers; the producer returns what the
// consumers take
constexpr int PRODUCER_REGS = 40;
constexpr int CONSUMER_REGS = 232;
static_assert(128 * PRODUCER_REGS + NCONSUMERS * CONSUMER_REGS <= NTHREADS * 168,
              "the consumers take no more registers than the producer returns");
constexpr int SLOT_BYTES = 16384;        // 128 weight rows x 64 k x fp16
constexpr int HALF_SLOT_BYTES = SLOT_BYTES / 2;   // rows [64g, 64g+64) of a slot: the half warpgroup g reads
constexpr int NSLOTS = 4;
constexpr int A_CHUNK_BYTES = 16384;     // 64 rows x 64 k x fp16, hi then lo
constexpr int A_BYTES = 8 * A_CHUNK_BYTES;
constexpr int AH_BYTES = 2 * A_CHUNK_BYTES;  // relu(H_c): 128 hidden features
constexpr int SLOTS_LIN_IN = 8;
constexpr int SLOTS_BLOCK = 128;         // fc_0 and fc_1 of one ResNet block, interleaved by hidden chunk
constexpr int SLOTS_TOTAL = SLOTS_LIN_IN + 5 * SLOTS_BLOCK;   // 648
constexpr int SLOTS_HEAD = SLOTS_LIN_IN + 3 * SLOTS_BLOCK;    // lin_in + blocks 0-2, run once per view
constexpr int SLOTS_TAIL = 2 * SLOTS_BLOCK;                   // blocks 3-4, run once per tile
constexpr int HEADER_BYTES = 256;

// shared memory map (offsets from the 1024-aligned base)
constexpr int SM_A = 0;
constexpr int SM_AH = SM_A + A_BYTES;                   // 131072
constexpr int SM_B = SM_AH + AH_BYTES;                  // 163840
constexpr int SM_GEO = SM_B + NSLOTS * SLOT_BYTES;      // [64][8] words: 4 tap offsets + 4 bilinear weights per row
constexpr int SM_PART = SM_A;                           // lin_out partials [64][2][4] floats alias A chunk 0 (free at tile end)
constexpr int SM_BAR = SM_GEO + ROWS * 8 * 4;          // [2][RING_BYTES]: each warpgroup's ring control
constexpr int BAR_FULL = 0;                             // [NSLOTS] mbarriers
constexpr int BAR_COUNT = BAR_FULL + NSLOTS;
constexpr int RING_RELEASED = BAR_COUNT * 8;            // [2] u32: the release counts of the ring's two slot pairs
constexpr int RING_BYTES = RING_RELEASED + 8;
constexpr int SM_NLIST = SM_BAR + 2 * RING_BYTES;       // fused render: number of rays this CTA completed in the current pass
constexpr int SM_PROF = SM_NLIST + 16;                  // phase counters of the profile build: [2][PH_COUNT] u64
#ifdef PNR_TC_PROFILE
constexpr int SMEM_BYTES = SM_PROF + 128;
#else
constexpr int SMEM_BYTES = SM_PROF;
#endif
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one H100 block");
constexpr int FLUSH_SCRATCH_BYTES = A_BYTES / NCONSUMER_WARPS;   // per-warp scratch (cdf + merged samples) in the idle A buffer


// One evaluation pass of the field: the coarse or the fine MLP over a set of points.
struct Pass {
  const uint8_t* packed;   // tensor-engine weight image of this pass's MLP (pnr_pack_mlp)
  const float* proj;       // [3][V][Hl][Wl][512] projected maps of this pass's MLP
  const float* fc0_b[5];
  const float* fc1_b[5];
  const float* lin_out_w;
  const float* lin_out_b;
  float* out;              // [total_points][4]
  int64_t total_points;
  int64_t n_tiles;
  int64_t P;               // points per object (sb = point / P)
  int K;                   // samples per ray (fused render)
};

// Fused render (NeRFRenderer.forward in ONE launch, src/render/nerf.py:251-303): pass 0 = coarse, pass 1 = fine.  The
// CTA that stores the last field value of a ray finishes the ray: compositing (+ importance / depth resampling and the
// sorted merge after the coarse pass) happens in that CTA at the end of its pass ("flush"), fine tiles wait for the
// `ready` flag of their rays.  rays == NULL: plain field evaluation (PixelNeRFNet.forward), one pass.
struct Render {
  const float* rays;       // [R][8]
  const float *lin, *u_c, *u_f, *u_j, *n_d;
  float *zc, *wc, *zf;     // [R][Kc], [R][Kc], [R][Kc+Kf]
  float *rgb_c, *depth_c, *rgb_f, *depth_f, *w_f;
  int* count;              // [2][R] field values stored so far per ray and pass
  int* ready;              // [R] 1 = the ray's fine samples are written
  int* lists;              // [gridDim.x][cap] rays completed by a CTA in the current pass
  int64_t R;
  int cap, Kc, Kf, Kfd, white;
  float depth_std;
};

struct Params {
  PnrScene sc;
  PointSource src;        // plain field evaluation only
  Pass pass[2];
  Render rn;
  float* scratch;         // [gridDim.x][512][64]
  int npass;
  int* status;
};

using namespace tcptx;

enum { MODE_GATHER = 0, MODE_BIAS_WB = 1, MODE_COMBINE = 2, MODE_OUT = 3 };

// Phase profile (built with -DPNR_TC_PROFILE into lib/libpnr_sm90_prof.so, scripts/tc_phase_profile.py): the first
// thread of each consumer warpgroup adds the clock64() time it spends in each phase to a shared-memory counter and, at
// kernel end, to the 8 counters that pnr_tc_counters returns.  The exception is PH_REFILL: the time each ring's
// producer lane spends issuing its refills (not waiting for releases), which it adds to the global counter itself when
// its ring is done (produce()).  The phases of the first thread are disjoint; the rest of PH_TOTAL is wgmma issue and
// the epilogue arithmetic.  The hooks are macros that the production build expands to nothing, so its kernels are the
// same instructions with or without them (tests/test_tc_profile.py).
#ifdef PNR_TC_PROFILE
extern __shared__ __align__(1024) uint8_t smem[];
enum { PH_FULL, PH_REFILL, PH_WGMMA_WAIT, PH_SYNC, PH_GATHER, PH_GEOM, PH_FLUSH, PH_TOTAL, PH_COUNT };
__device__ __forceinline__ void prof_add(int ph, long long t0) {
  const long long dt = clock64() - t0;
  if ((threadIdx.x & 127) == 0)
    reinterpret_cast<unsigned long long*>(smem + SM_PROF)[(threadIdx.x >> 7) * PH_COUNT + ph] += (unsigned long long)dt;
}
__device__ __forceinline__ void prof_finish(int* status, long long t_kernel) {
  prof_add(PH_TOTAL, t_kernel);
  if ((threadIdx.x & 127) == 0) {
    const unsigned long long* c = reinterpret_cast<const unsigned long long*>(smem + SM_PROF) + (threadIdx.x >> 7) * PH_COUNT;
    for (int i = 0; i < PH_COUNT; ++i) atomicAdd(reinterpret_cast<unsigned long long*>(status + 2) + i, c[i]);
  }
}
#define PROF_BEGIN(t) long long t = clock64()
#define PROF_RESTART(t) t = clock64()
#define PROF_END(ph, t) prof_add(ph, t)
// before the kernel's first __syncthreads
#define PROF_INIT() \
  if (threadIdx.x < 2 * PH_COUNT) reinterpret_cast<unsigned long long*>(smem + SM_PROF)[threadIdx.x] = 0
#define PROF_FINISH(status, t) prof_finish(status, t)
// a producer lane's private sum of one phase, added to the global counter when the lane is done
#define PROF_SUM_INIT(s) long long s = 0
#define PROF_SUM(s, t) s += clock64() - (t)
#define PROF_PUBLISH(status, ph, s) atomicAdd(reinterpret_cast<unsigned long long*>((status) + 2) + (ph), (unsigned long long)(s))
#else
#define PROF_BEGIN(t)
#define PROF_RESTART(t)
#define PROF_END(ph, t)
#define PROF_INIT()
#define PROF_FINISH(status, t)
#define PROF_SUM_INIT(s)
#define PROF_SUM(s, t)
#define PROF_PUBLISH(status, ph, s)
#endif

__device__ __forceinline__ void workers_sync() {
  PROF_BEGIN(t0);
  asm volatile("bar.sync 1, 256;" ::: "memory");
  PROF_END(PH_SYNC, t0);
}

__device__ __forceinline__ void st_evict_last(float* q, float v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(q), "f"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ float ld_evict_last(const float* q, uint64_t pol) {
  float v;
  asm volatile("ld.global.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(q), "l"(pol) : "memory");
  return v;
}
__device__ __forceinline__ float4 ldg_stream4(const float4* q, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(q), "l"(pol));
  return v;
}
__device__ __forceinline__ void st_shared_u32(uint32_t saddr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory");
}
// relu(y0), relu(y1) -> packed fp16 hi pair and lo pair (error-compensated split); F2FP packs two values per
// instruction on the fast pipe and saturates instead of producing inf.
__device__ __forceinline__ void split_relu2(float y0, float y1, uint32_t& hi, uint32_t& lo) {
  const float a0 = fmaxf(y0, 0.f), a1 = fmaxf(y1, 0.f);
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(a1), "f"(a0));
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(a1 - hf.y), "f"(a0 - hf.x));
}
// relu(y0), relu(y1) -> packed fp16 pair, the hi half of split_relu2 (single-pass engine)
__device__ __forceinline__ uint32_t relu_f16x2(float y0, float y1) {
  uint32_t hi;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(fmaxf(y1, 0.f)), "f"(fmaxf(y0, 0.f)));
  return hi;
}
// byte offset of the 16-bit pair (row m, k columns [k, k+2) of the 64-wide chunk), k even, in a 128B-swizzled tile
__device__ __forceinline__ uint32_t swz(int m, int k) {
  return (uint32_t)(m * 128 + ((((k >> 3) ^ (m & 7))) << 4) + (k & 7) * 2);
}

extern __shared__ __align__(1024) uint8_t smem[];

// The weight-slot sequence of one CTA, in consumption order: per pass, per tile of its pair, NS x (lin_in + blocks
// 0-2: slots [0, SLOTS_HEAD) of the pass's weight image) then blocks 3-4 (slots [SLOTS_HEAD, SLOTS_TOTAL)), i.e. runs
// of consecutive slots.  The producer lane of ring g walks it one step (two slots: W_hi, W_lo of one tile) at a time
// in registers; only the step that ends a run reads the kernel parameters to walk on to the next view, tile or pass.
struct Feed {
  const uint8_t* src;        // ring g's half of the next step's W_hi slot; nullptr: the sequence is done
  int64_t tile;              // tile of the current run
  int left;                  // steps left in the current run
  int ps, v;                 // pass (npass: sequence done), view of the current run (NS: the blocks 3-4 run)
  __device__ __forceinline__ void begin_run(const Params& p, int g) {
    while (ps < p.npass && tile >= p.pass[ps].n_tiles) {
      ++ps;
      tile = blockIdx.x >> 1;
    }
    const bool head = v < p.sc.NS;
    src = ps < p.npass ? p.pass[ps].packed + HEADER_BYTES + g * HALF_SLOT_BYTES +
                             (head ? 0 : (size_t)SLOTS_HEAD * SLOT_BYTES)
                       : nullptr;
    left = (head ? SLOTS_HEAD : SLOTS_TAIL) / 2;
  }
  __device__ __forceinline__ void next(const Params& p, int g) {
    if (--left > 0) {
      src += 2 * SLOT_BYTES;
      return;
    }
    if (++v > p.sc.NS) {
      v = 0;
      tile += gridDim.x >> 1;
    }
    begin_run(p, g);
  }
};
static_assert(SLOTS_HEAD % 2 == 0 && SLOTS_TAIL % 2 == 0, "a step's two slots lie in one run");
static_assert(SM_PROF <= SMEM_BYTES, "the two rings' barriers and release counts fit under the block limit");

__device__ __forceinline__ uint32_t atom_add_acq_rel(uint32_t saddr, uint32_t v) {
  uint32_t old;
  asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(saddr), "r"(v) : "memory");
  return old;
}

// Weight rings: one per consumer warpgroup.  Warpgroup g multiplies only rows [64g, 64g+64) of every 128-row weight
// tile, the contiguous 8 KB at byte 8192 g of each 16 KB slot, so each warpgroup has its own halves of the 4 slots
// with its own FULL mbarriers and release counts, and its own producer lane (produce()); the two rings share nothing.
// The halves are filled in exactly the order the warpgroup uses them; every step takes two consecutive slots (W_hi,
// W_lo of one 128-row x 64-k tile), so steps alternate between slots 0-1 and 2-3.  A step's halves are released once
// the wgmma that read them have completed: at the next step's acquire(), which retires the step (wait_group 0) and
// releases it BEFORE it waits for the next step's slots, or at the drain that ends an MMA run.  Each warp's lane 0
// releases a step with an acq_rel atomic add on the count of its slot pair; that is all the consumers do for the
// ring.  The producer lane of the ring issues steps 0 and 1 at kernel start and step s + 2 as soon as the count of
// s's slot pair shows all 4 releases of s, so while a warpgroup waits for step s + 1 to land, the copy of s + 2 is
// already in flight beside it.  A warpgroup never waits for the other one's ring, so the two may drift apart by up to
// a step between two workers_sync, which staggers their use of the tensor pipe and of L2.
//  * The count needs no reset: a warp releases step s + 2 (same slot pair) only after its FULL wait for s + 2, which
//    the producer issued only after the 4 releases of s, so the 4 releases of one step are the 4 consecutive adds on
//    their count and the count reaches 4 (s / 2 + 1) exactly when step s is released.
//  * No slot is freed under a reader: the producer issues s + 2 only after all 4 releases of s (its acquire load
//    reads the last of the acq_rel adds), and each release follows wait_group 0, when every wgmma of the warp's
//    warpgroup that read the step has completed.  Every warp runs the same wait_group sequence (none depends on data).
//  * Slot order: one lane issues a ring's refills, in sequence order.
//  * No deadlock: the producer waits only for the releases of step s, which every warp makes before any wait other than
//    the FULL wait of step s + 1 (issued before), since every MMA run ends with a drain before workers_sync, the flush
//    and the fine pass's `ready` wait.  So the producer never waits for anything that those can block.
//  * Pass change: the sequence runs on into the next pass's weight image, so the releases of the coarse pass's last
//    two steps (at the drains that end the pass) let the producer load the fine pass's first two, which arrive during
//    the flush and the `ready` wait.
// FAST (single-pass engine): the same sequence numbers and the same protocol on each step's first (W_hi) slot only;
// the barriers of the W_lo slots are never used.
template <bool FAST>
struct Ring {
  uint32_t bar_base, b_base;   // this warpgroup's ring control (barriers, release counts); its half of slot 0
  uint32_t seq;      // slot sequence number of the next step
  bool has_pend;     // step seq - 2 is still in flight
  int* status;
  __device__ __forceinline__ uint32_t slot_addr(uint32_t s) const { return b_base + (s % NSLOTS) * SLOT_BYTES; }
  // retire and release the step before (the producer refills its slots), then wait for this step's slots
  __device__ __forceinline__ void acquire() {
    if (has_pend) {
      PROF_BEGIN(t1);
      wgmma_wait<0>();
      PROF_END(PH_WGMMA_WAIT, t1);
      release(seq - 2);
      has_pend = false;
    }
    PROF_BEGIN(t0);
    for (uint32_t s = seq; s < seq + (FAST ? 1 : 2); ++s)
      mbar_wait(bar_base + (BAR_FULL + s % NSLOTS) * 8, (s / NSLOTS) & 1, status,
                210 + 4 * (int)(threadIdx.x >> 7) + (int)(s % NSLOTS));
    PROF_END(PH_FULL, t0);
  }
  __device__ __forceinline__ void release(uint32_t s) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) atom_add_acq_rel(bar_base + RING_RELEASED + ((s / 2) & 1) * 4, 1);
    __syncwarp();
  }
  // after the step's wgmma are issued: commit them as one group (the next acquire() or drain() retires it)
  __device__ __forceinline__ void issued() {
    wgmma_commit();
    has_pend = true;
    seq += 2;
  }
  __device__ __forceinline__ void drain() {
    PROF_BEGIN(t0);
    wgmma_wait<0>();
    PROF_END(PH_WGMMA_WAIT, t0);
    if (has_pend) release(seq - 2);
    has_pend = false;
  }
};

// The producer lane of ring g (lane 0 of warp 8 + g): loads ring g's halves of steps 0 and 1, then of each step
// s + 2 once the 4 warps of consumer warpgroup g have released step s, into ring slots (2 s) % 4 and (2 s) % 4 + 1.
// It walks on to the next step's source right after each issue, so the copy leaves as soon as the count completes.
// The single-pass engine loads the W_hi slot only (the weight image stores every tile as hi, lo) and steps over W_lo.
template <bool FAST>
__device__ __forceinline__ void produce(const Params& p, int g) {
  const uint32_t bar_base = smem_u32(smem + SM_BAR) + g * RING_BYTES;
  const uint32_t b_base = smem_u32(smem + SM_B) + g * HALF_SLOT_BYTES;
  // every CTA streams the same 2 x 10 MB of weight images; keep them in L2 ahead of the projected maps that the
  // gather streams past them (evict_first, stage_gather)
  uint64_t keep;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(keep));
  Feed f;
  f.tile = blockIdx.x >> 1;
  f.ps = 0;
  f.v = 0;
  f.begin_run(p, g);
  PROF_SUM_INIT(t_refill);
  for (uint32_t s = 0; f.src != nullptr; ++s) {
    const uint32_t pair = s & 1;
    if (s >= 2) wait_count(bar_base + RING_RELEASED + pair * 4, 4 * (s >> 1), p.status, 220 + 2 * g + (int)pair);
    PROF_BEGIN(t0);
#pragma unroll
    for (uint32_t k = 0; k < (FAST ? 1u : 2u); ++k) {
      const uint32_t full = bar_base + (BAR_FULL + 2 * pair + k) * 8;
      mbar_expect_tx(full, HALF_SLOT_BYTES);
      bulk_g2s_hint(b_base + (2 * pair + k) * SLOT_BYTES, f.src + k * SLOT_BYTES, HALF_SLOT_BYTES, full, keep);
    }
    PROF_SUM(t_refill, t0);
    f.next(p, g);
  }
  PROF_PUBLISH(p.status, PH_REFILL, t_refill);
}

// acc (+)= A[64 x 16 KSTEPS] * W^T over one step: Ahi*Whi + Alo*Whi + Ahi*Wlo (FAST: Ahi*Whi only)
template <bool FAST, int KSTEPS>
__device__ __forceinline__ void mma3(float* acc, uint64_t a_hi, uint64_t b_hi, uint64_t b_lo, bool zero) {
  const uint64_t a_lo = a_hi + (8192 >> 4);
#pragma unroll
  for (int kk = 0; kk < KSTEPS; ++kk) {
    wgmma_m64n64_f16(acc, a_hi + 2 * kk, b_hi + 2 * kk, (zero && kk == 0) ? 0u : 1u);
    if (FAST) continue;
    wgmma_m64n64_f16(acc, a_lo + 2 * kk, b_hi + 2 * kk, 1u);
    wgmma_m64n64_f16(acc, a_hi + 2 * kk, b_lo + 2 * kk, 1u);
  }
}

struct Cons {
  uint32_t smem_u;
  int tid, wg, lane;
  int r0, c0;           // row of accumulator elements with ((i >> 1) & 1) == 0; column offset 2 (lane % 4)
  float w_scale, w_inv;
  uint64_t l2_keep;     // createpolicy evict_last (view-sum scratch)
};

// The epilogues address ~64 loop-invariant locations per thread (operand pairs, biases, scratch lines).  Left to
// itself the compiler hoists all of them out of the tile loop and spills them; instead every epilogue call rebuilds
// one base per buffer behind an opaque move and reaches the individual elements with immediate offsets.
template <typename T>
__device__ __forceinline__ T* opaque(T* v) {
  asm volatile("" : "+l"(v));
  return v;
}
__device__ __forceinline__ uint32_t opaque(uint32_t v) {
  asm volatile("" : "+r"(v));
  return v;
}
// Shared-memory address of the thread's accumulator pair (i, i + 1) of N block q in a buffer of 128B-swizzled
// 64-wide k-chunks (A operand layout): swz(m, k) at m = r0 + 8 ((i >> 1) & 1), k = 8 (i >> 2) + c0 of chunk
// 2 q + wg.  swz only XORs the 16-byte unit index (address bits 4-6) with m & 7 = r0 & 7, and every other term is a
// multiple of 128 (the buffers are 1024-byte aligned) or below 16, so the XOR can be applied to the thread's base
// swz(r0, c0) of chunk wg.
__device__ __forceinline__ uint32_t acc_base(const Cons& c, uint32_t buf) {
  return opaque(c.smem_u + buf + c.wg * A_CHUNK_BYTES + swz(c.r0, c.c0));
}
__device__ __forceinline__ uint32_t acc_addr(uint32_t base, int q, int i) {
  return (base ^ (uint32_t)((i >> 2) << 4)) + q * 2 * A_CHUNK_BYTES + ((i >> 1) & 1) * 1024;
}

// lin_in (K = 42 -> 48) and the fc_1 steps over one 64-wide k-chunk: 4 steps of 128 output rows (N block q);
// warpgroup g accumulates rows [64g, 64g+64) of each into x[q].
template <bool FAST, int KSTEPS>
__device__ __forceinline__ void wide_steps(Ring<FAST>& rg, const Cons& c, float (&x)[4][32], uint64_t a_hi,
                                           bool zero) {
  const uint64_t desc0 = make_desc(0);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    rg.acquire();
    const uint64_t b_hi = desc0 + (rg.slot_addr(rg.seq) >> 4);
    const uint64_t b_lo = desc0 + (rg.slot_addr(rg.seq + 1) >> 4);
    fence_acc<32>(x[q]);
    wgmma_fence();
    mma3<FAST, KSTEPS>(x[q], a_hi, b_hi, b_lo, zero);
    rg.issued();
  }
}

// fc_0 and fc_1 of one ResNet block: X += W1 relu(W0 relu(X) + b0) (the fc_1 bias is added by the caller's epilogue).
template <bool FAST>
__device__ __forceinline__ void fc_block(Ring<FAST>& rg, const Cons& c, float (&x)[4][32],
                                         const float* __restrict__ b0, const int* status) {
  const uint64_t desc0 = make_desc(0);
  float h[32];
#pragma unroll 1
  for (int hc = 0; hc < 4; ++hc) {
    // ---- H_c = relu(X) W0[128 hc + 64 g, +64)^T over K = 512 ----
#pragma unroll 1
    for (int j = 0; j < 8; ++j) {
      rg.acquire();
      const uint64_t a_hi = desc0 + ((c.smem_u + SM_A + j * A_CHUNK_BYTES) >> 4);
      const uint64_t b_hi = desc0 + (rg.slot_addr(rg.seq) >> 4);
      const uint64_t b_lo = desc0 + (rg.slot_addr(rg.seq + 1) >> 4);
      fence_acc<32>(h);
      wgmma_fence();
      mma3<FAST, 4>(h, a_hi, b_hi, b_lo, j == 0);
      rg.issued();
    }
    rg.drain();
    fence_acc<32>(h);
    workers_sync();   // both warpgroups are done with relu(H_{c-1})
    // ---- relu(H_c + b0) -> fp16 hi/lo chunk g of the relu(H) buffer ----
    const float* bc = opaque(b0 + hc * 128 + c.wg * 64 + c.c0);
    const uint32_t ah = acc_base(c, SM_AH);
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const float2 bb = __ldg(reinterpret_cast<const float2*>(bc + 8 * (i >> 2)));
      if (FAST) {
        st_shared_u32(acc_addr(ah, 0, i), relu_f16x2(h[i] * c.w_inv + bb.x, h[i + 1] * c.w_inv + bb.y));
        continue;
      }
      uint32_t hi, lo;
      split_relu2(h[i] * c.w_inv + bb.x, h[i + 1] * c.w_inv + bb.y, hi, lo);
      const uint32_t a = acc_addr(ah, 0, i);
      st_shared_u32(a, hi);
      st_shared_u32(a + 8192, lo);
    }
    fence_proxy_async();
    workers_sync();
    // ---- X += relu(H_c) W1[:, 128 hc, +128)^T ----
#pragma unroll 1
    for (int jj = 0; jj < 2; ++jj)
      wide_steps<FAST, 4>(rg, c, x, desc0 + ((c.smem_u + SM_AH + jj * A_CHUNK_BYTES) >> 4), false);
  }
}

// Coalesced gather of the projected-latent map into the (idle) A buffer: G[row][:] = sum_k w_k * P_i[tap_k(row)][:].
// A warp-load covers two rows x 64 features with lane = feature (2 x 256 contiguous bytes per tap instead of the 32
// scattered lines a lane-per-row gather costs).  G[m][8u..8u+3] and G[m][8u+4..8u+7] of a k-chunk are parked in
// exactly the two 16-byte units (hi, lo) that the fp16 split of those 8 features overwrites later.
__device__ __forceinline__ void stage_gather(uint32_t smem_u, const float* __restrict__ proj_i, int warp, int lane) {
  const int sub = lane >> 4, l16 = lane & 15;
  uint64_t stream;   // the maps (2 x 50 MB at C2) pass through L2 without pushing out the weight images
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(stream));
#pragma unroll 1
  for (int j = 0; j < 8; ++j) {
    float4 t[4][4];
    uint32_t geo[4][4];
    float w[4][4];
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const uint32_t ga = smem_u + SM_GEO + (warp * 8 + it * 2 + sub) * 32;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        uint32_t wb;
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(geo[it][k]) : "r"(ga + 4 * k));
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(wb) : "r"(ga + 16 + 4 * k));
        w[it][k] = __uint_as_float(wb);
      }
    }
    // all 16 tap loads are issued before the first use (one L2 round trip)
#pragma unroll
    for (int it = 0; it < 4; ++it)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        t[it][k] = ldg_stream4(reinterpret_cast<const float4*>(proj_i + geo[it][k] + j * 64) + l16, stream);
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int row = warp * 8 + it * 2 + sub;
      float4 g;
      g.x = ((t[it][0].x * w[it][0] + t[it][1].x * w[it][1]) + t[it][2].x * w[it][2]) + t[it][3].x * w[it][3];
      g.y = ((t[it][0].y * w[it][0] + t[it][1].y * w[it][1]) + t[it][2].y * w[it][2]) + t[it][3].y * w[it][3];
      g.z = ((t[it][0].z * w[it][0] + t[it][1].z * w[it][1]) + t[it][2].z * w[it][2]) + t[it][3].z * w[it][3];
      g.w = ((t[it][0].w * w[it][0] + t[it][1].w * w[it][1]) + t[it][2].w * w[it][2]) + t[it][3].w * w[it][3];
      const uint32_t a = smem_u + SM_A + j * A_CHUNK_BYTES + swz(row, (l16 >> 1) * 8) + ((l16 & 1) ? 8192u : 0u);
      asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(g.x), "f"(g.y), "f"(g.z), "f"(g.w) : "memory");
    }
  }
}

// Epilogue of a layer that ends on the residual stream: y = X / s + (gathered projected latent | bias), then
//   GATHER / BIAS_WB: X = y, relu(y) -> fp16 hi/lo A operand;   COMBINE: view sum (mean after the last view), ditto
//   OUT: lin_out partial sums of relu(y) into out_part.
template <bool FAST, int MODE>
__device__ __forceinline__ void epilogue_x(Ring<FAST>& rg, const Cons& c, float (&x)[4][32], const float* __restrict__ bias,
                                           const float* __restrict__ proj_i, const float* __restrict__ lin_out_w,
                                           int view, int NS, float* __restrict__ scratch, float* out_part) {
  rg.drain();
#pragma unroll
  for (int q = 0; q < 4; ++q) fence_acc<32>(x[q]);
  workers_sync();   // every warpgroup's wgmma reading the A buffer are complete
  const bool produce = (MODE != MODE_OUT) && !(MODE == MODE_COMBINE && view != NS - 1);
  if (MODE == MODE_GATHER) {
    PROF_BEGIN(t0);
    stage_gather(c.smem_u, proj_i, c.tid >> 5, c.lane);
    PROF_END(PH_GATHER, t0);
    workers_sync();
  }
  float o[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  // feature f = 128 q + 64 wg + 8 (i >> 2) + c0 of row m = r0 + 8 ((i >> 1) & 1)
  const uint32_t xa = acc_base(c, SM_A);
  // the staged G pair of (m, f, f + 1) sits in the hi (c0 < 4) or lo unit of 8-feature group f & ~7 (stage_gather)
  const uint32_t ga = opaque(c.smem_u + SM_A + c.wg * A_CHUNK_BYTES + swz(c.r0, 0) + (c.c0 >= 4 ? 8192u : 0u) +
                             (c.c0 & 3) * 4);
  const float* bp = MODE == MODE_GATHER ? nullptr : opaque(bias + 64 * c.wg + c.c0);
  const float* wp = MODE == MODE_OUT ? opaque(lin_out_w + 64 * c.wg + c.c0) : nullptr;
  float* sp0 = MODE == MODE_COMBINE ? opaque(scratch + c.tid) : nullptr;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int r = (i >> 1) & 1;
      float y0 = x[q][i] * c.w_inv, y1 = x[q][i + 1] * c.w_inv;
      if (MODE == MODE_GATHER) {
        // the quad that shares the G pair's 16-byte units reads them all before any writes
        float2 g;
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(g.x), "=f"(g.y) : "r"(acc_addr(ga, q, i)) : "memory");
        __syncwarp();
        y0 += g.x;
        y1 += g.y;
      } else {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bp + 128 * q + 8 * (i >> 2)));
        y0 += bb.x;
        y1 += bb.y;
      }
      if (MODE == MODE_COMBINE && NS > 1) {
        // view-sum scratch (thread-private, coalesced): 128 KB per CTA that every CTA rewrites and re-reads NS-1
        // times per tile.  With both MLPs' projected maps and weight images streaming through the 50 MB L2, plain
        // LRU would evict DIRTY scratch lines to DRAM; evict_last keeps the small hot scratch resident instead
        float* sp = sp0 + (q * 32 + i) * NCONSUMERS;
        if (view == 0) {
          st_evict_last(sp, y0, c.l2_keep);
          st_evict_last(sp + NCONSUMERS, y1, c.l2_keep);
        } else {
          y0 = ld_evict_last(sp, c.l2_keep) + y0;
          y1 = ld_evict_last(sp + NCONSUMERS, c.l2_keep) + y1;
          if (view < NS - 1) {
            st_evict_last(sp, y0, c.l2_keep);
            st_evict_last(sp + NCONSUMERS, y1, c.l2_keep);
          } else {
            const float ns = (float)NS;
            y0 = y0 / ns;
            y1 = y1 / ns;
          }
        }
      }
      if (MODE == MODE_OUT) {
        const float a0 = fmaxf(y0, 0.f), a1 = fmaxf(y1, 0.f);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 w = __ldg(reinterpret_cast<const float2*>(wp + k * D + 128 * q + 8 * (i >> 2)));
          o[r][k] = fmaf(a1, w.y, fmaf(a0, w.x, o[r][k]));
        }
      } else if (produce) {
        x[q][i] = y0 * c.w_scale;
        x[q][i + 1] = y1 * c.w_scale;
        if (FAST) {
          st_shared_u32(acc_addr(xa, q, i), relu_f16x2(y0, y1));
          continue;
        }
        uint32_t hi, lo;
        split_relu2(y0, y1, hi, lo);
        const uint32_t a = acc_addr(xa, q, i);
        st_shared_u32(a, hi);
        st_shared_u32(a + 8192, lo);
      }
    }
  }
  if (MODE == MODE_OUT) {
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        o[r][k] += __shfl_xor_sync(0xffffffffu, o[r][k], 1);
        o[r][k] += __shfl_xor_sync(0xffffffffu, o[r][k], 2);
      }
    if ((c.lane & 3) == 0) {
#pragma unroll
      for (int r = 0; r < 2; ++r)
        reinterpret_cast<float4*>(out_part)[(c.r0 + 8 * r) * 2 + c.wg] = make_float4(o[r][0], o[r][1], o[r][2], o[r][3]);
    }
  } else if (produce) {
    fence_proxy_async();
  }
  workers_sync();
}

// Loads of values that OTHER CTAs wrote during this launch (field values, samples): L2, never a stale L1 line.
struct LdCg {
  __device__ __forceinline__ float operator()(const float* q) const { return __ldcg(q); }
};
struct LdCg4 {
  __device__ __forceinline__ float4 operator()(const float4* q) const { return __ldcg(q); }
};

// Fused render: finish ray `ray` of pass `ps` (one warp).  Coarse pass: compositing (nerf.py:222-249), then importance
// + depth-centred resampling and the sorted merge (nerf.py:120-161, 285-295) into zf, then the ray's `ready` flag.
// Fine pass: compositing into the fine outputs.
// The ray's field values and depths (written by other CTAs: L2 loads) are first staged into the warp's shared-memory
// scratch with coalesced loads, so the sequential transmittance / cdf loops of lane 0 run at shared-memory latency.
__device__ __forceinline__ void finish_ray(const Params& p, int ps, int64_t ray, float* scratch, int lane) {
  const Render& rn = p.rn;
  const float* rr = rn.rays + ray * 8;
  const float near = rr[6], far = rr[7];
  const int Kc = rn.Kc, K = rn.Kc + rn.Kf;
  const int Kp = ps == 0 ? Kc : K;
  const float* zg = ps == 0 ? rn.zc + ray * Kc : rn.zf + ray * K;
  const float4* fg = reinterpret_cast<const float4*>(p.pass[ps].out) + ray * Kp;
  float* wg = ps == 0 ? rn.wc + ray * Kc : (rn.w_f ? rn.w_f + ray * K : nullptr);
  float* rgb = ps == 0 ? rn.rgb_c + ray * 3 : rn.rgb_f + ray * 3;
  float* dep = ps == 0 ? rn.depth_c + ray : rn.depth_f + ray;
  // scratch: field [Kp] float4 | z [Kp] | w [Kp] | resampling scratch [Kc + 1 + K]
  const bool staged = (size_t)(6 * Kp + Kc + 1 + K) * sizeof(float) <= (size_t)FLUSH_SCRATCH_BYTES;
  float4* fs = reinterpret_cast<float4*>(scratch);
  float* zs = scratch + 4 * Kp;
  float* ws = zs + Kp;
  float* rs = staged ? ws + Kp : scratch;
  if (staged) {
    for (int k = lane; k < Kp; k += 32) {
      fs[k] = __ldcg(fg + k);
      zs[k] = __ldcg(zg + k);
    }
    __syncwarp();
    if (lane == 0) composite_ray(zs, fs, far, Kp, rn.white, ws, rgb, dep, LdPlain(), LdPlain4());
    __syncwarp();
    if (wg)
      for (int k = lane; k < Kp; k += 32) wg[k] = ws[k];
  } else {
    if (lane == 0) composite_ray(zg, fg, far, Kp, rn.white, wg, rgb, dep, LdCg(), LdCg4());
    __syncwarp();
  }
  if (ps == 0 && p.npass > 1) {
    const int Ku = rn.Kf - rn.Kfd;
    const float dc = rn.Kfd > 0 ? __ldcg(rn.depth_c + ray) : 0.f;
    if (staged)
      sample_fine_ray(near, far, zs, ws, dc, rn.u_f + ray * Ku, rn.u_j + ray * Ku, rn.n_d + ray * rn.Kfd, rn.depth_std,
                      rn.zf + ray * K, Kc, rn.Kf, rn.Kfd, rs, lane, LdPlain());
    else
      sample_fine_ray(near, far, zg, wg, dc, rn.u_f + ray * Ku, rn.u_j + ray * Ku, rn.n_d + ray * rn.Kfd, rn.depth_std,
                      rn.zf + ray * K, Kc, rn.Kf, rn.Kfd, rs, lane, LdCg());
    __threadfence();
    __syncwarp();
    if (lane == 0) *reinterpret_cast<volatile int*>(rn.ready + ray) = 1;
  }
}

template <bool FAST>
__device__ __forceinline__ void field_tc(const Params& p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = blockIdx.x & 1;        // which 64 points of the 128-point tile
  const int pair = blockIdx.x >> 1;
  const int n_pairs = gridDim.x >> 1;
  const int wg = threadIdx.x >> 7;        // consumer warpgroups 0-1; 2: the producer
  const bool producer = wg == 2;
  const uint32_t bar_base = smem_u32(smem + SM_BAR) + wg * RING_BYTES;   // this warpgroup's ring
  const uint32_t b_base = smem_u32(smem + SM_B) + wg * HALF_SLOT_BYTES;
  int* n_list = reinterpret_cast<int*>(smem + SM_NLIST);
  const int NS = p.sc.NS;
  const bool render = p.rn.rays != nullptr;
  PROF_BEGIN(t_kernel);
  PROF_INIT();

  if (!producer && (threadIdx.x & 127) == 0) {
    for (int i = 0; i < NSLOTS; ++i) mbar_init(bar_base + (BAR_FULL + i) * 8, 1);
    if (threadIdx.x == 0) *n_list = 0;
    uint32_t* released = reinterpret_cast<uint32_t*>(smem + SM_BAR + wg * RING_BYTES + RING_RELEASED);
    released[0] = released[1] = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // ptxas allocates each side for the budget its setmaxnreg sets, as long as the two paths never join again
  if (producer) {
    setmaxnreg_dec<PRODUCER_REGS>();
    // lane 0 of producer warp g refills ring g; the rest of the producer warpgroup has nothing to do
    if (lane == 0 && warp < NCONSUMER_WARPS + 2) produce<FAST>(p, warp - NCONSUMER_WARPS);
    return;
  }
  setmaxnreg_inc<CONSUMER_REGS>();
  const size_t map_stride = (size_t)p.sc.SB * NS * p.sc.Hl * p.sc.Wl * D;

  {
    Cons c;
    c.smem_u = smem_u32(smem);
    c.tid = threadIdx.x;
    c.wg = threadIdx.x >> 7;
    c.lane = lane;
    c.r0 = 16 * (warp & 3) + (lane >> 2);
    c.c0 = 2 * (lane & 3);
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(c.l2_keep));
    Ring<FAST> rg;
    rg.bar_base = bar_base;
    rg.b_base = b_base;
    rg.seq = 0;
    rg.has_pend = false;
    rg.status = p.status;
    float x[4][32];
    float* scratch = p.scratch + (size_t)blockIdx.x * D * ROWS;
    float* out_part = reinterpret_cast<float*>(smem + SM_PART);
    const int grow = threadIdx.x & 63;   // row handled in the geometry stage
    const int gsub = threadIdx.x >> 6;   // 0..3: which 12 of the 48 input channels
    const uint64_t a0_desc = make_desc(c.smem_u + SM_A);   // A chunk 0: the lin_in operand

    for (int ps = 0; ps < p.npass; ++ps) {
      const Pass& P = p.pass[ps];
      c.w_scale = reinterpret_cast<const float*>(P.packed)[0];
      c.w_inv = reinterpret_cast<const float*>(P.packed)[1];
      for (int64_t tile = pair; tile < P.n_tiles; tile += n_pairs) {
        PROF_BEGIN(t_geo);
        const int64_t pt_raw = tile * TILE_POINTS + rank * ROWS + grow;
        const int64_t pt = pt_raw < P.total_points ? pt_raw : P.total_points - 1;
        const int sb = (int)(pt / P.P);
        float xp[3], d[3];
        if (render) {
          // the sample depth is produced here: stratified draw (coarse, nerf.py:98-113) or the merged fine sample that
          // the CTA which finished the ray's coarse pass has written
          const int64_t ray = pt / P.K;
          const int k = (int)(pt - ray * P.K);
          const float* rr = p.rn.rays + ray * 8;
          float zz;
          if (ps == 0) {
            zz = coarse_sample(rr[6], rr[7], p.rn.lin ? p.rn.lin[k] : lin_step_value(k, P.K), p.rn.u_c[pt], P.K);
            if (gsub == 0 && pt_raw < P.total_points) p.rn.zc[pt] = zz;
          } else {
            // ONE poller per ray segment of this CTA's 64 rows (the first row of the CTA and every row that starts a
            // ray), with back-off: CTAs that run out of coarse tiles early wait here for a whole tile time, and
            // hundreds of threads spinning on a handful of L2 lines starve the weight stream of the CTAs still computing
            if (gsub == 0 && (k == 0 || grow == 0) && pt_raw < P.total_points) {
              const volatile int* flag = p.rn.ready + ray;
              if (*flag == 0) {
                const long long t0 = clock64();
                uint32_t spins = 0;
                while (*flag == 0) {
                  __nanosleep(400);
                  if ((++spins & 0xFF) == 0) {
                    if (*(volatile int*)p.status != 0) break;
                    if (clock64() - t0 > timeout_limit(p.status)) {
                      atomicCAS(p.status, 0, 160);
                      if (((volatile int*)p.status)[1]) __trap();
                      break;
                    }
                  }
                }
              }
              __threadfence();
            }
            PROF_END(PH_GEOM, t_geo);
            workers_sync();   // every ray of the tile has its merged samples in L2
            PROF_RESTART(t_geo);
            zz = __ldcg(p.rn.zf + pt);
          }
          for (int i = 0; i < 3; ++i) {
            d[i] = rr[3 + i];
            xp[i] = __fadd_rn(rr[i], __fmul_rn(zz, d[i]));  // nerf.py:185
          }
        } else {
          load_point(p.src, pt, xp, d);
        }
        PROF_END(PH_GEOM, t_geo);
        for (int v = 0; v < NS; ++v) {
          // ---- geometry + the 42 input channels -> A chunk 0 (lin_in operand) ----
          workers_sync();   // the previous view / tile is done with the geometry words and A chunk 0
          {
            PROF_BEGIN(t0);
            PointGeom pg = point_geometry(p.sc, sb, v, xp, d);
            if (gsub == 0) {
              uint32_t* geo = reinterpret_cast<uint32_t*>(smem + SM_GEO) + grow * 8;
              const uint32_t vbase = (uint32_t)(sb * NS + v) * p.sc.Hl * p.sc.Wl;
              geo[0] = (vbase + pg.y0 * p.sc.Wl + pg.x0) * D;
              geo[1] = (vbase + pg.y0 * p.sc.Wl + pg.x1) * D;
              geo[2] = (vbase + pg.y1 * p.sc.Wl + pg.x0) * D;
              geo[3] = (vbase + pg.y1 * p.sc.Wl + pg.x1) * D;
              geo[4] = __float_as_uint(pg.w_nw);
              geo[5] = __float_as_uint(pg.w_ne);
              geo[6] = __float_as_uint(pg.w_sw);
              geo[7] = __float_as_uint(pg.w_se);
            }
            uint8_t* row_hi = smem + SM_A + grow * 128;
            uint8_t* row_lo = row_hi + 8192;
#pragma unroll 1
            for (int e = 0; e < 12; e += 2) {
              const int ch = gsub * 12 + e;
              float f0 = feat_channel(pg, ch), f1 = feat_channel(pg, ch + 1);
              f0 = fmaxf(fminf(f0, 65504.f), -65504.f);
              f1 = fmaxf(fminf(f1, 65504.f), -65504.f);
              __half h0 = __float2half_rn(f0), h1 = __float2half_rn(f1);
              __half l0 = __float2half_rn(f0 - __half2float(h0)), l1 = __float2half_rn(f1 - __half2float(h1));
              const uint32_t hi = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
              const uint32_t lo = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
              const uint32_t byte = swz(grow, ch);
              *reinterpret_cast<uint32_t*>(row_hi - grow * 128 + byte) = hi;
              if (!FAST) *reinterpret_cast<uint32_t*>(row_lo - grow * 128 + byte) = lo;   // (FAST: lo is dead)
            }
            fence_proxy_async();
            PROF_END(PH_GEOM, t0);
            workers_sync();  // geometry and the lin_in operand visible to both warpgroups
          }
          // ---- lin_in (overwrites X), then blocks 0..2 ----
#pragma unroll
          for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int i = 0; i < 32; ++i) x[q][i] = 0.f;   // X is dead until here: no registers held across the geometry
          wide_steps<FAST, 3>(rg, c, x, a0_desc, true);
          epilogue_x<FAST, MODE_GATHER>(rg, c, x, nullptr, P.proj, nullptr, v, NS, nullptr, nullptr);
          for (int blk = 0; blk < 3; ++blk) {
            fc_block(rg, c, x, P.fc0_b[blk], p.status);
            if (blk < 2)
              epilogue_x<FAST, MODE_GATHER>(rg, c, x, nullptr, P.proj + (size_t)(blk + 1) * map_stride, nullptr, v,
                                            NS, nullptr, nullptr);
            else
              epilogue_x<FAST, MODE_COMBINE>(rg, c, x, P.fc1_b[2], nullptr, nullptr, v, NS, scratch, nullptr);
          }
        }
        fc_block(rg, c, x, P.fc0_b[3], p.status);
        epilogue_x<FAST, MODE_BIAS_WB>(rg, c, x, P.fc1_b[3], nullptr, nullptr, 0, NS, nullptr, nullptr);
        fc_block(rg, c, x, P.fc0_b[4], p.status);
        epilogue_x<FAST, MODE_OUT>(rg, c, x, P.fc1_b[4], nullptr, P.lin_out_w, 0, NS, nullptr, out_part);
        if (threadIdx.x < ROWS) {
          const int64_t opt = tile * TILE_POINTS + rank * ROWS + threadIdx.x;
          if (opt < P.total_points) {
            const float4 a = reinterpret_cast<const float4*>(out_part)[threadIdx.x * 2];
            const float4 b = reinterpret_cast<const float4*>(out_part)[threadIdx.x * 2 + 1];
            const float* bo = P.lin_out_b;
            const float r0 = (a.x + b.x) + bo[0], r1 = (a.y + b.y) + bo[1], r2 = (a.z + b.z) + bo[2],
                        r3 = (a.w + b.w) + bo[3];
            float4 o;
            o.x = 1.0f / (1.0f + expf(-r0));   // sigmoid rgb, relu sigma (models.py:260-264)
            o.y = 1.0f / (1.0f + expf(-r1));
            o.z = 1.0f / (1.0f + expf(-r2));
            o.w = fmaxf(r3, 0.f);
            reinterpret_cast<float4*>(P.out)[opt] = o;
            if (render) __threadfence();   // visible device-wide before this ray's completion count moves
          }
        }
        workers_sync();  // out_part is reused by the next tile; all field values of the tile are stored and fenced
        if (render && threadIdx.x < ROWS) {
          // ray completion: the first row of every ray segment inside this CTA's 64 rows adds the segment's length to
          // the ray's counter; whoever brings it to K owns the ray's compositing (and resampling)
          const int64_t opt = tile * TILE_POINTS + rank * ROWS + threadIdx.x;
          if (opt < P.total_points) {
            const int64_t ray = opt / P.K;
            const int k = (int)(opt - ray * P.K);
            if (k == 0 || threadIdx.x == 0) {
              int64_t seg = P.K - k;
              if (seg > ROWS - (int)threadIdx.x) seg = ROWS - (int)threadIdx.x;
              if (seg > P.total_points - opt) seg = P.total_points - opt;
              const int old = atomicAdd(p.rn.count + (size_t)ps * p.rn.R + ray, (int)seg);
              if (old + (int)seg == P.K) {
                const int idx = atomicAdd(n_list, 1);
                p.rn.lists[(size_t)blockIdx.x * p.rn.cap + idx] = (int)ray;
              }
            }
          }
        }
      }
      if (render) {
        // ---- flush: finish the rays whose last field value this CTA stored (A buffer is idle: per-warp scratch) ----
        workers_sync();
        const int n_done = *reinterpret_cast<volatile int*>(n_list);
        __threadfence();   // acquire side of the completion counters
        float* fs = reinterpret_cast<float*>(smem + SM_A + warp * FLUSH_SCRATCH_BYTES);
        PROF_BEGIN(t0);
        for (int i = warp; i < n_done; i += NCONSUMER_WARPS)
          finish_ray(p, ps, p.rn.lists[(size_t)blockIdx.x * p.rn.cap + i], fs, lane);
        PROF_END(PH_FLUSH, t0);
        workers_sync();
        if (threadIdx.x == 0) *n_list = 0;
        // (the next pass's first write to n_list happens after several workers_sync of its first tile)
      }
    }
  }
  PROF_FINISH(p.status, t_kernel);
}

// The exact engine (PNR_ENGINE_TC, 3 tensor passes per step) and the single-pass engine (PNR_ENGINE_TC_FAST).
__global__ void __launch_bounds__(NTHREADS, 1) k_field_tc(const __grid_constant__ Params p) { field_tc<false>(p); }
__global__ void __launch_bounds__(NTHREADS, 1) k_field_tc_fast(const __grid_constant__ Params p) { field_tc<true>(p); }

// ---------------------------------------------------------------------------------------
// weight packing: fp32 [512][K] -> fp16 hi/lo 16 KB slots (128 rows x 64 k, 128B-swizzled) in consumption order
// ---------------------------------------------------------------------------------------
__global__ void k_absmax(const float* __restrict__ w, int n, unsigned int* out) {
  float m = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = fmaxf(m, fabsf(w[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}

__global__ void k_pack_header(const unsigned int* absmax_bits, float* header) {
  float m = __uint_as_float(*absmax_bits);
  float s = 1.0f;
  if (m > 0.f && isfinite(m)) {
    int e = (int)floorf(log2f(16384.0f / m));
    e = max(0, min(e, 12));
    s = exp2f((float)e);
  }
  header[0] = s;
  header[1] = 1.0f / s;
}

// One block per slot.  lin_in (W1 == NULL, 8 slots): (N block q, part).
// A ResNet block (128 slots): per hidden chunk hc, 16 fc_0 slots (k-chunk j, part) of W0 rows [128 hc, +128), then
// 16 fc_1 slots (k-chunk jj of [128 hc, +128), N block q, part) of W1.
__global__ void k_pack_slots(const float* __restrict__ W0, const float* __restrict__ W1, int K, uint8_t* __restrict__ dst,
                             const float* __restrict__ header) {
  const int s = blockIdx.x;
  const float* W;
  int part, n0, k0;
  if (W1 == nullptr) {
    const int q = s >> 1;
    W = W0;
    part = s & 1;
    n0 = 128 * q;
    k0 = 0;
  } else {
    const int hc = s >> 5, r = s & 31;
    if (r < 16) {
      W = W0;
      part = r & 1;
      n0 = 128 * hc;
      k0 = 64 * (r >> 1);
    } else {
      const int r2 = r - 16, q = (r2 >> 1) & 3, jj = r2 >> 3;
      W = W1;
      part = r2 & 1;
      n0 = 128 * q;
      k0 = 64 * (2 * hc + jj);
    }
  }
  uint8_t* out = dst + (size_t)s * SLOT_BYTES;
  const float sc = header[0];
  for (int idx = threadIdx.x; idx < 128 * 64; idx += blockDim.x) {
    const int i = idx >> 6, kk = idx & 63;
    const int n = n0 + i, k = k0 + kk;
    float w = (k < K) ? W[(size_t)n * K + k] * sc : 0.f;
    __half hi = __float2half_rn(w);
    __half val = part ? __float2half_rn(w - __half2float(hi)) : hi;
    const int byte = i * 128 + (((kk >> 3) ^ (i & 7)) * 16) + (kk & 7) * 2;
    *reinterpret_cast<__half*>(out + byte) = val;
  }
}

__global__ void k_proj_bias(const float* a, const float* b, float* out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + b[i];
}

static int* g_status[64] = {nullptr};

static int get_status_buffer(int** out) {
  int dev = 0;
  PNR_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) {
    set_error("device index out of range");
    return PNR_ERR_INVALID;
  }
  if (!g_status[dev]) {
    PNR_CUDA(cudaMalloc(&g_status[dev], 256));
    PNR_CUDA(cudaMemset(g_status[dev], 0, 256));
    // word 0: tag of the first barrier wait that timed out; word 1: 1 = __trap() on a timeout (default: a protocol
    // failure must kill the launch loudly instead of returning garbage with rc == PNR_OK), 0 = record the tag and
    // carry on (PNR_TC_NO_TRAP=1, for scripts/tc_debug.py which then reads the tag with pnr_tc_status)
    const int init[2] = {0, getenv("PNR_TC_NO_TRAP") ? 0 : 1};
    PNR_CUDA(cudaMemcpy(g_status[dev], init, sizeof(init), cudaMemcpyHostToDevice));
    const int mult = getenv("PNR_TC_TIMEOUT_MULT") ? atoi(getenv("PNR_TC_TIMEOUT_MULT")) : 1;   // word 20, see timeout_limit
    PNR_CUDA(cudaMemcpy(g_status[dev] + 20, &mult, sizeof(int), cudaMemcpyHostToDevice));
  }
  *out = g_status[dev];
  return PNR_OK;
}

}  // namespace tc

int tc_status_buffer(int** out) { return tc::get_status_buffer(out); }   // shared with pnr_gemm_tc.cu

bool tc_supported(const PnrScene& sc, const PnrMlp& m) {
  // the kernel addresses the projected maps with 32-bit ELEMENT offsets (geo[0..3]): one map must stay below 2^32 floats
  const unsigned long long map_elems = (unsigned long long)sc.SB * sc.NS * sc.Hl * sc.Wl * tc::D;
  return m.d_hidden == tc::D && m.d_latent == tc::D && sc.C == tc::D && m.d_in == 42 && m.d_out == 4 &&
         m.n_blocks == 5 && m.combine_layer == 3 && sc.NS >= 1 && sc.NS <= 64 && map_elems < (1ull << 32);
}

static int tc_pairs(int64_t n_tiles) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int64_t pairs = sms / 2;
  if (pairs > n_tiles) pairs = n_tiles;
  return (int)(pairs < 1 ? 1 : pairs);
}

static size_t tc_packed_bytes() { return (size_t)tc::HEADER_BYTES + (size_t)tc::SLOTS_TOTAL * tc::SLOT_BYTES; }

size_t tc_workspace_bytes(const PnrScene&, const PnrMlp&, int64_t total_points) {
  int64_t n_tiles = (total_points + tc::TILE_POINTS - 1) / tc::TILE_POINTS;
  return (size_t)tc_pairs(n_tiles) * 2 * tc::D * tc::ROWS * sizeof(float) + 1024;
}

static void fill_pass(tc::Pass& P, const PnrMlp& mlp, const float* proj, float* out, int64_t total_points, int64_t P_obj,
                      int K) {
  P.packed = static_cast<const uint8_t*>(mlp.packed);
  P.proj = proj;
  for (int i = 0; i < 5; ++i) {
    P.fc0_b[i] = mlp.fc0_b[i];
    P.fc1_b[i] = mlp.fc1_b[i];
  }
  P.lin_out_w = mlp.lin_out_w;
  P.lin_out_b = mlp.lin_out_b;
  P.out = out;
  P.total_points = total_points;
  P.n_tiles = (total_points + tc::TILE_POINTS - 1) / tc::TILE_POINTS;
  P.P = P_obj;
  P.K = K;
}

static int tc_launch(tc::Params& p, int pairs, bool fast, cudaStream_t s) {
  int rc = tc::get_status_buffer(&p.status);
  if (rc) return rc;
  static bool attr_set[2][64] = {{false}};
  int dev = 0;
  cudaGetDevice(&dev);
  void (*kernel)(tc::Params) = fast ? tc::k_field_tc_fast : tc::k_field_tc;
  if (!attr_set[fast][dev]) {
    PNR_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES));
    attr_set[fast][dev] = true;
  }
  prof_before(s);
  kernel<<<dim3(pairs * 2), dim3(tc::NTHREADS), tc::SMEM_BYTES, s>>>(p);
  prof_after(s);
  PNR_LAUNCH_CHECK();
  return PNR_OK;
}

static int tc_field_launch(const PnrScene& sc, const PnrMlp& mlp, const float* proj, const PointSource& src,
                           int64_t total_points, float* out, void* ws, size_t ws_bytes, bool fast, cudaStream_t s) {
  if (!tc_supported(sc, mlp) || !mlp.packed || !proj) {
    set_error("tensor engine: unsupported shape or missing packed weights / projected latent");
    return PNR_ERR_UNSUPPORTED;
  }
  if (mlp.packed_bytes < pnr_pack_mlp_bytes(&mlp)) {
    set_error("packed weight buffer too small");
    return PNR_ERR_INVALID;
  }
  if (ws_bytes < tc_workspace_bytes(sc, mlp, total_points)) {
    set_error("workspace too small for the tensor engine");
    return PNR_ERR_WORKSPACE;
  }
  if (total_points == 0) return PNR_OK;
  tc::Params p{};
  p.sc = sc;
  p.src = src;
  p.npass = 1;
  fill_pass(p.pass[0], mlp, proj, out, total_points, src.P, src.K > 0 ? src.K : 1);
  p.rn.rays = nullptr;
  p.scratch = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
  return tc_launch(p, tc_pairs(p.pass[0].n_tiles), fast, s);
}

int tc_field_eval(const PnrScene& sc, const PnrMlp& mlp, const float* proj, const PointSource& src,
                  int64_t total_points, float* out, void* ws, size_t ws_bytes, cudaStream_t s) {
  return tc_field_launch(sc, mlp, proj, src, total_points, out, ws, ws_bytes, false, s);
}

int tc_field_eval_fast(const PnrScene& sc, const PnrMlp& mlp, const float* proj, const PointSource& src,
                       int64_t total_points, float* out, void* ws, size_t ws_bytes, cudaStream_t s) {
  return tc_field_launch(sc, mlp, proj, src, total_points, out, ws, ws_bytes, true, s);
}

// ---- fused render: NeRFRenderer.forward (nerf.py:251-303) in ONE launch of the tensor engine ----------------------
// Workspace: view-sum scratch | field values of both passes | completion counters + ready flags | completion lists.
static int tc_render_pairs(int64_t R, int Kc, int K) {
  const int64_t tiles = ((int64_t)R * (K > Kc ? K : Kc) + tc::TILE_POINTS - 1) / tc::TILE_POINTS;
  return tc_pairs(tiles);
}
static int tc_render_cap(int64_t R, int Kc, int K, int pairs) {
  // rays a CTA can complete in one pass: (tiles per pair) x (rays that end inside 64 rows)
  int64_t cap = 0;
  for (int Kp : {Kc, K}) {
    if (Kp <= 0) continue;
    const int64_t tiles = (R * Kp + tc::TILE_POINTS - 1) / tc::TILE_POINTS;
    const int64_t per_pair = (tiles + pairs - 1) / pairs;
    const int64_t c = per_pair * (tc::ROWS / Kp + 2);
    if (c > cap) cap = c;
  }
  return (int)(cap + 8);
}

size_t tc_render_workspace_bytes(const PnrScene& sc, int64_t R, int Kc, int Kf) {
  const int K = Kc + Kf;
  const int pairs = tc_render_pairs(R, Kc, K);
  size_t b = (size_t)pairs * 2 * tc::D * tc::ROWS * sizeof(float) + 1024;
  b += align_up((size_t)R * Kc * 16, 256) + align_up((size_t)R * K * 16, 256);
  b += align_up((size_t)R * 3 * sizeof(int), 256);
  b += align_up((size_t)pairs * 2 * tc_render_cap(R, Kc, K, pairs) * sizeof(int), 256);
  return b + 1024;
}

int tc_render(const PnrScene& sc, const PnrMlp& mc, const PnrMlp& mf, const float* proj_c, const float* proj_f,
              const PnrRenderCfg& cfg, const float* rays, const PnrNoise& noise, float* zc, float* wc, float* zf,
              const PnrRenderOut& out, int64_t B, void* ws, size_t ws_bytes, cudaStream_t s) {
  const int64_t R = B * sc.SB;
  const int Kc = cfg.n_coarse, Kf = cfg.n_fine, Kfd = cfg.n_fine_depth, K = Kc + Kf;
  if (ws_bytes < tc_render_workspace_bytes(sc, R, Kc, Kf)) {
    set_error("workspace too small for the fused render");
    return PNR_ERR_WORKSPACE;
  }
  if (K > 512) {
    set_error("n_coarse + n_fine = %d exceeds 512", K);
    return PNR_ERR_INVALID;
  }
  if ((int64_t)R * K >= (1ll << 31)) {
    set_error("too many sample points for one fused render call (R * K must stay below 2^31)");
    return PNR_ERR_INVALID;
  }
  const int pairs = tc_render_pairs(R, Kc, K);
  Arena ar(ws, ws_bytes);
  tc::Params p{};
  p.sc = sc;
  p.scratch = ar.take<float>((size_t)pairs * 2 * tc::D * tc::ROWS);
  float* field_c = ar.take<float>((size_t)R * Kc * 4);
  float* field_f = ar.take<float>((size_t)R * K * 4);
  int* flags = ar.take<int>((size_t)R * 3);
  p.rn.cap = tc_render_cap(R, Kc, K, pairs);
  p.rn.lists = ar.take<int>((size_t)pairs * 2 * p.rn.cap);
  PNR_CUDA(cudaMemsetAsync(flags, 0, (size_t)R * 3 * sizeof(int), s));
  p.npass = Kf > 0 ? 2 : 1;
  fill_pass(p.pass[0], mc, proj_c, field_c, R * Kc, B * Kc, Kc);
  if (Kf > 0) fill_pass(p.pass[1], mf, proj_f, field_f, R * K, B * K, K);
  tc::Render& rn = p.rn;
  rn.rays = rays;
  rn.lin = noise.lin_steps;
  rn.u_c = noise.u_coarse;
  rn.u_f = noise.u_fine;
  rn.u_j = noise.u_fine_jit;
  rn.n_d = noise.n_depth;
  rn.zc = zc;
  rn.wc = wc;
  rn.zf = zf;
  rn.rgb_c = out.rgb_coarse;
  rn.depth_c = out.depth_coarse;
  rn.rgb_f = out.rgb_fine;
  rn.depth_f = out.depth_fine;
  rn.w_f = out.weights_fine;
  rn.count = flags;
  rn.ready = flags + 2 * R;
  rn.R = R;
  rn.Kc = Kc;
  rn.Kf = Kf;
  rn.Kfd = Kfd;
  rn.white = cfg.white_bkgd;
  rn.depth_std = cfg.depth_std;
  return tc_launch(p, pairs, cfg.engine == PNR_ENGINE_TC_FAST, s);
}

}  // namespace pnr

using namespace pnr;

extern "C" {

size_t pnr_pack_mlp_bytes(const PnrMlp* mlp) {
  if (!mlp || mlp->d_hidden != tc::D || mlp->d_latent != tc::D || mlp->n_blocks != 5 || mlp->d_in != 42) return 0;
  return tc_packed_bytes();
}

int pnr_pack_mlp(const PnrMlp* mlp, void* packed, size_t packed_bytes, void* stream) {
  PNR_CHECK_ARG(mlp && packed, "NULL pointer");
  size_t need = pnr_pack_mlp_bytes(mlp);
  if (need == 0) {
    set_error("pnr_pack_mlp: the tensor engine needs d_hidden = d_latent = 512, 5 blocks, d_in = 42");
    return PNR_ERR_UNSUPPORTED;
  }
  PNR_CHECK_ARG(packed_bytes >= need, "packed buffer too small");
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* base = static_cast<uint8_t*>(packed);
  float* header = reinterpret_cast<float*>(base);
  unsigned int* absmax = reinterpret_cast<unsigned int*>(base + 64);
  PNR_CUDA(cudaMemsetAsync(base, 0, tc::HEADER_BYTES, s));
  // global |w| max over every tensor-engine layer (one power-of-two scale for the whole MLP)
  tc::k_absmax<<<64, 256, 0, s>>>(mlp->lin_in_w, tc::D * mlp->d_in, absmax);
  PNR_LAUNCH_CHECK();
  for (int i = 0; i < 5; ++i) {
    tc::k_absmax<<<64, 256, 0, s>>>(mlp->fc0_w[i], tc::D * tc::D, absmax);
    PNR_LAUNCH_CHECK();
    tc::k_absmax<<<64, 256, 0, s>>>(mlp->fc1_w[i], tc::D * tc::D, absmax);
    PNR_LAUNCH_CHECK();
  }
  tc::k_pack_header<<<1, 1, 0, s>>>(absmax, header);
  PNR_LAUNCH_CHECK();
  uint8_t* slots = base + tc::HEADER_BYTES;
  tc::k_pack_slots<<<tc::SLOTS_LIN_IN, 256, 0, s>>>(mlp->lin_in_w, nullptr, mlp->d_in, slots, header);
  PNR_LAUNCH_CHECK();
  for (int i = 0; i < 5; ++i) {
    uint8_t* dst = slots + (size_t)(tc::SLOTS_LIN_IN + i * tc::SLOTS_BLOCK) * tc::SLOT_BYTES;
    tc::k_pack_slots<<<tc::SLOTS_BLOCK, 256, 0, s>>>(mlp->fc0_w[i], mlp->fc1_w[i], tc::D, dst, header);
    PNR_LAUNCH_CHECK();
  }
  return PNR_OK;
}

size_t pnr_project_latent_bytes(const PnrScene* sc, const PnrMlp* mlp) {
  if (!sc || !mlp || !tc_supported(*sc, *mlp)) return 0;
  return (size_t)3 * sc->SB * sc->NS * sc->Hl * sc->Wl * tc::D * sizeof(float);
}

// proj[i] = lin_z[i](latent) + lin_z[i].bias + (i == 0 ? lin_in.bias : blocks[i-1].fc_1.bias)
int pnr_project_latent(const PnrScene* sc, const PnrMlp* mlp, float* proj, size_t proj_bytes, void* workspace,
                       size_t workspace_bytes, void* stream) {
  PNR_CHECK_ARG(sc && mlp && proj && workspace, "NULL pointer");
  size_t need = pnr_project_latent_bytes(sc, mlp);
  if (need == 0) {
    set_error("pnr_project_latent: unsupported shape for the tensor engine");
    return PNR_ERR_UNSUPPORTED;
  }
  PNR_CHECK_ARG(proj_bytes >= need, "proj buffer too small");
  PNR_CHECK_ARG(workspace_bytes >= 3 * tc::D * sizeof(float) + 256, "workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  float* bias = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  const int64_t rows = (int64_t)sc->SB * sc->NS * sc->Hl * sc->Wl;
  // deterministic mode: the rest of the workspace holds the GEMM's split-K partials
  const size_t used = (size_t)((reinterpret_cast<char*>(bias + 3 * tc::D) - static_cast<char*>(workspace)) + 255) & ~(size_t)255;
  SplitKScope splitk(reinterpret_cast<float*>(static_cast<char*>(workspace) + used),
                     workspace_bytes > used ? workspace_bytes - used : 0);
  for (int i = 0; i < 3; ++i) {
    const float* extra = (i == 0) ? mlp->lin_in_b : mlp->fc1_b[i - 1];
    tc::k_proj_bias<<<2, 256, 0, s>>>(mlp->lin_z_b[i], extra, bias + i * tc::D, tc::D);
    PNR_LAUNCH_CHECK();
    // fp16 hi/lo split tensor-core GEMM (22 mantissa bits, the precision of the fused kernel's own products);
    // PNR_PROJECT_SIMT=1 keeps the fp32 FFMA SGEMM of round 1
    static const bool simt = getenv("PNR_PROJECT_SIMT") != nullptr;
    int rc = simt ? sgemm(sc->latent_nhwc, tc::D, mlp->lin_z_w[i], bias + i * tc::D, proj + (size_t)i * rows * tc::D,
                          tc::D, (int)rows, tc::D, tc::D, false, false, s)
                  : gemm_f16x3(sc->latent_nhwc, tc::D, mlp->lin_z_w[i], tc::D, bias + i * tc::D,
                               proj + (size_t)i * rows * tc::D, tc::D, (int)rows, tc::D, tc::D, s);
    if (rc) return rc;
  }
  return PNR_OK;
}

// Debug / test hook: synchronises the device and returns the tensor-engine status word
// (0 = ok, otherwise the tag of the first barrier wait that timed out -- only observable with PNR_TC_NO_TRAP=1, by
// default a timeout traps and every later CUDA call fails); clears it.
int pnr_tc_status(int* out) {
  int* buf = nullptr;
  int rc = tc::get_status_buffer(&buf);
  if (rc) return rc;
  PNR_CUDA(cudaDeviceSynchronize());
  int v = 0;
  PNR_CUDA(cudaMemcpy(&v, buf, sizeof(int), cudaMemcpyDeviceToHost));
  PNR_CUDA(cudaMemset(buf, 0, sizeof(int)));
  if (out) *out = v;
  return PNR_OK;
}


// Debug: 8 cycle counters accumulated over all launches since the last call; clears them.  Only the profile build
// of the tensor engine (-DPNR_TC_PROFILE, lib/libpnr_sm90_prof.so) records them: its per-phase clocks, PH_FULL ..
// PH_TOTAL, summed over the first thread of each warpgroup of every CTA.  Otherwise they read 0.
int pnr_tc_counters(unsigned long long* out8) {
  int* buf = nullptr;
  int rc = tc::get_status_buffer(&buf);
  if (rc) return rc;
  PNR_CUDA(cudaDeviceSynchronize());
  PNR_CUDA(cudaMemcpy(out8, buf + 2, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  PNR_CUDA(cudaMemset(buf + 2, 0, 8 * sizeof(unsigned long long)));
  return PNR_OK;
}

}  // extern "C"
