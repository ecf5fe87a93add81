// clc_kernels.cuh -- the sm_90a kernels.
//
// K1  clc_sweep_kernel   fused residual + Jacobian + Cauchy weight + reduce over every laser point
//                        (HBM-bandwidth bound FP64 map-reduce; 24 B per residual streamed with 128-bit loads)
// K3  clc_lm_kernel      single-thread LM update (multi-rank path, after the all-reduce)
// K0  layout kernels     AoS -> SoA, frame pose -> board plane / edge planes, warp start table
// K5  generator kernels  synthetic boards on the device
#pragma once

#include <cuda_runtime.h>

#include <type_traits>

#include "clc_camera.cuh"
#include "clc_expand.cuh"
#include "clc_frames.cuh"
#include "clc_lm.cuh"

namespace clc {

// Launch shape: one 12-warp block per SM with 2 stages per warp.  On an H100 (sm_90a) 384 threads leave the streaming
// instantiations 168 registers and no spills; with 512 threads (128 registers) they spill ~0.5 KB per thread and run ~17 %
// slower at configs[1] and ~10 % at configs[2] (320 threads ties with 384, 448 is as slow as 512; a third stage or two
// 256-thread blocks per SM gain nothing).  Dynamic shared memory per block: ~111 KiB general, ~135 KiB planar.
#ifndef CLC_THREADS
#define CLC_THREADS 384
#endif
#ifndef CLC_BLOCKS_PER_SM
#define CLC_BLOCKS_PER_SM 1
#endif
#ifndef CLC_STAGES
#define CLC_STAGES 2
#endif
constexpr int kThreads = CLC_THREADS;
constexpr int kBlocksPerSM = CLC_BLOCKS_PER_SM;
constexpr int kWarps = kThreads / 32;
constexpr int kTileStride = 13;       // doubles per tile row: 10 moments, product, exponent, frame id
#ifndef CLC_CHUNK
#define CLC_CHUNK 128
#endif
constexpr int kChunk = CLC_CHUNK;     // points per pipeline stage and coordinate array (one bulk copy each, 8 B/point)
constexpr int kGroups = kChunk / 64;  // 64-point groups per stage: every lane takes 2 adjacent points of each group
constexpr int kStages = CLC_STAGES;   // bulk-copy stages in flight per warp (x 3 KiB)
constexpr int kMaxOut = 54;           // closed-form mode: 45 + 9
constexpr int kMaxRanks = 16;
constexpr int kMailboxSlot = 64;      // doubles per (parity, source rank) mailbox slot (>= kMaxOut)
#ifndef CLC_PLANAR_STAGES
#define CLC_PLANAR_STAGES CLC_STAGES
#endif
#ifndef CLC_PLANAR_CHUNK
#define CLC_PLANAR_CHUNK (CLC_CHUNK * 2)
#endif
// the two-stream (planar, z == 0) kernels: 256-point stages, one 2 KiB bulk copy per coordinate array
constexpr int kPlanarStages = CLC_PLANAR_STAGES;
constexpr int kPlanarChunk = CLC_PLANAR_CHUNK;
static_assert(kChunk % 64 == 0 && kPlanarChunk % 64 == 0, "stages are made of 64-point groups");
constexpr int kMaxChunk = kChunk > kPlanarChunk ? kChunk : kPlanarChunk;
// Soft lockstep of the warps of a block: a warp does not start stage c before every warp of its block has finished stage
// c - kLockstepSlack (0 = off).  The issue arbiter lets some warps run ahead; they then leave early and the block finishes
// its last stages with few loads in flight.  Holding the front-runners back hands their issue slots to the stragglers: the
// block's warps end together, at the block's mean finishing time, with the static (deterministic) partition untouched.
#ifndef CLC_LOCKSTEP_SLACK
#define CLC_LOCKSTEP_SLACK 0
#endif
constexpr int kLockstepSlack = CLC_LOCKSTEP_SLACK;
constexpr int kBarsPerWarp = kStages > kPlanarStages ? kStages : kPlanarStages;
constexpr int kTileDoublesPerWarp = 32 * kTileStride;
// dynamic shared memory of a kernel family: per-warp ring + per-warp tile + per-warp mbarriers
__host__ __device__ constexpr int ring_doubles_per_warp(bool planar) { return planar ? kPlanarStages * 2 * kPlanarChunk : kStages * 3 * kChunk; }
__host__ __device__ constexpr int dyn_smem_bytes(bool planar) {
  return kWarps * ring_doubles_per_warp(planar) * 8 + kWarps * kTileDoublesPerWarp * 8 + kWarps * kBarsPerWarp * 8;
}

// per-frame report mode: the tile keeps 3 more doubles per parked piece (sum e, sum e^2, max |e|) behind the mbarriers
constexpr int kFrameTileDoublesPerWarp = 32 * 3;
__host__ __device__ constexpr int frames_smem_bytes(bool planar) {
  return dyn_smem_bytes(planar) + kWarps * kFrameTileDoublesPerWarp * 8;
}

// kModeFrames: the per-frame report (clc_frame_report) -- every frame's residual statistics and its share of the normal
// equations go to a row of their own instead of being summed
// kModeSegments: independent solves over runs of frames (clc_*_segments) -- every frame's raw moments at its segment's pose go
// to a row of their own (clc_segment_fixup_kernel expands them); the frame constants m, c come from SweepArgs::seg_consts.
// A raw row: 10 moments, the cost (Cauchy: product of (1 + e^2/a^2) with its exponent taken out; other kinds: sum rho~(e),
// clc_expand.cuh) and that exponent -- the layout of the first 12 doubles of a split-frame slot.
constexpr int kSegRawDoubles = 12;
// kModePoses: one calibration at many poses (clc_eval_poses, clc_solve_lm_starts) -- every stage is read once and walked once per
// pose of a tile of at most kPoseTile poses, with that pose's frame constants; every piece leaves raw as in kModeSegments, to
// that pose's rows and slots.  A piece that continues past a stage waits in a per-warp, per-pose accumulator that takes the
// place of the tile (12 doubles per pose: 10 moments, cost, exponent).
constexpr int kPoseTile = 32;
static_assert(kPoseTile * kSegRawDoubles <= kTileDoublesPerWarp, "the open pieces of a pose tile live in the warp's tile");
// kModeRange: the extrinsic with the laser's range offset and scale (clc_range_bias.cuh) -- as kModeSegments, with the frame
// constants of SweepArgs::seg_consts, but every point is first moved to kappa p (kappa = 1 + s + b / r, (b, s) = pose7[7], [8]:
// the LM candidate) and every piece leaves kRangeRawDoubles: the 25 RangeMoments, the cost and its exponent.  A split frame's
// pieces go to per-warp head / tail slots of the same width.
constexpr int kRangeMoments = 25;
constexpr int kRangeRawDoubles = kRangeMoments + 2;
enum SweepMode { kModeLM = 0, kModeClosedForm = 1, kModeFrames = 2, kModeSegments = 3, kModePoses = 4, kModeRange = 5 };

// Device-resident problem (read-only for the sweeps).
struct ProblemView {
  const double* x;            // SoA coordinates, zero padded to a multiple of kMaxChunk (+ kMaxChunk)
  const double* y;
  const double* z;
  const double* plane;        // [n_frames*4]   n, d in the camera frame
  const int64_t* offsets;     // [n_frames+1]
  const int* warp_first_frame;  // [total warps of the launch grid] frame containing each warp's first point
  const double* edge_plane;   // [n_edges*4] or nullptr
  const double* edge_pt;      // [n_edges*3]
  int64_t n_frames;
  int64_t n_points;
  int64_t n_edges;            // 2 * n_frames or 0
  int64_t per_warp;           // points per warp (multiple of the kernel family's stage size)
  int resident_chunks;        // LM solves: the last resident_chunks stages of every warp's range are kept in L2 (clc_l2_plan.h)
  double inv_a2;              // 1 / a^2 of the problem's loss
  double a2;                  // a^2
};

struct SweepArgs {
  const double* pose7;        // device pointer: the pose to evaluate
  const int* done;            // device flag: non-zero -> the sweep is a no-op (LM finished); may be nullptr
  unsigned long long* partials_ll;  // [gridDim.x * kMaxOut * 2] block partial sums, every 8-byte word = 32 payload bits +
                                    // the 32-bit sequence number of the launch (no ticket, no fence: see the block reduction)
  double* sums;               // [kMaxOut] result of the launch
  unsigned int* launch_seq;   // sweeps completed on this problem (device counter, bumped by block 0 of every real sweep)
  LmState* lm;                // non-null: the last block also runs lm_update (single-rank fused mode)
  int use_loss;
  int use_edges;
  int l2_hints;               // LM solves only: the bulk copies carry L2 eviction priorities (pv.resident_chunks)
  int loop_sweeps;            // > 1 (LOOP instantiations with a fused LM update only): the kernel runs up to that many LM
                              // iterations by itself -- sweep, reduce, lm_update, next sweep -- instead of one per launch
  unsigned long long* pose_ll;  // [16] looping multi-block grids: block 0 hands the next pose (7 doubles) and the `done` flag to
                                // the other blocks as tagged words (same protocol as partials_ll)
  unsigned long long* timing;  // optional [gridDim.x * 8] globaltimer stamps (profiling hook), nullptr normally;
                               // followed by [gridDim.x * kWarps] per-warp "stream done" stamps
  // fused all-reduce over NVLink peer memory (nranks > 1): every rank's last block stores its sums into every rank's
  // mailbox with a low-latency protocol -- every 8-byte word carries 32 bits of payload and the 32-bit sequence number,
  // 8-byte stores are atomic, so no fence and no separate flag are needed -- then polls its own mailbox and adds the
  // contributions in rank order (identical bits on every rank)
  int nranks;
  int rank;
  unsigned long long* seq_counter;        // device counter of completed exchanges (local to the rank; all ranks agree)
  unsigned long long* peer_mailbox[kMaxRanks];  // peer_mailbox[r]: rank r's mailbox (IPC-mapped),
                                                // [2 parity][nranks source][kMailboxSlot values][2 words]
  int* error;                             // set to 1 on a peer time-out
  // kModeFrames only
  double* frame_rows;   // [n_frames * kRowDoubles] the report rows of the frames that lie in one warp range
  double* frame_slots;  // [total warps * 2 * kSlotDoubles] head / tail pieces of split frames (clc_frames.cuh)
  // kModeSegments only (frame_rows then holds [n_frames * kSegRawDoubles] raw rows; frame_slots as above); kModeRange: rows and
  // slots kRangeRawDoubles wide, and pose7 points at (pose7, b, s)
  const double* seg_consts;  // [(n_frames + n_edges) * 4] m, c of every frame, then of every edge residual, at its segment's pose
  // kModePoses only: pose k's constants at seg_consts + k * pose_consts_stride, its raw rows at frame_rows + k * pose_rows_stride,
  // its slots at frame_slots + k * pose_slots_stride; this launch walks the poses pose_active[pose_tile0 ..
  // min(pose_tile0 + kPoseTile, *pose_count))
  const int* pose_active;
  const int* pose_count;
  int pose_tile0;
  int64_t pose_consts_stride;
  int64_t pose_rows_stride;
  int64_t pose_slots_stride;
};

// ---- small device helpers ---------------------------------------------------------------------------------

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#define CLC_STAMP(slot)                                                                       \
  do {                                                                                        \
    if (args.timing != nullptr && threadIdx.x == 0) args.timing[(int64_t)blockIdx.x * 8 + (slot)] = globaltimer_ns(); \
  } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!done);
}
// 1-D bulk async copy global -> shared (TMA engine, SASS UBLKCP); completion is signalled on `bar` in bytes
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// the same copy with an L2 eviction priority for the lines it reads (a policy made by createpolicy)
__device__ __forceinline__ void bulk_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
               : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

__device__ __forceinline__ void st_relaxed_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// 16-byte store / load of two tagged words (each word carries its own tag, so the pair need not be atomic)
__device__ __forceinline__ void st_volatile_v2(unsigned long long* p, unsigned long long a, unsigned long long b) {
  asm volatile("st.volatile.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}
__device__ __forceinline__ void ld_volatile_v2(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
  asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}

__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// gpu-scope acq_rel fetch-add: releases this block's partial sums (ordered before it by the preceding block barrier)
// and acquires the other blocks' when it turns out to be the last ticket
__device__ __forceinline__ unsigned int atom_add_acq_rel_gpu(unsigned int* p, unsigned int v) {
  unsigned int old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}

// 1/a for a normal, positive a: MUFU.RCP64H seed (2^-23 relative) + two Newton steps (-> ~1 ulp).
__device__ __forceinline__ double rcp_pos(double a) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(a));
  double e = fma(-a, r, 1.0);
  r = fma(r, e, r);
  e = fma(-a, r, 1.0);
  r = fma(r, e, r);
  return r;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Transposing butterfly: on entry every lane holds N values v[0..N); on exit lane L holds, in v[0], the sum over all
// 32 lanes of slot (L mod N).  N + log2(32/N) - 1 shuffles instead of 5 N, in a fixed (deterministic) order.
template <int N>
__device__ __forceinline__ void warp_transpose_sum(double* v, int lane) {
#pragma unroll
  for (int half = N / 2; half >= 1; half >>= 1) {
    const bool upper = (lane & half) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      const double keep = upper ? v[i + half] : v[i];
      const double send = upper ? v[i] : v[i + half];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, half);
    }
  }
#pragma unroll
  for (int o = N; o < 32; o <<= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
}

// warp_transpose_sum with every round a template instance: the trip counts are compile-time constants, so the rounds unroll
// completely and v stays in registers (warp_transpose_sum's loop over a shifted bound is not fully unrolled, which sends v to
// local memory).  kModeSegments uses it so that nothing goes through local memory in the streaming loop.
template <int HALF>
__device__ __forceinline__ void transpose_round(double* v, int lane) {
  const bool upper = (lane & HALF) != 0;
#pragma unroll
  for (int i = 0; i < HALF; ++i) {
    const double keep = upper ? v[i + HALF] : v[i];
    const double send = upper ? v[i] : v[i + HALF];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, HALF);
  }
  if constexpr (HALF > 1) transpose_round<HALF / 2>(v, lane);
}
template <int N>
__device__ __forceinline__ void warp_transpose_sum_regs(double* v, int lane) {
  transpose_round<N / 2>(v, lane);
#pragma unroll
  for (int o = N; o < 32; o <<= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
}

// Per-lane streaming accumulators of one piece.
struct Moments {
  double S0, Sx, Sy, Sz, Sxx, Sxy, Sxz, Syy, Syz, Szz;
  double prod;  // Cauchy: running product of (1 + e^2/a^2), mantissa kept in [1,2); other kinds: running sum of rho~(e)
  int esum;     // exponent taken out of prod
};

template <int LOSS>
__device__ __forceinline__ void moments_clear(Moments& a) {
  a.S0 = a.Sx = a.Sy = a.Sz = a.Sxx = a.Sxy = a.Sxz = a.Syy = a.Syz = a.Szz = 0.0;
  a.prod = LOSS == kLossCauchy ? 1.0 : 0.0;
  a.esum = 0;
}

// PLANAR: every z of the problem is exactly 0 (a 2-D laser: reference utilities.cpp:207), so the z stream is neither
// stored nor read and the four z moments stay exactly 0 -- every per-point term is bit-identical to the general path.
template <bool PLANAR>
__device__ __forceinline__ void accumulate(Moments& a, double w, double x, double y, double z) {
  const double wx = w * x, wy = w * y;
  a.S0 += w;
  a.Sx += wx; a.Sy += wy;
  a.Sxx = fma(wx, x, a.Sxx); a.Sxy = fma(wx, y, a.Sxy);
  a.Syy = fma(wy, y, a.Syy);
  if (!PLANAR) {
    const double wz = w * z;
    a.Sz += wz;
    a.Sxz = fma(wx, z, a.Sxz); a.Syz = fma(wy, z, a.Syz); a.Szz = fma(wz, z, a.Szz);
  }
}

// The robust weights w0, w1 of two residuals e0, e1 (v0/v1: validity of the two points; an invalid point gets w = 0) and their
// cost terms added to prod (Cauchy: multiplied into it), with process2's arithmetic operation for operation.  LOSS: LossKind
// (clc_expand.cuh); COST: the no-loss kind also sums e^2.  ha: the loss parameter (Huber only), a2 = ha^2.  (process2 keeps its
// own inline copy: calling this from it changes the SASS of its no-loss and soft-L1 instantiations.)
template <int LOSS, bool COST>
__device__ __forceinline__ void weigh2(double& prod, double e0, double e1, bool v0, bool v1, double inv_a2, double ha, double a2,
                                       double& w0, double& w1) {
  if (LOSS == kLossHuber) {
    // w = a / max(|e|, a): one reciprocal of the product of the two denominators serves both weights (a NaN e stays NaN)
    const double ae0 = fabs(e0), ae1 = fabs(e1);
    double d0 = ae0 < ha ? ha : ae0, d1 = ae1 < ha ? ha : ae1;
    d0 = v0 ? d0 : ha;
    d1 = v1 ? d1 : ha;
    const double ar = ha * rcp_pos(d0 * d1);
    w0 = ar * d1;
    w1 = ar * d0;
    w0 = v0 ? w0 : 0.0;
    w1 = v1 ? w1 : 0.0;
    // rho~ = e^2 inside a, 2 a |e| - a^2 outside: summed directly, like e^2 without a loss
    const double r0 = ae0 <= ha ? e0 * e0 : fma(2.0 * ha, ae0, -a2);
    const double r1 = ae1 <= ha ? e1 * e1 : fma(2.0 * ha, ae1, -a2);
    prod += v0 ? r0 : 0.0;
    prod += v1 ? r1 : 0.0;
  } else if (LOSS == kLossSoftL1) {
    // w = 1/sqrt(u), u = 1 + e^2/a^2; rho~ = 2 e^2 / (1 + sqrt(u)) with sqrt(u) = u w -- one reciprocal for both points
    double u0 = fma(e0 * inv_a2, e0, 1.0);
    double u1 = fma(e1 * inv_a2, e1, 1.0);
    u0 = v0 ? u0 : 1.0;
    u1 = v1 ? u1 : 1.0;
    const double y0 = rsqrt(u0), y1 = rsqrt(u1);
    const double t0 = fma(u0, y0, 1.0), t1 = fma(u1, y1, 1.0);
    const double r = rcp_pos(t0 * t1);
    const double r0 = (2.0 * e0) * e0 * (r * t1), r1 = (2.0 * e1) * e1 * (r * t0);
    prod += v0 ? r0 : 0.0;
    prod += v1 ? r1 : 0.0;
    w0 = v0 ? y0 : 0.0;
    w1 = v1 ? y1 : 0.0;
  } else if (LOSS == kLossCauchy) {
    double u0 = fma(e0 * inv_a2, e0, 1.0);
    double u1 = fma(e1 * inv_a2, e1, 1.0);
    u0 = v0 ? u0 : 1.0;
    u1 = v1 ? u1 : 1.0;
    // batch inversion: one reciprocal of u0*u1 serves both weights and the cost product
    const double p = u0 * u1;
    const double r = rcp_pos(p);
    w0 = r * u1;
    w1 = r * u0;
    w0 = v0 ? w0 : 0.0;
    w1 = v1 ? w1 : 0.0;
    prod *= p;
  } else {
    if (COST) {
      prod = fma(v0 ? e0 : 0.0, e0, prod);
      prod = fma(v1 ? e1 : 0.0, e1, prod);
    }
    w0 = v0 ? 1.0 : 0.0;
    w1 = v1 ? 1.0 : 0.0;
  }
}

// Two points (one LDG.128 per coordinate array).  v0/v1: validity of the two points.  LOSS: LossKind (clc_expand.cuh); COST:
// the no-loss kind also sums e^2 (the other kinds always sum their cost term).  a: the loss parameter (Huber only), a2 = a^2.
template <int LOSS, bool COST, bool PLANAR>
__device__ __forceinline__ void process2(Moments& a, const double2 X, const double2 Y, const double2 Z, bool v0,
                                         bool v1, double m0, double m1, double m2, double c, double inv_a2, double ha = 0.0,
                                         double a2 = 0.0) {
  // fma(m2, 0, c) == c exactly for finite m2, so the planar form rounds like the general one
  const double e0 = fma(m0, X.x, fma(m1, Y.x, PLANAR ? c : fma(m2, Z.x, c)));
  const double e1 = fma(m0, X.y, fma(m1, Y.y, PLANAR ? c : fma(m2, Z.y, c)));
  if (LOSS == kLossHuber) {
    // w = a / max(|e|, a): one reciprocal of the product of the two denominators serves both weights (a NaN e stays NaN)
    const double ae0 = fabs(e0), ae1 = fabs(e1);
    double d0 = ae0 < ha ? ha : ae0, d1 = ae1 < ha ? ha : ae1;
    d0 = v0 ? d0 : ha;
    d1 = v1 ? d1 : ha;
    const double ar = ha * rcp_pos(d0 * d1);
    double w0 = ar * d1, w1 = ar * d0;
    w0 = v0 ? w0 : 0.0;
    w1 = v1 ? w1 : 0.0;
    // rho~ = e^2 inside a, 2 a |e| - a^2 outside: summed directly, like e^2 without a loss
    const double r0 = ae0 <= ha ? e0 * e0 : fma(2.0 * ha, ae0, -a2);
    const double r1 = ae1 <= ha ? e1 * e1 : fma(2.0 * ha, ae1, -a2);
    a.prod += v0 ? r0 : 0.0;
    a.prod += v1 ? r1 : 0.0;
    accumulate<PLANAR>(a, w0, X.x, Y.x, Z.x);
    accumulate<PLANAR>(a, w1, X.y, Y.y, Z.y);
  } else if (LOSS == kLossSoftL1) {
    // w = 1/sqrt(u), u = 1 + e^2/a^2; rho~ = 2 e^2 / (1 + sqrt(u)) with sqrt(u) = u w -- one reciprocal for both points
    double u0 = fma(e0 * inv_a2, e0, 1.0);
    double u1 = fma(e1 * inv_a2, e1, 1.0);
    u0 = v0 ? u0 : 1.0;
    u1 = v1 ? u1 : 1.0;
    const double y0 = rsqrt(u0), y1 = rsqrt(u1);
    const double t0 = fma(u0, y0, 1.0), t1 = fma(u1, y1, 1.0);
    const double r = rcp_pos(t0 * t1);
    const double r0 = (2.0 * e0) * e0 * (r * t1), r1 = (2.0 * e1) * e1 * (r * t0);
    a.prod += v0 ? r0 : 0.0;
    a.prod += v1 ? r1 : 0.0;
    accumulate<PLANAR>(a, v0 ? y0 : 0.0, X.x, Y.x, Z.x);
    accumulate<PLANAR>(a, v1 ? y1 : 0.0, X.y, Y.y, Z.y);
  } else if (LOSS == kLossCauchy) {
    double u0 = fma(e0 * inv_a2, e0, 1.0);
    double u1 = fma(e1 * inv_a2, e1, 1.0);
    u0 = v0 ? u0 : 1.0;
    u1 = v1 ? u1 : 1.0;
    // batch inversion: one reciprocal of u0*u1 serves both weights and the cost product
    const double p = u0 * u1;
    const double r = rcp_pos(p);
    double w0 = r * u1, w1 = r * u0;
    w0 = v0 ? w0 : 0.0;
    w1 = v1 ? w1 : 0.0;
    a.prod *= p;
    accumulate<PLANAR>(a, w0, X.x, Y.x, Z.x);
    accumulate<PLANAR>(a, w1, X.y, Y.y, Z.y);
  } else {
    if (COST) {
      a.prod = fma(v0 ? e0 : 0.0, e0, a.prod);
      a.prod = fma(v1 ? e1 : 0.0, e1, a.prod);
    }
    accumulate<PLANAR>(a, v0 ? 1.0 : 0.0, X.x, Y.x, Z.x);
    accumulate<PLANAR>(a, v1 ? 1.0 : 0.0, X.y, Y.y, Z.y);
  }
}

// kModeRange: the moments of a piece in the augmented vector a = (p, p/r, 1), r = |p| (clc_range_bias.cuh): Moments' 10
// (1, p, p p^T), then p/r, p p^T / r and p p^T / r^2 -- 25 in all, 14 of them non-zero on a planar problem.
struct RangeMoments : Moments {
  double Qx, Qy, Qz;                          // sum w p / r
  double Pxx, Pxy, Pxz, Pyy, Pyz, Pzz;        // sum w p p^T / r
  double P2xx, P2xy, P2xz, P2yy, P2yz, P2zz;  // sum w p p^T / r^2
};

template <int LOSS>
__device__ __forceinline__ void moments_clear(RangeMoments& a) {
  moments_clear<LOSS>(static_cast<Moments&>(a));
  a.Qx = a.Qy = a.Qz = 0.0;
  a.Pxx = a.Pxy = a.Pxz = a.Pyy = a.Pyz = a.Pzz = 0.0;
  a.P2xx = a.P2xy = a.P2xz = a.P2yy = a.P2yz = a.P2zz = 0.0;
}

// One point's share of the range moments: w, w / r, w / r^2 on the three blocks (inv_r = 1 / r, 0 at r == 0)
template <bool PLANAR>
__device__ __forceinline__ void accumulate_range(RangeMoments& a, double w, double inv_r, double x, double y, double z) {
  accumulate<PLANAR>(a, w, x, y, z);
  const double wr = w * inv_r, wrr = wr * inv_r;
  const double rx = wr * x, ry = wr * y, qx = wrr * x, qy = wrr * y;
  a.Qx += rx; a.Qy += ry;
  a.Pxx = fma(rx, x, a.Pxx); a.Pxy = fma(rx, y, a.Pxy); a.Pyy = fma(ry, y, a.Pyy);
  a.P2xx = fma(qx, x, a.P2xx); a.P2xy = fma(qx, y, a.P2xy); a.P2yy = fma(qy, y, a.P2yy);
  if (!PLANAR) {
    const double rz = wr * z, qz = wrr * z;
    a.Qz += rz;
    a.Pxz = fma(rx, z, a.Pxz); a.Pyz = fma(ry, z, a.Pyz); a.Pzz = fma(rz, z, a.Pzz);
    a.P2xz = fma(qx, z, a.P2xz); a.P2yz = fma(qy, z, a.P2yz); a.P2zz = fma(qz, z, a.P2zz);
  }
}

// 1 / r of a point with r^2 = x^2 + y^2 + z^2: one FP64 reciprocal square root; 0 at r == 0 (the p / r terms of the origin are
// 0), NaN for a NaN coordinate
__device__ __forceinline__ double range_inv_r(double x, double y, double z) {
  const double r2 = fma(x, x, fma(y, y, z * z));
  return r2 == 0.0 ? 0.0 : rsqrt(r2);
}

// kModeRange's process2: the same two points at the corrected positions kappa p, kappa = sigma + b / r (sigma = 1 + s), so
// e = kappa (m.p) + c.  Every residual of the loss is weighed as process2 weighs it (weigh2, COST = true).
template <int LOSS, bool PLANAR>
__device__ __forceinline__ void process2_range(RangeMoments& a, const double2 X, const double2 Y, const double2 Z, bool v0, bool v1,
                                               double m0, double m1, double m2, double c, double sigma, double b, double inv_a2,
                                               double ha, double a2) {
  const double ir0 = range_inv_r(X.x, Y.x, PLANAR ? 0.0 : Z.x);
  const double ir1 = range_inv_r(X.y, Y.y, PLANAR ? 0.0 : Z.y);
  const double y0 = fma(m0, X.x, fma(m1, Y.x, PLANAR ? 0.0 : m2 * Z.x));
  const double y1 = fma(m0, X.y, fma(m1, Y.y, PLANAR ? 0.0 : m2 * Z.y));
  const double e0 = fma(fma(b, ir0, sigma), y0, c);
  const double e1 = fma(fma(b, ir1, sigma), y1, c);
  double w0, w1;
  weigh2<LOSS, true>(a.prod, e0, e1, v0, v1, inv_a2, ha, a2, w0, w1);
  accumulate_range<PLANAR>(a, w0, ir0, X.x, Y.x, Z.x);
  accumulate_range<PLANAR>(a, w1, ir1, X.y, Y.y, Z.y);
}

__device__ __forceinline__ void renormalise(Moments& a) {
  // prod >= 1: move its binary exponent into esum (exact)
  const int hi = __double2hiint(a.prod);
  const int ex = (hi >> 20) - 1023;
  a.esum += ex;
  a.prod = __hiloint2double(hi - (ex << 20), __double2loint(a.prod));
}

// kModeFrames: the unweighted per-point statistics of a piece, next to its Moments (per lane)
struct FrameSums {
  double se, se2, emax;  // sum e, sum e^2, max |e| (NaN kept) of the raw distances
};

__device__ __forceinline__ void frame_sums_clear(FrameSums& s) { s.se = s.se2 = s.emax = 0.0; }

// the same two points as process2 (the same e, rounded the same way)
template <bool PLANAR>
__device__ __forceinline__ void frame_sums2(FrameSums& s, const double2 X, const double2 Y, const double2 Z, bool v0, bool v1,
                                            double m0, double m1, double m2, double c) {
  const double e0 = fma(m0, X.x, fma(m1, Y.x, PLANAR ? c : fma(m2, Z.x, c)));
  const double e1 = fma(m0, X.y, fma(m1, Y.y, PLANAR ? c : fma(m2, Z.y, c)));
  const double d0 = v0 ? e0 : 0.0, d1 = v1 ? e1 : 0.0;
  s.se += d0;
  s.se += d1;
  s.se2 = fma(d0, d0, s.se2);
  s.se2 = fma(d1, d1, s.se2);
  s.emax = nan_max(s.emax, fabs(d0));
  s.emax = nan_max(s.emax, fabs(d1));
}

// Expands the summed pieces of frame f into its report row (clc_frames.cuh layout): S = the 10 weighted moments, cost_term as
// expand_lm takes it, se / se2 / emax the unweighted statistics of its n points.  The frame's two edge residuals (edges) are
// expanded exactly as K1's edge tail does and added to the row.
__device__ __forceinline__ void frame_row_write(const ProblemView& pv, const PoseConsts& pc, int64_t f, int64_t n, const double* S,
                                                double cost_term, double se, double se2, double emax, int loss, bool edges,
                                                double* row) {
  double plane[4], m[3], c;
#pragma unroll
  for (int k = 0; k < 4; ++k) plane[k] = pv.plane[f * 4 + k];
  frame_consts(pc, plane, m, &c);
  const double s2 = 1.0 / (double)(pv.offsets[f + 1] - pv.offsets[f]);
  double out[kNumSums];
#pragma unroll
  for (int k = 0; k < kNumSums; ++k) out[k] = 0.0;
  expand_lm(plane, m, c, s2, S, loss, cost_term, pv.a2, out);
  double ee[2] = {0.0, 0.0};
  if (edges) {
#pragma unroll
    for (int k = 0; k < 2; ++k)
      ee[k] = edge_residual(pc, pv.edge_plane + (2 * f + k) * 4, pv.edge_pt + (2 * f + k) * 3, s2, loss, pv.a2, pv.inv_a2, out);
  }
  const double dn = (double)n;
  row[kRowN] = __longlong_as_double(n);
  row[kRowCost] = out[27];
  row[kRowChi] = s2 * se2;
  row[kRowMeanE] = se / dn;
  row[kRowRmsE] = sqrt(se2 / dn);
  row[kRowMaxE] = emax;
  row[kRowMeanW] = S[0] / dn;
  row[kRowEdgeE] = ee[0];
  row[kRowEdgeE + 1] = ee[1];
#pragma unroll
  for (int k = 0; k < 21; ++k) row[kRowH + k] = out[k];
#pragma unroll
  for (int k = 0; k < 6; ++k) row[kRowG + k] = out[21 + k];
}

// ---- K1: the fused sweep -------------------------------------------------------------------------------------
//
// Work decomposition: the P points are cut into equal contiguous ranges (a multiple of 128 points), one per warp of
// a grid that fills the machine exactly once (persistent: SM count x resident blocks).  Every warp owns a private
// 2-stage ring in shared memory that the TMA engine fills with 1 KiB bulk copies (cp.async.bulk, one per coordinate
// array and stage; completion on an mbarrier), so ~6 KiB per warp / ~96 KiB per SM are in flight regardless of
// register pressure and independent of the frame bookkeeping.  The warp consumes a stage with conflict-free 128-bit
// shared loads (4 points per lane), walks the frame pieces that overlap the stage, and keeps 10 weighted moments
// plus the running cost product per lane in registers.  When a frame ends, the lanes' moments are summed by warp
// shuffles and parked in a shared-memory tile; every 32 pieces (and at the end) the tile is expanded -- one piece
// per lane -- into the 28 normal-equation sums, which are shuffle-reduced into the warp's accumulator.  Block
// partials go to global memory; the last block to finish (ticket) adds them in a fixed order, so the result is
// bit-reproducible from run to run, and optionally runs the LM update.
// LOOP: the instantiation for single-block grids that runs the whole LM loop inside one launch (args.loop_sweeps sweeps at
// most); kept apart so that the streaming instantiations do not carry the loop's bookkeeping in registers.
// LOSS: the loss kind (LossKind, clc_expand.cuh).
template <int LOSS, int MODE, bool PLANAR, bool LOOP = false>
__global__ void __launch_bounds__(kThreads, kBlocksPerSM)
clc_sweep_kernel(ProblemView pv, SweepArgs args) {
  constexpr int NOUT = (MODE == kModeClosedForm) ? kMaxOut : kNumSums;
  // planar: two coordinate streams per stage; stages of kPlanarChunk points keep the bytes in flight per warp the same
  constexpr int NST = PLANAR ? kPlanarStages : kStages;
  constexpr int CH = PLANAR ? kPlanarChunk : kChunk;  // points per stage
  constexpr int G = CH / 64;
  constexpr int SST = (PLANAR ? 2 : 3) * CH;  // doubles per stage
  constexpr int RING = NST * SST;  // doubles per warp
  static_assert(RING == ring_doubles_per_warp(PLANAR), "ring size");
  extern __shared__ __align__(128) unsigned char s_dyn[];
  __shared__ double s_acc[kWarps][NOUT];
  __shared__ double s_red[kWarps][32];
  __shared__ unsigned long long s_core[kLmCoreWords];  // block 0: the hot LM state
  __shared__ double s_next[8];                           // looping grids: pose of the next sweep + the `done` flag
  __shared__ int s_prog[32];                             // stages finished by every warp (soft lockstep)

  CLC_STAMP(0);
  if (args.timing != nullptr && threadIdx.x == 0) {
    unsigned int smid;
    asm volatile("mov.u32 %0, %smid;" : "=r"(smid));
    args.timing[(int64_t)blockIdx.x * 8 + 7] = smid;
  }

  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int64_t gwarp = (int64_t)blockIdx.x * kWarps + warp;

  // ---- this warp's range and ring; start the copies before anything else (they do not depend on the pose) ----
  const int64_t P = pv.n_points;
  int64_t p0 = gwarp * pv.per_warp;
  if (p0 > P) p0 = P;
  int64_t p1 = p0 + pv.per_warp;
  if (p1 > P) p1 = P;
  const int n_chunks = (int)((p1 - p0 + CH - 1) / CH);
  double* ring = reinterpret_cast<double*>(s_dyn) + warp * RING;
  double* tile = reinterpret_cast<double*>(s_dyn) + kWarps * RING + warp * kTileDoublesPerWarp;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_dyn + (size_t)kWarps * (RING + kTileDoublesPerWarp) * 8) + warp * kBarsPerWarp;
  // kModeFrames: sum e, sum e^2, max |e| of every parked piece (tile row r -> ftile[3 r ..])
  double* ftile = reinterpret_cast<double*>(s_dyn + dyn_smem_bytes(PLANAR)) + warp * kFrameTileDoublesPerWarp;

  // Stage slots and mbarrier phases follow a running count of issued stages (`issued`, kept by every lane), so that a kernel
  // that loops over several sweeps (loop_sweeps > 1) keeps prefetching across the reduce + LM update between two sweeps.
  const int sweeps_max = (LOOP && args.loop_sweeps > 1 && MODE == kModeLM && args.lm != nullptr) ? args.loop_sweeps : 1;
  const int total_chunks = LOOP ? sweeps_max * n_chunks : n_chunks;
  int issued = 0, next_c = 0;  // next_c == issued mod n_chunks
  // L2 residency during LM solves: every sweep reads the same bytes in the same order.  The last resident_chunks stages of the
  // range are read with evict_last and stay in L2 from one sweep to the next; all other stages are read with evict_first, so
  // that the stream does not push the resident share out.  The last stages, because the warps that finish late (the
  // straggler tail, one or two stages in flight) then read from L2.  Only the eviction priority changes, not the arithmetic.
  const bool l2_hints = args.l2_hints != 0 && pv.resident_chunks > 0;
  auto issue_one = [&](bool slot_was_read) {
    if (lane == 0) {
      const int c = LOOP ? next_c : issued, st = issued % NST;
      double* dst = ring + st * SST;
      // always a whole stage (the arrays are zero padded beyond the last point; the ranges are whole stages)
      const int64_t src = p0 + (int64_t)c * CH;  // multiple of the stage size -> 1 KiB aligned
      if (slot_was_read) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      mbar_expect_tx(bars + st, (PLANAR ? 2 : 3) * CH * 8);
      if (l2_hints) {
        const uint64_t pol = c >= n_chunks - pv.resident_chunks ? policy_evict_last() : policy_evict_first();
        bulk_g2s_hint(dst, pv.x + src, CH * 8, bars + st, pol);
        bulk_g2s_hint(dst + CH, pv.y + src, CH * 8, bars + st, pol);
        if (!PLANAR) bulk_g2s_hint(dst + 2 * CH, pv.z + src, CH * 8, bars + st, pol);
      } else {
        bulk_g2s(dst, pv.x + src, CH * 8, bars + st);
        bulk_g2s(dst + CH, pv.y + src, CH * 8, bars + st);
        if (!PLANAR) bulk_g2s(dst + 2 * CH, pv.z + src, CH * 8, bars + st);
      }
    }
    ++issued;
    if (LOOP && ++next_c == n_chunks) next_c = 0;
  };
  // waits for the stages that are still in flight (g = first stage not yet consumed): a block must not exit before its bulk
  // copies have landed
  auto drain = [&](int g) {
    for (; g < issued; ++g) mbar_wait(bars + g % NST, (uint32_t)(g / NST) & 1u);
  };
  if (lane == 0) {
#pragma unroll
    for (int st = 0; st < NST; ++st) mbar_init(bars + st, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();
  // kModePoses: a tile with no running pose reads no point (the list of running poses is final before the launch: no PDL)
  int first_issue = total_chunks;
  if constexpr (MODE == kModePoses) {
    if (*args.pose_count <= args.pose_tile0) first_issue = 0;
  }
  for (int g = 0; g < NST && g < first_issue; ++g) issue_one(false);
  __syncwarp();

  // Programmatic dependent launch: everything above touched only constant data (the points), so it overlaps the
  // tail of the previous sweep (final reduce + LM update on its block 0).  From here on the pose, the `done` flag,
  // the partial sums and the ticket of the previous launch are needed: wait for it to complete.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (args.done != nullptr && (*args.done != 0 || (args.error != nullptr && *args.error != 0))) {
    // the LM finished (or an earlier sweep of this solve lost a peer): nothing to do, but the bulk copies already in flight must land before the block may exit
    drain(0);
    return;
  }

  if constexpr (MODE == kModePoses) {
    const int t1 = min(*args.pose_count, args.pose_tile0 + kPoseTile);
    const int nt = t1 - args.pose_tile0;
    if (nt <= 0 || n_chunks == 0) {  // no pose of this tile is running (or no points in this range)
      drain(0);
      return;
    }
    // the open piece of every pose of the tile: lane L < 12 keeps value L of it
    double* open = tile;
    for (int j = 0; j < nt; ++j)
      if (lane < kSegRawDoubles) open[j * kSegRawDoubles + lane] = (LOSS == kLossCauchy && lane == 10) ? 1.0 : 0.0;
    __syncwarp();
    const double huber_a = LOSS == kLossHuber ? sqrt(pv.a2) : 0.0;
    // adds this lane's share of one piece of pose j to its open piece: the lanes' moments are summed across the warp (and the
    // Cauchy products multiplied), so the sum of a piece does not depend on how many poses share the stage
    auto fold = [&](const Moments& a, int j) {
      double v[16] = {a.S0, a.Sx, a.Sy, a.Sz, a.Sxx, a.Sxy, a.Sxz, a.Syy, a.Syz, a.Szz, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      double pr = a.prod;
      int es = a.esum;
      if (LOSS == kLossCauchy) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          pr *= __shfl_xor_sync(0xffffffffu, pr, o);  // 32 mantissas in [1,2): product < 2^32
          es += __shfl_xor_sync(0xffffffffu, es, o);
        }
      } else {
        v[10] = pr;
      }
      warp_transpose_sum_regs<16>(v, lane);
      double* o = open + j * kSegRawDoubles;
      if (lane < 10 || (LOSS != kLossCauchy && lane == 10)) o[lane] += v[0];
      if (LOSS == kLossCauchy && lane == 10) {
        Moments m;
        m.prod = o[10] * pr;  // [1,2) x [1, 2^32): exact exponent bookkeeping as renormalise does
        m.esum = (int)o[11] + es;
        renormalise(m);
        o[10] = m.prod;
        o[11] = (double)m.esum;
      }
    };
    // the open piece of frame f of pose k leaves raw, as kModeSegments' pieces do, and the accumulator starts afresh
    auto emit = [&](int j, int k, int64_t f, int64_t f_end) {
      const int kind = frame_piece_kind(pv.offsets[f], f_end, p0, p1);
      double* dst = kind == kPieceWhole ? args.frame_rows + k * args.pose_rows_stride + f * kSegRawDoubles
                                        : args.frame_slots + k * args.pose_slots_stride +
                                              (gwarp * 2 + (kind == kPieceHead ? kSlotHead : kSlotTail)) * kSlotDoubles;
      double* o = open + j * kSegRawDoubles;
      __syncwarp();  // lane 10 of fold wrote the exponent that lane 11 reads here
      if (lane < kSegRawDoubles) {
        dst[lane] = o[lane];
        o[lane] = (LOSS == kLossCauchy && lane == 10) ? 1.0 : 0.0;
      }
      __syncwarp();
    };
    int64_t f = pv.warp_first_frame[gwarp];
    int64_t f_end = pv.offsets[f + 1];
    for (int ch = 0; ch < n_chunks; ++ch) {
      const int st = ch % NST;
      const int64_t cb = p0 + (int64_t)ch * CH;
      const int64_t ce = (cb + CH < p1) ? cb + CH : p1;
      mbar_wait(bars + st, (uint32_t)(ch / NST) & 1u);
      const double* sx = ring + st * SST;
      double2 X[G], Y[G], Z[G];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        X[g] = *reinterpret_cast<const double2*>(sx + 64 * g + 2 * lane);
        Y[g] = *reinterpret_cast<const double2*>(sx + CH + 64 * g + 2 * lane);
        Z[g] = PLANAR ? make_double2(0.0, 0.0) : *reinterpret_cast<const double2*>(sx + 2 * CH + 64 * g + 2 * lane);
      }
      const int64_t f_stage = f, f_end_stage = f_end;
      for (int j = 0; j < nt; ++j) {
        const int k = args.pose_active[args.pose_tile0 + j];
        const double* kc = args.seg_consts + k * args.pose_consts_stride;
        f = f_stage;
        f_end = f_end_stage;
        int64_t q = cb;
        while (q < ce) {
          while (f_end <= q) f_end = pv.offsets[++f + 1];  // next non-empty frame
          const double m0 = kc[f * 4], m1 = kc[f * 4 + 1], m2 = kc[f * 4 + 2], c = kc[f * 4 + 3];
          const int64_t hi = f_end < ce ? f_end : ce;
          Moments a;
          moments_clear<LOSS>(a);
          if (q == cb && hi == cb + CH) {
#pragma unroll
            for (int g = 0; g < G; ++g)
              process2<LOSS, true, PLANAR>(a, X[g], Y[g], Z[g], true, true, m0, m1, m2, c, pv.inv_a2, huber_a, pv.a2);
          } else {
#pragma unroll
            for (int g = 0; g < G; ++g) {
              // as kModeSegments: the points outside the piece are replaced before any arithmetic
              const int64_t i0 = cb + 64 * g + 2 * lane;
              const bool v0 = i0 >= q && i0 < hi, v1 = i0 + 1 >= q && i0 + 1 < hi;
              const double2 Xm = make_double2(v0 ? X[g].x : 0.0, v1 ? X[g].y : 0.0);
              const double2 Ym = make_double2(v0 ? Y[g].x : 0.0, v1 ? Y[g].y : 0.0);
              const double2 Zm = make_double2(v0 ? Z[g].x : 0.0, v1 ? Z[g].y : 0.0);
              process2<LOSS, true, PLANAR>(a, Xm, Ym, Zm, v0, v1, m0, m1, m2, c, pv.inv_a2, huber_a, pv.a2);
            }
          }
          if (LOSS == kLossCauchy) renormalise(a);
          fold(a, j);
          q = hi;
          if (hi == f_end) emit(j, k, f, f_end);
        }
      }
      __syncwarp();
      if (issued < total_chunks) issue_one(true);
    }
    // the last frame continues in the next warp's range: its piece leaves as this warp's tail (or head) slot
    if (f_end > p1)
      for (int j = 0; j < nt; ++j) emit(j, args.pose_active[args.pose_tile0 + j], f, f_end);
    return;
  }

  // sequence number of the first sweep of this launch (the previous sweep on this problem has completed: griddepcontrol.wait)
  const unsigned int launch_tag0 = *args.launch_seq + 1u;  // (plain load: one L2 request per SM, see the pose below)
  // block 0 runs the LM update: its state is fetched now, far away from the critical tail
  if (MODE == kModeLM && args.lm != nullptr && blockIdx.x == 0) {
    const unsigned long long* g_core = reinterpret_cast<const unsigned long long*>(&args.lm->core);
    for (int k = threadIdx.x; k < kLmCoreWords; k += kThreads) s_core[k] = __ldcg(g_core + k);
  }

  PoseConsts pc;
  int n_tile = 0;

  // expands the parked pieces (one per lane) and folds them into the warp accumulator
  auto flush_tile = [&]() {
    double out[NOUT];
#pragma unroll
    for (int k = 0; k < NOUT; ++k) out[k] = 0.0;
    __syncwarp();
    if (lane < n_tile) {
      const double* row = tile + lane * kTileStride;
      const int64_t f = __double_as_longlong(row[12]);
      double plane[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) plane[k] = pv.plane[f * 4 + k];
      if (MODE == kModeLM) {
        double m[3], c;
        frame_consts(pc, plane, m, &c);
        const double cnt = (double)(pv.offsets[f + 1] - pv.offsets[f]);
        double cost_term = row[10];  // other kinds: sum rho~(e)
        if (LOSS == kLossCauchy) cost_term = log(row[10]) + row[11] * 0.693147180559945309417232121458;
        expand_lm(plane, m, c, 1.0 / cnt, row, LOSS, cost_term, pv.a2, out);
      } else {
        expand_closed_form(plane, row, out);
      }
    }
    {
      // lane L ends up with the warp total of output L (and of output 32 + L in the 54-wide closed-form mode)
      double v[32];
#pragma unroll
      for (int k = 0; k < 32; ++k) v[k] = (k < NOUT) ? out[k] : 0.0;
      warp_transpose_sum<32>(v, lane);
      if (lane < NOUT) s_acc[warp][lane] += v[0];
      if (NOUT > 32) {
#pragma unroll
        for (int k = 0; k < 32; ++k) v[k] = (32 + k < NOUT) ? out[(32 + k < NOUT) ? 32 + k : 0] : 0.0;
        warp_transpose_sum<32>(v, lane);
        if (32 + lane < NOUT) s_acc[warp][32 + lane] += v[0];
      }
    }
    __syncwarp();
    n_tile = 0;
  };

  // kModeFrames: expands the parked whole frames (one per lane) straight into their report rows -- no warp reduction
  auto flush_frames = [&]() {
    __syncwarp();
    if (lane < n_tile) {
      const double* row = tile + lane * kTileStride;
      const double* rx = ftile + lane * 3;
      const int64_t f = __double_as_longlong(row[12]);
      // no loss: the frame's sum e^2 (the sweep does not accumulate it twice); Huber / soft-L1: the summed rho~(e)
      const double cost_term = LOSS == kLossCauchy ? log(row[10]) + row[11] * 0.693147180559945309417232121458
                               : LOSS == kLossNone ? rx[1] : row[10];
      frame_row_write(pv, pc, f, pv.offsets[f + 1] - pv.offsets[f], row, cost_term, rx[0], rx[1], rx[2], LOSS,
                      args.use_edges && pv.n_edges > 0, args.frame_rows + f * kRowDoubles);
    }
    __syncwarp();
    n_tile = 0;
  };

  int gc_base = 0;
  for (int sw = 0;; ++sw) {  // one pass per sweep (exactly one unless the kernel loops the LM by itself)
  const unsigned int launch_tag = LOOP ? launch_tag0 + (unsigned int)sw : launch_tag0;
  for (int k = lane; k < NOUT; k += 32) s_acc[warp][k] = 0.0;
  {
    double pose[7];
#pragma unroll
    // plain (L1-cached) loads: every warp of the grid reads the same 56 bytes -- one L2 request per SM instead of one per warp (L1 is
    // invalidated at every kernel launch, so the pose written by the previous sweep's block 0 is what arrives)
    for (int i = 0; i < 7; ++i) pose[i] = (LOOP && sw > 0) ? s_next[i] : args.pose7[i];
    make_pose_consts(pose, &pc);
  }

  // ---- main stream ----
  if (kLockstepSlack > 0) {
    if (lane == 0) s_prog[warp] = n_chunks > 0 ? 0 : 0x7fffffff;
    if (warp == 0 && lane >= kWarps) s_prog[lane] = 0x7fffffff;
    __syncthreads();
  }
  if (n_chunks > 0) {
    int64_t f = pv.warp_first_frame[gwarp];
    int64_t f_end = pv.offsets[f + 1];
    double m0 = 0.0, m1 = 0.0, m2 = 0.0, c = 0.0;
    // frame constants (every lane, redundantly); the next frame's plane and end offset are prefetched one piece
    // ahead so that a frame change does not stall the stream on a global-memory round trip
    // kModeSegments: every frame's m, c were computed at its segment's pose before the sweep; they take the place of its plane
    const double* fsrc = pv.plane;
    if constexpr (MODE == kModeSegments || MODE == kModeRange) fsrc = args.seg_consts;
    double nx_plane[4] = {0.0, 0.0, 0.0, 0.0};
    int64_t nx_end = 0;
    auto prefetch_next = [&]() {
      if (f + 1 < pv.n_frames) {
#pragma unroll
        for (int k = 0; k < 4; ++k) nx_plane[k] = fsrc[(f + 1) * 4 + k];
        nx_end = pv.offsets[f + 2];
      }
    };
    auto set_frame_consts = [&](const double* plane) {
      if constexpr (MODE == kModeSegments || MODE == kModeRange) {
        m0 = plane[0]; m1 = plane[1]; m2 = plane[2]; c = plane[3];
      } else {
        double m[3];
        frame_consts(pc, plane, m, &c);
        m0 = m[0]; m1 = m[1]; m2 = m[2];
      }
    };
    {
      double plane[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) plane[k] = fsrc[f * 4 + k];
      set_frame_consts(plane);
      prefetch_next();
    }
    std::conditional_t<MODE == kModeRange, RangeMoments, Moments> a;
    moments_clear<LOSS>(a);
    // Huber's a (sqrt(a^2) is exact, clc_expand.cuh), once per sweep
    const double huber_a = LOSS == kLossHuber ? sqrt(pv.a2) : 0.0;
    // kModeRange: the range offset b and 1 + s of the point being evaluated
    double range_b = 0.0, range_sigma = 1.0;
    if constexpr (MODE == kModeRange) {
      range_b = args.pose7[7];
      range_sigma = 1.0 + args.pose7[8];
    }
    bool open = false;  // the current piece has accumulated points
    FrameSums fx;       // kModeFrames only
    frame_sums_clear(fx);
    int64_t piece_n = 0;  // kModeFrames: points of the current piece

    // sums the lanes' moments of the finished piece and parks them in the tile
    auto park_piece = [&]() {
      if constexpr (MODE == kModeRange) {
        // as kModeSegments: every piece leaves raw, 25 moments, the cost and its exponent
        double v[32] = {a.S0, a.Sx, a.Sy, a.Sz, a.Sxx, a.Sxy, a.Sxz, a.Syy, a.Syz, a.Szz, a.Qx, a.Qy, a.Qz,
                        a.Pxx, a.Pxy, a.Pxz, a.Pyy, a.Pyz, a.Pzz, a.P2xx, a.P2xy, a.P2xz, a.P2yy, a.P2yz, a.P2zz,
                        0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        double pr = a.prod;
        int es = a.esum;
        if (LOSS == kLossCauchy) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            pr *= __shfl_xor_sync(0xffffffffu, pr, o);  // 32 mantissas in [1,2): product < 2^32
            es += __shfl_xor_sync(0xffffffffu, es, o);
          }
        } else {
          v[kRangeMoments] = pr;
        }
        warp_transpose_sum_regs<32>(v, lane);
        const int kind = frame_piece_kind(pv.offsets[f], f_end, p0, p1);
        double* dst = kind == kPieceWhole
                          ? args.frame_rows + f * kRangeRawDoubles
                          : args.frame_slots + (gwarp * 2 + (kind == kPieceHead ? kSlotHead : kSlotTail)) * kRangeRawDoubles;
        if (lane < kRangeMoments || (LOSS != kLossCauchy && lane == kRangeMoments)) dst[lane] = v[0];
        if (LOSS == kLossCauchy && lane == kRangeMoments) dst[kRangeMoments] = pr;
        if (lane == kRangeMoments + 1) dst[kRangeMoments + 1] = (double)es;
        moments_clear<LOSS>(a);
        open = false;
        return;
      }
      double v[16] = {a.S0, a.Sx, a.Sy, a.Sz, a.Sxx, a.Sxy, a.Sxz, a.Syy, a.Syz, a.Szz, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      double pr = a.prod;
      int es = a.esum;
      double em = 0.0;
      if (MODE == kModeFrames) {
        v[12] = fx.se;
        v[13] = fx.se2;
        em = fx.emax;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) em = nan_max(em, __shfl_xor_sync(0xffffffffu, em, o));
      }
      if (LOSS == kLossCauchy) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          pr *= __shfl_xor_sync(0xffffffffu, pr, o);  // 32 mantissas in [1,2): product < 2^32
          es += __shfl_xor_sync(0xffffffffu, es, o);
        }
      } else {
        v[10] = pr;  // sum of e^2 / rho~(e)
      }
      if constexpr (MODE == kModeSegments) {
        // every piece leaves raw -- the moments and the cost (loss: product and exponent): a whole frame to its row of
        // kSegRawDoubles, a piece of a split frame to this warp's head or tail slot.  clc_segment_fixup_kernel expands them all,
        // so no expansion state is live in the streaming loop, and the transpose keeps v in registers: nothing goes through
        // local memory between the stage loop's head and its back-edges.
        warp_transpose_sum_regs<16>(v, lane);
        const int kind = frame_piece_kind(pv.offsets[f], f_end, p0, p1);
        double* dst = kind == kPieceWhole
                          ? args.frame_rows + f * kSegRawDoubles
                          : args.frame_slots + (gwarp * 2 + (kind == kPieceHead ? kSlotHead : kSlotTail)) * kSlotDoubles;
        if (lane < 10 || (LOSS != kLossCauchy && lane == 10)) dst[lane] = v[0];
        if (LOSS == kLossCauchy && lane == 10) dst[10] = pr;
        if (lane == 11) dst[11] = (double)es;
        moments_clear<LOSS>(a);
        open = false;
        return;
      }
      warp_transpose_sum<16>(v, lane);  // lane L: total of moment (L mod 16)
      const int kind = MODE == kModeFrames ? frame_piece_kind(pv.offsets[f], f_end, p0, p1) : (int)kPieceWhole;
      if (kind != kPieceWhole) {
        // kModeFrames: a piece of a frame that crosses a range end -> this warp's head or tail slot, raw (clc_frames.cuh)
        double* slot = args.frame_slots + (gwarp * 2 + (kind == kPieceHead ? kSlotHead : kSlotTail)) * kSlotDoubles;
        if (lane < 10 || lane == 12 || lane == 13) slot[lane] = v[0];
        if (lane == 10) slot[10] = LOSS == kLossCauchy ? pr : LOSS == kLossNone ? 0.0 : v[0];
        if (lane == 11) slot[11] = (double)es;
        if (lane == 14) slot[14] = em;
        if (lane == 15) slot[15] = (double)piece_n;
      } else {
        {
          double* row = tile + n_tile * kTileStride;
          if (lane < 10 || (LOSS != kLossCauchy && lane == 10)) row[lane] = v[0];
          if (LOSS == kLossCauchy && lane == 10) row[10] = pr;
          if (lane == 11) row[11] = (double)es;
          if (lane == 12) row[12] = __longlong_as_double(f);
        }
        if (MODE == kModeFrames) {
          double* rx = ftile + n_tile * 3;
          if (lane == 12) rx[0] = v[0];
          if (lane == 13) rx[1] = v[0];
          if (lane == 14) rx[2] = em;
        }
        ++n_tile;
        if (n_tile == 32) {
          if (MODE == kModeFrames) flush_frames();
          else flush_tile();
        }
      }
      moments_clear<LOSS>(a);
      open = false;
      if (MODE == kModeFrames) {
        frame_sums_clear(fx);
        piece_n = 0;
      }
    };

    for (int ch = 0; ch < n_chunks; ++ch) {
      const int gc = LOOP ? gc_base + ch : ch;  // running stage number -> ring slot and mbarrier phase
      const int st = gc % NST;
      const int64_t cb = p0 + (int64_t)ch * CH;
      const int64_t ce = (cb + CH < p1) ? cb + CH : p1;
      if (kLockstepSlack > 0) {
        while (__reduce_min_sync(0xffffffffu, *(volatile int*)&s_prog[lane]) < ch - kLockstepSlack) __nanosleep(40);
      }
      mbar_wait(bars + st, (uint32_t)(gc / NST) & 1u);
      const double* sx = ring + st * SST;
      // this lane's points of the stage: local indices 64 g + 2 lane, 64 g + 2 lane + 1 (conflict-free LDS.128)
      double2 X[G], Y[G], Z[G];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        X[g] = *reinterpret_cast<const double2*>(sx + 64 * g + 2 * lane);
        Y[g] = *reinterpret_cast<const double2*>(sx + CH + 64 * g + 2 * lane);
        Z[g] = PLANAR ? make_double2(0.0, 0.0) : *reinterpret_cast<const double2*>(sx + 2 * CH + 64 * g + 2 * lane);
      }
      int64_t q = cb;
      while (q < ce) {
        while (f_end <= q) {  // next non-empty frame
          ++f;
          if (nx_end > q) {   // the prefetched frame is the one (the common case)
            f_end = nx_end;
            set_frame_consts(nx_plane);
          } else {
            f_end = pv.offsets[f + 1];
            if (f_end > q) {
              double plane[4];
#pragma unroll
              for (int k = 0; k < 4; ++k) plane[k] = fsrc[f * 4 + k];
              set_frame_consts(plane);
            }
          }
          if (f_end > q) prefetch_next();
          else nx_end = 0;
        }
        const int64_t hi = f_end < ce ? f_end : ce;
        if (q == cb && hi == cb + CH) {
          // the whole stage belongs to one frame: no masks
#pragma unroll
          for (int g = 0; g < G; ++g) {
            if constexpr (MODE == kModeRange) {
              process2_range<LOSS, PLANAR>(a, X[g], Y[g], Z[g], true, true, m0, m1, m2, c, range_sigma, range_b, pv.inv_a2, huber_a,
                                           pv.a2);
              continue;
            }
            process2<LOSS, MODE == kModeLM || MODE == kModeSegments, PLANAR>(a, X[g], Y[g], Z[g], true, true, m0, m1, m2, c, pv.inv_a2,
                                                                            huber_a, pv.a2);
            if (MODE == kModeFrames) frame_sums2<PLANAR>(fx, X[g], Y[g], Z[g], true, true, m0, m1, m2, c);
          }
        } else {
#pragma unroll
          for (int g = 0; g < G; ++g) {
            const int64_t i0 = cb + 64 * g + 2 * lane;
            if constexpr (MODE == kModeSegments) {
              // the points outside the piece may belong to another segment: their coordinates are replaced before any
              // arithmetic (a NaN there must not reach this frame through 0 * NaN), so every segment's rows depend on its
              // own points only
              const bool v0 = i0 >= q && i0 < hi, v1 = i0 + 1 >= q && i0 + 1 < hi;
              const double2 Xm = make_double2(v0 ? X[g].x : 0.0, v1 ? X[g].y : 0.0);
              const double2 Ym = make_double2(v0 ? Y[g].x : 0.0, v1 ? Y[g].y : 0.0);
              const double2 Zm = make_double2(v0 ? Z[g].x : 0.0, v1 ? Z[g].y : 0.0);
              process2<LOSS, true, PLANAR>(a, Xm, Ym, Zm, v0, v1, m0, m1, m2, c, pv.inv_a2, huber_a, pv.a2);
              continue;
            }
            if constexpr (MODE == kModeRange) {  // masked as kModeSegments masks (a NaN of another frame stays out)
              const bool v0 = i0 >= q && i0 < hi, v1 = i0 + 1 >= q && i0 + 1 < hi;
              const double2 Xm = make_double2(v0 ? X[g].x : 0.0, v1 ? X[g].y : 0.0);
              const double2 Ym = make_double2(v0 ? Y[g].x : 0.0, v1 ? Y[g].y : 0.0);
              const double2 Zm = make_double2(v0 ? Z[g].x : 0.0, v1 ? Z[g].y : 0.0);
              process2_range<LOSS, PLANAR>(a, Xm, Ym, Zm, v0, v1, m0, m1, m2, c, range_sigma, range_b, pv.inv_a2, huber_a, pv.a2);
              continue;
            }
            process2<LOSS, MODE == kModeLM, PLANAR>(a, X[g], Y[g], Z[g], i0 >= q && i0 < hi, i0 + 1 >= q && i0 + 1 < hi, m0, m1, m2,
                                            c, pv.inv_a2, huber_a, pv.a2);
            if (MODE == kModeFrames)
              frame_sums2<PLANAR>(fx, X[g], Y[g], Z[g], i0 >= q && i0 < hi, i0 + 1 >= q && i0 + 1 < hi, m0, m1, m2, c);
          }
        }
        if (LOSS == kLossCauchy) renormalise(a);
        open = true;
        if (MODE == kModeFrames) piece_n += hi - q;
        q = hi;
        if (hi == f_end) park_piece();
      }
      // every lane has consumed its registers' worth of the stage (data dependence), so the slot can be handed
      // back to the TMA engine: the other stage stays in flight meanwhile
      __syncwarp();
      if (issued < total_chunks) issue_one(true);
      if (kLockstepSlack > 0 && lane == 0) *(volatile int*)&s_prog[warp] = (ch + 1 == n_chunks) ? 0x7fffffff : ch + 1;
    }
    if (open) park_piece();  // the last frame continues in the next warp's range
  }
  if (MODE == kModeFrames) {
    // the rows of whole frames are written; split frames are finished by clc_frame_fixup_kernel -- no block reduction
    flush_frames();
    return;
  }
  if constexpr (MODE == kModeSegments || MODE == kModeRange) return;  // every piece has left raw (park_piece): no tile, no block reduction
  CLC_STAMP(1);
  if (args.timing != nullptr && lane == 0) args.timing[(int64_t)gridDim.x * 8 + gwarp] = globaltimer_ns();
  flush_tile();
  CLC_STAMP(2);

  // ---- board-edge residuals: one residual per lane, same moment/expansion path ----
  if (MODE == kModeLM && args.use_edges && pv.n_edges > 0) {
    const int64_t total_lanes = (int64_t)gridDim.x * kThreads;
    double out[NOUT];
#pragma unroll
    for (int k = 0; k < NOUT; ++k) out[k] = 0.0;
    bool any = false;
    for (int64_t i = gwarp * 32 + lane; i < pv.n_edges; i += total_lanes) {
      const int64_t f = i >> 1;
      const int64_t cnt = pv.offsets[f + 1] - pv.offsets[f];
      if (cnt <= 0) continue;
      any = true;
      double plane[4], m[3], c;
#pragma unroll
      for (int k = 0; k < 4; ++k) plane[k] = pv.edge_plane[i * 4 + k];
      frame_consts(pc, plane, m, &c);
      const double x = pv.edge_pt[i * 3], y = pv.edge_pt[i * 3 + 1], z = pv.edge_pt[i * 3 + 2];
      const double e = fma(m[0], x, fma(m[1], y, fma(m[2], z, c)));
      double w, cost_term;
      loss_weight(LOSS, e, pv.a2, pv.inv_a2, &w, &cost_term);
      const double S[10] = {w, w * x, w * y, w * z, w * x * x, w * x * y, w * x * z, w * y * y, w * y * z, w * z * z};
      expand_lm(plane, m, c, 1.0 / (double)cnt, S, LOSS, cost_term, pv.a2, out);
    }
    if (__any_sync(0xffffffffu, any)) {
      double v[32];
#pragma unroll
      for (int k = 0; k < 32; ++k) v[k] = (k < NOUT) ? out[k] : 0.0;
      warp_transpose_sum<32>(v, lane);
      if (lane < NOUT) s_acc[warp][lane] += v[0];
      __syncwarp();
    }
  }

  // ---- block reduction (fixed order) ----
  // The block's partial sums travel to block 0 with a low-latency protocol instead of "store, fence, ticket": every
  // 8-byte word carries 32 bits of the value and the 32-bit sequence number of this launch, 8-byte stores are single
  // transactions, so the reader needs no flag and the writer no fence -- one one-way trip through L2 instead of three
  // dependent ones (partials -> release ticket -> acquire poll -> partial loads).
  const unsigned long long ll_tag = (unsigned long long)launch_tag << 32;
  __syncthreads();
  double block_sum = 0.0;
  if (threadIdx.x < NOUT) {
#pragma unroll
    for (int wv = 0; wv < kWarps; ++wv) block_sum += s_acc[wv][threadIdx.x];
    if (gridDim.x > 1) {
      const unsigned long long bits = (unsigned long long)__double_as_longlong(block_sum);
      st_volatile_v2(args.partials_ll + ((int64_t)blockIdx.x * kMaxOut + threadIdx.x) * 2, ll_tag | (bits & 0xffffffffull),
                     ll_tag | (bits >> 32));
    }
  }
  CLC_STAMP(3);
  // let the next sweep's blocks be scheduled on the SMs this grid is vacating (they only prefetch until we complete)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // The final reduction (and the LM update) always runs on block 0 -- the persistent grid is fully co-resident, so
  // block 0 can wait for the other blocks -- rather than on whichever block happens to finish last: the ~1000 instructions
  // of that serial tail then stay warm in ONE SM's instruction cache from launch to launch.
  if (blockIdx.x != 0 && (!LOOP || sweeps_max == 1)) return;

  // ---- block 0: deterministic sum of the block partials ----
  if (blockIdx.x == 0) {
    // thread (part, k) polls the words of output k of blocks part, part + PARTS, ... (all its loads in flight at once)
    // and adds them in block order; the PARTS partial results are then added in part order: a fixed tree.
    constexpr int PARTS = kThreads / NOUT;
    constexpr int NB = 10;  // blocks per thread and round
    double* s_gather = &s_red[0][0];
    static_assert(kWarps * 32 >= PARTS * NOUT, "s_red holds one value per gathering thread");
    if (gridDim.x > 1 && threadIdx.x < PARTS * NOUT) {
      const int k = threadIdx.x % NOUT, part = threadIdx.x / NOUT;
      double acc = 0.0;
      for (int base = part; base < (int)gridDim.x; base += PARTS * NB) {
        unsigned long long w0[NB], w1[NB];
        unsigned int pending = 0u;
#pragma unroll
        for (int u = 0; u < NB; ++u)
          if (base + u * PARTS < (int)gridDim.x) pending |= 1u << u;
        unsigned int polls = 0;
        unsigned long long t0 = 0;
        while (pending != 0u) {
#pragma unroll
          for (int u = 0; u < NB; ++u)
            if ((pending >> u) & 1u)
              ld_volatile_v2(args.partials_ll + ((int64_t)(base + u * PARTS) * kMaxOut + k) * 2, w0[u], w1[u]);
#pragma unroll
          for (int u = 0; u < NB; ++u)
            if (((pending >> u) & 1u) && (w0[u] & 0xffffffff00000000ull) == ll_tag && (w1[u] & 0xffffffff00000000ull) == ll_tag)
              pending &= ~(1u << u);
          if (pending != 0u && (++polls & 0xffu) == 0u) {
            // The grid is sized to be fully co-resident (one block per SM), which is what lets block 0 wait here.  Should
            // that ever not hold (MPS with a reduced SM share, a foreign kernel pinning SMs), fail loudly instead of
            // hanging: after 2 s the error flag is raised, the host reports it and the LM is stopped.
            const unsigned long long now = globaltimer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 2000000000ull) {
              if (args.error != nullptr) *args.error = 2;
              break;
            }
          }
        }
#pragma unroll
        for (int u = 0; u < NB; ++u)
          if (base + u * PARTS < (int)gridDim.x) acc += __longlong_as_double((long long)((w1[u] << 32) | (w0[u] & 0xffffffffull)));
      }
      s_gather[threadIdx.x] = acc;
    }
    double total = block_sum;  // a single-block grid: nothing to gather
    if (gridDim.x > 1) {
      __syncthreads();
      total = 0.0;
      if (threadIdx.x < NOUT) {
#pragma unroll
        for (int part = 0; part < PARTS; ++part) total += s_gather[part * NOUT + threadIdx.x];
      }
    }
    if (args.nranks > 1) {
      // ---- fused all-reduce: NVLink stores into every rank's mailbox, tagged words, deterministic rank-order sum ----
      // the sequence number lives on the device: sweeps that no-op (LM already finished) must not consume one, or two
      // consecutive real exchanges could land in the same parity slot while a slow peer is still reading it
      double* s_tot = s_acc[0];                                 // [NOUT] this rank's totals
      double* s_x = reinterpret_cast<double*>(s_dyn) + kWarps * RING;  // [nranks][NOUT] in the tiles, idle between two sweeps
                                                                       // (not the rings: a looping grid is prefetching into them)
      static_assert(kWarps * kTileDoublesPerWarp >= kMaxRanks * kMaxOut, "the tiles hold one value per rank and output");
      __syncthreads();                                          // s_gather reads are done before s_acc/s_dyn are reused
      if (threadIdx.x < NOUT) s_tot[threadIdx.x] = total;
      __syncthreads();
      const unsigned long long seq = *args.seq_counter + 1ull;
      const unsigned long long tag = (seq & 0xffffffffull) << 32;  // never matches the zero-initialised mailbox for seq >= 1
      const int par = (int)(seq & 1ull);
      const int n_words = args.nranks * NOUT;
      // one (destination rank, output) pair per thread: all stores leave at once
      for (int idx = threadIdx.x; idx < n_words; idx += kThreads) {
        const int r = idx / NOUT, k = idx % NOUT;
        const unsigned long long bits = (unsigned long long)__double_as_longlong(s_tot[k]);
        const int64_t slot = (((int64_t)par * args.nranks + args.rank) * kMailboxSlot + k) * 2;
        st_relaxed_sys(args.peer_mailbox[r] + slot, tag | (bits & 0xffffffffull));
        st_relaxed_sys(args.peer_mailbox[r] + slot + 1, tag | (bits >> 32));
      }
      // one (source rank, output) pair per thread polls my own mailbox: the waits for all ranks overlap
      const unsigned long long t0 = globaltimer_ns();
      for (int idx = threadIdx.x; idx < n_words; idx += kThreads) {
        const int r = idx / NOUT, k = idx % NOUT;
        const unsigned long long* src = args.peer_mailbox[args.rank] + (((int64_t)par * args.nranks + r) * kMailboxSlot + k) * 2;
        unsigned long long a0, a1;
        unsigned int polls = 0;
        for (;;) {
          a0 = ld_relaxed_sys(src);
          a1 = ld_relaxed_sys(src + 1);
          if ((a0 & 0xffffffff00000000ull) == tag && (a1 & 0xffffffff00000000ull) == tag) break;
          if ((++polls & 0x3fu) == 0u && globaltimer_ns() - t0 > 5000000000ull) {  // 5 s: a peer died -- fail loudly
            if (args.error != nullptr) *args.error = 1;
            break;
          }
        }
        s_x[idx] = __longlong_as_double((long long)((a1 << 32) | (a0 & 0xffffffffull)));
      }
      __syncthreads();
      if (threadIdx.x < NOUT) {
        total = 0.0;
        for (int r = 0; r < args.nranks; ++r) total += s_x[r * NOUT + threadIdx.x];  // rank order: identical bits everywhere
      }
      if (threadIdx.x == 0) *args.seq_counter = seq;
    }
    __syncthreads();
    if (threadIdx.x < NOUT) {
      args.sums[threadIdx.x] = total;
      if (threadIdx.x < 32) s_red[0][threadIdx.x] = total;
    }
    __syncthreads();
    CLC_STAMP(4);
    if (threadIdx.x == 0) *args.launch_seq = launch_tag;
    if (MODE == kModeLM && args.lm != nullptr) {
      // the hot LM state sits in shared memory since the start of the kernel: no global round trip on the serial tail
      if (threadIdx.x == 0) {
        double sums[kNumSums];
        for (int k = 0; k < kNumSums; ++k) sums[k] = s_red[0][k];
        if (args.error != nullptr && *args.error != 0) {
          // a peer never answered / the grid was not co-resident: the sums are not the whole problem's -- stop the solve
          reinterpret_cast<LmCore*>(s_core)->done = CLC_TERM_FAILURE;
        } else {
          lm_update(reinterpret_cast<LmCore*>(s_core), args.lm->trace, sums);
        }
      }
      __syncthreads();
      if (LOOP && sweeps_max > 1 && threadIdx.x < 8) {
        // the next pose and the `done` flag: to this block through shared memory, to the other blocks as tagged words
        const LmCore* core = reinterpret_cast<const LmCore*>(s_core);
        const double v = threadIdx.x < 7 ? core->cand[threadIdx.x] : (double)core->done;
        s_next[threadIdx.x] = v;
        if (gridDim.x > 1) {
          const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
          st_volatile_v2(args.pose_ll + 2 * threadIdx.x, ll_tag | (bits & 0xffffffffull), ll_tag | (bits >> 32));
        }
      }
      unsigned long long* o_core = reinterpret_cast<unsigned long long*>(&args.lm->core);
      for (int k = threadIdx.x; k < kLmCoreWords; k += kThreads) o_core[k] = s_core[k];
    }
    CLC_STAMP(5);
  } else {
    // ---- looping grid, blocks other than 0: wait for the next pose from block 0 ----
    if (threadIdx.x < 8 && sw + 1 < sweeps_max) {
      unsigned long long a0, a1, t0 = 0;
      unsigned int polls = 0;
      for (;;) {
        ld_volatile_v2(args.pose_ll + 2 * threadIdx.x, a0, a1);
        if ((a0 & 0xffffffff00000000ull) == ll_tag && (a1 & 0xffffffff00000000ull) == ll_tag) break;
        if ((++polls & 0xffu) == 0u) {
          const unsigned long long now = globaltimer_ns();
          if (t0 == 0) t0 = now;
          else if (now - t0 > 10000000000ull) {  // 10 s without a pose: block 0 is gone -- stop instead of hanging
            if (args.error != nullptr) *args.error = 2;
            a0 = a1 = 0;
            break;
          }
        }
      }
      const bool lost = (a0 | a1) == 0ull;
      s_next[threadIdx.x] = lost ? (double)CLC_TERM_FAILURE : __longlong_as_double((long long)((a1 << 32) | (a0 & 0xffffffffull)));
    }
  }
  // ---- next sweep of the same launch (LOOP instantiations: the LM runs inside the kernel) ----
  if (!LOOP || sw + 1 >= sweeps_max) break;
  gc_base += n_chunks;
  __syncthreads();  // s_next is visible to the whole block
  if (s_next[7] != 0.0) {
    drain(gc_base);  // stages prefetched for a sweep that will not happen
    break;
  }
  }  // sweeps
}

// ---- K3: LM update as its own launch (multi-rank: runs after the all-reduce of `sums`) --------------------------
__global__ void clc_lm_kernel(LmState* lm, const double* sums) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double s[kNumSums];
    for (int k = 0; k < kNumSums; ++k) s[k] = sums[k];
    lm_update(&lm->core, lm->trace, s);
  }
}

// ---- K1 fix-up of the per-frame report (after a kModeFrames sweep) ---------------------------------------------------
// One thread per frame: an empty frame gets a row of zeros; a split frame (clc_frames.cuh) adds the tail slot of its first warp
// and the head slots of the following warps, in warp order (the row is bit-reproducible), and expands them into its row; the
// rows of the other frames were written by the sweep.
template <int LOSS>
__global__ void clc_frame_fixup_kernel(ProblemView pv, const double* pose7, int edges, const double* __restrict__ slots,
                                       double* __restrict__ rows) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= pv.n_frames) return;
  const int64_t fs = pv.offsets[f], fe = pv.offsets[f + 1];
  double* row = rows + f * kRowDoubles;
  if (fe <= fs) {
    for (int k = 0; k < kRowDoubles; ++k) row[k] = 0.0;
    return;
  }
  int64_t w0, w1;
  frame_warps(fs, fe, pv.per_warp, &w0, &w1);
  if (w0 == w1) return;
  double S[10] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  double cost_term = 0.0, se = 0.0, se2 = 0.0, emax = 0.0;
  int64_t n = 0;
  for (int64_t w = w0; w <= w1; ++w) {
    const double* s = slots + frame_slot(w, w0);
#pragma unroll
    for (int k = 0; k < 10; ++k) S[k] += s[k];
    cost_term += LOSS == kLossCauchy ? log(s[10]) + s[11] * 0.693147180559945309417232121458 : LOSS == kLossNone ? s[13] : s[10];
    se += s[12];
    se2 += s[13];
    emax = nan_max(emax, s[14]);
    n += (int64_t)s[15];
  }
  PoseConsts pc;
  make_pose_consts(pose7, &pc);
  frame_row_write(pv, pc, f, n, S, cost_term, se, se2, emax, LOSS, edges != 0, row);
}

// ---- K0: layout kernels ------------------------------------------------------------------------------------------

// AoS (x,y,z)[n] -> SoA at element offset `dst_off`
// *nonplanar is raised if any z is not exactly zero (NaN included): decides whether the z stream has to be kept
__global__ void clc_aos_to_soa_kernel(const double* __restrict__ aos, int64_t n, double* __restrict__ x,
                                      double* __restrict__ y, double* __restrict__ z, int64_t dst_off,
                                      int* __restrict__ nonplanar) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool off_plane = false;
  if (i < n) {
    x[dst_off + i] = aos[3 * i];
    y[dst_off + i] = aos[3 * i + 1];
    const double zi = aos[3 * i + 2];
    z[dst_off + i] = zi;
    off_plane = !(zi == 0.0);
  }
  if (__any_sync(0xffffffffu, off_plane) && (threadIdx.x & 31) == 0) atomicOr(nonplanar, 1);
}

// packed (x,y)[n] -> SoA: the upload format of planar data (the host packer checked every z == 0 and left it behind,
// so 16 instead of 24 bytes per point cross PCIe)
__global__ void clc_aos2_to_soa_kernel(const double2* __restrict__ xy, int64_t n, double* __restrict__ x,
                                       double* __restrict__ y, double* __restrict__ z, int64_t dst_off) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const double2 v = xy[i];
    x[dst_off + i] = v.x;
    y[dst_off + i] = v.y;
    if (z != nullptr) z[dst_off + i] = 0.0;
  }
}

__global__ void clc_soa_to_aos_kernel(const double* __restrict__ x, const double* __restrict__ y,
                                      const double* __restrict__ z, int64_t src_off, int64_t n,
                                      double* __restrict__ aos) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    aos[3 * i] = x[src_off + i];
    aos[3 * i + 1] = y[src_off + i];
    aos[3 * i + 2] = (z != nullptr) ? z[src_off + i] : 0.0;
  }
}

// frame pose -> board plane (a2) and the two edge planes (a7)
__global__ void clc_planes_kernel(const double* __restrict__ frame_pose, int64_t n_frames, double* __restrict__ plane,
                                  double* __restrict__ edge_plane) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frames) return;
  double fp[7], pl[4];
  for (int k = 0; k < 7; ++k) fp[k] = frame_pose[f * 7 + k];
  frame_plane(fp, pl);
  for (int k = 0; k < 4; ++k) plane[f * 4 + k] = pl[k];
  if (edge_plane != nullptr) {
    double p1[4], p2[4];
    edge_planes(fp, p1, p2);
    for (int k = 0; k < 4; ++k) {
      edge_plane[(2 * f) * 4 + k] = p1[k];
      edge_plane[(2 * f + 1) * 4 + k] = p2[k];
    }
  }
}

// frame containing the first point of every warp range (binary search done once at problem creation)
__global__ void clc_warp_table_kernel(const int64_t* __restrict__ offsets, int64_t n_frames, int64_t n_points,
                                      int64_t per_warp, int64_t n_warps, int* __restrict__ first_frame) {
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_warps) return;
  const int64_t p0 = w * per_warp;
  if (p0 >= n_points) { first_frame[w] = 0; return; }
  int64_t lo = 0, hi = n_frames;  // offsets[lo] <= p0 < offsets[hi]
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (offsets[mid] <= p0) lo = mid; else hi = mid;
  }
  first_frame[w] = (int)lo;
}

// ---- K5: synthetic generator (exact-M mode) ----------------------------------------------------------------------

__global__ void clc_gen_frames_kernel(uint64_t seed, int64_t frame_begin, int64_t n_local, int64_t beams, int with_edges,
                                      CameraDesc cam, int image_width, int image_height, double* __restrict__ frame_pose,
                                      double* __restrict__ frame_pose_true, int64_t* __restrict__ offsets,
                                      double* __restrict__ edge_pt) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) offsets[n_local] = n_local * beams;
  if (i >= n_local) return;
  double fp[7], fe[7];
  if (cam.model == kCameraNone) {
    gen_frame_pose(seed, frame_begin + i, with_edges != 0, fp);
    for (int k = 0; k < 7; ++k) fe[k] = fp[k];
  } else {
    // camera mode: the board must be fully in the image; the pose handed to the calibration is the PnP estimate
    float uv[2 * 256];  // up to 8 x 8 tags
    const bool in_view = gen_frame_pose_camera(cam, image_width, image_height, seed, frame_begin + i, with_edges != 0, fp);
    bool ok = in_view && grid_num_corners(cam) <= 256;
    if (ok) ok = camera_estimate_pose(cam, seed, frame_begin + i, fp, fe, uv);
    if (!ok)
      for (int k = 0; k < 7; ++k) fe[k] = fp[k];  // no usable image of the board: fall back to the exact pose
  }
  for (int k = 0; k < 7; ++k) {
    frame_pose[i * 7 + k] = fe[k];
    if (frame_pose_true != nullptr) frame_pose_true[i * 7 + k] = fp[k];
  }
  offsets[i] = i * beams;
  if (with_edges) {
    double ep[6];
    if (!gen_edge_points(fp, ep))
      for (int k = 0; k < 6; ++k) ep[k] = 0.0;
    for (int k = 0; k < 6; ++k) edge_pt[i * 6 + k] = ep[k];
  }
}

// one block per frame
__global__ void clc_gen_points_kernel(uint64_t seed, double sigma, int64_t frame_begin, int64_t beams,
                                      const double* __restrict__ frame_pose, double* __restrict__ x,
                                      double* __restrict__ y, double* __restrict__ z) {
  const int64_t i = blockIdx.x;
  __shared__ double s_nl[3], s_dl, s_a, s_b;
  if (threadIdx.x == 0) {
    double fp[7], nl[3], dl, a = 0.0, b = 0.0;
    for (int k = 0; k < 7; ++k) fp[k] = frame_pose[i * 7 + k];
    gen_plane_laser(fp, nl, &dl);
    gen_window(nl, dl, &a, &b);
    s_nl[0] = nl[0]; s_nl[1] = nl[1]; s_nl[2] = nl[2]; s_dl = dl; s_a = a; s_b = b;
  }
  __syncthreads();
  const double n0 = s_nl[0], n1 = s_nl[1], dl = s_dl, a = s_a, b = s_b;
  for (int64_t j = threadIdx.x; j < beams; j += blockDim.x) {
    const double theta = a + (b - a) * (((double)j + 0.5) / (double)beams);
    const double cx = cos(theta), sy = sin(theta);
    const double depth = -dl / (cx * n0 + sy * n1) + gen_noise(seed, sigma, frame_begin + i, j);
    const int64_t o = i * beams + j;
    x[o] = depth * cx;
    y[o] = depth * sy;
    if (z != nullptr) z[o] = 0.0;  // a 2-D laser: planar by construction, the z stream is not stored
  }
}

// L2 flush for the measurement hook: overwrite a buffer larger than L2, then read it back.  The read pass matters:
// after the write pass L2 is full of DIRTY lines whose write-back (~50 MB of DRAM writes) would otherwise be charged
// to the kernel being timed; after the read pass L2 holds clean, unrelated lines.
__global__ void clc_flush_kernel(double* buf, int64_t n, double v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    buf[i] = v;
}
__global__ void clc_flush_read_kernel(const double* buf, int64_t n, double* sink) {
  double acc = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    acc += __ldcg(buf + i);
  if (acc == 123.456) *sink = acc;  // never true: keeps the loads alive
}

// End of an LM solve: the lines its sweeps read with evict_last go back to the normal priority, so that they do not outlive
// the solve (other work on the GPU, the cold-L2 measurement hook).  One thread per 128-byte line of x in the resident share
// of every warp's range (the stages clc_sweep_kernel marks, same range arithmetic); it demotes the same line of y and z.
__global__ void clc_l2_demote_kernel(ProblemView pv, int64_t n_warps, int chunk) {
  const int k = pv.resident_chunks;
  const int64_t lines_per_warp = (int64_t)k * chunk / 16;  // 16 doubles per line
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_warps * lines_per_warp) return;
  const int64_t w = t / lines_per_warp;
  const int64_t P = pv.n_points;
  int64_t p0 = w * pv.per_warp;
  if (p0 > P) p0 = P;
  int64_t p1 = p0 + pv.per_warp;
  if (p1 > P) p1 = P;
  const int64_t n_chunks = (p1 - p0 + chunk - 1) / chunk;
  const int64_t c0 = n_chunks > k ? n_chunks - k : 0;  // first resident stage (a short last range may hold fewer than k)
  const int64_t i = p0 + c0 * chunk + (t - w * lines_per_warp) * 16;
  if (i >= p0 + n_chunks * chunk) return;
  asm volatile("applypriority.global.L2::evict_normal [%0], 128;" ::"l"(pv.x + i) : "memory");
  asm volatile("applypriority.global.L2::evict_normal [%0], 128;" ::"l"(pv.y + i) : "memory");
  if (pv.z != nullptr) asm volatile("applypriority.global.L2::evict_normal [%0], 128;" ::"l"(pv.z + i) : "memory");
}

}  // namespace clc
