// clc_quantiles.cuh -- the device side of clc_point_residuals, clc_residual_quantiles and clc_frame_quantiles: exact order
// statistics of the raw point-to-board distances |e| (include/clc_b200.h; the selection arithmetic is clc_quantile_plan.h).
//
// Every kernel recomputes e as the sweep kernel, the frame report and the trim compute it: frame_consts at the pose, then
// point_distance.  The ones that stream the whole problem load and walk their tiles as the trim mark kernel does (tile_load,
// tile_first_frame, trim_frame_of): the same tiles of kTrimTile points, the same 32-way search for a tile's first frame.  (The
// trim mark kernel keeps its own inline copy: calling these helpers from it changes its register allocation, and it is left
// byte-identical.)
//
// Problem-wide, a radix select on the 63-bit key of |e|: clc_quantile_pass_kernel runs on a persistent grid and, per pass,
//   - histograms the next digit of every key that matches an active prefix (uint32 bins in shared memory, added into global uint64
//     counts once per block, so counts stay exact past 2^32 points), or
//   - compacts the keys of the active buckets into a scratch buffer once each bucket holds at most kCompactCap keys (the order
//     of the scratch does not matter), after which the remaining digits read the scratch instead of the point streams.
// The host consumes each histogram (qsel_update) and launches the next pass.
//
// Per frame, clc_frame_quantiles_kernel: one block per frame.  A frame of at most kFrameSortMax points sorts its keys in shared
// memory (bitonic) and reads every rank off the sorted keys; a larger frame runs the radix select on its block, with one pass over
// its points in global memory per digit.
#pragma once

#include "clc_quantile_plan.h"
#include "clc_trim.cuh"

namespace clc {

constexpr int kQuantThreads = kTrimThreads;
constexpr int kFrameSortMax = 1 << kFrameBinsLog2;  // S: the largest frame sorted in shared memory (its buffer holds the bins too)
static_assert(kQuantThreads == 256, "the frame kernel's loops assume 256 threads");

// The points of the tile [t0, t0 + kTrimTile): slot i of a thread holds point t0 + i * kTrimThreads + threadIdx.x, 0 at or past
// n_end.  z == nullptr: every z is 0.  All loads are issued before any use: they do not depend on the frames.
__device__ __forceinline__ void tile_load(const double* x, const double* y, const double* z, int64_t t0, int64_t n_end,
                                          double* X, double* Y, double* Z) {
#pragma unroll
  for (int i = 0; i < kTrimPerThread; ++i) {
    const int64_t j = t0 + i * kTrimThreads + threadIdx.x;
    const bool in = j < n_end;
    X[i] = in ? x[j] : 0.0;
    Y[i] = in ? y[j] : 0.0;
    Z[i] = in && z != nullptr ? z[j] : 0.0;
  }
}

// The frame of point t0, called by every lane of one warp: a 32-way search, about log32(n_frames) dependent loads (a bisection's
// log2 chain of loads would hold every block for microseconds, longer than its share of the stream).
__device__ __forceinline__ int64_t tile_first_frame(const int64_t* offsets, int64_t n_frames, int64_t t0, int lane) {
  int64_t lo = 0, hi = n_frames;  // offsets[lo] <= t0 < offsets[hi]
  while (hi - lo > 1) {
    const int64_t probe = lo + 1 + (hi - lo - 1) * lane / 32;  // in (lo, hi), non-decreasing over the lanes
    const unsigned below = __ballot_sync(0xffffffffu, offsets[probe] <= t0);
    const int n = __popc(below);  // the lanes whose probe starts at or before t0 come first
    const int64_t new_lo = n > 0 ? __shfl_sync(0xffffffffu, probe, n - 1) : lo;
    hi = n < 32 ? __shfl_sync(0xffffffffu, probe, n < 32 ? n : 0) : hi;
    lo = new_lo;
  }
  return lo;
}

__device__ __forceinline__ uint64_t abs_key(double e) { return (uint64_t)__double_as_longlong(fabs(e)); }

struct PointStreams {
  const double* x;
  const double* y;
  const double* z;  // nullptr: every z is known to be 0
  const double* plane;
  const int64_t* offsets;
  int64_t n_frames, n_points;
  double pose7[7];
};

// Calls visit(i, j, e) for the points j of the tile [t0, t0 + kTrimTile) below n_end, slot i of every thread (tile_load), with e the
// point's raw distance; every lane of the block runs the calls (j >= n_end: e is NaN), so visit may use warp collectives.
// Ends with a barrier: the caller may run the next tile at once.
template <class Visit>
__device__ __forceinline__ void tile_distances(const PointStreams& a, const PoseConsts& pc, int64_t t0, int64_t n_end, int64_t* s_first,
                                               Visit&& visit) {
  double X[kTrimPerThread], Y[kTrimPerThread], Z[kTrimPerThread];
  tile_load(a.x, a.y, a.z, t0, n_end, X, Y, Z);
  if ((threadIdx.x >> 5) == 0) {
    const int64_t lo = tile_first_frame(a.offsets, a.n_frames, t0, threadIdx.x & 31);
    if (threadIdx.x == 0) *s_first = lo;
  }
  __syncthreads();
  int64_t f = *s_first, f_end = 0;
  double m[3], c = 0.0;
  auto set_frame = [&](int64_t g) {
    double plane[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) plane[k] = a.plane[g * 4 + k];
    frame_consts(pc, plane, m, &c);
    f = g;
    f_end = a.offsets[g + 1];
  };
  set_frame(f);
#pragma unroll
  for (int i = 0; i < kTrimPerThread; ++i) {
    const int64_t j = t0 + i * kTrimThreads + threadIdx.x;
    double e = __longlong_as_double(0x7FF8000000000000ll);
    if (j < n_end) {
      if (f_end <= j) set_frame(trim_frame_of(a.offsets, a.n_frames, f, j));
      e = point_distance(m, c, X[i], Y[i], Z[i]);
    }
    visit(i, j, e);
  }
  __syncthreads();  // s_first is overwritten by the next tile
}

// ---- the per-point dump: block b writes e of points [first + b kTrimTile, ...) below first + count into out[j - first] ----------
__global__ void __launch_bounds__(kQuantThreads) clc_point_residuals_kernel(PointStreams a, int64_t first, int64_t count, double* out) {
  __shared__ int64_t s_first;
  PoseConsts pc;
  make_pose_consts(a.pose7, &pc);
  const int64_t t0 = first + (int64_t)blockIdx.x * kTrimTile;
  tile_distances(a, pc, t0, first + count, &s_first, [&](int, int64_t j, double e) {
    if (j < first + count) out[j - first] = e;
  });
}

// ---- the problem-wide passes ------------------------------------------------------------------------------------------------------
enum QuantPassKind { kPassPoints = 0, kPassCompact = 1, kPassScratch = 2 };

struct QuantPassArgs {
  PointStreams pts;
  const uint64_t* keys;  // kPassScratch: the compacted keys [n_keys]
  int64_t n_keys;
  int bits, n_pre, d;  // the selection's state (QSel) and the digit width of this pass
  uint64_t pre[kQuantilesMax];
  unsigned long long* hist;       // [n_pre << d], zero on entry (kPassPoints, kPassScratch)
  uint64_t* out_keys;             // kPassCompact: [n_pre * kCompactCap]
  unsigned long long* out_count;  // kPassCompact: zero on entry
};

template <int KIND>
__global__ void __launch_bounds__(kQuantThreads) clc_quantile_pass_kernel(QuantPassArgs a) {
  __shared__ uint32_t s_hist[1 << kQuantileBinsLog2];
  __shared__ int64_t s_first;
  const int lane = threadIdx.x & 31;
  const int nb = a.n_pre << a.d;
  if (KIND != kPassCompact) {
    for (int b = threadIdx.x; b < nb; b += kQuantThreads) s_hist[b] = 0;
    __syncthreads();
  }
  // every lane calls it: warp-aggregated shared atomics (noisy data puts most keys of a pass into a few bins)
  auto take = [&](uint64_t key, bool in) {
    if (KIND == kPassCompact) {
      const bool hit = in && qsel_match(a.bits, a.n_pre, a.pre, key);
      const unsigned hits = __ballot_sync(0xffffffffu, hit);
      unsigned long long base = 0;
      if (lane == 0 && hits) base = atomicAdd(a.out_count, (unsigned long long)__popc(hits));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (hit) a.out_keys[base + __popc(hits & ((1u << lane) - 1u))] = key;
    } else {
      const int bin = in ? qsel_bin(a.bits, a.n_pre, a.pre, a.d, key) : -1;
      const unsigned same = __match_any_sync(0xffffffffu, bin);
      if (bin >= 0 && lane == __ffs(same) - 1) atomicAdd(&s_hist[bin], (uint32_t)__popc(same));
    }
  };
  if (KIND == kPassScratch) {
    for (int64_t base = (int64_t)blockIdx.x * kQuantThreads; base < a.n_keys; base += (int64_t)gridDim.x * kQuantThreads) {
      const int64_t j = base + threadIdx.x;
      take(j < a.n_keys ? a.keys[j] : 0, j < a.n_keys);
    }
  } else {
    PoseConsts pc;
    make_pose_consts(a.pts.pose7, &pc);
    const int64_t n_tiles = (a.pts.n_points + kTrimTile - 1) / kTrimTile;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x)
      tile_distances(a.pts, pc, t * kTrimTile, a.pts.n_points, &s_first, [&](int, int64_t, double e) { take(abs_key(e), true); });
  }
  if (KIND != kPassCompact) {
    __syncthreads();
    for (int b = threadIdx.x; b < nb; b += kQuantThreads)
      if (s_hist[b] != 0) atomicAdd(&a.hist[b], (unsigned long long)s_hist[b]);
  }
}

// ---- per frame ---------------------------------------------------------------------------------------------------------------
struct FrameQuantArgs {
  PointStreams pts;
  int n_q;
  double q[kQuantilesMax];
  double* values;    // [n_frames * n_q]
  int64_t* n_valid;  // [n_frames]
};

__global__ void __launch_bounds__(kQuantThreads) clc_frame_quantiles_kernel(FrameQuantArgs a) {
  __shared__ unsigned long long s_buf[kFrameSortMax];  // the sorted keys, or the bins of a large frame's passes
  __shared__ QSel s_sel;
  __shared__ unsigned long long s_valid;
  const int64_t f = blockIdx.x;
  const PointStreams& p = a.pts;
  const int64_t begin = p.offsets[f], n = p.offsets[f + 1] - begin;
  PoseConsts pc;
  make_pose_consts(p.pose7, &pc);
  double plane[4], m[3], c;
#pragma unroll
  for (int k = 0; k < 4; ++k) plane[k] = p.plane[f * 4 + k];
  frame_consts(pc, plane, m, &c);
  auto key_of = [&](int64_t j) {
    return abs_key(point_distance(m, c, p.x[j], p.y[j], p.z != nullptr ? p.z[j] : 0.0));
  };
  const double nan = __longlong_as_double(0x7FF8000000000000ll);
  if (n <= kFrameSortMax) {
    int P = 1;
    while (P < n) P <<= 1;
    if (threadIdx.x == 0) s_valid = 0;
    __syncthreads();
    unsigned valid = 0;
    for (int i = threadIdx.x; i < P; i += kQuantThreads) {
      uint64_t key = ~0ull;  // padding and NaN sort last
      if (i < n) {
        const uint64_t k = key_of(begin + i);
        if (k < kKeyNanMin) {
          key = k;
          ++valid;
        }
      }
      s_buf[i] = key;
    }
    if (valid) atomicAdd(&s_valid, (unsigned long long)valid);
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = threadIdx.x; i < P; i += kQuantThreads) {
          const int l = i ^ j;
          if (l > i) {
            const unsigned long long u = s_buf[i], v = s_buf[l];
            if ((u > v) == ((i & k) == 0)) {
              s_buf[i] = v;
              s_buf[l] = u;
            }
          }
        }
        __syncthreads();
      }
    }
    const uint64_t nv = s_valid;
    if ((int)threadIdx.x < a.n_q)
      a.values[f * a.n_q + threadIdx.x] = nv == 0 ? nan : __longlong_as_double((long long)s_buf[quantile_rank(a.q[threadIdx.x], nv)]);
    if (threadIdx.x == 0) a.n_valid[f] = (int64_t)nv;
    return;
  }
  // a large frame: the radix select of clc_quantile_plan.h on this block, one pass over the frame's points per digit
  if (threadIdx.x == 0) qsel_start(&s_sel, a.n_q, a.q);
  __syncthreads();
  while (!qsel_done(s_sel)) {
    const int d = qsel_digit(s_sel, kFrameBinsLog2), bits = s_sel.bits, n_pre = s_sel.n_pre;
    for (int b = threadIdx.x; b < (n_pre << d); b += kQuantThreads) s_buf[b] = 0;
    __syncthreads();
    for (int64_t j = threadIdx.x; j < n; j += kQuantThreads) {
      const int bin = qsel_bin(bits, n_pre, s_sel.pre, d, key_of(begin + j));
      if (bin >= 0) atomicAdd(&s_buf[bin], 1ull);
    }
    __syncthreads();
    if (threadIdx.x == 0) qsel_update(&s_sel, s_buf, d);
    __syncthreads();
  }
  if ((int)threadIdx.x < a.n_q)
    a.values[f * a.n_q + threadIdx.x] = s_sel.n_valid == 0 ? nan : __longlong_as_double((long long)qsel_key(s_sel, threadIdx.x));
  if (threadIdx.x == 0) a.n_valid[f] = (int64_t)s_sel.n_valid;
}

}  // namespace clc
