// clc_subset.cuh -- the gather of clc_problem_subset / clc_group_subset: the kept frames of a device-resident problem copied
// into the SoA arrays of a new one, without a host round trip of the points (the plan is clc_subset_plan.h).
//
// One launch per destination shard.  Blocks [0, n_tiles) each own kSubsetTile consecutive destination points and copy them from
// whichever runs of kept frames reach into the tile; the blocks after them copy the per-frame arrays, one thread per kept frame.
// A source shard on another device of an in-process group is read through its own device pointers: its arrays come from that
// device's default memory pool, which the host opens to the destination devices for the gather (subset_build, clc_api.cu).
#pragma once

#include "clc_kernels.cuh"

namespace clc {

constexpr int kSubsetThreads = 256;
constexpr int64_t kSubsetTile = 4096;  // destination points per block: 8 pairs of each stream per thread
constexpr int64_t kSubsetBlockRun = 2 * kSubsetThreads;  // pieces of runs this long are copied by the whole block ...
constexpr int64_t kSubsetWarpRun = 32;                   // ... this long by one warp, shorter ones by one thread

struct SubsetSource {
  const double* x;
  const double* y;
  const double* z;  // nullptr: every z of this source is known to be 0
  const double* frame_pose;
  const double* edge_pt;          // nullptr: no edge residuals
  const double* frame_pose_true;  // nullptr: none
};

struct SubsetArgs {
  SubsetSource src[kMaxRanks];
  const int64_t* runs;       // [n_runs][4]: source shard, source point, destination point, points -- runs with points, in order
  const int64_t* tile_run;   // [n_tiles]: the first run that reaches into tile t
  const int64_t* frame_src;  // [n_frames]: source shard * 2^40 + source frame of every destination frame
  int64_t n_runs, n_tiles, n_frames;
  double* x;
  double* y;
  double* z;  // nullptr: the destination has no z stream
  double* frame_pose;
  double* edge_pt;
  double* frame_pose_true;
  int* nonplanar;  // raised when a copied z is not exactly 0 (NaN included), the predicate of clc_aos_to_soa_kernel
};

constexpr int64_t kSubsetShardShift = 40;

// dst[i] = src[i + d] for every stream, i in [lo, hi).  The destination arrays are 16-byte aligned, so pairs starting at an even
// index are stored as double2; they are loaded as double2 too when d is even, else as two doubles.  Copied bit for bit.
// zmode 0: no z stream, 1: copy z, 2: write z = 0 (the source has none).  The copy is shared by `width` threads (the block,
// a warp or one thread), this one being number `rank`.  Returns whether a copied z is not exactly 0.
__device__ __forceinline__ bool subset_copy_run(const SubsetSource& s, const SubsetArgs& a, int64_t lo, int64_t hi, int64_t d,
                                                int zmode, int rank, int width) {
  bool off = false;
  auto one = [&](int64_t i) {
    a.x[i] = __ldcs(s.x + i + d);
    a.y[i] = __ldcs(s.y + i + d);
    if (zmode == 1) {
      const double v = __ldcs(s.z + i + d);
      a.z[i] = v;
      off |= !(v == 0.0);
    } else if (zmode == 2) {
      a.z[i] = 0.0;
    }
  };
  int64_t start = lo;
  if ((lo & 1) && lo < hi) {
    if (rank == 0) one(lo);
    start = lo + 1;
  }
  const int64_t end2 = start + ((hi - start) & ~(int64_t)1);
  if (end2 < hi && rank == width - 1) one(end2);
  const bool aligned = (d & 1) == 0;
  auto ld2 = [&](const double* p) -> double2 {
    if (aligned) return __ldcs(reinterpret_cast<const double2*>(p));
    return make_double2(__ldcs(p), __ldcs(p + 1));
  };
#pragma unroll 2
  for (int64_t i = start + 2 * (int64_t)rank; i < end2; i += 2 * (int64_t)width) {
    const double2 vx = ld2(s.x + i + d);
    const double2 vy = ld2(s.y + i + d);
    double2 vz = make_double2(0.0, 0.0);
    if (zmode == 1) vz = ld2(s.z + i + d);
    *reinterpret_cast<double2*>(a.x + i) = vx;
    *reinterpret_cast<double2*>(a.y + i) = vy;
    if (zmode != 0) *reinterpret_cast<double2*>(a.z + i) = vz;
    if (zmode == 1) off |= !(vz.x == 0.0) || !(vz.y == 0.0);
  }
  return off;
}

__global__ void __launch_bounds__(kSubsetThreads) clc_subset_gather_kernel(SubsetArgs a) {
  if ((int64_t)blockIdx.x < a.n_tiles) {
    const int64_t t0 = (int64_t)blockIdx.x * kSubsetTile, t1 = t0 + kSubsetTile;
    bool off = false;
    // The share of a run inside the tile goes to the whole block when it is long, to one warp (round robin over the warps) when
    // it is a few dozen points, to one thread (round robin) when it is shorter: many short runs -- a mask that keeps every
    // other small frame -- then keep every thread busy instead of costing one nearly empty block-wide pass each.
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int64_t n_mid = 0, n_short = 0;
    for (int64_t r = a.tile_run[blockIdx.x]; r < a.n_runs; ++r) {
      const int64_t dp = a.runs[4 * r + 2];
      if (dp >= t1) break;
      const int64_t lo = max(t0, dp), hi = min(t1, dp + a.runs[4 * r + 3]);
      int rank, width;
      if (hi - lo >= kSubsetBlockRun) {
        rank = threadIdx.x, width = kSubsetThreads;
      } else if (hi - lo >= kSubsetWarpRun) {
        if (n_mid++ % (kSubsetThreads / 32) != warp) continue;
        rank = lane, width = 32;
      } else {
        if (n_short++ % kSubsetThreads != threadIdx.x) continue;
        rank = 0, width = 1;
      }
      const SubsetSource& s = a.src[a.runs[4 * r]];
      const int zmode = a.z == nullptr ? 0 : (s.z != nullptr ? 1 : 2);
      off |= subset_copy_run(s, a, lo, hi, a.runs[4 * r + 1] - dp, zmode, rank, width);
    }
    if (a.z != nullptr && __syncthreads_or(off) && threadIdx.x == 0) atomicOr(a.nonplanar, 1);
    return;
  }
  const int64_t f = ((int64_t)blockIdx.x - a.n_tiles) * blockDim.x + threadIdx.x;
  if (f >= a.n_frames) return;
  const int64_t code = a.frame_src[f];
  const SubsetSource& s = a.src[code >> kSubsetShardShift];
  const int64_t g = code & (((int64_t)1 << kSubsetShardShift) - 1);
  for (int k = 0; k < 7; ++k) a.frame_pose[7 * f + k] = s.frame_pose[7 * g + k];
  if (a.edge_pt != nullptr)
    for (int k = 0; k < 6; ++k) a.edge_pt[6 * f + k] = s.edge_pt[6 * g + k];
  if (a.frame_pose_true != nullptr)
    for (int k = 0; k < 7; ++k) a.frame_pose_true[7 * f + k] = s.frame_pose_true[7 * g + k];
}

}  // namespace clc
