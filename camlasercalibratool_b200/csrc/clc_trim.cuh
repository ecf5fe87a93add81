// clc_trim.cuh -- the two device passes of clc_problem_trim / clc_group_trim: the points of a device-resident problem whose
// distance to their board exceeds their frame's threshold are dropped, and the kept ones copied into the SoA arrays of a new
// problem, without a host round trip of the points (the plan between the passes is clc_trim_plan.h).
//
// Mark pass, one launch per source shard: block b owns source points [b * kTrimTile, (b + 1) * kTrimTile).  It finds the frame of
// its first point once, every thread then walks the frame boundaries through its own points.  Output: a keep bitmask (bit `lane`
// of word w is point 32 w + lane), the kept count of every tile and of every frame (integer atomics, so the counts do not depend
// on the order the blocks run in).
//
// Gather pass, one launch per destination shard: block b owns destination points [b * kTrimTile, (b + 1) * kTrimTile) of its shard.
// It walks the source tiles that feed it (the first one is the plan's), ranks their kept points with __popc over the mask words and
// a scan of the tile's word counts, and copies the points whose rank falls into its own range.  The blocks after the tiles copy
// the per-frame arrays, one thread per frame.  A source shard on another device of an in-process group is read through its own
// device pointers, under the pool grants of the subset gather (gather_shards, clc_api.cu).
#pragma once

#include "clc_kernels.cuh"
#include "clc_trim_plan.h"

namespace clc {

constexpr int kTrimThreads = 256;
constexpr int kTrimPerThread = (int)(kTrimTile / kTrimThreads);  // points per thread and tile
constexpr int kTrimWords = (int)(kTrimTile / 32);                // mask words per tile
static_assert(kTrimTile % kTrimThreads == 0 && kTrimWords == 64, "the gather scans a tile's mask words two per lane");

struct TrimMarkArgs {
  const double* x;
  const double* y;
  const double* z;  // nullptr: every z is known to be 0
  const double* plane;
  const int64_t* offsets;
  const double* max_abs_e;  // [n_frames]
  int64_t n_frames, n_points;
  double pose7[7];
  uint32_t* mask;                   // [n_tiles * kTrimWords]
  int64_t* tile_kept;               // [n_tiles]
  unsigned long long* frame_kept;   // [n_frames], zero on entry
};

// The frame holding point j (the last frame whose start is <= j), searched forward from frame f, which starts at or before j:
// galloping, then bisection, so a thread that crosses many short or empty frames at once pays O(log) loads.
__device__ __forceinline__ int64_t trim_frame_of(const int64_t* off, int64_t n_frames, int64_t f, int64_t j) {
  int64_t lo = f, hi = f + 1, step = 1;
  while (hi < n_frames && off[hi] <= j) {
    lo = hi;
    step *= 2;
    hi = lo + step;
  }
  hi = min(hi, n_frames);  // off[lo] <= j < off[hi]
  while (hi - lo > 1) {
    const int64_t mid = lo + (hi - lo) / 2;
    if (off[mid] <= j) lo = mid;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kTrimThreads) clc_trim_mark_kernel(TrimMarkArgs a) {
  __shared__ int64_t s_first;
  __shared__ int s_count[kTrimThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t t0 = (int64_t)blockIdx.x * kTrimTile;
  // the loads first: they do not depend on the frames, so all of them are in flight at once
  double X[kTrimPerThread], Y[kTrimPerThread], Z[kTrimPerThread];
#pragma unroll
  for (int i = 0; i < kTrimPerThread; ++i) {
    const int64_t j = t0 + i * kTrimThreads + threadIdx.x;
    const bool in = j < a.n_points;
    X[i] = in ? a.x[j] : 0.0;
    Y[i] = in ? a.y[j] : 0.0;
    Z[i] = in && a.z != nullptr ? a.z[j] : 0.0;
  }
  if (warp == 0) {
    // the frame of the tile's first point: a 32-way search by warp 0, about log32(n_frames) dependent loads (a bisection's
    // log2 chain of loads would hold every block for microseconds, longer than its share of the stream)
    int64_t lo = 0, hi = a.n_frames;  // offsets[lo] <= t0 < offsets[hi]
    while (hi - lo > 1) {
      const int64_t probe = lo + 1 + (hi - lo - 1) * lane / 32;  // in (lo, hi), non-decreasing over the lanes
      const unsigned below = __ballot_sync(0xffffffffu, a.offsets[probe] <= t0);
      const int n = __popc(below);  // the lanes whose probe starts at or before t0 come first
      const int64_t new_lo = n > 0 ? __shfl_sync(0xffffffffu, probe, n - 1) : lo;
      hi = n < 32 ? __shfl_sync(0xffffffffu, probe, n < 32 ? n : 0) : hi;
      lo = new_lo;
    }
    if (lane == 0) s_first = lo;
  }
  PoseConsts pc;
  make_pose_consts(a.pose7, &pc);
  __syncthreads();
  int64_t f = -1, f_end = 0;
  double m[3], c = 0.0, tau = 0.0;
  auto set_frame = [&](int64_t g) {
    double plane[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) plane[k] = a.plane[g * 4 + k];
    frame_consts(pc, plane, m, &c);
    tau = a.max_abs_e[g];
    f = g;
    f_end = a.offsets[g + 1];
  };
  set_frame(s_first);
  int count = 0;
#pragma unroll
  for (int i = 0; i < kTrimPerThread; ++i) {
    const int64_t j = t0 + i * kTrimThreads + threadIdx.x;
    bool keep = false;
    int64_t fj = -1;
    if (j < a.n_points) {
      if (f_end <= j) set_frame(trim_frame_of(a.offsets, a.n_frames, f, j));
      keep = fabs(point_distance(m, c, X[i], Y[i], Z[i])) <= tau;  // a NaN distance is never kept
      fj = f;
    }
    const unsigned word = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) {
      a.mask[(int64_t)blockIdx.x * kTrimWords + i * (kTrimThreads / 32) + warp] = word;
      count += __popc(word);
    }
    // one atomic per frame and warp: the lowest kept lane of every frame adds the frame's kept lanes
    const unsigned same = __match_any_sync(0xffffffffu, fj) & word;
    if (keep && lane == __ffs(same) - 1) atomicAdd(&a.frame_kept[fj], (unsigned long long)__popc(same));
  }
  if (lane == 0) s_count[warp] = count;
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t total = 0;
#pragma unroll
    for (int w = 0; w < kTrimThreads / 32; ++w) total += s_count[w];
    a.tile_kept[blockIdx.x] = total;
  }
}

struct TrimSource {
  const double* x;
  const double* y;
  const double* z;  // nullptr: every z of this source is known to be 0
  const uint32_t* mask;
  const double* frame_pose;
  const double* edge_pt;          // nullptr: no edge residuals
  const double* frame_pose_true;  // nullptr: none
};

struct TrimGatherArgs {
  TrimSource src[kMaxRanks];
  int64_t src_tile_begin[kMaxRanks + 1];   // global index of every source shard's first tile; [n_src] = all tiles
  int64_t src_frame_begin[kMaxRanks + 1];  // global index of every source shard's first frame; [n_src] = all frames
  int n_src;
  const int64_t* tile_prefix;  // [all tiles + 1]: kept points before every source tile (TrimPlan)
  const int64_t* first_tile;   // [n_tiles]: the first source tile feeding every destination tile
  int64_t point_begin;         // global kept index of the shard's first point
  int64_t n_points, n_tiles;
  int64_t frame_begin, n_frames;  // global index of the shard's first frame, its frames
  double* x;
  double* y;
  double* z;  // nullptr: the destination has no z stream
  double* frame_pose;
  double* edge_pt;
  double* frame_pose_true;
  int* nonplanar;  // raised when a copied z is not exactly 0 (NaN included), the predicate of clc_aos_to_soa_kernel
};

__global__ void __launch_bounds__(kTrimThreads) clc_trim_gather_kernel(TrimGatherArgs a) {
  if ((int64_t)blockIdx.x < a.n_tiles) {
    __shared__ uint32_t s_word[kTrimWords];
    __shared__ int s_before[kTrimWords];  // kept points of the tile before word w
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned below = (1u << lane) - 1u;
    const int64_t lo = a.point_begin + (int64_t)blockIdx.x * kTrimTile;
    const int64_t hi = min(lo + kTrimTile, a.point_begin + a.n_points);
    const int64_t n_src_tiles = a.src_tile_begin[a.n_src];
    bool off = false;
    int s = 0;
    for (int64_t g = a.first_tile[blockIdx.x]; g < n_src_tiles; ++g) {
      const int64_t base = a.tile_prefix[g];
      if (base >= hi) break;
      if (a.tile_prefix[g + 1] == base) continue;  // no kept point
      while (g >= a.src_tile_begin[s + 1]) ++s;
      const TrimSource& src = a.src[s];
      const int64_t t0 = (g - a.src_tile_begin[s]) * kTrimTile;  // the tile's first point in its source shard
      if (warp == 0) {
        const uint32_t w0 = src.mask[t0 / 32 + 2 * lane], w1 = src.mask[t0 / 32 + 2 * lane + 1];
        const int n0 = __popc(w0), n = n0 + __popc(w1);
        int incl = n;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int v = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += v;
        }
        s_word[2 * lane] = w0;
        s_word[2 * lane + 1] = w1;
        s_before[2 * lane] = incl - n;
        s_before[2 * lane + 1] = incl - n + n0;
      }
      __syncthreads();
      const int zmode = a.z == nullptr ? 0 : (src.z != nullptr ? 1 : 2);  // no z stream, copy z, write z = 0
      double X[kTrimPerThread], Y[kTrimPerThread], Z[kTrimPerThread];
      int64_t dst[kTrimPerThread];
      // every load of the tile before any store: the source and destination arrays are not known to be apart
#pragma unroll
      for (int i = 0; i < kTrimPerThread; ++i) {
        const int w = i * (kTrimThreads / 32) + warp;
        const uint32_t word = s_word[w];
        const int64_t rank = base + s_before[w] + __popc(word & below);
        const bool take = ((word >> lane) & 1u) && rank >= lo && rank < hi;
        dst[i] = take ? rank - a.point_begin : -1;
        const int64_t j = t0 + i * kTrimThreads + threadIdx.x;
        X[i] = take ? src.x[j] : 0.0;
        Y[i] = take ? src.y[j] : 0.0;
        Z[i] = take && zmode == 1 ? src.z[j] : 0.0;
      }
#pragma unroll
      for (int i = 0; i < kTrimPerThread; ++i) {
        if (dst[i] < 0) continue;
        a.x[dst[i]] = X[i];
        a.y[dst[i]] = Y[i];
        if (zmode != 0) a.z[dst[i]] = Z[i];
        off |= zmode == 1 && !(Z[i] == 0.0);
      }
      __syncthreads();  // s_word / s_before are overwritten by the next tile
    }
    if (a.z != nullptr && __syncthreads_or(off) && threadIdx.x == 0) atomicOr(a.nonplanar, 1);
    return;
  }
  const int64_t f = ((int64_t)blockIdx.x - a.n_tiles) * blockDim.x + threadIdx.x;
  if (f >= a.n_frames) return;
  const int64_t F = a.frame_begin + f;
  int s = 0;
  while (F >= a.src_frame_begin[s + 1]) ++s;
  const TrimSource& src = a.src[s];
  const int64_t g = F - a.src_frame_begin[s];
  for (int k = 0; k < 7; ++k) a.frame_pose[7 * f + k] = src.frame_pose[7 * g + k];
  if (a.edge_pt != nullptr)
    for (int k = 0; k < 6; ++k) a.edge_pt[6 * f + k] = src.edge_pt[6 * g + k];
  if (a.frame_pose_true != nullptr)
    for (int k = 0; k < 7; ++k) a.frame_pose_true[7 * f + k] = src.frame_pose_true[7 * g + k];
}

}  // namespace clc
