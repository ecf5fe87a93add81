// clc_segments.cuh -- W independent LM solves over runs of consecutive frames (segments) of one problem, sharing every sweep
// (clc_eval_segments, clc_information_segments, clc_solve_lm_segments).
//
// Every residual depends on the pose of one segment only, so one pass over the points serves every segment.  One LM iteration:
//   1. clc_segment_consts_kernel   m = R^T n, c = n.t + d of every frame and edge residual at its segment's current pose;
//   2. clc_sweep_kernel<.., kModeSegments, ..>   every frame's raw moments and cost into its own row, a split frame's pieces into
//                                  per-warp slots (as the per-frame report, with the frame constants of step 1 and the points
//                                  outside a piece masked out);
//   3. clc_segment_fixup_kernel    every frame's share of the 28 sums at its segment's pose (zeros for an empty frame);
//   4. clc_segment_chunk_kernel    level 1 of the fixed reduction plan (clc_segment_plan.h): the rows of every chunk;
//   5. clc_segment_lm_kernel       level 2: the chunk partials of every segment, then lm_update on the segment's own LmCore.
// Steps 4 and 5 are templates on the row width and the number of tangent columns: the time offset (clc_time_offset.cuh) runs
// them as one segment of 36-wide rows and a 7-column LmCoreN<7>.
// Every kernel of the iteration is a no-op once every segment has terminated (`done`, raised by the last one).
// The kernels at the end of the file run the same iteration for one calibration at many poses.
#pragma once

#include "clc_kernels.cuh"
#include "clc_segment_plan.h"

namespace clc {

// The frame constants of frame f at `pose`: m, c of the frame (and, with edges, of its two edge residuals, behind the frames':
// SweepArgs::seg_consts).
__device__ __forceinline__ void frame_consts_at(const ProblemView& pv, const double* pose_src, int64_t f, int edges,
                                                double* __restrict__ consts) {
  double pose[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) pose[k] = pose_src[k];
  PoseConsts pc;
  make_pose_consts(pose, &pc);
  double plane[4], m[3], c;
#pragma unroll
  for (int k = 0; k < 4; ++k) plane[k] = pv.plane[f * 4 + k];
  frame_consts(pc, plane, m, &c);
  consts[f * 4] = m[0]; consts[f * 4 + 1] = m[1]; consts[f * 4 + 2] = m[2]; consts[f * 4 + 3] = c;
  if (edges) {
    for (int k = 0; k < 2; ++k) {
      const int64_t i = 2 * f + k;
      frame_consts(pc, pv.edge_plane + i * 4, m, &c);
      double* o = consts + (pv.n_frames + i) * 4;
      o[0] = m[0]; o[1] = m[1]; o[2] = m[2]; o[3] = c;
    }
  }
}

// One thread per frame: the frame constants at the pose of its segment, pose s at poses[s * pose_stride] (the caller's poses, or
// the candidate of segment s's LmCore).
__global__ void clc_segment_consts_kernel(ProblemView pv, const int32_t* __restrict__ frame_seg, const double* poses,
                                          int64_t pose_stride, int edges, const int* done, double* __restrict__ consts) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= pv.n_frames || (done != nullptr && *done != 0)) return;
  frame_consts_at(pv, poses + (int64_t)frame_seg[f] * pose_stride, f, edges, consts);
}

// Expands the summed pieces of frame f (S = 10 moments, cost_term as expand_lm takes it) into its row of kNumSums doubles at its
// segment's pose: m, c of the frame and of its two edge residuals come from `consts` (SweepArgs::seg_consts).
__device__ __forceinline__ void segment_row_write(const ProblemView& pv, const double* consts, int64_t f, const double* S,
                                                  double cost_term, int loss, bool edges, double* row) {
  double plane[4], m[3];
#pragma unroll
  for (int k = 0; k < 4; ++k) plane[k] = pv.plane[f * 4 + k];
#pragma unroll
  for (int k = 0; k < 3; ++k) m[k] = consts[f * 4 + k];
  const double c = consts[f * 4 + 3];
  const double s2 = 1.0 / (double)(pv.offsets[f + 1] - pv.offsets[f]);
  double out[kNumSums];
#pragma unroll
  for (int k = 0; k < kNumSums; ++k) out[k] = 0.0;
  expand_lm(plane, m, c, s2, S, loss, cost_term, pv.a2, out);
  if (edges) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int64_t i = 2 * f + k;
      const double* ec = consts + (pv.n_frames + i) * 4;
      edge_residual_at(pv.edge_plane + i * 4, ec, ec[3], pv.edge_pt + i * 3, s2, loss, pv.a2, pv.inv_a2, out);
    }
  }
#pragma unroll
  for (int k = 0; k < kNumSums; ++k) row[k] = out[k];
}

// The summed moments S[10] and cost_term (as expand_lm takes them) of frame f after a kModeSegments or kModePoses sweep: a whole
// frame's raw row (kSegRawDoubles), or a split frame's pieces added in warp order.  false, with S and cost_term untouched, for an
// empty frame.
template <int LOSS>
__device__ __forceinline__ bool segment_frame_moments(const ProblemView& pv, int64_t f, const double* __restrict__ raw,
                                                      const double* __restrict__ slots, double* S, double* cost_term) {
  const int64_t fs = pv.offsets[f], fe = pv.offsets[f + 1];
  if (fe <= fs) return false;
  int64_t w0, w1;
  frame_warps(fs, fe, pv.per_warp, &w0, &w1);
#pragma unroll
  for (int k = 0; k < 10; ++k) S[k] = 0.0;
  double ct = 0.0;
  for (int64_t w = w0; w <= w1; ++w) {
    const double* s = w0 == w1 ? raw + f * kSegRawDoubles : slots + frame_slot(w, w0);
#pragma unroll
    for (int k = 0; k < 10; ++k) S[k] += s[k];
    ct += LOSS == kLossCauchy ? log(s[10]) + s[11] * 0.693147180559945309417232121458 : s[10];
  }
  *cost_term = ct;
  return true;
}

// Expansion of frame f after a kModeSegments or kModePoses sweep, clc_frame_fixup_kernel's sibling.  An empty frame gets a row of
// zeros; the frame's summed moments (segment_frame_moments) are expanded at the pose of `consts`.
template <int LOSS>
__device__ __forceinline__ void segment_fixup_frame(const ProblemView& pv, const double* __restrict__ consts, int edges, int64_t f,
                                                    const double* __restrict__ raw, const double* __restrict__ slots,
                                                    double* __restrict__ rows) {
  double* row = rows + f * kNumSums;
  double S[10], cost_term;
  if (!segment_frame_moments<LOSS>(pv, f, raw, slots, S, &cost_term)) {
    for (int k = 0; k < kNumSums; ++k) row[k] = 0.0;
    return;
  }
  segment_row_write(pv, consts, f, S, cost_term, LOSS, edges != 0, row);
}

// One thread per frame, at its segment's pose.
template <int LOSS>
__global__ void clc_segment_fixup_kernel(ProblemView pv, const double* __restrict__ consts, int edges, const int* done,
                                         const double* __restrict__ raw, const double* __restrict__ slots,
                                         double* __restrict__ rows) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= pv.n_frames || (done != nullptr && *done != 0)) return;
  segment_fixup_frame<LOSS>(pv, consts, edges, f, raw, slots, rows);
}

// Level 1: one warp per chunk, lane k adds outputs k, k + 32, ... (< W) of the chunk's W-wide rows in frame order.
constexpr int kSegWarpsPerBlock = 4;
template <int W>
__global__ void __launch_bounds__(32 * kSegWarpsPerBlock)
clc_segment_chunk_kernel(const double* __restrict__ rows, const int64_t* __restrict__ chunk_offsets, int64_t n_chunks,
                         const int* done, double* __restrict__ partials) {
  const int64_t ch = (int64_t)blockIdx.x * kSegWarpsPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (ch >= n_chunks || lane >= W || (done != nullptr && *done != 0)) return;
  const int64_t a = chunk_offsets[ch], b = chunk_offsets[ch + 1];
#pragma unroll
  for (int j = 0; j < (W + 31) / 32; ++j) {
    const int k = lane + 32 * j;
    if (k >= W) break;
    double acc = 0.0;
    for (int64_t r = a; r < b; ++r) acc += rows[r * W + k];
    partials[ch * W + k] = acc;
  }
}

// Level 2 + LM over D tangent columns: one warp per segment.  Lane k adds outputs k, k + 32, ... (< kLmSums<D>) of the
// segment's chunk partials in chunk order (an empty segment sums to zeros) into sums[s] (may be nullptr); with cores, lane 0 then
// runs lm_update on segment s's LmCoreN<D>, staged in shared memory.  A segment that terminates in this call leaves `running`; the
// last one raises `done`.
template <int D>
__global__ void __launch_bounds__(32 * kSegWarpsPerBlock)
clc_segment_lm_kernel(const double* __restrict__ partials, const int64_t* __restrict__ seg_chunks, int64_t n_segments,
                      double* sums, LmCoreN<D>* cores, clc_lm_iteration* trace, int trace_cap, int* running, int* done) {
  constexpr int W = kLmSums<D>, kWords = kLmWords<D>;
  __shared__ unsigned long long s_core[kSegWarpsPerBlock][kWords];
  __shared__ double s_sums[kSegWarpsPerBlock][(W + 31) / 32 * 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * kSegWarpsPerBlock + warp;
  if (s >= n_segments || (done != nullptr && *done != 0)) return;
  const int64_t c0 = seg_chunks[s], c1 = seg_chunks[s + 1];
#pragma unroll
  for (int j = 0; j < (W + 31) / 32; ++j) {
    const int k = lane + 32 * j;
    if (k >= W) break;
    double acc = 0.0;
    for (int64_t c = c0; c < c1; ++c) acc += partials[c * W + k];
    s_sums[warp][k] = acc;
    if (sums != nullptr) sums[s * W + k] = acc;
  }
  if (cores == nullptr) return;
  unsigned long long* g_core = reinterpret_cast<unsigned long long*>(cores + s);
  for (int k = lane; k < kWords; k += 32) s_core[warp][k] = g_core[k];
  __syncwarp();
  if (lane == 0) {
    LmCoreN<D>* core = reinterpret_cast<LmCoreN<D>*>(s_core[warp]);
    const bool was_running = core->done == 0;
    lm_update(core, TraceRows{trace != nullptr ? trace + s * trace_cap : nullptr, trace_cap}, s_sums[warp]);
    if (was_running && core->done != 0 && atomicSub(running, 1) == 1) *done = 1;
  }
  __syncwarp();
  for (int k = lane; k < kWords; k += 32) g_core[k] = s_core[warp][k];
}


// ---- one calibration at many poses (clc_eval_poses, clc_solve_lm_starts) ----------------------------------------------------
// Pose k owns every frame, so the K poses form a pose-major virtual segmentation of K * n_frames rows (segment k = rows
// [k n_frames, (k + 1) n_frames)) that the chunk and LM kernels above reduce and update unchanged.  Only the running poses are
// evaluated: pose_active[0 .. *pose_count) lists them (clc_pose_compact_kernel), and blockIdx.y walks that list.

// One thread per frame and running pose: pose k's frame constants at poses[k * pose_stride], to consts + k * consts_stride.
__global__ void clc_pose_consts_kernel(ProblemView pv, const int* __restrict__ pose_active, const int* pose_count, const double* poses,
                                       int64_t pose_stride, int edges, double* __restrict__ consts, int64_t consts_stride) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= pv.n_frames || (int)blockIdx.y >= *pose_count) return;
  const int64_t k = pose_active[blockIdx.y];
  frame_consts_at(pv, poses + k * pose_stride, f, edges, consts + k * consts_stride);
}

// One thread per frame and running pose: the rows of pose k after a kModePoses sweep (strides as SweepArgs' pose_*_stride).
template <int LOSS>
__global__ void clc_pose_fixup_kernel(ProblemView pv, const int* __restrict__ pose_active, const int* pose_count,
                                      const double* __restrict__ consts, int64_t consts_stride, int edges,
                                      const double* __restrict__ raw, int64_t raw_stride, const double* __restrict__ slots,
                                      int64_t slots_stride, double* __restrict__ rows) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= pv.n_frames || (int)blockIdx.y >= *pose_count) return;
  const int64_t k = pose_active[blockIdx.y];
  segment_fixup_frame<LOSS>(pv, consts + k * consts_stride, edges, f, raw + k * raw_stride, slots + k * slots_stride,
                            rows + k * pv.n_frames * kNumSums);
}

// One block of kPoseCompactThreads: the poses whose LmCore is still running, in increasing order, to pose_active[0 .. *pose_count).
constexpr int kPoseCompactThreads = 1024;
__global__ void __launch_bounds__(kPoseCompactThreads)
clc_pose_compact_kernel(const LmCore* __restrict__ cores, int n_poses, int* __restrict__ pose_active, int* pose_count) {
  __shared__ int s_warp[kPoseCompactThreads / 32];
  const int k = threadIdx.x, lane = k & 31, warp = k >> 5;
  const bool running = k < n_poses && cores[k].done == 0;
  const unsigned ballot = __ballot_sync(0xffffffffu, running);
  if (lane == 0) s_warp[warp] = __popc(ballot);
  __syncthreads();
  int base = 0;
  for (int w = 0; w < warp; ++w) base += s_warp[w];
  if (running) pose_active[base + __popc(ballot & ((1u << lane) - 1u))] = k;
  if (k == kPoseCompactThreads - 1) *pose_count = base + __popc(ballot);
}

}  // namespace clc
