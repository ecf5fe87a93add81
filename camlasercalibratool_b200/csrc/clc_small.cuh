// clc_small.cuh -- the whole Levenberg-Marquardt solve of a SMALL problem in one launch of one thread-block cluster.
//
// The reference's own problems are tiny for an H100: 50 board poses x <= 180 laser points (reference
// main/calibr_simulation.cpp:34,79), a few thousand residuals.  The streaming sweep kernel (clc_kernels.cuh) is built for
// 10^7..10^9 points -- per-warp TMA rings, moment expansion, a one-block-per-SM gather -- and at this size spends its time
// in machinery even when it loops inside one launch.  Here instead
//   * one cluster of 8 CTAs x 256 threads; every thread loads its <= 8 residuals (point, frame index, 1/#points of the frame)
//     ONCE into registers and keeps them for the whole solve;
//   * per LM iteration every thread evaluates its residuals against the current pose and accumulates the 28 sums (21 of H,
//     6 of g, the robust cost) directly -- no moments: with a handful of points per thread the per-frame bookkeeping would
//     cost more than the 45 flops it saves;
//   * warp transposing butterfly -> shared memory -> distributed shared memory of CTA 0 (fixed order: the result is
//     bit-reproducible), lm_update on one thread of CTA 0 (the same Ceres state machine as everywhere, clc_lm.cuh), the next
//     pose handed back through distributed shared memory: two cluster barriers per iteration, no global-memory round trip.
// Same arithmetic per residual as reference src/LaseCamCalCeres.cpp:43-66 (+ CauchyLoss :249, scale :239-240, edge residuals
// :258-294); the sums differ from the streaming kernels' only by summation order.
#pragma once

#include <cooperative_groups.h>

#include "clc_kernels.cuh"

namespace clc {

namespace cg = cooperative_groups;

constexpr int kSmallThreads = 256;
constexpr int kSmallCluster = 8;
constexpr int kSmallItems = 8;  // residuals per thread
constexpr int64_t kSmallMaxResiduals = (int64_t)kSmallThreads * kSmallCluster * kSmallItems;  // 16384

// EVAL: one evaluation at `eval_pose` instead of the LM loop -- the 28 sums go to `eval_sums` (clc_eval / clc_information of a
// small problem: the same residual code, no LM state touched).
template <int LOSS, bool EVAL = false>
__global__ void __cluster_dims__(kSmallCluster, 1, 1) __launch_bounds__(kSmallThreads, 1)
clc_small_lm_kernel(ProblemView pv, LmState* lm, int max_sweeps, int use_edges, const double* eval_pose, double* eval_sums) {
#include "clc_small_body.inl"
}

// One launch of many clusters (clc_eval_poses, clc_solve_lm_starts): cluster k runs exactly what a one-cluster launch runs, with
// lm[k] (the LM loop), or eval_pose[7 k ..] and eval_sums[kNumSums k ..] (EVAL).
template <int LOSS, bool EVAL = false>
__global__ void __cluster_dims__(kSmallCluster, 1, 1) __launch_bounds__(kSmallThreads, 1)
clc_small_poses_kernel(ProblemView pv, LmState* lm, int max_sweeps, int use_edges, const double* eval_pose, double* eval_sums) {
  {
    const int64_t slot = blockIdx.x / kSmallCluster;
    if (EVAL) {
      eval_pose += 7 * slot;
      eval_sums += kNumSums * slot;
    } else {
      lm += slot;
    }
  }
#include "clc_small_body.inl"
}

}  // namespace clc
