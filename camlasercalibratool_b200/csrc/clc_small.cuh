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
template <bool LOSS, bool EVAL = false>
__global__ void __cluster_dims__(kSmallCluster, 1, 1) __launch_bounds__(kSmallThreads, 1)
clc_small_lm_kernel(ProblemView pv, LmState* lm, int max_sweeps, int use_edges, const double* eval_pose, double* eval_sums) {
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned int rank = cluster.block_rank();
  __shared__ double s_w[kSmallThreads / 32][32];  // per-warp totals of the 28 sums
  __shared__ double s_blk[32];                    // this CTA's totals
  __shared__ double s_tot[32];                    // CTA 0: the cluster's totals
  __shared__ double s_pose[8];                    // CTA 0: pose of the next sweep + the `done` flag
  __shared__ unsigned long long s_core[kLmCoreWords];  // CTA 0: the LM state

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t n_threads = (int64_t)kSmallThreads * kSmallCluster;
  const int64_t gtid = (int64_t)rank * kSmallThreads + tid;
  const int64_t P = pv.n_points;
  const int64_t n_res = P + ((use_edges && pv.n_edges > 0) ? pv.n_edges : 0);

  // ---- this thread's residuals, loaded once ----
  double px[kSmallItems], py[kSmallItems], pz[kSmallItems], s2[kSmallItems];
  int pl[kSmallItems];  // plane: >= 0 frame index (pv.plane), < 0: -(edge index + 1) (pv.edge_plane); INT_MIN-like: none
  constexpr int kNone = 0x7fffffff;
#pragma unroll
  for (int j = 0; j < kSmallItems; ++j) {
    const int64_t i = gtid + (int64_t)j * n_threads;
    px[j] = py[j] = pz[j] = s2[j] = 0.0;
    pl[j] = kNone;
    if (i < P) {
      px[j] = pv.x[i];
      py[j] = pv.y[i];
      pz[j] = pv.z != nullptr ? pv.z[i] : 0.0;
      int64_t lo = 0, hi = pv.n_frames;  // offsets[lo] <= i < offsets[hi]
      while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (pv.offsets[mid] <= i) lo = mid; else hi = mid;
      }
      // frames may be empty: the frame of point i is the LAST one that starts at or before i and is non-empty, which the
      // search above finds (offsets[lo] <= i < offsets[lo + 1] because offsets is non-decreasing and i < offsets[n_frames])
      while (pv.offsets[lo + 1] <= i) ++lo;
      pl[j] = (int)lo;
      s2[j] = 1.0 / (double)(pv.offsets[lo + 1] - pv.offsets[lo]);
    } else if (i < n_res) {
      const int64_t e = i - P, f = e >> 1;
      const int64_t cnt = pv.offsets[f + 1] - pv.offsets[f];
      if (cnt > 0) {  // a frame without points has no scale: the streaming kernels skip its edge residuals too
        px[j] = pv.edge_pt[e * 3];
        py[j] = pv.edge_pt[e * 3 + 1];
        pz[j] = pv.edge_pt[e * 3 + 2];
        pl[j] = -(int)(e + 1);
        s2[j] = 1.0 / (double)cnt;
      }
    }
  }

  double pose[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) pose[i] = EVAL ? __ldcg(eval_pose + i) : __ldcg(lm->core.cand + i);
  if (!EVAL && rank == 0) {
    const unsigned long long* g_core = reinterpret_cast<const unsigned long long*>(&lm->core);
    for (int k = tid; k < kLmCoreWords; k += kSmallThreads) s_core[k] = __ldcg(g_core + k);
  }
  __syncthreads();

  for (int sw = 0; sw < max_sweeps; ++sw) {
    PoseConsts pc;
    make_pose_consts(pose, &pc);
    double acc[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) acc[k] = 0.0;
#pragma unroll
    for (int j = 0; j < kSmallItems; ++j) {
      if (pl[j] == kNone) continue;
      const double* plane = pl[j] >= 0 ? pv.plane + (int64_t)pl[j] * 4 : pv.edge_plane + (int64_t)(-pl[j] - 1) * 4;
      double pln[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) pln[k] = plane[k];
      accumulate_residual(pc, pln, px[j], py[j], pz[j], s2[j], LOSS, pv.a2, pv.inv_a2, acc);
    }
    // ---- cluster reduction, fixed order ----
    warp_transpose_sum<32>(acc, lane);  // lane L: this warp's total of sum L
    s_w[warp][lane] = acc[0];
    __syncthreads();
    if (tid < 32) {
      double t = 0.0;
#pragma unroll
      for (int wv = 0; wv < kSmallThreads / 32; ++wv) t += s_w[wv][tid];
      s_blk[tid] = t;
    }
    cluster.sync();  // every CTA's totals are in its shared memory
    if (rank == 0) {
      if (tid < 32) {
        double t = 0.0;
        for (unsigned int r = 0; r < (unsigned int)kSmallCluster; ++r) t += *cluster.map_shared_rank(&s_blk[tid], r);
        s_tot[tid] = t;
      }
      if (EVAL && tid < kNumSums) eval_sums[tid] = s_tot[tid];
      __syncthreads();
      if (!EVAL && tid == 0) {
        double sums[kNumSums];
        for (int k = 0; k < kNumSums; ++k) sums[k] = s_tot[k];
        LmCore* core = reinterpret_cast<LmCore*>(s_core);
        lm_update(core, lm->trace, sums);
        for (int i = 0; i < 7; ++i) s_pose[i] = core->cand[i];
        s_pose[7] = (double)core->done;
      }
    }
    cluster.sync();  // the next pose is in CTA 0's shared memory (and CTA 0 is done reading the other CTAs' totals)
    if (EVAL) break;
    const double* next = cluster.map_shared_rank(&s_pose[0], 0);
#pragma unroll
    for (int i = 0; i < 7; ++i) pose[i] = next[i];
    if (next[7] != 0.0) break;
  }
  if (!EVAL && rank == 0) {
    __syncthreads();
    unsigned long long* o_core = reinterpret_cast<unsigned long long*>(&lm->core);
    for (int k = tid; k < kLmCoreWords; k += kSmallThreads) o_core[k] = s_core[k];
  }
  cluster.sync();  // no CTA leaves while another may still read its shared memory
}

}  // namespace clc
