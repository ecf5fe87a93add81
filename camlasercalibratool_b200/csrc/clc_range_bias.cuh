// clc_range_bias.cuh -- the laser's range offset b and range scale s, estimated together with the extrinsic (clc_eval_range_bias,
// clc_information_range_bias, clc_solve_lm_range_bias, clc_problem_range_correct).
//
// A point p the laser reported at range r = |p| along u = p / r is taken to lie at range (1 + s) r + b on the same ray:
//   p' = (1 + s) p + b u = kappa p,   kappa = (1 + s) + b / r         (r == 0: the p / r terms are 0, p' = (1 + s) p = 0)
// and its residual is the reference's at p':  e = m.p' + c = kappa (m.p) + c  (m = R^T n, c = n.t + d; times the frame's scale).
// The tangent space is (tx ty tz rx ry rz b s): the pose columns of expand_lm taken at p', J_b = (m.p) / r, J_s = m.p.  Every
// column and e are linear in a = (p, p / r, 1), so a frame's 45 sums are images of its weighted moments sum w a a^T: the 25 the
// sweep accumulates (RangeMoments, clc_kernels.cuh; 14 of them on a planar problem).  One iteration, on the segmented path with
// one segment (clc_segments.cuh):
//   1. clc_segment_consts_kernel   m, c of every frame at the pose of the point (pose7, b, s) -- the LM candidate in a solve;
//   2. clc_sweep_kernel<.., kModeRange, ..>   every frame's raw row of kRangeRawDoubles (b, s read from the same point);
//   3. clc_range_fixup_kernel     every frame's moments expanded into its row of kRangeSums (expand_lm_range);
//   4. clc_segment_chunk_kernel<kRangeSums>   level 1 of the segment plan;
//   5. clc_segment_lm_kernel<8>              level 2, then lm_update on LmCoreN<8> (clc_lm.cuh).
// The host part (everything CLC_HD) also compiles with g++ for the CPU tests.
#pragma once

#include "clc_expand.cuh"
#include "clc_lm.cuh"

namespace clc {

constexpr int kRangeSums = kLmSums<8>;  // 36 upper-tri of the 8x8 H (tx ty tz rx ry rz b s, row-major, i <= j) + 8 g + 1 cost
constexpr int kRangeMomentCount = 25;   // the layout of M below (== kRangeMoments of the sweep)

// M layout (the sweep's raw row): M[0] = sum w, M[1..3] = sum w p, M[4..9] = sum w p p^T (xx xy xz yy yz zz),
// M[10..12] = sum w p / r, M[13..18] = sum w p p^T / r, M[19..24] = sum w p p^T / r^2.
// Adds the piece's contribution to out[kRangeSums] at the frame normal n, m = R^T n, c = n.t + d and (b, s): the 6x6 block, g
// and the cost are expand_lm's on the moments of p' (sum w kappa p and sum w kappa^2 p p^T), and with
// Mb = (1 + s) P1 + b P2 = sum w kappa p (p / r)^T, Ms = (1 + s) P0 + b P1 = sum w kappa p p^T:
//   H_t,b = s2 n (m.Q)     H_theta,b = s2 (Mb m) x m    H_bb = s2 m^T P2 m    g_b = s2 (m^T Mb m + c m.Q)
//   H_t,s = s2 n (m.S1)    H_theta,s = s2 (Ms m) x m    H_bs = s2 m^T P1 m    g_s = s2 (m^T Ms m + c m.S1)
//                                                        H_ss = s2 m^T P0 m
// (P0 = sum w p p^T, P1 = sum w p p^T / r, P2 = sum w p p^T / r^2, Q = sum w p / r.)  cost_term, loss and a2 as expand_lm.
CLC_HD void expand_lm_range(const double* n, const double* m, double c, double b, double s, double s2, const double* M, int loss,
                            double cost_term, double a2, double* out) {
  const double sg = 1.0 + s;
  const double* S1 = M + 1;
  const double* P0 = M + 4;
  const double* Q = M + 10;
  const double* P1 = M + 13;
  const double* P2 = M + 19;
  // the moments of p': S0, sum w kappa p, sum w kappa^2 p p^T
  double Sp[10];
  Sp[0] = M[0];
  for (int i = 0; i < 3; ++i) Sp[1 + i] = sg * S1[i] + b * Q[i];
  for (int i = 0; i < 6; ++i) Sp[4 + i] = sg * sg * P0[i] + 2.0 * sg * b * P1[i] + b * b * P2[i];
  const double plane[4] = {n[0], n[1], n[2], 0.0};  // expand_lm reads the normal only
  double o[kNumSums];
  for (int k = 0; k < kNumSums; ++k) o[k] = 0.0;
  expand_lm(plane, m, c, s2, Sp, loss, cost_term, a2, o);
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) out[tri<8>(i, j)] += o[tri(i, j)];
  for (int i = 0; i < 6; ++i) out[36 + i] += o[21 + i];
  out[44] += o[27];
  // symmetric 3x3 (xx xy xz yy yz zz) times m
  auto symv = [](const double* A, const double* v, double* r) {
    r[0] = A[0] * v[0] + A[1] * v[1] + A[2] * v[2];
    r[1] = A[1] * v[0] + A[3] * v[1] + A[4] * v[2];
    r[2] = A[2] * v[0] + A[4] * v[1] + A[5] * v[2];
  };
  double Mb[6], Ms[6];
  for (int i = 0; i < 6; ++i) {
    Mb[i] = sg * P1[i] + b * P2[i];
    Ms[i] = sg * P0[i] + b * P1[i];
  }
  double Mbm[3], Msm[3], P0m[3], P1m[3], P2m[3];
  symv(Mb, m, Mbm);
  symv(Ms, m, Msm);
  symv(P0, m, P0m);
  symv(P1, m, P1m);
  symv(P2, m, P2m);
  const double mQ = m[0] * Q[0] + m[1] * Q[1] + m[2] * Q[2];
  const double mS = m[0] * S1[0] + m[1] * S1[1] + m[2] * S1[2];
  double hb[3], hs[3];
  cross3(Mbm, m, hb);
  cross3(Msm, m, hs);
  for (int i = 0; i < 3; ++i) {
    out[tri<8>(i, 6)] += s2 * n[i] * mQ;
    out[tri<8>(i, 7)] += s2 * n[i] * mS;
    out[tri<8>(3 + i, 6)] += s2 * hb[i];
    out[tri<8>(3 + i, 7)] += s2 * hs[i];
  }
  out[tri<8>(6, 6)] += s2 * (m[0] * P2m[0] + m[1] * P2m[1] + m[2] * P2m[2]);
  out[tri<8>(6, 7)] += s2 * (m[0] * P1m[0] + m[1] * P1m[1] + m[2] * P1m[2]);
  out[tri<8>(7, 7)] += s2 * (m[0] * P0m[0] + m[1] * P0m[1] + m[2] * P0m[2]);
  out[42] += s2 * (m[0] * Mbm[0] + m[1] * Mbm[1] + m[2] * Mbm[2] + c * mQ);
  out[43] += s2 * (m[0] * Msm[0] + m[1] * Msm[1] + m[2] * Msm[2] + c * mS);
}

// kappa of a point: (1 + s) + b / r, r = |p|; 1 + s at r == 0 (the corrected origin stays at the origin)
CLC_HD double range_kappa(double x, double y, double z, double b, double s) {
  const double r2 = x * x + y * y + z * z;
  return r2 == 0.0 ? 1.0 + s : (1.0 + s) + b / sqrt(r2);
}

using LmCoreRange = LmCoreN<8>;

}  // namespace clc

#if defined(__CUDACC__)
#include "clc_segments.cuh"

namespace clc {

// The summed range moments M[25] and cost_term (as expand_lm takes it) of frame f after a kModeRange sweep: a whole frame's raw
// row, or a split frame's pieces added in warp order (slots kRangeRawDoubles wide).  false for an empty frame.
template <int LOSS>
__device__ __forceinline__ bool range_frame_moments(const ProblemView& pv, int64_t f, const double* __restrict__ raw,
                                                    const double* __restrict__ slots, double* M, double* cost_term) {
  const int64_t fs = pv.offsets[f], fe = pv.offsets[f + 1];
  if (fe <= fs) return false;
  int64_t w0, w1;
  frame_warps(fs, fe, pv.per_warp, &w0, &w1);
#pragma unroll
  for (int k = 0; k < kRangeMoments; ++k) M[k] = 0.0;
  double ct = 0.0;
  for (int64_t w = w0; w <= w1; ++w) {
    const double* s = w0 == w1 ? raw + f * kRangeRawDoubles
                               : slots + (w * 2 + (w == w0 ? kSlotTail : kSlotHead)) * kRangeRawDoubles;
#pragma unroll
    for (int k = 0; k < kRangeMoments; ++k) M[k] += s[k];
    ct += LOSS == kLossCauchy ? log(s[kRangeMoments]) + s[kRangeMoments + 1] * 0.693147180559945309417232121458 : s[kRangeMoments];
  }
  *cost_term = ct;
  return true;
}

// One thread per frame after the kModeRange sweep: the frame's row of kRangeSums at x9 = (pose7, b, s) (zeros for an empty frame);
// m, c of the frame from consts (SweepArgs::seg_consts).
template <int LOSS>
__global__ void clc_range_fixup_kernel(ProblemView pv, const double* __restrict__ consts, const double* x9, const int* done,
                                       const double* __restrict__ raw, const double* __restrict__ slots, double* __restrict__ rows) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= pv.n_frames || (done != nullptr && *done != 0)) return;
  double* row = rows + f * kRangeSums;
  double M[kRangeMoments], cost_term;
  if (!range_frame_moments<LOSS>(pv, f, raw, slots, M, &cost_term)) {
    for (int k = 0; k < kRangeSums; ++k) row[k] = 0.0;
    return;
  }
  const double n[3] = {pv.plane[f * 4], pv.plane[f * 4 + 1], pv.plane[f * 4 + 2]};
  const double m[3] = {consts[f * 4], consts[f * 4 + 1], consts[f * 4 + 2]};
  const double s2 = 1.0 / (double)(pv.offsets[f + 1] - pv.offsets[f]);
  double out[kRangeSums];
#pragma unroll
  for (int k = 0; k < kRangeSums; ++k) out[k] = 0.0;
  expand_lm_range(n, m, consts[f * 4 + 3], x9[7], x9[8], s2, M, LOSS, cost_term, pv.a2, out);
#pragma unroll
  for (int k = 0; k < kRangeSums; ++k) row[k] = out[k];
}

// The corrected points of clc_problem_range_correct: (x, y, z)[i] -> kappa (x, y, z), kappa = range_kappa, for i < n (the
// padding beyond the last point stays as the destination's allocation left it: zeros).  z == nullptr: a planar problem (z = 0).
// One thread per two points, 16-byte loads and stores: an HBM-bound stream of 48 B (planar 32 B) per point pair each way.
__global__ void clc_range_correct_kernel(const double* __restrict__ x, const double* __restrict__ y, const double* __restrict__ z,
                                         int64_t n, double b, double s, double* __restrict__ ox, double* __restrict__ oy,
                                         double* __restrict__ oz) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2; i < n; i += 2 * stride) {
    if (i + 1 < n) {
      const double2 X = *reinterpret_cast<const double2*>(x + i);
      const double2 Y = *reinterpret_cast<const double2*>(y + i);
      const double2 Z = z != nullptr ? *reinterpret_cast<const double2*>(z + i) : make_double2(0.0, 0.0);
      const double k0 = range_kappa(X.x, Y.x, Z.x, b, s), k1 = range_kappa(X.y, Y.y, Z.y, b, s);
      *reinterpret_cast<double2*>(ox + i) = make_double2(k0 * X.x, k1 * X.y);
      *reinterpret_cast<double2*>(oy + i) = make_double2(k0 * Y.x, k1 * Y.y);
      if (z != nullptr) *reinterpret_cast<double2*>(oz + i) = make_double2(k0 * Z.x, k1 * Z.y);
    } else {
      const double zz = z != nullptr ? z[i] : 0.0;
      const double k = range_kappa(x[i], y[i], zz, b, s);
      ox[i] = k * x[i];
      oy[i] = k * y[i];
      if (z != nullptr) oz[i] = k * zz;
    }
  }
}

}  // namespace clc
#endif
