// clc_time_offset.cuh -- the camera-laser time offset td, estimated together with the extrinsic from a board trajectory that is
// interpolated on the device (clc_problem_set_trajectory, clc_eval_time_offset, clc_information_time_offset,
// clc_solve_lm_time_offset).
//
// Frame f's board plane is no longer the one stored at creation but the plane of the trajectory at tau_f = s_f + td (s_f: the
// scan's time, td: what is added to a laser time to put it on the camera clock).  The trajectory is K >= 2 knots of T_ac (the
// camera in the board frame): lerp on the translation, a shortest-arc slerp q_k (x) Exp(u w_k) on the rotation, clamped to the end
// knots outside [t_0, t_{K-1}].  The board is z = 0 in its own frame, so the plane in the camera frame is n = R_ac^T e_z (the third
// row of R_ac) and d = t_ac,z, and with dR/du = R [w]x:
//   dn/dtd = (n x w_k) / D_k,   dd/dtd = (t_{k+1},z - t_k,z) / D_k        (0 outside the knot span)
// The residual e = m.p + c (m = R_cl^T n, c = n.t_cl + d) gains one Jacobian column, J_td = s (mdot.p + cdot) with
// mdot = R_cl^T dn/dtd and cdot = dn/dtd.t_cl + dd/dtd: linear in p, so its sums are images of the same 10 moments the sweep
// accumulates (expand_lm_td).  One iteration, on the segmented path with one segment (clc_segments.cuh):
//   1. clc_time_consts_kernel   the plane of every frame at tau_f (td from the LM candidate), m, c into the sweep's seg_consts,
//                               n, mdot, cdot into a per-frame array;
//   2. clc_sweep_kernel<.., kModeSegments, ..>   unchanged;
//   3. clc_time_fixup_kernel    every frame's moments (segment_frame_moments) expanded into its row of kTdSums;
//   4. clc_segment_chunk_kernel<kTdSums>   level 1 of the segment plan;
//   5. clc_segment_lm_kernel<7>            level 2, then lm_update on LmCoreN<7> (Ceres' LM on the pose and td, clc_lm.cuh).
// The host part (everything CLC_HD) also compiles with g++ for the CPU tests.
#pragma once

#include "clc_expand.cuh"
#include "clc_lm.cuh"

namespace clc {

constexpr int kTdSums = kLmSums<7>;  // 28 upper-tri of the 7x7 H (tx ty tz rx ry rz td, row-major, i <= j) + 7 g + 1 cost
constexpr int kTdFrameDoubles = 8;         // per frame: n[3], mdot[3], cdot, unused
constexpr int kKnotDoubles = 7;            // per knot: q_ac (x, y, z, w), t_ac

// ---- the trajectory ----------------------------------------------------------------------------------------------------------

// Hamilton product of (x, y, z, w) quaternions
CLC_HD void quat_mul(const double* a, const double* b, double* c) {
  c[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  c[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  c[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  c[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
}

// the unit quaternion Exp(v) of a rotation vector v: (sin(h) / (2h) v, cos(h)), h = |v| / 2 (a series below |v| = 1e-2)
CLC_HD void quat_exp(const double* v, double* q) {
  const double t2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  double a, w;
  if (t2 < 1e-4) {
    const double h2 = 0.25 * t2;
    a = 0.5 * (1.0 - h2 / 6.0 * (1.0 - h2 / 20.0 * (1.0 - h2 / 42.0)));
    w = 1.0 - h2 / 2.0 * (1.0 - h2 / 12.0 * (1.0 - h2 / 30.0));
  } else {
    const double t = sqrt(t2);
    a = sin(0.5 * t) / t;
    w = cos(0.5 * t);
  }
  q[0] = a * v[0]; q[1] = a * v[1]; q[2] = a * v[2]; q[3] = w;
}

// Log of a unit quaternion on the shortest arc (the sign with w >= 0): the rotation vector v, |v| <= pi
CLC_HD void quat_log(const double* qin, double* v) {
  const double sg = qin[3] < 0.0 ? -1.0 : 1.0;
  const double q[4] = {sg * qin[0], sg * qin[1], sg * qin[2], sg * qin[3]};
  const double s = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  double a;  // |v| / s = 2 atan2(s, w) / s
  if (s < 1e-4 * q[3]) {
    const double r2 = (s / q[3]) * (s / q[3]);
    a = 2.0 / q[3] * (1.0 - r2 / 3.0 * (1.0 - 0.6 * r2));
  } else {
    a = 2.0 * atan2(s, q[3]) / s;
  }
  v[0] = a * q[0]; v[1] = a * q[1]; v[2] = a * q[2];
}

// A knot in the frame_pose convention (qx qy qz qw tx ty tz of T_ca) -> k7 = (q_ac, t_ac) of T_ac = T_ca^-1 with the normalised
// quaternion: q_ac = conj(q / |q|), t_ac = -R_ca^T t_ca.
CLC_HD void traj_knot(const double* fp, double* k7) {
  const double inv = 1.0 / sqrt(fp[0] * fp[0] + fp[1] * fp[1] + fp[2] * fp[2] + fp[3] * fp[3]);
  const double q[4] = {fp[0] * inv, fp[1] * inv, fp[2] * inv, fp[3] * inv};
  double R[9];
  quat_to_rot(q, R);
  k7[0] = -q[0]; k7[1] = -q[1]; k7[2] = -q[2]; k7[3] = q[3];
  for (int c = 0; c < 3; ++c) k7[4 + c] = -(R[c] * fp[4] + R[3 + c] * fp[5] + R[6 + c] * fp[6]);
}

// w_k = Log(q_a^-1 (x) q_b) of the interval between knots a and b (k7 layout), |w_k| <= pi
CLC_HD void traj_omega(const double* ka, const double* kb, double* w) {
  const double ca[4] = {-ka[0], -ka[1], -ka[2], ka[3]};
  double r[4];
  quat_mul(ca, kb, r);
  quat_log(r, w);
}

// The trajectory on the device: times t[K] relative to t_0, knots [K * kKnotDoubles], w [(K - 1) * 3].
struct TrajView {
  const double* t;
  const double* knot;
  const double* omega;
  int64_t K;
};

// The board plane (n, d) at tau and its derivative by td (dplane: dn, dd).  tau in [t_k, t_k+1) (the last interval includes its
// right end) interpolates interval k; outside [t_0, t_{K-1}] the plane is the end knot's, and its derivative 0.
CLC_HD void traj_plane(const TrajView& tv, double tau, double* plane, double* dplane) {
  const int64_t K = tv.K;
  const bool before = tau < tv.t[0], after = tau > tv.t[K - 1];
  double q[4], tz, u = 0.0;
  int64_t k;
  if (before || after) {
    k = before ? 0 : K - 1;
    const double* a = tv.knot + k * kKnotDoubles;
    for (int i = 0; i < 4; ++i) q[i] = a[i];
    tz = a[6];
  } else {
    int64_t lo = 0, hi = K - 1;  // t[lo] <= tau, and tau < t[hi] or hi == K - 1
    while (hi - lo > 1) {
      const int64_t mid = lo + (hi - lo) / 2;
      if (tv.t[mid] <= tau) lo = mid; else hi = mid;
    }
    k = lo;
    const double dt = tv.t[k + 1] - tv.t[k];
    u = (tau - tv.t[k]) / dt;
    const double* a = tv.knot + k * kKnotDoubles;
    const double* b = a + kKnotDoubles;
    const double* w = tv.omega + k * 3;
    const double uw[3] = {u * w[0], u * w[1], u * w[2]}, inv_dt = 1.0 / dt;
    double e[4];
    quat_exp(uw, e);
    quat_mul(a, e, q);
    tz = (1.0 - u) * a[6] + u * b[6];
    dplane[3] = (b[6] - a[6]) * inv_dt;
    double R[9];
    quat_to_rot(q, R);
    plane[0] = R[6]; plane[1] = R[7]; plane[2] = R[8]; plane[3] = tz;
    double nw[3];
    cross3(plane, w, nw);
    dplane[0] = nw[0] * inv_dt; dplane[1] = nw[1] * inv_dt; dplane[2] = nw[2] * inv_dt;
    return;
  }
  double R[9];
  quat_to_rot(q, R);
  plane[0] = R[6]; plane[1] = R[7]; plane[2] = R[8]; plane[3] = tz;
  dplane[0] = dplane[1] = dplane[2] = dplane[3] = 0.0;
}

// ---- the 36 sums -------------------------------------------------------------------------------------------------------------

// Adds the piece's contribution to out[kTdSums] (upper-tri 7x7, 7 g, cost): expand_lm's 6x6 block, g[0..5] and cost at the plane
// n (with m = R^T n, c = n.t + d), and the td row and column from mdot, cdot.  With Sm = S2 mdot + cdot S1, Ew = mdot.S1 + cdot S0
// (= sum w J_td / s) and v, E0 of expand_lm:
//   H_t,td = s2 n Ew    H_theta,td = s2 Sm x m    H_td,td = s2 (mdot.Sm + cdot Ew)    g_td = s2 (mdot.v + cdot E0)
CLC_HD void expand_lm_td(const double* n, const double* m, double c, const double* md, double cd, double s2, const double* S, int loss,
                         double cost_term, double a2, double* out) {
  const double plane[4] = {n[0], n[1], n[2], 0.0};  // expand_lm reads the normal only
  double o[kNumSums];
  for (int k = 0; k < kNumSums; ++k) o[k] = 0.0;
  expand_lm(plane, m, c, s2, S, loss, cost_term, a2, o);
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) out[tri<7>(i, j)] += o[tri(i, j)];
  for (int i = 0; i < 6; ++i) out[28 + i] += o[21 + i];
  out[35] += o[27];
  const double S0 = S[0];
  const double S1[3] = {S[1], S[2], S[3]};
  const double xx = S[4], xy = S[5], xz = S[6], yy = S[7], yz = S[8], zz = S[9];
  const double Sm[3] = {xx * md[0] + xy * md[1] + xz * md[2] + cd * S1[0],
                        xy * md[0] + yy * md[1] + yz * md[2] + cd * S1[1],
                        xz * md[0] + yz * md[1] + zz * md[2] + cd * S1[2]};
  const double Ew = md[0] * S1[0] + md[1] * S1[1] + md[2] * S1[2] + cd * S0;
  const double v[3] = {xx * m[0] + xy * m[1] + xz * m[2] + c * S1[0],
                       xy * m[0] + yy * m[1] + yz * m[2] + c * S1[1],
                       xz * m[0] + yz * m[1] + zz * m[2] + c * S1[2]};
  const double E0 = m[0] * S1[0] + m[1] * S1[1] + m[2] * S1[2] + c * S0;
  double smx[3];
  cross3(Sm, m, smx);
  for (int i = 0; i < 3; ++i) out[tri<7>(i, 6)] += s2 * n[i] * Ew;
  for (int i = 0; i < 3; ++i) out[tri<7>(3 + i, 6)] += s2 * smx[i];
  out[tri<7>(6, 6)] += s2 * (md[0] * Sm[0] + md[1] * Sm[1] + md[2] * Sm[2] + cd * Ew);
  out[34] += s2 * (md[0] * v[0] + md[1] * v[1] + md[2] * v[2] + cd * E0);
}

// ---- Ceres' LM on two parameter blocks, the pose (local size 6) and td (a 1-vector): clc_lm.cuh's state machine at D = 7 -------

using LmCoreTd = LmCoreN<7>;

CLC_HD void lm_init_td(LmCoreTd* s, const double* pose7, double td, const clc_lm_options& opt) {
  const double x8[8] = {pose7[0], pose7[1], pose7[2], pose7[3], pose7[4], pose7[5], pose7[6], td};
  lm_init(s, x8, opt);
}

CLC_HD void lm_update_td(LmCoreTd* s, TraceRows trace, const double* sums) { lm_update(s, trace, sums); }

}  // namespace clc

#if defined(__CUDACC__)
#include "clc_segments.cuh"

namespace clc {

// One thread per frame: the plane at tau_f = frame_time[f] + td and its td-derivative at pose8 = (pose7, td) on the device; m, c
// into consts (SweepArgs::seg_consts), n, mdot, cdot into tframe[f * kTdFrameDoubles].
__global__ void clc_time_consts_kernel(ProblemView pv, TrajView tv, const double* __restrict__ frame_time, const double* pose8,
                                       const int* done, double* __restrict__ consts, double* __restrict__ tframe) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= pv.n_frames || (done != nullptr && *done != 0)) return;
  double pose[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) pose[k] = pose8[k];
  PoseConsts pc;
  make_pose_consts(pose, &pc);
  double plane[4], dplane[4], m[3], c, md[3], cd;
  traj_plane(tv, frame_time[f] + pose8[7], plane, dplane);
  frame_consts(pc, plane, m, &c);
  frame_consts(pc, dplane, md, &cd);  // mdot = R^T dn, cdot = dn.t + dd
  consts[f * 4] = m[0]; consts[f * 4 + 1] = m[1]; consts[f * 4 + 2] = m[2]; consts[f * 4 + 3] = c;
  double* o = tframe + f * kTdFrameDoubles;
  o[0] = plane[0]; o[1] = plane[1]; o[2] = plane[2];
  o[3] = md[0]; o[4] = md[1]; o[5] = md[2]; o[6] = cd; o[7] = 0.0;
}

// One thread per frame after the kModeSegments sweep: the frame's row of kTdSums (zeros for an empty frame).
template <int LOSS>
__global__ void clc_time_fixup_kernel(ProblemView pv, const double* __restrict__ consts, const double* __restrict__ tframe,
                                      const int* done, const double* __restrict__ raw, const double* __restrict__ slots,
                                      double* __restrict__ rows) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= pv.n_frames || (done != nullptr && *done != 0)) return;
  double* row = rows + f * kTdSums;
  double S[10], cost_term;
  if (!segment_frame_moments<LOSS>(pv, f, raw, slots, S, &cost_term)) {
    for (int k = 0; k < kTdSums; ++k) row[k] = 0.0;
    return;
  }
  const double* tf = tframe + f * kTdFrameDoubles;
  const double n[3] = {tf[0], tf[1], tf[2]}, md[3] = {tf[3], tf[4], tf[5]};
  const double m[3] = {consts[f * 4], consts[f * 4 + 1], consts[f * 4 + 2]};
  const double s2 = 1.0 / (double)(pv.offsets[f + 1] - pv.offsets[f]);
  double out[kTdSums];
#pragma unroll
  for (int k = 0; k < kTdSums; ++k) out[k] = 0.0;
  expand_lm_td(n, m, consts[f * 4 + 3], md, tf[6], s2, S, LOSS, cost_term, pv.a2, out);
#pragma unroll
  for (int k = 0; k < kTdSums; ++k) row[k] = out[k];
}

}  // namespace clc
#endif
