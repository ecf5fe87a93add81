// clc_expand.cuh -- from the streamed moments of one "piece" (a run of points of one frame) to its contribution
// to the normal equations.
//
// For a frame with board plane (n, d) and the pose (R, t):   m = R^T n,  c = n.t + d,
//   raw distance        e_j = n^T(R p_j + t) + d = m.p_j + c
//   residual            r_j = s e_j,  s = 1/sqrt(#points of the frame)      (reference src/LaseCamCalCeres.cpp:239-240,:48)
//   Jacobian (1x6)      J_j = s [ n^T , (p_j x m)^T ]                         (:54-60:  n^T(-R [p]x) = (p x m)^T)
//   robust weight       w_j = rho'(r_j^2), e.g. Cauchy 1 / (1 + e_j^2 / a^2), a = 0.05  (:249; the scale s cancels)
// J_t = n is constant over the frame and J_theta = p x m = -[m]x p is linear in p, so everything the LM step
// needs is a linear image of the weighted moments  S0 = sum w, S1 = sum w p, S2 = sum w p p^T:
//   sum w J^T J = s^2 [ S0 n n^T        n (S1 x m)^T      ]      sum w e J^T = s^2 [ (m.S1 + c S0) n      ]
//                     [ .               [m]x S2 [m]x^T    ]                        [ (S2 m + c S1) x m    ]
// and the robust cost is 1/2 a^2 s^2 sum log(1 + e^2/a^2) = 1/2 a^2 s^2 log(prod (1 + e^2/a^2)).
// The kernel therefore keeps 10 moment accumulators + a running product per lane instead of 28 sums.
// This holds for every loss with rho'' <= 0 (LossKind below): Ceres' Corrector then scales r and J by sqrt(rho'), so
// sum w J^T J and sum w e J^T are the same linear images of the moments -- only w and the cost term change.
#pragma once

#include "clc_math.cuh"

namespace clc {

// Robust losses (include/clc_b200.h CLC_LOSS_*).  A frame with scale s uses loss parameter a s on r = s e (reference :249), so
// with z = e^2 / a^2 the scale cancels from the weight; the frame's cost is 1/2 s^2 sum rho~(e), and a^2 times that for Cauchy:
//   kind      w = rho'                       rho~(e)
//   none      1                              e^2
//   Cauchy    1 / (1 + z)                    log(1 + z)
//   Huber     1 if |e| <= a, else a / |e|    e^2 if |e| <= a, else 2 a |e| - a^2
//   soft-L1   1 / sqrt(1 + z)                2 e^2 / (1 + sqrt(1 + z))   (Ceres' 2 a^2 (sqrt(1 + z) - 1) without cancellation)
// Every kind has rho'' <= 0 (Ceres' simple corrector branch).  |e| == a is a Huber inlier.
enum LossKind { kLossNone = 0, kLossCauchy = 1, kLossHuber = 2, kLossSoftL1 = 3 };

// w and rho~ of one residual (the single-residual paths: the one-cluster kernel, the edge residuals).  a2 = a^2, inv_a2 = 1/a2.
// Huber takes a = sqrt(a2), which is exact: sqrt(fl(a * a)) == a in binary floating point when a^2 is normal.
CLC_HD void loss_weight(int kind, double e, double a2, double inv_a2, double* w, double* cost_term) {
  if (kind == kLossCauchy) {
    const double u = fma(e * inv_a2, e, 1.0);
    *w = 1.0 / u;
    *cost_term = log(u);
  } else if (kind == kLossHuber) {
    const double a = sqrt(a2), ae = fabs(e);
    *w = ae <= a ? 1.0 : a / ae;
    *cost_term = ae <= a ? e * e : fma(2.0 * a, ae, -a2);
  } else if (kind == kLossSoftL1) {
    const double t = sqrt(fma(e * inv_a2, e, 1.0));
    *w = 1.0 / t;
    *cost_term = 2.0 * e * e / (1.0 + t);
  } else {
    *w = 1.0;
    *cost_term = e * e;
  }
}

// Pose-dependent constants shared by all frames of one sweep.
struct PoseConsts {
  double R[9];
  double t[3];
};

CLC_HD void make_pose_consts(const double* pose7, PoseConsts* pc) {
  quat_to_rot(pose7 + 3, pc->R);
  pc->t[0] = pose7[0]; pc->t[1] = pose7[1]; pc->t[2] = pose7[2];
}

// m = R^T n, c = n.t + d
CLC_HD void frame_consts(const PoseConsts& pc, const double* plane, double* m, double* c) {
  const double n0 = plane[0], n1 = plane[1], n2 = plane[2];
  m[0] = pc.R[0] * n0 + pc.R[3] * n1 + pc.R[6] * n2;
  m[1] = pc.R[1] * n0 + pc.R[4] * n1 + pc.R[7] * n2;
  m[2] = pc.R[2] * n0 + pc.R[5] * n1 + pc.R[8] * n2;
  *c = (n0 * pc.t[0] + n1 * pc.t[1] + n2 * pc.t[2]) + plane[3];
}

// The raw point-to-plane distance e = m.p + c of one point, rounded exactly as the sweep kernel and the frame report round it
// (a point of a planar problem has z = 0: fma(m2, 0, c) == c).  The trim's thresholds compare against this value.
CLC_HD double point_distance(const double* m, double c, double x, double y, double z) {
  return fma(m[0], x, fma(m[1], y, fma(m[2], z, c)));
}

// Moments layout: S[0]=S0, S[1..3]=S1 (x,y,z), S[4..9]=S2 (xx,xy,xz,yy,yz,zz).
// Adds the piece's contribution to out[28] = 21 upper-tri H (row-major, i<=j), 6 g, 1 cost.
//   s2        = 1/(#points of the whole frame)
//   cost_term = sum rho~(e) over the piece (LossKind; accumulated directly: deriving it from the moments would cancel
//               catastrophically near the optimum)
//   loss      = LossKind, a2 = a^2
CLC_HD void expand_lm(const double* plane, const double* m, double c, double s2, const double* S, int loss,
                      double cost_term, double a2, double* out) {
  const double n[3] = {plane[0], plane[1], plane[2]};
  const double S0 = S[0];
  const double S1[3] = {S[1], S[2], S[3]};
  const double xx = S[4], xy = S[5], xz = S[6], yy = S[7], yz = S[8], zz = S[9];
  // u = S1 x m = sum w (p x m)
  double u[3];
  cross3(S1, m, u);
  // T = [m]x S2
  const double T00 = -m[2] * xy + m[1] * xz, T01 = -m[2] * yy + m[1] * yz, T02 = -m[2] * yz + m[1] * zz;
  const double T10 = m[2] * xx - m[0] * xz, T11 = m[2] * xy - m[0] * yz, T12 = m[2] * xz - m[0] * zz;
  const double T20 = -m[1] * xx + m[0] * xy, T21 = -m[1] * xy + m[0] * yy, T22 = -m[1] * xz + m[0] * yz;
  // Q = T [m]x^T (upper triangle)
  const double Q00 = -m[2] * T01 + m[1] * T02;
  const double Q01 = m[2] * T00 - m[0] * T02;
  const double Q02 = -m[1] * T00 + m[0] * T01;
  const double Q11 = m[2] * T10 - m[0] * T12;
  const double Q12 = -m[1] * T10 + m[0] * T11;
  const double Q22 = -m[1] * T20 + m[0] * T21;
  // v = S2 m + c S1 = sum w e p ;  E0 = m.S1 + c S0 = sum w e
  const double v[3] = {xx * m[0] + xy * m[1] + xz * m[2] + c * S1[0],
                       xy * m[0] + yy * m[1] + yz * m[2] + c * S1[1],
                       xz * m[0] + yz * m[1] + zz * m[2] + c * S1[2]};
  const double E0 = m[0] * S1[0] + m[1] * S1[1] + m[2] * S1[2] + c * S0;
  double vxm[3];
  cross3(v, m, vxm);
  const double sn[3] = {s2 * n[0], s2 * n[1], s2 * n[2]};
  // H_tt
  out[0] += sn[0] * n[0] * S0;  out[1] += sn[0] * n[1] * S0;  out[2] += sn[0] * n[2] * S0;
  out[6] += sn[1] * n[1] * S0;  out[7] += sn[1] * n[2] * S0;  out[11] += sn[2] * n[2] * S0;
  // H_t,theta
  out[3] += sn[0] * u[0];  out[4] += sn[0] * u[1];  out[5] += sn[0] * u[2];
  out[8] += sn[1] * u[0];  out[9] += sn[1] * u[1];  out[10] += sn[1] * u[2];
  out[12] += sn[2] * u[0]; out[13] += sn[2] * u[1]; out[14] += sn[2] * u[2];
  // H_theta,theta
  out[15] += s2 * Q00; out[16] += s2 * Q01; out[17] += s2 * Q02;
  out[18] += s2 * Q11; out[19] += s2 * Q12; out[20] += s2 * Q22;
  // g
  out[21] += sn[0] * E0; out[22] += sn[1] * E0; out[23] += sn[2] * E0;
  out[24] += s2 * vxm[0]; out[25] += s2 * vxm[1]; out[26] += s2 * vxm[2];
  // cost: 1/2 a^2 s^2 sum log(1 + e^2/a^2) with the Cauchy loss, 1/2 s^2 sum rho~(e) otherwise
  out[27] += loss == kLossCauchy ? 0.5 * a2 * s2 * cost_term : 0.5 * s2 * cost_term;
}

// One residual added DIRECTLY to acc[28] (21 upper-tri H, 6 g, cost) -- what the one-cluster kernel for small problems does
// (clc_small.cuh): no moments, the plain PointInPlaneFactor arithmetic of reference src/LaseCamCalCeres.cpp:43-66 with the
// Cauchy correction of :249.  plane = (n, d); (x, y, z) the laser point; s2 = 1/#points of the frame (the squared scale of
// :239-240); loss = LossKind, a2 = a^2, inv_a2 = 1/a2.  J = s [n, p x m] with m = R^T n; w = rho' (loss_weight).
CLC_HD void accumulate_residual(const PoseConsts& pc, const double* plane, double x, double y, double z, double s2, int loss,
                                double a2, double inv_a2, double* acc) {
  double m[3], c;
  frame_consts(pc, plane, m, &c);
  const double e = fma(m[0], x, fma(m[1], y, fma(m[2], z, c)));
  double w = 1.0, cost;
  if (loss == kLossCauchy) {
    const double u = fma(e * inv_a2, e, 1.0);
    w = 1.0 / u;
    cost = 0.5 * a2 * s2 * log(u);
  } else if (loss == kLossNone) {
    cost = 0.5 * s2 * e * e;
  } else {
    double t;
    loss_weight(loss, e, a2, inv_a2, &w, &t);
    cost = 0.5 * s2 * t;
  }
  const double J[6] = {plane[0], plane[1], plane[2], y * m[2] - z * m[1], z * m[0] - x * m[2], x * m[1] - y * m[0]};
  const double ws = w * s2;
  int k = 0;
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    const double wa = ws * J[a];
#pragma unroll
    for (int b = a; b < 6; ++b) {
      acc[k] = fma(wa, J[b], acc[k]);
      ++k;
    }
  }
  const double we = ws * e;
#pragma unroll
  for (int a = 0; a < 6; ++a) acc[21 + a] = fma(we, J[a], acc[21 + a]);
  acc[27] += cost;
}

// One board-edge residual (plane = an edge plane, pt = its edge point) expanded through its moments into out[28], as the edge
// tail of the sweep kernel does; returns the raw distance e.  s2 = 1/#points of the frame.
// m, c: the edge plane's constants at the pose (frame_consts).
CLC_HD double edge_residual_at(const double* plane, const double* m, double c, const double* pt, double s2, int loss,
                               double a2, double inv_a2, double* out) {
  const double x = pt[0], y = pt[1], z = pt[2];
  const double e = fma(m[0], x, fma(m[1], y, fma(m[2], z, c)));
  double w, cost_term;
  loss_weight(loss, e, a2, inv_a2, &w, &cost_term);
  const double S[10] = {w, w * x, w * y, w * z, w * x * x, w * x * y, w * x * z, w * y * y, w * y * z, w * z * z};
  expand_lm(plane, m, c, s2, S, loss, cost_term, a2, out);
  return e;
}

// edge_residual_at with m, c = frame_consts(pc, plane)
CLC_HD double edge_residual(const PoseConsts& pc, const double* plane, const double* pt, double s2, int loss, double a2,
                            double inv_a2, double* out) {
  double m[3], c;
  frame_consts(pc, plane, m, &c);
  return edge_residual_at(plane, m, c, pt, s2, loss, a2, inv_a2, out);
}

// Closed-form initialisation (reference src/LaseCamCalCeres.cpp:144-161): row A_k = n (x) (x, y, 1), b_k = -d, so
// A^T A = sum_frames M (x) n n^T with M = sum_j pbar pbar^T (unweighted moments, z ignored) and
// A^T b = sum_frames -d (M e_3) (x) n.   out[54] = 45 upper-tri of the 9x9 (row-major) then 9 of A^T b.
CLC_HD void expand_closed_form(const double* plane, const double* S, double* out) {
  const double n[3] = {plane[0], plane[1], plane[2]};
  const double M[3][3] = {{S[4], S[5], S[1]}, {S[5], S[7], S[2]}, {S[1], S[2], S[0]}};
  int k = 0;
  for (int i = 0; i < 9; ++i) {
    const int a = i / 3, r = i % 3;
    for (int j = i; j < 9; ++j) {
      const int b = j / 3, q = j % 3;
      out[k++] += M[a][b] * n[r] * n[q];
    }
  }
  for (int i = 0; i < 9; ++i) out[45 + i] += -plane[3] * M[i / 3][2] * n[i % 3];
}

}  // namespace clc
