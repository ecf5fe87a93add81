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
//   4. clc_time_chunk_kernel    level 1 of the segment plan at width kTdSums;
//   5. clc_time_lm_kernel       level 2, then lm_update_td (Ceres' LM on the pose and td) by lane 0.
// The host part (everything CLC_HD) also compiles with g++ for the CPU tests.
#pragma once

#include "clc_expand.cuh"
#include "clc_lm.cuh"

namespace clc {

constexpr int kTdSums = 36;          // 28 upper-tri of the 7x7 H (tx ty tz rx ry rz td, row-major, i <= j) + 7 g + 1 cost
constexpr int kTdFrameDoubles = 8;   // per frame: n[3], mdot[3], cdot, unused
constexpr int kKnotDoubles = 7;      // per knot: q_ac (x, y, z, w), t_ac

CLC_HD int tri7(int i, int j) { return i * 7 - (i * (i - 1)) / 2 + (j - i); }  // upper-tri index of the 7x7, i <= j

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
    for (int j = i; j < 6; ++j) out[tri7(i, j)] += o[tri(i, j)];
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
  for (int i = 0; i < 3; ++i) out[tri7(i, 6)] += s2 * n[i] * Ew;
  for (int i = 0; i < 3; ++i) out[tri7(3 + i, 6)] += s2 * smx[i];
  out[tri7(6, 6)] += s2 * (md[0] * Sm[0] + md[1] * Sm[1] + md[2] * Sm[2] + cd * Ew);
  out[34] += s2 * (md[0] * v[0] + md[1] * v[1] + md[2] * v[2] + cd * E0);
}

// ---- Ceres' LM on two parameter blocks: the pose (local size 6) and td (a 1-vector) --------------------------------------------
// lm_update's state machine over 7 columns: x = (pose7, td), the parameter tolerance on the 8-vector, gradient_max_norm =
// max(|x - Plus(x, -g)|_inf over the pose, |g_td|).  fixed_mask bit 6 holds td (its start bits kept), bits 0-5 as in lm_hold.

struct LmCoreTd {
  int done;  // as LmCore
  int phase;
  int iteration;
  int num_invalid;
  int reuse_diagonal;
  int n_trace;
  int num_successful;
  int num_unsuccessful;
  int sweeps;
  int pad0;
  double x[8];     // pose7, td
  double cand[8];  // the point the next sweep evaluates
  double x_cost, x_norm;
  double H[28], g[7];
  double scale[7], diag[7];
  double radius, decrease_factor, model_cost_change;
  double initial_cost;
  clc_lm_options opt;
};
static_assert(sizeof(LmCoreTd) % 8 == 0, "LmCoreTd is copied as 8-byte words");
constexpr int kLmCoreTdWords = (int)(sizeof(LmCoreTd) / 8);

CLC_HD double norm8(const double* a) {
  double s = 0.0;
  for (int i = 0; i < 8; ++i) s += a[i] * a[i];
  return sqrt(s);
}

CLC_HD double gradient_max_norm_td(const double* x, const double* g) {
  const double m = gradient_max_norm(x, g), a = fabs(g[6]);
  return a > m ? a : m;
}

// Cholesky solve of the SPD 7x7 system A y = b (chol6_solve's arithmetic).  false if not positive definite.
CLC_HD bool chol7_solve(const double* A, const double* b, double* y) {
  constexpr int N = 7;
  double L[N * N], inv[N];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < N; ++j) {
    double s = A[j * N + j];
#pragma unroll
    for (int k = 0; k < j; ++k) s -= L[j * N + k] * L[j * N + k];
    ok = ok && (s > 0.0);
    const double d = sqrt(s);
    L[j * N + j] = d;
    inv[j] = 1.0 / d;
#pragma unroll
    for (int i = j + 1; i < N; ++i) {
      double t = A[i * N + j];
#pragma unroll
      for (int k = 0; k < j; ++k) t -= L[i * N + k] * L[j * N + k];
      L[i * N + j] = t * inv[j];
    }
  }
  if (!ok) return false;
  double z[N];
#pragma unroll
  for (int i = 0; i < N; ++i) {
    double s = b[i];
#pragma unroll
    for (int k = 0; k < i; ++k) s -= L[i * N + k] * z[k];
    z[i] = s * inv[i];
  }
#pragma unroll
  for (int i = N - 1; i >= 0; --i) {
    double s = z[i];
#pragma unroll
    for (int k = i + 1; k < N; ++k) s -= L[k * N + i] * y[k];
    y[i] = s * inv[i];
  }
  return true;
}

// lm_hold over 7 columns
CLC_HD void lm_hold_td(LmCoreTd* s, int fixed) {
#pragma unroll 1
  for (int k = 0; k < 7; ++k) {
    if (!(fixed >> k & 1)) continue;
#pragma unroll 1
    for (int j = 0; j < 7; ++j) s->H[j < k ? tri7(j, k) : tri7(k, j)] = 0.0;
    s->H[tri7(k, k)] = 1.0;
    s->g[k] = 0.0;
  }
}

// a held translation coordinate or td keeps the bits of x
CLC_HD void lm_hold_cand_td(LmCoreTd* s, int fixed) {
#pragma unroll 1
  for (int k = 0; k < 3; ++k)
    if (fixed >> k & 1) s->cand[k] = s->x[k];
  if (fixed >> 6 & 1) s->cand[7] = s->x[7];
}

CLC_HD void lm_record(LmCoreTd* s, TraceRows trace, const clc_lm_iteration& it) {
  if (s->n_trace < trace.cap) trace.rows[s->n_trace] = it;
  s->n_trace++;
}

CLC_HD void lm_init_td(LmCoreTd* s, const double* pose7, double td, const clc_lm_options& opt) {
  s->done = 0; s->phase = 0; s->iteration = 0; s->num_invalid = 0; s->reuse_diagonal = 0; s->n_trace = 0;
  s->num_successful = 0; s->num_unsuccessful = 0; s->sweeps = 0; s->pad0 = 0;
  for (int i = 0; i < 7; ++i) { s->x[i] = pose7[i]; s->cand[i] = pose7[i]; }
  s->x[7] = td; s->cand[7] = td;
  s->x_cost = 0.0;
  s->x_norm = norm8(s->x);
  s->radius = opt.initial_trust_region_radius;
  s->decrease_factor = 2.0;
  s->model_cost_change = 0.0;
  s->initial_cost = 0.0;
  s->opt = opt;
}

// lm_update on the kTdSums sums of the sweep that has just evaluated s->cand.
CLC_HD void lm_update_td(LmCoreTd* s, TraceRows trace, const double* sums) {
  if (s->done) return;
  s->sweeps++;
  const clc_lm_options& o = s->opt;
  clc_lm_iteration last;
  last.reserved = 0;
  bool sums_ok = true;
  for (int i = 0; i < kTdSums; ++i) sums_ok = sums_ok && is_finite(sums[i]);
  if (s->phase == 0) {
    if (!sums_ok) { s->done = CLC_TERM_FAILURE; return; }
    s->x_cost = sums[35];
    for (int i = 0; i < 28; ++i) s->H[i] = sums[i];
    for (int i = 0; i < 7; ++i) s->g[i] = sums[28 + i];
    if (o.fixed_mask) lm_hold_td(s, o.fixed_mask);
    for (int k = 0; k < 7; ++k) s->scale[k] = o.jacobi_scaling ? 1.0 / (1.0 + sqrt(s->H[tri7(k, k)])) : 1.0;
    s->initial_cost = s->x_cost;
    last.iteration = 0; last.step_is_valid = 1; last.step_is_successful = 1;
    last.cost = s->x_cost; last.cost_change = 0.0; last.gradient_max_norm = gradient_max_norm_td(s->x, s->g);
    last.step_norm = 0.0; last.relative_decrease = 0.0; last.trust_region_radius = s->radius;
  } else {
    const double cand_cost = sums_ok ? sums[35] : DBL_MAX;
    last.iteration = s->iteration + 1; last.step_is_valid = 1; last.step_is_successful = 0;
    double d[8];
    for (int i = 0; i < 8; ++i) d[i] = s->x[i] - s->cand[i];
    last.step_norm = norm8(d);
    last.cost_change = s->x_cost - cand_cost;
    last.cost = cand_cost;
    last.gradient_max_norm = 0.0; last.relative_decrease = 0.0; last.trust_region_radius = s->radius;
    if (last.step_norm <= o.parameter_tolerance * (s->x_norm + o.parameter_tolerance)) {
      s->done = CLC_TERM_CONVERGENCE_PARAMETER;
      lm_record(s, trace, last);
      return;
    }
    if (fabs(last.cost_change) <= o.function_tolerance * s->x_cost) {
      s->done = CLC_TERM_CONVERGENCE_FUNCTION;
      lm_record(s, trace, last);
      return;
    }
    last.relative_decrease = last.cost_change / s->model_cost_change;
    if (last.relative_decrease > o.min_relative_decrease) {
      for (int i = 0; i < 8; ++i) s->x[i] = s->cand[i];
      s->x_norm = norm8(s->x);
      s->x_cost = cand_cost;
      for (int i = 0; i < 28; ++i) s->H[i] = sums[i];
      for (int i = 0; i < 7; ++i) s->g[i] = sums[28 + i];
      if (o.fixed_mask) lm_hold_td(s, o.fixed_mask);
      last.step_is_successful = 1;
      last.gradient_max_norm = gradient_max_norm_td(s->x, s->g);
      const double q = 2.0 * last.relative_decrease - 1.0;
      double den = 1.0 - q * q * q;
      if (den < 1.0 / 3.0) den = 1.0 / 3.0;
      s->radius = s->radius / den;
      if (s->radius > o.max_trust_region_radius) s->radius = o.max_trust_region_radius;
      s->decrease_factor = 2.0;
      s->reuse_diagonal = 0;
    } else {
      s->radius = s->radius / s->decrease_factor;
      s->decrease_factor *= 2.0;
      s->reuse_diagonal = 1;
    }
  }

  for (;;) {
    if (last.step_is_successful) s->num_successful++; else s->num_unsuccessful++;
    last.trust_region_radius = s->radius;
    lm_record(s, trace, last);
    s->iteration = last.iteration;
    if (last.iteration >= o.max_num_iterations) { s->done = CLC_TERM_NO_CONVERGENCE; return; }
    if (last.step_is_successful && last.gradient_max_norm <= o.gradient_tolerance) {
      s->done = CLC_TERM_CONVERGENCE_GRADIENT;
      return;
    }
    if (!(s->radius > o.min_trust_region_radius)) { s->done = CLC_TERM_CONVERGENCE_MIN_RADIUS; return; }

    double Hs[49], gs[7], A[49], step[7];
#pragma unroll
    for (int i = 0; i < 7; ++i) {
      gs[i] = s->scale[i] * s->g[i];
#pragma unroll
      for (int j = i; j < 7; ++j) {
        const double v = s->scale[i] * s->scale[j] * s->H[tri7(i, j)];
        Hs[i * 7 + j] = v;
        Hs[j * 7 + i] = v;
      }
    }
    if (!s->reuse_diagonal)
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        double dd = Hs[k * 7 + k];
        dd = dd > o.min_lm_diagonal ? dd : o.min_lm_diagonal;
        dd = dd < o.max_lm_diagonal ? dd : o.max_lm_diagonal;
        s->diag[k] = dd;
      }
#pragma unroll
    for (int i = 0; i < 49; ++i) A[i] = Hs[i];
    const double inv_radius = 1.0 / s->radius;
#pragma unroll
    for (int k = 0; k < 7; ++k) A[k * 7 + k] += s->diag[k] * inv_radius;
    bool ok = chol7_solve(A, gs, step);
    s->reuse_diagonal = 1;
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      if (!is_finite(step[k])) ok = false;
      step[k] = -step[k];
    }
    double mcc = 0.0;
    if (ok) {
      double gs_s = 0.0, sHs = 0.0;
#pragma unroll
      for (int i = 0; i < 7; ++i) {
        gs_s += gs[i] * step[i];
        double r = 0.0;
#pragma unroll
        for (int j = 0; j < 7; ++j) r += Hs[i * 7 + j] * step[j];
        sHs += step[i] * r;
      }
      mcc = -gs_s - 0.5 * sHs;
    }
    if (!(ok && mcc > 0.0)) {
      if (++s->num_invalid >= o.max_num_consecutive_invalid_steps) { s->done = CLC_TERM_FAILURE; return; }
      s->radius = s->radius / s->decrease_factor;
      s->decrease_factor *= 2.0;
      s->reuse_diagonal = 1;
      const double prev_gmax = last.gradient_max_norm;
      last.iteration = s->iteration + 1; last.step_is_valid = 0; last.step_is_successful = 0;
      last.cost = s->x_cost; last.cost_change = 0.0; last.gradient_max_norm = prev_gmax;
      last.step_norm = 0.0; last.relative_decrease = 0.0;
      continue;
    }
    s->num_invalid = 0;
    double delta[7];
    for (int k = 0; k < 7; ++k) delta[k] = step[k] * s->scale[k];
    pose_plus(s->x, delta, s->cand);
    s->cand[7] = s->x[7] + delta[6];
    if (o.fixed_mask) lm_hold_cand_td(s, o.fixed_mask);
    s->model_cost_change = mcc;
    s->phase = 1;
    return;
  }
}

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

// Level 1 at width kTdSums: one warp per chunk, lane k adds outputs k and k + 32 of the chunk's rows in frame order.
__global__ void __launch_bounds__(32 * kSegWarpsPerBlock)
clc_time_chunk_kernel(const double* __restrict__ rows, const int64_t* __restrict__ chunk_offsets, int64_t n_chunks, const int* done,
                      double* __restrict__ partials) {
  const int64_t ch = (int64_t)blockIdx.x * kSegWarpsPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (ch >= n_chunks || (done != nullptr && *done != 0)) return;
  const int64_t a = chunk_offsets[ch], b = chunk_offsets[ch + 1];
  for (int k = lane; k < kTdSums; k += 32) {
    double acc = 0.0;
    for (int64_t r = a; r < b; ++r) acc += rows[r * kTdSums + k];
    partials[ch * kTdSums + k] = acc;
  }
}

// Level 2 + LM, one warp: the chunk partials in chunk order into sums (may be nullptr); with a core, lane 0 then runs lm_update_td
// on it, staged in shared memory, and raises `done` when it terminates.
__global__ void __launch_bounds__(32)
clc_time_lm_kernel(const double* __restrict__ partials, int64_t n_chunks, double* sums, LmCoreTd* core, clc_lm_iteration* trace,
                   int trace_cap, int* done) {
  __shared__ unsigned long long s_core[kLmCoreTdWords];
  __shared__ double s_sums[kTdSums];
  const int lane = threadIdx.x & 31;
  if (done != nullptr && *done != 0) return;
  for (int k = lane; k < kTdSums; k += 32) {
    double acc = 0.0;
    for (int64_t c = 0; c < n_chunks; ++c) acc += partials[c * kTdSums + k];
    s_sums[k] = acc;
    if (sums != nullptr) sums[k] = acc;
  }
  if (core == nullptr) return;
  unsigned long long* g_core = reinterpret_cast<unsigned long long*>(core);
  for (int k = lane; k < kLmCoreTdWords; k += 32) s_core[k] = g_core[k];
  __syncwarp();
  if (lane == 0) {
    LmCoreTd* s = reinterpret_cast<LmCoreTd*>(s_core);
    lm_update_td(s, TraceRows{trace, trace_cap}, s_sums);
    if (s->done != 0) *done = 1;
  }
  __syncwarp();
  for (int k = lane; k < kLmCoreTdWords; k += 32) g_core[k] = s_core[k];
}

}  // namespace clc
#endif
