/*
 * loss_oracle.c -- plain-C oracle of the calibration solve under Ceres' HuberLoss and SoftLOneLoss (and CauchyLoss / no
 * loss, for cross-checks).  TEST INFRASTRUCTURE ONLY, built by the tests and linked against oracle/libclc_oracle.so, whose
 * public restatements of the reference's cost model it reuses unchanged: the board and edge planes
 * (oracle_frame_plane, oracle_edge_planes: reference src/LaseCamCalCeres.cpp:227-231, :262-276), PointInPlaneFactor::Evaluate
 * (oracle_factor_evaluate, :43-66) and PoseLocalParameterization::Plus (oracle_pose_plus).  What is new here:
 *
 *   - the loss objects of Ceres' internal/ceres/loss_function.cc: HuberLoss::Evaluate, SoftLOneLoss::Evaluate and
 *     CauchyLoss::Evaluate on s = r^2 with parameter a*scale (the reference scales its CauchyLoss that way, :249);
 *   - ResidualBlock::Evaluate + corrector.cc: all three losses have rho'' <= 0, so the Corrector takes its simple branch and
 *     scales the residual and the Jacobian by sqrt(rho');
 *   - the trust-region Levenberg-Marquardt loop of trust_region_minimizer.cc / levenberg_marquardt_strategy.cc with DENSE_QR
 *     (dense_qr_solver.cc: Householder QR of [J; D]), the reference's solver settings (:302-304, Ceres defaults otherwise).
 *
 * The loss kind travels in oracle_problem.use_loss (0 none, 1 Cauchy, 2 Huber, 3 soft-L1, the library's CLC_LOSS_*) and its
 * parameter a in oracle_problem.cauchy_a.  Huber's outlier test is Ceres' `s > b` taken as |r| > a*scale: the library's rule
 * |e| <= a (an inlier) up to the rounding of r = scale*e, where rho and rho' are continuous.  Soft-L1's cost is Ceres' own
 * 2b (sqrt(1 + s/b) - 1).
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "clc_oracle.h"

enum { LOSS_NONE = 0, LOSS_CAUCHY = 1, LOSS_HUBER = 2, LOSS_SOFT_L1 = 3 };

/* Ceres loss_function.cc, rho[3] = (rho(s), rho'(s), rho''(s)) with parameter a (b = a^2, c = 1/b). */
static void loss_evaluate(int kind, double a, double s, double rho[3]) {
  const double b = a * a;
  if (kind == LOSS_CAUCHY) { /* CauchyLoss::Evaluate */
    const double c = 1.0 / b, sum = 1.0 + s * c, inv = 1.0 / sum;
    rho[0] = b * log(sum);
    rho[1] = inv > DBL_MIN ? inv : DBL_MIN;
    rho[2] = -c * (inv * inv);
  } else if (kind == LOSS_HUBER) { /* HuberLoss::Evaluate */
    const double r = sqrt(s);
    if (r > a) { /* outlying region */
      rho[0] = 2.0 * a * r - b;
      rho[1] = a / r > DBL_MIN ? a / r : DBL_MIN;
      rho[2] = -rho[1] / (2.0 * s);
    } else { /* inlying region */
      rho[0] = s;
      rho[1] = 1.0;
      rho[2] = 0.0;
    }
  } else if (kind == LOSS_SOFT_L1) { /* SoftLOneLoss::Evaluate */
    const double c = 1.0 / b, sum = 1.0 + s * c, tmp = sqrt(sum);
    rho[0] = 2.0 * b * (tmp - 1.0);
    rho[1] = 1.0 / tmp > DBL_MIN ? 1.0 / tmp : DBL_MIN;
    rho[2] = -(c * rho[1]) / (2.0 * sum);
  } else {
    rho[0] = s;
    rho[1] = 1.0;
    rho[2] = 0.0;
  }
}

/* ResidualBlock::Evaluate + Corrector (simple branch, rho'' <= 0): cost 1/2 rho, r~ = sqrt(rho') r, J~ = sqrt(rho') J. */
static void residual_block(const oracle_problem* p, const double plane[4], const double pt[3], double scale, const double x[7],
                           double* cost, double* r_out, double* j6) {
  double r, j7[7], rho[3];
  oracle_factor_evaluate(plane, pt, scale, x, &r, j7);
  loss_evaluate(p->use_loss, p->cauchy_a * scale, r * r, rho);
  const double sq = sqrt(rho[1]);
  *cost = 0.5 * rho[0];
  *r_out = r * sq;
  for (int k = 0; k < 6; ++k) j6[k] = j7[k] * sq; /* local Jacobian: the first six columns (PoseLocalParameterization) */
}

/* One evaluation in the reference's AddResidualBlock order (:241-294: a frame's points, then its two edge residuals).
 * residuals [R], jacobian [R*6] and gradient [6] may be NULL. */
int loss_oracle_evaluate(const oracle_problem* p, const double x[7], double* cost, double* residuals, double* jacobian,
                         double* gradient) {
  double c = 0.0, g[6] = {0, 0, 0, 0, 0, 0};
  int64_t row = 0;
  for (int64_t f = 0; f < p->n_frames; ++f) {
    const int64_t b = p->offsets[f], e = p->offsets[f + 1];
    if (e <= b) continue;
    const double scale = 1.0 / sqrt((double)(e - b));
    double planes[3][4];
    const double* pts[3];
    int n_extra = 0;
    oracle_frame_plane(p->frame_pose + 7 * f, planes[0]);
    if (p->edge_points) {
      oracle_edge_planes(p->frame_pose + 7 * f, planes[1], planes[2]);
      pts[1] = p->edge_points + 6 * f;
      pts[2] = p->edge_points + 6 * f + 3;
      n_extra = 2;
    }
    for (int64_t j = b; j < e + n_extra; ++j, ++row) {
      const int k = j < e ? 0 : (int)(j - e) + 1;
      double ci, ri, j6[6];
      residual_block(p, planes[k], k == 0 ? p->points + 3 * j : pts[k], scale, x, &ci, &ri, j6);
      c += ci;
      if (residuals) residuals[row] = ri;
      if (jacobian) memcpy(jacobian + 6 * row, j6, sizeof(j6));
      for (int q = 0; q < 6; ++q) g[q] += j6[q] * ri;
    }
  }
  if (cost) *cost = c;
  if (gradient) memcpy(gradient, g, sizeof(g));
  return 0;
}

/* min ||A y - b|| by Householder QR of the rows x 6 row-major A (dense_qr_solver.cc); A and b are overwritten. */
static void householder_ls6(double* A, double* b, int64_t rows, double y[6]) {
  for (int k = 0; k < 6; ++k) {
    double nrm2 = 0.0;
    for (int64_t i = k; i < rows; ++i) nrm2 += A[i * 6 + k] * A[i * 6 + k];
    const double nrm = sqrt(nrm2), akk = A[k * 6 + k];
    if (!(nrm > 0.0)) { A[k * 6 + k] = 0.0; continue; }
    const double alpha = akk > 0.0 ? -nrm : nrm, v0 = akk - alpha, vtv = nrm2 - akk * akk + v0 * v0;
    if (vtv > 0.0) {
      const double beta = 2.0 / vtv;
      for (int j = k + 1; j < 7; ++j) { /* columns k+1..5 of A, then b */
        double s = v0 * (j < 6 ? A[k * 6 + j] : b[k]);
        for (int64_t i = k + 1; i < rows; ++i) s += A[i * 6 + k] * (j < 6 ? A[i * 6 + j] : b[i]);
        s *= beta;
        if (j < 6) {
          A[k * 6 + j] -= s * v0;
          for (int64_t i = k + 1; i < rows; ++i) A[i * 6 + j] -= s * A[i * 6 + k];
        } else {
          b[k] -= s * v0;
          for (int64_t i = k + 1; i < rows; ++i) b[i] -= s * A[i * 6 + k];
        }
      }
    }
    A[k * 6 + k] = alpha;
  }
  for (int k = 5; k >= 0; --k) {
    double s = b[k];
    for (int j = k + 1; j < 6; ++j) s -= A[k * 6 + j] * y[j];
    y[k] = s / A[k * 6 + k];
  }
}

static double norm7(const double* a) {
  double s = 0.0;
  for (int i = 0; i < 7; ++i) s += a[i] * a[i];
  return sqrt(s);
}

/* trust_region_minimizer.cc: |x - Plus(x, -g)| in the max norm */
static double gradient_max_norm(const double x[7], const double g[6]) {
  double ng[6], xp[7], m = 0.0;
  for (int i = 0; i < 6; ++i) ng[i] = -g[i];
  oracle_pose_plus(x, ng, xp);
  for (int i = 0; i < 7; ++i) m = fabs(x[i] - xp[i]) > m ? fabs(x[i] - xp[i]) : m;
  return m;
}

static void record(oracle_iteration* trace, int cap, int* n, const oracle_iteration* it) {
  if (trace && *n < cap) trace[*n] = *it;
  (*n)++;
}

/* TrustRegionMinimizer::Minimize with LevenbergMarquardtStrategy and DENSE_QR (opt->linear_solver is ignored). */
int loss_oracle_solve(const oracle_problem* p, double pose7[7], const oracle_options* opt, oracle_summary* summary,
                      oracle_iteration* trace, int trace_cap) {
  const int64_t R = oracle_num_residuals(p);
  double* res = malloc(sizeof(double) * (size_t)(R + 1));
  double* jac = malloc(sizeof(double) * (size_t)(R + 1) * 6);
  double* A = malloc(sizeof(double) * (size_t)(R + 6) * 6);
  double* rhs = malloc(sizeof(double) * (size_t)(R + 6));
  oracle_summary sm;
  memset(&sm, 0, sizeof(sm));
  int n_trace = 0, reuse_diagonal = 0, num_invalid = 0;
  double x[7], cand[7], x_cost, cand_cost, grad[6], scale[6], diag[6], colnorm2[6];
  memcpy(x, pose7, sizeof(x));
  double x_norm = norm7(x), radius = opt->initial_trust_region_radius, decrease_factor = 2.0;

  /* EvaluateGradientAndJacobian, with the Jacobi scaling of the first evaluation kept for the whole solve */
#define EVALUATE_JACOBIAN(first)                                                                              \
  do {                                                                                                        \
    loss_oracle_evaluate(p, x, &x_cost, res, jac, grad);                                                      \
    if (first) {                                                                                              \
      for (int k = 0; k < 6; ++k) colnorm2[k] = 0.0;                                                          \
      for (int64_t i = 0; i < R; ++i)                                                                         \
        for (int k = 0; k < 6; ++k) colnorm2[k] += jac[i * 6 + k] * jac[i * 6 + k];                           \
      for (int k = 0; k < 6; ++k) scale[k] = opt->jacobi_scaling ? 1.0 / (1.0 + sqrt(colnorm2[k])) : 1.0;     \
    }                                                                                                         \
    for (int k = 0; k < 6; ++k) colnorm2[k] = 0.0;                                                            \
    for (int64_t i = 0; i < R; ++i)                                                                           \
      for (int k = 0; k < 6; ++k) {                                                                           \
        jac[i * 6 + k] *= scale[k];                                                                           \
        colnorm2[k] += jac[i * 6 + k] * jac[i * 6 + k];                                                       \
      }                                                                                                       \
    sm.num_residual_evaluations++;                                                                            \
    sm.num_jacobian_evaluations++;                                                                            \
  } while (0)

  oracle_iteration it;
  memset(&it, 0, sizeof(it));
  EVALUATE_JACOBIAN(1);
  sm.initial_cost = x_cost;
  if (!isfinite(x_cost)) {
    sm.termination = ORACLE_TERM_FAILURE;
    sm.final_cost = x_cost;
    goto done;
  }
  it.cost = x_cost;
  it.gradient_max_norm = gradient_max_norm(x, grad);
  it.step_is_valid = it.step_is_successful = 1;
  for (;;) {
    if (it.step_is_successful) {
      sm.num_successful_steps++;
      memcpy(pose7, x, sizeof(x));
    } else {
      sm.num_unsuccessful_steps++;
    }
    it.trust_region_radius = radius;
    record(trace, trace_cap, &n_trace, &it);
    if (it.iteration >= opt->max_num_iterations) { sm.termination = ORACLE_TERM_NO_CONVERGENCE; break; }
    if (it.step_is_successful && it.gradient_max_norm <= opt->gradient_tolerance) {
      sm.termination = ORACLE_TERM_CONVERGENCE_GRADIENT;
      break;
    }
    if (!(radius > opt->min_trust_region_radius)) { sm.termination = ORACLE_TERM_CONVERGENCE_MIN_RADIUS; break; }
    const oracle_iteration prev = it;
    memset(&it, 0, sizeof(it));
    it.iteration = prev.iteration + 1;

    /* LevenbergMarquardtStrategy::ComputeStep: solve [J; D] y = [r; 0] by QR, step = -y */
    if (!reuse_diagonal)
      for (int k = 0; k < 6; ++k)
        diag[k] = fmin(fmax(colnorm2[k], opt->min_lm_diagonal), opt->max_lm_diagonal);
    double step[6];
    memcpy(A, jac, sizeof(double) * (size_t)R * 6);
    memset(A + R * 6, 0, sizeof(double) * 36);
    for (int k = 0; k < 6; ++k) A[(R + k) * 6 + k] = sqrt(diag[k] / radius);
    memcpy(rhs, res, sizeof(double) * (size_t)R);
    memset(rhs + R, 0, sizeof(double) * 6);
    householder_ls6(A, rhs, R + 6, step);
    reuse_diagonal = 1;
    int finite = 1;
    for (int k = 0; k < 6; ++k) {
      finite = finite && isfinite(step[k]);
      step[k] = -step[k];
    }
    /* model cost change -(J s)^T (r + J s / 2) */
    double model_change = 0.0;
    if (finite)
      for (int64_t i = 0; i < R; ++i) {
        double mr = 0.0;
        for (int k = 0; k < 6; ++k) mr += jac[i * 6 + k] * step[k];
        model_change -= mr * (res[i] + mr / 2.0);
      }
    it.step_is_valid = finite && model_change > 0.0;
    if (!it.step_is_valid) { /* HandleInvalidStep */
      if (++num_invalid >= opt->max_num_consecutive_invalid_steps) { sm.termination = ORACLE_TERM_FAILURE; break; }
      radius /= decrease_factor;
      decrease_factor *= 2.0;
      it.cost = x_cost;
      it.gradient_max_norm = prev.gradient_max_norm;
      continue;
    }
    num_invalid = 0;
    double delta[6];
    for (int k = 0; k < 6; ++k) delta[k] = step[k] * scale[k];
    oracle_pose_plus(x, delta, cand);
    loss_oracle_evaluate(p, cand, &cand_cost, NULL, NULL, NULL);
    sm.num_residual_evaluations++;
    if (!isfinite(cand_cost)) cand_cost = DBL_MAX;
    {
      double d[7];
      for (int i = 0; i < 7; ++i) d[i] = x[i] - cand[i];
      it.step_norm = norm7(d);
    }
    it.cost_change = x_cost - cand_cost;
    it.cost = cand_cost;
    if (it.step_norm <= opt->parameter_tolerance * (x_norm + opt->parameter_tolerance)) {
      sm.termination = ORACLE_TERM_CONVERGENCE_PARAMETER;
      it.trust_region_radius = radius;
      record(trace, trace_cap, &n_trace, &it);
      break;
    }
    if (fabs(it.cost_change) <= opt->function_tolerance * x_cost) {
      sm.termination = ORACLE_TERM_CONVERGENCE_FUNCTION;
      it.trust_region_radius = radius;
      record(trace, trace_cap, &n_trace, &it);
      break;
    }
    it.relative_decrease = it.cost_change / model_change;
    if (it.relative_decrease > opt->min_relative_decrease) { /* HandleSuccessfulStep + StepAccepted */
      memcpy(x, cand, sizeof(x));
      x_norm = norm7(x);
      EVALUATE_JACOBIAN(0);
      it.cost = x_cost;
      it.gradient_max_norm = gradient_max_norm(x, grad);
      it.step_is_successful = 1;
      const double q = 2.0 * it.relative_decrease - 1.0;
      radius = fmin(radius / fmax(1.0 / 3.0, 1.0 - q * q * q), opt->max_trust_region_radius);
      decrease_factor = 2.0;
      reuse_diagonal = 0;
    } else { /* HandleUnsuccessfulStep + StepRejected */
      radius /= decrease_factor;
      decrease_factor *= 2.0;
    }
  }
#undef EVALUATE_JACOBIAN
  sm.final_cost = x_cost;
done:
  sm.num_iterations = n_trace;
  if (summary) *summary = sm;
  free(res);
  free(jac);
  free(A);
  free(rhs);
  return 0;
}
