/*
 * fixed_oracle.c -- plain-C oracle of the calibration solve with some tangent coordinates of the extrinsic held at their
 * start value (clc_lm_options.fixed_mask).  TEST INFRASTRUCTURE ONLY, built by the tests and linked against
 * oracle/libclc_oracle.so, whose public restatements it reuses unchanged: the Ceres-shaped evaluation (oracle_evaluate: the
 * corrected residuals and local Jacobian, no loss or CauchyLoss), the streaming one (oracle_evaluate_normal: H, g) and
 * PoseLocalParameterization::Plus (oracle_pose_plus).  What is new here is the minimiser on the reduced local
 * parameterization -- a Ceres 2.1 local parameterization of local size 6 - k wrapped around the reference's:
 *
 *   - the trust-region Levenberg-Marquardt loop of trust_region_minimizer.cc / levenberg_marquardt_strategy.cc over the free
 *     coordinates only: Jacobi scaling, the LM diagonal, the linear solve and the model cost change see the free columns of J
 *     (or the free rows and columns of H and the free entries of g); the gradient norm is that of the free gradient embedded
 *     with zeros; Plus takes the free increment embedded with zeros; the parameter tolerance measures the 7-vector;
 *   - two linear solvers, as the main oracle has: opt->linear_solver 0 = DENSE_QR (Householder QR of [J_s; D] on the free
 *     columns, dense_qr_solver.cc), 1 = Cholesky of the free block of the scaled normal equations plus D^2.
 *
 * Bit k of fixed_mask holds tangent coordinate k (dt_x, dt_y, dt_z, dtheta_x, dtheta_y, dtheta_z); the mask is a separate
 * argument, so oracle_options keeps its layout.
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "clc_oracle.h"

/* min ||A y - b|| by Householder QR of the rows x n row-major A, n <= 6 (dense_qr_solver.cc); A and b are overwritten. */
static void householder_ls(double* A, double* b, int64_t rows, int n, double* y) {
  for (int k = 0; k < n; ++k) {
    double nrm2 = 0.0;
    for (int64_t i = k; i < rows; ++i) nrm2 += A[i * n + k] * A[i * n + k];
    const double nrm = sqrt(nrm2), akk = A[k * n + k];
    if (!(nrm > 0.0)) { A[k * n + k] = 0.0; continue; }
    const double alpha = akk > 0.0 ? -nrm : nrm, v0 = akk - alpha, vtv = nrm2 - akk * akk + v0 * v0;
    if (vtv > 0.0) {
      const double beta = 2.0 / vtv;
      for (int j = k + 1; j <= n; ++j) { /* columns k+1..n-1 of A, then b */
        double s = v0 * (j < n ? A[k * n + j] : b[k]);
        for (int64_t i = k + 1; i < rows; ++i) s += A[i * n + k] * (j < n ? A[i * n + j] : b[i]);
        s *= beta;
        if (j < n) {
          A[k * n + j] -= s * v0;
          for (int64_t i = k + 1; i < rows; ++i) A[i * n + j] -= s * A[i * n + k];
        } else {
          b[k] -= s * v0;
          for (int64_t i = k + 1; i < rows; ++i) b[i] -= s * A[i * n + k];
        }
      }
    }
    A[k * n + k] = alpha;
  }
  for (int k = n - 1; k >= 0; --k) {
    double s = b[k];
    for (int j = k + 1; j < n; ++j) s -= A[k * n + j] * y[j];
    y[k] = s / A[k * n + k];
  }
}

/* Cholesky solve of the SPD n x n row-major A y = b, n <= 6.  Returns 0 on success. */
static int cholesky_solve(const double* A, const double* b, int n, double* y) {
  double L[36], z[6];
  for (int i = 0; i < n; ++i)
    for (int j = 0; j <= i; ++j) {
      double s = A[i * n + j];
      for (int k = 0; k < j; ++k) s -= L[i * n + k] * L[j * n + k];
      if (i == j) {
        if (!(s > 0.0)) return 1;
        L[i * n + i] = sqrt(s);
      } else {
        L[i * n + j] = s / L[j * n + j];
      }
    }
  for (int i = 0; i < n; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s -= L[i * n + k] * z[k];
    z[i] = s / L[i * n + i];
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = z[i];
    for (int k = i + 1; k < n; ++k) s -= L[k * n + i] * y[k];
    y[i] = s / L[i * n + i];
  }
  return 0;
}

static double norm7(const double* a) {
  double s = 0.0;
  for (int i = 0; i < 7; ++i) s += a[i] * a[i];
  return sqrt(s);
}

/* trust_region_minimizer.cc: |x - Plus(x, -g)| in the max norm, g the free gradient embedded with zeros */
static double gradient_max_norm(const double x[7], const double g[6], int fixed_mask) {
  double ng[6], xp[7], m = 0.0;
  for (int i = 0; i < 6; ++i) ng[i] = (fixed_mask >> i & 1) ? 0.0 : -g[i];
  oracle_pose_plus(x, ng, xp);
  for (int i = 0; i < 7; ++i) m = fabs(x[i] - xp[i]) > m ? fabs(x[i] - xp[i]) : m;
  return m;
}

static void record(oracle_iteration* trace, int cap, int* n, const oracle_iteration* it) {
  if (trace && *n < cap) trace[*n] = *it;
  (*n)++;
}

/* TrustRegionMinimizer::Minimize with LevenbergMarquardtStrategy on the free coordinates of fixed_mask (0 <= mask < 63). */
int fixed_oracle_solve(const oracle_problem* p, double pose7[7], const oracle_options* opt, int fixed_mask, oracle_summary* summary,
                       oracle_iteration* trace, int trace_cap) {
  const int qr = opt->linear_solver == 0;
  int fc[6], nf = 0;
  for (int k = 0; k < 6; ++k)
    if (!(fixed_mask >> k & 1)) fc[nf++] = k;
  const int64_t R = qr ? oracle_num_residuals(p) : 0;
  double* res = qr ? malloc(sizeof(double) * (size_t)(R + 1)) : NULL;
  double* jac = qr ? malloc(sizeof(double) * (size_t)(R + 1) * 6) : NULL;
  double* js = qr ? malloc(sizeof(double) * (size_t)(R + 1) * 6) : NULL; /* the scaled free columns [R x nf] */
  double* A = qr ? malloc(sizeof(double) * (size_t)(R + 6) * 6) : NULL;
  double* rhs = qr ? malloc(sizeof(double) * (size_t)(R + 6)) : NULL;
  oracle_summary sm;
  memset(&sm, 0, sizeof(sm));
  int n_trace = 0, reuse_diagonal = 0, num_invalid = 0;
  double x[7], cand[7], x_cost, cand_cost, grad[6], H[36], scale[6], diag[6], colnorm2[6];
  memcpy(x, pose7, sizeof(x));
  double x_norm = norm7(x), radius = opt->initial_trust_region_radius, decrease_factor = 2.0;

  /* EvaluateGradientAndJacobian on the free coordinates, with the Jacobi scaling of the first evaluation kept */
#define EVALUATE_JACOBIAN(first)                                                                                   \
  do {                                                                                                             \
    if (qr) {                                                                                                      \
      oracle_evaluate(p, x, &x_cost, res, jac, grad, opt->num_threads);                                            \
      if (first) {                                                                                                 \
        for (int c = 0; c < nf; ++c) {                                                                             \
          double s2 = 0.0;                                                                                         \
          for (int64_t i = 0; i < R; ++i) s2 += jac[i * 6 + fc[c]] * jac[i * 6 + fc[c]];                           \
          scale[c] = opt->jacobi_scaling ? 1.0 / (1.0 + sqrt(s2)) : 1.0;                                           \
        }                                                                                                          \
      }                                                                                                            \
      for (int c = 0; c < nf; ++c) colnorm2[c] = 0.0;                                                              \
      for (int64_t i = 0; i < R; ++i)                                                                              \
        for (int c = 0; c < nf; ++c) {                                                                             \
          js[i * nf + c] = jac[i * 6 + fc[c]] * scale[c];                                                          \
          colnorm2[c] += js[i * nf + c] * js[i * nf + c];                                                          \
        }                                                                                                          \
    } else {                                                                                                       \
      oracle_evaluate_normal(p, x, &x_cost, H, grad, opt->num_threads);                                            \
      if (first)                                                                                                   \
        for (int c = 0; c < nf; ++c) scale[c] = opt->jacobi_scaling ? 1.0 / (1.0 + sqrt(H[fc[c] * 7])) : 1.0;      \
      for (int c = 0; c < nf; ++c) colnorm2[c] = scale[c] * scale[c] * H[fc[c] * 7];                               \
    }                                                                                                              \
    sm.num_residual_evaluations++;                                                                                 \
    sm.num_jacobian_evaluations++;                                                                                 \
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
  it.gradient_max_norm = gradient_max_norm(x, grad, fixed_mask);
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

    /* LevenbergMarquardtStrategy::ComputeStep on the free coordinates, step = -y */
    if (!reuse_diagonal)
      for (int c = 0; c < nf; ++c) diag[c] = fmin(fmax(colnorm2[c], opt->min_lm_diagonal), opt->max_lm_diagonal);
    double y[6] = {0, 0, 0, 0, 0, 0}, step[6], gs[6], Hs[36];
    int failed = 0;
    if (qr) { /* [J_s; D] y = [r; 0] */
      memcpy(A, js, sizeof(double) * (size_t)R * nf);
      memset(A + R * nf, 0, sizeof(double) * (size_t)(nf * nf));
      for (int c = 0; c < nf; ++c) A[(R + c) * nf + c] = sqrt(diag[c] / radius);
      memcpy(rhs, res, sizeof(double) * (size_t)R);
      memset(rhs + R, 0, sizeof(double) * (size_t)nf);
      householder_ls(A, rhs, R + nf, nf, y);
    } else { /* (H_s + D^2) y = g_s */
      for (int a = 0; a < nf; ++a) {
        gs[a] = scale[a] * grad[fc[a]];
        for (int b = 0; b < nf; ++b) Hs[a * nf + b] = scale[a] * scale[b] * H[fc[a] * 6 + fc[b]];
      }
      double Ad[36];
      memcpy(Ad, Hs, sizeof(double) * (size_t)(nf * nf));
      for (int c = 0; c < nf; ++c) Ad[c * nf + c] += diag[c] / radius;
      failed = cholesky_solve(Ad, gs, nf, y);
    }
    reuse_diagonal = 1;
    int finite = !failed;
    for (int c = 0; c < nf; ++c) {
      finite = finite && isfinite(y[c]);
      step[c] = -y[c];
    }
    /* model cost change -(J s)^T (r + J s / 2) = -g_s.s - 1/2 s^T H_s s */
    double model_change = 0.0;
    if (finite) {
      if (qr) {
        for (int64_t i = 0; i < R; ++i) {
          double mr = 0.0;
          for (int c = 0; c < nf; ++c) mr += js[i * nf + c] * step[c];
          model_change -= mr * (res[i] + mr / 2.0);
        }
      } else {
        double gs_s = 0.0, sHs = 0.0;
        for (int a = 0; a < nf; ++a) {
          gs_s += gs[a] * step[a];
          for (int b = 0; b < nf; ++b) sHs += step[a] * Hs[a * nf + b] * step[b];
        }
        model_change = -gs_s - 0.5 * sHs;
      }
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
    double delta[6] = {0, 0, 0, 0, 0, 0}; /* the free increment embedded with zeros */
    for (int c = 0; c < nf; ++c) delta[fc[c]] = step[c] * scale[c];
    oracle_pose_plus(x, delta, cand);
    if (qr) oracle_evaluate(p, cand, &cand_cost, NULL, NULL, NULL, opt->num_threads);
    else oracle_evaluate_normal(p, cand, &cand_cost, NULL, NULL, opt->num_threads);
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
      it.gradient_max_norm = gradient_max_norm(x, grad, fixed_mask);
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
  free(js);
  free(A);
  free(rhs);
  return 0;
}
