/*
 * frame_oracle.c -- per-frame restatement of clc_frame_report, built on the C oracle's exported functions (the factor as the
 * reference writes it, oracle_factor_evaluate, and the board / edge planes).  TEST INFRASTRUCTURE ONLY: compiled by
 * tests/test_frame_report_cpu.py and linked against oracle/libclc_oracle.so.
 *
 * Every residual of frame f goes through PointInPlaneFactor::Evaluate (reference src/LaseCamCalCeres.cpp:43-66) and, with the
 * loss, the Ceres Cauchy corrector (residual and Jacobian scaled by sqrt(rho'), cost 1/2 rho; :249).  The row is the frame's
 * share of the sums the oracle's evaluation forms: H_f = sum J~^T J~, g_f = sum J~^T r~, cost_f = 1/2 sum rho over its points and
 * its two edge residuals, chi_f = sum r^2 over its points (no loss, no edges: the analysis tail, :318-381), plus the unweighted
 * statistics of the raw distances e = r / scale.  Row layout: that of clc_frame_row (36 doubles, n_points as int64 bits).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../oracle/clc_oracle.h"

enum { ROW = 36, COST = 1, CHI = 2, MEAN_E = 3, RMS_E = 4, MAX_E = 5, MEAN_W = 6, EDGE_E = 7, H21 = 9, G6 = 30 };

/* Ceres CauchyLoss::Evaluate (b = a^2, c = 1/b): rho(s) = b log(1 + s c), rho'(s) = 1 / (1 + s c) */
static void cauchy(double a, double s, double* rho0, double* rho1) {
  const double b = a * a, c = 1.0 / b;
  const double sum = 1.0 + s * c;
  const double inv = 1.0 / sum;
  *rho0 = b * log(sum);
  *rho1 = inv > DBL_MIN ? inv : DBL_MIN;
}

/* adds one residual block to the row; returns r (uncorrected) and rho' (1 without the loss) */
static double add_residual(const oracle_problem* p, const double plane[4], const double pt[3], double scale, const double pose7[7],
                           double* row, double* w_out) {
  double r, j7[7];
  oracle_factor_evaluate(plane, pt, scale, pose7, &r, j7);
  double cost = 0.5 * r * r, sq = 1.0, w = 1.0;
  if (p->use_loss) {
    double rho0;
    cauchy(p->cauchy_a * scale, r * r, &rho0, &w);
    cost = 0.5 * rho0;
    sq = sqrt(w);
  }
  double J[6];
  for (int k = 0; k < 6; ++k) J[k] = j7[k] * sq;
  const double rc = r * sq;
  row[COST] += cost;
  int k = 0;
  for (int a = 0; a < 6; ++a)
    for (int b = a; b < 6; ++b) row[H21 + k++] += J[a] * J[b];
  for (int a = 0; a < 6; ++a) row[G6 + a] += J[a] * rc;
  *w_out = w;
  return r;
}

int oracle_frame_report(const oracle_problem* p, const double pose7[7], double* rows) {
  for (int64_t f = 0; f < p->n_frames; ++f) {
    double* row = rows + ROW * f;
    memset(row, 0, sizeof(double) * ROW);
    const int64_t b = p->offsets[f], e = p->offsets[f + 1], n = e - b;
    if (n <= 0) continue; /* no residual exists (the reference would divide by zero) */
    double plane[4];
    oracle_frame_plane(p->frame_pose + 7 * f, plane);
    const double scale = 1. / sqrt((double)n); /* :239-240 */
    double se = 0.0, se2 = 0.0, emax = 0.0, sw = 0.0, chi = 0.0;
    for (int64_t j = b; j < e; ++j) {
      double w;
      const double r = add_residual(p, plane, p->points + 3 * j, scale, pose7, row, &w);
      const double ev = r / scale;
      chi += r * r;
      se += ev;
      se2 += ev * ev;
      const double ae = fabs(ev);
      if (ae > emax || ae != ae) emax = ae; /* a NaN stays */
      sw += w;
    }
    if (p->edge_points != NULL) {
      double pi[2][4];
      oracle_edge_planes(p->frame_pose + 7 * f, pi[0], pi[1]);
      for (int k = 0; k < 2; ++k) {
        double w;
        row[EDGE_E + k] = add_residual(p, pi[k], p->edge_points + 6 * f + 3 * k, scale, pose7, row, &w) / scale;
      }
    }
    memcpy(row, &n, sizeof(n));
    row[CHI] = chi;
    row[MEAN_E] = se / (double)n;
    row[RMS_E] = sqrt(se2 / (double)n);
    row[MAX_E] = emax;
    row[MEAN_W] = sw / (double)n;
  }
  return 0;
}
