// clc_lm.cuh -- the Levenberg-Marquardt trust-region state machine, run ON THE DEVICE by one thread after every
// sweep of the fused residual+Jacobian+reduce kernel (either as the tail of that kernel's last block, or as its
// own single-thread kernel after the NCCL all-reduce when several ranks share the problem).
//
// It restates what ceres::Solve() does for the reference at src/LaseCamCalCeres.cpp:299-307 (DENSE_QR,
// max_num_iterations 100, every other option a Ceres default): Ceres' TrustRegionMinimizer loop with the
// LevenbergMarquardtStrategy, Jacobi scaling fixed at iteration 0, monotonic steps.  Two deliberate differences,
// both exact in exact arithmetic:
//   * the damped step solves the 6x6 normal equations (J_s^T J_s + D^2) y = J_s^T r by Cholesky instead of a
//     Householder QR of the (P+6)x6 matrix [J_s; D] -- the Jacobian is never materialised;
//   * every candidate point is evaluated with its Jacobian in the same sweep ("speculative" evaluation), so an
//     accepted step needs no second sweep: one LM iteration = one pass over the points.
#pragma once

#include "clc_math.cuh"
#include "../../include/clc_b200.h"

namespace clc {

constexpr int kTraceMax = 256;

// The state machine runs over D tangent columns: D = 6, the pose (its local parameterization); D = 7, the pose and the
// camera-laser time offset td as a plain 1-vector (clc_time_offset.cuh); D = 8, the pose and the laser's range offset b and
// scale s (clc_range_bias.cuh).  Tangent coordinate k >= 6 is the plain parameter x[k + 1].  Its sums are [upper-tri H | g | cost].
template <int D>
constexpr int kLmSums = D * (D + 1) / 2 + D + 1;
constexpr int kNumSums = kLmSums<6>;  // 21 upper-tri H + 6 g + 1 cost

// Hot state of the minimiser (about 600 bytes): staged through shared memory around lm_update so that the single
// thread running it does not pay a global-memory round trip per field.
template <int D>
struct LmCoreN {
  int done;            // CLC_TERM_*; 0 while running
  int phase;           // 0: the pending sweep evaluates the start point; 1: it evaluates a candidate
  int iteration;       // index of the last finalised iteration
  int num_invalid;
  int reuse_diagonal;
  int n_trace;
  int num_successful;
  int num_unsuccessful;
  int sweeps;
  int pad0;
  double x[D + 1];     // pose7, then the D - 6 plain parameters (td; or b, s)
  double cand[D + 1];  // the point the next sweep evaluates
  double x_cost, x_norm;
  double H[D * (D + 1) / 2], g[D];  // at x: loss-corrected, unscaled
  double scale[D], diag[D];
  double radius, decrease_factor, model_cost_change;
  double initial_cost;
  clc_lm_options opt;
};
using LmCore = LmCoreN<6>;
static_assert(sizeof(LmCore) % 8 == 0 && sizeof(LmCoreN<7>) % 8 == 0 && sizeof(LmCoreN<8>) % 8 == 0,
              "LmCoreN is copied as 8-byte words");
template <int D>
constexpr int kLmWords = (int)(sizeof(LmCoreN<D>) / 8);
constexpr int kLmCoreWords = kLmWords<6>;

struct LmState {
  LmCore core;
  clc_lm_iteration trace[kTraceMax];
};

// -DCLC_LM_PROFILE: clock stamps at the section boundaries of the last lm_update that ran on the device (experiment builds only;
// read back with clc_debug_lm_profile)
#if defined(CLC_LM_PROFILE) && defined(__CUDACC__)
__device__ long long g_lm_profile[16];
#endif
#if defined(CLC_LM_PROFILE) && defined(__CUDA_ARCH__)
#define CLC_LM_STAMP(i) g_lm_profile[i] = clock64()
#else
#define CLC_LM_STAMP(i) ((void)0)
#endif

template <int N>
CLC_HD double vec_norm(const double* a) {
  double s = 0.0;
  for (int i = 0; i < N; ++i) s += a[i] * a[i];
  return sqrt(s);
}

// Ceres EvaluateGradientAndJacobian: |x - Plus(x, -g)|_inf, over the pose and the plain parameters (|g_k|, k >= 6)
template <int D>
CLC_HD double gradient_max_norm(const double* x, const double* g) {
  double ng[6], xp[7], m = 0.0;
  for (int i = 0; i < 6; ++i) ng[i] = -g[i];
  pose_plus(x, ng, xp);
  for (int i = 0; i < 7; ++i) {
    const double d = fabs(x[i] - xp[i]);
    if (d > m) m = d;
  }
  for (int k = 6; k < D; ++k) {
    const double a = fabs(g[k]);
    if (a > m) m = a;
  }
  return m;
}

// Held coordinates (clc_lm_options.fixed_mask): Ceres' LM on the reduced local parameterization.  Each held coordinate leaves
// the H and g just stored at x: its row and column of H become 0 but for a unit diagonal, its entry of g 0.  Every later use
// then sees the free coordinates only -- gradient_max_norm (g embedded with zeros), the Jacobi-scaled system and its LM
// diagonal, whose positive pivot makes the Cholesky step of a held coordinate exactly 0 and that of the free ones the step of
// the reduced system (every product with a held entry is 0), and the model cost change.  Done in place on the state (shared
// memory on the device), off the register-resident step code.  Bit k >= 6 holds plain parameter k (td; b, s).
template <int D>
CLC_HD void lm_hold(LmCoreN<D>* s, int fixed) {
#pragma unroll 1
  for (int k = 0; k < D; ++k) {
    if (!(fixed >> k & 1)) continue;
#pragma unroll 1
    for (int j = 0; j < D; ++j) s->H[j < k ? tri<D>(j, k) : tri<D>(k, j)] = 0.0;
    s->H[tri<D>(k, k)] = 1.0;
    s->g[k] = 0.0;
  }
}

// a held translation of the candidate (or plain parameter) keeps the bits of x (x + 0 would turn a -0.0 into +0.0)
template <int D>
CLC_HD void lm_hold_cand(LmCoreN<D>* s, int fixed) {
#pragma unroll 1
  for (int k = 0; k < 3; ++k)
    if (fixed >> k & 1) s->cand[k] = s->x[k];
  for (int k = 6; k < D; ++k)
    if (fixed >> k & 1) s->cand[k + 1] = s->x[k + 1];
}

template <int D>
CLC_HD void lm_record(LmCoreN<D>* s, clc_lm_iteration* trace, const clc_lm_iteration& it) {
  if (s->n_trace < kTraceMax) trace[s->n_trace] = it;
  s->n_trace++;
}

// A trace of `cap` rows (cap 0: none, rows may be NULL): the segmented solve (clc_solve_lm_segments) keeps one per segment and
// allocates them only when the caller asks for a trace.
struct TraceRows {
  clc_lm_iteration* rows;
  int cap;
};

template <int D>
CLC_HD void lm_record(LmCoreN<D>* s, TraceRows trace, const clc_lm_iteration& it) {
  if (s->n_trace < trace.cap) trace.rows[s->n_trace] = it;
  s->n_trace++;
}

// x0: pose7, then the plain parameters
template <int D>
CLC_HD void lm_init(LmCoreN<D>* s, const double* x0, const clc_lm_options& opt) {
  s->done = 0; s->phase = 0; s->iteration = 0; s->num_invalid = 0; s->reuse_diagonal = 0; s->n_trace = 0;
  s->num_successful = 0; s->num_unsuccessful = 0; s->sweeps = 0; s->pad0 = 0;
  for (int i = 0; i < D + 1; ++i) { s->x[i] = x0[i]; s->cand[i] = x0[i]; }
  s->x_cost = 0.0;
  s->x_norm = vec_norm<D + 1>(x0);
  s->radius = opt.initial_trust_region_radius;
  s->decrease_factor = 2.0;
  s->model_cost_change = 0.0;
  s->initial_cost = 0.0;
  s->opt = opt;
}

// Consumes the kLmSums<D> sums of the sweep that has just evaluated s->cand and advances the minimiser until it either
// terminates (s->done != 0) or has a new candidate in s->cand for the next sweep.  Trace: a clc_lm_iteration* of kTraceMax
// rows, or TraceRows.  With D > 6 the parameter tolerance measures the (D + 1)-vector (pose7, plain parameters),
// gradient_max_norm also takes their |g| and a candidate's plain parameter is x's plus its step.
template <int D, class Trace>
CLC_HD void lm_update(LmCoreN<D>* s, Trace trace, const double* sums) {
  constexpr int kH = D * (D + 1) / 2, kSums = kLmSums<D>;
  if (s->done) return;
  CLC_LM_STAMP(0);
  s->sweeps++;
  const clc_lm_options& o = s->opt;
  clc_lm_iteration last;
  last.reserved = 0;
  // Ceres rejects an evaluation that produced a non-finite residual or Jacobian entry (residual_block.cc
  // IsArrayValid): at the start point that is a FAILURE, at a candidate it is "a step with infinite cost".
  bool sums_ok = true;
  for (int i = 0; i < kSums; ++i) sums_ok = sums_ok && is_finite(sums[i]);
  if (s->phase == 0) {
    // ---- iteration 0 (Ceres: IterationZero) ----
    if (!sums_ok) { s->done = CLC_TERM_FAILURE; return; }
    s->x_cost = sums[kSums - 1];
    for (int i = 0; i < kH; ++i) s->H[i] = sums[i];
    for (int i = 0; i < D; ++i) s->g[i] = sums[kH + i];
    if (o.fixed_mask) lm_hold(s, o.fixed_mask);
    for (int k = 0; k < D; ++k) s->scale[k] = o.jacobi_scaling ? 1.0 / (1.0 + sqrt(s->H[tri<D>(k, k)])) : 1.0;
    s->initial_cost = s->x_cost;
    last.iteration = 0; last.step_is_valid = 1; last.step_is_successful = 1;
    last.cost = s->x_cost; last.cost_change = 0.0; last.gradient_max_norm = gradient_max_norm<D>(s->x, s->g);
    last.step_norm = 0.0; last.relative_decrease = 0.0; last.trust_region_radius = s->radius;
  } else {
    // ---- a candidate has been evaluated ----
    const double cand_cost = sums_ok ? sums[kSums - 1] : DBL_MAX;
    last.iteration = s->iteration + 1; last.step_is_valid = 1; last.step_is_successful = 0;
    double d[D + 1];
    for (int i = 0; i < D + 1; ++i) d[i] = s->x[i] - s->cand[i];
    last.step_norm = vec_norm<D + 1>(d);
    last.cost_change = s->x_cost - cand_cost;
    last.cost = cand_cost;
    last.gradient_max_norm = 0.0; last.relative_decrease = 0.0; last.trust_region_radius = s->radius;
    // Ceres: ParameterToleranceReached
    if (last.step_norm <= o.parameter_tolerance * (s->x_norm + o.parameter_tolerance)) {
      s->done = CLC_TERM_CONVERGENCE_PARAMETER;
      lm_record(s, trace, last);
      return;
    }
    // Ceres: FunctionToleranceReached (tested before the accept/reject decision; the candidate is not applied)
    if (fabs(last.cost_change) <= o.function_tolerance * s->x_cost) {
      s->done = CLC_TERM_CONVERGENCE_FUNCTION;
      lm_record(s, trace, last);
      return;
    }
    last.relative_decrease = last.cost_change / s->model_cost_change;
    if (last.relative_decrease > o.min_relative_decrease) {
      // Ceres: HandleSuccessfulStep + LevenbergMarquardtStrategy::StepAccepted
      for (int i = 0; i < D + 1; ++i) s->x[i] = s->cand[i];
      s->x_norm = vec_norm<D + 1>(s->x);
      s->x_cost = cand_cost;
      for (int i = 0; i < kH; ++i) s->H[i] = sums[i];
      for (int i = 0; i < D; ++i) s->g[i] = sums[kH + i];
      if (o.fixed_mask) lm_hold(s, o.fixed_mask);
      last.step_is_successful = 1;
      last.gradient_max_norm = gradient_max_norm<D>(s->x, s->g);
      const double q = 2.0 * last.relative_decrease - 1.0;
      double den = 1.0 - q * q * q;
      if (den < 1.0 / 3.0) den = 1.0 / 3.0;
      s->radius = s->radius / den;
      if (s->radius > o.max_trust_region_radius) s->radius = o.max_trust_region_radius;
      s->decrease_factor = 2.0;
      s->reuse_diagonal = 0;
    } else {
      // Ceres: HandleUnsuccessfulStep + StepRejected
      s->radius = s->radius / s->decrease_factor;
      s->decrease_factor *= 2.0;
      s->reuse_diagonal = 1;
    }
  }

  CLC_LM_STAMP(1);  // accept / reject decided (incl. gradient_max_norm of an accepted step)
  for (;;) {
    // ---- Ceres: FinalizeIterationAndCheckIfMinimizerCanContinue ----
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

    CLC_LM_STAMP(2);  // iteration recorded, termination tests done
    // ---- Ceres: LevenbergMarquardtStrategy::ComputeStep on the Jacobi-scaled system ----
    double Hs[D * D], gs[D], A[D * D], step[D];
#pragma unroll
    for (int i = 0; i < D; ++i) {
      gs[i] = s->scale[i] * s->g[i];
#pragma unroll
      for (int j = i; j < D; ++j) {
        const double v = s->scale[i] * s->scale[j] * s->H[tri<D>(i, j)];
        Hs[i * D + j] = v;
        Hs[j * D + i] = v;
      }
    }
    if (!s->reuse_diagonal)
#pragma unroll
      for (int k = 0; k < D; ++k) {
        double dd = Hs[k * D + k];
        dd = dd > o.min_lm_diagonal ? dd : o.min_lm_diagonal;
        dd = dd < o.max_lm_diagonal ? dd : o.max_lm_diagonal;
        s->diag[k] = dd;
      }
#pragma unroll
    for (int i = 0; i < D * D; ++i) A[i] = Hs[i];
    const double inv_radius = 1.0 / s->radius;
#pragma unroll
    for (int k = 0; k < D; ++k) A[k * D + k] += s->diag[k] * inv_radius;  // D^2 = diag / radius
    CLC_LM_STAMP(3);  // scaled, damped system built
    bool ok = chol_solve<D>(A, gs, step);
    CLC_LM_STAMP(4);  // Cholesky solve done
    s->reuse_diagonal = 1;
#pragma unroll
    for (int k = 0; k < D; ++k) {
      if (!is_finite(step[k])) ok = false;
      step[k] = -step[k];
    }
    // Ceres: model_cost_change = -(J s)^T (r + J s / 2) = -g_s.s - 1/2 s^T H_s s
    double mcc = 0.0;
    if (ok) {
      double gs_s = 0.0, sHs = 0.0;
#pragma unroll
      for (int i = 0; i < D; ++i) {
        gs_s += gs[i] * step[i];
        double r = 0.0;
#pragma unroll
        for (int j = 0; j < D; ++j) r += Hs[i * D + j] * step[j];
        sHs += step[i] * r;
      }
      mcc = -gs_s - 0.5 * sHs;
    }
    if (!(ok && mcc > 0.0)) {
      // ---- Ceres: HandleInvalidStep ----
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
    double delta[D];
    for (int k = 0; k < D; ++k) delta[k] = step[k] * s->scale[k];
    CLC_LM_STAMP(5);  // model cost change done
    pose_plus(s->x, delta, s->cand);
    for (int k = 6; k < D; ++k) s->cand[k + 1] = s->x[k + 1] + delta[k];
    if (o.fixed_mask) lm_hold_cand(s, o.fixed_mask);
    s->model_cost_change = mcc;
    s->phase = 1;
    CLC_LM_STAMP(6);  // candidate pose done
    return;
  }
}

}  // namespace clc
