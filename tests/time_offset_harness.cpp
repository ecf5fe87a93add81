// Test-only harness for the time offset: the product's CLC_HD trajectory interpolation, 36-sum expansion and 7-column LM state
// machine (clc_time_offset.cuh), compiled with g++ so that the code the GPU runs can be checked on a machine without a GPU.  Never
// shipped, never linked into libclc_b200.so.
#include <cstring>
#include <vector>

#include "../camlasercalibratool_b200/csrc/clc_time_offset.cuh"

extern "C" {

// K knots (frame_pose convention) -> the device layout: knots [K * 7] (q_ac, t_ac) and w [(K - 1) * 3]
void td_prepare(int64_t K, const double* knot_poses, double* knots, double* omega) {
  for (int64_t k = 0; k < K; ++k) clc::traj_knot(knot_poses + 7 * k, knots + 7 * k);
  for (int64_t k = 0; k + 1 < K; ++k) clc::traj_omega(knots + 7 * k, knots + 7 * (k + 1), omega + 3 * k);
}
// the plane (n, d) of the trajectory at each tau[i] and its td-derivative (t: knot times relative to the first knot)
void td_planes(int64_t K, const double* t, const double* knots, const double* omega, int64_t n, const double* tau, double* planes,
               double* dplanes) {
  const clc::TrajView tv{t, knots, omega, K};
  for (int64_t i = 0; i < n; ++i) clc::traj_plane(tv, tau[i], planes + 4 * i, dplanes + 4 * i);
}
// the moments of one piece -> the 36 sums at pose7 with the plane (n, d) and its derivative (dn, dd)
void td_expand(const double* plane, const double* dplane, const double* pose7, double count, const double* S10, int kind,
               double cost_term, double a, double* out36) {
  clc::PoseConsts pc;
  clc::make_pose_consts(pose7, &pc);
  double m[3], c, md[3], cd;
  clc::frame_consts(pc, plane, m, &c);
  clc::frame_consts(pc, dplane, md, &cd);
  clc::expand_lm_td(plane, m, c, md, cd, 1.0 / count, S10, kind, cost_term, a * a, out36);
}

struct TdState {
  clc::LmCoreTd core;
  clc_lm_iteration trace[clc::kTraceMax];
};
int td_lm_state_size() { return (int)sizeof(TdState); }
void td_lm_init(void* st, const double* pose7, double td, const clc_lm_options* opt) {
  clc::lm_init_td(&static_cast<TdState*>(st)->core, pose7, td, *opt);
}
void td_lm_update(void* st, const double* sums36) {
  TdState* s = static_cast<TdState*>(st);
  clc::lm_update_td(&s->core, clc::TraceRows{s->trace, clc::kTraceMax}, sums36);
}
int td_lm_done(const void* st) { return static_cast<const TdState*>(st)->core.done; }
int td_lm_ntrace(const void* st) { return static_cast<const TdState*>(st)->core.n_trace; }
int td_lm_sweeps(const void* st) { return static_cast<const TdState*>(st)->core.sweeps; }
void td_lm_cand(const void* st, double* out8) { std::memcpy(out8, static_cast<const TdState*>(st)->core.cand, 64); }
void td_lm_x(const void* st, double* out8) { std::memcpy(out8, static_cast<const TdState*>(st)->core.x, 64); }
void td_lm_trace(const void* st, int i, clc_lm_iteration* out) { *out = static_cast<const TdState*>(st)->trace[i]; }

}  // extern "C"
