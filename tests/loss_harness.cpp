// Test-only harness for the robust losses: the product's CLC_HD per-residual and expansion code (clc_expand.cuh) and the LM
// state machine (clc_lm.cuh), compiled with g++ so that the code the GPU runs for every loss kind can be checked against the
// references on a machine without a GPU.  Never shipped, never linked into libclc_b200.so.
#include <cstring>

#include "../camlasercalibratool_b200/csrc/clc_expand.cuh"
#include "../camlasercalibratool_b200/csrc/clc_lm.cuh"

extern "C" {

// w and rho~ of one residual (loss_weight)
void loss_weight(int kind, double e, double a, double* w, double* cost_term) {
  const double a2 = a * a;
  clc::loss_weight(kind, e, a2, 1.0 / a2, w, cost_term);
}
// one residual added directly to acc28: the per-residual code of the one-cluster kernel
void loss_accumulate_residual(const double* plane, const double* pose7, const double* xyz, double count, int kind, double a,
                              double* acc28) {
  clc::PoseConsts pc;
  clc::make_pose_consts(pose7, &pc);
  const double a2 = a * a;
  clc::accumulate_residual(pc, plane, xyz[0], xyz[1], xyz[2], 1.0 / count, kind, a2, 1.0 / a2, acc28);
}
// R residuals (plane r: planes[4 r..], point pts[3 r..], frame size counts[r]) added in order to acc28
void loss_accumulate_all(const double* planes, const double* pose7, const double* pts, const double* counts, int64_t R, int kind,
                         double a, double* acc28) {
  clc::PoseConsts pc;
  clc::make_pose_consts(pose7, &pc);
  const double a2 = a * a;
  for (int64_t r = 0; r < R; ++r)
    clc::accumulate_residual(pc, planes + 4 * r, pts[3 * r], pts[3 * r + 1], pts[3 * r + 2], 1.0 / counts[r], kind, a2, 1.0 / a2,
                             acc28);
}
// one edge residual through its moments (the sweep kernel's edge tail and fix-up kernels); returns e
double loss_edge_residual(const double* plane, const double* pose7, const double* pt, double count, int kind, double a,
                          double* out28) {
  clc::PoseConsts pc;
  clc::make_pose_consts(pose7, &pc);
  const double a2 = a * a;
  return clc::edge_residual(pc, plane, pt, 1.0 / count, kind, a2, 1.0 / a2, out28);
}
// the moments of one piece (computed by the caller) -> the 28 sums
void loss_expand_lm(const double* plane, const double* pose7, double count, const double* S10, int kind, double cost_term,
                    double a, double* out28) {
  clc::PoseConsts pc;
  clc::make_pose_consts(pose7, &pc);
  double m[3], c;
  clc::frame_consts(pc, plane, m, &c);
  clc::expand_lm(plane, m, c, 1.0 / count, S10, kind, cost_term, a * a, out28);
}

int loss_lm_state_size() { return (int)sizeof(clc::LmState); }
void loss_lm_init(void* st, const double* pose7, const clc_lm_options* opt) {
  clc::lm_init(&static_cast<clc::LmState*>(st)->core, pose7, *opt);
}
void loss_lm_update(void* st, const double* sums28) {
  clc::LmState* s = static_cast<clc::LmState*>(st);
  clc::lm_update(&s->core, s->trace, sums28);
}
int loss_lm_done(const void* st) { return static_cast<const clc::LmState*>(st)->core.done; }
int loss_lm_ntrace(const void* st) { return static_cast<const clc::LmState*>(st)->core.n_trace; }
void loss_lm_cand(const void* st, double* out) { std::memcpy(out, static_cast<const clc::LmState*>(st)->core.cand, 56); }
void loss_lm_x(const void* st, double* out) { std::memcpy(out, static_cast<const clc::LmState*>(st)->core.x, 56); }
void loss_lm_trace(const void* st, int i, clc_lm_iteration* out) { *out = static_cast<const clc::LmState*>(st)->trace[i]; }

}  // extern "C"
