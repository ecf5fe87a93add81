// Test-only harness for the range bias: the product's CLC_HD 45-sum expansion and 8-column LM state machine
// (clc_range_bias.cuh), compiled with g++ so that the code the GPU runs can be checked on a machine without a GPU.  Never
// shipped, never linked into libclc_b200.so.
#include <cstring>

#include "../camlasercalibratool_b200/csrc/clc_range_bias.cuh"

extern "C" {

// the 25 moments of one piece -> the 45 sums at pose7 and (b, s) with the frame's plane (n, d)
void rb_expand(const double* plane, const double* pose7, double b, double s, double count, const double* M25, int kind,
               double cost_term, double a, double* out45) {
  clc::PoseConsts pc;
  clc::make_pose_consts(pose7, &pc);
  double m[3], c;
  clc::frame_consts(pc, plane, m, &c);
  clc::expand_lm_range(plane, m, c, b, s, 1.0 / count, M25, kind, cost_term, a * a, out45);
}
double rb_kappa(double x, double y, double z, double b, double s) { return clc::range_kappa(x, y, z, b, s); }

struct RbState {
  clc::LmCoreRange core;
  clc_lm_iteration trace[clc::kTraceMax];
};
int rb_lm_state_size() { return (int)sizeof(RbState); }
void rb_lm_init(void* st, const double* x9, const clc_lm_options* opt) { clc::lm_init(&static_cast<RbState*>(st)->core, x9, *opt); }
void rb_lm_update(void* st, const double* sums45) {
  RbState* s = static_cast<RbState*>(st);
  clc::lm_update(&s->core, clc::TraceRows{s->trace, clc::kTraceMax}, sums45);
}
int rb_lm_done(const void* st) { return static_cast<const RbState*>(st)->core.done; }
int rb_lm_ntrace(const void* st) { return static_cast<const RbState*>(st)->core.n_trace; }
void rb_lm_cand(const void* st, double* out9) { std::memcpy(out9, static_cast<const RbState*>(st)->core.cand, 72); }
void rb_lm_x(const void* st, double* out9) { std::memcpy(out9, static_cast<const RbState*>(st)->core.x, 72); }
void rb_lm_trace(const void* st, int i, clc_lm_iteration* out) { *out = static_cast<const RbState*>(st)->trace[i]; }

}  // extern "C"
