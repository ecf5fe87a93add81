// Test-only harness for the frame selection: the product's CLC_HD Cholesky and gain (clc_select.cuh), compiled with g++ so that
// the arithmetic every step kernel thread runs can be checked on a machine without a GPU.  Never shipped, never linked into
// libclc_b200.so.
#include "../camlasercalibratool_b200/csrc/clc_select.cuh"

extern "C" {

// A [36] -> L [36], inv [6]; returns 1 when every pivot is positive and finite
int sel_chol(const double* A, double* L, double* inv) { return clc::sel_chol6(A, L, inv) ? 1 : 0; }

// the gains of m blocks H [m * 36] against the factor of A [36] (sel_chol6, then sel_gain6 per block)
int sel_gains(const double* A, int64_t m, const double* H, double* gain) {
  double L[36], inv[6];
  if (!clc::sel_chol6(A, L, inv)) return 0;
  for (int64_t i = 0; i < m; ++i) gain[i] = clc::sel_gain6(L, inv, H + 36 * i);
  return 1;
}

// the gains of m blocks H [m * 36] at a given factor L [36] (lower, as sel_chol6 writes it) with inv[k] = 1 / L_kk
void sel_gains_at(const double* L, const double* inv, int64_t m, const double* H, double* gain) {
  for (int64_t i = 0; i < m; ++i) gain[i] = clc::sel_gain6(L, inv, H + 36 * i);
}

}  // extern "C"
