// clc_math.cuh -- small host/device math shared by the kernels and the C-ABI host code.
//
// SE(3) conventions follow the reference: pose7 = (t, qx,qy,qz,qw) (src/LaseCamCalCeres.cpp:219), the
// right-multiplicative first-order quaternion update of src/pose_local_parameterization.cpp:3-32, and Eigen's
// quaternion <-> matrix conversions (used by the reference at :215 and :311-313).
#pragma once

#include <cstdint>
#include <cmath>
#include <cfloat>

#if defined(__CUDACC__)
#define CLC_HD __host__ __device__ __forceinline__
#else
#define CLC_HD inline
#endif

namespace clc {

CLC_HD bool is_finite(double v) { return fabs(v) <= DBL_MAX; }  // false for NaN and +-inf

// ---- Eigen-equivalent conversions -----------------------------------------------------------------------

// Eigen QuaternionBase::toRotationMatrix, q = (x,y,z,w), row-major R; q is NOT normalised here.
CLC_HD void quat_to_rot(const double* q, double* R) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w;
  const double txx = tx * x, txy = ty * x, txz = tz * x;
  const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1.0 - (tyy + tzz); R[1] = txy - twz;         R[2] = txz + twy;
  R[3] = txy + twz;         R[4] = 1.0 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;         R[7] = tyz + twx;         R[8] = 1.0 - (txx + tyy);
}

// Eigen Quaternion(Matrix3) (Shoemake); row-major R -> (x,y,z,w).
CLC_HD void rot_to_quat(const double* R, double* q) {
  double t = R[0] + R[4] + R[8];
  if (t > 0.0) {
    t = sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (R[7] - R[5]) * t;
    q[1] = (R[2] - R[6]) * t;
    q[2] = (R[3] - R[1]) * t;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[i * 4]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(R[i * 4] - R[j * 4] - R[k * 4] + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (R[k * 3 + j] - R[j * 3 + k]) * t;
    q[j] = (R[j * 3 + i] + R[i * 3 + j]) * t;
    q[k] = (R[k * 3 + i] + R[i * 3 + k]) * t;
  }
}

// x (+) delta of PoseLocalParameterization::Plus.
CLC_HD void pose_plus(const double* x, const double* d, double* xp) {
  xp[0] = x[0] + d[0]; xp[1] = x[1] + d[1]; xp[2] = x[2] + d[2];
  const double ax = x[3], ay = x[4], az = x[5], aw = x[6];
  const double bx = 0.5 * d[3], by = 0.5 * d[4], bz = 0.5 * d[5];
  const double w = aw - ax * bx - ay * by - az * bz;
  const double xx = aw * bx + ax + ay * bz - az * by;
  const double yy = aw * by + ay + az * bx - ax * bz;
  const double zz = aw * bz + az + ax * by - ay * bx;
  const double inv = 1.0 / sqrt(xx * xx + yy * yy + zz * zz + w * w);
  xp[3] = xx * inv; xp[4] = yy * inv; xp[5] = zz * inv; xp[6] = w * inv;
}

// ---- planes ----------------------------------------------------------------------------------------------

// Board plane in the camera frame, reference src/LaseCamCalCeres.cpp:227-231: (Tctag^-1)^T (0,0,1,0) =
// (row 2 of A^-1, -(row 2 of A^-1).t) with A = R(Qca) (general inverse: A is not assumed orthonormal).
CLC_HD void frame_plane(const double* fp, double* plane) {
  double A[9];
  quat_to_rot(fp, A);
  const double c0 = A[3] * A[7] - A[4] * A[6];
  const double c1 = A[1] * A[6] - A[0] * A[7];
  const double c2 = A[0] * A[4] - A[1] * A[3];
  const double inv_det = 1.0 / (A[2] * c0 + A[5] * c1 + A[8] * c2);
  const double n0 = c0 * inv_det, n1 = c1 * inv_det, n2 = c2 * inv_det;
  plane[0] = n0; plane[1] = n1; plane[2] = n2;
  plane[3] = -(n0 * fp[4] + n1 * fp[5] + n2 * fp[6]);
}

CLC_HD void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// Board-edge planes through the optical centre, reference :262-276 with pi_from_ppp (utilities.cpp:267-272)
// evaluated at x3 = 0: pi = (x1 x x2, 0).  Normals are deliberately left un-normalised, as in the reference.
CLC_HD void edge_planes(const double* fp, double* pi1, double* pi2) {
  const double o = 0.0265 + 0.0165;
  const double pm[3][3] = {{-o, -o, 0.0}, {0.5 - o, -o, 0.0}, {-o, 0.5 - o, 0.0}};
  double R[9], pc[3][3];
  quat_to_rot(fp, R);
  for (int k = 0; k < 3; ++k)
    for (int r = 0; r < 3; ++r)
      pc[k][r] = (R[r * 3] * pm[k][0] + R[r * 3 + 1] * pm[k][1] + R[r * 3 + 2] * pm[k][2]) + fp[4 + r];
  cross3(pc[0], pc[1], pi1);
  cross3(pc[0], pc[2], pi2);
  pi1[3] = 0.0;
  pi2[3] = 0.0;
}

// ---- counter-based RNG + synthetic board poses (reference main/calibr_simulation.cpp:10-108) --------------

CLC_HD void philox4x32(uint64_t seed, uint64_t ctr_lo, uint64_t ctr_hi, uint32_t* out) {
  uint32_t c0 = (uint32_t)ctr_lo, c1 = (uint32_t)(ctr_lo >> 32), c2 = (uint32_t)ctr_hi, c3 = (uint32_t)(ctr_hi >> 32);
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    const uint32_t n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    const uint32_t n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

CLC_HD double u53(uint32_t hi, uint32_t lo) {
  return (double)((((uint64_t)hi << 32) | lo) >> 11) * (1.0 / 9007199254740992.0);
}

constexpr uint64_t kStreamPose = (uint64_t)1 << 56;
constexpr uint64_t kStreamNoise = (uint64_t)2 << 56;
constexpr double kPi = 3.14159265358979323846;

// Ground truth of the generator: Rlc rows (0,0,1),(-1,0,0),(0,-1,0), tlc = (0.1,0.2,0.3)  (:15-20)
CLC_HD void gen_to_laser(const double* pc, double* pl) {  // p_l = Rlc p_c + tlc
  pl[0] = pc[2] + 0.1;
  pl[1] = -pc[0] + 0.2;
  pl[2] = -pc[1] + 0.3;
}

// yaw,pitch,roll ~ U(-pi/6,pi/6), Rca = Rz Ry Rx; tca = (U(-3,3),U(-3,3),U(1,5))   (:30-32,42-44,58)
CLC_HD void gen_draw_pose(uint64_t seed, int64_t frame, int attempt, double* fp) {
  double u[6];
  for (int b = 0; b < 3; ++b) {
    uint32_t o[4];
    philox4x32(seed, (uint64_t)frame, kStreamPose | ((uint64_t)attempt << 8) | (uint64_t)b, o);
    u[2 * b] = u53(o[0], o[1]);
    u[2 * b + 1] = u53(o[2], o[3]);
  }
  const double lim = kPi / 6.;
  const double yaw = -lim + 2.0 * lim * u[0], pitch = -lim + 2.0 * lim * u[1], roll = -lim + 2.0 * lim * u[2];
  const double cz = cos(yaw), sz = sin(yaw), cy = cos(pitch), sy = sin(pitch), cx = cos(roll), sx = sin(roll);
  const double R[9] = {cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx,
                       sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx,
                       -sy,     cy * sx,                cy * cx};
  rot_to_quat(R, fp);
  fp[4] = -3.0 + 6.0 * u[3];
  fp[5] = -3.0 + 6.0 * u[4];
  fp[6] = 1.0 + 4.0 * u[5];
}

// Board plane in the laser frame (:62-73).
CLC_HD void gen_plane_laser(const double* fp, double* nl, double* dl) {
  double Rca[9];
  quat_to_rot(fp, Rca);
  const double nc[3] = {Rca[2], Rca[5], Rca[8]};
  nl[0] = nc[2]; nl[1] = -nc[0]; nl[2] = -nc[1];  // Rlc nc
  double tla[3];
  gen_to_laser(fp + 4, tla);
  *dl = -(nl[0] * tla[0] + nl[1] * tla[1] + nl[2] * tla[2]);
}

// Valid beam window of a frame: the part of the line nx x + ny y + d = 0 inside 0 <= x < 5, |y| < 5
// (equivalent to the validity filter :83-94).  false if shorter than 0.2 m.
CLC_HD bool gen_window(const double* nl, double dl, double* th_a, double* th_b) {
  const double rho2 = nl[0] * nl[0] + nl[1] * nl[1];
  if (!(rho2 > 1e-12) || !(fabs(dl) > 1e-9)) return false;
  const double rho = sqrt(rho2);
  const double uu[2] = {-nl[1] / rho, nl[0] / rho};
  const double pp[2] = {-dl * nl[0] / rho2, -dl * nl[1] / rho2};
  const double lim = 5.0 * (1.0 - 1e-3);
  const double lo[2] = {0.0, -lim}, hi[2] = {lim, lim};
  double s0 = -1e30, s1 = 1e30;
  for (int a = 0; a < 2; ++a) {
    if (fabs(uu[a]) < 1e-14) {
      if (pp[a] < lo[a] || pp[a] > hi[a]) return false;
    } else {
      double ta = (lo[a] - pp[a]) / uu[a], tb = (hi[a] - pp[a]) / uu[a];
      if (ta > tb) { const double t = ta; ta = tb; tb = t; }
      if (ta > s0) s0 = ta;
      if (tb < s1) s1 = tb;
    }
  }
  if (!(s1 - s0 >= 0.2)) return false;
  *th_a = atan2(pp[1] + s0 * uu[1], pp[0] + s0 * uu[0]);
  *th_b = atan2(pp[1] + s1 * uu[1], pp[0] + s1 * uu[0]);
  return true;
}

// Edge-residual points: board-edge lines p1p2 / p1p3 (corners of reference :262-268) intersected with the scan
// plane z_l = 0, so both edge residuals vanish at ground truth.
CLC_HD bool gen_edge_points(const double* fp, double* ep) {
  const double o = 0.0265 + 0.0165;
  const double pm[3][3] = {{-o, -o, 0.0}, {0.5 - o, -o, 0.0}, {-o, 0.5 - o, 0.0}};
  double Rca[9], pl[3][3];
  quat_to_rot(fp, Rca);
  for (int k = 0; k < 3; ++k) {
    double pc[3];
    for (int r = 0; r < 3; ++r)
      pc[r] = (Rca[r * 3] * pm[k][0] + Rca[r * 3 + 1] * pm[k][1] + Rca[r * 3 + 2] * pm[k][2]) + fp[4 + r];
    gen_to_laser(pc, pl[k]);
  }
  for (int e = 0; e < 2; ++e) {
    const double* a = pl[0];
    const double* b = pl[1 + e];
    const double dz = b[2] - a[2];
    if (!(fabs(dz) > 1e-9)) return false;
    const double lam = -a[2] / dz;
    if (!(fabs(lam) <= 8.0)) return false;
    ep[3 * e] = a[0] + lam * (b[0] - a[0]);
    ep[3 * e + 1] = a[1] + lam * (b[1] - a[1]);
    ep[3 * e + 2] = 0.0;
  }
  return true;
}

// exact-M accept/redraw rule (up to 64 attempts per frame).
CLC_HD void gen_frame_pose(uint64_t seed, int64_t frame, bool with_edges, double* fp) {
  for (int attempt = 0; attempt < 64; ++attempt) {
    gen_draw_pose(seed, frame, attempt, fp);
    double nl[3], dl, a, b;
    gen_plane_laser(fp, nl, &dl);
    bool ok = gen_window(nl, dl, &a, &b);
    if (ok && with_edges) {
      double ep[6];
      ok = gen_edge_points(fp, ep);
    }
    if (ok) return;
  }
}

CLC_HD double gen_noise(uint64_t seed, double sigma, int64_t frame, int64_t beam) {
  if (!(sigma > 0.0)) return 0.0;
  uint32_t o[4];
  philox4x32(seed, (uint64_t)frame, kStreamNoise | (uint64_t)beam, o);
  const double u1 = u53(o[0], o[1]), u2 = u53(o[2], o[3]);
  return sigma * sqrt(-2.0 * log(1.0 - u1)) * cos(2.0 * kPi * u2);
}

// ---- dense pieces of the LM step (6 columns: the pose; 7: the pose and the time offset) ------------------------------

template <int N = 6>
CLC_HD int tri(int i, int j) { return i * N - (i * (i - 1)) / 2 + (j - i); }  // upper-tri index of the NxN, i <= j

// Cholesky solve of the SPD NxN system A y = b (A full row-major).  false if not positive definite.
template <int N>
CLC_HD bool chol_solve(const double* A, const double* b, double* y) {
  // fully unrolled (L, z, inv live in registers): it always runs on the same SM (block 0), whose instruction cache keeps it.
  // One reciprocal per pivot instead of one division per entry (divisions are ~100-cycle subroutines in FP64).
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

CLC_HD bool chol6_solve(const double* A, const double* b, double* y) { return chol_solve<6>(A, b, y); }

}  // namespace clc
