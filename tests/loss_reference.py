"""References for the Huber and soft-L1 losses (clc_problem_set_loss), next to the Cauchy / no-loss references of
oracle/ and tests/exact_sums.py, which stay as they are.

Three restatements:
  * the C oracle of the new losses (`COracle`, tests/loss_oracle.c, linked against oracle/libclc_oracle.so for the reference's
    cost model): HuberLoss / SoftLOneLoss / CauchyLoss::Evaluate of Ceres' internal/ceres/loss_function.cc, the Corrector and the
    trust-region LM with DENSE_QR, in plain C;
  * its numpy twin, written apart (`ceres_rho`, `evaluate`, `solve`): the same loss objects on the squared scaled residual
    s = r^2 with parameter a*scale, the Corrector's simple branch (rho'' <= 0: r~ = sqrt(rho') r, J~ = sqrt(rho') J), on
    oracle_np's numpy factor and TrustRegionMinimizer restatement (itself written apart from oracle/clc_oracle.c).
    Soft-L1's cost is Ceres' 2 b (sqrt(1 + s/b) - 1).  The Huber boundary is |e| <= a (inlier), the rule the library uses; it
    is Ceres' `s > b` up to the rounding of (s e)^2 against (a s)^2.
  * Long double (`lm_sums`): every per-residual term of the 28 sums in extended precision, with the magnitudes A_k of
    tests/exact_sums.py generalised to the kind's weight w and w' = dw/de.  The soft-L1 cost uses the cancellation-free
    2 e^2 / (1 + sqrt(1 + z)).  kind "none" / "cauchy" return exactly what exact_sums.lm_sums returns.

Test infrastructure only.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import exact_sums as X
from oracle import oracle as O
from oracle import oracle_np as ONP

LD = X.LD
KINDS = ("none", "cauchy", "huber", "soft_l1")
TINY = np.finfo(float).tiny


# ---- the C oracle of the new losses (tests/loss_oracle.c) ----------------------------------------------------------------
class COracle:
    """ctypes view of tests/loss_oracle.c, compiled into `out_dir` against oracle/libclc_oracle.so."""

    def __init__(self, out_dir):
        lib_path = O.build()
        here = os.path.dirname(os.path.abspath(__file__))
        odir = os.path.dirname(lib_path)
        out = os.path.join(str(out_dir), "libloss_oracle.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([cc, "-O2", "-std=c11", "-Wall", "-Wextra", "-shared", "-fPIC", "-I", odir, "-o", out,
                               os.path.join(here, "loss_oracle.c"), lib_path, "-Wl,-rpath," + odir, "-lm"])
        L = C.CDLL(out)
        dp = C.POINTER(C.c_double)
        L.loss_oracle_evaluate.argtypes = [C.POINTER(O._Problem), dp, dp, dp, dp, dp]
        L.loss_oracle_solve.argtypes = [C.POINTER(O._Problem), dp, C.POINTER(O.Options), C.POINTER(O.Summary),
                                        C.POINTER(O.Iteration), C.c_int]
        self.L = L

    @staticmethod
    def _problem(p, kind, a):
        c = O._Problem()
        C.pointer(c)[0] = p._c
        c.use_loss = KINDS.index(kind)  # CLC_LOSS_*: the kind travels in use_loss, a in cauchy_a
        c.cauchy_a = float(a)
        return c

    def evaluate(self, p, pose7, kind, a=0.05):
        """cost, corrected residuals [R], corrected local Jacobian [R, 6] of the oracle.Problem p."""
        c = self._problem(p, kind, a)
        R = p.num_residuals()
        cost, r, J, g = C.c_double(), np.empty(R), np.empty((R, 6)), np.empty(6)
        x = np.ascontiguousarray(pose7, dtype=np.float64)
        self.L.loss_oracle_evaluate(C.byref(c), O._dp(x), C.byref(cost), O._dp(r), O._dp(J), O._dp(g))
        return cost.value, r, J

    def solve(self, p, pose7, kind, a=0.05, options=None, trace_cap=256):
        """(pose7, oracle Summary, [Iteration...]) of the Ceres LM under the loss."""
        c = self._problem(p, kind, a)
        x = np.array(pose7, dtype=np.float64)
        s, tr = O.Summary(), (O.Iteration * trace_cap)()
        self.L.loss_oracle_solve(C.byref(c), O._dp(x), C.byref(options or O.default_options()), C.byref(s), tr, trace_cap)
        return x, s, list(tr[: min(s.num_iterations, trace_cap)])


# ---- Ceres' loss objects, on s = r^2 with parameter `a` (already scaled) --------------------------------------------
def ceres_rho(kind, s, a):
    """rho[3] = (rho(s), rho'(s), rho''(s)) of Ceres' loss `kind` with parameter a, vectorised over s (float64)."""
    s = np.asarray(s, dtype=np.float64)
    b = a * a
    if kind == "none":
        return s.copy(), np.ones_like(s), np.zeros_like(s)
    if kind == "cauchy":  # CauchyLoss::Evaluate
        c = 1.0 / b
        summ = 1.0 + s * c
        inv = 1.0 / summ
        return b * np.log(summ), np.maximum(TINY, inv), -c * (inv * inv)
    if kind == "huber":  # HuberLoss::Evaluate, outlier test on |r| > a (see the module docstring)
        r = np.sqrt(s)
        out = r > a
        with np.errstate(divide="ignore", invalid="ignore"):
            rho1_out = np.maximum(TINY, a / r)
            rho2_out = -rho1_out / (2.0 * s)
        return (np.where(out, 2.0 * a * r - b, s), np.where(out, rho1_out, 1.0), np.where(out, rho2_out, 0.0))
    if kind == "soft_l1":  # SoftLOneLoss::Evaluate
        c = 1.0 / b
        summ = 1.0 + s * c
        tmp = np.sqrt(summ)
        rho1 = np.maximum(TINY, 1.0 / tmp)
        return 2.0 * b * (tmp - 1.0), rho1, -(c * rho1) / (2.0 * summ)
    raise ValueError(kind)


def evaluate(table, pose7, kind, a=0.05):
    """PointInPlaneFactor::Evaluate (reference :43-66) of every row of oracle_np.residual_table with the frame's loss
    `kind`(a * scale) and the Corrector: cost, corrected residuals [R], corrected local Jacobian [R, 6]."""
    cost, r, J = ONP.evaluate(table, pose7, use_loss=False)
    s = table[2]
    rho = ceres_rho(kind, r * r, a * s)
    if kind == "huber":  # the library's inlier rule |e| <= a, decided on the unscaled distance
        e = r / s
        inl = np.abs(e) <= a
        rho = (np.where(inl, r * r, rho[0]), np.where(inl, 1.0, rho[1]), np.where(inl, 0.0, rho[2]))
    assert np.all(rho[2] <= 0.0)  # Corrector: the simple branch
    sq = np.sqrt(rho[1])
    return 0.5 * float(np.sum(rho[0])), r * sq, J * sq[:, None]


def solve(table, pose7, kind, a=0.05, max_num_iterations=100):
    """Ceres' LM (oracle_np.trust_region_lm, the defaults of the reference's solve) with the loss `kind`(a * scale)."""
    return ONP.trust_region_lm(lambda x: evaluate(table, x, kind, a), ONP.pose_plus, pose7, max_num_iterations,
                               ONP.gradient_max_norm)


# ---- closed forms of w = rho' and the cost term rho~ per unscaled distance e (DESIGN section 2) ------------------------
def weight_and_cost(kind, e, a):
    """(w, rho~, |dw/de|) in long double for raw distances e: the frame's cost is 1/2 s^2 sum rho~."""
    e = np.asarray(e).astype(LD)
    a = LD(a)
    a2 = a * a
    if kind == "none":
        return np.ones_like(e), e * e, np.zeros_like(e)
    if kind == "cauchy":
        q = e * e / a2
        w = LD(1) / (LD(1) + q)
        return w, a2 * np.log1p(q), 2 * np.abs(e) * w * w / a2
    if kind == "huber":
        ae = np.abs(e)
        inl = ae <= a
        with np.errstate(divide="ignore"):
            w = np.where(inl, LD(1), a / np.where(inl, LD(1), ae))
            dw = np.where(inl, LD(0), a / np.where(inl, LD(1), ae * ae))
        return w, np.where(inl, e * e, 2 * a * ae - a2), dw
    if kind == "soft_l1":
        u = LD(1) + e * e / a2
        t = np.sqrt(u)
        w = LD(1) / t
        return w, 2 * e * e / (LD(1) + t), np.abs(e) / a2 * w * w * w
    raise ValueError(kind)


def lm_sums(frame_pose, offsets, points, pose7, kind, a=0.05, edge_points=None):
    """The 28 sums of one LM sweep under the loss `kind` in long double, and their magnitudes A_k (float64)."""
    return lm_sums_of_blocks(X._residual_blocks(frame_pose, offsets, points, edge_points), pose7, kind, a)


def lm_sums_of_blocks(blocks, pose7, kind, a=0.05):
    if kind in ("none", "cauchy"):
        return X.lm_sums_of_blocks(blocks, pose7, kind == "cauchy", a)
    pose = np.asarray(pose7, dtype=np.float64).astype(LD)
    R, t = X._rot(pose[3:7]), pose[:3]
    val = np.zeros(28, dtype=LD)
    mag = np.zeros(28)
    for plane, p, s2 in blocks:
        n, d = plane[:, :3], plane[:, 3]
        m = n @ R
        c = n @ t + d
        e = np.sum(m * p, axis=-1) + c
        L_e = X._norm(m) * X._norm(p) + X._norm(n) * X._norm(t) + np.abs(d)
        J = np.concatenate([n, X._cross(p, m)], axis=1)
        Jabs = np.concatenate([np.abs(n), np.repeat((X._norm(p) * X._norm(m))[:, None], 3, axis=1)], axis=1)
        w, rho, dw = weight_and_cost(kind, e, a)
        cost = LD(0.5) * s2 * rho
        cost_mag = LD(0.5) * s2 * np.abs(rho) + s2 * w * np.abs(e) * L_e
        sw = s2 * w
        H = (J * sw[:, None]).T @ J
        val[:21] += H[X.IU6]
        val[21:27] += (J * (sw * e)[:, None]).sum(axis=0)
        val[27] += cost.sum()
        Jf = Jabs.astype(np.float64)
        Hm = (Jf * (s2 * (w + dw * L_e)).astype(np.float64)[:, None]).T @ Jf
        mag[:21] += Hm[X.IU6]
        mag[21:27] += (Jf * (sw * L_e).astype(np.float64)[:, None]).sum(axis=0)
        mag[27] += float(cost_mag.sum())
    return val, mag


def frame_sums(frame_pose, offsets, points, pose7, kind, a=0.05, edge_points=None):
    """lm_sums of every frame on its own (its points and, with edge_points, its two edge residuals): [N] (val, mag) pairs."""
    offsets = np.asarray(offsets, dtype=np.int64)
    out = []
    for f in range(len(offsets) - 1):
        b, e = int(offsets[f]), int(offsets[f + 1])
        ep = None if edge_points is None else np.asarray(edge_points)[f:f + 1]
        out.append(lm_sums(np.asarray(frame_pose)[f:f + 1], np.array([0, e - b]), np.asarray(points)[b:e], pose7, kind, a, ep))
    return out
