"""Long-double and numpy restatements of the range bias (csrc/clc_range_bias.cuh) for the CPU and GPU tests, and synthetic
scenes with a known range offset b and scale s.  Test infrastructure only.

The model: a reported point p (r = |p|) lies at kappa p, kappa = 1 + s + b / r (r == 0: kappa p = 0); the residual is
e = kappa (m.p) + c, and the Jacobian over (tx ty tz rx ry rz b s) is [n, kappa (p x m), (m.p) / r, m.p], each times the frame's
scale 1/sqrt(#points)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import exact_sums as X
import loss_reference as LR
from oracle import oracle_np as ONP

LD = X.LD
IU8 = np.triu_indices(8)
GROUPS_RB = {"H_pose": [k for k, (i, j) in enumerate(zip(*IU8)) if j < 6],
             "H_bias": [k for k, (i, j) in enumerate(zip(*IU8)) if j >= 6],
             "g": list(range(36, 44)), "cost": [44]}


class RbHarness:
    def __init__(self, out_dir):
        here = os.path.dirname(os.path.abspath(__file__))
        out = os.path.join(str(out_dir), "librange_bias_harness.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", out,
                               os.path.join(here, "range_bias_harness.cpp")])
        from camlasercalibratool_b200._lib import LmIteration, LmOptions

        L = C.CDLL(out)
        dp = C.POINTER(C.c_double)
        L.rb_expand.argtypes = [dp, dp, C.c_double, C.c_double, C.c_double, dp, C.c_int, C.c_double, C.c_double, dp]
        L.rb_kappa.argtypes = [C.c_double] * 5
        L.rb_kappa.restype = C.c_double
        L.rb_lm_init.argtypes = [C.c_void_p, dp, C.POINTER(LmOptions)]
        L.rb_lm_update.argtypes = [C.c_void_p, dp]
        for f in ("rb_lm_done", "rb_lm_ntrace"):
            getattr(L, f).argtypes = [C.c_void_p]
        L.rb_lm_cand.argtypes = [C.c_void_p, dp]
        L.rb_lm_x.argtypes = [C.c_void_p, dp]
        L.rb_lm_trace.argtypes = [C.c_void_p, C.c_int, C.POINTER(LmIteration)]
        self.L, self.LmIteration, self.LmOptions = L, LmIteration, LmOptions

    @staticmethod
    def dp(a):
        return a.ctypes.data_as(C.POINTER(C.c_double))

    def expand(self, plane, pose7, b, s, count, M25, kind, cost_term, a):
        out = np.zeros(45)
        pl, x, M = (np.ascontiguousarray(v, dtype=np.float64) for v in (plane, pose7, M25))
        self.L.rb_expand(self.dp(pl), self.dp(x), float(b), float(s), float(count), self.dp(M), LR.KINDS.index(kind),
                         float(cost_term), float(a), self.dp(out))
        return out

    def default_options(self, **kw):
        o = self.LmOptions(100, 1e4, 1e16, 1e-32, 1e-3, 1e-6, 1e32, 1e-6, 1e-10, 1e-8, 5, 1, 8, 0)
        for k, v in kw.items():
            setattr(o, k, v)
        return o

    def lm_run(self, sums_fn, x9, options, max_sweeps=300):
        """lm_update<8> driven as the device loop drives it: sums_fn(x9) -> the 45 sums at x9 = (pose7, b, s)."""
        st = C.create_string_buffer(self.L.rb_lm_state_size())
        x0 = np.ascontiguousarray(x9, dtype=np.float64)
        self.L.rb_lm_init(st, self.dp(x0), C.byref(options))
        cand, n = np.empty(9), 0
        while not self.L.rb_lm_done(st) and n < max_sweeps:
            self.L.rb_lm_cand(st, self.dp(cand))
            sums = np.ascontiguousarray(sums_fn(cand.copy()), dtype=np.float64)
            self.L.rb_lm_update(st, self.dp(sums))
            n += 1
        x = np.empty(9)
        self.L.rb_lm_x(st, self.dp(x))
        trace = []
        for i in range(min(self.L.rb_lm_ntrace(st), 256)):
            it = self.LmIteration()
            self.L.rb_lm_trace(st, i, C.byref(it))
            trace.append(it)
        return x, self.L.rb_lm_done(st), trace


# ---- the 45 sums in long double -------------------------------------------------------------------------------------------
def moments25(points, w):
    """The 25 range moments (RangeMoments order) of points [P, 3] with weights w [P], long double."""
    p = np.asarray(points, dtype=np.float64).astype(LD)
    w = np.asarray(w, dtype=LD)
    r = np.sqrt(np.sum(p * p, axis=1))
    ir = np.where(r > 0, LD(1) / np.where(r > 0, r, 1), LD(0))
    out = [w.sum()]
    out += list((w[:, None] * p).sum(0))
    pp = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]
    out += [(w * p[:, i] * p[:, j]).sum() for i, j in pp]
    out += list((w[:, None] * p * ir[:, None]).sum(0))
    out += [(w * p[:, i] * p[:, j] * ir).sum() for i, j in pp]
    out += [(w * p[:, i] * p[:, j] * ir * ir).sum() for i, j in pp]
    return np.array(out, dtype=LD)


def residuals_ld(plane, points, pose7, b, s):
    """(e [P], J [P, 8] without the frame scale, the bound L_e of e's rounding) of one frame, long double."""
    pose = np.asarray(pose7, dtype=np.float64).astype(LD)
    R, t = X._rot(pose[3:7]), pose[:3]
    pl = np.asarray(plane, dtype=LD)
    n, d = pl[:3], pl[3]
    m, c = n @ R, n @ t + d
    p = np.asarray(points, dtype=np.float64).astype(LD)
    r = np.sqrt(np.sum(p * p, axis=1))
    ir = np.where(r > 0, LD(1) / np.where(r > 0, r, 1), LD(0))
    kap = LD(1) + LD(s) + LD(b) * ir
    y = p @ m
    e = kap * y + c
    J = np.concatenate([np.tile(n, (len(p), 1)), kap[:, None] * X._cross(p, np.tile(m, (len(p), 1))), (y * ir)[:, None],
                        y[:, None]], axis=1)
    L_e = np.abs(kap) * X._norm(m) * r + X._norm(n) * X._norm(t) + np.abs(d)
    return e, J, L_e, kap, r, m


def rb_sums(planes, offsets, points, pose7, b, s, kind, a=0.05):
    """The 45 sums (36 upper-tri H over tx ty tz rx ry rz b s, 8 g, cost) by direct accumulation of every residual's 8-column
    Jacobian in long double, and their magnitudes A_k (exact_sums' bounds, extended to the two bias columns: |J_b| <= |m|,
    |J_s| <= |m| r, each taken twice for the rounding of kappa and 1/r)."""
    offsets = np.asarray(offsets, dtype=np.int64)
    val, mag = np.zeros(45, dtype=LD), np.zeros(45)
    for f in range(len(offsets) - 1):
        a0, a1 = offsets[f], offsets[f + 1]
        if a1 <= a0:
            continue
        s2 = LD(1) / LD(a1 - a0)
        e, J, L_e, kap, r, m = residuals_ld(planes[f], points[a0:a1], pose7, b, s)
        w, rho, dw = LR.weight_and_cost(kind, e, a)
        sw = s2 * w
        val[:36] += ((J * sw[:, None]).T @ J)[IU8]
        val[36:44] += (J * (sw * e)[:, None]).sum(axis=0)
        val[44] += (LD(0.5) * s2 * rho).sum()
        nm = X._norm(m)
        pm = np.abs(kap) * r * nm
        n = np.asarray(planes[f], dtype=LD)[:3]
        Jabs = np.concatenate([np.tile(np.abs(n) + 1, (len(e), 1)), np.repeat((2 * pm)[:, None], 3, axis=1),
                               np.repeat((2 * nm), len(e))[:, None], (2 * nm * r)[:, None]], axis=1).astype(np.float64)
        mag[:36] += ((Jabs * (s2 * (w + dw * L_e)).astype(np.float64)[:, None]).T @ Jabs)[IU8]
        mag[36:44] += (Jabs * (sw * L_e).astype(np.float64)[:, None]).sum(axis=0)
        cm = LD(0.5) * s2 * np.abs(rho) + s2 * w * np.abs(e) * L_e
        if kind == "cauchy":
            cm = cm + LD(0.5) * s2 * LD(a) ** 2 * LD(X.U_PROD)
        mag[44] += float(cm.sum())
    return val, mag


def sums_at(scene, x9, kind, a=0.05):
    """The 45 sums at x9 = (pose7, b, s), rounded to float64 (what the LM harness is fed)."""
    val, _ = rb_sums(scene.planes, scene.offsets, scene.points, x9[:7], x9[7], x9[8], kind, a)
    return val.astype(np.float64)


# ---- the numpy restatement of the solve -------------------------------------------------------------------------------------
def evaluate8(scene, x9, kind, a=0.05):
    """(cost, corrected residuals [P], corrected Jacobian [P, 8]) at x9, float64 (the Corrector's simple branch)."""
    counts = np.diff(scene.offsets)
    f_of = np.repeat(np.arange(len(counts)), counts)
    sc = 1.0 / np.sqrt(counts[f_of].astype(np.float64))
    P = np.asarray(scene.planes, dtype=np.float64)
    R, t = ONP.quat_to_rot(x9[3:7]), x9[:3]
    n, d = P[f_of, :3], P[f_of, 3]
    m = n @ R
    pts = scene.points
    rr = np.linalg.norm(pts, axis=1)
    ir = np.where(rr > 0, 1.0 / np.where(rr > 0, rr, 1.0), 0.0)
    kap = 1.0 + x9[8] + x9[7] * ir
    y = np.sum(m * pts, axis=1)
    e = kap * y + np.sum(n * t, axis=1) + d
    r = sc * e
    J = sc[:, None] * np.concatenate([n, kap[:, None] * np.cross(pts, m), (y * ir)[:, None], y[:, None]], axis=1)
    rho = LR.ceres_rho(kind, r * r, a * sc)
    if kind == "huber":
        inl = np.abs(e) <= a
        rho = (np.where(inl, r * r, rho[0]), np.where(inl, 1.0, rho[1]), np.where(inl, 0.0, rho[2]))
    sq = np.sqrt(rho[1])
    return 0.5 * float(np.sum(rho[0])), r * sq, J * sq[:, None]


def solve8(scene, x9, kind, a=0.05, fixed_mask=0, max_num_iterations=100):
    """Ceres' LM on the pose (PoseLocalParameterization), b and s through oracle_np.trust_region_lm; the held coordinates of
    fixed_mask are dropped from the Jacobian and embedded as zeros.  Returns (x9, termination name, trace dicts)."""
    free = [k for k in range(8) if not (fixed_mask >> k) & 1]

    def embed(v):
        full = np.zeros(8)
        full[free] = v
        return full

    def ev(x):
        cost, r, J = evaluate8(scene, x, kind, a)
        return cost, r, J[:, free]

    def plus(x, dv):
        dfull = embed(dv)
        out = np.concatenate([ONP.pose_plus(x[:7], dfull[:6]), x[7:9] + dfull[6:8]])
        for k in (0, 1, 2, 6, 7):
            if fixed_mask >> k & 1:
                out[k if k < 3 else k + 1] = x[k if k < 3 else k + 1]
        return out

    def gnorm(x, gv):
        g = embed(gv)
        return max(ONP.gradient_max_norm(x[:7], g[:6]), abs(g[6]), abs(g[7]))

    return ONP.trust_region_lm(ev, plus, np.asarray(x9, dtype=np.float64), max_num_iterations, gnorm)


# ---- scenes ---------------------------------------------------------------------------------------------------------------
def truth_pose7():
    """T_cl of the scenes: the laser 5 cm beside and 3 cm below the camera, turned a few degrees."""
    ax = np.array([0.2, -0.5, 0.3])
    ang = 0.08
    q = np.concatenate([np.sin(ang / 2) * ax / np.linalg.norm(ax), [np.cos(ang / 2)]])
    return np.concatenate([[0.05, -0.03, 0.02], q])


class Scene:
    pass


def _quat_from_rot(R):
    w = np.sqrt(max(1e-300, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    return np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])


def scene(n_frames=40, beams=120, b=0.025, s=0.005, sigma=0.0, ranges=(0.8, 4.0), planar=False, seed=0, pose7=None):
    """Boards at distances spread over `ranges` in front of the laser, seen by `beams` rays each.  The true points lie on the
    boards at T_cl = pose7 (truth_pose7 by default); the reported ones are the true ones moved along their rays to the range
    (r_true - b) / (1 + s), plus sigma of noise along the ray, so that kappa p of the true (b, s) puts them back on the board.
    planar: every ray in the laser's z = 0 plane; otherwise the rays fan out +-0.3 rad in elevation as well."""
    rng = np.random.default_rng(seed)
    x = truth_pose7() if pose7 is None else np.asarray(pose7, dtype=np.float64)
    R, t = ONP.quat_to_rot(x[3:]), x[:3]
    frame_pose, pts, off = [], [], [0]
    while len(frame_pose) < n_frames:
        dist = rng.uniform(*ranges)
        az = rng.uniform(-0.6, 0.6)
        center_l = dist * np.array([np.cos(az), np.sin(az), 0.0])
        center_c = R @ center_l + t
        # the board faces the camera with a tilt; its z axis is the normal
        nz = -center_c / np.linalg.norm(center_c) + 0.4 * rng.standard_normal(3)
        nz /= np.linalg.norm(nz)
        xa = np.cross([0.0, 1.0, 0.0], nz)
        xa /= np.linalg.norm(xa)
        Rb = np.stack([xa, np.cross(nz, xa), nz], axis=1)
        fp = np.concatenate([_quat_from_rot(Rb), center_c])
        n = Rb[:, 2]
        d = -n @ center_c
        ang = rng.uniform(-0.25, 0.25, beams) + az
        el = np.zeros(beams) if planar else rng.uniform(-0.3, 0.3, beams)
        u = np.stack([np.cos(ang) * np.cos(el), np.sin(ang) * np.cos(el), np.sin(el)], axis=1)
        den = (u @ R.T) @ n
        r_true = -(n @ t + d) / den
        ok = (r_true > 0.2) & (r_true < 3 * ranges[1])
        if ok.sum() < 5:
            continue
        r_rep = (r_true[ok] - b) / (1.0 + s) + sigma * rng.standard_normal(int(ok.sum()))
        p = u[ok] * r_rep[:, None]
        if planar:
            p[:, 2] = 0.0
        frame_pose.append(fp)
        pts.append(p)
        off.append(off[-1] + len(p))
    sc = Scene()
    sc.frame_pose = np.array(frame_pose)
    sc.offsets = np.array(off, dtype=np.int64)
    sc.points = np.concatenate(pts)
    sc.planes = np.asarray(X.frame_planes(sc.frame_pose), dtype=np.float64)
    sc.pose7, sc.b, sc.s = x, b, s
    return sc
