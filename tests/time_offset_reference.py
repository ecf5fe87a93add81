"""References of the time-offset calls (clc_*_time_offset).  TEST INFRASTRUCTURE ONLY.

* TdHarness: ctypes view of tests/time_offset_harness.cpp (the product's CLC_HD trajectory, expansion and 7-column LM code,
  compiled with g++);
* a long-double restatement of the trajectory (knots, shortest-arc slerp / lerp, clamping) and of the plane's td-derivative;
* td_sums: the 36 sums by direct per-residual accumulation of the 7-column Jacobian in long double, with magnitudes A_k in the
  sense of tests/exact_sums.py, extended to the td row and column;
* evaluate7 / solve7: an independent numpy restatement of the solve through oracle_np.trust_region_lm (7 columns, Plus =
  pose_plus on the pose and + on td, the 8-vector gradient norm and tolerances);
* scene: a recording whose camera trajectory IS the piecewise slerp / lerp of its knots, scans at another rate, a true offset, and
  laser points from the board at each scan's true time.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import exact_sums as X
import loss_reference as LR
from oracle import oracle_np as ONP

LD = X.LD
IU7 = np.triu_indices(7)
GROUPS_TD = {"H": list(range(28)), "g": list(range(28, 35)), "cost": [35]}
# the generator's extrinsic (reference main/calibr_simulation.cpp:15-20): T_lc, and T_cl as the solver's pose7
R_LC = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])
T_LC = np.array([0.1, 0.2, 0.3])


class TdHarness:
    def __init__(self, out_dir):
        here = os.path.dirname(os.path.abspath(__file__))
        out = os.path.join(str(out_dir), "libtime_offset_harness.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", out,
                               os.path.join(here, "time_offset_harness.cpp")])
        from camlasercalibratool_b200._lib import LmIteration, LmOptions

        L = C.CDLL(out)
        dp = C.POINTER(C.c_double)
        L.td_prepare.argtypes = [C.c_int64, dp, dp, dp]
        L.td_planes.argtypes = [C.c_int64, dp, dp, dp, C.c_int64, dp, dp, dp]
        L.td_expand.argtypes = [dp, dp, dp, C.c_double, dp, C.c_int, C.c_double, C.c_double, dp]
        L.td_lm_init.argtypes = [C.c_void_p, dp, C.c_double, C.POINTER(LmOptions)]
        L.td_lm_update.argtypes = [C.c_void_p, dp]
        for f in ("td_lm_done", "td_lm_ntrace", "td_lm_sweeps"):
            getattr(L, f).argtypes = [C.c_void_p]
        L.td_lm_cand.argtypes = [C.c_void_p, dp]
        L.td_lm_x.argtypes = [C.c_void_p, dp]
        L.td_lm_trace.argtypes = [C.c_void_p, C.c_int, C.POINTER(LmIteration)]
        self.L, self.LmIteration, self.LmOptions = L, LmIteration, LmOptions

    @staticmethod
    def dp(a):
        return a.ctypes.data_as(C.POINTER(C.c_double))

    def planes(self, knot_times, knot_poses, tau):
        """(planes [n, 4], dplanes [n, 4]) of the product's code at tau (relative to the first knot)."""
        K = len(knot_times)
        kp = np.ascontiguousarray(knot_poses, dtype=np.float64)
        knots, om = np.empty((K, 7)), np.empty((max(K - 1, 1), 3))
        self.L.td_prepare(K, self.dp(kp), self.dp(knots), self.dp(om))
        t = np.ascontiguousarray(np.asarray(knot_times, dtype=np.float64) - knot_times[0])
        tau = np.ascontiguousarray(tau, dtype=np.float64)
        P, D = np.empty((len(tau), 4)), np.empty((len(tau), 4))
        self.L.td_planes(K, self.dp(t), self.dp(knots), self.dp(om), len(tau), self.dp(tau), self.dp(P), self.dp(D))
        return P, D

    def expand(self, plane, dplane, pose7, count, S10, kind, cost_term, a):
        out = np.zeros(36)
        args = [np.ascontiguousarray(v, dtype=np.float64) for v in (plane, dplane, pose7, S10)]
        self.L.td_expand(self.dp(args[0]), self.dp(args[1]), self.dp(args[2]), float(count), self.dp(args[3]),
                         LR.KINDS.index(kind), float(cost_term), float(a), self.dp(out))
        return out

    def default_options(self, **kw):
        o = self.LmOptions(100, 1e4, 1e16, 1e-32, 1e-3, 1e-6, 1e32, 1e-6, 1e-10, 1e-8, 5, 1, 8, 0)
        for k, v in kw.items():
            setattr(o, k, v)
        return o

    def lm_run(self, sums_fn, pose7, td, options, max_sweeps=300):
        """lm_update_td driven as the device loop drives it: sums_fn(x8) -> the 36 sums at x8 = (pose7, td)."""
        st = C.create_string_buffer(self.L.td_lm_state_size())
        x0 = np.ascontiguousarray(pose7, dtype=np.float64)
        self.L.td_lm_init(st, self.dp(x0), float(td), C.byref(options))
        cand, n = np.empty(8), 0
        while not self.L.td_lm_done(st) and n < max_sweeps:
            self.L.td_lm_cand(st, self.dp(cand))
            sums = np.ascontiguousarray(sums_fn(cand.copy()), dtype=np.float64)
            self.L.td_lm_update(st, self.dp(sums))
            n += 1
        x = np.empty(8)
        self.L.td_lm_x(st, self.dp(x))
        trace = []
        for i in range(min(self.L.td_lm_ntrace(st), 256)):
            it = self.LmIteration()
            self.L.td_lm_trace(st, i, C.byref(it))
            trace.append(it)
        return x, self.L.td_lm_done(st), trace


# ---- the trajectory in long double -----------------------------------------------------------------------------------------
def _qmul(a, b):
    return np.stack([a[..., 3] * b[..., 0] + a[..., 0] * b[..., 3] + a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                     a[..., 3] * b[..., 1] + a[..., 1] * b[..., 3] + a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 3] * b[..., 2] + a[..., 2] * b[..., 3] + a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0],
                     a[..., 3] * b[..., 3] - a[..., 0] * b[..., 0] - a[..., 1] * b[..., 1] - a[..., 2] * b[..., 2]], axis=-1)


def knots_ld(knot_poses):
    """(q_ac [K, 4], t_ac [K, 3]) of T_ac = T_ca^-1 with the normalised quaternion, long double."""
    fp = np.asarray(knot_poses, dtype=np.float64).reshape(-1, 7).astype(LD)
    q = fp[:, :4] / X._norm(fp[:, :4])[:, None]
    R = X._rot(q)
    t_ac = -np.einsum("kji,kj->ki", R, fp[:, 4:])
    return np.concatenate([-q[:, :3], q[:, 3:]], axis=1), t_ac


def omegas_ld(q_ac):
    """w_k = Log(q_k^-1 (x) q_k+1) on the shortest arc, [K - 1, 3]."""
    conj = np.concatenate([-q_ac[:-1, :3], q_ac[:-1, 3:]], axis=1)
    r = _qmul(conj, q_ac[1:])
    r = np.where(r[:, 3:] < 0, -r, r)
    s = X._norm(r[:, :3])
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.where(s > 0, 2 * np.arctan2(s, r[:, 3]) / np.where(s > 0, s, 1), 2 / r[:, 3])
    return r[:, :3] * a[:, None]


def planes_ld(knot_times, knot_poses, tau):
    """(planes [n, 4], dplanes [n, 4]) in long double at tau (float64, relative to the first knot): the model of the header."""
    t = (np.asarray(knot_times, dtype=np.float64) - knot_times[0]).astype(LD)
    K = len(t)
    q_ac, t_ac = knots_ld(knot_poses)
    om = omegas_ld(q_ac)
    tau = np.asarray(tau, dtype=np.float64)
    taul = tau.astype(LD)
    before, after = taul < t[0], taul > t[-1]
    k = np.clip(np.searchsorted(t, taul, side="right") - 1, 0, K - 2)
    dt = t[k + 1] - t[k]
    u = (taul - t[k]) / dt
    v = u[:, None] * om[k]
    th = X._norm(v)
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.where(th > 0, np.sin(th / 2) / np.where(th > 0, th, 1), LD(0.5))
    e = np.concatenate([v * a[:, None], np.cos(th / 2)[:, None]], axis=1)
    q = _qmul(q_ac[k], e)
    tz = (1 - u) * t_ac[k, 2] + u * t_ac[k + 1, 2]
    dn = X._cross(X._rot(q)[:, 2, :], om[k]) / dt[:, None]
    dd = (t_ac[k + 1, 2] - t_ac[k, 2]) / dt
    clamp = before | after
    kc = np.where(before, 0, K - 1)
    q = np.where(clamp[:, None], q_ac[kc], q)
    tz = np.where(clamp, t_ac[kc, 2], tz)
    n = X._rot(q)[:, 2, :]
    dn = np.where(clamp[:, None], LD(0), dn)
    dd = np.where(clamp, LD(0), dd)
    return np.concatenate([n, tz[:, None]], axis=1), np.concatenate([dn, dd[:, None]], axis=1)


# ---- the 36 sums ----------------------------------------------------------------------------------------------------------
def pack_td(cost, H, g):
    return np.concatenate([np.asarray(H, dtype=np.float64)[IU7], np.asarray(g, dtype=np.float64), [float(cost)]])


def td_sums(planes, dplanes, offsets, points, pose7, td_unused, kind, a_loss=0.05):
    """The 36 sums (28 upper-tri H over tx ty tz rx ry rz td, 7 g, cost) at pose7 with the frames' planes and derivatives
    [N, 4] (long double), by direct accumulation of every residual's 7-column Jacobian in long double, and their magnitudes A_k.
    A_k extends exact_sums' to the td column (|J_td| <= L_td = |mdot||p| + |dn||t| + |dd|) and carries the rounding of the
    planes, which the device computes from the trajectory: each |J_i| is taken as |J_i| + its scale (1 for the translation
    columns, |p||m| for the rotation ones, L_td)."""
    offsets = np.asarray(offsets, dtype=np.int64)
    counts = np.diff(offsets)
    f_all = np.repeat(np.arange(len(counts)), counts)
    live = counts > 0
    s2f = np.zeros(len(counts), dtype=LD)
    s2f[live] = LD(1) / counts[live].astype(LD)
    planes, dplanes = np.asarray(planes, dtype=LD), np.asarray(dplanes, dtype=LD)
    val, mag = np.zeros(36, dtype=LD), np.zeros(36)
    for a in range(0, len(f_all), X.CHUNK):
        f_of = f_all[a:a + X.CHUNK]
        v, m_ = _td_block(planes[f_of], dplanes[f_of], s2f[f_of], np.asarray(points[a:a + X.CHUNK], dtype=np.float64), pose7,
                          kind, a_loss)
        val += v
        mag += m_
    return val, mag


def _td_block(pl, dpl, s2, points, pose7, kind, a):
    pose = np.asarray(pose7, dtype=np.float64).astype(LD)
    R, t = X._rot(pose[3:7]), pose[:3]
    p = points.astype(LD)
    n, d, dn, dd = pl[:, :3], pl[:, 3], dpl[:, :3], dpl[:, 3]
    m, md = n @ R, dn @ R
    c, cd = n @ t + d, dn @ t + dd
    e = np.sum(m * p, axis=-1) + c
    jtd = np.sum(md * p, axis=-1) + cd
    J = np.concatenate([n, X._cross(p, m), jtd[:, None]], axis=1)
    L_e = X._norm(m) * X._norm(p) + X._norm(n) * X._norm(t) + np.abs(d)
    L_td = X._norm(md) * X._norm(p) + X._norm(dn) * X._norm(t) + np.abs(dd)
    pm = X._norm(p) * X._norm(m)
    Jabs = np.concatenate([np.abs(n) + 1, np.repeat((2 * pm)[:, None], 3, axis=1), (2 * L_td)[:, None]], axis=1)
    w, rho, dw = LR.weight_and_cost(kind, e, a)
    sw = s2 * w
    val = np.zeros(36, dtype=LD)
    val[:28] = ((J * sw[:, None]).T @ J)[IU7]
    val[28:35] = (J * (sw * e)[:, None]).sum(axis=0)
    val[35] = (LD(0.5) * s2 * rho).sum()
    Jf = Jabs.astype(np.float64)
    mag = np.zeros(36)
    mag[:28] = ((Jf * (s2 * (w + dw * L_e)).astype(np.float64)[:, None]).T @ Jf)[IU7]
    mag[28:35] = (Jf * (sw * L_e).astype(np.float64)[:, None]).sum(axis=0)
    cost_mag = LD(0.5) * s2 * np.abs(rho) + s2 * w * np.abs(e) * L_e
    if kind == "cauchy":
        cost_mag = cost_mag + LD(0.5) * s2 * LD(a) ** 2 * LD(X.U_PROD)
    mag[35] = float(cost_mag.sum())
    return val, mag


# ---- the numpy restatement of the solve -------------------------------------------------------------------------------------
def evaluate7(scene, x8, kind, a=0.05):
    """(cost, corrected residuals [P], corrected Jacobian [P, 7]) at x8 = (pose7, td), float64 (the Corrector's simple branch)."""
    tau = scene.s_rel + x8[7]
    P, D = planes_ld(scene.knot_times, scene.knot_poses, tau)
    P, D = P.astype(np.float64), D.astype(np.float64)
    counts = np.diff(scene.offsets)
    f_of = np.repeat(np.arange(len(counts)), counts)
    s = 1.0 / np.sqrt(counts[f_of].astype(np.float64))
    R, t = ONP.quat_to_rot(x8[3:7]), x8[:3]
    n, d, dn, dd = P[f_of, :3], P[f_of, 3], D[f_of, :3], D[f_of, 3]
    m, md = n @ R, dn @ R
    pts = scene.points
    e = np.sum(m * pts, axis=1) + n @ t + d
    r = s * e
    J = s[:, None] * np.concatenate([n, np.cross(pts, m), (np.sum(md * pts, axis=1) + dn @ t + dd)[:, None]], axis=1)
    rho = LR.ceres_rho(kind, r * r, a * s)
    if kind == "huber":
        inl = np.abs(e) <= a
        rho = (np.where(inl, r * r, rho[0]), np.where(inl, 1.0, rho[1]), np.where(inl, 0.0, rho[2]))
    sq = np.sqrt(rho[1])
    return 0.5 * float(np.sum(rho[0])), r * sq, J * sq[:, None]


def solve7(scene, pose7, td, kind, a=0.05, fixed_mask=0, max_num_iterations=100):
    """Ceres' LM on the pose (PoseLocalParameterization) and td, through oracle_np.trust_region_lm: the held coordinates of
    fixed_mask (bits 0-5 the pose's tangent coordinates, bit 6 td) are dropped from the Jacobian and embedded as zeros.
    Returns (x8, termination name, trace dicts)."""
    free = [k for k in range(7) if not (fixed_mask >> k) & 1]

    def embed(v):
        full = np.zeros(7)
        full[free] = v
        return full

    def ev(x):
        cost, r, J = evaluate7(scene, x, kind, a)
        return cost, r, J[:, free]

    def plus(x, dv):
        dfull = embed(dv)
        out = np.concatenate([ONP.pose_plus(x[:7], dfull[:6]), [x[7] + dfull[6]]])
        if fixed_mask >> 6 & 1:
            out[7] = x[7]
        for k in range(3):
            if fixed_mask >> k & 1:
                out[k] = x[k]
        return out

    def gnorm(x, gv):
        g = embed(gv)
        return max(ONP.gradient_max_norm(x[:7], g[:6]), abs(g[6]))

    x0 = np.concatenate([np.asarray(pose7, dtype=np.float64), [float(td)]])
    return ONP.trust_region_lm(ev, plus, x0, max_num_iterations, gnorm)


def sums_at(scene, x8, kind, a=0.05):
    """The 36 sums at x8 from the long-double reference, rounded to float64 (what the LM harness is fed)."""
    P, D = planes_ld(scene.knot_times, scene.knot_poses, scene.s_rel + x8[7])
    val, _ = td_sums(P, D, scene.offsets, scene.points, x8[:7], None, kind, a)
    return val.astype(np.float64)


# ---- scenes ---------------------------------------------------------------------------------------------------------------
def _rot_to_quat(R):
    w = np.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    if w > 1e-3:
        return np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])
    raise ValueError("rotation too close to pi for this helper")


def truth_pose7():
    """T_cl of the generator as the solver's pose7 (tx ty tz qx qy qz qw)."""
    R_cl = R_LC.T
    return np.concatenate([-R_cl @ T_LC, _rot_to_quat(R_cl)])


class Scene:
    pass


def scene(n_knots=40, knot_rate=30.0, scan_rate=40.0, n_frames=None, beams=80, td_true=0.012, sigma=0.0, seed=0,
          epoch=1.7e9, static=False, outside=0, motion=1.0):
    """A recording (beams: points per scan, or one count per scan): knots of T_ca at knot_rate (times from `epoch`), a board whose motion IS the slerp / lerp of the knots;
    scans at scan_rate with jittered stamps on the laser clock, each scan's points taken from the board at its true camera time
    s_f + td_true (range noise sigma along the ray).  outside: that many scans at each end whose true time lies outside the knot
    span (clamped).  static: every knot equal.  frame_pose: the nearest knot's pose (the matching of
    formats.observations_from_segments), offsets / points of the laser."""
    rng = np.random.default_rng(seed)
    kt = epoch + np.arange(n_knots) / knot_rate + rng.uniform(-1e-3, 1e-3, n_knots) * (np.arange(n_knots) > 0)
    ph = rng.uniform(0, 2 * np.pi, 6)
    tt = np.arange(n_knots) / knot_rate
    kp = np.empty((n_knots, 7))
    for k in range(n_knots):
        tk = 0.0 if static else tt[k]
        yaw, pitch, roll = (motion * 0.35 * np.sin(2.1 * tk + ph[0]), motion * 0.3 * np.sin(1.7 * tk + ph[1]),
                            motion * 0.25 * np.sin(2.9 * tk + ph[2]))
        cz, sz, cy, sy, cx, sx = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
        R = np.array([[cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx],
                      [sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx],
                      [-sy, cy * sx, cy * cx]])
        kp[k, :4] = _rot_to_quat(R)
        kp[k, 4:] = [motion * 0.3 * np.sin(1.3 * tk + ph[3]), motion * 0.2 * np.sin(1.1 * tk + ph[4]),
                     2.0 + motion * 0.4 * np.sin(0.9 * tk + ph[5])]
    span = tt[-1]
    if n_frames is None:
        n_frames = int((span - 0.05) * scan_rate)
    s_true_rel = 0.02 + np.arange(n_frames) / scan_rate + rng.uniform(-3e-3, 3e-3, n_frames)
    if outside:
        s_true_rel[:outside] = -0.01 - 0.02 * np.arange(outside)[::-1]
        s_true_rel[-outside:] = span + 0.01 + 0.02 * np.arange(outside)
    s_rel = s_true_rel - td_true          # laser stamps, relative to the first knot
    frame_times = kt[0] + s_rel           # absolute laser stamps
    s_rel = frame_times - kt[0]           # what the library computes (exact by Sterbenz)
    P, _ = planes_ld(kt, kp, s_rel + td_true)
    P = P.astype(np.float64)
    Rcl, tcl = R_LC.T, -R_LC.T @ T_LC
    pts, off = [], [0]
    counts = np.broadcast_to(np.asarray(beams, dtype=np.int64), (n_frames,))
    for f in range(n_frames):
        m = Rcl.T @ P[f, :3]
        c = P[f, :3] @ tcl + P[f, 3]
        th = np.linspace(-0.25, 0.25, counts[f])
        den = m[0] * np.cos(th) + m[1] * np.sin(th)
        r = -c / den + (sigma * rng.standard_normal(counts[f]) if sigma > 0 else 0.0)
        pts.append(np.stack([r * np.cos(th), r * np.sin(th), np.zeros(counts[f])], axis=1))
        off.append(off[-1] + counts[f])
    sc = Scene()
    sc.knot_times, sc.knot_poses, sc.frame_times, sc.s_rel = kt, kp, frame_times, s_rel
    sc.offsets, sc.points = np.array(off, dtype=np.int64), np.concatenate(pts)
    nearest = np.clip(np.searchsorted(kt, frame_times), 1, n_knots - 1)
    nearest = np.where(np.abs(kt[nearest - 1] - frame_times) <= np.abs(kt[nearest] - frame_times), nearest - 1, nearest)
    sc.frame_pose = kp[nearest].copy()
    sc.td_true = td_true
    return sc
