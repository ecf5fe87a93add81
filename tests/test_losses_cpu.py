"""CPU tests of the Huber and soft-L1 losses (clc_problem_set_loss), no GPU needed:

* the Ceres-shaped restatement of HuberLoss / SoftLOneLoss (tests/loss_reference.py) against closed forms at the points where a
  loss changes behaviour, and the library's |e| == a Huber boundary;
* the product's per-residual and expansion code (csrc/clc_expand.cuh, compiled with g++ by tests/loss_harness.cpp) against
  the long-double reference, and the moment expansion against direct accumulation, for every kind;
* the product's LM state machine (csrc/clc_lm.cuh) fed by that per-residual code makes the decisions of the Ceres-shaped
  oracle, on clean data and on a scene with 5 % gross outliers;
* the third-party pin: scipy.optimize.least_squares(loss="huber" | "soft_l1") reaches the oracle's minimum;
* the C ABI and Python argument checks of set_loss.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import exact_sums as X
import loss_reference as LR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KIND = {"none": 0, "cauchy": 1, "huber": 2, "soft_l1": 3}
NEW = ("huber", "soft_l1")
A = 0.05
X0 = np.array([0, 0, 0, 0, 0, 0, 1.0])
TERM = {"CONVERGENCE_FUNCTION": 1, "CONVERGENCE_PARAMETER": 2, "CONVERGENCE_GRADIENT": 3, "CONVERGENCE_MIN_RADIUS": 4,
        "NO_CONVERGENCE": 5, "FAILURE": 6}


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    from camlasercalibratool_b200._lib import LmIteration

    out = str(tmp_path_factory.mktemp("loss_harness") / "libloss_harness.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "loss_harness.cpp")])
    L = C.CDLL(out)
    dp = C.POINTER(C.c_double)
    L.loss_weight.argtypes = [C.c_int, C.c_double, C.c_double, dp, dp]
    L.loss_accumulate_residual.argtypes = [dp, dp, dp, C.c_double, C.c_int, C.c_double, dp]
    L.loss_accumulate_all.argtypes = [dp, dp, dp, dp, C.c_int64, C.c_int, C.c_double, dp]
    L.loss_edge_residual.argtypes = [dp, dp, dp, C.c_double, C.c_int, C.c_double, dp]
    L.loss_edge_residual.restype = C.c_double
    L.loss_expand_lm.argtypes = [dp, dp, C.c_double, dp, C.c_int, C.c_double, C.c_double, dp]
    L.loss_lm_init.argtypes = [C.c_void_p, dp, C.c_void_p]
    L.loss_lm_update.argtypes = [C.c_void_p, dp]
    L.loss_lm_done.argtypes = [C.c_void_p]
    L.loss_lm_ntrace.argtypes = [C.c_void_p]
    L.loss_lm_cand.argtypes = [C.c_void_p, dp]
    L.loss_lm_x.argtypes = [C.c_void_p, dp]
    L.loss_lm_trace.argtypes = [C.c_void_p, C.c_int, C.POINTER(LmIteration)]
    L.LmIteration = LmIteration
    return L


@pytest.fixture(scope="module")
def CO(tmp_path_factory):
    return LR.COracle(tmp_path_factory.mktemp("loss_oracle"))


def host_weight(H, kind, e, a=A):
    w, t = C.c_double(), C.c_double()
    H.loss_weight(KIND[kind], float(e), a, C.byref(w), C.byref(t))
    return w.value, t.value


# ---- the losses themselves ---------------------------------------------------------------------------------------------
def closed_form(kind, s, a):
    """rho, rho', rho'' of HuberLoss / SoftLOneLoss(a) at s = r^2 (float64 closed forms)."""
    b = a * a
    if kind == "huber":
        if s <= b:
            return s, 1.0, 0.0
        r = np.sqrt(s)
        return 2 * a * r - b, a / r, -a / (2 * s * r)
    u = 1 + s / b
    return 2 * s / (1 + np.sqrt(u)), 1 / np.sqrt(u), -1 / (2 * b * u ** 1.5)


@pytest.mark.parametrize("kind", NEW)
@pytest.mark.parametrize("z", [0.0, 1e-8, 1 - 2 ** -40, 1.0, 1 + 2 ** -40, 1e4])
def test_rho_known_answers(H, kind, z):
    a = 0.05 * 0.3  # a scaled parameter, as a frame of ~11 points sees it
    s = z * a * a
    got = LR.ceres_rho(kind, np.array([s]), a)
    want = closed_form(kind, s, a)
    # Ceres' soft-L1 rho = 2b (sqrt(1 + s/b) - 1) cancels for s << b: to 1e-7 relative at z = 1e-8, exact elsewhere
    tol0 = 2e-7 if (kind == "soft_l1" and 0 < z < 1e-6) else 1e-14
    np.testing.assert_allclose(got[0][0], want[0], rtol=tol0, atol=0)
    np.testing.assert_allclose(got[1][0], want[1], rtol=1e-14, atol=0)
    np.testing.assert_allclose(got[2][0], want[2], rtol=1e-13, atol=0)
    assert got[2][0] <= 0.0  # Ceres' Corrector takes its simple branch
    # the product's per-residual code, on the unscaled distance e (rho~ = rho(s)/scale^2 with s = (scale e)^2)
    e = np.sqrt(z) * A
    w, t = host_weight(H, kind, e)
    wl, rl, _ = LR.weight_and_cost(kind, np.array([e]), A)
    np.testing.assert_allclose(w, float(wl[0]), rtol=2e-16, atol=0)
    np.testing.assert_allclose(t, float(rl[0]), rtol=4e-16, atol=0)
    np.testing.assert_allclose(w, want[1], rtol=1e-14)


def test_huber_boundary_is_an_inlier(H):
    for e in (A, -A):
        w, t = host_weight(H, "huber", e)
        assert w == 1.0 and t == e * e
        wl, rl, _ = LR.weight_and_cost("huber", np.array([e]), A)
        assert wl[0] == 1 and rl[0] == np.longdouble(e) * np.longdouble(e)
    up = np.nextafter(A, 1.0)
    w, t = host_weight(H, "huber", up)
    assert w < 1.0 and w == A / up
    dn = np.nextafter(A, 0.0)
    assert host_weight(H, "huber", dn) == (1.0, dn * dn)
    # continuity: the two branches meet at |e| = a to rounding
    assert abs(host_weight(H, "huber", up)[1] - A * A) <= 4e-16 * A * A


# ---- the product's per-residual code against the long-double reference ---------------------------------------------------
def _residuals(oracle, seed, outliers=0.0):
    p = oracle.generate(12, 60, seed=seed, sigma=0.01, exact_m=False, with_edges=True)
    pts = p.points.copy()
    if outliers:
        rng = np.random.default_rng(seed)
        k = rng.choice(len(pts), size=max(1, int(outliers * len(pts))), replace=False)
        pts[k, :2] += rng.uniform(0.3, 1.0, size=(len(k), 2)) * rng.choice([-1, 1], size=(len(k), 2))
    return oracle.Problem(p.frame_pose, p.offsets, pts, p.edge_points)


@pytest.mark.parametrize("kind", KIND)
def test_host_residual_code_matches_reference(oracle, oracle_np, H, kind):
    p = _residuals(oracle, 3, outliers=0.1)
    pl, pts, s = oracle_np.residual_table(p.frame_pose, p.offsets, p.points, p.edge_points)
    counts = np.rint(1.0 / (s * s))
    pose = oracle.pose_plus(oracle.ground_truth()[1], 0.02 * np.array([1.0, -0.7, 0.4, -1.0, 0.6, 0.3]))
    ref = LR.lm_sums_of_blocks([(pl.astype(LR.LD), pts.astype(LR.LD), (1 / counts).astype(LR.LD))], pose, kind, A)
    # the one-cluster kernel's per-residual code
    acc = np.zeros(32)
    H.loss_accumulate_all(_dp(np.ascontiguousarray(pl)), _dp(pose), _dp(np.ascontiguousarray(pts)), _dp(counts), len(s), KIND[kind],
                          A, _dp(acc))
    X.assert_within(acc[:28], *ref, X.GROUPS_LM, f"accumulate_residual/{kind}")
    # the moment path of the edge residuals (edge_residual_at): every residual through it
    out = np.zeros(28)
    for r in range(len(s)):
        e = H.loss_edge_residual(_dp(np.ascontiguousarray(pl[r])), _dp(pose), _dp(np.ascontiguousarray(pts[r])), counts[r],
                                 KIND[kind], A, _dp(out))
        assert np.isfinite(e)
    X.assert_within(out, *ref, X.GROUPS_LM, f"edge_residual_at/{kind}")


@pytest.mark.parametrize("kind", KIND)
def test_moment_expansion_equals_direct_accumulation(oracle, oracle_np, H, kind):
    p = _residuals(oracle, 5, outliers=0.05)
    pose = oracle.pose_plus(oracle.ground_truth()[1], 0.01 * np.array([0.3, 1.0, -0.4, 0.2, -0.6, 0.9]))
    off = p.offsets
    for f in range(4):
        b, e = int(off[f]), int(off[f + 1])
        plane = oracle_np.frame_plane(p.frame_pose[f])
        P = p.points[b:e]
        direct = np.zeros(32)
        cnt = float(e - b)
        for j in range(e - b):
            H.loss_accumulate_residual(_dp(plane), _dp(pose), _dp(np.ascontiguousarray(P[j])), cnt, KIND[kind], A, _dp(direct))
        # moments with the kind's weights, as the sweep kernel streams them
        R = oracle_np.quat_to_rot(pose[3:7])
        ed = P @ (R.T @ plane[:3]) + (plane[:3] @ pose[:3] + plane[3])
        ws, ts = zip(*(host_weight(H, kind, v) for v in ed))
        w, t = np.array(ws), np.array(ts)
        S = np.array([w.sum(), *(w[:, None] * P).sum(0), *[(w * P[:, i] * P[:, j]).sum() for i, j in
                                                          ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))]])
        out = np.zeros(28)
        H.loss_expand_lm(_dp(plane), _dp(pose), cnt, _dp(S), KIND[kind], float(t.sum()), A, _dp(out))
        ref = LR.lm_sums(p.frame_pose[f:f + 1], np.array([0, e - b]), P, pose, kind, A)
        X.assert_within(direct[:28], *ref, X.GROUPS_LM, f"direct/{kind}")
        X.assert_within(out, *ref, X.GROUPS_LM, f"moments/{kind}")


# ---- the product's LM, fed by its per-residual code, against the Ceres-shaped oracle ---------------------------------------
def host_solve(H, table, pose7, kind, a=A, max_sweeps=400):
    from camlasercalibratool_b200._lib import LmOptions

    pl, pts, s = (np.ascontiguousarray(v) for v in table)
    counts = np.rint(1.0 / (s * s))
    st = C.create_string_buffer(H.loss_lm_state_size())
    opt = LmOptions(100, 1e4, 1e16, 1e-32, 1e-3, 1e-6, 1e32, 1e-6, 1e-10, 1e-8, 5, 1, 8, 0)
    x0 = np.ascontiguousarray(pose7, dtype=np.float64)
    H.loss_lm_init(st, _dp(x0), C.byref(opt))
    cand = np.empty(7)
    for _ in range(max_sweeps):
        if H.loss_lm_done(st):
            break
        H.loss_lm_cand(st, _dp(cand))
        acc = np.zeros(32)
        H.loss_accumulate_all(_dp(pl), _dp(cand), _dp(pts), _dp(counts), len(s), KIND[kind], a, _dp(acc))
        H.loss_lm_update(st, _dp(acc))
    x = np.empty(7)
    H.loss_lm_x(st, _dp(x))
    tr = []
    for i in range(H.loss_lm_ntrace(st)):
        it = H.LmIteration()
        H.loss_lm_trace(st, i, C.byref(it))
        tr.append(it)
    return x, H.loss_lm_done(st), tr


def config1(oracle, seed, scene):
    """Config 1 (50 x 180, sigma = 1 cm); "outliers": 5 % of the points moved 0.3-1 m off their board."""
    p = oracle.generate(50, 180, seed=seed, sigma=0.01)
    if scene == "outliers":
        rng = np.random.default_rng(100 + seed)
        pts = p.points.copy()
        k = rng.choice(len(pts), size=len(pts) // 20, replace=False)
        pts[k, :2] += rng.uniform(0.3, 1.0, size=(len(k), 2)) * rng.choice([-1, 1], size=(len(k), 2))
        p = oracle.Problem(p.frame_pose, p.offsets, pts)
    return p


def STARTS(oracle):
    """The identity and a perturbed truth."""
    return (X0, oracle.pose_plus(oracle.ground_truth()[1], 0.05 * np.array([1.0, -0.5, 0.3, 0.2, -0.4, 0.6])))


@pytest.mark.parametrize("scene", ["clean", "outliers"])
@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("kind", NEW)
def test_c_oracle_equals_numpy_twin(oracle, oracle_np, CO, kind, seed, scene):
    """tests/loss_oracle.c against its numpy twin (loss_reference.evaluate / solve): eval cost, H and g to ~1e-15, and full
    solves with the same accept/reject sequence and termination, poses within 1e-12."""
    p = config1(oracle, seed, scene)
    table = oracle_np.residual_table(p.frame_pose, p.offsets, p.points)
    for x in STARTS(oracle) + (oracle.ground_truth()[1],):
        c1, r1, J1 = CO.evaluate(p, x, kind, A)
        c2, r2, J2 = LR.evaluate(table, x, kind, A)
        H1, H2 = J1.T @ J1, J2.T @ J2
        assert abs(c1 - c2) <= 1e-15 * 8 * c2, (c1, c2)
        assert np.abs(H1 - H2).max() <= 1e-15 * 8 * np.abs(H2).max()
        assert np.abs(J1.T @ r1 - J2.T @ r2).max() <= 1e-15 * 8 * np.abs(H2).max()
    for x0 in STARTS(oracle):
        xo, so, tro = CO.solve(p, x0, kind, A)
        xn, term, trn = LR.solve(table, x0, kind, A)
        assert so.termination == TERM[term]
        # the numpy restatement does not record the iteration whose candidate terminates the solve
        assert so.num_iterations in (len(trn), len(trn) + 1)
        assert [bool(t.step_is_successful) for t in tro[:len(trn)]] == [bool(t["ok"]) for t in trn]
        np.testing.assert_allclose([t.cost for t in tro[:len(trn)]], [t["cost"] for t in trn], rtol=1e-12)
        ang, dt = oracle.pose_error(xo, xn)
        assert ang < 1e-12 and dt < 1e-12, (ang, dt)


def test_c_oracle_cauchy_is_the_oracle(oracle, CO):
    """With the Cauchy kind (and none) the loss oracle reproduces oracle/clc_oracle.c's own solve."""
    p = config1(oracle, 2, "outliers")
    for kind, use_loss in (("cauchy", True), ("none", False)):
        q = oracle.Problem(p.frame_pose, p.offsets, p.points, use_loss=use_loss)
        xo, so, tro = oracle.solve(q, X0)
        x, s, tr = CO.solve(p, X0, kind, 0.05)
        assert s.termination == so.termination and s.num_iterations == so.num_iterations
        assert [t.step_is_successful for t in tr] == [t.step_is_successful for t in tro]
        ang, dt = oracle.pose_error(x, xo)
        assert ang < 1e-12 and dt < 1e-12, (ang, dt)


@pytest.mark.parametrize("scene", ["clean", "outliers"])
@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("kind", NEW)
def test_host_lm_makes_the_oracle_decisions(oracle, oracle_np, H, CO, kind, seed, scene):
    p = config1(oracle, seed, scene)
    table = oracle_np.residual_table(p.frame_pose, p.offsets, p.points)
    for x0 in STARTS(oracle):
        xo, so, tro = CO.solve(p, x0, kind, A)
        x, done, tr = host_solve(H, table, x0, kind)
        assert done == so.termination and len(tr) == so.num_iterations, (so.termination, done)
        assert [(t.step_is_valid, t.step_is_successful) for t in tr] == [(t.step_is_valid, t.step_is_successful) for t in tro]
        np.testing.assert_allclose([t.cost for t in tr], [t.cost for t in tro], rtol=1e-9)
        ang, dt = oracle.pose_error(x, xo)
        assert ang < 1e-9 and dt < 1e-9, (ang, dt)


@pytest.mark.parametrize("kind", NEW)
def test_noise_free_host_solve_reaches_the_truth(oracle, oracle_np, H, kind):
    p = oracle.generate(50, 180, seed=1, sigma=0.0)
    x, done, _ = host_solve(H, oracle_np.residual_table(p.frame_pose, p.offsets, p.points), X0, kind)
    ang, dt = oracle.pose_error(x, oracle.ground_truth()[1])
    assert done in (1, 2, 3) and ang < 1e-9 and dt < 1e-9, (ang, dt)


# ---- third-party pin ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", NEW)
def test_scipy_least_squares_reaches_the_oracle_minimum(oracle, oracle_np, kind):
    """Exact-M frames share one scale s, so the library's cost is s^2 times scipy's 1/2 f_scale^2 sum rho(e^2 / f_scale^2) on
    the raw distances e: both minimise the same function of the pose."""
    least_squares = pytest.importorskip("scipy.optimize").least_squares
    from scipy.spatial.transform import Rotation

    p = oracle.generate(30, 120, seed=4, sigma=0.01, exact_m=True)
    rng = np.random.default_rng(9)
    pts = p.points.copy()
    k = rng.choice(len(pts), size=len(pts) // 20, replace=False)
    pts[k, :2] += rng.uniform(0.3, 1.0, size=(len(k), 2))
    table = oracle_np.residual_table(p.frame_pose, p.offsets, pts)
    s2 = float(table[2][0]) ** 2
    gt = oracle.ground_truth()[1]
    xo, term, _ = LR.solve(table, gt, kind, A)
    cost_ceres = LR.evaluate(table, xo, kind, A)[0]
    # Ceres stops at function_tolerance 1e-6; Gauss-Newton steps on the same corrected model converge it tightly
    for _ in range(40):
        _, r, J = LR.evaluate(table, xo, kind, A)
        xo = oracle_np.pose_plus(xo, -np.linalg.lstsq(J, r, rcond=None)[0])
    planes, P = table[0], table[1]

    def raw(v):
        R = Rotation.from_rotvec(v[3:]).as_matrix()
        return np.einsum("ij,ij->i", planes[:, :3], P @ R.T + v[:3]) + planes[:, 3]

    v0 = np.concatenate([gt[:3], Rotation.from_quat(gt[3:]).as_rotvec()])
    res = least_squares(raw, v0, loss=kind, f_scale=A, xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=2000)
    xs = np.concatenate([res.x[:3], Rotation.from_rotvec(res.x[3:]).as_quat()])
    ang, dt = oracle.pose_error(xs, xo)
    assert ang < 1e-8 and dt < 1e-8, (ang, dt)
    cost_o = LR.evaluate(table, xo, kind, A)[0]
    np.testing.assert_allclose(cost_o, s2 * res.cost, rtol=1e-12)
    assert 0.0 <= cost_ceres - cost_o <= 1e-6 * cost_o


# ---- ABI and argument checks ------------------------------------------------------------------------------------------
def test_set_loss_rejects_bad_arguments_before_device_work():
    from camlasercalibratool_b200 import Group, Problem, _lib

    L = _lib.load()
    k, a = C.c_int(), C.c_double()
    assert L.clc_problem_set_loss(None, 2, 0.05) == 1  # CLC_ERR_INVALID
    assert L.clc_problem_get_loss(None, C.byref(k), C.byref(a)) == 1
    assert L.clc_group_set_loss(None, 2, 0.05) == 1
    # the library checks kind and a before it touches the handle: a dangling one is never dereferenced
    dangling = C.c_void_p(16)
    for kind, bad_a in ((4, 0.05), (-1, 0.05), (2, 0.0), (2, -0.05), (3, float("nan")), (1, float("inf")), (2, 1e-160),
                        (3, 1e160)):
        assert L.clc_problem_set_loss(dangling, kind, bad_a) == 1, (kind, bad_a)
        assert L.clc_group_set_loss(dangling, kind, bad_a) == 1, (kind, bad_a)
    fake = Problem.__new__(Problem)
    fake._h, fake._L, fake._comm = None, L, None
    grp = Group.__new__(Group)
    grp._h, grp._L = None, L
    for obj in (fake, grp):
        for bad in (("tukey", 0.05), (4, 0.05), ("Huber", 0.05), ("huber", 0.0), ("huber", -1.0), ("soft_l1", float("nan")),
                    ("cauchy", float("inf")), ("huber", 1e-160), ("soft_l1", 1e160), (None, -0.0)):
            with pytest.raises(ValueError):
                obj.set_loss(*bad)
    fake._h = grp._h = None  # nothing to close
