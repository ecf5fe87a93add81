"""The camera-laser time offset (clc_problem_set_trajectory, clc_eval_time_offset, clc_information_time_offset,
clc_solve_lm_time_offset) on the GPU, on both kernel families, with and without a loss.  Scenes come from
time_offset_reference.scene: a board whose motion IS the slerp / lerp of its knots, scans at another rate with a true offset,
laser points from the board at each scan's true time.
"""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

import exact_sums as X
import time_offset_reference as TR

pytestmark = pytest.mark.gpu

FAMILIES = {"general": dict(CLC_PLANAR="0"), "planar": dict(CLC_PLANAR="1", CLC_PLANAR_MIN_POINTS="0")}
LOSSES = ("none", "cauchy")
TERM = {1: "CONVERGENCE_FUNCTION", 2: "CONVERGENCE_PARAMETER", 3: "CONVERGENCE_GRADIENT", 4: "CONVERGENCE_MIN_RADIUS",
        5: "NO_CONVERGENCE", 6: "FAILURE"}
ALL6 = ("tx", "ty", "tz", "rx", "ry", "rz")


@contextlib.contextmanager
def env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def problem(sc, family, kind, trajectory=True):
    from camlasercalibratool_b200 import Problem

    with env(**FAMILIES[family]):
        p = Problem.from_arrays(sc.frame_pose, sc.offsets, sc.points, use_loss=kind == "cauchy")
    assert p.planar == (family == "planar")
    p.set_loss(kind)
    if trajectory:
        p.set_trajectory(sc.knot_times, sc.knot_poses, sc.frame_times)
    return p


def tight(**kw):
    from camlasercalibratool_b200 import default_options

    return default_options(function_tolerance=1e-20, parameter_tolerance=1e-15, gradient_tolerance=1e-20, **kw)


def x8_near_truth(seed, td, scale=0.01):
    from oracle import oracle_np as ONP

    rng = np.random.default_rng(seed)
    return ONP.pose_plus(TR.truth_pose7(), scale * rng.standard_normal(6)), td + 0.003 * rng.standard_normal()


def ragged_scene(n_frames, seed, big=20000):
    rng = np.random.default_rng(seed)
    counts = rng.choice([0, 1, 3, 40, 700, 3000, big], size=n_frames, p=[0.06, 0.08, 0.1, 0.3, 0.3, 0.1, 0.06])
    return TR.scene(n_knots=int(n_frames * 0.8) + 4, n_frames=n_frames, beams=counts, seed=seed, sigma=0.003, outside=2)


def check_sums(p, sc, x, td, kind, what):
    cost, H, g = p.eval_time_offset(x, td)
    P, D = TR.planes_ld(sc.knot_times, sc.knot_poses, sc.s_rel + td)
    val, mag = TR.td_sums(P, D, sc.offsets, sc.points, x, td, kind)
    X.assert_within(TR.pack_td(cost, H, g), val, mag, TR.GROUPS_TD, f"{what}/eval")
    Hi, b, chi, sv = p.information_time_offset(x, td)
    val, mag = TR.td_sums(P, D, sc.offsets, sc.points, x, td, "none")
    X.assert_within(TR.pack_td(chi / 2, Hi, -b), val, mag, TR.GROUPS_TD, f"{what}/information")
    return cost, H, g


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("kind", LOSSES)
def test_sums_against_long_double(family, kind):
    """Every one of the 36 sums within GAMMA * A_k, on ragged layouts (empty, one-point and multi-warp frames, frames clamped at
    both ends of the trajectory); two calls return identical bytes."""
    sc = ragged_scene(700, seed=4)
    with problem(sc, family, kind) as p:
        part = p.partition(warp_table=False)
        assert part["grid"] > 1 and part["per_warp"] < 20000  # frames cross warp ranges
        for i in range(3):
            x, td = x8_near_truth(i, 0.012)
            cost, H, g = check_sums(p, sc, x, td, kind, f"{family}/{kind}/{i}")
            c2, H2, g2 = p.eval_time_offset(x, td)
            assert c2 == cost and H2.tobytes() == H.tobytes() and g2.tobytes() == g.tobytes()


@pytest.mark.parametrize("family", list(FAMILIES))
def test_sums_at_ten_million_points(family):
    sc = TR.scene(n_knots=760, n_frames=1000, beams=10000, seed=8, sigma=0.005, outside=3)
    assert len(sc.points) >= 10**7
    with problem(sc, family, "cauchy") as p:
        x, td = x8_near_truth(5, 0.012)
        check_sums(p, sc, x, td, "cauchy", f"{family}/1e7")


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("kind", LOSSES)
def test_consistency_with_the_existing_solve(oracle, family, kind):
    """Knots equal to each frame's own pose and scan times on the knots: with td = 0 the 6x6 block, g[0..5] and the cost are
    clc_eval's on the frame_pose problem, and the solve with td held makes clc_solve_lm's decisions and reaches its pose."""
    from camlasercalibratool_b200 import Problem

    d = oracle.generate(60, 400, seed=7, sigma=0.01)
    kt = 1.7e9 + 0.05 * np.arange(60)
    with env(**FAMILIES[family]):
        p = Problem.from_arrays(d.frame_pose, d.offsets, d.points, use_loss=kind == "cauchy")
    with p:
        p.set_loss(kind)
        p.set_trajectory(kt, d.frame_pose, kt)
        rng = np.random.default_rng(1)
        x = oracle.pose_plus(oracle.ground_truth()[1], 0.02 * rng.standard_normal(6))
        cost, H, g = p.eval_time_offset(x, 0.0)
        c6, H6, g6 = p.eval(x)
        assert abs(cost - c6) <= 1e-12 * c6
        assert np.abs(H[:6, :6] - H6).max() <= 1e-12 * np.abs(H6).max()
        assert np.abs(g[:6] - g6).max() <= 1e-12 * np.abs(H6).max()
        x0 = np.array([0, 0, 0, 0, 0, 0, 1.0])
        xs, s6, tr6 = p.solve(x0)
        xt, td, st, trt = p.solve_time_offset(x0, 0.0, fixed="td")
        assert td == 0.0 and TERM[st.termination] == TERM[s6.termination]
        assert [(t.step_is_valid, t.step_is_successful) for t in trt] == [(t.step_is_valid, t.step_is_successful) for t in tr6]
        assert np.abs(xt - xs).max() < 1e-9, xt - xs


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("kind", LOSSES)
def test_recovery(family, kind):
    """Noise-free: from the nearest-pose closed form and td = 0 the solve recovers td* and T_cl; the plain solve on the same
    nearest-pose frames is biased.  With 5 mm range noise the solve makes the numpy restatement's decisions and reaches its x8."""
    from camlasercalibratool_b200 import T_to_pose7

    sc = TR.scene(n_knots=60, beams=120, seed=12, td_true=0.012, motion=2.0)
    gt = TR.truth_pose7()
    with problem(sc, family, kind) as p:
        x0 = T_to_pose7(np.linalg.inv(p.closed_form()[0]))
        xb, sb, _ = p.solve(x0, tight())
        x, td, s, _ = p.solve_time_offset(x0, 0.0, tight())
        assert TERM[s.termination] != "FAILURE"
        assert abs(td - sc.td_true) < 1e-9, td - sc.td_true
        from oracle import oracle_np as ONP

        def off(y):
            return max(np.abs(y[:3] - gt[:3]).max(), np.abs(ONP.quat_to_rot(y[3:]) - ONP.quat_to_rot(gt[3:])).max())

        bias, err = off(xb), off(x)
        print(f"{family}/{kind}: nearest-pose solve off by {bias:.3e}, time-offset solve off by {err:.3e} and td by "
              f"{abs(td - sc.td_true):.3e} s")
        # Under the Cauchy loss the cost is a^2 log of a running product: near a zero-residual optimum its changes fall below the
        # product's resolution and the function tolerance stops the solve within about 1e-8 of the truth (as for every solve of
        # the library: tests/test_fixed_cpu.py); without a loss the truth is reached to 1e-9
        assert err < (1e-9 if kind == "none" else 2e-8), err
        assert bias > 1e-4
    noisy = TR.scene(n_knots=40, beams=60, seed=13, td_true=0.012, sigma=0.005, motion=2.0)
    with problem(noisy, family, kind) as p:
        x0 = T_to_pose7(np.linalg.inv(p.closed_form()[0]))
        x, td, s, tr = p.solve_time_offset(x0, 0.0)
        xn, term, trn = TR.solve7(noisy, x0, 0.0, kind)
        assert TERM[s.termination] == term
        assert [r["ok"] for r in trn] == [bool(t.step_is_successful) for t in tr[:len(trn)]]
        assert np.abs(np.concatenate([x, [td]]) - xn).max() < 1e-9


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("kind", LOSSES)
def test_static_board_leaves_td_unobservable(family, kind):
    sc = TR.scene(n_knots=30, beams=100, seed=14, static=True)
    with problem(sc, family, kind) as p:
        x0 = TR.truth_pose7()  # one plane leaves the extrinsic unobservable too: noise-free, from the truth
        H, b, chi, sv = p.information_time_offset(x0, 0.0)
        assert sv[-1] == 0.0 and sv[0] > 0
        assert abs(abs(p.last_V[6, 6]) - 1.0) < 1e-12
        start = np.nextafter(0.01, 1.0)
        x, td, s, _ = p.solve_time_offset(x0, start)
        assert np.float64(td).tobytes() == np.float64(start).tobytes()
        xs, s6, _ = p.solve(x0)
        assert np.abs(x - xs).max() < 1e-9


@pytest.mark.parametrize("family", list(FAMILIES))
def test_clamped_frames_say_nothing_about_td(family):
    sc = TR.scene(n_knots=40, beams=100, seed=15, outside=4, sigma=0.003, motion=2.0)
    tau_true = sc.s_rel + sc.td_true
    span = sc.knot_times[-1] - sc.knot_times[0]
    out = (tau_true < -0.005) | (tau_true > span + 0.005)
    assert out.sum() == 8
    with problem(sc, family, "cauchy") as p:
        with p.subset(out) as q:
            q.set_trajectory(sc.knot_times, sc.knot_poses, sc.frame_times[out])
            cost, H, g = q.eval_time_offset(TR.truth_pose7(), sc.td_true)
            assert not np.any(H[6]) and not np.any(H[:, 6]) and g[6] == 0.0 and cost > 0
        x, td, s, _ = p.solve_time_offset(TR.truth_pose7(), 0.0)
        assert TERM[s.termination] != "FAILURE" and abs(td - sc.td_true) < 1e-3


@pytest.mark.parametrize("family", list(FAMILIES))
def test_masks(family):
    from oracle import oracle_np as ONP

    sc = TR.scene(n_knots=40, beams=80, seed=16, td_true=0.012, motion=2.0)
    gt = TR.truth_pose7()
    x0 = ONP.pose_plus(gt, 0.02 * np.random.default_rng(3).standard_normal(6))
    with problem(sc, family, "none") as p:
        # td alone: the extrinsic known and held
        x, td, s, _ = p.solve_time_offset(gt, 0.0, tight(), fixed=ALL6)
        assert x[:3].tobytes() == gt[:3].tobytes() and np.abs(x - gt).max() < 1e-15 and abs(td - sc.td_true) < 1e-9
        # the extrinsic alone: td held at its start bits
        x, td, s, _ = p.solve_time_offset(x0, 0.004, fixed="td")
        assert td == 0.004 and TERM[s.termination] != "FAILURE"
        # mixed: a held translation keeps its bits, the rest recovers the truth
        x, td, s, _ = p.solve_time_offset(x0, 0.0, fixed=("tz", "ry"))
        assert x[2] == x0[2] and TERM[s.termination] != "FAILURE"
        for bad in (ALL6 + ("td",), ("yaw",)):
            with pytest.raises(ValueError):
                p.solve_time_offset(x0, 0.0, fixed=bad)


def test_rejections():
    from camlasercalibratool_b200 import Problem, _lib
    from camlasercalibratool_b200.api import default_options

    L = _lib.load()
    sc = TR.scene(n_knots=12, beams=50, seed=17)
    N = len(sc.offsets) - 1
    dp = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))  # noqa
    with Problem.from_arrays(sc.frame_pose, sc.offsets, sc.points) as p:
        h = p._h
        x = TR.truth_pose7()
        H, g, cost = np.empty(49), np.empty(7), C.c_double()
        td = C.c_double(0.0)
        # no trajectory yet
        assert L.clc_eval_time_offset(h, dp(x), 0.0, dp(H), dp(g), C.byref(cost)) == 4
        assert b"trajectory" in L.clc_last_error()
        assert L.clc_solve_lm_time_offset(h, dp(x), C.byref(td), None, None, None, 0) == 4

        kt, kp, ft = sc.knot_times, sc.knot_poses, sc.frame_times
        bad = []
        bad.append(("n_knots", lambda: L.clc_problem_set_trajectory(h, 1, dp(kt), dp(kp), dp(ft))))
        bad.append(("n_knots", lambda: L.clc_problem_set_trajectory(h, -2, dp(kt), dp(kp), dp(ft))))
        bad.append(("NULL", lambda: L.clc_problem_set_trajectory(h, len(kt), None, dp(kp), dp(ft))))
        bad.append(("NULL", lambda: L.clc_problem_set_trajectory(h, len(kt), dp(kt), dp(kp), None)))
        t2 = kt.copy(); t2[3] = t2[2]
        bad.append(("knot_times", lambda: L.clc_problem_set_trajectory(h, len(kt), dp(t2), dp(kp), dp(ft))))
        t3 = kt.copy(); t3[5] = np.nan
        bad.append(("knot_times", lambda: L.clc_problem_set_trajectory(h, len(kt), dp(t3), dp(kp), dp(ft))))
        q2 = kp.copy(); q2[4, 6] = np.inf
        bad.append(("knot_poses", lambda: L.clc_problem_set_trajectory(h, len(kt), dp(kt), dp(q2), dp(ft))))
        q3 = kp.copy(); q3[2, :4] = 0.0
        bad.append(("quaternion", lambda: L.clc_problem_set_trajectory(h, len(kt), dp(kt), dp(q3), dp(ft))))
        f2 = ft.copy(); f2[N // 2] = np.nan
        bad.append(("frame_times", lambda: L.clc_problem_set_trajectory(h, len(kt), dp(kt), dp(kp), dp(f2))))
        for word, call in bad:
            assert call() == 1, word
            assert word.encode() in L.clc_last_error(), (word, L.clc_last_error())
        assert L.clc_eval_time_offset(h, dp(x), 0.0, None, None, None) == 4  # still no trajectory: nothing changed

        p.set_trajectory(kt, kp, ft)
        ref = p.eval_time_offset(x, 0.01)
        for word, call in bad:
            assert call() == 1, word
        again = p.eval_time_offset(x, 0.01)  # the rejected calls left the trajectory as it was
        assert again[0] == ref[0] and again[1].tobytes() == ref[1].tobytes()
        xn = x.copy(); xn[4] = np.nan
        assert L.clc_eval_time_offset(h, dp(xn), 0.0, None, None, None) == 1 and b"pose7" in L.clc_last_error()
        assert L.clc_eval_time_offset(h, dp(x), float("inf"), None, None, None) == 1 and b"td" in L.clc_last_error()
        assert L.clc_eval_time_offset(None, dp(x), 0.0, None, None, None) == 1
        assert L.clc_information_time_offset(h, None, 0.0, None, None, None, None, None) == 1
        assert L.clc_solve_lm_time_offset(h, dp(x), None, None, None, None, 0) == 1
        for mask in (127, 128, -1):
            o = default_options()
            o.fixed_mask = mask
            assert L.clc_solve_lm_time_offset(h, dp(x), C.byref(td), C.byref(o), None, None, 0) == 1
            assert b"fixed_mask" in L.clc_last_error()
        for cap in (-1, 257):
            assert L.clc_solve_lm_time_offset(h, dp(x), C.byref(td), None, None, None, cap) == 1
            assert b"trace_cap" in L.clc_last_error()
        ms = (C.c_float * 1)()
        assert L.clc_bench_time_offset(h, dp(xn), 0.0, 1, 0, ms) == 1
        # the existing entry points keep rejecting masks >= 63
        o = default_options()
        o.fixed_mask = 64
        assert L.clc_solve_lm(h, dp(x), C.byref(o), None, None, 0) == 1
        # subsets and trims carry no trajectory
        with p.subset(np.ones(N, dtype=bool)) as q:
            assert L.clc_eval_time_offset(q._h, dp(x), 0.0, None, None, None) == 4
        with p.trim(x, np.inf) as q:
            assert L.clc_eval_time_offset(q._h, dp(x), 0.0, None, None, None) == 4
        # n_knots = 0 removes it
        p.set_trajectory(None, None, None)
        assert L.clc_eval_time_offset(h, dp(x), 0.0, None, None, None) == 4
    # edge residuals are not modelled
    from oracle import oracle as O

    d = O.generate(10, 50, seed=2, with_edges=True)
    with Problem.from_arrays(d.frame_pose, d.offsets, d.points, d.edge_points) as p:
        kt = np.arange(10) * 0.05
        assert L.clc_problem_set_trajectory(p._h, 10, dp(kt), dp(d.frame_pose), dp(kt)) == 1
        assert b"edge" in L.clc_last_error()


@pytest.mark.parametrize("family", list(FAMILIES))
def test_reproducible_and_bench(family):
    sc = TR.scene(n_knots=30, beams=200, seed=18, sigma=0.003, motion=2.0)
    with problem(sc, family, "cauchy") as p:
        x0 = TR.truth_pose7()
        a = p.solve_time_offset(x0, 0.0)
        b = p.solve_time_offset(x0, 0.0)
        assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1]
        assert [bytes(t) for t in a[3]] == [bytes(t) for t in b[3]]
        ms = p.bench_time_offset(x0, 0.0, 3)
        assert ms.shape == (3,) and np.all(ms > 0)


def test_offline_glue_recovers_the_offset():
    """calibrate_offline(..., time_offset=True) on a generated recording (tag poses at 30 Hz, scans at 40 Hz with a 12 ms clock
    offset, 2 mm range noise) recovers the offset; with time_offset=False it returns what the plain call returns."""
    from camlasercalibratool_b200 import formats as fmt

    sc = TR.scene(n_knots=90, beams=200, seed=19, td_true=0.012, sigma=0.002, motion=2.0)
    tagpose = []
    for t, kp in zip(sc.knot_times, sc.knot_poses):
        qwc = fmt.quat_inverse(kp[:4])
        tagpose.append(fmt.CamPose(float(t), qwc, -fmt.quat_to_rot(qwc) @ kp[4:]))
    scans = [(float(sc.frame_times[f]), sc.points[sc.offsets[f]:sc.offsets[f + 1]]) for f in range(len(sc.offsets) - 1)]
    Tlc_a, rep_a = fmt.calibrate_offline(tagpose, scans)
    Tlc_b, rep_b = fmt.calibrate_offline(tagpose, scans, time_offset=False)
    assert Tlc_a.tobytes() == Tlc_b.tobytes() and set(rep_a) == set(rep_b) and "time_offset" not in rep_a
    Tlc, rep = fmt.calibrate_offline(tagpose, scans, time_offset=True)
    print(f"offline: td {rep['time_offset'] * 1e3:.3f} ms (true {sc.td_true * 1e3:.1f} ms) from {rep['n_obs']} scans, "
          f"singular values {rep['time_offset_singular_values']}")
    assert abs(rep["time_offset"] - sc.td_true) < 1e-3
    assert rep["time_offset_summary"].termination != 6 and len(rep["time_offset_singular_values"]) == 7
    Tlc_true = np.eye(4)
    Tlc_true[:3, :3], Tlc_true[:3, 3] = TR.R_LC, TR.T_LC
    assert np.abs(Tlc - Tlc_true).max() < np.abs(rep["Tlc_without_time_offset"] - Tlc_true).max()
