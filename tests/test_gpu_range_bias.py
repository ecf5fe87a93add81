"""The laser's range offset and scale (clc_eval_range_bias, clc_information_range_bias, clc_solve_lm_range_bias,
clc_problem_range_correct) on the GPU, on both kernel families.  Scenes come from range_bias_reference.scene: boards at known
poses, points reported at the range (r_true - b) / (1 + s) along their rays.
"""
import contextlib
import os

import numpy as np
import pytest

import exact_sums as X
import layouts as LY
import loss_reference as LR
import range_bias_reference as RB

pytestmark = pytest.mark.gpu

FAMILIES = {"general": dict(CLC_PLANAR="0"), "planar": dict(CLC_PLANAR="1", CLC_PLANAR_MIN_POINTS="0")}
B_TRUE, S_TRUE = 0.025, 0.005


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


def problem(frame_pose, offsets, points, family, kind):
    from camlasercalibratool_b200 import Problem

    with env(**FAMILIES[family]):
        p = Problem.from_arrays(frame_pose, offsets, points, use_loss=kind == "cauchy")
    assert p.planar == (family == "planar")
    p.set_loss(kind)
    return p


def tight(**kw):
    from camlasercalibratool_b200 import default_options

    return default_options(function_tolerance=1e-20, parameter_tolerance=1e-15, gradient_tolerance=1e-20, **kw)


def pack(cost, H, g):
    return np.concatenate([H[RB.IU8], g, [cost]])


def check_sums(p, planes, offsets, points, x, bias, kind, what):
    cost, H, g = p.eval_range_bias(x, bias)
    val, mag = RB.rb_sums(planes, offsets, points, x, bias[0], bias[1], kind)
    X.assert_within(pack(cost, H, g), val, mag, RB.GROUPS_RB, what)


def ragged(sc, seed, planar, n_frames=300, big=60000):
    """sc's boards re-cut into frames of ragged sizes (0 ... big points): splits at every partition boundary kind."""
    rng = np.random.default_rng(seed)
    counts = rng.choice([0, 1, 3, 40, 700, 3000, big], size=n_frames, p=[0.06, 0.08, 0.1, 0.3, 0.3, 0.1, 0.06])
    counts[0] = 5
    base = type("B", (), {})()
    base.n_frames = len(sc.offsets) - 1
    base.offsets, base.points, base.frame_pose, base.edge_points = sc.offsets, sc.points, sc.frame_pose, None
    lay = LY.recut(base, counts, "ragged", (), with_edges=False, z_sigma=0.0 if planar else 0.2, seed=seed)
    return lay.frame_pose, lay.offsets, lay.points


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("kind", LR.KINDS)
def test_sums_ragged_multi_block(family, kind):
    sc = RB.scene(n_frames=60, beams=150, seed=3, sigma=0.004, planar=family == "planar")
    fp, off, pts = ragged(sc, 5 + LR.KINDS.index(kind), family == "planar")
    planes = np.asarray(X.frame_planes(fp), dtype=np.float64)
    with problem(fp, off, pts, family, kind) as p:
        for bias in ((0.0, 0.0), (B_TRUE, S_TRUE), (-0.04, -0.01)):
            check_sums(p, planes, off, pts, sc.pose7, bias, kind, f"{family} {kind} {bias}")


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", ["L1_aligned", "L3_empty_runs", "L4_giant_frame"])
def test_sums_layouts(oracle, family, name):
    """Layouts of tests/layouts.py: frame ends on stage, warp and block boundaries, empty runs, one frame over many blocks."""
    from camlasercalibratool_b200 import Problem

    with Problem.synthetic(600, 1000) as probe:  # every block of the device has stages
        grid_full = probe.partition(warp_table=False)["grid"]
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    lay = LY.build(name, LY.base_problem(oracle), grid_full, 256, stage)
    planes = np.asarray(X.frame_planes(lay.frame_pose), dtype=np.float64)
    with problem(lay.frame_pose, lay.offsets, lay.points, family, "cauchy") as p:
        check_sums(p, planes, lay.offsets, lay.points, RB.truth_pose7(), (B_TRUE, S_TRUE), "cauchy", f"{family} {name}")


def test_sums_ten_million_points():
    sc = RB.scene(n_frames=1000, beams=10000, seed=8, sigma=0.003)
    with problem(sc.frame_pose, sc.offsets, sc.points, "general", "cauchy") as p:
        check_sums(p, sc.planes, sc.offsets, sc.points, sc.pose7, (B_TRUE, S_TRUE), "cauchy", "1e7")


@pytest.mark.parametrize("family", list(FAMILIES))
def test_recovery_noise_free(family):
    """From the closed form and b = s = 0 the solve reaches T_cl, b and s to 1e-9; the plain solve is visibly biased."""
    from oracle import oracle as O

    sc = RB.scene(n_frames=60, beams=200, b=B_TRUE, s=S_TRUE, seed=11, planar=family == "planar", ranges=(0.8, 6.0))
    with problem(sc.frame_pose, sc.offsets, sc.points, family, "none") as p:
        T, _, _, _ = p.closed_form()
        from camlasercalibratool_b200 import T_to_pose7

        x0 = T_to_pose7(np.linalg.inv(T))
        x, bias, s, _ = p.solve_range_bias(x0, (0.0, 0.0), tight())
        assert s.termination != 6
        ang, dt = O.pose_error(x, sc.pose7)
        assert ang < 1e-9 and dt < 1e-9, (ang, dt)
        assert abs(bias[0] - B_TRUE) < 1e-9 and abs(bias[1] - S_TRUE) < 1e-9, bias
        xp, _, _ = p.solve(x0)
        _, dtp = O.pose_error(xp, sc.pose7)
        assert dtp > 1e-3, dtp  # the uncorrected offset goes into t_cl


def test_recovery_noisy_matches_least_squares():
    """With noise the solution is scipy least_squares' on the same residuals, to 1e-6."""
    from scipy.optimize import least_squares

    from oracle import oracle_np as ONP

    sc = RB.scene(n_frames=50, beams=150, seed=12, sigma=0.003, ranges=(0.8, 6.0))
    with problem(sc.frame_pose, sc.offsets, sc.points, "general", "none") as p:
        x0 = np.concatenate([ONP.pose_plus(sc.pose7, 0.01 * np.random.default_rng(1).standard_normal(6))])
        x, bias, s, _ = p.solve_range_bias(x0, (0.0, 0.0), tight())

    def res(v):
        x9 = np.concatenate([ONP.pose_plus(x, v[:6]), v[6:8]])
        return RB.evaluate8(sc, x9, "none")[1]

    ls = least_squares(res, np.concatenate([np.zeros(6), bias]), xtol=1e-15, ftol=1e-15, gtol=1e-15)
    xl = ONP.pose_plus(x, ls.x[:6])
    assert np.abs(xl[:3] - x[:3]).max() < 1e-6 and np.abs(ls.x[6:] - bias).max() < 1e-6, (xl - x, ls.x[6:] - bias)


def test_observability_narrow_band():
    """Boards in a narrow band of ranges: the weakest direction of the information lies in span(t, e_b, e_s) and has a large
    e_s share (the scale cannot be told from the offset); holding s lifts the smallest eigenvalue.  Boards over a wide band of
    ranges: the weakest direction has almost no e_s share (what remains is the offset against the translation along the
    viewing direction)."""
    sc = RB.scene(n_frames=40, beams=200, seed=13, ranges=(2.0, 2.05), planar=True)
    wide = RB.scene(n_frames=40, beams=200, seed=13, ranges=(0.8, 6.0), planar=True)
    with problem(sc.frame_pose, sc.offsets, sc.points, "general", "none") as p, \
            problem(wide.frame_pose, wide.offsets, wide.points, "general", "none") as q:
        H, _, _, sv = p.information_range_bias(sc.pose7, (B_TRUE, S_TRUE))
        v = p.last_V[:, -1]
        _, _, _, svw = q.information_range_bias(wide.pose7, (B_TRUE, S_TRUE))
        vw = q.last_V[:, -1]
    print(f"narrow: sv {sv}, V {v}; wide: sv {svw}, V {vw}")
    assert np.linalg.norm(v[[0, 1, 2, 6, 7]]) > 0.95, v
    assert abs(v[7]) > 0.3 and abs(vw[7]) < 0.1, (v, vw)
    held = np.linalg.eigvalsh(H[:7, :7])  # s held: its row and column leave the system
    assert held[0] / held[-1] > 2 * sv[-1] / sv[0], (held, sv)


@pytest.mark.parametrize("family", list(FAMILIES))
def test_range_corrected(family):
    sc = RB.scene(n_frames=40, beams=300, seed=14, sigma=0.002, planar=family == "planar")
    with problem(sc.frame_pose, sc.offsets, sc.points, family, "cauchy") as p:
        c1, H1, g1 = p.eval_range_bias(sc.pose7, (B_TRUE, S_TRUE))
        with env(**FAMILIES[family]):  # a copy picks its kernel family as a fresh creation does
            q, q2 = p.range_corrected((B_TRUE, S_TRUE)), p.range_corrected((B_TRUE, S_TRUE))
        with q, q2:
            assert q.planar == p.planar and q2.planar == p.planar
            c2, H2, g2 = q.eval(sc.pose7)
            assert q.eval(sc.pose7)[0] == q2.eval(sc.pose7)[0]
            assert np.array_equal(q.frame_report(sc.pose7)["max_abs_e"], q2.frame_report(sc.pose7)["max_abs_e"])
        val, mag = RB.rb_sums(sc.planes, sc.offsets, sc.points, sc.pose7, B_TRUE, S_TRUE, "cauchy")
        six = [k for k, (i, j) in enumerate(zip(*RB.IU8)) if j < 6]
        got = np.concatenate([H2[np.triu_indices(6)], g2, [c2]])
        idx = six + list(range(36, 42)) + [44]
        X.assert_within(got, val[idx], mag[idx], X.GROUPS_LM, "range_corrected")
        assert abs(c1 - c2) <= X.GAMMA * mag[44]


def test_rejections_and_reproducibility():
    from camlasercalibratool_b200 import ClcError, Problem, default_options
    from oracle import oracle as O

    sc = RB.scene(n_frames=30, beams=200, seed=15, sigma=0.003)
    with problem(sc.frame_pose, sc.offsets, sc.points, "general", "cauchy") as p:
        a = p.solve_range_bias(sc.pose7, (0.0, 0.0))
        b = p.solve_range_bias(sc.pose7, (0.0, 0.0))
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
        assert [bytes(t) for t in a[3]] == [bytes(t) for t in b[3]]
        e1, e2 = p.eval_range_bias(sc.pose7, (0.01, 0.0)), p.eval_range_bias(sc.pose7, (0.01, 0.0))
        assert e1[1].tobytes() == e2[1].tobytes() and e1[0] == e2[0]
        o = default_options()
        o.fixed_mask = 255
        with pytest.raises(ClcError):
            p.solve_range_bias(sc.pose7, (0.0, 0.0), o)
        with pytest.raises(ValueError):
            p.solve_range_bias(sc.pose7, (0.0, 0.0), fixed=("tx", "ty", "tz", "rx", "ry", "rz", "range_offset", "range_scale"))
        with pytest.raises(ValueError):
            p.range_corrected((0.0, -1.0))
        # held b and s keep their start bits
        x, bias, _, _ = p.solve_range_bias(sc.pose7, (0.01, -0.0), fixed=("range_offset", "range_scale"))
        assert bias[0] == 0.01 and np.signbit(bias[1])
    g = O.generate(20, 100, seed=2, sigma=0.01, with_edges=True)
    with Problem.from_arrays(g.frame_pose, g.offsets, g.points, edge_points=g.edge_points) as pe:
        with pytest.raises(ClcError):
            pe.eval_range_bias(sc.pose7, (0.0, 0.0))
        with pytest.raises(ClcError):
            pe.range_corrected((0.01, 0.0))


def test_offline_glue():
    """calibrate_offline(..., range_bias=True) reports the bias; range_bias=False returns what the plain call returns."""
    import time_offset_reference as TR
    from camlasercalibratool_b200 import formats as fmt

    sc = TR.scene(n_knots=90, beams=200, seed=19, td_true=0.0, sigma=0.001, motion=2.0)
    r = np.linalg.norm(sc.points, axis=1)
    pts = sc.points * (((r - B_TRUE) / (1 + S_TRUE)) / r)[:, None]
    tagpose = []
    for t, kp in zip(sc.knot_times, sc.knot_poses):
        qwc = fmt.quat_inverse(kp[:4])
        tagpose.append(fmt.CamPose(float(t), qwc, -fmt.quat_to_rot(qwc) @ kp[4:]))
    scans = [(float(sc.frame_times[f]), pts[sc.offsets[f]:sc.offsets[f + 1]]) for f in range(len(sc.offsets) - 1)]
    Tlc_a, rep_a = fmt.calibrate_offline(tagpose, scans)
    Tlc_b, rep_b = fmt.calibrate_offline(tagpose, scans, range_bias=False)
    assert Tlc_a.tobytes() == Tlc_b.tobytes() and "range_offset" not in rep_a
    Tlc, rep = fmt.calibrate_offline(tagpose, scans, range_bias=True)
    print(f"offline: b {rep['range_offset'] * 1e3:.2f} mm, s {rep['range_scale'] * 1e3:.2f} per mille, "
          f"singular values {rep['range_bias_singular_values']}")
    assert rep["range_bias_summary"].termination != 6 and len(rep["range_bias_singular_values"]) == 8
    assert np.isfinite(rep["range_offset"]) and np.isfinite(rep["range_scale"])
    assert rep["Tlc_without_range_bias"].tobytes() == Tlc_a.tobytes()
    with pytest.raises(ValueError):
        fmt.calibrate_offline(tagpose, scans, time_offset=True, range_bias=True)
