"""CPU side of tests/test_gpu_small_path.py: the small layouts hit what they were cut to hit under K2's slot mapping and the
single-block partition; between them they cover the residual totals and point counts where those kernels change state; the
residual list in K2's order sums to the extended-precision reference; and the reference bound catches the mistakes a slot
mapping can make.  Also: the oracle's QR path declares the steps of a rank-deficient damped system invalid exactly as the
device's Cholesky path does, so the GPU tests of the invalid-step termination compare like with like."""
import numpy as np
import pytest

import exact_sums as X
import layouts as LY
import small_layouts as SL

from conftest import pack_sums

STAGES = {"general": LY.STAGE_GENERAL, "planar": LY.STAGE_PLANAR}
X0 = np.array([0, 0, 0, 0, 0, 0, 1.0])


@pytest.fixture(scope="module")
def base(oracle):
    return SL.base_problems(oracle)


@pytest.fixture(scope="module")
def near(oracle):
    return oracle.pose_plus(oracle.ground_truth()[1], 1e-3 * np.array([1.0, -0.7, 0.4, -1.0, 0.6, 0.3]))


def test_small_slot_mapping():
    assert SL.SMALL_MAX == 16384 and SL.SLOT == 2048
    assert SL.small_slot(0) == (0, 0, 0, 0)
    assert SL.small_slot(31) == (0, 0, 31, 0) and SL.small_slot(32) == (0, 1, 0, 0)
    assert SL.small_slot(255) == (0, 7, 31, 0) and SL.small_slot(256) == (1, 0, 0, 0)
    assert SL.small_slot(2047) == (7, 7, 31, 0) and SL.small_slot(2048) == (0, 0, 0, 1)
    assert SL.small_slot(16383) == (7, 7, 31, 7)
    P, R, live = SL.small_residuals([0, 0, 3, 3, 5], True)
    assert (P, R) == (5, 13) and live.tolist() == [True] * 5 + [False, False, True, True, False, False, True, True]


@pytest.mark.parametrize("family", list(STAGES))
@pytest.mark.parametrize("name", SL.LAYOUTS)
def test_small_layout_hits_its_targets(base, name, family):
    stage = STAGES[family]
    lay = SL.build(name, base, stage)
    hits = SL.classify(lay, stage)
    assert lay.targets and lay.targets <= hits, (name, family, lay.targets - hits)


@pytest.mark.parametrize("family", list(STAGES))
def test_small_layouts_cover_the_thresholds(base, family):
    stage = STAGES[family]
    totals, points = set(), set()
    for name in SL.LAYOUTS:
        lay = SL.build(name, base, stage)
        hits = SL.classify(lay, stage)
        totals |= {int(t.split("=")[1]) for t in hits if t.startswith("k2:total=")}
        points |= {int(t.split("=")[1]) for t in hits if t.startswith("k1:P=") and t[5:].isdigit()}
    assert SL.K2_TOTALS <= totals, SL.K2_TOTALS - totals
    want = SL.K1_POINTS | {stage - 1, stage + 1, 12 * stage - 1, 12 * stage + 1}
    assert want <= points, want - points


@pytest.mark.parametrize("name", ["empty_edges_at_seam", "one_point_frames_edges", "seam_2049", "edges_total_16383"])
def test_k2_residual_order_sums_to_the_reference(oracle, base, near, name):
    lay = SL.build(name, base, LY.STAGE_GENERAL)
    plane, point, s2, live = SL.k2_residuals(lay.frame_pose, lay.offsets, lay.points, lay.edge_points)
    ref = X.lm_sums(lay.frame_pose, lay.offsets, lay.points, near, True, 0.05, lay.edge_points)
    got = X.lm_sums_of_residuals(plane[live], point[live], s2[live], near)
    assert np.max(X.error_ratios(got[0].astype(np.float64), *ref)) < 1e-3 * X.GAMMA


def _mutated_breaks_bound(lay, pose, mutate):
    plane, point, s2, live = SL.k2_residuals(lay.frame_pose, lay.offsets, lay.points, lay.edge_points)
    ref = X.lm_sums(lay.frame_pose, lay.offsets, lay.points, pose, True, 0.05, lay.edge_points)
    plane, point, s2, live = mutate(plane.copy(), point.copy(), s2.copy(), live.copy())
    got = X.lm_sums_of_residuals(plane[live], point[live], s2[live], pose)
    return np.max(X.error_ratios(got[0].astype(np.float64), *ref)) > X.GAMMA


@pytest.mark.parametrize("name", ["empty_edges_at_seam", "seam_2048", "seam_2049", "edges_total_16384"])
def test_reference_side_mutations_break_the_bound(oracle, base, near, name):
    """What a wrong slot mapping would compute, summed exactly, must fall outside GAMMA * A_k of the true sums: the seam edge
    moved by one slot (the first live edge residual evaluated as its neighbour), the residual at the last slot end dropped,
    and the edge residuals of an empty frame counted (at the scale of a one-point frame)."""
    lay = SL.build(name, base, LY.STAGE_GENERAL)
    P = lay.n_points
    for pose in (X0, near):
        def seam_moved(plane, point, s2, live):
            e = P + int(np.argmax(live[P:]))  # the first edge residual that exists
            plane[e], point[e], s2[e] = plane[e + 1], point[e + 1], s2[e + 1]
            return plane, point, s2, live

        def slot_end_dropped(plane, point, s2, live):
            i = (len(live) // SL.SLOT) * SL.SLOT - 1 if len(live) >= SL.SLOT else len(live) - 1
            live[i] = False
            return plane, point, s2, live

        assert _mutated_breaks_bound(lay, pose, seam_moved), name
        assert _mutated_breaks_bound(lay, pose, slot_end_dropped), name
        if not SL.small_residuals(lay.offsets, True)[2].all():
            def empty_edges_counted(plane, point, s2, live):
                dead = np.nonzero(~live)[0]
                s2[dead] = 1
                live[dead] = True
                return plane, point, s2, live

            assert _mutated_breaks_bound(lay, pose, empty_edges_counted), name


@pytest.mark.parametrize("max_invalid", [1, 5])
def test_oracle_qr_and_device_cholesky_agree_on_invalid_steps(oracle, harness, max_invalid):
    """The "ONLY pitch" teaching boards (every board normal has n_y = 0, so the t_y column of J is identically 0) with
    min_lm_diagonal = 0: the damped system is singular.  Ceres' DENSE_QR (Eigen householderQr) back-substitutes through
    R_kk = 0 and returns a non-finite step, which LevenbergMarquardtStrategy reports as LINEAR_SOLVER_FAILURE -> an invalid
    step; the device's Cholesky meets a zero pivot.  Both must record the same invalid iterations and stop with FAILURE
    after max_num_consecutive_invalid_steps of them."""
    from test_gpu_degenerate import simulate

    p = simulate(oracle, "only_pitch", seed=11, sigma=0.01)
    c, H, g = oracle.evaluate_normal(p, X0)
    assert not H[1].any() and not H[:, 1].any()
    xo, so, tro = oracle.solve(p, X0, oracle.default_options(min_lm_diagonal=0.0, max_num_consecutive_invalid_steps=max_invalid))
    assert so.termination == 6 and so.num_iterations == max_invalid
    assert [(t.iteration, t.step_is_valid, t.step_is_successful) for t in tro] == \
        [(0, 1, 1)] + [(k, 0, 0) for k in range(1, max_invalid)]
    assert np.array_equal(xo, X0)

    def sums(x):
        c, H, g = oracle.evaluate_normal(p, x)
        return pack_sums(c, H, g)

    o = harness.default_options(min_lm_diagonal=0.0, max_num_consecutive_invalid_steps=max_invalid)
    x, done, tr, sweeps = harness.lm_run(sums, X0, o)
    assert done == 6 and sweeps == 1 and np.array_equal(x, X0)
    assert [(t.iteration, t.step_is_valid, t.step_is_successful) for t in tr] == \
        [(t.iteration, t.step_is_valid, t.step_is_successful) for t in tro]
    for a, b in zip(tr, tro):
        assert a.cost == b.cost or abs(a.cost - b.cost) <= 1e-12 * b.cost
        assert a.trust_region_radius == b.trust_region_radius
