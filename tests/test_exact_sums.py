"""CPU tests of the test infrastructure the partition tests stand on: the extended-precision reference (tests/exact_sums.py)
against the oracle, its numpy twin and exactly rounded float64 sums, and the adversarial layouts (tests/layouts.py) against
a Python restatement of partition() for several SM counts."""
import math

import numpy as np
import pytest

import exact_sums as X
import layouts as LY

from conftest import pack_sums

G = X.GAMMA


def small_problems(oracle):
    """Edges, empty frames, z != 0, loss on and off -- at most a few hundred residuals, so that the oracle's own float64
    sums stay well inside GAMMA * A_k."""
    rng = np.random.default_rng(4)
    base = oracle.generate(12, 30, seed=7, sigma=0.01, exact_m=True, with_edges=True)
    counts = np.array([0, 3, 30, 0, 0, 1, 2, 17, 30, 0, 5, 0])
    keep = np.concatenate([np.arange(base.offsets[f], base.offsets[f] + c) for f, c in enumerate(counts)]).astype(int)
    off = np.concatenate([[0], np.cumsum(counts)])
    pts = base.points[keep].copy()
    out = []
    for loss in (True, False):
        out.append(oracle.Problem(base.frame_pose, off, pts, base.edge_points, use_loss=loss))
        out.append(oracle.Problem(base.frame_pose, off, pts, None, use_loss=loss))
    ptz = pts.copy()
    ptz[:, 2] = rng.normal(size=len(ptz)) * 0.3
    out.append(oracle.Problem(base.frame_pose, off, ptz, base.edge_points, use_loss=True))
    out.append(oracle.Problem(base.frame_pose, off, ptz, None, use_loss=False))
    return out


def test_long_double_is_extended_precision():
    assert np.finfo(np.longdouble).nmant >= 63


def test_reference_equals_oracle_and_numpy_twin(oracle, oracle_np):
    gt = oracle.ground_truth()[1]
    poses = [np.array([0, 0, 0, 0, 0, 0, 1.0]), gt, oracle.pose_plus(gt, np.full(6, 1e-3)),
             np.array([0.3, -0.2, 0.4, 0.1, 0.7, -0.1, 0.7])]  # a far pose with a non-unit quaternion
    for p in small_problems(oracle):
        for x in poses:
            val, mag = X.lm_sums(p.frame_pose, p.offsets, p.points, x, p.use_loss, p.cauchy_a, p.edge_points)
            X.assert_within(pack_sums(*oracle.evaluate_normal(p, x)), val, mag, X.GROUPS_LM, "oracle")
            table = oracle_np.residual_table(p.frame_pose, p.offsets, p.points, p.edge_points)
            cost, r, J = oracle_np.evaluate(table, x, p.use_loss, p.cauchy_a)
            X.assert_within(pack_sums(cost, J.T @ J, J.T @ r), val, mag, X.GROUPS_LM, "numpy twin")
        # information: loss off, no edges, chi = 2 cost
        H, b, chi, sv = oracle.information(p, gt)
        val, mag = X.lm_sums(p.frame_pose, p.offsets, p.points, gt, False, p.cauchy_a, None)
        X.assert_within(pack_sums(chi / 2, H, -b), val, mag, X.GROUPS_LM, "information")
        _, _, AtA, Atb = oracle.closed_form(p)
        cval, cmag = X.closed_form_sums(p.frame_pose, p.offsets, p.points)
        X.assert_within(X.pack_closed_form(AtA, Atb), cval, cmag, X.GROUPS_CF, "closed form")
        _, _, AtA2, Atb2 = oracle_np.closed_form(p.frame_pose, p.offsets, p.points)
        X.assert_within(X.pack_closed_form(AtA2, Atb2), cval, cmag, X.GROUPS_CF, "closed form, numpy twin")


def _fsum_lm(p, x, use_loss, edges):
    """Every per-residual term in float64 (the plain PointInPlaneFactor arithmetic), summed exactly by math.fsum."""
    R = np.array(X._rot(np.asarray(x[3:7]).astype(np.longdouble)), dtype=np.float64)
    t = np.asarray(x[:3])
    a2 = p.cauchy_a ** 2
    rows = []
    counts = np.diff(p.offsets)
    for f in range(p.n_frames):
        if counts[f] == 0:
            continue
        s2 = 1.0 / counts[f]
        pl = X.frame_planes(p.frame_pose[f:f + 1]).astype(np.float64)[0]
        res = [(pl, p.points[j]) for j in range(p.offsets[f], p.offsets[f + 1])]
        if edges:
            e2 = X.edge_planes(p.frame_pose[f:f + 1]).astype(np.float64)[0]
            res += [(e2[0], p.edge_points[f, :3]), (e2[1], p.edge_points[f, 3:])]
        for plane, pt in res:
            n, m = plane[:3], R.T @ plane[:3]
            e = m @ pt + (n @ t + plane[3])
            w = 1.0 / (1.0 + e * e / a2) if use_loss else 1.0
            cost = 0.5 * s2 * a2 * math.log1p(e * e / a2) if use_loss else 0.5 * s2 * e * e
            J = np.concatenate([n, np.cross(pt, m)])
            rows.append(np.concatenate([(s2 * w * np.outer(J, J))[X.IU6], s2 * w * e * J, [cost]]))
    rows = np.array(rows)
    return np.array([math.fsum(rows[:, k]) for k in range(28)])


@pytest.mark.parametrize("use_loss,edges", [(True, False), (False, False), (True, True)])
def test_reference_equals_exactly_rounded_float64_sums(oracle, use_loss, edges):
    p = oracle.generate(4, 50, seed=9, sigma=0.01, exact_m=True, with_edges=True)
    assert p.n_points == 200
    for x in (oracle.ground_truth()[1], np.array([0.1, 0.2, -0.1, 0.0, 0.0, 0.6, 0.8])):
        val, mag = X.lm_sums(p.frame_pose, p.offsets, p.points, x, use_loss, p.cauchy_a, p.edge_points if edges else None)
        X.assert_within(_fsum_lm(p, x, use_loss, edges), val, mag, X.GROUPS_LM, "fsum")


def test_the_bound_is_tight_enough_to_fail(oracle):
    """A one-ulp-scale error would pass; dropping a single point of a frame does not."""
    p = oracle.generate(20, 100, seed=3, sigma=0.01, exact_m=True)
    x = oracle.pose_plus(oracle.ground_truth()[1], np.full(6, 1e-3))
    val, mag = X.lm_sums(p.frame_pose, p.offsets, p.points, x, True)
    off = p.offsets.copy()
    off[5] -= 1  # the last point of frame 4 counted in frame 5
    v2, _ = X.lm_sums(p.frame_pose, off, p.points, x, True)
    assert np.max(X.error_ratios(v2.astype(np.float64), val, mag)) > 1e3 * G


# ---- layouts --------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def base(oracle):
    return LY.base_problem(oracle)


def _shape(grid_full, stage):
    """(grid, per_warp) the layouts are built for: warp ranges of 256 points on a full grid, 4 stages on one block."""
    if grid_full == 1:
        return 1, 4 * stage
    return grid_full, 256


@pytest.mark.parametrize("grid_full", [132, 114, 1])
@pytest.mark.parametrize("stage", [LY.STAGE_GENERAL, LY.STAGE_PLANAR])
@pytest.mark.parametrize("name", LY.LAYOUTS)
def test_layout_hits_its_boundaries(base, grid_full, stage, name):
    grid, W = _shape(grid_full, stage)
    if stage == LY.STAGE_PLANAR and name.endswith("_z"):
        pytest.skip("z != 0: general kernels only")
    lay = LY.build(name, base, grid, W, stage)
    P = lay.n_points
    assert len(lay.offsets) == len(lay.frame_pose) + 1 and lay.points.shape == (P, 3)
    g, pw = LY.partition(P, grid_full, stage)
    hits = LY.classify(lay.offsets, g, pw, stage)
    missing = (lay.targets - {"partial_resident"}) - hits
    assert not missing, (name, missing, sorted(hits))
    if not name.startswith(("L6_jump", "L7")):
        assert (g, pw) == (grid, W), "the layout was cut for a different partition than the one its size gives"
    if "partial_resident" in lay.targets:
        k = LY.resident_chunks(P, g, pw, stage)
        assert 0 < k < pw // stage, (k, pw // stage)
    if grid_full > 1:
        assert P >= 200_000


def test_partition_restatement_known_values():
    assert LY.partition(9000, 132, 128) == (1, 768)            # one block: up to 12 288 points
    assert LY.partition(12_289, 132, 128) == (9, 128)          # blocks for the stages there are
    assert LY.partition(10_000_000, 132, 128) == (132, 6400)   # configs[1]
    assert LY.partition(10_000_000, 132, 256) == (132, 6400)
    assert LY.partition(132 * 12 * 256 + 1, 132, 128) == (132, 384)
