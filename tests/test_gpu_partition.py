"""The sweep kernel's multi-block work partition against the extended-precision reference (tests/exact_sums.py), on frame
layouts that put frame boundaries, empty-frame runs and huge frames exactly at stage, warp-range and block boundaries of the
partition the device really uses (tests/layouts.py, read back through clc_debug_partition).  Every output k of eval,
information and the closed form must lie within GAMMA * A_k of the reference; solves must take the oracle's decisions.
Both kernel families run: the general three-stream kernels and the planar two-stream kernels."""
import contextlib
import os

import numpy as np
import pytest

import exact_sums as X
import layouts as LY

from conftest import pack_sums

pytestmark = pytest.mark.gpu

X0 = np.array([0, 0, 0, 0, 0, 0, 1.0])
FAR = np.array([0.4, -0.3, 0.25, 0.2, -0.5, 0.3, 0.78])
FAR[3:] /= np.linalg.norm(FAR[3:])
FAMILIES = {"general": dict(CLC_PLANAR="0"), "planar": dict(CLC_PLANAR="1", CLC_PLANAR_MIN_POINTS="0")}
MODES = {"loss": (True, False), "no_loss": (False, False), "edges": (True, True)}  # use_loss, edge residuals
WORST = {}  # largest |err| / A_k per output group over the module (printed by the last test)
_REF = {}   # reference sums, keyed by (problem content, pose, mode): shared by the two families


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


def gpu_problem(lay_or_p, use_loss=True, edges=False):
    from camlasercalibratool_b200 import Problem

    return Problem.from_arrays(lay_or_p.frame_pose, lay_or_p.offsets, lay_or_p.points, lay_or_p.edge_points if edges else None,
                               use_loss=use_loss)


def _key(p):
    return (hash(np.asarray(p.offsets).tobytes()), hash(np.asarray(p.points).tobytes()), hash(np.asarray(p.frame_pose).tobytes()))


def ref_lm(p, pose, mode):
    k = (_key(p), tuple(np.asarray(pose).tolist()), mode)
    if k not in _REF:
        loss, edges = MODES[mode]
        _REF[k] = X.lm_sums(p.frame_pose, p.offsets, p.points, pose, loss, 0.05, p.edge_points if edges else None)
    return _REF[k]


def ref_cf(p):
    k = (_key(p), "closed_form")
    if k not in _REF:
        _REF[k] = X.closed_form_sums(p.frame_pose, p.offsets, p.points)
    return _REF[k]


def AtA_of(cf_sums):
    A = np.zeros((9, 9))
    A[X.IU9] = np.asarray(cf_sums[:45], dtype=np.float64)
    return A + np.triu(A, 1).T


def check(got, ref, groups, what):
    r = X.assert_within(got, *ref, groups, what)
    for name, v in X.worst_by_group(r, groups).items():
        WORST[name] = max(WORST.get(name, 0.0), v)


def near_optimum(oracle, scale=1e-3):
    return oracle.pose_plus(oracle.ground_truth()[1], scale * np.array([1.0, -0.7, 0.4, -1.0, 0.6, 0.3]))


@pytest.fixture(scope="module")
def grid_full():
    from camlasercalibratool_b200 import Problem

    with Problem.synthetic(600, 1000) as probe:  # 600 000 points: every block of the device has stages
        return probe.partition(warp_table=False)["grid"]


@pytest.fixture(scope="module")
def base(oracle):
    return LY.base_problem(oracle)


def assert_partition(g, lay, grid_full, stage):
    """The device's partition is the restated one, its warp table is a binary search of the offsets, and the layout hits
    what it was cut to hit under it."""
    part = g.partition()
    P = lay.n_points
    assert part["stage"] == stage
    assert (part["grid"], part["per_warp"]) == LY.partition(P, grid_full, stage)
    w = np.arange(part["grid"] * LY.WARPS, dtype=np.int64)
    p0 = w * part["per_warp"]
    want = np.where(p0 < P, np.searchsorted(lay.offsets, np.minimum(p0, P), side="right") - 1, 0)
    np.testing.assert_array_equal(part["warp_first_frame"], want)
    hits = LY.classify(lay.offsets, part["grid"], part["per_warp"], stage)
    if 0 < part["resident_chunks"] < part["per_warp"] // stage:
        hits.add("partial_resident")
    assert lay.targets <= hits, (lay.name, lay.targets - hits)
    return part


def boundary_mutations_fail(oracle, lay, pose):
    """Reference side of the proof that these checks can fail: at one of the layout's frame boundaries, dropping the
    boundary point, counting it in the neighbouring frame, and counting an edge residual for an empty frame each move some
    output by more than GAMMA * A_k."""
    p = lay.problem(oracle)
    val, mag = ref_lm(p, pose, "edges")
    counts = np.diff(lay.offsets)
    ends = lay.offsets[1:-1]
    cand = np.nonzero((counts[:-1] > 1) & (counts[1:] > 0))[0]
    at_stage = cand[np.isin(ends[cand] % LY.STAGE_GENERAL, (0, 1, LY.STAGE_GENERAL - 1))]  # a boundary the layout placed
    cand = at_stage if at_stage.size else cand
    f = int(cand[len(cand) // 2]) if cand.size else 0
    e = int(lay.offsets[f + 1])  # first point after frame f (its boundary)
    dropped = np.delete(lay.points, e - 1, axis=0)
    off_d = lay.offsets.copy()
    off_d[f + 1:] -= 1
    moved = lay.offsets.copy()
    moved[f + 1] -= 1
    variants = [(off_d, dropped)] + ([(moved, lay.points)] if len(counts) > 1 else [])
    for off, pts in variants:
        v2, _ = X.lm_sums(lay.frame_pose, off, pts, pose, True, 0.05, lay.edge_points)
        assert np.max(X.error_ratios(v2.astype(np.float64), val, mag)) > X.GAMMA
    empty = np.nonzero(counts == 0)[0]
    if empty.size and lay.edge_points is not None:
        k = int(empty[0])  # the edge residuals of an empty frame, at the scale of a one-point frame
        one = lay.frame_pose[k:k + 1], np.array([0, 1]), lay.edge_points[k:k + 1, :3]
        with_e = X.lm_sums(*one, pose, True, 0.05, lay.edge_points[k:k + 1])[0]
        without = X.lm_sums(*one, pose, True, 0.05, None)[0]
        assert np.max(X.error_ratios((val + with_e - without).astype(np.float64), val, mag)) > X.GAMMA


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", LY.LAYOUTS)
def test_layout_against_exact_sums(oracle, base, grid_full, name, family):
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    if family == "planar" and name.endswith("_z"):
        pytest.skip("z != 0: general kernels only")
    lay = LY.build(name, base, grid_full, 256, stage)
    gt_near, P = near_optimum(oracle), lay.n_points
    with env(**FAMILIES[family]):
        # the partition depends on (P, family, device) only: a one-frame problem of the same size has the same one
        with gpu_problem(LY.recut(base, [P], "probe", set())) as probe:
            before = probe.partition(warp_table=False)
        for mode, (loss, edges) in MODES.items():
            p = lay.problem(oracle, use_loss=loss, edges=edges)
            with gpu_problem(lay, loss, edges) as g:
                assert g.planar == (family == "planar")
                part = assert_partition(g, lay, grid_full, stage)
                assert {k: part[k] for k in before} == before
                for x in (X0, gt_near, FAR):
                    got = pack_sums(*g.eval(x))
                    check(got, ref_lm(p, x, mode), X.GROUPS_LM, f"{name}/{family}/{mode} eval")
                    if mode == "loss" and x is X0:
                        assert np.array_equal(pack_sums(*g.eval(x)), got), "not bit-reproducible"
                if mode == "no_loss":
                    H, b, chi, sv = g.information(gt_near)
                    check(pack_sums(chi / 2, H, -b), ref_lm(p, gt_near, "no_loss"), X.GROUPS_LM, f"{name}/{family} information")
                    svo = oracle.information(p, gt_near)[3]
                    np.testing.assert_allclose(sv, svo, rtol=0, atol=1e-11 * svo[0])
                    T, un, AtA, Atb = g.closed_form()
                    check(X.pack_closed_form(AtA, Atb), ref_cf(p), X.GROUPS_CF, f"{name}/{family} closed form")
                    # T and the flag only where A^T A is clearly regular: laser points of one board lie on a line, so a board
                    # adds rank 2 and the one- and two-frame layouts sit at rounding level of the 1e-10 threshold
                    sv_ref = np.linalg.svd(np.asarray(AtA_of(ref_cf(p)[0])), compute_uv=False)
                    if sv_ref[-1] > 1e-6 * sv_ref[0]:
                        To, uno, _, _ = oracle.closed_form(p)
                        assert un == uno
                        np.testing.assert_allclose(T, To, rtol=0, atol=1e-8)
    if family == "general":
        boundary_mutations_fail(oracle, lay, gt_near)


def _solve_both_drivers(lay, family):
    out = []
    for loop in ("0", "2"):
        with env(CLC_LOOP_IN_KERNEL=loop, **FAMILIES[family]), gpu_problem(lay, True, False) as g:
            x, s, tr = g.solve(X0)
            out.append((x, s.termination, s.num_iterations, [(t.cost, t.step_is_successful) for t in tr]))
    return out


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", LY.LAYOUTS)
def test_layout_solve(oracle, base, grid_full, name, family):
    """One solve per layout with one launch per LM iteration and with the LM looping inside the persistent kernel: the two
    drivers are bit-identical, and both take the oracle's decisions."""
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    if family == "planar" and name.endswith("_z"):
        pytest.skip("z != 0: general kernels only")
    lay = LY.build(name, base, grid_full, 256, stage)
    (x0, t0, n0, tr0), (x2, t2, n2, tr2) = _solve_both_drivers(lay, family)
    assert np.array_equal(x0, x2) and (t0, n0) == (t2, n2) and tr0 == tr2
    xo, so, _ = oracle.solve(lay.problem(oracle), X0)
    assert (t0, n0) == (so.termination, so.num_iterations)
    ang, dt = oracle.pose_error(x0, xo)
    assert ang < 1e-6 and dt < 1e-6


def _threshold_problem(oracle, counts, edges):
    base = oracle.generate(40, 500, seed=13, sigma=0.01, exact_m=True, with_edges=True)
    lay = LY.recut(base, counts, "threshold", set(), with_edges=edges)
    return lay


@pytest.mark.parametrize("small_kernel", ["0", "1"])
@pytest.mark.parametrize("case", ["points_12288", "points_12289", "residuals_16384", "residuals_16385"])
def test_dispatch_thresholds(oracle, case, small_kernel):
    """Problems at the single-block limit (12 288 points) and at the one-cluster kernel's limit counted with the edge
    residuals (16 384): points <= 16 384 < points + edges takes the sweep kernel for eval and solve, although partition()
    sizes the L2 plan by points alone."""
    if case.startswith("points"):
        P = int(case.split("_")[1])
        counts, edges = [97] * (P // 97) + ([P % 97] if P % 97 else []), False
    else:
        R = int(case.split("_")[1])
        n = 192
        P = R - 2 * n
        counts, edges = [83] * (n - 1) + [P - 83 * (n - 1)], True
        assert P <= LY.SMALL_MAX_RESIDUALS and P + 2 * n == R
    lay = _threshold_problem(oracle, counts, edges)
    assert lay.n_points == P
    x_near = near_optimum(oracle)
    with env(CLC_SMALL_KERNEL=small_kernel, CLC_PLANAR="0"):
        for loss in (True, False):
            p = lay.problem(oracle, use_loss=loss, edges=edges)
            mode = "edges" if edges else ("loss" if loss else "no_loss")
            if edges and not loss:
                continue
            with gpu_problem(lay, loss, edges) as g:
                assert (g.partition(warp_table=False)["grid"] == 1) == (P <= LY.SINGLE_BLOCK_MAX)
                for x in (X0, x_near, FAR):
                    check(pack_sums(*g.eval(x)), ref_lm(p, x, mode), X.GROUPS_LM, f"{case}/{small_kernel}/{mode}")
                xs, s, _ = g.solve(X0)
            xo, so, _ = oracle.solve(p, X0)
            assert s.termination == so.termination
            ang, dt = oracle.pose_error(xs, xo)
            assert ang < 1e-6 and dt < 1e-6


@pytest.mark.parametrize("family", list(FAMILIES))
def test_far_range_conditioning(oracle, family):
    """Boards 6-30 m away (an oracle.generate scene scaled by 6, within the 30 m range cap of the scan conversion), 1 mm
    noise: near the optimum g = (S2 m + c S1) x m cancels by orders of magnitude, and must still be within GAMMA * A_k."""
    k = 6.0
    p0 = oracle.generate(200, 1000, seed=17, sigma=0.001 / k, exact_m=True)
    fp = p0.frame_pose.copy()
    fp[:, 4:] *= k
    p = oracle.Problem(fp, p0.offsets, p0.points * k)
    gt = oracle.ground_truth()[1].copy()
    gt[:3] *= k
    near = oracle.pose_plus(gt, 1e-5 * np.array([1.0, -0.7, 0.4, -1.0, 0.6, 0.3]))
    with env(**FAMILIES[family]):
        for loss in (True, False):
            q = oracle.Problem(fp, p0.offsets, p0.points * k, use_loss=loss)
            with gpu_problem(q, loss) as g:
                assert g.planar == (family == "planar")
                for x in (gt, near):
                    check(pack_sums(*g.eval(x)), ref_lm(q, x, "loss" if loss else "no_loss"), X.GROUPS_LM,
                          f"far/{family}/{loss}")
                xs, s, _ = g.solve(near)
            xo, so, _ = oracle.solve(q, near)
            assert (s.termination, s.num_iterations) == (so.termination, so.num_iterations)
            ang, dt = oracle.pose_error(xs, xo)
            assert ang < 1e-6 and dt < 1e-6


def test_zz_report_headroom():
    """Largest |err| / A_k per output group seen by this module (run with -s to read it), against GAMMA."""
    print("\nlargest |err|/A_k by group (GAMMA = %.0e):" % X.GAMMA)
    for name, v in sorted(WORST.items()):
        print(f"  {name:14s} {v:.3e}  ({v / X.GAMMA:.3f} GAMMA)")
    assert all(v <= X.GAMMA for v in WORST.values())
