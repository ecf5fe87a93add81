"""Trims of device-resident problems and groups (clc_problem_trim / clc_group_trim) on the GPU.

The reference of every case is a fresh Problem.from_arrays (Group.from_arrays) of the kept points, and every comparison is on the
bytes: the trim is the problem that fresh creation builds, so its data, partition, dispatch and every output -- eval,
information, closed form, frame report, solve (pose, summary, trace) -- are bit-identical to the fresh problem's.  The scenes
are layouts with points far off their board inserted between the layout's points, so that the trim returns exactly the layout:
it then hits the one-cluster kernel's limit, the single-block limit, the planar family's threshold and the stage, warp-range and
block-range ends of its own partition.
"""
import ctypes as C

import numpy as np
import pytest

import layouts as LY
from test_gpu_subset import FAMILIES, MODES, Scene, assert_same_data, assert_same_outputs, env, near_optimum, outcomes

pytestmark = pytest.mark.gpu

TAU = 0.1  # the layouts' points lie within a few cm of their boards near the optimum, the inserted ones 0.3 - 1 m off


@pytest.fixture(scope="module")
def base(oracle):
    return LY.base_problem(oracle)


@pytest.fixture(scope="module")
def grid_full():
    from camlasercalibratool_b200 import Problem

    with Problem.synthetic(600, 1000) as probe:
        return probe.partition(warp_table=False)["grid"]


def laser_normals(oracle, fp, x):
    """m = R^T n and c = n.t + d of every frame at pose x (host arithmetic: only used to place points far from the threshold)."""
    R = oracle.quat_to_rot(x[3:])
    planes = np.array([oracle.frame_plane(f) for f in fp]).reshape(-1, 4)
    return planes[:, :3] @ R, planes[:, :3] @ x[:3] + planes[:, 3]


def inject(oracle, lay, x, rng, per_frame=(0, 6)):
    """The layout's frames with outliers -- points moved 0.3 - 1 m along their board's normal -- inserted at random places between
    their points (empty frames get outliers on their own board).  Returns the scene and the mask of the layout's points."""
    counts = np.diff(lay.offsets)
    N = len(counts)
    m, c = laser_normals(oracle, lay.frame_pose, x)
    k = rng.integers(per_frame[0], per_frame[1] + 1, size=N)
    fb = np.repeat(np.arange(N), k)
    own = lay.offsets[fb] + (rng.random(len(fb)) * np.maximum(counts[fb], 1)).astype(np.int64)
    on_board = np.where((counts[fb] > 0)[:, None], lay.points[np.minimum(own, max(lay.n_points - 1, 0))] if lay.n_points else 0.0,
                        -c[fb][:, None] * m[fb])
    bad = on_board + (rng.uniform(0.3, 1.0, size=len(fb)) * rng.choice([-1, 1], size=len(fb)))[:, None] * m[fb]
    where = lay.offsets[fb] + (rng.random(len(fb)) * (counts[fb] + 1)).astype(np.int64)
    order = np.lexsort((where, fb))
    pts = np.insert(lay.points, where[order], bad[order], axis=0)
    keep = np.insert(np.ones(lay.n_points, dtype=bool), where[order], False)
    off = lay.offsets + np.concatenate([[0], np.cumsum(k)]).astype(np.int64)
    new_counts = np.diff(off)
    e = np.abs(np.einsum("ij,ij->i", pts, np.repeat(m, new_counts, axis=0)) + np.repeat(c, new_counts))
    assert np.all(e[keep] < TAU / 2) and np.all(e[~keep] > 2 * TAU), "the scene is not cleanly separated"
    return Scene(lay.frame_pose, off, pts, lay.edge_points), keep


def np_trim(scene, keep, edges):
    """The kept points as from_arrays takes them: every frame stays."""
    ck = np.concatenate([[0], np.cumsum(keep)]).astype(np.int64)
    new_off = ck[scene.off]
    return scene.fp, new_off, scene.pts[keep], scene.edge if edges else None


def fresh(scene, keep, loss=True, edges=False):
    from camlasercalibratool_b200 import Problem

    return Problem.from_arrays(*np_trim(scene, keep, edges), use_loss=loss)


def check_trim(scene, keep, x0, x, tau=TAU, loss=True, edges=False, solve=True, what=""):
    """trim(x, tau) of the scene's problem against a fresh problem of the kept points: data, partition, dispatch, outputs; the
    trimmed problem's frame report at x stays within the thresholds.  Returns the fresh problem's dispatch, partition, planarity."""
    with scene.problem(loss, edges) as src, src.trim(x, tau) as t, fresh(scene, keep, loss, edges) as f:
        assert_same_data(t, f, what)
        assert_same_outputs(outcomes(t, x0, x, solve), outcomes(f, x0, x, solve), what)
        rows = t.frame_report(x)
        taus = np.broadcast_to(np.asarray(tau, dtype=np.float64), (scene.n_frames,))
        assert np.all(rows["max_abs_e"] <= taus), what
        return f.dispatch(), f.partition(warp_table=False), f.planar


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", ["L1_aligned", "L2_off_by_one", "L3_empty_runs", "L5_confetti"])
def test_trims_that_are_partition_layouts(oracle, base, grid_full, name, family):
    """A tests/layouts.py layout with outliers between its points: the trim is the layout, so it hits the stage, warp-range and
    block-range ends the layout was cut for under its own partition."""
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    lay = LY.build(name, base, grid_full, 256, stage)
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    scene, keep = inject(oracle, lay, x, np.random.default_rng(11))
    with env(**FAMILIES[family]):
        for mode, (loss, edges) in MODES.items():
            _, part, planar = check_trim(scene, keep, x0, x, TAU, loss, edges, what=f"{name}/{family}/{mode}")
            assert planar == (family == "planar")
            assert (part["grid"], part["per_warp"]) == LY.partition(lay.n_points, grid_full, stage)
            assert lay.targets <= LY.classify(lay.offsets, part["grid"], part["per_warp"], stage)


def test_small_layout_trims(oracle):
    """tests/small_layouts.py layouts as trims: the one-cluster kernel's slot ends, the seam and one-point frames."""
    import small_layouts as SL

    bases = SL.base_problems(oracle)
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    for name in ("seam_2048", "empty_edges_at_seam", "one_point_frames_edges", "total_2049", "sb_12stage+1"):
        lay = SL.build(name, bases, LY.STAGE_GENERAL)
        scene, keep = inject(oracle, lay, x, np.random.default_rng(13), per_frame=(0, 3))
        for mode, (loss, edges) in MODES.items():
            if edges and lay.edge_points is None:
                continue
            check_trim(scene, keep, x0, x, TAU, loss, edges, what=f"{name}/{mode}")


def exact_counts(rng, total, extra=0, lo=1, hi=180):
    """Frame sizes whose residuals -- points plus `extra` per frame (its edge residuals) -- add up to exactly `total`."""
    out, s = [], 0
    while s < total:
        k = int(rng.integers(lo, hi + 1))
        if s + k + extra > total:
            k = total - s - extra
            if k < 1:  # not enough room for a frame with edges: grow the previous one
                out[-1] += total - s
                break
        out.append(k)
        s += k + extra
    assert sum(out) + extra * len(out) == total
    return out


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("target", ["k2_limit", "single_block_limit"])
def test_trims_on_the_small_path_limits(oracle, base, family, target):
    """A multi-block source trimmed down to the one-cluster kernel's limit (16 384 residuals) and one either side, and to the
    single-block limit (12 288 points) and one either side; with and without the loss and the edge residuals."""
    rng = np.random.default_rng(7)
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    with env(**FAMILIES[family]):
        for mode, (loss, edges) in MODES.items():
            for d in (-1, 0, 1):
                if target == "k2_limit":  # with edges, the two edge residuals of every kept frame count too
                    counts = exact_counts(rng, 16384 + d, extra=2 if edges else 0)
                else:
                    counts = exact_counts(rng, 12288 + d)
                lay = LY.recut(base, counts, "limit", set())
                scene, keep = inject(oracle, lay, x, rng, per_frame=(60, 140))  # 15 000+ more points: several blocks
                with scene.problem(loss, edges) as src:
                    assert src.dispatch()["eval"] == "multi_block"
                disp, part, _ = check_trim(scene, keep, x0, x, TAU, loss, edges, what=f"{target}{d:+d}/{family}/{mode}")
                if target == "k2_limit":
                    assert (disp["eval"] == "one_cluster") == (d <= 0), (d, disp)
                else:
                    assert (part["grid"] == 1) == (d <= 0), (d, part)


def test_planar_threshold_with_off_plane_outliers(oracle, base, grid_full):
    """Default planar mode.  The outliers are off the laser plane (they move along the board normal), so the source is general;
    the trim that drops them is planar when it has planar_min_points points, general (z materialised as zeros, as a fresh
    problem) one below."""
    rng = np.random.default_rng(17)
    pmin = grid_full * LY.WARPS * LY.STAGE_PLANAR
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    for d, want in ((0, True), (-1, False), (1, True)):
        lay = LY.recut(base, exact_counts(rng, pmin + d, lo=500, hi=1000), "planar_threshold", set())
        scene, keep = inject(oracle, lay, x, rng, per_frame=(0, 3))
        with scene.problem() as src:
            assert not src.planar
        assert check_trim(scene, keep, x0, x, what=f"P = min{d:+d}")[2] == want


def identity_scene(z_rows):
    """Frames with identity tag poses (board plane z = 0 of the laser frame at the identity pose): there e == z exactly."""
    counts = [len(z) for z in z_rows]
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    P = int(off[-1])
    pts = np.zeros((P, 3))
    pts[:, 0] = np.linspace(0.5, 3.0, P)
    pts[:, 1] = np.linspace(-1.0, 1.0, P)
    pts[:, 2] = np.concatenate([np.asarray(z, dtype=np.float64) for z in z_rows])
    fp = np.zeros((len(counts), 7))
    fp[:, 3] = 1.0
    return Scene(fp, off, pts)


def test_exact_boundary(oracle):
    """|e| == tau is kept, nextafter(tau, +inf) dropped; tau = 0 keeps e = 0 only."""
    ident = np.array([0, 0, 0, 0, 0, 0, 1.0])
    taus = np.array([0.0625, 0.3, 1e-3, 0.0])
    up = [np.nextafter(t, np.inf) for t in taus]
    z_rows = [[taus[f], -taus[f], up[f], -up[f], 0.5 * taus[f], 0.0] * 40 for f in range(4)]
    scene = identity_scene(z_rows)
    keep = np.concatenate([np.array([True, True, False, False, True, True] * 40) for _ in range(4)])
    with scene.problem() as src:
        assert np.array_equal(src.download()["planes"], np.tile([0.0, 0.0, 1.0, 0.0], (4, 1)))
        with src.trim(ident, taus) as t:
            assert t.sizes()[1] == int(keep.sum())
            assert t.download()["points"].tobytes() == scene.pts[keep].tobytes()
    check_trim(scene, keep, ident, ident, taus, solve=False, what="exact boundary")


def test_nan_points_and_infinite_thresholds(oracle, base):
    """A point with a NaN coordinate is dropped at any threshold, and the frames around it then give the fresh problem's outputs
    (a NaN kept in a frame would spread through the moments into its stage neighbours); tau = +inf keeps every other point."""
    rng = np.random.default_rng(19)
    lay = LY.recut(base, rng.integers(50, 400, size=300), "nan", set())
    pts = lay.points.copy()
    bad = [lay.offsets[40] + 3, lay.offsets[41], lay.offsets[41] + 1, lay.offsets[200] + 7]
    pts[bad[0], 2] = np.nan
    pts[bad[1], 0] = np.nan
    pts[bad[2], 1] = np.nan
    pts[bad[3], :] = np.nan
    scene = Scene(lay.frame_pose, lay.offsets, pts, lay.edge_points)
    keep = np.ones(len(pts), dtype=bool)
    keep[bad] = False
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    with env(CLC_PLANAR_MIN_POINTS="0"):
        _, _, planar = check_trim(scene, keep, x0, x, np.inf, True, True, what="nan, tau = inf")
        assert planar  # the NaN z went with its point
        tau = np.full(300, np.inf)
        tau[100] = 1e-12  # and one frame emptied by its own threshold, the others untouched
        keep2 = keep.copy()
        keep2[lay.offsets[100]:lay.offsets[101]] = False
        check_trim(scene, keep2, x0, x, tau, True, True, what="nan, one frame emptied")
    with scene.problem() as src, src.trim(x, tau) as t:
        assert t.sizes()[0] == 300 and np.diff(t.download()["offsets"])[100] == 0


def test_combinations_invariants_and_the_source(oracle, base):
    """Per-frame thresholds from the frame report, both families, loss / no loss / edges: the trim equals the fresh problem, two
    trims give identical bytes, and the source's outputs are the same before and after."""
    rng = np.random.default_rng(23)
    lay = LY.recut(base, rng.integers(0, 600, size=400), "ragged", set())
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    scene, keep = inject(oracle, lay, x, rng, per_frame=(0, 4))
    for family, fam_env in FAMILIES.items():
        with env(**fam_env):
            for mode, (loss, edges) in MODES.items():
                with scene.problem(loss, edges) as src:
                    before = outcomes(src, x0, x)
                    # thresholds between the layout's points and the outliers, per frame
                    tau = np.where(rng.random(400) < 0.5, TAU, 2 * TAU)
                    with src.trim(x, tau) as a, src.trim(x, tau) as b, fresh(scene, keep, loss, edges) as f:
                        assert_same_data(a, f, f"{family}/{mode}")
                        assert_same_data(a, b, f"{family}/{mode} twice")
                        oa = outcomes(a, x0, x)
                        assert_same_outputs(oa, outcomes(b, x0, x), f"{family}/{mode} twice")
                        assert_same_outputs(oa, outcomes(f, x0, x), f"{family}/{mode}")
                        assert np.all(a.frame_report(x)["max_abs_e"] <= tau)
                    assert_same_outputs(outcomes(src, x0, x), before, f"{family}/{mode}: source after trimming")


def test_true_poses_of_a_camera_mode_source():
    from camlasercalibratool_b200 import Problem

    x = np.array([0, 0, 0, 0, 0, 0, 1.0])
    with Problem.synthetic(300, 50, seed=4, sigma=0.01, camera="radtan", pixel_sigma=0.3) as src, src.trim(x, 0.05) as t:
        assert t.download_true_poses().tobytes() == src.download_true_poses().tobytes()
        assert t.download()["frame_pose"].tobytes() == src.download()["frame_pose"].tobytes()
        assert 0 < t.sizes()[1] < src.sizes()[1]


def _group_check(scene, devices, keep, x0, x, what):
    from camlasercalibratool_b200 import Group

    with scene.group(devices, True, True) as src, src.trim(x, TAU) as t, \
            Group.from_arrays(*np_trim(scene, keep, True), devices=devices, use_loss=True) as f:
        assert t.sizes() == f.sizes(), what
        for i in range(t.sizes()[0]):
            ds, df = t.problem(i).download(), f.problem(i).download()
            for k in ds:
                assert (ds[k] is None and df[k] is None) or ds[k].tobytes() == df[k].tobytes(), f"{what}: shard {i} {k}"
            assert t.problem(i).dispatch() == f.problem(i).dispatch(), what
        assert_same_outputs(outcomes(t, x0, x), outcomes(f, x0, x), what)
        assert np.all(t.frame_report(x)["max_abs_e"] <= TAU)


def test_group_of_one_device(oracle, base):
    rng = np.random.default_rng(29)
    lay = LY.recut(base, rng.integers(0, 500, size=2000), "ragged", set())
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    scene, keep = inject(oracle, lay, x, rng)
    _group_check(scene, (0,), keep, x0, x, "group of 1")


def test_group_of_two_devices(oracle, base):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    rng = np.random.default_rng(31)
    lay = LY.recut(base, rng.integers(0, 500, size=2000), "ragged", set())
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    scene, keep = inject(oracle, lay, x, rng)
    _group_check(scene, (0, 1), keep, x0, x, "group of 2")
    # outliers only in the first 700 frames: the shard boundary moves back and kept points of shard 1 move to device 0
    head = LY.recut(base, np.diff(lay.offsets)[:700], "head", set())
    head_scene, head_keep = inject(oracle, head, x, rng, per_frame=(300, 300))
    tail = slice(lay.offsets[700], lay.offsets[-1])
    off = np.concatenate([head_scene.off, head_scene.off[-1] + lay.offsets[701:] - lay.offsets[700]])
    moved = Scene(lay.frame_pose, off, np.concatenate([head_scene.pts, lay.points[tail]]), lay.edge_points)
    _group_check(moved, (0, 1), np.concatenate([head_keep, np.ones(lay.offsets[-1] - lay.offsets[700], dtype=bool)]), x0, x,
                 "group of 2, head trimmed")


def test_invalid_arguments_raise_before_device_work(base):
    from camlasercalibratool_b200 import _lib, launch_count

    lay = LY.recut(base, [100] * 20, "small", set())
    scene = Scene(lay.frame_pose, lay.offsets, lay.points)
    x = np.array([0, 0, 0, 0, 0, 0, 1.0])
    with scene.problem() as src, scene.group((0,)) as grp:
        n0 = launch_count()
        for p in (src, grp):
            with pytest.raises(ValueError):
                p.trim(x, np.ones(19))
            with pytest.raises(ValueError):
                p.trim(x, np.ones((20, 1)))
            with pytest.raises(ValueError):
                p.trim(x, np.nan)
        L = _lib.load()
        out = C.c_void_p()
        dp = C.POINTER(C.c_double)
        for what, pose, tau in (("max_abs_e[5]", x, np.where(np.arange(20) == 5, np.nan, 1.0)),
                                ("max_abs_e[7]", x, np.where(np.arange(20) == 7, -1e-300, 1.0)),
                                ("pose7[2]", np.array([0, 0, np.inf, 0, 0, 0, 1.0]), np.ones(20)),
                                ("pose7[6]", np.array([0, 0, 0, 0, 0, 0, np.nan]), np.ones(20))):
            for fn, h in ((L.clc_problem_trim, src._h), (L.clc_group_trim, grp._h)):
                assert fn(h, pose.ctypes.data_as(dp), tau.ctypes.data_as(dp), C.byref(out)) == 1 and out.value is None
                assert what.encode() in L.clc_last_error()
            ms = (C.c_float * 1)()
            assert L.clc_bench_trim(src._h, pose.ctypes.data_as(dp), tau.ctypes.data_as(dp), 1, 1, ms, ms) == 1
        assert launch_count() == n0
