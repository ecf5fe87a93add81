"""Subsets of device-resident problems and groups (clc_problem_subset / clc_group_subset) on the GPU.

The reference of every case is a fresh Problem.from_arrays (Group.from_arrays) of the kept frames, and every comparison is on the
bytes: the subset is the problem that fresh creation builds, so its data, partition, dispatch and every output -- eval,
information, closed form, frame report, solve (pose, summary, trace) -- are bit-identical to the fresh problem's.  The masks
put the subset on the one-cluster kernel's limit, the single-block limit, the planar family's threshold and the warp-range ends
of its own partition (a tests/layouts.py layout whose frames are interleaved with frames the mask drops).
"""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

import layouts as LY

pytestmark = pytest.mark.gpu

FAMILIES = {"general": dict(CLC_PLANAR="0"), "planar": dict(CLC_PLANAR="1", CLC_PLANAR_MIN_POINTS="0")}
MODES = {"loss": (True, False), "no_loss": (False, False), "edges": (True, True)}  # use_loss, edge residuals
SUMMARY_FIELDS = ("termination", "num_iterations", "num_successful_steps", "num_unsuccessful_steps", "num_sweeps",
                  "initial_cost", "final_cost")  # device_ms is a time


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


def near_optimum(oracle, scale=1e-3):
    return oracle.pose_plus(oracle.ground_truth()[1], scale * np.array([1.0, -0.7, 0.4, -1.0, 0.6, 0.3]))


def np_subset(fp, off, pts, edge, keep):
    """The kept frames as from_arrays takes them."""
    keep = np.asarray(keep, dtype=bool)
    off = np.asarray(off, dtype=np.int64)
    counts = np.diff(off)
    new_off = np.concatenate([[0], np.cumsum(counts[keep])]).astype(np.int64)
    return fp[keep], new_off, pts[np.repeat(keep, counts)], None if edge is None else edge[keep]


class Scene:
    """Host arrays of a source problem (frame poses, offsets, points, edge points)."""

    def __init__(self, fp, off, pts, edge=None):
        self.fp, self.off, self.pts, self.edge = fp, np.asarray(off, dtype=np.int64), pts, edge

    @property
    def n_frames(self):
        return len(self.off) - 1

    def problem(self, loss=True, edges=False, keep=None):
        from camlasercalibratool_b200 import Problem

        e = self.edge if edges else None
        if keep is None:
            return Problem.from_arrays(self.fp, self.off, self.pts, e, use_loss=loss)
        return Problem.from_arrays(*np_subset(self.fp, self.off, self.pts, e, keep), use_loss=loss)

    def group(self, devices, loss=True, edges=False, keep=None):
        from camlasercalibratool_b200 import Group

        e = self.edge if edges else None
        arrays = (self.fp, self.off, self.pts, e) if keep is None else np_subset(self.fp, self.off, self.pts, e, keep)
        return Group.from_arrays(*arrays, devices=devices, use_loss=loss)


def interleave(lay, rng, junk_every=3):
    """The layout's frames with extra frames between them (random sizes, points and poses of other frames): returns the scene
    and the mask that keeps exactly the layout."""
    counts = np.diff(lay.offsets)
    out_counts, keep, src = [], [], []
    for f in range(len(counts)):
        if f % junk_every == 0:
            out_counts.append(int(rng.integers(0, 300)))
            keep.append(False)
            src.append(-1)
        out_counts.append(int(counts[f]))
        keep.append(True)
        src.append(f)
    out_counts.append(7)
    keep.append(False)
    src.append(-1)
    src = np.array(src)
    off = np.concatenate([[0], np.cumsum(out_counts)]).astype(np.int64)
    pts = np.empty((off[-1], 3))
    fp = np.empty((len(src), 7))
    edge = None if lay.edge_points is None else np.empty((len(src), 6))
    for i, f in enumerate(src):
        g = f if f >= 0 else int(rng.integers(0, len(counts)))
        fp[i] = lay.frame_pose[g]
        if edge is not None:
            edge[i] = lay.edge_points[g]
        if f >= 0:
            pts[off[i]:off[i + 1]] = lay.points[lay.offsets[f]:lay.offsets[f + 1]]
        else:
            pts[off[i]:off[i + 1]] = lay.points[rng.integers(0, lay.n_points, size=out_counts[i])] if lay.n_points else 0.0
    return Scene(fp, off, pts, edge), np.array(keep)


def exact_mask(counts, target, rng, extra=0, allowed=None):
    """Random big frames (all of one size) and one-point frames whose residuals -- points, plus `extra` per frame (its edge
    residuals) -- add up to exactly `target`; only frames in `allowed` are kept."""
    counts = np.asarray(counts)
    allowed = np.ones(len(counts), dtype=bool) if allowed is None else allowed
    big_idx, one_idx = np.nonzero((counts > 1) & allowed)[0], np.nonzero((counts == 1) & allowed)[0]
    big = int(counts[big_idx[0]]) + extra
    assert np.all(counts[big_idx] + extra == big)
    for a in range(min(len(big_idx), target // big), -1, -1):
        b, r = divmod(target - a * big, 1 + extra)
        if r == 0 and b <= len(one_idx):
            keep = np.zeros(len(counts), dtype=bool)
            keep[rng.choice(big_idx, a, replace=False)] = True
            keep[rng.choice(one_idx, b, replace=False)] = True
            return keep
    raise AssertionError(f"no mask reaches {target}")


def outcomes(p, x0, x, solve=True):
    """Every output of a problem or group, as bytes (or the status of the error it raised)."""
    from camlasercalibratool_b200 import ClcError

    out = {}

    def rec(name, fn):
        try:
            out[name] = ("ok", fn())
        except ClcError as exc:
            out[name] = ("error", str(exc).split(":")[0])

    rec("eval", lambda: b"".join(np.asarray(v).tobytes() for v in p.eval(x)))
    rec("information", lambda: b"".join(np.asarray(v).tobytes() for v in p.information(x)) + p.last_V.tobytes())
    rec("closed_form", lambda: b"".join(np.asarray(v).tobytes() for v in p.closed_form()))
    rec("frame_report", lambda: p.frame_report(x).tobytes())
    if solve:
        def run():
            xs, s, trace = p.solve(x0)
            return xs.tobytes() + repr([getattr(s, k) for k in SUMMARY_FIELDS]).encode() + b"".join(bytes(t) for t in trace)
        rec("solve", run)
    return out


def assert_same_outputs(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k] == b[k], f"{what}: {k} differs"


def assert_same_data(sub, fresh, what):
    ds, df = sub.download(), fresh.download()
    for k in ds:
        if ds[k] is None or df[k] is None:
            assert ds[k] is None and df[k] is None, f"{what}: {k}"
        else:
            assert ds[k].tobytes() == df[k].tobytes(), f"{what}: {k} differs"
    assert sub.planar == fresh.planar, what
    a, b = sub.partition(), fresh.partition()
    assert a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a), what
    assert sub.dispatch() == fresh.dispatch(), what


def check_subset(scene, keep, x0, x, loss=True, edges=False, solve=True, what=""):
    """subset(keep) of the scene's problem against a fresh problem of the kept frames: data, partition, dispatch, outputs.
    Returns the fresh problem's dispatch."""
    with scene.problem(loss, edges) as src, src.subset(keep) as sub, scene.problem(loss, edges, keep) as fresh:
        assert_same_data(sub, fresh, what)
        assert_same_outputs(outcomes(sub, x0, x, solve), outcomes(fresh, x0, x, solve), what)
        return fresh.dispatch(), fresh.partition(warp_table=False), fresh.planar


@pytest.fixture(scope="module")
def base(oracle):
    return LY.base_problem(oracle)


@pytest.fixture(scope="module")
def grid_full():
    from camlasercalibratool_b200 import Problem

    with Problem.synthetic(600, 1000) as probe:
        return probe.partition(warp_table=False)["grid"]


def mixed_scene(base, rng, n_big, big=180, n_one=400):
    """Frames of `big` points and one-point frames, shuffled, with the base's poses, points and edge points."""
    counts = np.array([big] * n_big + [1] * n_one)
    rng.shuffle(counts)
    lay = LY.recut(base, counts, "mixed", set())
    return Scene(lay.frame_pose, lay.offsets, lay.points, lay.edge_points)


def test_download_equals_the_numpy_subset(oracle, base):
    """The subset's data is the numpy subset of the source's download: points, offsets, poses, planes, edge points."""
    rng = np.random.default_rng(1)
    lay = LY.recut(base, rng.integers(0, 400, size=900), "ragged", set())
    scene = Scene(lay.frame_pose, lay.offsets, lay.points, lay.edge_points)
    for name, keep in (("random", rng.random(900) < 0.5), ("every_tenth_dropped", np.arange(900) % 10 != 0)):
        with scene.problem(True, True) as src, src.subset(keep) as sub:
            d, s = src.download(), sub.download()
            counts = np.diff(d["offsets"])
            assert np.array_equal(s["offsets"], np.concatenate([[0], np.cumsum(counts[keep])])), name
            assert s["points"].tobytes() == d["points"][np.repeat(keep, counts)].tobytes(), name
            for k in ("frame_pose", "planes", "edge_points"):
                assert s[k].tobytes() == d[k][keep].tobytes(), f"{name}: {k}"
            assert sub.sizes() == (int(keep.sum()), int(counts[keep].sum()), True)


def test_true_poses_of_a_camera_mode_source():
    from camlasercalibratool_b200 import Problem

    keep = np.arange(300) % 3 != 1
    with Problem.synthetic(300, 50, seed=4, sigma=0.01, camera="radtan", pixel_sigma=0.3) as src, src.subset(keep) as sub:
        assert sub.download_true_poses().tobytes() == src.download_true_poses()[keep].tobytes()
        assert sub.download()["frame_pose"].tobytes() == src.download()["frame_pose"][keep].tobytes()
        assert not np.array_equal(sub.download_true_poses(), sub.download()["frame_pose"])


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("target", ["k2_limit", "single_block_limit"])
def test_subsets_on_the_small_path_limits(oracle, base, family, target):
    """A multi-block source cut down to the one-cluster kernel's limit (16 384 residuals) and one either side, and to the
    single-block limit (12 288 points) and one either side; with and without the loss and the edge residuals."""
    rng = np.random.default_rng(7)
    scene = mixed_scene(base, rng, 150)  # 27 400 points: the sweep kernel on several blocks
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    with env(**FAMILIES[family]):
        with scene.problem() as src:
            assert src.dispatch()["eval"] == "multi_block"
        for mode, (loss, edges) in MODES.items():
            for d in (-1, 0, 1):
                if target == "k2_limit":  # with edges, the two edge residuals of every kept frame count too
                    keep = exact_mask(np.diff(scene.off), 16384 + d, rng, extra=2 if edges else 0)
                else:
                    keep = exact_mask(np.diff(scene.off), 12288 + d, rng)
                disp, part, _ = check_subset(scene, keep, x0, x, loss, edges, what=f"{target}{d:+d}/{family}/{mode}")
                if target == "k2_limit":
                    assert (disp["eval"] == "one_cluster") == (d <= 0), (d, disp)
                else:
                    assert (part["grid"] == 1) == (d <= 0), (d, part)


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", ["L1_aligned", "L2_off_by_one", "L3_empty_runs", "L5_confetti"])
def test_subsets_that_are_partition_layouts(oracle, base, grid_full, name, family):
    """A tests/layouts.py layout with other frames between its frames: the subset that drops them is the layout, so it hits
    the stage, warp-range and block-range ends the layout was cut for under its own partition."""
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    lay = LY.build(name, base, grid_full, 256, stage)
    scene, keep = interleave(lay, np.random.default_rng(11))
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    with env(**FAMILIES[family]):
        for mode, (loss, edges) in MODES.items():
            _, part, planar = check_subset(scene, keep, x0, x, loss, edges, what=f"{name}/{family}/{mode}")
            assert planar == (family == "planar")
            assert (part["grid"], part["per_warp"]) == LY.partition(lay.n_points, grid_full, stage)
            assert lay.targets <= LY.classify(lay.offsets, part["grid"], part["per_warp"], stage)


def test_small_layout_subsets(oracle):
    """tests/small_layouts.py layouts as subsets: the one-cluster kernel's slot ends, the seam and one-point frames."""
    import small_layouts as SL

    bases = SL.base_problems(oracle)
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    for name in ("seam_2048", "empty_edges_at_seam", "one_point_frames_edges", "total_2049", "sb_12stage+1"):
        lay = SL.build(name, bases, LY.STAGE_GENERAL)
        scene, keep = interleave(lay, np.random.default_rng(13), junk_every=2)
        for mode, (loss, edges) in MODES.items():
            if edges and lay.edge_points is None:
                continue
            check_subset(scene, keep, x0, x, loss, edges, what=f"{name}/{mode}")


def test_heavy_tailed_off_plane_layout(oracle, base, grid_full):
    lay = LY.build("L7_heavy_tailed_z", base, grid_full, 256, LY.STAGE_GENERAL)
    scene = Scene(lay.frame_pose, lay.offsets, lay.points, lay.edge_points)
    keep = np.random.default_rng(3).random(scene.n_frames) < 0.6
    _, _, planar = check_subset(scene, keep, near_optimum(oracle, 1e-2), near_optimum(oracle), True, True, what="L7_z")
    assert not planar


def planar_min_points(grid_full):
    return grid_full * LY.WARPS * LY.STAGE_PLANAR


def test_planar_threshold_and_dropped_off_plane_frames(oracle, base, grid_full):
    """Default planar mode.  A planar source (z stream freed) cut to planar_min_points and one below: planar, then general with
    the z stream re-materialised, as a fresh problem.  A source whose only z != 0 lie in dropped frames gives a planar subset
    when it is large enough, a general one below that."""
    rng = np.random.default_rng(17)
    pmin = planar_min_points(grid_full)
    counts = np.array([1000] * (pmin // 1000 + 8) + [1] * 2000)
    rng.shuffle(counts)
    lay = LY.recut(base, counts, "planar_source", set())
    scene = Scene(lay.frame_pose, lay.offsets, lay.points, lay.edge_points)
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    with scene.problem() as src:
        assert src.planar
    for d, want in ((0, True), (-1, False)):
        keep = exact_mask(counts, pmin + d, rng)
        assert check_subset(scene, keep, x0, x, what=f"planar source, P = min{d:+d}")[2] == want
    # off-plane frames that the mask drops
    bad = np.zeros(len(counts), dtype=bool)
    bad[rng.choice(np.nonzero(counts == 1000)[0], 5, replace=False)] = True
    pts = scene.pts.copy()
    pts[np.repeat(bad, counts), 2] = rng.normal(size=5000) * 0.2
    z_scene = Scene(scene.fp, scene.off, pts, scene.edge)
    with z_scene.problem() as src:
        assert not src.planar
    for P, want in ((pmin + 500, True), (pmin - 1, False), (40_000, False)):
        keep = exact_mask(counts, P, rng, allowed=~bad)
        assert not np.any(keep & bad)
        assert check_subset(z_scene, keep, x0, x, what=f"off-plane frames dropped, P = {P}")[2] == want


def test_a_nan_z_in_a_kept_frame_makes_the_subset_non_planar(oracle, base):
    rng = np.random.default_rng(19)
    lay = LY.recut(base, rng.integers(50, 400, size=300), "nan_z", set())
    pts = lay.points.copy()
    pts[lay.offsets[40] + 3, 2] = np.nan
    scene = Scene(lay.frame_pose, lay.offsets, pts, lay.edge_points)
    keep = rng.random(300) < 0.5
    keep[40] = True
    with env(CLC_PLANAR_MIN_POINTS="0"):
        _, _, planar = check_subset(scene, keep, near_optimum(oracle, 1e-2), near_optimum(oracle), solve=False, what="nan z")
        assert not planar
        keep[40] = False
        _, _, planar = check_subset(scene, keep, near_optimum(oracle, 1e-2), near_optimum(oracle), solve=False, what="nan dropped")
        assert planar


def test_keep_all_keep_none_and_the_source_is_unchanged(oracle, base):
    from camlasercalibratool_b200 import Problem

    rng = np.random.default_rng(23)
    lay = LY.recut(base, rng.integers(0, 300, size=400), "ragged", set())
    scene = Scene(lay.frame_pose, lay.offsets, lay.points, lay.edge_points)
    x0, x = near_optimum(oracle, 1e-2), near_optimum(oracle)
    with scene.problem(True, True) as src:
        before = outcomes(src, x0, x)
        with src.subset(np.ones(400, dtype=bool)) as sub:
            assert_same_data(sub, src, "keep all")
            assert_same_outputs(outcomes(sub, x0, x), before, "keep all")
        with src.subset(np.zeros(400, dtype=bool)) as sub, \
                Problem.from_arrays(np.zeros((0, 7)), [0], np.zeros((0, 3)), np.zeros((0, 6))) as empty:
            assert sub.sizes() == (0, 0, False)
            assert_same_data(sub, empty, "keep none")
            assert_same_outputs(outcomes(sub, x0, x, solve=False), outcomes(empty, x0, x, solve=False), "keep none")
        with src.subset(rng.random(400) < 0.3):
            pass
        assert_same_outputs(outcomes(src, x0, x), before, "source after subsetting")


def test_dropping_a_shifted_tag_pose(oracle):
    """The frame report's workflow: frame 137's tag pose is shifted 5 cm along its board normal.  The report ranks it first;
    the subset without it solves bit-identically to a fresh problem without it, lands closer to the ground truth than the
    solve with it, and the report's one-step frame_influence agrees with that re-solve."""
    from camlasercalibratool_b200 import frame_influence

    base = oracle.generate(500, 180, seed=31, sigma=0.01, exact_m=True)
    fp = base.frame_pose.copy()
    k = 137
    fp[k, 4:] += 0.05 * oracle.quat_to_rot(fp[k, :4])[:, 2]
    scene = Scene(fp, base.offsets, base.points)
    gt = oracle.ground_truth()[1]
    x0 = near_optimum(oracle, 1e-2)
    keep = np.arange(500) != k
    with scene.problem() as src:
        x, _, _ = src.solve(x0)
        rows = src.frame_report(x)
        _, H, g = src.eval(x)
        assert int(np.argmax(np.abs(rows["mean_e"]))) == k
        with src.subset(keep) as sub, scene.problem(keep=keep) as fresh:
            a, b = outcomes(sub, x, x), outcomes(fresh, x, x)
            assert_same_outputs(a, b, "without the shifted frame")
            x2, _, _ = sub.solve(x)
    delta, t_norm, r_norm = frame_influence(rows, H, g)
    assert int(np.argmax(t_norm)) == k
    err_with, err_without = oracle.pose_error(x, gt), oracle.pose_error(x2, gt)
    assert err_without[1] < err_with[1], (err_with, err_without)  # the shift biases the translation
    dt = np.linalg.norm(x2[:3] - x[:3])
    dr = oracle.pose_error(x2, x)[0]
    print(f"\nwithout frame {k}: error {err_with[1]:.3e} m -> {err_without[1]:.3e} m, {err_with[0]:.3e} -> {err_without[0]:.3e} rad; "
          f"one-step / re-solve: t {t_norm[k] / dt:.4f}, r {r_norm[k] / dr:.4f}")
    assert abs(t_norm[k] / dt - 1) < 0.01 and abs(r_norm[k] / dr - 1) < 0.01


def _group_check(scene, devices, keep, x0, x, what):
    with scene.group(devices, True, True) as src, src.subset(keep) as sub, scene.group(devices, True, True, keep) as fresh:
        assert sub.sizes() == fresh.sizes(), what
        for i in range(sub.sizes()[0]):
            ds, df = sub.problem(i).download(), fresh.problem(i).download()
            for k in ds:
                assert (ds[k] is None and df[k] is None) or ds[k].tobytes() == df[k].tobytes(), f"{what}: shard {i} {k}"
            assert sub.problem(i).dispatch() == fresh.problem(i).dispatch(), what
        # groups have no per-shard closed form / information differences: the collective outputs
        assert_same_outputs(outcomes(sub, x0, x), outcomes(fresh, x0, x), what)


def test_group_of_one_device(oracle, base):
    rng = np.random.default_rng(29)
    lay = LY.recut(base, rng.integers(0, 500, size=2000), "ragged", set())
    scene = Scene(lay.frame_pose, lay.offsets, lay.points, lay.edge_points)
    for keep in (rng.random(2000) < 0.5, np.arange(2000) % 10 != 0):
        _group_check(scene, (0,), keep, near_optimum(oracle, 1e-2), near_optimum(oracle), "group of 1")


def test_group_of_two_devices(oracle, base):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    rng = np.random.default_rng(31)
    lay = LY.recut(base, rng.integers(0, 500, size=2000), "ragged", set())
    scene = Scene(lay.frame_pose, lay.offsets, lay.points, lay.edge_points)
    keep_head = np.arange(2000) >= 700  # most of shard 0 dropped: kept frames of shard 1 move to device 0
    for keep in (rng.random(2000) < 0.5, keep_head, np.arange(2000) % 10 != 0):
        _group_check(scene, (0, 1), keep, near_optimum(oracle, 1e-2), near_optimum(oracle), "group of 2")


def test_invalid_masks_raise_before_device_work(base):
    from camlasercalibratool_b200 import _lib, launch_count

    lay = LY.recut(base, [100] * 20, "small", set())
    scene = Scene(lay.frame_pose, lay.offsets, lay.points)
    with scene.problem() as src, scene.group((0,)) as grp:
        n0 = launch_count()
        for p in (src, grp):
            with pytest.raises(ValueError):
                p.subset(np.ones(19, dtype=bool))
            with pytest.raises(ValueError):
                p.subset(np.ones((20, 1), dtype=bool))
            with pytest.raises(TypeError):
                p.subset(np.ones(20, dtype=np.int64))
        L = _lib.load()
        bad = np.ones(20, dtype=np.uint8)
        bad[5] = 2
        out = C.c_void_p()
        assert L.clc_problem_subset(src._h, bad.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(out)) == 1 and out.value is None
        assert b"keep[5]" in L.clc_last_error()
        assert L.clc_group_subset(grp._h, bad.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(out)) == 1 and out.value is None
        assert launch_count() == n0
