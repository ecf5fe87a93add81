"""The per-frame report (clc_frame_report) on the GPU.

* Every field of every frame within GAMMA * A of a long-double per-frame reference (tests/frame_exact.py) on the adversarial
  layouts of tests/layouts.py (multi-block partition) and tests/small_layouts.py (single-block and one-cluster sizes, which the
  report also runs on the sweep kernel), for both kernel families, with and without the loss and the edge residuals.
* Summed over the frames, the rows give clc_eval's cost, H, g and clc_information's chi; two calls return identical bytes.
* An in-process group of two devices returns the single-device rows.
* A frame whose tag pose is shifted 5 cm along its board normal has the largest |mean_e| and the largest influence.
"""
import contextlib
import os

import numpy as np
import pytest

import exact_sums as X
import frame_exact as FE
import layouts as LY
import small_layouts as SL

pytestmark = pytest.mark.gpu

FAR = np.array([0.4, -0.3, 0.25, 0.2, -0.5, 0.3, 0.78])
FAR[3:] /= np.linalg.norm(FAR[3:])
FAMILIES = {"general": dict(CLC_PLANAR="0"), "planar": dict(CLC_PLANAR="1", CLC_PLANAR_MIN_POINTS="0")}
MODES = {"loss": (True, False), "no_loss": (False, False), "edges": (True, True)}  # use_loss, edge residuals
WORST = {}


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


def gpu_problem(lay, use_loss=True, edges=False):
    from camlasercalibratool_b200 import Problem

    return Problem.from_arrays(lay.frame_pose, lay.offsets, lay.points, lay.edge_points if edges else None, use_loss=use_loss)


def near_optimum(oracle, scale=1e-3):
    return oracle.pose_plus(oracle.ground_truth()[1], scale * np.array([1.0, -0.7, 0.4, -1.0, 0.6, 0.3]))


def split_frames(offsets, per_warp):
    """Frames that cross a warp-range end under the partition (their rows come from the fix-up kernel)."""
    off = np.asarray(offsets, dtype=np.int64)
    live = off[1:] > off[:-1]
    return int(np.sum(live & (off[:-1] // per_warp != (np.maximum(off[1:], 1) - 1) // per_warp)))


def check_rows(rows, lay, x, loss, edges, what):
    assert np.array_equal(rows["n_points"], np.diff(lay.offsets)), what
    val, mag = FE.frame_sums(lay.frame_pose, lay.offsets, lay.points, x, loss, 0.05, lay.edge_points if edges else None)
    worst = FE.assert_within(FE.comparable(rows), val, mag, what=what)
    for k, v in worst.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
    empty = np.diff(lay.offsets) == 0
    assert all(np.all(rows[name][empty] == 0) for name in rows.dtype.names), what


@pytest.fixture(scope="module")
def grid_full():
    from camlasercalibratool_b200 import Problem

    with Problem.synthetic(600, 1000) as probe:
        return probe.partition(warp_table=False)["grid"]


@pytest.fixture(scope="module")
def base(oracle):
    return LY.base_problem(oracle)


@pytest.fixture(scope="module")
def small_bases(oracle):
    return SL.base_problems(oracle)


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", LY.LAYOUTS)
def test_partition_layouts_against_long_double(oracle, base, grid_full, name, family):
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    if family == "planar" and name.endswith("_z"):
        pytest.skip("z != 0: general kernels only")
    lay = LY.build(name, base, grid_full, 256, stage)
    with env(**FAMILIES[family]):
        for mode, (loss, edges) in MODES.items():
            with gpu_problem(lay, loss, edges) as g:
                assert g.planar == (family == "planar")
                part = g.partition(warp_table=False)
                assert (part["grid"], part["per_warp"]) == LY.partition(lay.n_points, grid_full, stage)
                assert split_frames(lay.offsets, part["per_warp"]) > 0, "the layout has no split frame"
                for x in (near_optimum(oracle), FAR):
                    check_rows(g.frame_report(x), lay, x, loss, edges, f"{name}/{family}/{mode}")


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", SL.LAYOUTS)
def test_small_layouts_against_long_double(oracle, small_bases, grid_full, name, family):
    """The reference-sized problems: eval runs them on the one-cluster kernel or one block, the report on the sweep kernel."""
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    lay = SL.build(name, small_bases, stage)
    if family == "planar" and lay.general_only:
        pytest.skip("z != 0: general kernels only")
    x = SL.far_range_poses(oracle)[1] if name.startswith("far_range") else near_optimum(oracle)
    modes = MODES if lay.edge_points is not None else {k: v for k, v in MODES.items() if not v[1]}
    with env(**FAMILIES[family]):
        for mode, (loss, edges) in modes.items():
            with gpu_problem(lay, loss, edges) as g:
                part = g.partition(warp_table=False)
                assert (part["grid"], part["per_warp"]) == LY.partition(lay.n_points, grid_full, stage)
                if split_frames(lay.offsets, part["per_warp"]) == 0:
                    pytest.skip("no frame crosses a warp-range end here")  # e.g. one or two residuals
                check_rows(g.frame_report(x), lay, x, loss, edges, f"{name}/{family}/{mode}")


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("edges", [False, True])
def test_rows_sum_to_eval_and_information(oracle, base, grid_full, family, edges):
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    for lay in (LY.build("L3_empty_runs", base, grid_full, 256, stage), LY.recut(base, [180] * 50, "reference_size", set())):
        x = near_optimum(oracle)
        with env(**FAMILIES[family]), gpu_problem(lay, True, edges) as g:
            rows = g.frame_report(x)
            assert rows.tobytes() == g.frame_report(x).tobytes(), "not bit-reproducible"
            cost, H, gg = g.eval(x)
            chi = g.information(x)[2]
            val, mag = X.lm_sums(lay.frame_pose, lay.offsets, lay.points, x, True, 0.05, lay.edge_points if edges else None)
            got = np.concatenate([rows["H21"].sum(axis=0), rows["g6"].sum(axis=0), [rows["cost"].sum()]])
            X.assert_within(got, val, mag, X.GROUPS_LM, f"summed rows/{family}/edges={edges}")
            # the report and clc_eval are two summation orders of the same terms: each within GAMMA * A_k of the reference
            assert np.all(np.abs(got - X.pack_lm(cost, H, gg)) <= 2 * X.GAMMA * mag), "rows do not sum to clc_eval"
            vi, mi = X.lm_sums(lay.frame_pose, lay.offsets, lay.points, x, False, 0.05, None)
            assert abs(rows["chi"].sum() - 2 * float(vi[27])) <= X.GAMMA * 2 * mi[27]
            assert abs(rows["chi"].sum() - chi) <= 2 * X.GAMMA * 2 * mi[27], "chi does not sum to clc_information"


def test_group_of_two_devices_returns_single_device_rows(oracle, base, grid_full):
    import torch

    from camlasercalibratool_b200 import Group

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    lay = LY.build("L3_empty_runs", base, grid_full, 256, LY.STAGE_GENERAL)
    x = near_optimum(oracle)
    with gpu_problem(lay, True, True) as p:
        single = p.frame_report(x)
    with Group.from_arrays(lay.frame_pose, lay.offsets, lay.points, lay.edge_points, devices=(0, 1)) as g:
        rows = g.frame_report(x)
    check_rows(rows, lay, x, True, True, "group of 2")
    assert np.array_equal(rows["n_points"], single["n_points"])
    val, mag = FE.frame_sums(lay.frame_pose, lay.offsets, lay.points, x, True, 0.05, lay.edge_points)
    assert np.all(FE.ratios(FE.comparable(rows), FE.comparable(single).astype(FE.LD), mag) <= 2 * X.GAMMA)


def test_a_shifted_tag_pose_is_found(oracle):
    """500 frames x 180 beams, 1 cm noise; frame 137's tag pose is shifted 5 cm along its board normal.  After the solve it has
    the largest |mean_e| and the largest one-step influence on the translation.  The one-step estimate is compared with a
    re-solve of the problem without that frame (printed: run with -s)."""
    from camlasercalibratool_b200 import Problem, frame_influence

    base = oracle.generate(500, 180, seed=31, sigma=0.01, exact_m=True)
    fp = base.frame_pose.copy()
    k = 137
    fp[k, 4:] += 0.05 * oracle.quat_to_rot(fp[k, :4])[:, 2]
    x0 = near_optimum(oracle, 1e-2)
    with Problem.from_arrays(fp, base.offsets, base.points) as g:
        x, s, _ = g.solve(x0)
        rows = g.frame_report(x)
        _, H, gg = g.eval(x)
    delta, t_norm, r_norm = frame_influence(rows, H, gg)
    assert int(np.argmax(np.abs(rows["mean_e"]))) == k
    assert int(np.argmax(t_norm)) == k
    keep = np.arange(500) != k
    counts = np.diff(base.offsets)[keep]
    off = np.concatenate([[0], np.cumsum(counts)])
    pts = np.concatenate([base.points[base.offsets[f]:base.offsets[f + 1]] for f in np.nonzero(keep)[0]])
    with Problem.from_arrays(fp[keep], off, pts) as g2:
        x2, s2, _ = g2.solve(x)
    dt = np.linalg.norm(x2[:3] - x[:3])
    dr = oracle.pose_error(x2, x)[0]
    print(f"\nshifted frame {k}: |mean_e| = {abs(rows['mean_e'][k]):.4f} m (next {np.sort(np.abs(rows['mean_e']))[-2]:.4f}); "
          f"one-step |dt| = {t_norm[k]:.3e} m, |dr| = {r_norm[k]:.3e} rad; re-solve |dt| = {dt:.3e} m, |dr| = {dr:.3e} rad; "
          f"ratio t {t_norm[k] / dt:.3f}, r {r_norm[k] / dr:.3f}")


def test_zz_report_headroom():
    """Largest |err| / A per field group seen by this module (run with -s to read it), against GAMMA."""
    print("\nlargest |err|/A by group (GAMMA = %.0e):" % X.GAMMA)
    for name, v in sorted(WORST.items()):
        print(f"  {name:14s} {v:.3e}  ({v / X.GAMMA:.3f} GAMMA)")
    assert all(v <= X.GAMMA for v in WORST.values())
