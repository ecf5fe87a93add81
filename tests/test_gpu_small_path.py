"""The reference-sized solve path against the extended-precision reference and the Ceres restatement (-m gpu).

The reference's own calls (50 boards x <= 180 beams, a few thousand residuals) run on the one-cluster kernel K2
(csrc/clc_small.cuh) and, for the closed form or with CLC_SMALL_KERNEL=0, on the single-block sweep kernel.  Here:
  * every layout of tests/small_layouts.py -- residual totals and the point/edge seam at K2's slot, CTA and warp ends and one
    either side, empty frames whose edges sit at the seam, one-point frames with edges, one 16 384-point frame, 16 384
    one-point frames, the single-block partition's stage and warp-range ends, off-plane points, boards 6-30 m away -- runs eval (loss, no loss,
    edges), information and the closed form with K2 on and off, for both kernel families, and every summed output must lie
    within GAMMA * A_k of tests/exact_sums.py.  Each problem first asserts, through clc_debug_dispatch, which kernel serves
    each call, so the test exercises the path it names;
  * the on-device LM runs every termination path under every driver (K2, the single-block loop, one launch per iteration
    with and without programmatic dependent launch, the persistent looping grid on a multi-block problem) and must take the
    oracle's decisions; the sweep-kernel drivers must be bit-identical to one another, K2 equal to 1e-12."""
import time

import numpy as np
import pytest

import exact_sums as X
import layouts as LY
import small_layouts as SL

from conftest import pack_sums
from test_gpu_partition import AtA_of, FAMILIES, FAR, MODES, X0, env, gpu_problem, near_optimum, ref_cf, ref_lm

pytestmark = pytest.mark.gpu

KERNELS = {"k2_on": "1", "k2_off": "0"}
WORST = {}  # largest |err| / A_k per (path, output group) over the module
_T0 = time.time()


def check(got, ref, groups, what, path):
    if what.startswith("far_range"):  # reported on its own: the scene where g cancels the most
        path += " far"
    r = X.assert_within(got, *ref, groups, f"{what} [{path}]")
    for name, v in X.worst_by_group(r, groups).items():
        WORST[(path, name)] = max(WORST.get((path, name), 0.0), v)


def expected_dispatch(P, N, edges, small_kernel):
    """The kernel each call must run on: K2 up to 16 384 residuals (edge residuals counted where the call has them; the
    information matrix never has them), the sweep kernel on one block up to 12 288 points, on several blocks beyond."""
    sweep = "single_block" if P <= SL.SINGLE_BLOCK_MAX else "multi_block"
    R = P + (2 * N if edges else 0)
    k2 = small_kernel == "1"
    return dict(eval="one_cluster" if k2 and R <= SL.SMALL_MAX else sweep,
                information="one_cluster" if k2 and P <= SL.SMALL_MAX else sweep,
                closed_form=sweep,
                solve="one_cluster" if k2 and R <= SL.SMALL_MAX else sweep + "_loop" if sweep == "single_block" else sweep,
                small_shape=(SL.SMALL_THREADS, SL.SMALL_CLUSTER, SL.SMALL_ITEMS))


@pytest.fixture(scope="module")
def base(oracle):
    return SL.base_problems(oracle)


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", SL.LAYOUTS)
def test_small_layout_against_exact_sums(oracle, base, name, family, kernel):
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    lay = SL.build(name, base, stage)
    if family == "planar" and lay.general_only:
        pytest.skip("z != 0: general kernels only")
    assert lay.targets <= SL.classify(lay, stage)
    P, N = lay.n_points, len(lay.offsets) - 1
    if name.startswith("far_range"):  # g = (S2 m + c S1) x m cancels by orders of magnitude near the optimum
        gt, gt_near = SL.far_range_poses(oracle)
        poses = (gt, gt_near)
    else:
        gt_near = near_optimum(oracle)
        poses = (X0, gt_near, FAR)
    with env(CLC_SMALL_KERNEL=KERNELS[kernel], **FAMILIES[family]):
        for mode, (loss, edges) in MODES.items():
            if edges and lay.edge_points is None:
                continue
            p = lay.problem(oracle, use_loss=loss, edges=edges)
            with gpu_problem(lay, loss, edges) as g:
                assert g.planar == (family == "planar")
                d = g.dispatch()
                assert d == expected_dispatch(P, N, edges, KERNELS[kernel]), (name, mode, d)
                part = g.partition(warp_table=False)
                if P <= SL.SINGLE_BLOCK_MAX:
                    assert (part["grid"], part["per_warp"], part["stage"]) == (1, SL.single_block_per_warp(P, stage), stage)
                for x in poses:
                    check(pack_sums(*g.eval(x)), ref_lm(p, x, mode), X.GROUPS_LM, f"{name}/{family}/{mode} eval", d["eval"])
                if mode == "edges":  # the information matrix has neither the loss nor the edge residuals of the problem
                    H, b, chi, sv = g.information(gt_near)
                    check(pack_sums(chi / 2, H, -b), ref_lm(p, gt_near, "no_loss"), X.GROUPS_LM,
                          f"{name}/{family} information of a problem with edges", d["information"])
                if mode != "no_loss":
                    continue
                H, b, chi, sv = g.information(gt_near)
                check(pack_sums(chi / 2, H, -b), ref_lm(p, gt_near, "no_loss"), X.GROUPS_LM, f"{name}/{family} information",
                      d["information"])
                svo = oracle.information(p, gt_near)[3]
                np.testing.assert_allclose(sv, svo, rtol=0, atol=1e-11 * svo[0])
                T, un, AtA, Atb = g.closed_form()
                check(X.pack_closed_form(AtA, Atb), ref_cf(p), X.GROUPS_CF, f"{name}/{family} closed form", d["closed_form"])
                sv_ref = np.linalg.svd(np.asarray(AtA_of(ref_cf(p)[0])), compute_uv=False)
                if sv_ref[-1] > 1e-6 * sv_ref[0]:  # T and the flag only where A^T A is clearly regular
                    To, uno, _, _ = oracle.closed_form(p)
                    assert un == uno
                    np.testing.assert_allclose(T, To, rtol=0, atol=1e-8)


# ---- the on-device LM on every termination path, under every driver ------------------------------------------------

BAD = np.array([3.0, -2.0, 4.0, 0.7, 0.1, -0.7, 0.1])  # test_gpu_parity's bad start
BAD[3:] /= np.linalg.norm(BAD[3:])
X0_NAN = np.array([np.nan, 0, 0, 0, 0, 0, 1.0])  # a non-finite start pose
NO_CONV, FUNCTION, PARAMETER, GRADIENT, MIN_RADIUS, FAILURE = 5, 1, 2, 3, 4, 6
# case -> (problem, start, options, termination the oracle reaches on the small problem or None)
CASES = {
    "max_it_0": ("plain", X0, dict(max_num_iterations=0), NO_CONV),
    "max_it_1": ("plain", X0, dict(max_num_iterations=1), NO_CONV),
    "max_it_2": ("plain", X0, dict(max_num_iterations=2), NO_CONV),
    "max_it_7": ("plain", X0, dict(max_num_iterations=7), NO_CONV),
    "default": ("plain", X0, dict(), FUNCTION),
    "default_bad_start": ("plain", BAD, dict(), FUNCTION),
    "gradient_tolerance": ("plain", X0, dict(gradient_tolerance=1e-3), GRADIENT),
    "min_radius_bad_start": ("plain", BAD, dict(min_relative_decrease=2.0, min_trust_region_radius=1e3), MIN_RADIUS),
    "min_radius_initial": ("plain", X0, dict(initial_trust_region_radius=1e-3, min_trust_region_radius=1e-3), MIN_RADIUS),
    "min_relative_decrease": ("plain", BAD, dict(min_relative_decrease=2.0), None),
    "no_jacobi_scaling": ("plain", BAD, dict(jacobi_scaling=0), FUNCTION),
    "max_radius_300": ("plain", BAD, dict(max_trust_region_radius=1e-2, max_num_iterations=300), NO_CONV),
    "per_sync_1": ("plain", X0, dict(iterations_per_sync=1), FUNCTION),
    "per_sync_3": ("plain", X0, dict(iterations_per_sync=3), FUNCTION),
    "per_sync_50": ("plain", X0, dict(iterations_per_sync=50), FUNCTION),
    "nan_point": ("nan", X0, dict(), FAILURE),
    "nan_start_pose": ("plain", X0_NAN, dict(), FAILURE),
    "invalid_1": ("pitch", X0, dict(min_lm_diagonal=0.0, max_num_consecutive_invalid_steps=1), FAILURE),
    "invalid_5": ("pitch", X0, dict(min_lm_diagonal=0.0, max_num_consecutive_invalid_steps=5), FAILURE),
}
# driver -> (knobs, the solve path clc_debug_dispatch must report)
SMALL_DRIVERS = {
    "k2": (dict(CLC_SMALL_KERNEL="1"), "one_cluster"),
    "single_block_loop": (dict(CLC_SMALL_KERNEL="0"), "single_block_loop"),
    "per_iteration": (dict(CLC_SMALL_KERNEL="0", CLC_LOOP_IN_KERNEL="0"), "single_block"),
    "per_iteration_no_pdl": (dict(CLC_SMALL_KERNEL="0", CLC_LOOP_IN_KERNEL="0", CLC_PDL="0"), "single_block"),
}
BIG_DRIVERS = {
    "persistent_loop": (dict(CLC_LOOP_IN_KERNEL="2"), "multi_block_loop"),
    "per_iteration": (dict(CLC_LOOP_IN_KERNEL="0"), "multi_block"),
    "per_iteration_no_pdl": (dict(CLC_LOOP_IN_KERNEL="0", CLC_PDL="0"), "multi_block"),
}
_PROBLEMS = {}


def lm_problem(oracle, kind, size):
    k = (kind, size)
    if k not in _PROBLEMS:
        if kind == "pitch":
            from test_gpu_degenerate import simulate

            p = simulate(oracle, "only_pitch", n_frames=50 if size == "small" else 150, seed=11, sigma=0.01)
        else:
            p = oracle.generate(50, 180, seed=2, sigma=0.02) if size == "small" else \
                oracle.generate(60, 400, seed=5, sigma=0.01, exact_m=True)
            if kind == "nan":
                pts = p.points.copy()
                pts[17, 1] = np.nan
                p = oracle.Problem(p.frame_pose, p.offsets, pts)
        assert (p.n_points <= SL.SINGLE_BLOCK_MAX) == (size == "small")
        _PROBLEMS[k] = p
    return _PROBLEMS[k]


def _rows(tr):
    return [(t.iteration, t.step_is_valid, t.step_is_successful) for t in tr]


def _summary(s):
    return (s.termination, s.num_iterations, s.num_successful_steps, s.num_unsuccessful_steps, s.num_sweeps, s.initial_cost,
            s.final_cost)


def _fields(tr):
    return [(t.iteration, t.step_is_valid, t.step_is_successful, t.cost, t.cost_change, t.gradient_max_norm, t.step_norm,
             t.relative_decrease, t.trust_region_radius) for t in tr]


def assert_follows_oracle(s, tr, so, tro, what):
    assert (s.termination, s.num_iterations, s.num_successful_steps, s.num_unsuccessful_steps) == \
        (so.termination, so.num_iterations, so.num_successful_steps, so.num_unsuccessful_steps), what
    assert len(tr) == min(so.num_iterations, 256) and _rows(tr) == _rows(tro[:len(tr)]), what

    def close(a, b, rtol, floor=0.0):
        return a == b or abs(a - b) <= rtol * abs(b) + floor

    for a, b in zip(tr, tro):
        w = f"{what} iteration {b.iteration}"
        assert close(a.cost, b.cost, 1e-9), (w, a.cost, b.cost)
        assert close(a.cost_change, b.cost_change, 1e-9, 1e-9 * abs(b.cost)), (w, a.cost_change, b.cost_change)
        assert close(a.trust_region_radius, b.trust_region_radius, 1e-6), (w, a.trust_region_radius, b.trust_region_radius)
        assert close(a.relative_decrease, b.relative_decrease, 1e-6, 1e-9), (w, a.relative_decrease, b.relative_decrease)
        assert close(a.step_norm, b.step_norm, 1e-6, 1e-13), (w, a.step_norm, b.step_norm)
        assert close(a.gradient_max_norm, b.gradient_max_norm, 1e-6, 1e-13), (w, a.gradient_max_norm, b.gradient_max_norm)


@pytest.mark.parametrize("size", ["small", "multi_block"])
@pytest.mark.parametrize("case", list(CASES))
def test_lm_termination_under_every_driver(oracle, case, size):
    from camlasercalibratool_b200 import default_options

    kind, x0, opts, want = CASES[case]
    sz = "small" if size == "small" else "big"
    p = lm_problem(oracle, kind, sz)
    xo, so, tro = oracle.solve(p, x0, oracle.default_options(**{k: v for k, v in opts.items() if k != "iterations_per_sync"}),
                               trace_cap=400)
    if want is not None and sz == "small":
        assert so.termination == want, (case, so.termination)  # the case reaches the path it is named after
    if case == "max_radius_300":
        assert so.num_iterations > 256
    drivers = SMALL_DRIVERS if sz == "small" else BIG_DRIVERS
    runs = {}
    for drv, (knobs, path) in drivers.items():
        with env(CLC_PLANAR="0", **knobs), gpu_problem(p) as g:
            assert g.dispatch()["solve"] == path, (drv, g.dispatch())
            x, s, tr = g.solve(x0, default_options(**opts))
            assert len(tr) == min(s.num_iterations, 256)
            if case == "max_radius_300":
                x5, s5, tr5 = g.solve(x0, default_options(**opts), trace_cap=5)
                assert s5.num_iterations == s.num_iterations > 256 and len(tr5) == 5
                assert _fields(tr5) == _fields(tr[:5]) and np.array_equal(x5, x)
        runs[drv] = (x, s, tr)
        assert_follows_oracle(s, tr, so, tro, f"{case}/{drv}")
        if so.termination == FAILURE and so.num_iterations == 0:
            assert np.array_equal(x, x0, equal_nan=True)
        elif kind != "pitch":
            ang, dt = oracle.pose_error(x, xo)
            assert ang < 1e-6 and dt < 1e-6, (case, drv, ang, dt)
        else:
            assert np.array_equal(x, x0)
    k1 = [d for d in runs if d != "k2"]
    x1, s1, tr1 = runs[k1[0]]
    for d in k1[1:]:  # the sweep kernel's drivers share the data path: bit for bit
        x, s, tr = runs[d]
        assert np.array_equal(x, x1, equal_nan=True) and _summary(s)[:5] == _summary(s1)[:5], (case, d)
        assert np.array_equal(_summary(s)[5:], _summary(s1)[5:], equal_nan=True), (case, d)
        assert np.array_equal(np.array(_fields(tr), dtype=float), np.array(_fields(tr1), dtype=float), equal_nan=True), (case, d)
    if "k2" in runs:  # the one-cluster kernel adds the same residuals in another order: same decisions, pose to 1e-12
        x, s, tr = runs["k2"]
        assert _summary(s)[:5] == _summary(s1)[:5] and _rows(tr) == _rows(tr1), case
        if not np.isnan(x1).any():
            np.testing.assert_allclose(x, x1, rtol=0, atol=1e-12)


def test_zz_report_headroom():
    """Largest |err| / A_k per kernel path and output group seen by this module (run with -s), and the module's runtime."""
    print("\nlargest |err|/A_k by path and group (GAMMA = %.0e):" % X.GAMMA)
    for (path, name), v in sorted(WORST.items()):
        print(f"  {path:22s} {name:14s} {v:.3e}  ({v / X.GAMMA:.3f} GAMMA)")
    print(f"module runtime so far: {time.time() - _T0:.1f} s")
    assert all(v <= X.GAMMA for v in WORST.values())
