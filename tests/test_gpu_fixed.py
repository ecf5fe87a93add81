"""GPU tests (-m gpu) of held extrinsic coordinates (clc_lm_options.fixed_mask):

* every solve path -- the one-cluster kernel, the single-block sweep with and without the in-kernel loop, multi-block sweeps
  launched per iteration and the persistent grid -- on both kernel families, with and without edge residuals, under all four
  losses, makes the decisions of Ceres' LM on the reduced parameterization (tests/fixed_oracle.c for no loss and Cauchy, the
  numpy twin fixed_reference.solve_fixed over the losses' reference evaluation for Huber and soft-L1), to 1e-6; held
  translations keep the start's bits;
* the reference's degenerate teaching geometries with the null space held at the truth's values: full parity with the oracle,
  noise-free data reaching the truth; rotation-only and translation-only solves reaching the truth;
* solve_segments and solve_starts under a mask equal single solves (bytes on the one-cluster starts path), best follows its
  rule; Group.solve equals Problem.solve;
* a bad mask is rejected on a real problem before any device work.
"""
import tempfile

import numpy as np
import pytest

import fixed_reference as FR
import loss_reference as LR
from test_gpu_degenerate import simulate
from test_gpu_partition import FAMILIES, env
from test_gpu_small_path import BIG_DRIVERS, SMALL_DRIVERS, assert_follows_oracle

pytestmark = pytest.mark.gpu

A = 0.05
X0 = np.array([0, 0, 0, 0, 0, 0, 1.0])
KIND_MASK = {"none": 0b000001, "cauchy": 0b011010, "huber": 0b100001, "soft_l1": 0b111000}
_PROBLEMS = {}
_FO = []


def fixed_oracle():
    if not _FO:
        _FO.append(FR.FixedOracle(tempfile.mkdtemp(prefix="fixed_oracle")))
    return _FO[0]


def problem(oracle, size, edges):
    k = (size, edges)
    if k not in _PROBLEMS:
        _PROBLEMS[k] = oracle.generate(50, 180, seed=2, sigma=0.02, with_edges=edges) if size == "small" else \
            oracle.generate(60, 400, seed=5, sigma=0.01, exact_m=True, with_edges=edges)
    return _PROBLEMS[k]


def gpu(p, kind="cauchy"):
    from camlasercalibratool_b200 import Problem

    g = Problem.from_arrays(p.frame_pose, p.offsets, p.points, p.edge_points, use_loss=True, cauchy_a=A)
    g.set_loss(kind, A)
    return g


def held_t(mask):
    return [k for k in range(3) if mask >> k & 1]


def free_start(oracle, x, mask, rng, s):
    d = s * rng.standard_normal(6)
    d[[k for k in range(6) if mask >> k & 1]] = 0.0
    return oracle.pose_plus(x, d)


def reduced_oracle(oracle, p, x0, kind, mask):
    """(pose, termination code, [step_is_successful]) of Ceres' LM on the reduced parameterization under the loss `kind`."""
    if kind in ("none", "cauchy"):
        q = oracle.Problem(p.frame_pose, p.offsets, p.points, p.edge_points, use_loss=kind == "cauchy", cauchy_a=A)
        xo, so, tro = fixed_oracle().solve(q, x0, mask)
        return xo, so.termination, [bool(t.step_is_successful) for t in tro], (so, tro)
    from oracle import oracle_np as ONP

    table = ONP.residual_table(p.frame_pose, p.offsets, p.points, p.edge_points)
    xn, term, trn = FR.solve_fixed(lambda y: LR.evaluate(table, y, kind, A), x0, mask)
    code = {v: k for k, v in oracle.TERMINATION.items()}[term]
    return xn, code, [r["ok"] for r in trn], None


def assert_reduced_parity(oracle, p, x0, kind, mask, x, s, tr, what, noise_free=False):
    """The oracle's decisions and pose to 1e-6; with the C oracle also its per-row trace fields, except on noise-free data,
    where the costs near 0 are cancellation and only the decisions are compared."""
    xo, term, ok, full = reduced_oracle(oracle, p, x0, kind, mask)
    if full is not None and not noise_free:
        assert_follows_oracle(s, tr, *full, what)
    elif full is not None:
        so, tro = full
        assert (s.termination, s.num_iterations, s.num_successful_steps, s.num_unsuccessful_steps) == \
            (so.termination, so.num_iterations, so.num_successful_steps, so.num_unsuccessful_steps), what
        assert [(t.step_is_valid, t.step_is_successful) for t in tr] == [(t.step_is_valid, t.step_is_successful) for t in tro], what
    else:
        assert s.termination == term, (what, s.termination, term)
        assert len(ok) in (len(tr), len(tr) - 1) and ok == [bool(t.step_is_successful) for t in tr[:len(ok)]], what
    ang, dt = oracle.pose_error(x, xo)
    assert ang < 1e-6 and dt < 1e-6, (what, ang, dt)
    assert x[held_t(mask)].tobytes() == np.asarray(x0)[held_t(mask)].tobytes(), what


@pytest.mark.parametrize("edges", [False, True])
@pytest.mark.parametrize("kind", list(KIND_MASK))
@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("size", ["small", "multi_block"])
def test_every_path_makes_the_reduced_oracles_decisions(oracle, size, family, kind, edges):
    from camlasercalibratool_b200 import default_options

    mask = KIND_MASK[kind]
    p = problem(oracle, size, edges)
    x0 = free_start(oracle, oracle.ground_truth()[1], 0, np.random.default_rng(3), 0.05)
    drivers = SMALL_DRIVERS if size == "small" else BIG_DRIVERS
    for drv, (knobs, path) in drivers.items():
        with env(**FAMILIES[family], **knobs), gpu(p, kind) as g:
            if family == "general":
                assert g.dispatch()["solve"] == path, (drv, g.dispatch())
            x, s, tr = g.solve(x0, default_options(fixed_mask=mask))
        assert_reduced_parity(oracle, p, x0, kind, mask, x, s, tr, f"{size}/{family}/{kind}/edges={edges}/{drv}/mask={mask}")


@pytest.mark.parametrize("variant,mask", [("only_roll", 0b000001), ("only_pitch", 0b011010)])
@pytest.mark.parametrize("seed,centred", [(3, False), (11, True)])
def test_degenerate_geometries_with_the_null_space_held(oracle, variant, mask, seed, centred):
    """The coordinates the reference's null-space report names, held at the truth's values: the solve is well posed, so the
    full north-star parity applies (test_gpu_degenerate.py can only compare the observable projection without them)."""
    from camlasercalibratool_b200 import default_options

    gt = oracle.ground_truth()[1]
    rng = np.random.default_rng(seed)
    for sigma in (0.0, 0.01):
        p = simulate(oracle, variant, seed=seed, sigma=sigma, centred=centred)
        x0 = free_start(oracle, gt, mask, rng, 0.05)
        with gpu(p) as g:
            x, s, tr = g.solve(x0, default_options(fixed_mask=mask))
        assert_reduced_parity(oracle, p, x0, "cauchy", mask, x, s, tr, f"{variant} sigma={sigma}", noise_free=sigma == 0.0)
        if sigma == 0.0:
            # Ceres stops once a step is shorter than parameter_tolerance * |x| (1e-8 * ~1.1 here) and does not apply it
            ang, dt = oracle.pose_error(x, gt)
            assert ang < 2e-8 and dt < 2e-8, (variant, ang, dt)


@pytest.mark.parametrize("mask", [0b000111, 0b111000])  # rotation only, translation only
@pytest.mark.parametrize("size", ["small", "multi_block"])
def test_extreme_masks_reach_the_truth(oracle, mask, size):
    from camlasercalibratool_b200 import default_options

    p = oracle.generate(50, 180, seed=6, sigma=0.0) if size == "small" else oracle.generate(60, 400, seed=6, sigma=0.0)
    gt = oracle.ground_truth()[1]
    x0 = free_start(oracle, gt, mask, np.random.default_rng(1), 0.1)
    with gpu(p) as g:
        x, s, tr = g.solve(x0, default_options(fixed_mask=mask))
    assert s.termination != 6
    assert x[held_t(mask)].tobytes() == x0[held_t(mask)].tobytes()
    ang, dt = oracle.pose_error(x, gt)
    assert ang < 2e-8 and dt < 2e-8, (mask, size, ang, dt, s.termination)
    assert_reduced_parity(oracle, p, x0, "cauchy", mask, x, s, tr, f"extreme mask={mask} {size}", noise_free=True)


@pytest.mark.parametrize("family", list(FAMILIES))
def test_segments_equal_single_solves(oracle, family):
    from camlasercalibratool_b200 import Problem, default_options

    p = oracle.generate(90, 300, seed=7, sigma=0.01, with_edges=True)
    seg = np.array([0, 30, 55, 90], dtype=np.int64)
    gt = oracle.ground_truth()[1]
    rng = np.random.default_rng(2)
    mask = 0b001010  # ty, rx
    x0 = np.array([free_start(oracle, gt, 0, rng, 0.05) for _ in range(3)])
    o = default_options(fixed_mask=mask)
    with env(**FAMILIES[family]), gpu(p) as g:
        xs, summ, traces = g.solve_segments(seg, x0, o, trace_cap=256)
    for s in range(3):
        b, e = int(seg[s]), int(seg[s + 1])
        off = p.offsets[b:e + 1] - p.offsets[b]
        with env(**FAMILIES[family]), Problem.from_arrays(p.frame_pose[b:e], off, p.points[p.offsets[b]:p.offsets[e]],
                                                          p.edge_points[b:e], use_loss=True, cauchy_a=A) as gs:
            x1, s1, t1 = gs.solve(x0[s], o)
        assert (summ[s].termination, summ[s].num_iterations) == (s1.termination, s1.num_iterations), s
        assert [r.step_is_successful for r in traces[s]] == [r.step_is_successful for r in t1], s
        assert np.abs(xs[s] - x1).max() <= 1e-12, (s, np.abs(xs[s] - x1).max())
        assert xs[s][held_t(mask)].tobytes() == x0[s][held_t(mask)].tobytes()


@pytest.mark.parametrize("path", ["one_cluster", "sweep"])
def test_starts_equal_single_solves(oracle, path):
    from camlasercalibratool_b200 import default_options

    p = oracle.generate(50, 180, seed=3, sigma=0.02) if path == "one_cluster" else oracle.generate(120, 400, seed=4, sigma=0.01)
    gt = oracle.ground_truth()[1]
    rng = np.random.default_rng(8)
    mask = 0b100100  # tz, rz
    x = np.array([X0] + [free_start(oracle, gt, 0, rng, s) for s in (1e-3, 1e-2, 0.1, 0.3)])
    o = default_options(fixed_mask=mask)
    with env(CLC_PLANAR="0"), gpu(p) as g:
        assert (g.dispatch()["solve"] == "one_cluster") == (path == "one_cluster"), g.dispatch()
        xs, sums, traces, best = g.solve_starts(x, o, trace_cap=256)
        for k in range(len(x)):
            xk, sk, tk = g.solve(x[k], o)
            if path == "one_cluster":
                assert xk.tobytes() == xs[k].tobytes(), k
                assert (sk.termination, sk.num_iterations, sk.final_cost) == (sums[k].termination, sums[k].num_iterations,
                                                                             sums[k].final_cost), k
                assert [bytes(r) for r in tk] == [bytes(r) for r in traces[k]], k
            else:
                assert (sk.termination, sk.num_iterations) == (sums[k].termination, sums[k].num_iterations), k
                assert [r.step_is_successful for r in tk] == [r.step_is_successful for r in traces[k]], k
                assert np.abs(xk - xs[k]).max() < 1e-12, (k, np.abs(xk - xs[k]).max())
            assert xs[k][held_t(mask)].tobytes() == x[k][held_t(mask)].tobytes()
    ok = [k for k in range(len(x)) if sums[k].termination != 6]
    assert best == (min(ok, key=lambda k: (sums[k].final_cost, k)) if ok else -1)


def test_group_solve_equals_problem_solve(oracle):
    from camlasercalibratool_b200 import Group, default_options

    p = oracle.generate(60, 400, seed=9, sigma=0.01, with_edges=True)
    x0 = free_start(oracle, oracle.ground_truth()[1], 0, np.random.default_rng(4), 0.05)
    o = default_options(fixed=("ty", "rz"))
    with gpu(p) as g:
        x1, s1, t1 = g.solve(x0, o)
    with Group.from_arrays(p.frame_pose, p.offsets, p.points, p.edge_points, devices=(0,)) as grp:
        x2, s2, t2 = grp.solve(x0, o)
    assert x1.tobytes() == x2.tobytes() and [bytes(r) for r in t1] == [bytes(r) for r in t2]
    assert (s1.termination, s1.num_iterations, s1.final_cost) == (s2.termination, s2.num_iterations, s2.final_cost)


def test_bad_mask_is_rejected_on_a_real_problem(oracle):
    from camlasercalibratool_b200 import ClcError, default_options

    p = oracle.generate(20, 100, seed=1, sigma=0.01)
    with gpu(p) as g:
        x, s, _ = g.solve(X0)
        for mask in (63, 64, -1):
            o = default_options()
            o.fixed_mask = mask
            with pytest.raises(ClcError, match="fixed_mask"):
                g.solve(X0, o)
            with pytest.raises(ClcError, match="fixed_mask"):
                g.solve_starts(X0[None], o)
            with pytest.raises(ClcError, match="fixed_mask"):
                g.solve_segments([0, 20], X0[None], o)
        x2, s2, _ = g.solve(X0)  # the problem is untouched
        assert x.tobytes() == x2.tobytes()
