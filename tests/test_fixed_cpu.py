"""CPU tests of held extrinsic coordinates (clc_lm_options.fixed_mask) that need no GPU:

* the host build of lm_update (tests/host_harness.cpp, the source the device runs), fed the C oracle's sums at its own
  candidates, makes the decisions of the reduced-parameterization C oracle's Cholesky and Householder-QR solves
  (tests/fixed_oracle.c) and of the numpy twin (fixed_reference.solve_fixed, an independent restatement through
  oracle_np.trust_region_lm): every single-bit mask and a few multi-bit ones, on random problems and on the reference's
  degenerate teaching geometries.  Held translations keep their bits;
* mask 0 is the unmasked solve: byte for byte in lm_update, and the reduced oracle with nothing held is the main oracle;
* the C entry points reject a mask with bits above 5 or with all six bits set, before anything else;
* the coordinate names of default_options(fixed=...).
"""
import ctypes as C

import numpy as np
import pytest

import fixed_reference as FR
from conftest import pack_sums
from test_gpu_degenerate import simulate

NAMES = ("tx", "ty", "tz", "rx", "ry", "rz")
MASKS = [1 << k for k in range(6)] + [0b000111, 0b111000, 0b011010, 0b100001]  # singles, {tx,ty,tz}, {rx,ry,rz}, {ty,rx,ry}, {tx,rz}


@pytest.fixture(scope="module")
def FO(tmp_path_factory):
    return FR.FixedOracle(tmp_path_factory.mktemp("fixed_oracle"))


def harness_solve(harness, oracle, p, x0, mask):
    return harness.lm_run(lambda x: pack_sums(*oracle.evaluate_normal(p, x)), x0, harness.default_options(fixed_mask=mask))


def decisions(trace):
    return [(int(t.step_is_valid), int(t.step_is_successful)) for t in trace]


def free_start(oracle, x, mask, rng, s):
    """x moved by a random increment in the free coordinates only (held ones keep x's values)."""
    d = s * rng.standard_normal(6)
    d[[k for k in range(6) if mask >> k & 1]] = 0.0
    return oracle.pose_plus(x, d)


def check_against_oracles(harness, oracle, oracle_np, FO, p, x0, mask, ctx):
    x, done, tr, _ = harness_solve(harness, oracle, p, x0, mask)
    held_t = [k for k in range(3) if mask >> k & 1]
    assert x[held_t].tobytes() == np.asarray(x0)[held_t].tobytes(), ctx
    for solver in (1, 0):  # the C oracle's Cholesky, then its Householder QR of [J_s; D], both on the free columns
        xo, so, tro = FO.solve(p, x0, mask, linear_solver=solver)
        c = f"{ctx} solver={solver}"
        assert done == so.termination and len(tr) == so.num_iterations, (c, done, so.termination, len(tr), so.num_iterations)
        assert decisions(tr) == [(t.step_is_valid, t.step_is_successful) for t in tro], c
        assert np.abs(x - xo).max() < 1e-9, (c, x - xo)
        assert xo[held_t].tobytes() == np.asarray(x0)[held_t].tobytes(), c
    # the numpy twin: the reduced parameterization restated through trust_region_lm
    table = oracle_np.residual_table(p.frame_pose, p.offsets, p.points, p.edge_points)
    xn, term, trn = FR.solve_fixed(lambda y: oracle_np.evaluate(table, y, p.use_loss, p.cauchy_a), x0, mask)
    assert term == oracle.TERMINATION[done], (ctx, term)
    assert len(trn) in (len(tr), len(tr) - 1), ctx  # the twin records no row for a tolerance that stops on a candidate
    assert [r["ok"] for r in trn] == [bool(t.step_is_successful) for t in tr[:len(trn)]], ctx
    assert np.abs(xn - x).max() < 1e-9, (ctx, xn - x)
    return x, done, tr


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("seed", [2, 7])
def test_host_lm_update_makes_the_reduced_oracles_decisions(harness, oracle, oracle_np, FO, mask, seed):
    p = oracle.generate(30, 120, seed=seed, sigma=0.01, with_edges=seed == 7)
    gt = oracle.ground_truth()[1]
    rng = np.random.default_rng(seed)
    for i, x0 in enumerate([np.array([0, 0, 0, 0, 0, 0, 1.0]), free_start(oracle, gt, 0, rng, 0.05)]):
        check_against_oracles(harness, oracle, oracle_np, FO, p, x0, mask, f"mask={mask} seed={seed} start={i}")


@pytest.mark.parametrize("variant,mask", [("only_roll", 0b000001), ("only_pitch", 0b011010)])
@pytest.mark.parametrize("seed,centred", [(3, False), (11, True)])
def test_degenerate_geometries_become_well_posed(harness, oracle, oracle_np, FO, variant, mask, seed, centred):
    """With the coordinates the null space names held at the truth's values, the solve on the reference's degenerate
    geometries is well posed: all three restatements agree, and noise-free data reach the truth."""
    gt = oracle.ground_truth()[1]
    rng = np.random.default_rng(seed)
    for sigma in (0.0, 0.01):
        p = simulate(oracle, variant, seed=seed, sigma=sigma, centred=centred)
        x0 = free_start(oracle, gt, mask, rng, 0.05)
        x, done, _ = check_against_oracles(harness, oracle, oracle_np, FO, p, x0, mask, f"{variant} sigma={sigma}")
        assert done != 6
        if sigma == 0.0:
            # Ceres stops once a step is shorter than parameter_tolerance * |x| (1e-8 * ~1.1 here) and does not apply it
            ang, dt = oracle.pose_error(x, gt)
            assert ang < 2e-8 and dt < 2e-8, (variant, ang, dt)


def test_mask_zero_is_the_unmasked_solve(harness, oracle, FO):
    p = oracle.generate(40, 150, seed=4, sigma=0.01)
    x0 = np.array([0, 0, 0, 0, 0, 0, 1.0])
    sums = lambda x: pack_sums(*oracle.evaluate_normal(p, x))  # noqa: E731
    a = harness.lm_run(sums, x0)
    b = harness.lm_run(sums, x0, harness.default_options(fixed_mask=0))
    assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1] and a[3] == b[3]
    assert [bytes(t) for t in a[2]] == [bytes(t) for t in b[2]]
    for solver in (0, 1):  # with nothing held the reduced oracle is the main oracle, solver for solver
        xo, so, tro = oracle.solve(p, x0, oracle.default_options(linear_solver=solver))
        xz, sz, trz = FO.solve(p, x0, 0, linear_solver=solver)
        assert (sz.termination, sz.num_iterations) == (so.termination, so.num_iterations), solver
        assert decisions(trz) == [(t.step_is_valid, t.step_is_successful) for t in tro], solver
        assert np.abs(xz - xo).max() < 1e-12, (solver, xz - xo)
    xo, so, tro = oracle.solve(p, x0)
    assert a[1] == so.termination and len(a[2]) == so.num_iterations and np.abs(a[0] - xo).max() < 1e-9


@pytest.mark.parametrize("mask", [63, 64, 127, 1 << 20, -1])
def test_abi_rejects_bad_masks_first(mask):
    from camlasercalibratool_b200 import _lib
    from camlasercalibratool_b200.api import default_options

    L = _lib.load()
    o = default_options()
    o.fixed_mask = mask
    x = np.array([0, 0, 0, 0, 0, 0, 1.0])
    dp = x.ctypes.data_as(C.POINTER(C.c_double))
    off = np.array([0, 0], dtype=np.int64).ctypes.data_as(C.POINTER(C.c_int64))
    best = C.c_int64()
    calls = {
        "clc_solve_lm": lambda opt: L.clc_solve_lm(None, dp, opt, None, None, 0),
        "clc_group_solve_lm": lambda opt: L.clc_group_solve_lm(None, dp, opt, None, None, 0),
        "clc_solve_lm_segments": lambda opt: L.clc_solve_lm_segments(None, 1, off, dp, opt, None, None, 0),
        "clc_solve_lm_starts": lambda opt: L.clc_solve_lm_starts(None, 1, dp, opt, None, None, 0, C.byref(best)),
    }
    for name, call in calls.items():
        assert call(C.byref(o)) == 1, name
        assert b"fixed_mask" in L.clc_last_error(), (name, L.clc_last_error())
        ok = default_options()
        ok.fixed_mask = 62
        assert call(C.byref(ok)) == 1, name  # the NULL problem, now
        assert b"fixed_mask" not in L.clc_last_error(), (name, L.clc_last_error())


def test_default_options_names():
    from camlasercalibratool_b200 import default_options

    assert default_options().fixed_mask == 0
    assert default_options(fixed=()).fixed_mask == 0
    assert default_options(fixed=("ty", "rx")).fixed_mask == 0b001010
    assert default_options(fixed="tz").fixed_mask == 0b000100
    for k, n in enumerate(NAMES):
        assert default_options(fixed=[n]).fixed_mask == 1 << k
    assert default_options(fixed=("rx", "ry", "rz"), max_num_iterations=7).max_num_iterations == 7
    assert default_options(fixed=NAMES[:5]).fixed_mask == 31
    for bad in (("tx", "yaw"), ("TX",), ("x",), NAMES):
        with pytest.raises(ValueError):
            default_options(fixed=bad)
