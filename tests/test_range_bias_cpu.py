"""CPU tests of the range bias (clc_range_bias.cuh) that need no GPU: the product's CLC_HD code, compiled with g++
(tests/range_bias_harness.cpp), against the long-double and numpy restatements of tests/range_bias_reference.py.

* expand_lm_range of the 25 moments of random points against direct accumulation of the 8-column Jacobian, every loss kind,
  within GAMMA * A_k; a point at r == 0 and a NaN coordinate;
* lm_update<8> fed the reference's sums makes the numpy restatement's decisions and reaches its x9, for several masks;
* b = s = 0 with both held is the 6-column state machine: the same decisions and a pose that agrees to 1e-12.
"""
import math

import numpy as np
import pytest

import exact_sums as X
import loss_reference as LR
import range_bias_reference as RB

LD = X.LD


@pytest.fixture(scope="module")
def RH(tmp_path_factory):
    return RB.RbHarness(tmp_path_factory.mktemp("rb_harness"))


def _piece(rng, planar, P):
    pts = np.stack([rng.uniform(0.5, 4, P), rng.uniform(-2, 2, P), np.zeros(P) if planar else rng.normal(0, 0.3, P)], 1)
    n = rng.standard_normal(3)
    n /= np.linalg.norm(n)
    return pts, np.concatenate([n, [rng.uniform(-3, 3)]])


def _expand_ld(RH, plane, pts, x, b, s, kind):
    """(got, ref, mag): the harness's expansion of the long-double moments against direct accumulation."""
    e, _, _, _, _, _ = RB.residuals_ld(plane, pts, x, b, s)
    w, rho, _ = LR.weight_and_cost(kind, e, 0.05)
    M = RB.moments25(pts, w)
    ct = rho.sum() / (LD(0.05) ** 2 if kind == "cauchy" else 1)
    got = RH.expand(plane, x, b, s, len(pts), M.astype(np.float64), kind, float(ct), 0.05)
    val, mag = RB.rb_sums(plane[None], [0, len(pts)], pts, x, b, s, kind)
    return got, val, mag


@pytest.mark.parametrize("kind", LR.KINDS)
def test_expansion_against_direct_accumulation(RH, kind):
    rng = np.random.default_rng(LR.KINDS.index(kind) + 31)
    x = RB.truth_pose7()
    for trial in range(8):
        pts, plane = _piece(rng, trial % 2 == 0, int(rng.integers(1, 300)))
        b, s = (0.0, 0.0) if trial < 2 else (rng.uniform(-0.05, 0.05), rng.uniform(-0.02, 0.02))
        got, val, mag = _expand_ld(RH, plane, pts, x, b, s, kind)
        X.assert_within(got, val, mag, RB.GROUPS_RB, f"{kind} trial {trial}")


def test_origin_point(RH):
    """r == 0: the p / r terms are 0, kappa p = 0 -- the point contributes e = c, J = [n, 0, 0, 0]."""
    rng = np.random.default_rng(4)
    pts, plane = _piece(rng, False, 20)
    pts[3] = 0.0
    x = RB.truth_pose7()
    got, val, mag = _expand_ld(RH, plane, pts, x, 0.03, 0.01, "cauchy")
    X.assert_within(got, val, mag, RB.GROUPS_RB, "origin")
    assert RH.L.rb_kappa(0.0, 0.0, 0.0, 0.03, 0.01) == 1.01
    assert RH.L.rb_kappa(3.0, 4.0, 0.0, 0.5, 0.0) == 1.1


def test_nan_propagates(RH):
    rng = np.random.default_rng(6)
    pts, plane = _piece(rng, False, 10)
    M = RB.moments25(pts, np.ones(len(pts))).astype(np.float64)
    M[1] = np.nan
    got = RH.expand(plane, RB.truth_pose7(), 0.01, 0.0, len(pts), M, "none", 1.0, 0.05)
    assert np.isnan(got).any()
    assert math.isnan(RH.L.rb_kappa(np.nan, 1.0, 0.0, 0.01, 0.0))


MASKS_RB = [0, 1 << 7, (1 << 6) | (1 << 7), 0b00111111, 0b10000011, 0b01001000]
NAMES = {1: "CONVERGENCE_FUNCTION", 2: "CONVERGENCE_PARAMETER", 3: "CONVERGENCE_GRADIENT", 4: "CONVERGENCE_MIN_RADIUS",
         5: "NO_CONVERGENCE", 6: "FAILURE"}


@pytest.mark.parametrize("mask", MASKS_RB)
@pytest.mark.parametrize("case", ["noisy_cauchy", "noise_free_none"])
def test_lm_makes_the_restatements_decisions(RH, mask, case):
    kind = "cauchy" if case == "noisy_cauchy" else "none"
    sc = RB.scene(n_frames=24, beams=40, sigma=0.0 if kind == "none" else 0.003, seed=len(case))
    rng = np.random.default_rng(mask + 3)
    from oracle import oracle_np as ONP

    d = 0.02 * rng.standard_normal(6)
    d[[k for k in range(6) if mask >> k & 1]] = 0.0
    x0 = np.concatenate([ONP.pose_plus(sc.pose7, d), [0.0 if not mask >> 6 & 1 else sc.b, 0.0 if not mask >> 7 & 1 else sc.s]])
    x, done, tr = RH.lm_run(lambda y: RB.sums_at(sc, y, kind), x0, RH.default_options(fixed_mask=mask))
    xn, term, trn = RB.solve8(sc, x0, kind, fixed_mask=mask)
    assert NAMES[done] == term, (case, mask, done, term)
    assert len(trn) in (len(tr), len(tr) - 1)
    assert [r["ok"] for r in trn] == [bool(t.step_is_successful) for t in tr][:len(trn)], (case, mask)
    assert np.abs(x - xn).max() < 1e-10, (case, mask, x - xn)
    for k in (0, 1, 2):
        if mask >> k & 1:
            assert x[k] == x0[k]
    for k in (6, 7):
        if mask >> k & 1:
            assert x[k + 1] == x0[k + 1]


def test_held_zero_bias_is_the_six_column_solve(RH, harness):
    """b = s = 0, both held: the 8-column machine makes the 6-column one's decisions and reaches its pose to 1e-12."""
    sc = RB.scene(n_frames=20, beams=50, b=0.0, s=0.0, sigma=0.004, seed=9)
    from oracle import oracle_np as ONP

    x0 = ONP.pose_plus(sc.pose7, 0.03 * np.random.default_rng(2).standard_normal(6))
    six = [k for k, (i, j) in enumerate(zip(*RB.IU8)) if j < 6]

    def sums28(y7):
        s = RB.sums_at(sc, np.concatenate([y7, [0.0, 0.0]]), "cauchy")
        return np.concatenate([s[six], s[36:42], [s[44]]])

    x7, done7, tr7, _ = harness.lm_run(sums28, x0)
    x9, done9, tr9 = RH.lm_run(lambda y: RB.sums_at(sc, y, "cauchy"), np.concatenate([x0, [0.0, 0.0]]),
                               RH.default_options(fixed_mask=(1 << 6) | (1 << 7)))
    assert done7 == done9 and len(tr7) == len(tr9)
    assert [bool(t.step_is_successful) for t in tr7] == [bool(t.step_is_successful) for t in tr9]
    assert np.abs(x9[:7] - x7).max() < 1e-12 and x9[7] == 0.0 and x9[8] == 0.0


def test_python_checks_run_before_the_library():
    from camlasercalibratool_b200 import api

    assert api.range_bias_mask(("range_offset", "tz")) == (1 << 6) | (1 << 2)
    assert api.range_bias_mask("range_scale") == 1 << 7
    with pytest.raises(ValueError):
        api.range_bias_mask(api.RANGE_BIAS_NAMES)
    with pytest.raises(ValueError):
        api.range_bias_mask("td")
    with pytest.raises(ValueError):
        api._pose_bias(np.zeros(7), (0.0,))
    with pytest.raises(ValueError):
        api._pose_bias(np.zeros(7), (np.nan, 0.0))
    with pytest.raises(ValueError):
        api._pose_bias(np.zeros(6), (0.0, 0.0))
