"""CPU tests of the time offset (clc_time_offset.cuh) that need no GPU: the product's CLC_HD code, compiled with g++
(tests/time_offset_harness.cpp), against the long-double and numpy restatements of tests/time_offset_reference.py.

* the interpolated plane and its td-derivative to 1e-12, the derivative against a central difference, knots 0, a few micro-
  radians and nearly pi apart, tau on a knot and clamped at both ends;
* expand_lm_td of the moments of random points against direct accumulation of the 7-column Jacobian, every loss kind;
* lm_update_td fed the reference's sums makes the numpy restatement's decisions and reaches its x8, every mask with bit 6;
* mask 0 on a board that never moves (td column identically 0) is the 6-column state machine.
"""
import numpy as np
import pytest

import exact_sums as X
import loss_reference as LR
import time_offset_reference as TR

LD = X.LD


@pytest.fixture(scope="module")
def TH(tmp_path_factory):
    return TR.TdHarness(tmp_path_factory.mktemp("td_harness"))


def _axis_angle_pose(axis, angle, t):
    axis = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    return np.concatenate([np.sin(angle / 2) * axis, [np.cos(angle / 2)], t])


def _knot_sets():
    rng = np.random.default_rng(5)
    sc = TR.scene(n_knots=12, seed=1)
    base = _axis_angle_pose([0.3, -0.2, 1.0], 0.4, [0.1, -0.2, 2.0])
    same = np.array([base, base, base])  # 0 degrees between knots
    small = np.array([base, _axis_angle_pose([0.3, -0.2, 1.0], 0.4 + 3e-6, [0.1, -0.2, 2.01]),
                      _axis_angle_pose([0.3, -0.2, 1.0], 0.4 + 9e-6, [0.1, -0.19, 2.02])])
    near_pi = np.array([_axis_angle_pose([1, 0, 0], 0.1, [0, 0, 2.0]), _axis_angle_pose([1, 0, 0], 0.1 + np.pi - 1e-7, [0, 0, 2.1]),
                        _axis_angle_pose([0, 1, 0], 0.3, [0, 0.1, 2.1])])
    near_pi[1, :4] *= -1.0  # the other sign of the same rotation: the slerp takes the shorter arc anyway
    scaled = sc.knot_poses.copy()
    scaled[:, :4] *= rng.uniform(0.5, 2.0, (len(scaled), 1))  # non-unit quaternions: the library normalises
    return {"motion": (sc.knot_times, sc.knot_poses), "scaled": (sc.knot_times, scaled),
            "zero_angle": (1.7e9 + np.array([0.0, 0.033, 0.07]), same),
            "small_angle": (np.array([0.0, 0.05, 0.1]), small), "near_pi": (np.array([0.0, 0.04, 0.08]), near_pi)}


@pytest.mark.parametrize("name", list(_knot_sets()))
def test_planes_and_derivatives(TH, name):
    kt, kp = _knot_sets()[name]
    t = kt - kt[0]
    span = t[-1]
    rng = np.random.default_rng(3)
    tau = np.concatenate([t, rng.uniform(0, span, 50), [-1e-3, -5.0, span + 1e-9, span + 2.0, np.nextafter(span, 0)]])
    P, D = TH.planes(kt, kp, tau)
    Pl, Dl = TR.planes_ld(kt, kp, tau)
    scale = np.maximum(1.0, np.abs(np.asarray(Dl, dtype=np.float64)).max())
    assert np.abs(P - np.asarray(Pl, dtype=np.float64)).max() < 1e-12, name
    assert np.abs(D - np.asarray(Dl, dtype=np.float64)).max() < 1e-12 * scale, name
    # clamped: the end knot's plane, no derivative; on a knot (u = 0): that knot's frame_plane
    out = (tau < 0) | (tau > span)
    assert not np.any(D[out]), name
    unit = kp.copy()
    unit[:, :4] /= np.linalg.norm(unit[:, :4], axis=1, keepdims=True)  # frame_plane takes the quaternion as it is
    for k in range(len(kt)):
        fp = np.asarray(X.frame_planes(unit[k:k + 1]), dtype=np.float64)[0]
        assert np.abs(P[k] - fp).max() < 1e-12, (name, k)
    for i in np.nonzero(tau < 0)[0]:
        assert P[i].tobytes() == TH.planes(kt, kp, [-10.0])[0][0].tobytes()
    # the derivative against a central difference of the long-double plane, away from the knots
    inner = rng.uniform(0, span, 20)
    k = np.clip(np.searchsorted(t, inner) - 1, 0, len(t) - 2)
    h = 1e-6 * (t[k + 1] - t[k])
    keep = (inner - h > t[k]) & (inner + h < t[k + 1])
    inner, h = inner[keep], h[keep]
    Pp, _ = TR.planes_ld(kt, kp, inner + h)
    Pm, _ = TR.planes_ld(kt, kp, inner - h)
    fd = np.asarray((Pp - Pm) / (2 * h.astype(LD))[:, None], dtype=np.float64)
    _, Dg = TH.planes(kt, kp, inner)
    assert np.abs(fd - Dg).max() < 1e-7 * scale, (name, np.abs(fd - Dg).max())


@pytest.mark.parametrize("kind", LR.KINDS)
def test_expansion_against_direct_accumulation(TH, kind):
    rng = np.random.default_rng(LR.KINDS.index(kind) + 11)
    x = TR.truth_pose7()
    for trial in range(6):
        n = rng.standard_normal(3)
        n /= np.linalg.norm(n)
        plane = np.concatenate([n, [rng.uniform(-3, 3)]])
        dplane = rng.standard_normal(4) * [0.5, 0.5, 0.5, 0.3]
        P = int(rng.integers(1, 300))
        pts = np.stack([rng.uniform(0.5, 4, P), rng.uniform(-2, 2, P), rng.normal(0, 0.1, P) if trial % 2 else np.zeros(P)], 1)
        # moments and cost term as the sweep forms them, in long double then rounded
        R, t = X._rot(np.asarray(x[3:], dtype=np.float64).astype(LD)), x[:3].astype(LD)
        pl = plane.astype(LD)
        m, c = pl[:3] @ R, pl[:3] @ t + pl[3]
        e = pts.astype(LD) @ m + c
        w, rho, _ = LR.weight_and_cost(kind, e, 0.05)
        pL = pts.astype(LD)
        S = np.array([w.sum(), *(w[:, None] * pL).sum(0), (w * pL[:, 0] ** 2).sum(), (w * pL[:, 0] * pL[:, 1]).sum(),
                      (w * pL[:, 0] * pL[:, 2]).sum(), (w * pL[:, 1] ** 2).sum(), (w * pL[:, 1] * pL[:, 2]).sum(),
                      (w * pL[:, 2] ** 2).sum()], dtype=LD)
        ct = rho.sum() / (LD(0.05) ** 2 if kind == "cauchy" else 1)
        got = TH.expand(plane, dplane, x, P, S.astype(np.float64), kind, float(ct), 0.05)
        val, mag = TR.td_sums(plane[None].astype(LD), dplane[None].astype(LD), [0, P], pts, x, None, kind)
        X.assert_within(got, val, mag, TR.GROUPS_TD, f"{kind} trial {trial}")


MASKS_TD = [0, 1 << 6, 0b0111111, 0b1000011, 0b1101000, 0b0000110]


def _decisions(trace):
    return [bool(t.step_is_successful) for t in trace]


@pytest.mark.parametrize("mask", MASKS_TD)
@pytest.mark.parametrize("case", ["noisy_cauchy", "noise_free_none", "noisy_huber"])
def test_lm_makes_the_restatements_decisions(TH, mask, case):
    kind = {"noisy_cauchy": "cauchy", "noise_free_none": "none", "noisy_huber": "huber"}[case]
    sigma = 0.0 if case == "noise_free_none" else 0.005
    sc = TR.scene(n_knots=40, beams=40, sigma=sigma, seed=len(case), td_true=0.011, motion=2.0)
    rng = np.random.default_rng(mask + 3)
    gt = TR.truth_pose7()
    d = 0.02 * rng.standard_normal(6)
    d[[k for k in range(6) if mask >> k & 1]] = 0.0
    from oracle import oracle_np as ONP

    x0 = ONP.pose_plus(gt, d)
    td0 = 0.0 if not mask >> 6 & 1 else 0.011
    x, done, tr = TH.lm_run(lambda y: TR.sums_at(sc, y, kind), x0, td0, TH.default_options(fixed_mask=mask))
    xn, term, trn = TR.solve7(sc, x0, td0, kind, fixed_mask=mask)
    names = {1: "CONVERGENCE_FUNCTION", 2: "CONVERGENCE_PARAMETER", 3: "CONVERGENCE_GRADIENT", 4: "CONVERGENCE_MIN_RADIUS",
             5: "NO_CONVERGENCE", 6: "FAILURE"}
    assert names[done] == term, (case, mask, done, term)
    assert len(trn) in (len(tr), len(tr) - 1)  # the restatement records no row for a tolerance that stops on a candidate
    assert [r["ok"] for r in trn] == _decisions(tr)[:len(trn)], (case, mask)
    assert np.abs(x - xn).max() < 1e-12, (case, mask, x - xn)
    if mask >> 6 & 1:
        assert x[7] == td0
    for k in range(3):
        if mask >> k & 1:
            assert x[k] == x0[k]


def test_mask_zero_static_board_is_the_six_column_solve(TH, harness):
    """A board that never moves: the td column is identically 0, and the 7-column machine reproduces the 6-column one's poses,
    decisions and termination bit for bit."""
    sc = TR.scene(n_knots=6, beams=50, sigma=0.004, static=True, seed=9)
    from oracle import oracle_np as ONP

    x0 = ONP.pose_plus(TR.truth_pose7(), 0.03 * np.random.default_rng(2).standard_normal(6))
    cache = {}

    def sums36(y):
        key = y.tobytes()
        if key not in cache:
            cache[key] = TR.sums_at(sc, y, "cauchy")
        return cache[key]

    probe = sums36(np.concatenate([x0, [0.0]]))
    td_entries = [k for k, (i, j) in enumerate(zip(*TR.IU7)) if j == 6] + [34]
    assert not np.any(probe[td_entries])
    six = [k for k, (i, j) in enumerate(zip(*TR.IU7)) if j < 6]

    def sums28(y7):
        s = sums36(np.concatenate([y7, [0.0]]))
        return np.concatenate([s[six], s[28:34], [s[35]]])

    x7, done7, tr7, _ = harness.lm_run(sums28, x0)
    x8, done8, tr8 = TH.lm_run(sums36, x0, 0.0, TH.default_options())
    assert done7 == done8 and len(tr7) == len(tr8)
    assert x8[:7].tobytes() == x7.tobytes() and x8[7] == 0.0
    assert [bytes(a) for a in tr7] == [bytes(b) for b in tr8]
