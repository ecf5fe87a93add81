"""Greedy D-optimal frame selection (clc_select_frames, clc_select_frames_rows, clc_group_select_frames) on the GPU.

1. Known answers through the rows path: diagonal blocks (closed-form gains), exact duplicates, NaN and zero rows, forced frames,
   the three stop rules, a coordinate without information (held or not), and 0 or 1 frames and budget 0.
2. Problem.select_frames equals the rows path on the problem's own report, byte for byte, and two calls do too: both kernel
   families, with and without edge residuals.
3. On synthetic problems with noise and a camera chain (2 000 frames, budget 300, Cauchy and no loss, with and without held
   coordinates) every device pick is the long-double maximum of its step within 1e-10 (1 + g), its gain matches, and the pick
   sequence equals the float64 reference up to the reference's first near tie.
4. The same at 10^5 frames for the first 200 steps.
5. Pipeline: 30 of 2 000 noise-free frames solve to the ground truth and have a full-rank information matrix.
6. A group of two devices returns the rows path's bytes on the group's report and the single-device picks.
"""
import contextlib
import os

import numpy as np
import pytest

import select_reference as SR

pytestmark = pytest.mark.gpu

FAMILIES = {"general": dict(CLC_PLANAR="0"), "planar": dict(CLC_PLANAR="1", CLC_PLANAR_MIN_POINTS="0")}
RTOL = 1e-10


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


def rows_of(H):
    """FRAME_ROW_DTYPE rows holding the blocks H [n, 6, 6] (every other field 0)."""
    from camlasercalibratool_b200 import FRAME_ROW_DTYPE

    rows = np.zeros(len(H), dtype=FRAME_ROW_DTYPE)
    rows["H21"] = SR.pack(np.asarray(H, dtype=np.float64)) if len(H) else np.zeros((0, 21))
    return rows


def sel_rows(rows, budget, **kw):
    from camlasercalibratool_b200 import select_frames_from_report

    return select_frames_from_report(rows, budget, device=0, **kw)


def same_bytes(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes() for x, y in zip(a, b))


def near_truth(oracle, scale=1e-3):
    return oracle.pose_plus(oracle.ground_truth()[1], scale * np.array([1.0, -0.7, 0.4, -1.0, 0.6, 0.3]))


# ---- 1. known answers --------------------------------------------------------------------------------------------------------
def _diag_rows(rng, n):
    d = rng.permutation(n * 6).reshape(n, 6) + 1.0  # distinct positive values
    H = np.zeros((n, 6, 6))
    H[:, np.arange(6), np.arange(6)] = d
    return d, H


def test_diagonal_blocks_closed_form():
    rng = np.random.default_rng(1)
    n, budget = 40, 12
    diag, H = _diag_rows(rng, n)
    sel = sel_rows(rows_of(H), budget)
    T = diag.sum(axis=0)
    ht = diag / T
    a = np.full(6, SR.RIDGE / n)
    rem = list(range(n))
    for s in range(budget):
        g = np.array([np.sum(np.log1p(ht[f] / a)) for f in rem])
        k = int(np.argmax(g))
        assert sel.order[s] == rem[k], s
        assert abs(sel.gain[s] - g[k]) <= 1e-12 * abs(g[k]), s
        a = a + ht[rem[k]]
        rem.pop(k)
    assert len(sel.order) == budget and sel.keep.sum() == budget and np.all(sel.keep[sel.order])


def test_duplicates_lowest_index_wins():
    # dyadic values: T is exact in any summation order, so the duplicates' gains are equal bit for bit wherever they sit
    H = np.zeros((10, 6, 6))
    for f in range(10):
        H[f][np.arange(6), np.arange(6)] = 2.0 ** -(f % 4)
    H[3] = H[7] = np.diag([4.0, 4.0, 4.0, 4.0, 4.0, 4.0])
    sel = sel_rows(rows_of(H), 1)
    assert sel.order.tolist() == [3]
    rev = sel_rows(rows_of(H[::-1].copy()), 1)
    assert rev.order.tolist() == [9 - 7]
    assert rev.gain.tobytes() == sel.gain.tobytes()


def test_nan_and_zero_rows():
    rng = np.random.default_rng(2)
    _, H = _diag_rows(rng, 12)
    H[4] = 1e6 * np.eye(6)
    H[4, 2, 3] = H[4, 3, 2] = np.nan
    H[6] = 0.0
    H[9] = 0.0
    sel = sel_rows(rows_of(H), 50)
    assert 4 not in sel.order and 6 not in sel.order and 9 not in sel.order
    assert len(sel.order) == 9  # every other frame adds information; then only zero rows are left
    excl = np.ones(12, dtype=bool)
    excl[4] = False
    ref = sel_rows(rows_of(np.where(np.arange(12)[:, None, None] == 4, 0.0, H)), 50, candidates=excl)
    assert same_bytes(sel, ref)  # the NaN row is never summed: as if it were excluded with zeros


def test_forced_frames():
    rng = np.random.default_rng(3)
    _, H = _diag_rows(rng, 30)
    H += 0.3 * np.einsum("fi,fj->fij", rng.standard_normal((30, 6)), rng.standard_normal((30, 6)))
    H = 0.5 * (H + H.transpose(0, 2, 1)) + 40 * np.eye(6)
    forced = np.zeros(30, dtype=bool)
    forced[[2, 11, 17]] = True
    sel = sel_rows(rows_of(H), 8, forced=forced)
    assert not np.any(forced[sel.order])
    assert np.all(sel.keep[forced]) and sel.keep.sum() == 3 + len(sel.order)
    state = np.where(forced, 2, 1).astype(np.uint8)
    order, gain, keep, _ = SR.greedy(SR.pack(H), 8, state=state)
    assert sel.order.tolist() == order.tolist()
    assert np.all(np.abs(sel.gain - gain) <= 1e-12 * np.abs(gain))
    free = sel_rows(rows_of(H), 8)
    assert free.gain[0] > sel.gain[0]  # forced frames already count


def test_stop_rules():
    rng = np.random.default_rng(4)
    _, H = _diag_rows(rng, 20)
    full = sel_rows(rows_of(H), 100)
    assert len(full.order) == 20  # exhausted: budget above the candidates
    five = sel_rows(rows_of(H), 5)
    assert five.order.tolist() == full.order[:5].tolist() and same_bytes((five.gain,), (full.gain[:5],))
    cut = 0.5 * (full.gain[6] + full.gain[7])
    early = sel_rows(rows_of(H), 100, min_gain=cut)
    assert len(early.order) == int(np.sum(full.gain > cut))
    cand = np.zeros(20, dtype=bool)
    cand[[1, 5, 8]] = True
    few = sel_rows(rows_of(H), 100, candidates=cand)
    assert sorted(few.order.tolist()) == [1, 5, 8] and few.keep.sum() == 3


def test_coordinate_without_information():
    from camlasercalibratool_b200 import ClcError

    rng = np.random.default_rng(5)
    _, H = _diag_rows(rng, 15)
    H += 0.2 * np.einsum("fi,fj->fij", rng.standard_normal((15, 6)), rng.standard_normal((15, 6)))
    H = 0.5 * (H + H.transpose(0, 2, 1)) + 20 * np.eye(6)
    H[:, 2, :] = 0.0
    H[:, :, 2] = 0.0
    with pytest.raises(ClcError, match="tz"):
        sel_rows(rows_of(H), 5)
    with pytest.raises(SR.NoInformation):
        SR.prepare(SR.pack(H))
    sel = sel_rows(rows_of(H), 5, fixed=("tz",))
    order, gain, _, _ = SR.greedy(SR.pack(H), 5, mask=0b100)
    assert sel.order.tolist() == order.tolist()
    assert np.all(np.abs(sel.gain - gain) <= 1e-12 * np.abs(gain))


def test_edge_sizes():
    empty = sel_rows(rows_of(np.zeros((0, 6, 6))), 10)
    assert empty.order.size == 0 and empty.gain.size == 0 and empty.keep.size == 0
    one = sel_rows(rows_of(np.eye(6)[None]), 10)
    assert one.order.tolist() == [0] and one.keep.tolist() == [True] and one.gain[0] > 0
    rng = np.random.default_rng(6)
    _, H = _diag_rows(rng, 8)
    forced = np.zeros(8, dtype=bool)
    forced[3] = True
    none = sel_rows(rows_of(H), 0, forced=forced)
    assert none.order.size == 0 and none.keep.tolist() == forced.tolist()


def test_invalid_arguments_before_device_work():
    import ctypes as C

    from camlasercalibratool_b200 import _lib, launch_count
    from camlasercalibratool_b200._lib import SelectDesc

    L = _lib.load()
    rows = rows_of(np.eye(6)[None].repeat(4, axis=0))
    n_sel = C.c_int64()
    order, gain, keep = np.zeros(4, dtype=np.int64), np.zeros(4), np.zeros(4, dtype=np.uint8)
    st = np.array([1, 3, 1, 1], dtype=np.uint8)
    n0 = launch_count()
    for budget, min_gain, mask, state in ((-1, 0.0, 0, None), (2, float("nan"), 0, None), (2, -1.0, 0, None),
                                          (2, float("inf"), 0, None), (2, 0.0, 63, None), (2, 0.0, 64, None), (2, 0.0, -1, None),
                                          (2, 0.0, 0, st)):
        d = SelectDesc()
        d.budget, d.min_gain, d.fixed_mask = budget, min_gain, mask
        d.state = st.ctypes.data_as(C.POINTER(C.c_uint8)) if state is not None else None
        rc = L.clc_select_frames_rows(0, 4, rows.ctypes.data_as(C.c_void_p), C.byref(d), C.byref(n_sel),
                                      order.ctypes.data_as(_lib.c_int64_p), gain.ctypes.data_as(_lib.c_double_p),
                                      keep.ctypes.data_as(C.POINTER(C.c_uint8)))
        assert rc == 1, (budget, min_gain, mask)
    assert launch_count() == n0


# ---- 2. same rows, same answer -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("edges", [False, True])
def test_problem_equals_rows_path(oracle, family, edges):
    from camlasercalibratool_b200 import Problem, select_frames_from_report

    x = near_truth(oracle)
    with env(**FAMILIES[family]), Problem.synthetic(600, 400, seed=3, sigma=0.01, with_edges=edges, device=0) as p:
        a = p.select_frames(x, 60)
        b = p.select_frames(x, 60)
        c = select_frames_from_report(p.frame_report(x), 60, device=0)
        assert len(a.order) == 60
        assert same_bytes(a, b) and same_bytes(a, c)
        forced = np.arange(600) % 50 == 0
        d = p.select_frames(x, 30, forced=forced, fixed=("rz",), min_gain=1e-3)
        e = select_frames_from_report(p.frame_report(x), 30, forced=forced, fixed=("rz",), min_gain=1e-3, device=0)
        assert same_bytes(d, e)


# ---- 3. / 4. the greedy rule on real data ------------------------------------------------------------------------------------
def _check_real(p, x, budget, fixed=(), steps=None):
    from camlasercalibratool_b200.api import FIXED_NAMES

    sel = p.select_frames(x, budget, fixed=fixed)
    H21 = p.frame_report(x)["H21"]
    mask = sum(1 << FIXED_NAMES.index(k) for k in fixed)
    n_check = len(sel.order) if steps is None else steps
    SR.check_picks(H21, sel.order, sel.gain, budget, mask=mask, steps=steps, rtol=RTOL)
    ref_order, ref_gain, _, ref_sep = SR.greedy(H21, n_check, mask=mask)
    compared = SR.agreeing_prefix(sel.order[:n_check], ref_order, ref_sep, RTOL, ref_gain)
    return sel, compared


@pytest.mark.parametrize("loss", ["cauchy", "none"])
@pytest.mark.parametrize("fixed", [(), ("tz", "rx")])
def test_greedy_rule_on_real_data(oracle, loss, fixed):
    from camlasercalibratool_b200 import Problem

    x = near_truth(oracle, 1e-2)
    with Problem.synthetic(2000, 200, seed=7, sigma=0.01, camera="radtan", pixel_sigma=0.5, device=0) as p:
        p.set_loss(loss if loss != "none" else None)
        sel, compared = _check_real(p, x, 300, fixed)
    assert len(sel.order) == 300
    assert compared >= 20, compared


def test_greedy_rule_at_scale(oracle):
    from camlasercalibratool_b200 import Problem

    x = near_truth(oracle, 1e-2)
    with Problem.synthetic(100_000, 100, seed=11, sigma=0.01, device=0) as p:
        sel, compared = _check_real(p, x, 200, steps=200)
    assert len(sel.order) == 200
    assert compared >= 20, compared


# ---- 5. pipeline -------------------------------------------------------------------------------------------------------------
def test_pipeline_select_subset_solve(oracle):
    from camlasercalibratool_b200 import Problem, default_options

    gt = oracle.ground_truth()[1]
    x0 = near_truth(oracle, 1e-2)
    opt = default_options(function_tolerance=1e-20, parameter_tolerance=1e-20, gradient_tolerance=1e-30)
    with Problem.synthetic(2000, 200, seed=5, sigma=0.0, device=0) as p:
        sel = p.select_frames(x0, 30)
        assert len(sel.order) == 30 and sel.keep.sum() == 30
        with p.subset(sel.keep) as q:
            x, s, _ = q.solve(x0, opt)
            _, _, _, sv = q.information(x)
    ang, dt = oracle.pose_error(x, gt)
    assert ang < 1e-9 and dt < 1e-9, (ang, dt, s.termination)
    assert np.all(sv > 1e-8), sv


# ---- 6. group ----------------------------------------------------------------------------------------------------------------
def test_group_of_two_devices(oracle):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    from camlasercalibratool_b200 import Group, Problem, select_frames_from_report

    x = near_truth(oracle, 1e-2)
    with Group.synthetic(1500, 200, seed=9, sigma=0.01, devices=(0, 1)) as g:
        a = g.select_frames(x, 100)
        b = select_frames_from_report(g.frame_report(x), 100, device=0)
        assert same_bytes(a, b)
    with Problem.synthetic(1500, 200, seed=9, sigma=0.01, device=0) as p:
        H21 = p.frame_report(x)["H21"]
        c = p.select_frames(x, 100)
    _, _, _, sep = SR.greedy(H21, 100)
    n = SR.agreeing_prefix(a.order, c.order, sep, 1e-8)
    assert n >= 20, n
