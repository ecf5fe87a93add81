"""Every entry point returns the device scratch it allocates: the bytes in use in the device's default memory pool (which every
call's stream-ordered scratch comes from) are the same before and after a call, when it succeeds and when it is rejected.

The first call of each pair is a warm-up, so that what a problem keeps for its life (the L2 flush buffer of the bench hooks,
events) exists before the count is taken."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import time_offset_reference as TR

pytestmark = pytest.mark.gpu

CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7  # cuda.h, CUmemPool_attribute
X0 = np.array([0, 0, 0, 0, 0, 0, 1.0])


def _pool_used(device=0):
    import torch

    torch.cuda.synchronize(device)
    cu = C.CDLL("libcuda.so.1")
    dev, pool, used = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuDeviceGet(C.byref(dev), device) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT, C.byref(used)) == 0
    return used.value


def _no_scratch_left(name, call):
    call()
    before = _pool_used()
    call()
    assert _pool_used() == before, f"{name} left device scratch allocated"


def _rejected(call, code=None):
    """call() through the C ABI, which must return an error status (code, when given)"""
    def run():
        rc = call()
        assert rc != 0 and (code is None or rc == code), rc
    return run


def _close(p):
    p.close()


@pytest.fixture(scope="module", params=["K2", "K1"])
def problem(request):
    from camlasercalibratool_b200 import Problem

    # K2: the reference's size (the one-cluster kernel serves it); K1: the sweep kernel's multi-block size
    n_frames, beams = (50, 180) if request.param == "K2" else (700, 1000)
    with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01, device=0) as p:
        yield p


def test_problem_entry_points_free_their_scratch(problem):
    p = problem
    N = p.sizes()[0]
    seg = np.array([0, N // 3, N], dtype=np.int64)
    seg_poses = np.tile(X0, (2, 1))
    starts = np.tile(X0, (4, 1))
    starts[1:, :3] += np.array([[0.01, 0, 0], [0, 0.01, 0], [0, 0, 0.01]])
    keep = np.ones(N, dtype=bool)
    keep[::3] = False
    q = [0.1, 0.5, 0.9]
    calls = {
        "eval": lambda: p.eval(X0),
        "information": lambda: p.information(X0),
        "closed_form": lambda: p.closed_form(),
        "solve": lambda: p.solve(X0),
        "download": lambda: p.download(),
        "line_fit": lambda: p.line_fit(),
        "frame_report": lambda: p.frame_report(X0),
        "select_frames": lambda: p.select_frames(X0, 5),
        "residual_quantiles": lambda: p.residual_quantiles(X0, q),
        "frame_quantiles": lambda: p.frame_quantiles(X0, q),
        "point_residuals": lambda: p.point_residuals(X0),
        "eval_segments": lambda: p.eval_segments(seg, seg_poses),
        "information_segments": lambda: p.information_segments(seg, seg_poses),
        "solve_segments": lambda: p.solve_segments(seg, seg_poses, trace_cap=4),
        "eval_poses": lambda: p.eval_poses(starts),
        "solve_starts": lambda: p.solve_starts(starts, trace_cap=4),
        "subset": lambda: _close(p.subset(keep)),
        "trim": lambda: _close(p.trim(X0, 0.05)),
        "bench_eval": lambda: p.bench_eval(X0, 2),
        "bench_frame_report": lambda: p.bench_frame_report(X0, 2),
        "bench_select": lambda: p.bench_select(X0, 5, 2),
        "bench_segments": lambda: p.bench_segments(seg, seg_poses, 2),
        "bench_poses": lambda: p.bench_poses(starts, 2),
        "bench_subset": lambda: p.bench_subset(keep, 2),
        "bench_trim": lambda: p.bench_trim(X0, 0.05, 2),
        "bench_quantiles": lambda: p.bench_quantiles(X0, q, 2),
    }
    for name, call in calls.items():
        _no_scratch_left(name, call)


def test_rejected_calls_free_their_scratch(problem):
    from camlasercalibratool_b200 import ClcError, _lib

    p, L, h = problem, _lib.load(), problem._h
    N = p.sizes()[0]
    dp = lambda a: np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    ip = lambda a: np.ascontiguousarray(a, dtype=np.int64).ctypes.data_as(C.POINTER(C.c_int64))  # noqa: E731
    seg = np.array([0, N], dtype=np.int64)
    bad_pose = X0.copy()
    bad_pose[4] = np.nan
    H, g, cost = np.empty(36), np.empty(6), np.empty(4)
    summaries = (_lib.LmSummary * 4)()
    values, n_valid = np.empty(8), C.c_int64()
    invalid = 1  # CLC_ERR_INVALID
    calls = {
        "eval_segments": _rejected(lambda: L.clc_eval_segments(h, 1, ip(seg), dp(bad_pose), dp(H), dp(g), dp(cost)), invalid),
        "solve_segments": _rejected(lambda: L.clc_solve_lm_segments(h, 1, ip(seg), dp(X0.copy()), None, summaries, None, 999),
                                    invalid),
        "eval_poses": _rejected(lambda: L.clc_eval_poses(h, 0, dp(X0), dp(H), dp(g), dp(cost)), invalid),
        "solve_starts": _rejected(lambda: L.clc_solve_lm_starts(h, 1, dp(bad_pose.copy()), None, summaries, None, 0, None), invalid),
        "eval_time_offset": _rejected(lambda: L.clc_eval_time_offset(h, dp(X0), 0.0, dp(np.empty(49)), dp(np.empty(7)),
                                                                     dp(cost))),
        "residual_quantiles": _rejected(lambda: L.clc_residual_quantiles(h, dp(X0), 1, dp([1.5]), dp(values), C.byref(n_valid)),
                                        invalid),
        "point_residuals": _rejected(lambda: L.clc_point_residuals(h, dp(X0), 0, p.sizes()[1] + 1, dp(np.empty(1))), invalid),
    }
    for name, call in calls.items():
        _no_scratch_left(name, call)

    # a selection whose frames observe nothing is refused after its scratch exists
    def no_information():
        with pytest.raises(ClcError):
            p.select_frames(X0, 3, candidates=np.zeros(N, dtype=bool))

    _no_scratch_left("select_frames (refused)", no_information)


def test_time_offset_entry_points_free_their_scratch():
    from camlasercalibratool_b200 import Problem

    sc = TR.scene(n_knots=12, beams=50, seed=17)
    x = TR.truth_pose7()
    with Problem.from_arrays(sc.frame_pose, sc.offsets, sc.points, device=0) as p:
        p.set_trajectory(sc.knot_times, sc.knot_poses, sc.frame_times)
        calls = {
            "eval_time_offset": lambda: p.eval_time_offset(x, 0.01),
            "information_time_offset": lambda: p.information_time_offset(x, 0.01),
            "solve_time_offset": lambda: p.solve_time_offset(x, 0.0, trace_cap=8),
            "solve_time_offset (td held)": lambda: p.solve_time_offset(x, 0.01, fixed=("td",)),
            "bench_time_offset": lambda: p.bench_time_offset(x, 0.01, 2),
        }
        for name, call in calls.items():
            _no_scratch_left(name, call)


def test_group_and_standalone_entry_points_free_their_scratch():
    from camlasercalibratool_b200 import Group, LineFittingCeres
    from camlasercalibratool_b200 import formats as fmt

    q = [0.25, 0.75]
    with Group.synthetic(60, 200, seed=3, sigma=0.01, devices=(0,)) as g:
        N = g.sizes()[1]
        keep = np.ones(N, dtype=bool)
        keep[1::4] = False
        calls = {
            "group eval": lambda: g.eval(X0),
            "group solve": lambda: g.solve(X0),
            "group frame_report": lambda: g.frame_report(X0),
            "group select_frames": lambda: g.select_frames(X0, 4),
            "group residual_quantiles": lambda: g.residual_quantiles(X0, q),
            "group frame_quantiles": lambda: g.frame_quantiles(X0, q),
            "group subset": lambda: _close(g.subset(keep)),
            "group trim": lambda: _close(g.trim(X0, 0.05)),
        }
        for name, call in calls.items():
            _no_scratch_left(name, call)
    points = np.random.default_rng(5).normal(size=(40, 3))
    points[:, 2] = 0.0
    det = [(np.array([0], dtype=np.int32), np.zeros((1, 4, 2), dtype=np.float32))] * 3
    ranges = np.random.default_rng(6).uniform(1.0, 5.0, size=(4, 200)).astype(np.float32)
    calls = {
        "LineFittingCeres": lambda: LineFittingCeres(points, np.zeros(2)),
        "estimate_board_poses": lambda: fmt.estimate_board_poses("equi", det, device=0),
        "auto_get_line_segments": lambda: fmt.auto_get_line_segments(ranges, -1.0, 0.02, 0.05),
    }
    for name, call in calls.items():
        _no_scratch_left(name, call)
