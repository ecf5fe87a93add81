"""CPU tests of one calibration at many poses (clc_eval_poses, clc_solve_lm_starts) that need no GPU:

* the Python argument checks and the C entry points' NULL / bad-argument errors;
* the choice of the best start (csrc/clc_segment_plan.h, compiled with g++ from the source the library uses): FAILURE excluded,
  ties to the lowest index, -1 when every start failed;
* the pose-major virtual segmentation put through the library's reduction plan, against numpy;
* K LmCores advanced side by side by the host build of lm_update, each fed the oracle's sums at its own candidate, make the
  decisions of K oracle solves from the same starts.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import exact_sums as X
from test_segment_plan import numpy_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAILURE = 6  # CLC_TERM_FAILURE

SHIM = r'''
#include "clc_segment_plan.h"
extern "C" long long best(long long K, const int* term, const double* cost, int failure) {
  return clc::best_start(K, term, cost, failure);
}
extern "C" long long pose_plan(long long n, long long K, long long* off, long long* chunk_off, long long* seg_chunks) {
  const std::vector<int64_t> o = clc::pose_segment_offsets(n, K);
  for (size_t i = 0; i < o.size(); ++i) off[i] = o[i];
  const clc::SegmentPlan p = clc::segment_plan(n * K, K, o.data());
  for (size_t i = 0; i < p.chunk_offsets.size(); ++i) chunk_off[i] = p.chunk_offsets[i];
  for (size_t i = 0; i < p.seg_chunks.size(); ++i) seg_chunks[i] = p.seg_chunks[i];
  return (long long)p.chunk_offsets.size() - 1;
}
extern "C" long long chunk_rows() { return clc::kSegChunkRows; }
'''


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("starts")
    src = d / "starts.cpp"
    src.write_text(SHIM)
    out = str(d / "libstarts.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I",
                    os.path.join(ROOT, "camlasercalibratool_b200", "csrc"), str(src), "-o", out], check=True)
    L = C.CDLL(out)
    ll = C.POINTER(C.c_longlong)
    L.best.argtypes = [C.c_longlong, C.POINTER(C.c_int), C.POINTER(C.c_double), C.c_int]
    L.best.restype = C.c_longlong
    L.pose_plan.argtypes = [C.c_longlong, C.c_longlong, ll, ll, ll]
    L.pose_plan.restype = C.c_longlong
    L.chunk_rows.restype = C.c_longlong
    return L


def best(lib, term, cost):
    t = np.ascontiguousarray(term, dtype=np.int32)
    c = np.ascontiguousarray(cost, dtype=np.float64)
    return lib.best(len(t), t.ctypes.data_as(C.POINTER(C.c_int)), c.ctypes.data_as(C.POINTER(C.c_double)), FAILURE)


def test_best_start(lib):
    assert best(lib, [1, 2, 3], [3.0, 1.0, 2.0]) == 1
    assert best(lib, [1, 2, 1, 2], [2.0, 1.0, 1.0, 1.0]) == 1  # ties: lowest index
    assert best(lib, [1, FAILURE, 5], [2.0, 0.5, 3.0]) == 0  # a failed start never wins, whatever its cost
    assert best(lib, [FAILURE, FAILURE], [1.0, 2.0]) == -1
    assert best(lib, [5, 4], [np.nan, 7.0]) == 1  # a NaN cost loses to any other
    assert best(lib, [5, 4], [np.nan, np.nan]) == 0
    rng = np.random.default_rng(0)
    for _ in range(200):
        K = int(rng.integers(1, 40))
        term = rng.choice([1, 2, 3, 4, 5, FAILURE], size=K)
        cost = rng.choice([0.5, 1.0, 2.0, 3.0], size=K)
        ok = [k for k in range(K) if term[k] != FAILURE]
        assert best(lib, term, cost) == (min(ok, key=lambda k: (cost[k], k)) if ok else -1)


@pytest.mark.parametrize("n", [0, 1, 7, 255, 256, 257, 1000])
@pytest.mark.parametrize("K", [1, 2, 35, 1024])
def test_pose_major_plan_against_numpy(lib, n, K):
    R = lib.chunk_rows()
    off = np.zeros(K + 1, dtype=np.int64)
    cap = n * K + K + 2
    co, sc = np.zeros(cap, dtype=np.int64), np.zeros(K + 1, dtype=np.int64)
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_longlong))  # noqa: E731
    m = lib.pose_plan(n, K, p(off), p(co), p(sc))
    assert off.tolist() == [k * n for k in range(K + 1)]
    rco, rsc, _ = numpy_plan(n * K, off, R)
    assert np.array_equal(co[:m + 1], rco) and np.array_equal(sc, rsc)
    # every pose owns the same chunk layout, shifted by n rows: its sums cannot depend on K or on the other poses
    per = np.diff(sc)
    assert np.all(per == per[0])
    for k in range(K):
        assert np.array_equal(co[sc[k]:sc[k + 1] + 1] - k * n, co[sc[0]:sc[1] + 1])


def test_argument_checks():
    from camlasercalibratool_b200 import _lib
    from camlasercalibratool_b200.api import MAX_POSES, _poses

    x = np.tile([0, 0, 0, 0, 0, 0, 1.0], (3, 1))
    for bad in (x[0], x[:, :6], np.zeros((0, 7)), np.tile(x[0], (MAX_POSES + 1, 1)), x.astype(complex), [["a"] * 7]):
        with pytest.raises(ValueError):
            _poses(bad)
    for v in (np.nan, np.inf):
        b = x.copy()
        b[2, 5] = v
        with pytest.raises(ValueError):
            _poses(b)
    y, K = _poses(x.astype(np.float32))
    assert K == 3 and y.dtype == np.float64 and y.flags.c_contiguous
    assert _poses(np.tile(x[0], (MAX_POSES, 1)))[1] == MAX_POSES
    L = _lib.load()
    dp = x.ctypes.data_as(C.POINTER(C.c_double))
    cost = np.zeros(3)
    cp = cost.ctypes.data_as(C.POINTER(C.c_double))
    best = C.c_int64()
    assert L.clc_eval_poses(None, 3, dp, None, None, cp) == 1
    assert L.clc_solve_lm_starts(None, 3, dp, None, None, None, 0, C.byref(best)) == 1
    assert L.clc_bench_poses(None, 3, dp, 1, 0, None) == 1


def test_side_by_side_cores_make_the_oracles_decisions(oracle, harness):
    """K LmCores over ALL frames, one start each, advanced one shared sweep at a time (the host restatement of
    clc_solve_lm_starts' update loop on the sweep kernel, with finished starts skipped): every start ends as the oracle's solve
    from that start ends."""
    p = oracle.generate(60, 180, seed=5, sigma=0.01)
    x_gt = oracle.ground_truth()[1]
    rng = np.random.default_rng(5)
    x0 = [np.array([0, 0, 0, 0, 0, 0, 1.0]), x_gt.copy()] + [oracle.pose_plus(x_gt, s * rng.standard_normal(6))
                                                              for s in (1e-3, 1e-2, 1e-1, 3e-1)]
    K = len(x0)
    L = harness.L
    states = [C.create_string_buffer(L.harness_lm_state_size()) for _ in range(K)]
    opt = harness.default_options()
    for k in range(K):
        L.harness_lm_init(states[k], harness.dp(np.ascontiguousarray(x0[k])), C.byref(opt))
    cand = np.empty(7)
    for _ in range(opt.max_num_iterations + 2):
        running = [k for k in range(K) if not L.harness_lm_done(states[k])]  # the device's compacted list
        if not running:
            break
        for k in running:
            L.harness_lm_cand(states[k], harness.dp(cand))
            cost, H, g = oracle.evaluate_normal(p, cand.copy())
            L.harness_lm_update(states[k], harness.dp(np.ascontiguousarray(X.pack_lm(cost, H, g))))
    for k in range(K):
        xo, so, _ = oracle.solve(p, x0[k])
        x = np.empty(7)
        L.harness_lm_x(states[k], harness.dp(x))
        assert L.harness_lm_done(states[k]) == so.termination and L.harness_lm_ntrace(states[k]) == so.num_iterations, k
        assert np.abs(x - xo).max() < 1e-9, k
