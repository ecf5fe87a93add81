"""CPU tests of the segmented solves (clc_*_segments) that need no GPU:

* the segmentation check and the two-level reduction plan (csrc/clc_segment_plan.h, compiled with g++ from the source the
  library uses) against a numpy restatement;
* W LmCores advanced side by side by the host build of lm_update, each fed its segment's oracle sums, make the decisions of W
  separate oracle solves;
* the Python argument checks and the C entry points' NULL / bad-argument errors.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import exact_sums as X

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHIM = r'''
#include "clc_segment_plan.h"
extern "C" int valid(long long n, long long W, const long long* off) {
  return clc::segments_valid(n, W, reinterpret_cast<const int64_t*>(off)) ? 1 : 0;
}
extern "C" long long plan(long long n, long long W, const long long* off, long long* chunk_off, long long* seg_chunks, int* frame_seg) {
  const clc::SegmentPlan p = clc::segment_plan(n, W, reinterpret_cast<const int64_t*>(off));
  for (size_t i = 0; i < p.chunk_offsets.size(); ++i) chunk_off[i] = p.chunk_offsets[i];
  for (size_t i = 0; i < p.seg_chunks.size(); ++i) seg_chunks[i] = p.seg_chunks[i];
  for (size_t i = 0; i < p.frame_seg.size(); ++i) frame_seg[i] = p.frame_seg[i];
  return (long long)p.chunk_offsets.size() - 1;
}
extern "C" long long chunk_rows() { return clc::kSegChunkRows; }
'''


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("segplan")
    src = d / "plan.cpp"
    src.write_text(SHIM)
    out = str(d / "libsegplan.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I",
                    os.path.join(ROOT, "camlasercalibratool_b200", "csrc"), str(src), "-o", out], check=True)
    L = C.CDLL(out)
    ll = C.POINTER(C.c_longlong)
    L.valid.argtypes = [C.c_longlong, C.c_longlong, ll]
    L.plan.argtypes = [C.c_longlong, C.c_longlong, ll, ll, ll, C.POINTER(C.c_int)]
    L.plan.restype = C.c_longlong
    L.chunk_rows.restype = C.c_longlong
    return L


def _ll(a):
    return a.ctypes.data_as(C.POINTER(C.c_longlong))


def numpy_plan(n, off, R):
    chunk = [0]
    seg_chunks = [0]
    for s in range(len(off) - 1):
        a, b = off[s], off[s + 1]
        chunk += list(range(a + R, b, R)) + ([b] if b > a else [])
        seg_chunks.append(len(chunk) - 1)
    frame_seg = np.repeat(np.arange(len(off) - 1), np.diff(off))
    return np.array(chunk), np.array(seg_chunks), frame_seg


def run_plan(lib, n, off):
    off = np.ascontiguousarray(off, dtype=np.int64)
    W = len(off) - 1
    cap = n + W + 2
    co, sc, fs = np.zeros(cap, dtype=np.int64), np.zeros(W + 1, dtype=np.int64), np.zeros(max(n, 1), dtype=np.int32)
    k = lib.plan(n, W, _ll(off), _ll(co), _ll(sc), fs.ctypes.data_as(C.POINTER(C.c_int)))
    return co[:k + 1], sc, fs[:n]


SEGMENTATIONS = {
    "one": lambda n, rng: [0, n],
    "every_frame": lambda n, rng: list(range(n + 1)),
    "empty_segments": lambda n, rng: sorted([0, 0, min(3, n), min(3, n), min(3, n), n // 2, n, n]),
    "random": lambda n, rng: [0] + sorted(rng.integers(0, n + 1, size=40).tolist()) + [n],
    "long": lambda n, rng: sorted([0, min(1, n), max(n - 1, 0), n]),
}


@pytest.mark.parametrize("name", list(SEGMENTATIONS))
@pytest.mark.parametrize("n", [1, 7, 1000, 100_000])
def test_plan_against_numpy(lib, name, n):
    R = lib.chunk_rows()
    off = np.array(SEGMENTATIONS[name](n, np.random.default_rng(n)), dtype=np.int64)
    assert lib.valid(n, len(off) - 1, _ll(off)) == 1
    co, sc, fs = run_plan(lib, n, off)
    rco, rsc, rfs = numpy_plan(n, off, R)
    assert np.array_equal(co, rco) and np.array_equal(sc, rsc) and np.array_equal(fs, rfs)
    assert np.all(np.diff(co) >= 1) and np.all(np.diff(co) <= R)  # no empty chunk, none longer than R rows


def test_segments_of_empty_frames_and_validation(lib):
    off = np.array([0, 2, 5], dtype=np.int64)
    co, sc, fs = run_plan(lib, 5, off)
    assert co.tolist() == [0, 2, 5] and sc.tolist() == [0, 1, 2] and fs.tolist() == [0, 0, 1, 1, 1]
    for bad, n in (([1, 5], 5), ([0, 4], 5), ([0, 3, 2, 5], 5), ([0, 6], 5)):
        a = np.array(bad, dtype=np.int64)
        assert lib.valid(n, len(a) - 1, _ll(a)) == 0
    z = np.array([0], dtype=np.int64)
    assert lib.valid(0, 0, _ll(z)) == 0  # W >= 1


def test_side_by_side_cores_make_the_oracles_decisions(oracle, harness):
    """W LmCores advanced one sweep at a time, side by side, each on its own segment's oracle sums: every segment ends as the
    oracle's solve of its slice ends (the host restatement of clc_solve_lm_segments' update loop)."""
    p = oracle.generate(240, 180, seed=7, sigma=0.01)
    off = [0, 30, 31, 31, 120, 240]
    W = len(off) - 1
    rng = np.random.default_rng(7)
    x_gt = oracle.ground_truth()[1]
    x0 = [np.array([0, 0, 0, 0, 0, 0, 1.0]) if s % 2 else oracle.pose_plus(x_gt, 1e-2 * rng.standard_normal(6)) for s in range(W)]
    slices = []
    for s in range(W):
        a, b = off[s], off[s + 1]
        o = p.offsets[a:b + 1] - p.offsets[a]
        slices.append(oracle.Problem(p.frame_pose[a:b], o, p.points[p.offsets[a]:p.offsets[b]]))
    L = harness.L
    states = [C.create_string_buffer(L.harness_lm_state_size()) for _ in range(W)]
    opt = harness.default_options()
    for s in range(W):
        L.harness_lm_init(states[s], harness.dp(np.ascontiguousarray(x0[s])), C.byref(opt))
    cand = np.empty(7)
    for _ in range(opt.max_num_iterations + 2):
        for s in range(W):
            if L.harness_lm_done(states[s]):
                continue
            L.harness_lm_cand(states[s], harness.dp(cand))
            if len(slices[s].frame_pose):
                cost, H, g = oracle.evaluate_normal(slices[s], cand.copy())
                sums = X.pack_lm(cost, H, g)
            else:
                sums = np.zeros(28)
            L.harness_lm_update(states[s], harness.dp(np.ascontiguousarray(sums)))
    for s in range(W):
        if not len(slices[s].frame_pose):
            assert L.harness_lm_done(states[s]) != 0
            continue
        xo, so, to = oracle.solve(slices[s], x0[s])
        x = np.empty(7)
        L.harness_lm_x(states[s], harness.dp(x))
        assert L.harness_lm_done(states[s]) == so.termination and L.harness_lm_ntrace(states[s]) == so.num_iterations, s
        assert np.abs(x - xo).max() < 1e-9


def test_argument_checks():
    from camlasercalibratool_b200 import _lib
    from camlasercalibratool_b200.api import _segments

    x = np.tile([0, 0, 0, 0, 0, 0, 1.0], (2, 1))
    for off, poses in (([0, 5, 9], x), ([1, 5, 10], x), ([0, 6, 5, 10], np.tile(x[0], (3, 1))), ([0, 10], x),
                       ([0, 5, 10], x[:1]), ([0.0, 5.0, 10.0], x)):
        with pytest.raises(ValueError):
            _segments(off, poses, 10)
    bad = x.copy()
    bad[1, 2] = np.nan
    with pytest.raises(ValueError):
        _segments([0, 5, 10], bad, 10)
    off, poses, W = _segments([0, 0, 10], x, 10)
    assert W == 2 and off.dtype == np.int64
    L = _lib.load()
    o = np.array([0, 10], dtype=np.int64)
    p7 = np.array([0, 0, 0, 0, 0, 0, 1.0])
    dp = p7.ctypes.data_as(C.POINTER(C.c_double))
    op = o.ctypes.data_as(C.POINTER(C.c_int64))
    cost = np.zeros(1)
    assert L.clc_eval_segments(None, 1, op, dp, None, None, cost.ctypes.data_as(C.POINTER(C.c_double))) == 1
    assert L.clc_information_segments(None, 1, op, dp, None, None, None, None, None) == 1
    assert L.clc_solve_lm_segments(None, 1, op, dp, None, None, None, 0) == 1
