"""CPU tests of the quantile selection (csrc/clc_quantile_plan.h, compiled with g++ from the source the library uses): a complete
simulated multi-pass radix select on numpy key arrays -- the histogram passes over every key, the compaction of the active buckets
and the passes over the compacted keys, with the histograms of several shards summed -- compared bitwise with np.sort.  Also: the
Python argument checks (no library call on a rejected argument) and the C entry points' argument checks, which answer without a
GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHIM = r'''
#include <cstring>
#include <vector>
#include "clc_quantile_plan.h"
extern "C" int quantiles_max() { return clc::kQuantilesMax; }
// The selection of q[n_q] over the |e| of e[n], the keys split into `shards` contiguous parts whose histograms are summed, with
// `bins_log2` bins per pass and compaction at `cap` keys per bucket (cap 0: never).  Returns the passes over all keys.
extern "C" int run_select(const double* e, long long n, int shards, int n_q, const double* q, int bins_log2, unsigned long long cap,
                      double* values, long long* n_valid) {
  std::vector<uint64_t> keys((size_t)n);
  for (long long i = 0; i < n; ++i) {
    const double a = std::fabs(e[i]);
    std::memcpy(&keys[i], &a, 8);
  }
  clc::QSel s;
  clc::qsel_start(&s, n_q, q);
  bool compacted = false;
  int passes = 0;
  std::vector<uint64_t> src = keys;
  while (!clc::qsel_done(s)) {
    const int d = clc::qsel_digit(s, bins_log2);
    std::vector<unsigned long long> hist((size_t)s.n_pre << d, 0);
    const long long m = (long long)src.size();
    for (int sh = 0; sh < shards; ++sh) {
      std::vector<unsigned long long> part(hist.size(), 0);
      for (long long i = m * sh / shards; i < m * (sh + 1) / shards; ++i) {
        const int b = clc::qsel_bin(s.bits, s.n_pre, s.pre, d, src[i]);
        if (b >= 0) ++part[b];
      }
      for (size_t b = 0; b < hist.size(); ++b) hist[b] += part[b];
    }
    passes += compacted ? 0 : 1;
    clc::qsel_update(&s, hist.data(), d);
    if (compacted || clc::qsel_done(s) || cap == 0 || !clc::qsel_fits(s, cap)) continue;
    std::vector<uint64_t> kept;
    for (uint64_t k : keys)
      if (clc::qsel_match(s.bits, s.n_pre, s.pre, k)) kept.push_back(k);
    if (kept.size() > (size_t)s.n_pre * cap) return -1;  // the scratch would overflow
    src.swap(kept);
    compacted = true;
    ++passes;
  }
  for (int r = 0; r < n_q; ++r) {
    const uint64_t k = s.n_valid ? clc::qsel_key(s, r) : 0x7FF8000000000000ull;
    std::memcpy(&values[r], &k, 8);
  }
  *n_valid = (long long)s.n_valid;
  return passes;
}
extern "C" unsigned long long rank(double q, unsigned long long n) { return clc::quantile_rank(q, n); }
'''


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("quantplan")
    src = d / "plan.cpp"
    src.write_text(SHIM)
    out = str(d / "libplan.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I",
                    os.path.join(ROOT, "camlasercalibratool_b200", "csrc"), str(src), "-o", out], check=True)
    L = C.CDLL(out)
    dp = C.POINTER(C.c_double)
    L.run_select.restype = C.c_int
    L.run_select.argtypes = [dp, C.c_longlong, C.c_int, C.c_int, dp, C.c_int, C.c_ulonglong, dp, C.POINTER(C.c_longlong)]
    L.rank.restype = C.c_ulonglong
    L.rank.argtypes = [C.c_double, C.c_ulonglong]
    assert L.quantiles_max() == 16
    return L


def run(lib, e, q, shards=1, bins_log2=13, cap=1 << 16):
    e = np.ascontiguousarray(e, dtype=np.float64)
    q = np.ascontiguousarray(np.atleast_1d(q), dtype=np.float64)
    values = np.empty(q.size)
    nv = C.c_longlong()
    dp = C.POINTER(C.c_double)
    passes = lib.run_select(e.ctypes.data_as(dp), e.size, shards, q.size, q.ctypes.data_as(dp), bins_log2, cap,
                        values.ctypes.data_as(dp), C.byref(nv))
    assert passes >= 0, "compaction overflowed its scratch"
    return values, nv.value, passes


def expected(e, q):
    """The rank rule of include/clc_b200.h on numpy: sort the valid |e|, take k = clamp(ceil(q n) - 1, 0, n - 1)."""
    a = np.abs(np.asarray(e, dtype=np.float64))
    a = np.sort(a[~np.isnan(a)])
    n = a.size
    out = []
    for qq in np.atleast_1d(q):
        if n == 0:
            out.append(np.nan)
            continue
        k = int(min(max(np.ceil(float(qq) * float(n)) - 1.0, 0.0), n - 1))
        out.append(a[k])
    return np.array(out), n


def same_bits(a, b):
    """Equal bytes, NaN where NaN (the sign of a zero counts)."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64))


Q_EDGE = [0.0, 1.0, 0.5, 1e-300, 1.0 - 2.0 ** -53]


def cases():
    rng = np.random.default_rng(7)
    sub = np.array([5e-324, 1e-310, -2.5e-320, 0.0, -0.0, 1e-300])
    yield "all_equal", np.full(1000, 0.25)
    yield "all_zero", np.zeros(5000)
    yield "signed_zeros", np.array([0.0, -0.0, -0.0, 0.0, 1.0, -1.0])
    yield "two_values", np.where(rng.random(3000) < 0.3, 1e-3, -2e-3)
    yield "subnormals", np.concatenate([sub, -sub * 3, rng.normal(0, 1e-300, 50)])
    yield "inf", np.array([np.inf, -np.inf, 1.0, 0.0, -np.inf, 2.0])
    yield "nan", np.array([np.nan, 1.0, -np.nan, 0.5, np.nan])
    yield "all_nan", np.full(10, np.nan)
    yield "n0", np.zeros(0)
    yield "n1", np.array([-3.5])
    yield "n2", np.array([2.0, -1.0])
    yield "noisy", np.concatenate([rng.normal(0, 0.01, 200_000), rng.normal(0, 0.15, 5_000), [np.nan] * 17, [np.inf] * 3])
    yield "wide", rng.standard_cauchy(50_000) * 10.0 ** rng.integers(-300, 300, 50_000)
    yield "ties_dense", rng.integers(0, 5, 100_000).astype(np.float64) * 1e-3


@pytest.mark.parametrize("name,e", list(cases()), ids=[c[0] for c in cases()])
def test_selection_matches_sort(lib, name, e):
    rng = np.random.default_rng(11)
    qs = [np.array(Q_EDGE), rng.random(16), np.array([0.5] * 16), np.array([0.3, 0.3, 0.0, 1.0, 0.3, 0.7, 0.7, 0.0])]
    for q in qs:
        want, n = expected(e, q)
        for shards, bins, cap in ((1, 13, 1 << 16), (3, 13, 1 << 16), (2, 12, 0), (1, 5, 64), (4, 13, 1)):
            got, nv, passes = run(lib, e, q, shards, bins, cap)
            assert nv == n
            assert same_bits(got, want), (name, q, shards, bins, cap, got, want)


def test_every_R_with_colliding_ranks(lib):
    rng = np.random.default_rng(3)
    e = np.concatenate([rng.normal(0, 0.01, 20_000), np.zeros(500), np.full(300, 0.02)])
    for R in range(1, 17):
        q = rng.choice([0.0, 0.25, 0.5, 0.5, 0.999, 1.0], size=R) if R % 2 else rng.random(R)
        want, _ = expected(e, q)
        got, _, _ = run(lib, e, q)
        assert same_bits(got, want), R


def test_pass_counts(lib):
    """Noisy data compacts after its histogram passes; massive ties never compact and finish after the full digit sequence."""
    rng = np.random.default_rng(5)
    _, _, passes = run(lib, rng.normal(0, 0.01, 1_000_000), [0.5])
    assert passes <= 3, passes
    _, _, passes = run(lib, rng.normal(0, 0.01, 1_000_000), np.linspace(0, 1, 16))
    assert passes <= 4, passes
    # 63 bits: 13 bits in the first pass, then 13 per pass with one prefix -> 5 passes; at most ceil(63 / 9) = 7 with 16 prefixes
    _, _, passes = run(lib, np.zeros(200_000), [0.5], cap=1 << 16)
    assert passes == 5, passes
    _, _, passes = run(lib, np.zeros(200_000), np.linspace(0, 1, 16), cap=1 << 16)
    assert passes <= 7, passes


def test_rank_rule(lib):
    for n in (1, 2, 3, 10, 1001, 2 ** 33 + 1):
        for q in Q_EDGE + [0.25, 0.75, 1.0 / 3.0]:
            k = int(min(max(np.ceil(q * float(n)) - 1.0, 0.0), n - 1))
            assert lib.rank(q, n) == k, (n, q)
    assert lib.rank(0.5, 4) == 1 and lib.rank(0.5, 5) == 2  # the lower median


# ---- argument checks ---------------------------------------------------------------------------------------------------------

class _Recorder:
    """A stand-in for the library: records every call, answers 0."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append(name)
            return 0
        return fn


def _fake_problem(n_frames=3, n_points=100):
    from camlasercalibratool_b200 import Problem

    p = Problem.__new__(Problem)
    p._h = None
    p._L = _Recorder()
    p.sizes = lambda: (n_frames, n_points, False)
    return p


BAD_Q = [np.nan, -0.1, 1.5, [0.5, np.nan], [], np.zeros(17), np.zeros((2, 2)), "0.5", [True]]
BAD_POSE = [np.zeros(6), np.array([0, 0, 0, 0, 0, 0, np.inf]), np.array([np.nan] + [0.0] * 6)]
X = np.array([0, 0, 0, 0, 0, 0, 1.0])


def test_python_checks_before_any_library_call():
    p = _fake_problem()
    for q in BAD_Q:
        for call in (p.residual_quantiles, p.frame_quantiles):
            with pytest.raises((ValueError, TypeError)):
                call(X, q)
        with pytest.raises((ValueError, TypeError)):
            p.bench_quantiles(X, q, 2)
    for x in BAD_POSE:
        for call in (p.residual_quantiles, p.frame_quantiles):
            with pytest.raises(ValueError):
                call(x, 0.5)
        with pytest.raises(ValueError):
            p.point_residuals(x)
    for first, count in ((-1, None), (0, 101), (101, None), (50, 51), (0, -1), (1.5, None), (0, True)):
        with pytest.raises((ValueError, TypeError)):
            p.point_residuals(X, first, count)
    assert p._L.calls == []
    # accepted arguments reach the library
    p.residual_quantiles(X, 0.5)
    p.frame_quantiles(X, [0.0, 1.0])
    p.point_residuals(X, 100)
    p.point_residuals(X, 10, 90)
    assert p._L.calls == ["clc_residual_quantiles", "clc_frame_quantiles", "clc_point_residuals", "clc_point_residuals"]


def test_c_entry_points_reject_bad_arguments_without_a_gpu():
    from camlasercalibratool_b200 import _lib

    L = _lib.load()
    dp = _lib.c_double_p
    fake = C.create_string_buffer(4096)  # a zeroed stand-in handle: the checks run before the handle's device data is touched
    h = C.cast(fake, C.c_void_p)
    x = np.ascontiguousarray(X)
    q = np.array([0.5, 0.9])
    v, nv = np.zeros(16), C.c_int64()
    assert L.clc_residual_quantiles(None, x.ctypes.data_as(dp), 1, q.ctypes.data_as(dp), v.ctypes.data_as(dp), C.byref(nv)) == 1
    assert L.clc_residual_quantiles(h, None, 1, q.ctypes.data_as(dp), v.ctypes.data_as(dp), C.byref(nv)) == 1
    assert L.clc_residual_quantiles(h, x.ctypes.data_as(dp), 1, None, v.ctypes.data_as(dp), C.byref(nv)) == 1
    assert L.clc_group_residual_quantiles(None, x.ctypes.data_as(dp), 1, q.ctypes.data_as(dp), v.ctypes.data_as(dp), C.byref(nv)) == 1
    assert L.clc_group_frame_quantiles(None, x.ctypes.data_as(dp), 1, q.ctypes.data_as(dp), v.ctypes.data_as(dp), None) == 1
    for n_q in (0, 17, -1):
        for fn in (L.clc_residual_quantiles, L.clc_frame_quantiles):
            assert fn(h, x.ctypes.data_as(dp), n_q, np.zeros(20).ctypes.data_as(dp), v.ctypes.data_as(dp), C.byref(nv)) == 1
            assert b"n_q" in L.clc_last_error()
    for bad in (np.nan, -1e-300, 1.0 + 2.0 ** -52):
        qq = np.array([0.5, bad])
        for fn in (L.clc_residual_quantiles, L.clc_frame_quantiles):
            assert fn(h, x.ctypes.data_as(dp), 2, qq.ctypes.data_as(dp), v.ctypes.data_as(dp), C.byref(nv)) == 1
            assert b"q[1]" in L.clc_last_error()
    xb = x.copy()
    xb[3] = np.inf
    assert L.clc_residual_quantiles(h, xb.ctypes.data_as(dp), 1, q.ctypes.data_as(dp), v.ctypes.data_as(dp), C.byref(nv)) == 1
    assert b"pose7[3]" in L.clc_last_error()
    # the stand-in holds 0 points: every non-empty range lies outside it, and a non-finite pose is rejected first
    assert L.clc_point_residuals(h, x.ctypes.data_as(dp), 0, 1, v.ctypes.data_as(dp)) == 1
    assert L.clc_point_residuals(h, x.ctypes.data_as(dp), -1, 0, v.ctypes.data_as(dp)) == 1
    assert L.clc_point_residuals(h, xb.ctypes.data_as(dp), 0, 0, v.ctypes.data_as(dp)) == 1
    assert L.clc_point_residuals(None, x.ctypes.data_as(dp), 0, 0, v.ctypes.data_as(dp)) == 1
    fms, ms, passes = (C.c_float * 2)(), (C.c_float * 2)(), C.c_int()
    assert L.clc_bench_quantiles(h, x.ctypes.data_as(dp), 17, q.ctypes.data_as(dp), 2, 0, ms, fms, C.byref(passes)) == 1
    assert L.clc_bench_quantiles(h, x.ctypes.data_as(dp), 1, q.ctypes.data_as(dp), 0, 0, ms, fms, C.byref(passes)) == 1
