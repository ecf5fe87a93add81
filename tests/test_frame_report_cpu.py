"""The per-frame report without a GPU.

* Split-frame bookkeeping: the CLC_HD functions of csrc/clc_frames.cuh (which warps hold a frame, whether a warp's first and last
  piece is a whole frame, a head or a tail, which slots the fix-up adds) compiled for the host, against a restatement over every
  layout of tests/layouts.py and tests/small_layouts.py under the partition those modules compute for an H100 (132 SMs).
* The two per-frame restatements (tests/frame_oracle.c on the C oracle, tests/frame_report_np.py on numpy) agree, sum to the
  oracle's evaluation and analysis tail, report zeros for empty frames and keep a NaN point inside its own frame.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import frame_exact as FE
import frame_report_np as FN
import layouts as LY
import small_layouts as SL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "camlasercalibratool_b200", "csrc")
H100_SMS = 132
HEAD, WHOLE, TAIL = 1, 0, 2

SHIM = r"""
#include <algorithm>
#include "clc_frames.cuh"
extern "C" {
void frame_warps(const int64_t* off, int64_t n_frames, int64_t per_warp, int64_t* first, int64_t* last) {
  for (int64_t f = 0; f < n_frames; ++f) {
    first[f] = last[f] = -1;
    if (off[f + 1] > off[f]) clc::frame_warps(off[f], off[f + 1], per_warp, first + f, last + f);
  }
}
// kind of the first and the last piece of every warp range (-1: an idle warp), as the sweep kernel classifies them
void piece_kinds(const int64_t* off, int64_t n_frames, int64_t per_warp, int64_t n_warps, int32_t* kind_first, int32_t* kind_last) {
  const int64_t P = off[n_frames];
  for (int64_t w = 0; w < n_warps; ++w) {
    const int64_t p0 = std::min(w * per_warp, P), p1 = std::min(p0 + per_warp, P);
    kind_first[w] = kind_last[w] = -1;
    if (p0 >= p1) continue;
    const int64_t fa = std::upper_bound(off, off + n_frames + 1, p0) - off - 1;
    const int64_t fb = std::upper_bound(off, off + n_frames + 1, p1 - 1) - off - 1;
    kind_first[w] = clc::frame_piece_kind(off[fa], off[fa + 1], p0, p1);
    kind_last[w] = clc::frame_piece_kind(off[fb], off[fb + 1], p0, p1);
  }
}
int64_t frame_slot(int64_t w, int64_t w0) { return clc::frame_slot(w, w0); }
int slot_doubles(void) { return clc::kSlotDoubles; }
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("frames")
    src, out = d / "shim.cpp", d / "libframes.so"
    src.write_text(SHIM)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, "-o", str(out), str(src)])
    L = C.CDLL(str(out))
    L.frame_slot.restype = C.c_int64
    L.frame_slot.argtypes = [C.c_int64, C.c_int64]
    return L


def _ptr(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def restated(off, per_warp, n_warps):
    """Python restatement: first / last warp of every frame, and the kind of every warp's first and last piece."""
    off = np.asarray(off, dtype=np.int64)
    P = int(off[-1])
    fs, fe = off[:-1], off[1:]
    live = fe > fs
    first = np.where(live, fs // per_warp, -1)
    last = np.where(live, (np.maximum(fe, 1) - 1) // per_warp, -1)
    w = np.arange(n_warps, dtype=np.int64)
    p0 = np.minimum(w * per_warp, P)
    p1 = np.minimum(p0 + per_warp, P)
    busy = p0 < p1

    def kind(point):
        f = np.searchsorted(off, point, side="right") - 1
        return np.where(off[f] < p0, HEAD, np.where(off[f + 1] > p1, TAIL, WHOLE))

    kf = np.where(busy, kind(np.where(busy, p0, 0)), -1)
    kl = np.where(busy, kind(np.where(busy, p1 - 1, 0)), -1)
    return first, last, kf, kl


def check_layout(shim, off, grid, per_warp):
    off = np.ascontiguousarray(off, dtype=np.int64)
    N = len(off) - 1
    n_warps = grid * LY.WARPS
    first, last = np.empty(N, dtype=np.int64), np.empty(N, dtype=np.int64)
    kf, kl = np.empty(n_warps, dtype=np.int32), np.empty(n_warps, dtype=np.int32)
    shim.frame_warps(_ptr(off, C.c_int64), C.c_int64(N), C.c_int64(per_warp), _ptr(first, C.c_int64), _ptr(last, C.c_int64))
    shim.piece_kinds(_ptr(off, C.c_int64), C.c_int64(N), C.c_int64(per_warp), C.c_int64(n_warps), _ptr(kf, C.c_int32),
                     _ptr(kl, C.c_int32))
    rf, rl, rkf, rkl = restated(off, per_warp, n_warps)
    np.testing.assert_array_equal(first, rf)
    np.testing.assert_array_equal(last, rl)
    np.testing.assert_array_equal(kf, rkf)
    np.testing.assert_array_equal(kl, rkl)
    # the fix-up of every split frame adds the tail slot of its first warp and the head slots of the following warps, and
    # these pieces are exactly the frame
    P = int(off[-1])
    split = np.nonzero((first >= 0) & (first != last))[0]
    for f in split[:: max(1, len(split) // 200)]:
        w0, w1 = int(first[f]), int(last[f])
        assert kl[w0] == TAIL and all(kf[w] == HEAD for w in range(w0 + 1, w1 + 1))
        slots = [shim.frame_slot(w, w0) for w in range(w0, w1 + 1)]
        k = shim.slot_doubles()
        assert slots == [(2 * w0 + 1) * k] + [2 * w * k for w in range(w0 + 1, w1 + 1)]
        cover = sum(min(int(off[f + 1]), min((w + 1) * per_warp, P)) - max(int(off[f]), w * per_warp) for w in range(w0, w1 + 1))
        assert cover == off[f + 1] - off[f]
    return len(split)


@pytest.fixture(scope="module")
def bases(oracle):
    return LY.base_problem(oracle), SL.base_problems(oracle)


@pytest.mark.parametrize("stage", [LY.STAGE_GENERAL, LY.STAGE_PLANAR])
def test_split_bookkeeping_on_partition_layouts(shim, bases, stage):
    n_split = 0
    for name in LY.LAYOUTS:
        if stage == LY.STAGE_PLANAR and name.endswith("_z"):
            continue
        lay = LY.build(name, bases[0], H100_SMS, 256, stage)
        grid, per_warp = LY.partition(lay.n_points, H100_SMS, stage)
        n_split += check_layout(shim, lay.offsets, grid, per_warp)
    assert n_split > 0


@pytest.mark.parametrize("stage", [LY.STAGE_GENERAL, LY.STAGE_PLANAR])
def test_split_bookkeeping_on_small_layouts(shim, bases, stage):
    n_split = 0
    for name in SL.LAYOUTS:
        lay = SL.build(name, bases[1], stage)
        grid, per_warp = LY.partition(lay.n_points, H100_SMS, stage)
        n_split += check_layout(shim, lay.offsets, grid, per_warp)
    assert n_split > 0


# ---- the per-frame restatements ---------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def frame_oracle(oracle, tmp_path_factory):
    d = tmp_path_factory.mktemp("frame_oracle")
    out = d / "libframe_oracle.so"
    odir = os.path.dirname(oracle.build())
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    subprocess.check_call([cc, "-O2", "-std=c99", "-shared", "-fPIC", "-o", str(out), os.path.join(ROOT, "tests", "frame_oracle.c"),
                           "-L", odir, "-lclc_oracle", "-Wl,-rpath," + odir, "-lm"])
    L = C.CDLL(str(out))
    L.oracle_frame_report.argtypes = [C.POINTER(oracle._Problem), C.POINTER(C.c_double), C.POINTER(C.c_double)]

    def report(p, pose7):
        rows = np.zeros((p.n_frames, FN.ROW))
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        L.oracle_frame_report(C.byref(p._c), _ptr(pose7, C.c_double), _ptr(rows, C.c_double))
        rows[:, FN.N_POINTS] = rows[:, FN.N_POINTS].copy().view(np.int64)
        return rows

    return report


POSES = [np.array([0.0, 0, 0, 0, 0, 0, 1]), np.array([0.4, -0.3, 0.25, 0.2, -0.5, 0.3, 0.78])]


def _problem(oracle, use_loss, edges, counts=None, seed=5):
    base = oracle.generate(40, 120, seed=seed, sigma=0.01, exact_m=True, with_edges=True)
    if counts is None:
        return oracle.Problem(base.frame_pose, base.offsets, base.points, base.edge_points if edges else None, use_loss=use_loss)
    lay = LY.recut(base, counts, "cpu", set(), with_edges=edges)
    return oracle.Problem(lay.frame_pose, lay.offsets, lay.points, lay.edge_points, use_loss=use_loss)


def _np_report(p, pose7):
    return FN.frame_report(p.frame_pose, p.offsets, p.points, pose7, p.use_loss, p.cauchy_a, p.edge_points)


def _assert_rows_close(p, x, a, b, rtol=1e-13):
    """Agreement to rtol relative to what each field sums (tests/frame_exact.py's magnitudes: a frame's share of g or its
    mean e nearly cancels near the optimum)."""
    val, mag = FE.frame_sums(p.frame_pose, p.offsets, p.points, x, p.use_loss, p.cauchy_a, p.edge_points)
    FE.assert_within(FE.comparable(a), FE.comparable(b).astype(FE.LD), mag, rtol, "C vs numpy")
    FE.assert_within(FE.comparable(a), val, mag, rtol, "C vs long double")
    return mag


@pytest.mark.parametrize("use_loss,edges", [(True, False), (False, False), (True, True), (False, True)])
def test_restatements_agree_and_sum_to_the_oracle(oracle, frame_oracle, use_loss, edges):
    p = _problem(oracle, use_loss, edges, counts=[0, 37, 120, 0, 0, 1, 2, 300, 77, 0, 5])
    for x in POSES + [oracle.ground_truth()[1]]:
        rc, rn = frame_oracle(p, x), _np_report(p, x)
        A = _assert_rows_close(p, x, rc, rn).sum(axis=0)
        cost, H, g = oracle.evaluate_normal(p, x)
        chi = oracle.information(p, x)[2]
        want = np.concatenate([[cost, chi], H[np.triu_indices(6)], g])
        cols = [FE.C_COST, FE.C_CHI] + list(range(FE.C_H, FE.K))
        got = FE.comparable(rc)[:, cols].sum(axis=0)
        assert np.all(np.abs(got - want) <= 1e-13 * A[cols]), np.abs(got - want) / A[cols]
        if not use_loss:
            np.testing.assert_array_equal(rc[:, FN.MEAN_W][rc[:, 0] > 0], 1.0)


def test_empty_frames_report_zeros(oracle, frame_oracle):
    p = _problem(oracle, True, True, counts=[0, 0, 50, 0, 60, 0])
    x = POSES[1]
    for rows in (frame_oracle(p, x), _np_report(p, x)):
        empty = np.diff(p.offsets) == 0
        assert np.all(rows[empty] == 0.0)
        assert np.all(rows[~empty, FN.N_POINTS] == [50, 60])


def test_nan_point_stays_in_its_frame(oracle, frame_oracle):
    p = _problem(oracle, True, True, counts=[30, 40, 50])
    x = POSES[1]
    clean_c, clean_n = frame_oracle(p, x), _np_report(p, x)
    pts = p.points.copy()
    pts[45, 1] = np.nan  # frame 1
    q = oracle.Problem(p.frame_pose, p.offsets, pts, p.edge_points, use_loss=True)
    for rows, clean in ((frame_oracle(q, x), clean_c), (_np_report(q, x), clean_n)):
        # (rho' of a NaN is clamped to DBL_MIN by the corrector's comparison, so H_tt and mean_weight may stay finite)
        fields = [FN.COST, FN.CHI, FN.MEAN_E, FN.RMS_E, FN.MAX_E] + list(range(FN.G6, FN.ROW))
        assert np.all(np.isnan(rows[1, fields])) and np.any(np.isnan(rows[1, FN.H21:FN.G6]))
        np.testing.assert_array_equal(rows[[0, 2]], clean[[0, 2]])
