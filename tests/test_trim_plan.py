"""CPU tests of the trim plan (csrc/clc_trim_plan.h, compiled with g++ from the source the library uses): from the kept counts of
every source frame and every source tile, the new offsets, the destination shard ranges of a group and the first source tile of
every destination tile, against a numpy restatement.  Also: the Python threshold checks and the NULL-argument checks of the trim
entry points, which answer without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import layouts as LY
from test_subset_plan import _layout_counts, numpy_shard_ranges

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 2048  # clc::kTrimTile

SHIM = r'''
#include "clc_trim_plan.h"
extern "C" long long tile() { return clc::kTrimTile; }
extern "C" void plan(int n_src, const long long* frames, const long long* all_fk, const long long* tiles, const long long* all_tk,
                     int n_dst, long long* offsets, long long* shard_frame, long long* tile_prefix, long long* tile_begin,
                     long long* first_tile) {
  std::vector<const int64_t*> fk, tk;
  const int64_t* f = reinterpret_cast<const int64_t*>(all_fk);
  const int64_t* t = reinterpret_cast<const int64_t*>(all_tk);
  for (int s = 0; s < n_src; ++s) { fk.push_back(f); f += frames[s]; tk.push_back(t); t += tiles[s]; }
  const clc::TrimPlan p = clc::trim_plan(n_src, reinterpret_cast<const int64_t*>(frames), fk.data(),
                                         reinterpret_cast<const int64_t*>(tiles), tk.data(), n_dst);
  for (size_t i = 0; i < p.offsets.size(); ++i) offsets[i] = p.offsets[i];
  for (size_t i = 0; i < p.shard_frame.size(); ++i) shard_frame[i] = p.shard_frame[i];
  for (size_t i = 0; i < p.tile_prefix.size(); ++i) tile_prefix[i] = p.tile_prefix[i];
  for (size_t i = 0; i < p.tile_begin.size(); ++i) tile_begin[i] = p.tile_begin[i];
  for (size_t i = 0; i < p.first_tile.size(); ++i) first_tile[i] = p.first_tile[i];
}
'''


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("trimplan")
    src = d / "plan.cpp"
    src.write_text(SHIM)
    out = str(d / "libplan.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I",
                    os.path.join(ROOT, "camlasercalibratool_b200", "csrc"), str(src), "-o", out], check=True)
    L = C.CDLL(out)
    ll = C.POINTER(C.c_longlong)
    L.tile.restype = C.c_longlong
    L.plan.argtypes = [C.c_int, ll, ll, ll, ll, C.c_int, ll, ll, ll, ll, ll]
    assert L.tile() == TILE
    return L


def _ll(a):
    return a.ctypes.data_as(C.POINTER(C.c_longlong))


def run_plan(lib, frame_kept, tile_kept, n_dst):
    """frame_kept / tile_kept: one array per source shard."""
    frames = np.array([len(f) for f in frame_kept], dtype=np.int64)
    tiles = np.array([len(t) for t in tile_kept], dtype=np.int64)
    fk = np.concatenate([np.asarray(f, dtype=np.int64) for f in frame_kept] + [np.zeros(1, dtype=np.int64)])
    tk = np.concatenate([np.asarray(t, dtype=np.int64) for t in tile_kept] + [np.zeros(1, dtype=np.int64)])
    N, T, K = int(frames.sum()), int(tiles.sum()), int(fk.sum())
    offsets, shard_frame, tile_prefix = np.zeros(N + 1, dtype=np.int64), np.zeros(n_dst + 1, dtype=np.int64), np.zeros(T + 1, dtype=np.int64)
    tile_begin = np.zeros(n_dst + 1, dtype=np.int64)
    first_tile = np.full(K // TILE + n_dst + 1, -7, dtype=np.int64)
    lib.plan(len(frame_kept), _ll(frames), _ll(fk), _ll(tiles), _ll(tk), n_dst, _ll(offsets), _ll(shard_frame), _ll(tile_prefix),
             _ll(tile_begin), _ll(first_tile))
    return offsets, shard_frame, tile_prefix, tile_begin, first_tile[:tile_begin[-1]]


def check_plan(lib, frame_kept, tile_kept, n_dst, what=""):
    """The plan against the numpy restatement, and the property the gather relies on: destination tile t's first kept point
    lies in its first source tile, and every source tile before that one has its kept points before the destination tile."""
    offsets, shard_frame, tile_prefix, tile_begin, first_tile = run_plan(lib, frame_kept, tile_kept, n_dst)
    fk = np.concatenate([np.asarray(f, dtype=np.int64) for f in frame_kept] + [np.zeros(0, dtype=np.int64)])
    tk = np.concatenate([np.asarray(t, dtype=np.int64) for t in tile_kept] + [np.zeros(0, dtype=np.int64)])
    assert fk.sum() == tk.sum(), "the counts of one mark pass agree"
    want_off = np.concatenate([[0], np.cumsum(fk)]).astype(np.int64)
    assert np.array_equal(offsets, want_off), what
    want_prefix = np.concatenate([[0], np.cumsum(tk)]).astype(np.int64)
    assert np.array_equal(tile_prefix, want_prefix), what
    assert np.array_equal(shard_frame, numpy_shard_ranges(want_off, n_dst)), what
    want_first, want_begin = [], [0]
    for d in range(n_dst):
        p0, p1 = want_off[shard_frame[d]], want_off[shard_frame[d + 1]]
        for start in range(int(p0), int(p1), TILE):
            g = int(np.searchsorted(want_prefix[1:], start, side="right"))  # the tile holding kept point `start`
            assert want_prefix[g] <= start < want_prefix[g + 1], what
            want_first.append(g)
        want_begin.append(len(want_first))
    assert np.array_equal(tile_begin, want_begin), what
    assert np.array_equal(first_tile, want_first), what
    return offsets, shard_frame, tile_prefix, tile_begin, first_tile


def counts_from_keep(offsets, keep, shard_frames=None):
    """Per-frame and per-tile kept counts of a keep mask over the points of frames cut at `offsets`, as the mark pass of every
    source shard (frames split into shards of shard_frames[s] frames, each shard's points tiled from its own first point)."""
    offsets = np.asarray(offsets, dtype=np.int64)
    N = len(offsets) - 1
    shard_frames = [N] if shard_frames is None else shard_frames
    fks, tks, f0 = [], [], 0
    for n in shard_frames:
        a, b = offsets[f0], offsets[f0 + n]
        k = keep[a:b]
        ck = np.concatenate([[0], np.cumsum(k)]).astype(np.int64)
        fks.append(ck[offsets[f0 + 1:f0 + n + 1] - a] - ck[offsets[f0:f0 + n] - a])
        T = (b - a + TILE - 1) // TILE
        tks.append(np.array([int(k[t * TILE:(t + 1) * TILE].sum()) for t in range(T)], dtype=np.int64))
        f0 += n
    return fks, tks


KEEPS = ["all", "none", "random01", "random50", "random99", "runs", "every_other_tile"]


def keep_mask(name, P, rng):
    if name == "all":
        return np.ones(P, dtype=np.int64)
    if name == "none":
        return np.zeros(P, dtype=np.int64)
    if name.startswith("random"):
        return (rng.random(P) < int(name[6:]) / 100).astype(np.int64)
    if name == "runs":  # long kept and dropped runs
        k = np.zeros(P, dtype=np.int64)
        for a in rng.integers(0, max(P, 1), size=20):
            k[a:a + int(rng.integers(1, 5000))] = 1
        return k
    t = (np.arange(P) // TILE) % 2 == 0  # tiles with no kept point between full ones
    return t.astype(np.int64)


@pytest.mark.parametrize("name", KEEPS)
def test_keeps_on_one_shard(lib, name):
    rng = np.random.default_rng(5)
    counts = rng.integers(0, 700, size=300)
    counts[rng.random(300) < 0.2] = 0  # empty frames, some of them in runs
    counts[:3] = 0
    off = np.concatenate([[0], np.cumsum(counts)])
    fk, tk = counts_from_keep(off, keep_mask(name, int(off[-1]), rng))
    check_plan(lib, fk, tk, 1, name)


def test_random_counts(lib):
    """Per-frame and per-tile counts that only agree in their sum (the plan uses nothing else of them together)."""
    rng = np.random.default_rng(2)
    for _ in range(50):
        N, T = int(rng.integers(0, 200)), int(rng.integers(1, 60))
        tk = rng.integers(0, TILE + 1, size=T)
        tk[rng.random(T) < 0.3] = 0
        K = int(tk.sum())
        cuts = np.sort(rng.integers(0, K + 1, size=max(N - 1, 0)))
        fk = np.diff(np.concatenate([[0], cuts, [K]])) if N else np.zeros(0, dtype=np.int64)
        if N == 0:
            tk[:] = 0
        check_plan(lib, [fk], [tk], int(rng.integers(1, 9)), "random")


def test_no_points_and_no_frames(lib):
    offsets, shard_frame, tile_prefix, tile_begin, first_tile = check_plan(lib, [np.zeros(3, dtype=np.int64)], [np.zeros(2, dtype=np.int64)], 3)
    assert offsets.tolist() == [0, 0, 0, 0] and tile_prefix.tolist() == [0, 0, 0] and len(first_tile) == 0
    assert tile_begin.tolist() == [0, 0, 0, 0]
    check_plan(lib, [np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)], [np.zeros(0, dtype=np.int64)] * 2, 2)


def test_keep_all_maps_tiles_one_to_one(lib):
    counts = np.random.default_rng(1).integers(0, 500, size=200)
    off = np.concatenate([[0], np.cumsum(counts)])
    fk, tk = counts_from_keep(off, np.ones(int(off[-1]), dtype=np.int64))
    first_tile = check_plan(lib, fk, tk, 1)[4]
    assert first_tile.tolist() == list(range(len(tk[0])))


def split_frames(counts, G, by_points):
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    if by_points:
        b = numpy_shard_ranges(off, G)
    else:
        b = [len(counts) * i // G for i in range(G + 1)]
    return [int(b[i + 1] - b[i]) for i in range(G)]


@pytest.mark.parametrize("name", ["L2_off_by_one", "L3_empty_runs", "L4_giant_frame", "L5_confetti", "L7_heavy_tailed"])
def test_groups_of_one_to_eight_on_ragged_layouts(lib, name):
    """Source groups of 1, 3 and 8 shards, split by points (from_frames) or by frames (synthetic), each shard tiled from its own
    first point, trimmed and re-sharded over 1 ... 8 devices: shard boundaries move with the new point counts."""
    counts = _layout_counts(name)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    rng = np.random.default_rng(len(name))
    keeps = ("random50", "random99", "runs", "every_other_tile")
    for G in range(1, 9):
        G_src, by_points, k = (1, 3, 8)[G % 3], G % 2 == 0, keeps[G % 4]
        fk, tk = counts_from_keep(off, keep_mask(k, int(off[-1]), rng), split_frames(counts, G_src, by_points))
        check_plan(lib, fk, tk, G, f"{name}/{G_src}/{by_points}/{k}/{G}")


def test_thresholds_are_checked_in_python():
    """A scalar is broadcast; a wrong shape, NaN or a negative threshold raise ValueError before the library is called."""
    from camlasercalibratool_b200.api import _thresholds

    assert _thresholds(0.5, 3).tolist() == [0.5, 0.5, 0.5]
    assert _thresholds(np.inf, 2).tolist() == [np.inf, np.inf]
    assert _thresholds([0.0, 1.0], 2).dtype == np.float64
    for bad in (np.ones(2), np.ones((3, 1)), [[1.0, 2.0, 3.0]]):
        with pytest.raises(ValueError, match="shape"):
            _thresholds(bad, 3)
    for bad in (np.nan, -1.0, [0.1, np.nan, 0.2], [0.1, -0.0, -1e-300]):
        with pytest.raises(ValueError, match="NaN or negative"):
            _thresholds(bad, 3)
    assert _thresholds([0.1, -0.0, 0.2], 3)[1] == 0.0  # -0.0 is not negative


def test_trim_entry_points_reject_null_arguments():
    from camlasercalibratool_b200 import _lib

    L = _lib.load()
    out = C.c_void_p()
    pose = (C.c_double * 7)(0, 0, 0, 0, 0, 0, 1)
    tau = (C.c_double * 1)(1.0)
    for fn, name in ((L.clc_problem_trim, "clc_problem_trim"), (L.clc_group_trim, "clc_group_trim")):
        assert fn(None, pose, tau, C.byref(out)) == 1, name  # CLC_ERR_INVALID
        assert b"NULL" in L.clc_last_error(), name
        assert out.value is None
    ms = (C.c_float * 1)()
    assert L.clc_bench_trim(None, pose, tau, 1, 1, ms, ms) == 1
