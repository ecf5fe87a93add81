"""CPU tests of the subset plan (csrc/clc_subset_plan.h, compiled with g++ from the source the library uses): from the source
shards' frame offsets and a keep mask, the new offsets, the new -> old frame map, the destination shard ranges of a group and the
copy runs of the gather kernel, against a numpy restatement.  Also: the subset entry points reject NULL arguments without a GPU."""
import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

import layouts as LY

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEG_FIELDS = 8  # src_shard, dst_shard, src_frame, dst_frame, n_frames, src_point, dst_point, n_points

SHIM = r'''
#include "clc_subset_plan.h"
extern "C" void shard(long long n, const long long* off, int nr, int r, long long* b, long long* e) {
  int64_t bb = 0, ee = 0;
  clc::balanced_shard_range(n, reinterpret_cast<const int64_t*>(off), nr, r, &bb, &ee);
  *b = bb; *e = ee;
}
extern "C" void plan(int n_src, const long long* frames, const long long* all_off, const unsigned char* keep, int n_dst,
                     long long* offsets, long long* map, long long* shard_frame, long long* seg, long long* sizes) {
  std::vector<const int64_t*> ptr;
  const int64_t* o = reinterpret_cast<const int64_t*>(all_off);
  for (int s = 0; s < n_src; ++s) { ptr.push_back(o); o += frames[s] + 1; }
  const clc::SubsetPlan p = clc::subset_plan(n_src, ptr.data(), reinterpret_cast<const int64_t*>(frames), keep, n_dst);
  for (size_t i = 0; i < p.offsets.size(); ++i) offsets[i] = p.offsets[i];
  for (size_t i = 0; i < p.frame_map.size(); ++i) map[i] = p.frame_map[i];
  for (size_t i = 0; i < p.shard_frame.size(); ++i) shard_frame[i] = p.shard_frame[i];
  for (size_t i = 0; i < p.segments.size(); ++i) {
    const clc::SubsetSegment& c = p.segments[i];
    const long long v[8] = {c.src_shard, c.dst_shard, c.src_frame, c.dst_frame, c.n_frames, c.src_point, c.dst_point, c.n_points};
    for (int k = 0; k < 8; ++k) seg[8 * i + k] = v[k];
  }
  sizes[0] = (long long)p.frame_map.size();
  sizes[1] = (long long)p.segments.size();
}
'''


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("subsetplan")
    src = d / "plan.cpp"
    src.write_text(SHIM)
    out = str(d / "libplan.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I",
                    os.path.join(ROOT, "camlasercalibratool_b200", "csrc"), str(src), "-o", out], check=True)
    L = C.CDLL(out)
    ll = C.POINTER(C.c_longlong)
    L.shard.argtypes = [C.c_longlong, ll, C.c_int, C.c_int, ll, ll]
    L.plan.argtypes = [C.c_int, ll, ll, C.POINTER(C.c_ubyte), C.c_int, ll, ll, ll, ll, ll]
    return L


def _ll(a):
    return a.ctypes.data_as(C.POINTER(C.c_longlong))


def run_plan(lib, shard_offsets, keep, n_dst):
    frames = np.array([len(o) - 1 for o in shard_offsets], dtype=np.int64)
    all_off = np.concatenate([np.asarray(o, dtype=np.int64) for o in shard_offsets])
    keep = np.ascontiguousarray(keep, dtype=np.uint8)
    assert keep.size == frames.sum()
    N = int(frames.sum())
    offsets, fmap = np.zeros(N + 1, dtype=np.int64), np.zeros(max(N, 1), dtype=np.int64)
    shard_frame, seg = np.zeros(n_dst + 1, dtype=np.int64), np.zeros(max(N, 1) * SEG_FIELDS, dtype=np.int64)
    sizes = np.zeros(2, dtype=np.int64)
    lib.plan(len(shard_offsets), _ll(frames), _ll(all_off), keep.ctypes.data_as(C.POINTER(C.c_ubyte)), n_dst, _ll(offsets),
             _ll(fmap), _ll(shard_frame), _ll(seg), _ll(sizes))
    K, S = int(sizes[0]), int(sizes[1])
    return offsets[:K + 1], fmap[:K], shard_frame, seg[:S * SEG_FIELDS].reshape(S, SEG_FIELDS)


def numpy_shard_ranges(offsets, G):
    """clc_shard_range restated: boundary r = first frame whose start >= r * P // G."""
    off = np.asarray(offsets, dtype=np.int64)
    N, P = len(off) - 1, int(off[-1])
    bounds = [0] + [int(np.searchsorted(off, P * r // G, side="left")) for r in range(1, G)] + [N]
    return np.maximum.accumulate(np.array(bounds, dtype=np.int64))


def check_plan(lib, shard_offsets, keep, n_dst, what=""):
    """The plan against the numpy restatement: every field, and the runs copy every destination point (and frame) exactly once
    from the right source point (frame), merged as far as the shards allow."""
    keep = np.asarray(keep, dtype=bool)
    offsets, fmap, shard_frame, seg = run_plan(lib, shard_offsets, keep, n_dst)
    counts = np.concatenate([np.diff(np.asarray(o, dtype=np.int64)) for o in shard_offsets])
    shard_of = np.concatenate([np.full(len(o) - 1, s) for s, o in enumerate(shard_offsets)]).astype(np.int64)
    local_frame = np.concatenate([np.arange(len(o) - 1) for o in shard_offsets]).astype(np.int64)
    local_start = np.concatenate([np.asarray(o, dtype=np.int64)[:-1] for o in shard_offsets])
    kept = np.nonzero(keep)[0]
    assert np.array_equal(fmap, kept), what
    new_off = np.concatenate([[0], np.cumsum(counts[kept])]).astype(np.int64)
    assert np.array_equal(offsets, new_off), what
    assert np.array_equal(shard_frame, numpy_shard_ranges(new_off, n_dst)), what
    K = len(kept)
    # coverage: destination (shard, local point) -> source (shard, local point), and the same for frames
    got_pt = {d: np.full(new_off[shard_frame[d + 1]] - new_off[shard_frame[d]], -1, dtype=np.int64) for d in range(n_dst)}
    got_fr = np.full(K, -1, dtype=np.int64)
    src_pt_of = {}
    last_dst = -1
    for s_sh, d_sh, s_fr, d_fr, nf, s_pt, d_pt, npt in seg:
        assert 0 <= d_sh < n_dst and d_sh >= last_dst and nf >= 1, what
        last_dst = d_sh
        g0 = shard_frame[d_sh] + d_fr  # new global frame of the run's first frame
        assert np.all(got_fr[g0:g0 + nf] == -1), what
        got_fr[g0:g0 + nf] = np.arange(nf) + s_fr
        src = kept[g0:g0 + nf]
        assert np.all(shard_of[src] == s_sh) and np.array_equal(local_frame[src], np.arange(nf) + s_fr), what
        assert s_pt == local_start[src[0]] and npt == counts[src].sum(), what
        assert d_pt == new_off[g0] - new_off[shard_frame[d_sh]], what
        assert np.all(got_pt[d_sh][d_pt:d_pt + npt] == -1), what
        got_pt[d_sh][d_pt:d_pt + npt] = s_pt + np.arange(npt)
        src_pt_of.setdefault(d_sh, []).append(s_sh)
    assert np.all(got_fr >= 0), what
    # every destination point has exactly one source, and it is the right one
    for d in range(n_dst):
        fb, fe = shard_frame[d], shard_frame[d + 1]
        want = np.concatenate([local_start[f] + np.arange(counts[f]) for f in kept[fb:fe]] or [np.zeros(0, dtype=np.int64)])
        assert np.array_equal(got_pt[d], want), what
    # runs are maximal: two consecutive runs of one destination shard could not have been merged
    for a, b in zip(seg[:-1], seg[1:]):
        assert not (a[1] == b[1] and a[0] == b[0] and a[2] + a[4] == b[2]), what
    return offsets, fmap, shard_frame, seg


def shards_by_points(counts, G):
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    b = numpy_shard_ranges(off, G)
    return [np.concatenate([[0], np.cumsum(counts[b[i]:b[i + 1]])]).astype(np.int64) for i in range(G)]


def shards_by_frames(counts, G):
    N = len(counts)
    return [np.concatenate([[0], np.cumsum(counts[N * i // G:N * (i + 1) // G])]).astype(np.int64) for i in range(G)]


MASKS = ["all", "none", "alternating", "only_empty", "first", "last", "one", "random10", "random50", "random90"]


def mask(name, counts, rng):
    N = len(counts)
    k = np.zeros(N, dtype=bool)
    if name == "all":
        k[:] = True
    elif name == "alternating":
        k[::2] = True
    elif name == "only_empty":
        k = counts == 0
    elif name == "first":
        k[:1] = True
    elif name == "last":
        k[-1:] = True
    elif name == "one":
        k[N // 3] = True
    elif name.startswith("random"):
        k = rng.random(N) < int(name[6:]) / 100
    return k


@pytest.mark.parametrize("name", MASKS)
def test_masks_on_one_shard(lib, name):
    rng = np.random.default_rng(5)
    counts = rng.integers(0, 40, size=300)
    counts[rng.random(300) < 0.2] = 0  # empty frames, some of them in runs
    counts[:3] = 0
    check_plan(lib, [np.concatenate([[0], np.cumsum(counts)])], mask(name, counts, rng), 1, name)


def test_keep_none_and_no_frames(lib):
    offsets, fmap, shard_frame, seg = check_plan(lib, [np.array([0, 5, 5, 9])], np.zeros(3, dtype=bool), 3)
    assert offsets.tolist() == [0] and len(fmap) == 0 and shard_frame.tolist() == [0, 0, 0, 0] and len(seg) == 0
    offsets, fmap, shard_frame, seg = check_plan(lib, [np.array([0]), np.array([0])], np.zeros(0, dtype=bool), 2)
    assert offsets.tolist() == [0] and len(seg) == 0


def test_keep_all_is_one_run_per_shard(lib):
    counts = np.random.default_rng(1).integers(0, 50, size=200)
    off = [np.concatenate([[0], np.cumsum(counts)])]
    seg = check_plan(lib, off, np.ones(200, dtype=bool), 1)[3]
    assert len(seg) == 1 and seg[0].tolist() == [0, 0, 0, 0, 200, 0, 0, counts.sum()]


def test_runs_straddling_source_shards(lib):
    """A kept run crossing a source shard boundary is split there; a destination shard fed by three source shards."""
    counts = np.full(60, 10, dtype=np.int64)
    src = shards_by_frames(counts, 4)  # 15 frames per source shard
    keep = np.zeros(60, dtype=bool)
    keep[10:50] = True  # frames 10-49: the tail of shard 0, all of shards 1 and 2, the head of shard 3
    offsets, fmap, shard_frame, seg = check_plan(lib, src, keep, 1)
    assert [tuple(s[[0, 2, 4]]) for s in seg] == [(0, 10, 5), (1, 0, 15), (2, 0, 15), (3, 0, 5)]
    # the same into two destination shards
    offsets, fmap, shard_frame, seg = check_plan(lib, src, keep, 2)
    assert shard_frame.tolist() == [0, 20, 40]
    assert sorted({int(s[0]) for s in seg if s[1] == 0}) == [0, 1] and sorted({int(s[0]) for s in seg if s[1] == 1}) == [2, 3]
    # eight source shards of 7-8 frames: the first destination shard (frames 10-29) takes frames of three of them
    seg = check_plan(lib, shards_by_frames(counts, 8), keep, 2)[3]
    assert sorted({int(s[0]) for s in seg if s[1] == 0}) == [1, 2, 3]
    # and a destination shard whose frames come from three source shards, with drops inside
    keep2 = keep.copy()
    keep2[[12, 20, 33, 47]] = False
    check_plan(lib, src, keep2, 1)
    check_plan(lib, src, keep2, 3)


def test_shard_ranges_match_the_library(lib):
    """balanced_shard_range is clc_shard_range (libclc_b200.so, host code) and the numpy restatement."""
    from camlasercalibratool_b200 import shard_range

    rng = np.random.default_rng(3)
    for G in range(1, 9):
        cnt = rng.integers(0, 200, size=int(rng.integers(0, 400)))
        cnt[rng.random(cnt.size) < 0.1] = 0
        off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        want = numpy_shard_ranges(off, G)
        for r in range(G):
            b, e = C.c_longlong(), C.c_longlong()
            lib.shard(len(cnt), _ll(off), G, r, C.byref(b), C.byref(e))
            assert (b.value, e.value) == shard_range(len(cnt), G, r, off) == (want[r], want[r + 1])


def _layout_counts(name):
    """Frame sizes of a tests/layouts.py layout cut for the full grid of an H100 (132 blocks), without its points."""
    base = SimpleNamespace(n_frames=1, offsets=np.array([0, 1]), points=np.zeros((1, 3)), frame_pose=np.zeros((1, 7)),
                           edge_points=None)
    grid, per_warp = LY.partition(132 * 12 * 256 * 3, 132, LY.STAGE_GENERAL)
    return np.diff(LY.build(name, base, grid, per_warp, LY.STAGE_GENERAL).offsets)


@pytest.mark.parametrize("name", ["L2_off_by_one", "L3_empty_runs", "L4_giant_frame", "L5_confetti", "L7_heavy_tailed"])
def test_groups_of_one_to_eight_on_ragged_layouts(lib, name):
    """Source groups of 1, 3 and 8 shards, split by points (from_frames) or by frames (synthetic), into 1 ... 8 shards."""
    counts = _layout_counts(name)
    rng = np.random.default_rng(len(name))
    masks = ("random10", "random50", "random90", "alternating")
    for G in range(1, 9):
        G_src, split, m = (1, 3, 8)[G % 3], (shards_by_points, shards_by_frames)[G % 2], masks[G % 4]
        check_plan(lib, split(counts, G_src), mask(m, counts, rng), G, f"{name}/{G_src}/{split.__name__}/{m}/{G}")


def test_subset_entry_points_reject_null_arguments():
    """Argument checks come before any device work, so they answer without a GPU too."""
    from camlasercalibratool_b200 import _lib

    L = _lib.load()
    out = C.c_void_p()
    keep = (C.c_uint8 * 1)(1)
    for fn, name in ((L.clc_problem_subset, "clc_problem_subset"), (L.clc_group_subset, "clc_group_subset")):
        assert fn(None, keep, C.byref(out)) == 1, name  # CLC_ERR_INVALID
        assert b"NULL" in L.clc_last_error(), name
        assert out.value is None
    ms = (C.c_float * 1)()
    assert L.clc_bench_subset(None, keep, 1, 1, ms) == 1
