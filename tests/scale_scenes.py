"""Bench-sized scenes for tests/test_gpu_at_scale.py, and the long-double references spread over the host's cores.

The references of tests/exact_sums.py, tests/frame_exact.py and tests/loss_reference.py are linear in frames: the sums (and their
magnitudes) of two frame ranges add up to those of both, exactly up to the long-double rounding of one addition.  `spread` cuts a
problem into frame ranges of about equal point counts and evaluates them in forked worker processes, which read the host arrays
of the parent without copying them.  Test infrastructure only.
"""
from __future__ import annotations

import multiprocessing as mp
import os

import numpy as np

import exact_sums as X
import frame_exact as F
import loss_reference as LR

# (n_frames, beams, with_edges) of the scenes; every one is Problem.synthetic(..., seed=SEED, sigma=SIGMA)
SCENES = {"S1": (10_000, 1_000, False),      # configs[1]
          "S2": (100_000, 2_000, False),     # configs[2]
          "S3": (100, 2_000_000, False),     # deep lanes: every frame spans ~16 warp ranges
          "S2e": (100_000, 2_000, True)}     # configs[2] with the board-edge residuals (config 5)
SEED, SIGMA, A = 1, 0.01, 0.05

_DATA = {}  # frame_pose, offsets, points, edge_points of the problem being referenced (read by the forked workers)


def workers():
    return max(1, len(os.sched_getaffinity(0)))


def _slice(a, b):
    fp, off, pts, edge = _DATA["arrays"]
    oa, ob = int(off[a]), int(off[b])
    return fp[a:b], off[a:b + 1] - oa, pts[oa:ob], None if edge is None else edge[a:b]


def _job(items):
    """items: (what, frame_begin, frame_end, args) -> the reference of that frame range."""
    out = []
    for what, a, b, args in items:
        fp, off, pts, edge = _slice(a, b)
        if what == "lm":  # args: pose, loss kind, with edges
            pose, kind, edges = args
            out.append(LR.lm_sums(fp, off, pts, pose, kind, A, edge if edges else None))
        elif what == "frames":  # args: pose, use_loss (Cauchy), with edges
            pose, use_loss, edges = args
            out.append(F.frame_sums(fp, off, pts, pose, use_loss, A, edge if edges else None))
        elif what == "cf":
            out.append(X.closed_form_sums(fp, off, pts))
        else:
            raise ValueError(what)
    return out


def _run(arrays, batches):
    _DATA["arrays"] = arrays
    try:
        n = min(workers(), len(batches))
        if n <= 1:
            return [r for b in batches for r in _job(b)]
        with mp.get_context("fork").Pool(n) as pool:
            return [r for rs in pool.map(_job, batches, chunksize=1) for r in rs]
    finally:
        _DATA.clear()


def chunks(offsets, pieces):
    """Frame boundaries [0, ..., N] cutting the problem into about `pieces` ranges of equal point counts."""
    off = np.asarray(offsets, dtype=np.int64)
    N, P = len(off) - 1, int(off[-1])
    cut = np.searchsorted(off, np.linspace(0, P, pieces + 1).astype(np.int64), side="left")
    return np.unique(np.concatenate([[0], np.clip(cut, 0, N), [N]]))


def spread(arrays, what, args=None):
    """The reference `what` ("lm" -> (val, mag) of the 28 sums, "frames" -> per-frame (val, mag), "cf" -> the 54 closed-form
    sums) of the whole problem, from frame ranges evaluated in parallel."""
    cut = chunks(arrays[1], 4 * workers())
    parts = _run(arrays, [[(what, int(a), int(b), args)] for a, b in zip(cut[:-1], cut[1:])])
    if what == "frames":
        return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    val = sum((p[0] for p in parts), np.zeros_like(parts[0][0]))
    mag = sum((p[1] for p in parts), np.zeros_like(parts[0][1]))
    return val, mag


def segment_sums(arrays, seg_offsets, poses, kind):
    """lm_sums of every segment [seg_offsets[s], seg_offsets[s + 1]) at its own pose poses[s] under the loss `kind`, without
    edges: [W] (val, mag), in segment order."""
    off = np.asarray(seg_offsets, dtype=np.int64)
    items = [("lm", int(off[s]), int(off[s + 1]), (poses[s], kind, False)) for s in range(len(off) - 1)]
    k = min(len(items), 4 * workers())
    cut = np.linspace(0, len(items), k + 1).astype(np.int64)
    return _run(arrays, [items[a:b] for a, b in zip(cut[:-1], cut[1:]) if b > a])


def totals(val, mag):
    """The 28 sums (kernel order) of a whole problem from its per-frame reference (frame_exact COLUMNS)."""
    idx = list(range(F.C_H, F.C_H + 21)) + list(range(F.C_G, F.C_G + 6)) + [F.C_COST]
    return val[:, idx].sum(axis=0), mag[:, idx].sum(axis=0)


H_TT = ((0, 0, 0), (1, 0, 1), (2, 0, 2), (6, 1, 1), (7, 1, 2), (11, 2, 2))  # (H21 index, i, j) of the six H_tt entries


def frame_plane_slack(frame_pose, offsets):
    """Per frame, what the rounding of its board plane adds to the H_tt magnitudes of its row: the library rounds the plane once
    (|n| = 1) and exact_sums' A does not carry that input rounding.  |dH_ij / dn| |n| = (|n_i| + |n_j|) s^2 sum w <= |n_i| + |n_j|,
    as test_gpu_segments.plane_slack adds per segment; it matters in a frame whose normal has a tiny component.  [N, K]."""
    off = np.asarray(offsets, dtype=np.int64)
    n = np.abs(np.asarray(X.frame_planes(frame_pose), dtype=np.float64)[:, :3])
    slack = np.zeros((len(off) - 1, F.K))
    live = np.diff(off) > 0
    for k, i, j in H_TT:
        slack[live, F.C_H + k] = n[live, i] + n[live, j]
    return slack


def lane_depth(offsets, per_warp):
    """The most points one lane adds before its moments leave it: a lane takes 2 of every 64 points of its warp range and keeps
    adding until the frame or the warp range ends."""
    off = np.asarray(offsets, dtype=np.int64)
    P = int(off[-1])
    cuts = np.union1d(np.union1d(off, np.arange(0, P, int(per_warp), dtype=np.int64)), [P])
    return int(-(-np.diff(cuts).max() // 32)) if P else 0


def split_ranges(offsets, per_warp):
    """(frames per warp range [n_ranges], whether a frame crosses into or out of the range [n_ranges])."""
    off = np.asarray(offsets, dtype=np.int64)
    P = int(off[-1])
    lo = np.arange(0, P, int(per_warp), dtype=np.int64)
    hi = np.minimum(lo + int(per_warp), P)
    first = np.searchsorted(off, lo, side="right") - 1
    last = np.searchsorted(off, hi - 1, side="right") - 1
    n_frames = last - first + 1 - _empty_between(off, first, last)
    crosses = (off[first] < lo) | (off[last + 1] > hi)
    return n_frames, crosses


def _empty_between(off, first, last):
    empty = np.concatenate([[0], np.cumsum(np.diff(off) == 0)])
    return empty[last + 1] - empty[first]
