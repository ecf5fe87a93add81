"""Adversarial frame layouts for the sweep kernel's static work partition.

The sweep kernel cuts the P points into equal warp ranges of `per_warp` points (whole pipeline stages of `stage` points),
12 warps per block, `grid` blocks (partition() in csrc/clc_api.cu).  Each layout here places frame boundaries, empty frames
and huge frames exactly where that bookkeeping changes state -- stage, warp-range and block-range ends, the first and last
point of a range, the partial last warp, warps with no work -- for a given (grid, per_warp, stage).  Every builder returns
the boundary kinds it was meant to hit; `classify` recomputes which kinds a problem really hits under a given partition,
so a test can assert that the layout still hits them on the device in use (a different SM count cannot quietly weaken it).

The points and board poses come from an `oracle.generate` problem: frames are re-cut, and frame f takes the board pose of
base frame f mod n_base and that frame's points, cyclically.  Test infrastructure only.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

WARPS = 12                    # warps per block (kThreads = 384)
SINGLE_BLOCK_MAX = 12 * 8 * 128  # partition(): problems up to this size run on one block
SMALL_MAX_RESIDUALS = 16384   # the one-cluster kernel's limit (kSmallMaxResiduals)
STAGE_GENERAL, STAGE_PLANAR = 128, 256
L2_H100 = 50 * 1024 * 1024


def partition(n_points, grid_full, stage):
    """Python restatement of partition() in csrc/clc_api.cu: (grid, per_warp)."""
    grid = grid_full
    stages = -(-n_points // stage)
    grid = min(grid, max(1, -(-stages // WARPS)))
    if n_points <= SINGLE_BLOCK_MAX:
        grid = 1
    n_warps = grid * WARPS
    per_warp = max(stage, -(-(-(-n_points // n_warps)) // stage) * stage)
    return grid, per_warp


def resident_chunks(n_points, grid, per_warp, stage, l2_bytes=L2_H100):
    """clc_l2_plan.h at the default budget (half of L2)."""
    stage_bytes = (2 if stage == STAGE_PLANAR else 3) * stage * 8
    if grid <= 1 or n_points <= SMALL_MAX_RESIDUALS:
        return 0
    return min(per_warp // stage, int(l2_bytes * 0.5) // (grid * WARPS * stage_bytes))


def classify(offsets, grid, per_warp, stage):
    """The boundary kinds a problem with these frame offsets hits under the partition (grid, per_warp, stage)."""
    off = np.asarray(offsets, dtype=np.int64)
    P, N = int(off[-1]), len(off) - 1
    W, B = int(per_warp), int(per_warp) * WARPS
    n_warps = grid * WARPS
    counts = np.diff(off)
    tags = set()
    ends = off[1:N]
    ends = ends[(ends > 0) & (ends < P)]
    for d in (-1, 0, 1):
        v = ends - d
        for kind, mask in (("block", v % B == 0), ("warp", (v % W == 0) & (v % B != 0)),
                           ("stage", (v % stage == 0) & (v % W != 0))):
            if np.any(mask & (v > 0) & (v < P)):
                tags.add(f"end@{kind}{'' if d == 0 else f'{d:+d}'}")
    starts = off[:N]
    if np.any((starts % W == 0) & (counts == W)):
        tags.add("frame=warp_range")
    if N and counts.max() > B:
        tags.add("frame>block_range")
    empty = counts == 0
    if np.any(empty & (starts % W == 0) & (starts > 0) & (starts < P)):
        tags.add("empty_run@warp_start")
    if N and empty[0]:
        tags.add("leading_empty")
    if N and empty[-1]:
        tags.add("trailing_empty")
    if ends.size and np.bincount(ends // stage).max() > 32:
        tags.add(">32_pieces_per_stage")
    if P <= (n_warps - 1) * W:
        tags.add("idle_warps")
    if P <= (n_warps - WARPS) * W:
        tags.add("idle_block")
    if P > (n_warps - 1) * W:
        tags.add("all_warps_busy")
    if P % stage == 1:
        tags.add("P%stage==1")
    if (P + 1) % (n_warps * stage) == 0:
        tags.add("P=k*warps*stage-1")
    if (P - 1) % (n_warps * stage) == 0:
        tags.add("P=k*warps*stage+1")
    if N == 1:
        tags.add("one_frame")
    last_warp = -(-P // W) - 1
    if N == 2 and P % W != 0 and last_warp * W < off[1] < P:
        tags.add("split_in_last_partial_warp")
    return tags


@dataclass
class Layout:
    name: str
    frame_pose: np.ndarray
    offsets: np.ndarray
    points: np.ndarray
    edge_points: np.ndarray | None
    targets: set = field(default_factory=set)
    general_only: bool = False  # z != 0: the planar kernels do not apply

    @property
    def n_points(self):
        return int(self.offsets[-1])

    def problem(self, oracle, use_loss=True, edges=False):
        return oracle.Problem(self.frame_pose, self.offsets, self.points, self.edge_points if edges else None,
                              use_loss=use_loss)


def recut(base, counts, name, targets, with_edges=True, z_sigma=0.0, seed=0):
    """Frame f of the new problem: board pose of base frame f mod n_base, that frame's points (cyclically)."""
    counts = np.asarray(counts, dtype=np.int64)
    assert counts.min() >= 0
    n_base = base.n_frames
    base_cnt = np.diff(base.offsets)
    assert base_cnt.min() > 0
    N = len(counts)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    b = np.arange(N) % n_base
    frame_of = np.repeat(np.arange(N), counts)
    local = np.arange(off[-1]) - off[:-1][frame_of]
    bf = b[frame_of]
    pts = base.points[base.offsets[bf] + local % base_cnt[bf]].copy()
    if z_sigma:
        pts[:, 2] = np.random.default_rng(seed).normal(size=len(pts)) * z_sigma
    edge = base.edge_points[b].copy() if with_edges and base.edge_points is not None else None
    return Layout(name, base.frame_pose[b].copy(), off, pts, edge, set(targets), general_only=bool(z_sigma))


def _counts_from_cuts(cuts, P):
    """Frame sizes from a set of cut positions (0 < cut < P; repeats make empty frames)."""
    c = np.sort(np.asarray(list(cuts), dtype=np.int64))
    c = c[(c >= 0) & (c <= P)]
    return np.diff(np.concatenate([[0], c, [P]]))


def _fill(rng, total, lo, hi):
    """Random frame sizes in [lo, hi] adding up to exactly `total`."""
    out, s = [], 0
    while s < total:
        k = int(min(rng.integers(lo, hi + 1), total - s))
        out.append(k)
        s += k
    return out


BLOCK_TAGS = {"end@block", "end@block+1", "end@block-1", "idle_block", "frame>block_range"}


def build(name, base, grid, per_warp, stage, seed=0):
    """Layout `name` (L1 ... L7 and their variants, see LAYOUTS) for the partition (grid, per_warp, stage).  A single-block
    grid has no block boundary inside the problem: the block-level targets are dropped there."""
    lay = _build(name, base, grid, per_warp, stage, seed)
    if grid == 1:
        lay.targets -= BLOCK_TAGS | {"partial_resident"}
    return lay


def _build(name, base, grid, per_warp, stage, seed):
    rng = np.random.default_rng(seed)
    W = per_warp
    B = W * WARPS
    n_warps = grid * WARPS
    full = n_warps * W
    inner = W > stage  # warp ranges of several stages: stage ends inside a range exist
    if name == "L1_aligned":
        P = full
        cuts = {k * B for k in range(1, grid)} | {w * W for w in range(1, n_warps) if w % 3 != 2}
        cuts |= {w * W + j * stage for w in range(n_warps) if w % 5 == 1 for j in range(1, W // stage)}
        t = {"end@block", "end@warp", "frame=warp_range"} | ({"end@stage"} if inner else set())
        return recut(base, _counts_from_cuts(cuts, P), name, t)
    if name == "L2_off_by_one":
        P = full - 1
        cuts = {k * B + (1 if k % 2 else -1) for k in range(1, grid)}
        cuts |= {w * W + (1 if w % 2 else -1) for w in range(1, n_warps) if w % WARPS}
        cuts |= {w * W + j * stage + (1 if w % 4 == 1 else -1) for w in range(n_warps) if w % 2 == 1 for j in range(1, W // stage)}
        cuts |= {w * W + 1 + 2 * int(rng.integers(1, W // 2 - 1)) for w in range(0, n_warps, 7)}  # odd starts inside ranges
        t = {"end@block+1", "end@block-1", "end@warp+1", "end@warp-1"} | ({"end@stage+1", "end@stage-1"} if inner else set())
        return recut(base, _counts_from_cuts(cuts, P), name, t)
    if name == "L3_empty_runs":
        P = full - 37
        sizes = _fill(rng, P, 50, 400)
        off = np.concatenate([[0], np.cumsum(sizes)])
        cuts = list(off[1:-1]) + [w * W for w in range(1, n_warps) if w % 4 == 0]
        counts = list(_counts_from_cuts(cuts, P))
        # runs of 1-50 empty frames in front of the frames that start at a warp range (and elsewhere)
        starts = np.concatenate([[0], np.cumsum(counts)])[:-1]
        out = [0] * int(rng.integers(1, 51))  # leading empty frames: offsets 0, 0, ...
        for s, c in zip(starts, counts):
            if (s % W == 0 and s > 0) or rng.random() < 0.02:
                out += [0] * int(rng.integers(1, 51))
            out.append(int(c))
        out += [0] * int(rng.integers(1, 51))  # trailing empty frames: offsets P, P, ...
        return recut(base, out, name, {"empty_run@warp_start", "leading_empty", "trailing_empty"})
    if name == "L4_giant_frame":
        P = full - 100
        head = _fill(rng, max(0, grid // 2 - 1) * B + 3, 1, 700)  # the giant frame starts at an odd offset
        giant = min(B + B // 2 + 7, P - sum(head) - 1)
        tail = _fill(rng, P - sum(head) - giant, 100, 700)
        return recut(base, head + [giant] + tail, name, {"frame>block_range"})
    if name == "L4_one_frame":
        return recut(base, [full - 3], name, {"one_frame", "frame>block_range"})
    if name == "L4_two_frames":
        P = full - W // 2 - 1
        last = (-(-P // W) - 1) * W
        return recut(base, [last + (P - last) // 2 + 1, P - last - (P - last) // 2 - 1], name, {"split_in_last_partial_warp"})
    if name == "L5_confetti":
        P = full - 5
        half = P // 2 // 2 * 2
        sizes = [2] * (half // 2) + _fill(rng, P - half, 1, 3)
        return recut(base, sizes, name, {">32_pieces_per_stage", "all_warps_busy"})
    if name == "L6_short_tail":
        # the last block and one more warp have no stage at all.  With one stage per warp range the grid shrinks to the
        # blocks there are stages for (partition()), so there only the last warp can be idle; likewise on a single block.
        idle_block = grid > 1 and inner
        P = (n_warps - (WARPS + 1 if idle_block else 2)) * W + 1
        return recut(base, _fill(rng, P, 1, 700), name, {"P%stage==1", "idle_warps"} | ({"idle_block"} if idle_block else set()))
    if name == "L6_jump_below":
        P = n_warps * stage * (W // stage) - 1
        return recut(base, _fill(rng, P, 1, 700), name, {"P=k*warps*stage-1", "all_warps_busy"})
    if name == "L6_jump_above":
        P = n_warps * stage * (W // stage) + 1  # per_warp grows by one stage: a long tail of idle warps
        return recut(base, _fill(rng, P, 1, 700), name, {"P=k*warps*stage+1", "idle_warps", "P%stage==1"})
    if name in ("L7_heavy_tailed", "L7_heavy_tailed_z"):
        counts = np.minimum(5000, np.floor(rng.pareto(1.2, size=200_000) * 60)).astype(np.int64)
        counts = counts[np.cumsum(counts) <= 1_300_000]
        z = name.endswith("_z")
        # general family: 7 stages per warp, 5 of them resident in half of a 50 MB L2 (planar: 4 of 4)
        t = {"partial_resident"} if stage == STAGE_GENERAL and not z else set()
        return recut(base, counts, name, t, z_sigma=0.3 if z else 0.0, seed=seed)
    raise KeyError(name)


LAYOUTS = ["L1_aligned", "L2_off_by_one", "L3_empty_runs", "L4_giant_frame", "L4_one_frame", "L4_two_frames", "L5_confetti",
           "L6_short_tail", "L6_jump_below", "L6_jump_above", "L7_heavy_tailed", "L7_heavy_tailed_z"]


def base_problem(oracle, seed=21):
    """The board poses and points the layouts re-cut: 200 boards x 1000 beams, sigma = 1 cm, with edge points."""
    return oracle.generate(200, 1000, seed=seed, sigma=0.01, exact_m=True, with_edges=True)
