"""Frame layouts for the reference-sized solve path: the one-cluster kernel K2 and the single-block sweep kernel.

K2 (csrc/clc_small.cuh) gives residual i to thread i mod 2048 of its cluster (8 CTAs x 256 threads), in item slot i / 2048
(8 slots, 16 384 residuals).  Points come first; edge residual e (frame e >> 1) follows at index P + e, and the edges of
empty frames are skipped.  `small_slot` and `k2_residuals` restate that mapping; `classify_small` reports the boundary kinds a
problem really hits under it: totals and the point/edge seam at slot, CTA and warp ends and one residual either side, idle
CTAs and slots, empty frames whose edges sit at the seam or at the end, one-point frames with edges, a single 16 384-point
frame and 16 384 one-point frames.  The single-block sweep kernel (partition() with grid 1: 12 warps, whole stages of 128
points, 256 for the planar kernels, up to 8 stages per warp, 12 288 points) is classified by `classify_single_block`, which
reuses the multi-block restatement of tests/layouts.py.

Every layout declares the tags it was cut to hit, prefixed "k2:" or "k1:"; tests check them against the classifiers and, on
the device, against clc_debug_partition and clc_debug_dispatch.  Test infrastructure only.
"""
from __future__ import annotations

import numpy as np

import exact_sums as X
import layouts as LY

SMALL_THREADS, SMALL_CLUSTER, SMALL_ITEMS = 256, 8, 8  # kSmallThreads, kSmallCluster, kSmallItems
SLOT = SMALL_THREADS * SMALL_CLUSTER                   # residuals per item slot (one per thread of the cluster)
SMALL_MAX = SLOT * SMALL_ITEMS                         # 16 384
WARP = 32
SINGLE_BLOCK_MAX = LY.SINGLE_BLOCK_MAX                 # 12 288

# residual totals and single-block point counts the layouts must cover between them
K2_TOTALS = {1, 2, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 14336, 16383, 16384}
K1_POINTS = {1, 12287, 12288, 12289}  # plus stage +- 1 and 12 * stage +- 1 of each family


def small_slot(i):
    """(cta, warp, lane, item slot) of K2's residual i."""
    i = np.asarray(i, dtype=np.int64)
    t = i % SLOT
    return t // SMALL_THREADS, (t % SMALL_THREADS) // WARP, t % WARP, i // SLOT


def small_residuals(offsets, edges):
    """(P, R, live): K2's residual count R (edge slots of empty frames included) and which of them exist."""
    off = np.asarray(offsets, dtype=np.int64)
    P, N = int(off[-1]), len(off) - 1
    R = P + (2 * N if edges else 0)
    live = np.ones(R, dtype=bool)
    if edges:
        live[P:] = np.repeat(np.diff(off) > 0, 2)
    return P, R, live


def k2_residuals(frame_pose, offsets, points, edge_points=None):
    """K2's residuals in its index order: plane [R,4], point [R,3], s2 [R] (long double) and live [R]."""
    off = np.asarray(offsets, dtype=np.int64)
    counts = np.diff(off)
    P, R, live = small_residuals(off, edge_points is not None)
    planes = X.frame_planes(frame_pose)
    s2f = np.zeros(len(counts), dtype=X.LD)
    s2f[counts > 0] = X.LD(1) / counts[counts > 0].astype(X.LD)
    frame_of = np.repeat(np.arange(len(counts)), counts)
    plane = np.zeros((R, 4), dtype=X.LD)
    point = np.zeros((R, 3), dtype=X.LD)
    s2 = np.zeros(R, dtype=X.LD)
    plane[:P], point[:P], s2[:P] = planes[frame_of], np.asarray(points, dtype=np.float64).astype(X.LD), s2f[frame_of]
    if edge_points is not None:
        e = np.arange(R - P)
        f = e >> 1
        plane[P:] = X.edge_planes(frame_pose)[f, e & 1]
        point[P:] = np.asarray(edge_points, dtype=np.float64).reshape(-1, 2, 3)[f, e & 1].astype(X.LD)
        s2[P:] = s2f[f]
    return plane, point, s2, live


def _unit_tags(what, v, tags):
    """what@slot / @cta / @warp (the largest unit that divides v - d), with d in -1, 0, +1."""
    for d in (-1, 0, 1):
        u = v - d
        if u <= 0:
            continue
        kind = "slot" if u % SLOT == 0 else "cta" if u % SMALL_THREADS == 0 else "warp" if u % WARP == 0 else None
        if kind:
            tags.add(f"{what}@{kind}{'' if d == 0 else f'{d:+d}'}")


def classify_small(offsets, edges):
    """The boundary kinds K2's slot mapping meets on this problem (with or without the edge residuals)."""
    off = np.asarray(offsets, dtype=np.int64)
    counts = np.diff(off)
    N = len(counts)
    P, R, live = small_residuals(off, edges)
    tags = set()
    if R > SMALL_MAX:
        if edges and P <= SMALL_MAX:
            tags.add("points<=small<residuals")
        return tags
    tags.add(f"total={R}")
    if R:
        _unit_tags("total", R, tags)
    if edges and N and 0 < P:
        _unit_tags("seam", P, tags)
    ends = off[1:N]
    for v in np.unique(ends[(ends > 0) & (ends < P)]):
        if v % WARP in (0, 1, WARP - 1):
            _unit_tags("frame_end", int(v), tags)
    if R <= (SMALL_CLUSTER - 1) * SMALL_THREADS:
        tags.add("idle_cta")
    tags.add("idle_slot" if R <= (SMALL_ITEMS - 1) * SLOT else "all_slots")
    if edges and N:
        if counts[0] == 0:
            tags.add("empty_edges@seam")
        if counts[-1] == 0:
            tags.add("empty_edges@end")
        if np.any(counts == 1):
            tags.add("one_point_frame_edges")
        if not live.all():
            tags.add("dead_edge_slots")
    if N and counts[0] == 0:
        tags.add("leading_empty")
    if N and counts[-1] == 0:
        tags.add("trailing_empty")
    if N == 1 and P == SMALL_MAX:
        tags.add("one_frame_16384")
    if N == SMALL_MAX and np.all(counts == 1):
        tags.add("16384_one_point_frames")
    return tags


def single_block_per_warp(P, stage):
    """partition() on one block: whole stages, at least one per warp."""
    return max(stage, -(-(-(-P // LY.WARPS)) // stage) * stage)


def classify_single_block(offsets, stage):
    """The boundary kinds the single-block sweep kernel meets (tests/layouts.py's classify with grid 1), plus P itself."""
    off = np.asarray(offsets, dtype=np.int64)
    P = int(off[-1])
    if P > SINGLE_BLOCK_MAX:
        return {"multi_block", f"P={P}"}
    pw = single_block_per_warp(P, stage)
    tags = LY.classify(off, 1, pw, stage) | {f"P={P}", f"stages_per_warp={pw // stage}"}
    if P in (stage - 1, stage + 1):
        tags.add(f"P=stage{P - stage:+d}")
    return tags


def classify(lay, stage):
    """Every tag of a layout under both kernels, prefixed k2: (with edges when the layout has them) and k1:."""
    k2 = classify_small(lay.offsets, lay.edge_points is not None)
    return {f"k2:{t}" for t in k2} | {f"k1:{t}" for t in classify_single_block(lay.offsets, stage)}


def _counts(rng, total, lo=1, hi=180):
    return LY._fill(rng, total, lo, hi)


def _even(P, N):
    """N frame sizes as equal as possible, adding up to P."""
    return [P // N + (1 if k < P % N else 0) for k in range(N)]


def _one_point_mix(rng, P):
    out, s = [], 0
    while s < P:
        k = 1 if len(out) % 2 == 0 else int(rng.integers(1, 61))
        k = min(k, P - s)
        out.append(k)
        s += k
    return out


def _spec(name, stage, rng):
    """(counts, edges, z_sigma, targets) of layout `name` for the sweep kernel family with this stage size."""
    if name.startswith("total_"):
        R = int(name.split("_")[1])
        counts = [R] if R <= 2 else _counts(rng, R)
        t = {f"k2:total={R}"}
        if R <= (SMALL_CLUSTER - 1) * SMALL_THREADS:
            t.add("k2:idle_cta")
        t.add("k2:idle_slot" if R <= 7 * SLOT else "k2:all_slots")
        return counts, False, 0.0, t
    if name.startswith("seam_"):
        P = int(name.split("_")[1])
        kind = {32: "warp", 256: "cta", 2047: "slot-1", 2048: "slot", 2049: "slot+1", 4096: "slot"}[P]
        return _counts(rng, P), True, 0.0, {f"k2:seam@{kind}"}
    if name == "empty_edges_at_seam":
        counts = [0, 0, 0] + _counts(rng, 2 * SLOT) + [0, 0]
        return counts, True, 0.0, {"k2:seam@slot", "k2:empty_edges@seam", "k2:empty_edges@end", "k2:leading_empty",
                                   "k2:trailing_empty", "k2:dead_edge_slots", "k1:leading_empty", "k1:trailing_empty"}
    if name == "edges_total_16384":
        return _even(SMALL_MAX - 128, 64), True, 0.0, {"k2:total=16384", "k2:total@slot", "k2:all_slots"}
    if name == "edges_total_16383":
        return _even(SMALL_MAX - 129, 64), True, 0.0, {"k2:total=16383", "k2:total@slot-1", "k2:all_slots"}
    if name == "one_point_frames_edges":
        return _one_point_mix(rng, 3000), True, 0.0, {"k2:one_point_frame_edges"}
    if name == "one_frame_16384":
        return [SMALL_MAX], False, 0.0, {"k2:one_frame_16384", "k2:total@slot", "k1:multi_block"}
    if name == "one_frame_16384_edges":
        return [SMALL_MAX], True, 0.0, {"k2:points<=small<residuals", "k1:multi_block"}
    if name == "one_point_frames_16384":
        return [1] * SMALL_MAX, False, 0.0, {"k2:16384_one_point_frames", "k2:total=16384"}
    if name == "edges_beyond_small_single_block":
        # points <= 12 288 < 16 384 < points + edges: eval and solve take the single-block sweep kernel, information K2
        return _counts(rng, 12000, 1, 9), True, 0.0, {"k2:points<=small<residuals", "k1:P=12000"}
    if name == "offplane_4097_edges":
        return _counts(rng, 2 * SLOT + 1), True, 0.3, {"k2:seam@slot+1"}
    if name == "offplane_16384":
        return _counts(rng, SMALL_MAX), False, 0.3, {"k2:total=16384"}
    if name.startswith("sb_"):
        what = name[3:]
        P = {"P1": 1, "stage-1": stage - 1, "stage+1": stage + 1, "12stage-1": 12 * stage - 1, "12stage+1": 12 * stage + 1,
             "12287": 12287, "12288": 12288, "12289": 12289}[what]
        t = {f"k1:P={P}"}
        if what.startswith("stage"):
            t.add(f"k1:P=stage{what[5:]}")
        if what.startswith("12stage"):
            t.add(f"k1:P=k*warps*stage{what[7:]}")
        if P == 12289:
            t.add("k1:multi_block")
        return _counts(rng, P), False, 0.0, t
    raise KeyError(name)


# tests/layouts.py's layouts cut for one block with warp ranges of k * 128 points (L6_short_tail and L6_jump_above change
# the single-block partition they were cut for, L4_giant_frame and L7 need several blocks)
SB_RECUTS = [("L1_aligned", 8), ("L2_off_by_one", 8), ("L3_empty_runs", 8), ("L4_one_frame", 8), ("L4_two_frames", 8),
             ("L5_confetti", 8), ("L6_jump_below", 8), ("L1_aligned", 2), ("L2_off_by_one", 2)]

LAYOUTS = ([f"total_{R}" for R in sorted(K2_TOTALS)]
           + [f"seam_{P}" for P in (32, 256, 2047, 2048, 2049)]
           + ["empty_edges_at_seam", "edges_total_16384", "edges_total_16383", "one_point_frames_edges", "one_frame_16384",
              "one_frame_16384_edges", "one_point_frames_16384", "edges_beyond_small_single_block", "offplane_4097_edges",
              "offplane_16384", "far_range", "far_range_edges"]
           + [f"sb_{w}" for w in ("P1", "stage-1", "stage+1", "12stage-1", "12stage+1", "12287", "12288", "12289")]
           + [f"recut_{n}_x{k}" for n, k in SB_RECUTS])


def build(name, bases, stage, seed=0):
    """Layout `name` (see LAYOUTS) for the kernel family with this stage size (128 general, 256 planar); `bases` is what
    base_problems returns."""
    rng = np.random.default_rng(seed + sum(map(ord, name)))
    base = bases["near"]
    if name.startswith("far_range"):
        far = bases["far"]
        counts = np.diff(far.offsets)
        edges = name.endswith("_edges")
        t = {f"k1:P={far.n_points}"} | ({f"k2:total={far.n_points + 2 * far.n_frames}"} if edges else set())
        return LY.recut(far, counts, name, t, with_edges=edges)
    if name.startswith("recut_"):
        lname, k = name[6:].rsplit("_x", 1)
        k = int(k)
        # planar stages are twice as long: the same point count per warp range is half as many stages
        per_warp = k * LY.STAGE_GENERAL
        lay = LY.build(lname, base, 1, per_warp, stage, seed=seed)
        lay.name = name
        lay.targets = {f"k1:{t}" for t in lay.targets}
        return lay
    counts, edges, z, targets = _spec(name, stage, rng)
    lay = LY.recut(base, counts, name, targets, with_edges=edges, z_sigma=z, seed=seed)
    return lay


FAR_SCALE = 6.0  # the far-range scene: boards 6-30 m away, within the 30 m range cap of the scan conversion


def base_problems(oracle, seed=23):
    """The boards and points the small layouts re-cut: "near", 60 boards x 400 beams, sigma = 1 cm, with edge points; and
    "far", the reference's 50 boards x 180 beams at 1 mm noise with every distance scaled by FAR_SCALE (near the optimum g
    cancels by orders of magnitude there)."""
    k = FAR_SCALE
    f = oracle.generate(50, 180, seed=17, sigma=0.001 / k, exact_m=True, with_edges=True)
    fp = f.frame_pose.copy()
    fp[:, 4:] *= k
    far = oracle.Problem(fp, f.offsets, f.points * k, f.edge_points * k)
    return dict(near=oracle.generate(60, 400, seed=seed, sigma=0.01, exact_m=True, with_edges=True), far=far)


def far_range_poses(oracle):
    """The far-range scene's ground truth and a pose 1e-5 away from it."""
    gt = oracle.ground_truth()[1].copy()
    gt[:3] *= FAR_SCALE
    return gt, oracle.pose_plus(gt, 1e-5 * np.array([1.0, -0.7, 0.4, -1.0, 0.6, 0.3]))
