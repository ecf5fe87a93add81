"""Exact quantiles of the point-to-board distances on the GPU (clc_point_residuals, clc_residual_quantiles, clc_frame_quantiles and
their group forms).

The reference of every quantile is the residual dump itself: a quantile is one element of the multiset of |e|, so every comparison
is on the bytes, against np.sort of the dump.  The dump is held to the trim's decisions, the frame report's max_abs_e and a float64
host recomputation.  Scenes with a board at the laser origin (identity board pose, identity extrinsic) have e == z exactly, so any
multiset of e -- ties, signed zeros, NaN, inf -- can be written down directly.
"""
import numpy as np
import pytest

import layouts as LY
from test_gpu_subset import FAMILIES, Scene, env, near_optimum
from test_gpu_trim import inject, laser_normals
from test_quantiles_cpu import Q_EDGE, expected, same_bits

pytestmark = pytest.mark.gpu

IDENT = np.array([0, 0, 0, 0, 0, 0, 1.0])
S = 4096  # clc::kFrameSortMax
QS = [np.array(Q_EDGE), np.linspace(0.0, 1.0, 16), np.array([0.5, 0.5, 0.9, 0.0])]


def z_problem(counts, z):
    """Frames at the identity board pose whose point j has e == z[j] at IDENT (x, y spread so that the points differ)."""
    from camlasercalibratool_b200 import Problem

    counts = np.asarray(counts, dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    P = int(off[-1])
    rng = np.random.default_rng(P)
    pts = np.column_stack([rng.uniform(-1, 1, P), rng.uniform(-1, 1, P), np.asarray(z, dtype=np.float64)])
    fp = np.tile([0, 0, 0, 1.0, 0, 0, 0], (len(counts), 1))
    return Problem.from_arrays(fp, off, pts)


def check(p, x, qs=QS, frames=True):
    """Problem-wide and per-frame quantiles of p at x against np.sort of its own dump, bitwise; returns the dump."""
    n_frames, n_points, _ = p.sizes()
    e = p.point_residuals(x)
    assert e.shape == (n_points,)
    off = p.download()["offsets"] if frames else None
    for q in qs:
        v, nv = p.residual_quantiles(x, q)
        want, n = expected(e, q)
        assert nv == n and same_bits(v, want), (q, v, want)
        v2, _ = p.residual_quantiles(x, q)
        assert v.tobytes() == v2.tobytes()  # determinism
        if frames:
            fv, fnv = p.frame_quantiles(x, q)
            assert fv.shape == (n_frames, len(np.atleast_1d(q)))
            for f in range(n_frames):
                want, n = expected(e[off[f]:off[f + 1]], q)
                assert fnv[f] == n and same_bits(fv[f], want), (f, q, fv[f], want)
            fv2, fnv2 = p.frame_quantiles(x, q)
            assert fv.tobytes() == fv2.tobytes() and fnv.tobytes() == fnv2.tobytes()
    return e


@pytest.fixture(scope="module")
def base(oracle):
    return LY.base_problem(oracle)


@pytest.fixture(scope="module")
def grid_full():
    from camlasercalibratool_b200 import Problem

    with Problem.synthetic(600, 1000) as probe:
        return probe.partition(warp_table=False)["grid"]


def test_dump_matches_trim_report_and_host(oracle, base, grid_full):
    lay = LY.build("L3_empty_runs", base, grid_full, 256, LY.STAGE_GENERAL)
    x = near_optimum(oracle)
    scene, _ = inject(oracle, lay, x, np.random.default_rng(3))
    rng = np.random.default_rng(4)
    with scene.problem() as p:
        e = p.point_residuals(x)
        # paging gives the same bytes
        cut = len(e) // 3
        assert np.concatenate([p.point_residuals(x, 0, cut), p.point_residuals(x, cut)]).tobytes() == e.tobytes()
        counts = np.diff(scene.off)
        frame_of = np.repeat(np.arange(scene.n_frames), counts)
        # the trim keeps exactly |e| <= t_f
        t = rng.choice([0.0, 0.005, 0.02, 0.05, 0.5, np.inf], size=scene.n_frames) * rng.uniform(0.5, 1.5, scene.n_frames)
        t = np.where(np.isnan(t), np.inf, t)
        with p.trim(x, t) as tr:
            kept = np.diff(tr.download()["offsets"])
        assert np.array_equal(kept, np.bincount(frame_of, weights=np.abs(e) <= t[frame_of], minlength=scene.n_frames).astype(int))
        # per-frame max |e| is the report's max_abs_e
        rows = p.frame_report(x)
        for f in np.nonzero(counts > 0)[0]:
            seg = np.abs(e[scene.off[f]:scene.off[f + 1]])
            assert seg.max().tobytes() == rows["max_abs_e"][f].tobytes(), f
    m, c = laser_normals(oracle, scene.fp, x)
    host = np.einsum("ij,ij->i", scene.pts, m[frame_of]) + c[frame_of]
    scale = np.abs(scene.pts) @ np.ones(3) * np.abs(m[frame_of]).max(axis=1) + np.abs(c[frame_of])
    assert np.all(np.abs(e - host) <= 1e-12 * np.maximum(scale, 1e-300))


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", ["L1_aligned", "L2_off_by_one", "L3_empty_runs", "L4_giant_frame", "L5_confetti"])
def test_layouts(oracle, base, grid_full, name, family):
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    lay = LY.build(name, base, grid_full, 256, stage)
    x = near_optimum(oracle)
    with env(**FAMILIES[family]), Scene(lay.frame_pose, lay.offsets, lay.points).problem() as p:
        assert p.planar == (family == "planar")
        check(p, x, frames=name != "L4_giant_frame")
        if name == "L4_giant_frame":  # one frame of most of the points: the one-block radix select
            check(p, x, qs=QS[:1])


def test_special_values():
    rng = np.random.default_rng(8)
    z = rng.normal(0, 0.01, 50_000)
    z[rng.integers(0, z.size, 300)] = np.nan
    z[rng.integers(0, z.size, 30)] = np.inf
    z[rng.integers(0, z.size, 30)] = -np.inf
    z[rng.integers(0, z.size, 500)] = 0.0
    z[rng.integers(0, z.size, 500)] = -0.0
    with z_problem([100, 20_000, 0, 29_900], z) as p:
        e = check(p, IDENT)
        assert np.isnan(e).sum() > 0 and np.isinf(e).sum() > 0 and (e == 0).sum() > 0
    # every e is 0: massive ties, no compaction
    with z_problem([5000] * 40, np.zeros(200_000)) as p:
        v, nv = p.residual_quantiles(IDENT, np.linspace(0, 1, 16))
        assert nv == 200_000 and np.all(v.view(np.uint64) == 0)
        check(p, IDENT, qs=QS[:1])
    # every e is NaN
    with z_problem([10, 5000], np.full(5010, np.nan)) as p:
        v, nv = p.residual_quantiles(IDENT, [0.0, 1.0])
        assert nv == 0 and np.all(np.isnan(v))
        fv, fnv = p.frame_quantiles(IDENT, 0.5)
        assert np.all(fnv == 0) and np.all(np.isnan(fv))


def test_empty_and_single_point():
    with z_problem([0, 0, 0], np.zeros(0)) as p:
        v, nv = p.residual_quantiles(IDENT, [0.0, 0.5])
        assert nv == 0 and np.all(np.isnan(v))
        fv, fnv = p.frame_quantiles(IDENT, 0.5)
        assert fv.shape == (3, 1) and np.all(np.isnan(fv)) and np.all(fnv == 0)
        assert p.point_residuals(IDENT).shape == (0,)
    with z_problem([1], [-0.25]) as p:
        v, nv = p.residual_quantiles(IDENT, Q_EDGE)
        assert nv == 1 and np.all(v == 0.25)
        check(p, IDENT)


def test_frame_sizes():
    """Frames of 0, 1, S - 1, S, S + 1 and 1e5 points, and an all-NaN frame, with ties; q = 1 is the report's max_abs_e."""
    rng = np.random.default_rng(9)
    counts = [0, 1, S - 1, S, S + 1, 100_000, 3000, 7]
    P = sum(counts)
    z = np.round(rng.normal(0, 0.01, P), 4)  # ties
    nan_frame = slice(sum(counts[:6]), sum(counts[:7]))
    z[nan_frame] = np.nan
    with z_problem(counts, z) as p:
        check(p, IDENT)
        fv, _ = p.frame_quantiles(IDENT, 1.0)
        rows = p.frame_report(IDENT)
        for f in (1, 2, 3, 4, 5, 7):
            assert fv[f, 0].tobytes() == rows["max_abs_e"][f].tobytes(), f


def test_subsets_and_trims(oracle, base, grid_full):
    lay = LY.build("L2_off_by_one", base, grid_full, 256, LY.STAGE_GENERAL)
    x = near_optimum(oracle)
    scene, _ = inject(oracle, lay, x, np.random.default_rng(5))
    keep = np.random.default_rng(6).random(scene.n_frames) < 0.6
    with scene.problem() as p, p.subset(keep) as s, p.trim(x, 0.1) as t:
        check(s, x)
        check(t, x)


def test_group_equals_problem(oracle, base, grid_full):
    import torch

    from camlasercalibratool_b200 import Group

    lay = LY.build("L5_confetti", base, grid_full, 256, LY.STAGE_GENERAL)
    x = near_optimum(oracle)
    devs = list(range(torch.cuda.device_count()))
    with Scene(lay.frame_pose, lay.offsets, lay.points).problem() as p:
        want = [(p.residual_quantiles(x, q), p.frame_quantiles(x, q)) for q in QS]
    for devices in [[d] for d in devs] + ([devs] if len(devs) > 1 else []):
        with Group.from_arrays(lay.frame_pose, lay.offsets, lay.points, devices=devices) as g:
            for q, ((v, nv), (fv, fnv)) in zip(QS, want):
                gv, gnv = g.residual_quantiles(x, q)
                gfv, gfnv = g.frame_quantiles(x, q)
                assert gv.tobytes() == v.tobytes() and gnv == nv, devices
                assert gfv.tobytes() == fv.tobytes() and gfnv.tobytes() == fnv.tobytes(), devices


def test_median_trim_pipeline(oracle):
    """Outliers as the trim tests inject them, and a frame of wall returns: 180 points with noise up to 1 cm and 40 points 15 cm
    off the board.  A trim at 3 * 1.4826 * the per-frame median removes exactly the injected points, where 3 * rms_e keeps the
    wall returns; the re-solve is the solve of the clean points, bit for bit, and reaches the ground truth."""
    from camlasercalibratool_b200 import Problem

    rng = np.random.default_rng(12)
    gt = oracle.ground_truth()[1]
    g = oracle.generate(60, 180, seed=5, sigma=0.0)
    fp, off = np.asarray(g.frame_pose), np.asarray(g.offsets, dtype=np.int64)
    counts = np.diff(off)
    frame_of = np.repeat(np.arange(len(counts)), counts)
    m, c = laser_normals(oracle, fp, gt)
    pts = np.asarray(g.points) + rng.uniform(-0.01, 0.01, len(frame_of))[:, None] * m[frame_of]
    clean = Scene(fp, off, pts)

    class Lay:  # the layout interface inject() reads
        frame_pose, offsets, points, edge_points, n_points = fp, off, pts, None, len(pts)

    scene, keep = inject(oracle, Lay, gt, rng, per_frame=(0, 6))
    # frame 0 also gets 40 wall returns 15 cm behind its board
    w = scene.pts[scene.off[0]:scene.off[0] + 40] + 0.15 * m[0]
    pts2 = np.insert(scene.pts, scene.off[1], w, axis=0)
    keep = np.insert(keep, scene.off[1], False)
    off2 = scene.off + np.concatenate([[0], np.full(len(counts), 40)])
    scene = Scene(fp, off2, pts2)
    with scene.problem() as p:
        med = p.frame_quantiles(gt, 0.5)[0][:, 0]
        rms = p.frame_report(gt)["rms_e"]
        e0 = np.abs(p.point_residuals(gt, int(off2[0]), int(off2[1] - off2[0])))
        assert np.sum(e0 > 3 * rms[0]) < 40  # the rms threshold keeps wall returns
        with p.trim(gt, 3 * 1.4826 * med) as t, clean.problem() as ref:
            d, r = t.download(), ref.download()
            assert np.array_equal(d["offsets"], r["offsets"]) and d["points"].tobytes() == r["points"].tobytes()
            x0 = oracle.pose_plus(gt, np.array([0.02, -0.01, 0.01, 0.01, -0.02, 0.01]))
            xt, st, _ = t.solve(x0)
            xr, _, _ = ref.solve(x0)
            assert xt.tobytes() == xr.tobytes()
            ang, dt = oracle.pose_error(xt, gt)
            assert ang < 1e-3 and dt < 1e-3 and st.termination in (1, 2, 3), (ang, dt, st.termination)


BIG_FRAMES, BIG_BEAMS, BIG_SEED, BIG_GB = 1_100_000, 2_000, 3, 45


def test_past_2_31_points(oracle):
    """The scene of test_gpu_at_scale.test_past_2_31_points: every value v of rank k brackets count(|e| < v) <= k < count(|e| <= v),
    counted over paged point_residuals; the per-frame rows of sampled frames equal their slices' sorted values."""
    import torch

    free, _ = torch.cuda.mem_get_info()
    if free < BIG_GB * 2 ** 30:
        pytest.skip(f"needs {BIG_GB} GB of free device memory for 2.2e9 points (36 GB), {free / 2 ** 30:.1f} GB free")
    from camlasercalibratool_b200 import Problem

    P = BIG_FRAMES * BIG_BEAMS
    x = near_optimum(oracle)
    q = np.array([0.0, 0.5, 0.95, 1.0])
    with Problem.synthetic(BIG_FRAMES, BIG_BEAMS, seed=BIG_SEED, sigma=0.01) as p:
        assert p.sizes()[1] == P > 2 ** 31
        v, nv = p.residual_quantiles(x, q)
        fv, fnv = p.frame_quantiles(x, q)
        below, at = np.zeros(len(q), dtype=np.int64), np.zeros(len(q), dtype=np.int64)
        n = 0
        chunk = 1 << 26
        for first in range(0, P, chunk):
            a = np.abs(p.point_residuals(x, first, min(chunk, P - first)))
            n += int(np.sum(~np.isnan(a)))
            below += (a[None, :] < v[:, None]).sum(axis=1)
            at += (a[None, :] <= v[:, None]).sum(axis=1)
        assert nv == n
        k = np.array([min(max(int(np.ceil(qq * n)) - 1, 0), n - 1) for qq in q])
        assert np.all(below <= k) and np.all(k < at), (below, k, at)
        for f in (0, 2 ** 29 // BIG_BEAMS, 2 ** 31 // BIG_BEAMS, BIG_FRAMES - 1):
            want, nf = expected(p.point_residuals(x, f * BIG_BEAMS, BIG_BEAMS), q)
            assert fnv[f] == nf and same_bits(fv[f], want), f
