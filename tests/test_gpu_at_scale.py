"""Every sweep-based operation against the extended-precision reference at the sizes the benchmarks run (10^7 - 2*10^8 points,
and past 2^31 points).

Scenes (tests/scale_scenes.py): S1 = configs[1] (10^4 x 10^3), S2 = configs[2] (10^5 x 2*10^3), S3 = 100 frames of 2*10^6 points
(every frame spans ~16 warp ranges, so every lane adds ~3 900 points of one frame before its moments leave it, and every warp
range uses the split-frame head / tail slots), S2e = S2 with the board-edge residuals.  Each is Problem.synthetic(sigma = 0.01),
downloaded once; the general kernel family runs on the same data created under CLC_PLANAR=0.  The long-double references are
computed once per (scene, pose, loss, edges) on the host's cores.

* eval (no loss, Cauchy, Huber, soft-L1 at the closed-form pose; Cauchy at the identity), information, the closed form and
  every field of every frame of the frame report within GAMMA * A_k; rows sum to eval;
* solves from the identity bit-identical with the L2-resident share off and on, and launch-per-iteration vs the persistent
  grid; eval at the final pose within GAMMA * A_k; noise-free S2 reaches the truth;
* subsets (bench's drop-every-10th mask and a contiguous run) and trims (bench_trim's edited S2, tau = 0.2 and +inf) bytes-equal
  to fresh problems of the kept data;
* segments (10^4 rigs x 50 x 180, and 100 windows of configs[1]) within GAMMA * A_k of their slices; every window, and 1 000
  random rigs plus the rig with the most iterations, solving as a fresh problem of its slice;
* a 2.2*10^9-point problem: frame-report rows around point indices 2^29, 2^30, 2^31 and of the last frame against the same
  frames generated as a small problem, rows summing to eval, and a noise-free solve reaching the truth.
"""
import time

import numpy as np
import pytest

import exact_sums as X
import frame_exact as F
import scale_scenes as SS

from conftest import pack_sums
from test_gpu_segments import Data, plane_slack
from test_gpu_subset import FAMILIES, SUMMARY_FIELDS, assert_same_data, assert_same_outputs, env, np_subset, outcomes
from test_gpu_trim import Scene, check_trim

pytestmark = pytest.mark.gpu

IDENT = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
LOSSES = ("none", "cauchy", "huber", "soft_l1")
WORST = {}   # scene -> largest |err| / A_k over every checked output
HITS = {}    # scene / family -> what the partition made it hit
TIMES = {}   # phase -> seconds
T_START = []


def record(scene, r):
    WORST[scene] = max(WORST.get(scene, 0.0), float(np.max(r)) if np.size(r) else 0.0)


def check_lm(scene, got, ref, what, slack=None):
    val, mag = ref
    r = X.assert_within(got, val, mag if slack is None else mag + slack, X.GROUPS_LM, f"{scene}: {what}")
    record(scene, r)


def pose_of_closed_form(p):
    from camlasercalibratool_b200 import T_to_pose7

    return T_to_pose7(np.linalg.inv(p.closed_form()[0]))


def synthetic(name, **kw):
    from camlasercalibratool_b200 import Problem

    n, beams, edges = SS.SCENES[name]
    return Problem.synthetic(n, beams, seed=SS.SEED, sigma=kw.pop("sigma", SS.SIGMA), with_edges=edges, **kw)


class SceneData:
    """Host arrays of a scene, its closed-form pose and its references (computed on first use)."""

    def __init__(self, name):
        self.name = name
        with synthetic(name) as p:
            d = p.download()
            self.cf_pose = pose_of_closed_form(p)
        self.arrays = (d["frame_pose"], d["offsets"], d["points"], d["edge_points"])
        self.edges = SS.SCENES[name][2]
        self._ref = {}

    def ref(self, what, pose=None, kind="cauchy"):
        key = (what, None if pose is None else tuple(np.asarray(pose).tolist()), kind)
        if key not in self._ref:
            t0 = time.perf_counter()
            if what == "frames":
                self._ref[key] = SS.spread(self.arrays, "frames", (pose, kind == "cauchy", self.edges))
            elif what == "lm":
                self._ref[key] = SS.spread(self.arrays, "lm", (pose, kind, self.edges))
            else:
                self._ref[key] = SS.spread(self.arrays, "cf")
            TIMES[f"{self.name} reference {what}/{kind}"] = time.perf_counter() - t0
        return self._ref[key]

    def lm(self, pose, kind):
        """The 28 sums under `kind`: the Cauchy ones come from the per-frame reference (the same terms, summed per frame)."""
        if kind == "cauchy" and np.array_equal(pose, self.cf_pose):
            return SS.totals(*self.ref("frames", pose))
        return self.ref("lm", pose, kind)


@pytest.fixture(scope="module", autouse=True)
def wall_clock():
    T_START.append(time.perf_counter())
    yield


@pytest.fixture(scope="module")
def scene(request):
    return SceneData(request.param)


def test_00_host():
    print(f"\nhost reference workers: {SS.workers()}")


# ---- 1. what each scene hits -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", list(SS.SCENES), indirect=True)
def test_scene_hits(scene):
    off = scene.arrays[1]
    P = int(off[-1])
    for family, knobs in FAMILIES.items():
        with env(**knobs), synthetic(scene.name) as p:
            part = p.partition(warp_table=False)
            assert p.planar == (family == "planar")
            n_warps = part["grid"] * 12
            depth = SS.lane_depth(off, part["per_warp"])
            frames_per_range, crosses = SS.split_ranges(off, part["per_warp"])
            hits = dict(points=P, grid=part["grid"], per_warp=part["per_warp"], stage=part["stage"],
                        stages_per_warp=part["per_warp"] // part["stage"], resident_chunks=part["resident_chunks"],
                        max_lane_depth=depth, ranges_with_split_frames=int(crosses.sum()), ranges=len(crosses))
            HITS[f"{scene.name}/{family}"] = hits
            print(f"\n{scene.name}/{family}: {hits}")
            assert part["grid"] * 12 == n_warps and part["per_warp"] // part["stage"] > 1  # several stages per warp range
            assert part["resident_chunks"] > 0
            if scene.name == "S3":
                assert depth >= 3500, depth
                assert frames_per_range.max() <= 2 and np.all(crosses), (frames_per_range.max(), int(crosses.sum()))


# ---- 2. sums against long double ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", list(SS.SCENES), indirect=True)
def test_sums_against_long_double(scene):
    name, x = scene.name, scene.cf_pose
    full = name in ("S1", "S2")
    evals = [(k, x) for k in (LOSSES if full else ("cauchy",))] + ([("cauchy", IDENT)] if full else [])
    fails = []

    def attempt(fn):  # every check runs; the failures are listed together
        try:
            fn()
        except AssertionError as exc:
            print(f"\nFAILED CHECK {exc}"[:3000])
            fails.append(str(exc)[:300])

    for family, knobs in FAMILIES.items():
        with env(**knobs), synthetic(name) as p:
            assert p.planar == (family == "planar")
            for kind, pose in evals:
                p.set_loss(kind, SS.A)
                got = pack_sums(*p.eval(pose))
                at = "the identity" if pose is IDENT else "the closed-form pose"
                attempt(lambda: check_lm(name, got, scene.lm(pose, kind), f"{family} eval {kind} at {at}"))
            p.set_loss("cauchy", SS.A)
            if not scene.edges:  # information and the closed form have no edge residuals
                H, b, chi, _ = p.information(x)
                attempt(lambda: check_lm(name, pack_sums(chi / 2, H, -b), scene.lm(x, "none"), f"{family} information"))
                _, _, AtA, Atb = p.closed_form()
                attempt(lambda: record(name, X.assert_within(X.pack_closed_form(AtA, Atb), *scene.ref("cf"), X.GROUPS_CF,
                                                             f"{name}: {family} closed form")))
            rows = p.frame_report(x)
            val, mag = scene.ref("frames", x)

            def frames():
                slack = SS.frame_plane_slack(scene.arrays[0], scene.arrays[1])
                worst = F.assert_within(F.comparable(rows), val, mag + slack, what=f"{name}: {family} frame report")
                WORST[name] = max(WORST.get(name, 0.0), max(worst.values()))
            attempt(frames)
            assert np.array_equal(rows["n_points"], np.diff(scene.arrays[1]))
            tot = np.concatenate([rows["H21"].sum(axis=0), rows["g6"].sum(axis=0), [rows["cost"].sum()]])
            attempt(lambda: check_lm(name, tot, SS.totals(val, mag), f"{family} frame report rows summed"))
    assert not fails, fails


# ---- 3. solves at scale ------------------------------------------------------------------------------------------------------
def _solve(name, **knobs):
    with env(**knobs), synthetic(name) as p:
        x, s, tr = p.solve(IDENT)
        return p.partition(warp_table=False)["resident_chunks"], x, [getattr(s, k) for k in SUMMARY_FIELDS], \
            b"".join(bytes(t) for t in tr)


@pytest.mark.parametrize("scene", ["S2", "S3"], indirect=True)
def test_solves_at_scale(scene, oracle):
    name = scene.name
    finals = {}
    for family, knobs in FAMILIES.items():
        res, x, summ, trace = _solve(name, **knobs)
        assert res > 0
        res0, x0, summ0, trace0 = _solve(name, CLC_L2_RESIDENT_MB="0", **knobs)
        assert res0 == 0
        _, x2, summ2, trace2 = _solve(name, CLC_LOOP_IN_KERNEL="2", **knobs)
        for what, (xb, sb, tb) in (("L2 residency off", (x0, summ0, trace0)), ("persistent grid", (x2, summ2, trace2))):
            assert xb.tobytes() == x.tobytes() and sb == summ and tb == trace, f"{name}/{family}: {what} differs"
        assert summ[0] in (1, 2, 3), summ
        finals[family] = x
        print(f"\n{name}/{family}: {summ[1]} iterations, termination {summ[0]}, pose error vs truth "
              f"{oracle.pose_error(x, oracle.ground_truth()[1])}")
    xf = finals["planar"]
    ref = scene.ref("lm", xf, "cauchy")
    for family, knobs in FAMILIES.items():
        with env(**knobs), synthetic(name) as p:
            check_lm(name, pack_sums(*p.eval(xf)), ref, f"{family} eval at the final pose")


def test_noise_free_S2_reaches_the_truth(oracle):
    with synthetic("S2", sigma=0.0) as p:
        x, s, _ = p.solve(IDENT)
    ang, dt = oracle.pose_error(x, oracle.ground_truth()[1])
    assert ang < 1e-7 and dt < 1e-7 and s.termination in (1, 2, 3), (ang, dt, s.termination)


# ---- 4. subsets at bench size ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["S1", "S2"])
def test_subsets_at_bench_size(name):
    from camlasercalibratool_b200 import Problem

    n_frames, beams, _ = SS.SCENES[name]
    f = np.arange(n_frames)
    b, e = 3 * n_frames // 10 + 7, 7 * n_frames // 10 - 3
    masks = {"drop_every_10th": f % 10 != 9, "contiguous": (f >= b) & (f < e)}
    for family, knobs in FAMILIES.items():
        with env(**knobs):
            with synthetic(name) as src:
                d = src.download()
                x = pose_of_closed_form(src)
                if family == "planar":  # the generator's frame ranges are slices of the whole problem
                    with synthetic(name, frame_begin=b, frame_end=e) as gen:
                        g = gen.download()
                    o = d["offsets"]
                    assert g["offsets"].tobytes() == (o[b:e + 1] - o[b]).tobytes()
                    assert g["points"].tobytes() == d["points"][o[b]:o[e]].tobytes()
                    for k in ("frame_pose", "planes"):
                        assert g[k].tobytes() == d[k][b:e].tobytes(), k
                for mask, keep in masks.items():
                    what = f"{name}/{family}/{mask}"
                    with src.subset(keep) as sub:
                        with Problem.from_arrays(*np_subset(d["frame_pose"], d["offsets"], d["points"], None, keep)) as fresh:
                            assert_same_data(sub, fresh, what)
                            got = outcomes(sub, IDENT, x)
                            assert_same_outputs(got, outcomes(fresh, IDENT, x), what)
                        if mask == "contiguous":
                            with synthetic(name, frame_begin=b, frame_end=e) as gen:
                                assert_same_data(sub, gen, what + " vs the generator")
                                assert_same_outputs(got, outcomes(gen, IDENT, x), what + " vs the generator")
            del d


# ---- 5. trims at bench size --------------------------------------------------------------------------------------------------
def edited_source(oracle, name):
    """bench_trim.py's source: the scene with a seeded 1 % of its points moved 0.3 - 1 m off their board inside the laser plane
    (z stays 0), and the pose its clean version solves to.  Returns the scene, that pose and the mask of the unmoved points."""
    with synthetic(name) as syn:
        x, _, _ = syn.solve(IDENT)
        d = syn.download()
    rng = np.random.default_rng(2024)
    P = len(d["points"])
    idx = rng.choice(P, P // 100, replace=False)
    R = oracle.quat_to_rot(x[3:])
    m = d["planes"][:, :3] @ R
    fi = np.searchsorted(d["offsets"], idx, side="right") - 1
    mxy = m[fi, :2]
    shift = rng.uniform(0.3, 1.0, size=len(idx)) * rng.choice([-1.0, 1.0], size=len(idx))
    d["points"][idx, :2] += (shift / np.einsum("ij,ij->i", mxy, mxy))[:, None] * mxy
    moved = np.zeros(P, dtype=bool)
    moved[idx] = True
    return Scene(d["frame_pose"], d["offsets"], d["points"]), x, ~moved, d["planes"]


def test_trims_at_bench_size(oracle):
    scene, x, unmoved, planes = edited_source(oracle, "S2")
    tau = 0.2
    # on the host in float64: the unmoved points lie well inside tau, the moved ones well outside, so the device's rounding of
    # e (a few ulp of |m||p|) cannot move a point across
    R = oracle.quat_to_rot(x[3:])
    counts = np.diff(scene.off)
    e = np.empty(len(scene.pts))
    for a in range(0, len(counts), 10_000):  # frame blocks: bounded temporaries
        b = min(len(counts), a + 10_000)
        pa, pb = scene.off[a], scene.off[b]
        m = np.repeat(planes[a:b, :3] @ R, counts[a:b], axis=0)
        c = np.repeat(planes[a:b, :3] @ x[:3] + planes[a:b, 3], counts[a:b])
        e[pa:pb] = np.abs(np.einsum("ij,ij->i", scene.pts[pa:pb], m) + c)
    print(f"\ntrim: unmoved max |e| {e[unmoved].max():.4f} m, moved min |e| {e[~unmoved].min():.4f} m, tau {tau} m")
    assert e[unmoved].max() <= tau / 2 and e[~unmoved].min() >= 1.2 * tau
    del e
    for family, knobs in FAMILIES.items():
        with env(**knobs):
            for t, keep in ((tau, unmoved), (np.inf, np.ones(len(unmoved), dtype=bool))):
                check_trim(scene, keep, IDENT, x, t, what=f"S2/{family}/tau={t}")


# ---- 6. segments at bench size -----------------------------------------------------------------------------------------------
def _segment_poses(oracle, W, seed):
    rng = np.random.default_rng(seed)
    gt = oracle.ground_truth()[1]
    return np.stack([oracle.pose_plus(gt, 1e-2 * rng.standard_normal(6)) for _ in range(W)])


def _check_segments(oracle, label, n_frames, beams, per, knobs, fresh_max=10 ** 9):
    from camlasercalibratool_b200 import Problem

    off = np.arange(0, n_frames + 1, per, dtype=np.int64)
    W = len(off) - 1
    poses = _segment_poses(oracle, W, seed=W)
    with env(**knobs), Problem.synthetic(n_frames, beams, seed=SS.SEED, sigma=SS.SIGMA) as p:
        d = p.download()
        cost, H, g = p.eval_segments(off, poses)
        Hi, b, chi, _ = p.information_segments(off, poses)
        xs, summ, _ = p.solve_segments(off, np.tile(IDENT, (W, 1)))
    arrays = (d["frame_pose"], d["offsets"], d["points"], None)
    t0 = time.perf_counter()
    ref_c = SS.segment_sums(arrays, off, poses, "cauchy")
    ref_n = SS.segment_sums(arrays, off, poses, "none")
    TIMES[f"{label} reference"] = time.perf_counter() - t0
    o = d["offsets"]
    for s in range(W):
        slack = plane_slack(Data(d["frame_pose"][off[s]:off[s + 1]], o[off[s]:off[s + 1] + 1] - o[off[s]], None, None))
        check_lm(label, pack_sums(cost[s], H[s], g[s]), ref_c[s], f"eval segment {s}", slack)
        check_lm(label, pack_sums(chi[s] / 2, Hi[s], -b[s]), ref_n[s], f"information segment {s}", slack)
    del d, arrays
    t0 = time.perf_counter()
    worst = 0.0
    rng = np.random.default_rng(W)
    its = np.array([sm.num_iterations for sm in summ])
    sample = np.arange(W) if W <= fresh_max else np.unique(np.r_[rng.choice(W, fresh_max, replace=False), np.argmax(its)])
    with env(**knobs):
        for s in sample:
            with Problem.synthetic(n_frames, beams, seed=SS.SEED, sigma=SS.SIGMA, frame_begin=int(off[s]),
                                   frame_end=int(off[s + 1])) as f:
                xf, sf, _ = f.solve(IDENT)
            a, c = summ[s], sf
            assert (a.termination, a.num_iterations, a.num_successful_steps, a.num_unsuccessful_steps) == \
                (c.termination, c.num_iterations, c.num_successful_steps, c.num_unsuccessful_steps), f"{label}: segment {s}"
            dx = float(np.abs(xs[s] - xf).max())
            worst = max(worst, dx)
            assert dx <= 1e-12, (label, s, dx)
    TIMES[f"{label} fresh solves"] = time.perf_counter() - t0
    print(f"\n{label}: {W} segments, {len(sample)} fresh solves, largest pose difference to them {worst:.2e}")


def test_segments_fleet(oracle):
    """Every rig's sums; the solves of 1 000 random rigs and of the rig with the most iterations against fresh solves."""
    _check_segments(oracle, "fleet 10^4 rigs", 10_000 * 50, 180, 50, {}, fresh_max=1000)


@pytest.mark.parametrize("family", list(FAMILIES))
def test_segments_windows(oracle, family):
    _check_segments(oracle, f"windows/{family}", 10_000, 1_000, 100, FAMILIES[family])


# ---- 7. past 2^29 and 2^31 points --------------------------------------------------------------------------------------------
BIG_FRAMES, BIG_BEAMS, BIG_SEED = 1_100_000, 2_000, 3
BIG_GB = 45


def test_past_2_31_points(oracle):
    import torch

    free, _ = torch.cuda.mem_get_info()
    if free < BIG_GB * 2 ** 30:
        pytest.skip(f"needs {BIG_GB} GB of free device memory for 2.2e9 points (36 GB), {free / 2 ** 30:.1f} GB free")
    from camlasercalibratool_b200 import Problem

    P = BIG_FRAMES * BIG_BEAMS
    assert P > 2 ** 31
    gt = oracle.ground_truth()[1]
    xe = oracle.pose_plus(gt, np.array([0.01, -0.02, 0.015, 0.004, -0.003, 0.002]))
    frames = sorted({f for i in (2 ** 29, 2 ** 30, 2 ** 31) for f in (i // BIG_BEAMS - 1, i // BIG_BEAMS, i // BIG_BEAMS + 1)} |
                    {BIG_FRAMES - 1})
    with Problem.synthetic(BIG_FRAMES, BIG_BEAMS, seed=BIG_SEED, sigma=SS.SIGMA) as p:
        assert p.sizes()[1] == P and p.planar
        rows = p.frame_report(xe)
        whole = pack_sums(*p.eval(xe))
    assert np.all(rows["n_points"] == BIG_BEAMS)
    worst = 0.0
    for f in frames:
        with Problem.synthetic(BIG_FRAMES, BIG_BEAMS, seed=BIG_SEED, sigma=SS.SIGMA, frame_begin=f, frame_end=f + 1) as q:
            d = q.download()
        val, mag = F.frame_sums(d["frame_pose"], d["offsets"], d["points"], xe, True, SS.A)
        mag = mag + SS.frame_plane_slack(d["frame_pose"], d["offsets"])
        w = F.assert_within(F.comparable(rows[f:f + 1]), val, mag, what=f"frame {f} (points {f * BIG_BEAMS}...)")
        worst = max(worst, max(w.values()))
    WORST["2.2e9"] = worst
    # rows sum to eval.  A_k of the whole problem is at least the sum over frames of |row_k|: 1e-11 of that is a bound at most
    # 100 GAMMA * A_k
    tot = np.concatenate([rows["H21"].sum(axis=0), rows["g6"].sum(axis=0), [rows["cost"].sum()]])
    absum = np.concatenate([np.abs(rows["H21"]).sum(axis=0), np.abs(rows["g6"]).sum(axis=0), [np.abs(rows["cost"]).sum()]])
    assert np.all(np.abs(tot - whole) <= 100 * X.GAMMA * absum), np.abs(tot - whole) / absum
    del rows
    with Problem.synthetic(BIG_FRAMES, BIG_BEAMS, seed=BIG_SEED, sigma=0.0) as p:
        x, s, _ = p.solve(IDENT)
    ang, dt = oracle.pose_error(x, gt)
    print(f"\n2.2e9 points: frames {frames} worst |err|/A {worst:.2e}; noise-free solve: {s.num_iterations} iterations, "
          f"error {ang:.2e} rad {dt:.2e} m")
    assert ang < 1e-7 and dt < 1e-7 and s.termination in (1, 2, 3), (ang, dt, s.termination)


def test_zz_report():
    print(f"\nworst |err|/A_k per scene (GAMMA = {X.GAMMA:.0e}): {({k: f'{v:.2e}' for k, v in WORST.items()})}")
    for k, v in HITS.items():
        print(f"  {k}: {v}")
    for k, v in TIMES.items():
        print(f"  {k}: {v:.1f} s")
    if T_START:
        print(f"wall time of the module: {time.perf_counter() - T_START[0]:.0f} s")
    assert all(v <= X.GAMMA for v in WORST.values())
