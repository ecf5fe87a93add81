"""GPU tests (-m gpu) of the Huber and soft-L1 losses (clc_problem_set_loss).

* eval within GAMMA * A_k of the long-double reference (tests/loss_reference.py) on the adversarial layouts of the sweep kernel's
  partition and of the one-cluster kernel, both kernel families, with and without edge residuals, with the one-cluster kernel
  on and off, each layout on the kernel clc_debug_dispatch names;
* the Huber boundary |e| == a (and one ulp either side) at the identity pose, in frames split across warp ranges;
* the frame report's rows and the segments' sums within GAMMA * A of the reference, rows summing to eval;
* solves making the decisions of the losses' C oracle (tests/loss_oracle.c) under every driver, the sweep kernel's drivers
  bit for bit, segments equal to fresh problems, noise-free data reaching the truth;
* no behaviour change, by bytes: set_loss("cauchy", a) on a use_loss = 0 problem is a use_loss = 1 problem; switching kinds and
  back restores every byte; information and the closed form ignore the loss; subset / trim and a group of one inherit it.
"""
import numpy as np
import pytest

import exact_sums as X
import layouts as LY
import loss_reference as LR
import small_layouts as SL

from conftest import pack_sums
from test_gpu_partition import FAMILIES, FAR, X0, env, near_optimum
from test_gpu_segments import Data, ragged, seams
from test_gpu_small_path import KERNELS, expected_dispatch

pytestmark = pytest.mark.gpu

A = 0.05
NEW = ("huber", "soft_l1")
WORST = {}


def check(got, ref, what):
    r = X.assert_within(got, *ref, X.GROUPS_LM, what)
    for name, v in X.worst_by_group(r, X.GROUPS_LM).items():
        WORST[name] = max(WORST.get(name, 0.0), v)


def make(d, kind, edges=False, a=A, use_loss=True):
    from camlasercalibratool_b200 import Problem

    g = Problem.from_arrays(d.frame_pose, d.offsets, d.points, d.edge_points if edges else None, use_loss=use_loss, cauchy_a=A)
    g.set_loss(kind, a)
    return g


_REF = {}  # reference sums by (problem content, pose, kind, edges, a): shared by the kernel families and the K2 on/off runs


def ref(d, pose, kind, edges, a=A):
    k = (hash(np.asarray(d.offsets).tobytes()), hash(np.asarray(d.points).tobytes()), hash(np.asarray(d.frame_pose).tobytes()),
         tuple(np.asarray(pose).tolist()), kind, edges, a)
    if k not in _REF:
        _REF[k] = LR.lm_sums(d.frame_pose, d.offsets, d.points, pose, kind, a, d.edge_points if edges else None)
    return _REF[k]


@pytest.fixture(scope="module")
def grid_full():
    from camlasercalibratool_b200 import Problem

    with Problem.synthetic(600, 1000) as probe:
        return probe.partition(warp_table=False)["grid"]


@pytest.fixture(scope="module")
def CO(tmp_path_factory):
    return LR.COracle(tmp_path_factory.mktemp("loss_oracle"))


@pytest.fixture(scope="module")
def lbase(oracle):
    return LY.base_problem(oracle)


@pytest.fixture(scope="module")
def sbase(oracle):
    return SL.base_problems(oracle)


@pytest.mark.parametrize("kind", NEW)
@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", LY.LAYOUTS)
def test_partition_layouts(oracle, lbase, grid_full, name, family, kind):
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    if family == "planar" and name.endswith("_z"):
        pytest.skip("z != 0: general kernels only")
    lay = LY.build(name, lbase, grid_full, 256, stage)
    with env(**FAMILIES[family]):
        for edges in (False, True):
            with make(lay, kind, edges) as g:
                assert g.planar == (family == "planar") and g.loss == (kind, A)
                d = g.dispatch()["eval"]
                assert d == expected_dispatch(lay.n_points, len(lay.offsets) - 1, edges, "1")["eval"]
                hits = LY.classify(lay.offsets, *(g.partition(warp_table=False)[k] for k in ("grid", "per_warp")), stage)
                assert lay.targets <= hits | {"partial_resident"}, lay.targets - hits
                for x in (near_optimum(oracle), FAR):
                    check(pack_sums(*g.eval(x)), ref(lay, x, kind, edges), f"{name}/{family}/{kind}/edges={edges} [{d}]")


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("kind", NEW)
@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", SL.LAYOUTS)
def test_small_layouts(oracle, sbase, name, family, kind, kernel):
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    lay = SL.build(name, sbase, stage)
    if family == "planar" and lay.general_only:
        pytest.skip("z != 0: general kernels only")
    P, N = lay.n_points, len(lay.offsets) - 1
    poses = SL.far_range_poses(oracle) if name.startswith("far_range") else (near_optimum(oracle), FAR)
    with env(CLC_SMALL_KERNEL=KERNELS[kernel], **FAMILIES[family]):
        for edges in (False, True):
            if edges and lay.edge_points is None:
                continue
            with make(lay, kind, edges) as g:
                d = g.dispatch()
                assert d == expected_dispatch(P, N, edges, KERNELS[kernel]), (name, d)
                for x in poses:
                    check(pack_sums(*g.eval(x)), ref(lay, x, kind, edges), f"{name}/{family}/{kind}/edges={edges} [{d['eval']}]")


@pytest.mark.parametrize("family", list(FAMILIES))
def test_huber_boundary_scene(oracle, grid_full, family):
    """A scene where every distance is exact: boards with the (unnormalised) quaternion (0, 0.5, 0, 0.5), i.e. the plane
    x + z = 0.5 at the identity pose, and laser points with z = 0, so e = x - 0.5 without rounding.  Points at |e| == a and at
    the neighbouring x either side, in frames that cross warp ranges.  a is 0.05 on the grid of x, so that 0.5 +- a is a
    double."""
    from camlasercalibratool_b200 import Problem

    ab = (0.5 + A) - 0.5
    n_frames, per = 40, 4000 if family == "general" else 12000
    rng = np.random.default_rng(3)
    fp = np.tile([0.0, 0.5, 0.0, 0.5, 0.5, 0.0, 0.0], (n_frames, 1))  # (qx qy qz qw tx ty tz)
    off = np.arange(n_frames + 1, dtype=np.int64) * per
    hi, lo = 0.5 + ab, 0.5 - ab
    x = rng.choice([hi, lo, np.nextafter(hi, 1), np.nextafter(hi, 0), np.nextafter(lo, 0), np.nextafter(lo, 1), 0.51, 0.8],
                   size=n_frames * per)
    e = x - 0.5
    pts = np.column_stack([x, rng.uniform(-1, 1, n_frames * per), np.zeros(n_frames * per)])
    np.testing.assert_array_equal(X.frame_planes(fp[:1]).astype(np.float64), [[1.0, 0.0, 1.0, -0.5]])
    with env(**FAMILIES[family]), Problem.from_arrays(fp, off, pts) as g:
        g.set_loss("huber", ab)
        assert g.planar == (family == "planar")
        assert g.partition(warp_table=False)["per_warp"] < per
        # the device's distances are the exact ones: every frame's max |e| and mean e
        rows = g.frame_report(X0)
        fo = np.repeat(np.arange(n_frames), per)
        assert np.array_equal(rows["max_abs_e"], np.array([np.abs(e[fo == f]).max() for f in range(n_frames)]))
        got = pack_sums(*g.eval(X0))
        check(got, LR.lm_sums(fp, off, pts, X0, "huber", ab), f"huber boundary/{family}")
        # the inlier rule, cost term by cost term: |e| == a adds e^2, the next x beyond adds 2a|e| - a^2
        ld = np.longdouble
        inl = np.abs(e) <= ab
        assert np.sum(np.abs(e) == ab) > 0 and np.sum(~inl & (np.abs(e) < 1e-12 + ab)) > 0
        rho = np.where(inl, e.astype(ld) ** 2, 2 * ld(ab) * np.abs(e).astype(ld) - ld(ab) ** 2)
        np.testing.assert_allclose(float(0.5 * rho.sum() / per), got[27], rtol=1e-13)


@pytest.mark.parametrize("kind", NEW)
@pytest.mark.parametrize("family", list(FAMILIES))
def test_frame_report(oracle, lbase, grid_full, family, kind):
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    lay = LY.build("L3_empty_runs", lbase, grid_full, 256, stage)
    x = FAR
    with env(**FAMILIES[family]):
        for edges in (False, True):
            with make(lay, kind, edges) as g, make(lay, "cauchy", edges) as gc:
                rows, rc = g.frame_report(x), gc.frame_report(x)
                # the loss-free fields are the Cauchy report's, bit for bit
                for f in ("n_points", "chi", "mean_e", "rms_e", "max_abs_e", "edge_e"):
                    assert np.array_equal(rows[f], rc[f], equal_nan=True), f
                per = LR.frame_sums(lay.frame_pose, lay.offsets, lay.points, x, kind, A, lay.edge_points if edges else None)
                for fr, (val, mag) in enumerate(per):
                    got = np.concatenate([rows["H21"][fr], rows["g6"][fr], [rows["cost"][fr]]])
                    check(got, (val, mag), f"frame {fr}/{family}/{kind}/edges={edges}")
                cost, H, gr = g.eval(x)
                tot = np.concatenate([rows["H21"].sum(axis=0), rows["g6"].sum(axis=0), [rows["cost"].sum()]])
                check(tot, ref(lay, x, kind, edges), f"rows sum/{family}/{kind}")
                # mean weight: sum w / n of the frame's points
                c = np.diff(lay.offsets)
                R = LR.X._rot(np.asarray(x, dtype=np.float64).astype(LR.LD)[3:7])
                pl = LR.X.frame_planes(lay.frame_pose)
                fo = np.repeat(np.arange(len(c)), c)
                m = np.einsum("ij,jk->ik", pl[fo, :3], R)
                ee = np.sum(m * lay.points.astype(LR.LD), axis=1) + pl[fo, :3] @ np.asarray(x[:3]).astype(LR.LD) + pl[fo, 3]
                w = LR.weight_and_cost(kind, ee, A)[0]
                mw = np.zeros(len(c), dtype=LR.LD)
                np.add.at(mw, fo, w)
                live = c > 0
                np.testing.assert_allclose(rows["mean_weight"][live], (mw[live] / c[live]).astype(float), rtol=1e-12)


@pytest.mark.parametrize("kind", NEW)
@pytest.mark.parametrize("family", list(FAMILIES))
def test_segments(oracle, family, kind):
    d = ragged(oracle, 400 if family == "general" else 1500, seed=11)
    with env(**FAMILIES[family]):
        for edges in (False, True):
            with make(d, kind, edges) as g:
                off = seams(g.partition(warp_table=False), d.offsets, len(d.offsets) - 1)
                W = len(off) - 1
                poses = np.stack([oracle.pose_plus(FAR, 0.01 * s * np.array([1.0, -0.5, 0.2, 0.3, 0.1, -0.4])) for s in range(W)])
                cost, H, gr = g.eval_segments(off, poses)
                for s in range(W):
                    sl = d.slice(int(off[s]), int(off[s + 1]))
                    got = pack_sums(cost[s], H[s], gr[s])
                    check(got, ref(sl, poses[s], kind, edges), f"segment {s}/{family}/{kind}/edges={edges}")
            # solve_segments equals fresh-problem solves (a reference-sized rig per segment)
    rig = oracle.generate(120, 180, seed=2, sigma=0.01)
    dd = Data(rig.frame_pose, rig.offsets, rig.points, None)
    off = np.array([0, 40, 80, 120])
    with env(**FAMILIES[family]), make(dd, kind) as g:
        xs, sms, _ = g.solve_segments(off, np.tile(X0, (3, 1)))
        for s in range(3):
            with make(dd.slice(int(off[s]), int(off[s + 1])), kind) as gs:
                x, sm, _ = gs.solve(X0)
            assert sms[s].termination == sm.termination and sms[s].num_iterations == sm.num_iterations
            np.testing.assert_allclose(xs[s], x, rtol=0, atol=1e-12)


def _solve(d, kind, **knobs):
    with env(**knobs), make(d, kind) as g:
        x, s, tr = g.solve(X0)
        return g.dispatch()["solve"], x, s, tr


@pytest.mark.parametrize("kind", NEW)
@pytest.mark.parametrize("scene", ["config1", "outliers", "multi_block"])
def test_solves_follow_the_oracle_under_every_driver(oracle, CO, kind, scene):
    if scene == "multi_block":
        p = oracle.generate(300, 700, seed=5, sigma=0.01, exact_m=True)
    else:
        p = oracle.generate(50, 180, seed=1, sigma=0.01)
    pts = p.points.copy()
    if scene == "outliers":
        rng = np.random.default_rng(7)
        k = rng.choice(len(pts), size=len(pts) // 20, replace=False)
        pts[k, :2] += rng.uniform(0.3, 1.0, size=(len(k), 2)) * rng.choice([-1, 1], size=(len(k), 2))
    d = Data(p.frame_pose, p.offsets, pts, None)
    base = dict(CLC_PLANAR="0")
    runs = {"launch_pdl": _solve(d, kind, CLC_LOOP_IN_KERNEL="0", CLC_SMALL_KERNEL="0", **base),
            "launch_no_pdl": _solve(d, kind, CLC_LOOP_IN_KERNEL="0", CLC_SMALL_KERNEL="0", CLC_PDL="0", **base),
            "persistent": _solve(d, kind, CLC_LOOP_IN_KERNEL="2", CLC_SMALL_KERNEL="0", **base)}
    if scene != "multi_block":
        runs["single_block_loop"] = _solve(d, kind, CLC_LOOP_IN_KERNEL="1", CLC_SMALL_KERNEL="0", **base)
        runs["k2"] = _solve(d, kind, CLC_LOOP_IN_KERNEL="1", CLC_SMALL_KERNEL="1", **base)
        assert runs["single_block_loop"][0] == "single_block_loop" and runs["k2"][0] == "one_cluster"
    ref_run = runs["launch_pdl"]
    for name, (path, x, s, tr) in runs.items():
        same = name != "k2"
        if same:  # the sweep kernel's drivers: bit for bit
            assert np.array_equal(x, ref_run[1]), name
            assert [t.cost for t in tr] == [t.cost for t in ref_run[3]], name
        else:
            np.testing.assert_allclose(x, ref_run[1], rtol=0, atol=1e-12)
        assert s.termination == ref_run[2].termination and s.num_iterations == ref_run[2].num_iterations, name
        assert [(t.step_is_valid, t.step_is_successful) for t in tr] == [(t.step_is_valid, t.step_is_successful) for t in ref_run[3]]
    # the C oracle of the losses (tests/loss_oracle.c): the same decisions, termination and counts
    xo, so, tro = CO.solve(oracle.Problem(d.frame_pose, d.offsets, d.points), X0, kind, A)
    x, s, tr = ref_run[1:]
    assert s.termination == so.termination and s.num_iterations == so.num_iterations
    assert (s.num_successful_steps, s.num_unsuccessful_steps) == (so.num_successful_steps, so.num_unsuccessful_steps)
    assert [(t.step_is_valid, t.step_is_successful) for t in tr] == [(t.step_is_valid, t.step_is_successful) for t in tro]
    ang, dt = oracle.pose_error(x, xo)
    assert ang < 1e-9 and dt < 1e-9, (ang, dt)


@pytest.mark.parametrize("kind", NEW)
def test_noise_free_reaches_the_truth(oracle, kind):
    p = oracle.generate(50, 180, seed=1, sigma=0.0)
    with make(Data(p.frame_pose, p.offsets, p.points, None), kind) as g:
        x, s, _ = g.solve(X0)
    ang, dt = oracle.pose_error(x, oracle.ground_truth()[1])
    assert ang < 1e-9 and dt < 1e-9, (ang, dt)


# ---- no behaviour change, by bytes ------------------------------------------------------------------------------------
def _everything(g, d, x):
    cost, H, gr = g.eval(x)
    xs, s, tr = g.solve(X0)
    summ = (s.termination, s.num_iterations, s.num_successful_steps, s.num_unsuccessful_steps, s.num_sweeps, s.initial_cost,
            s.final_cost)
    trace = [(t.iteration, t.step_is_valid, t.step_is_successful, t.cost, t.cost_change, t.gradient_max_norm, t.step_norm,
              t.relative_decrease, t.trust_region_radius) for t in tr]
    rows = g.frame_report(x).tobytes()
    off = np.array([0, len(d.offsets) // 3, len(d.offsets) - 1])
    seg = g.eval_segments(off, np.stack([x, FAR]))
    return (pack_sums(cost, H, gr).tobytes(), xs.tobytes(), summ, trace, rows, b"".join(np.asarray(v).tobytes() for v in seg))


def _analysis(g, x):
    H, b, chi, sv = g.information(x)
    T, un, AtA, Atb = g.closed_form()
    return b"".join(np.asarray(v).tobytes() for v in (H, b, chi, sv, T, AtA, Atb)) + bytes([un])


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("size", ["k2", "multi_block"])
def test_set_loss_cauchy_is_the_use_loss_problem(oracle, family, size):
    from camlasercalibratool_b200 import Problem

    p = oracle.generate(50, 180, seed=1, sigma=0.01, with_edges=True) if size == "k2" else \
        oracle.generate(200, 1000, seed=3, sigma=0.01, exact_m=True, with_edges=True)
    d = Data(p.frame_pose, p.offsets, p.points, p.edge_points)
    x = near_optimum(oracle)
    with env(**FAMILIES[family]):
        with Problem.from_arrays(d.frame_pose, d.offsets, d.points, d.edge_points, use_loss=True, cauchy_a=0.07) as g1:
            want, ana = _everything(g1, d, x), _analysis(g1, x)
            assert g1.loss == ("cauchy", 0.07)
        with Problem.from_arrays(d.frame_pose, d.offsets, d.points, d.edge_points, use_loss=False, cauchy_a=0.07) as g0:
            assert g0.loss == ("none", 0.07)
            none = _everything(g0, d, x)
            g0.set_loss("cauchy", 0.07)
            assert _everything(g0, d, x) == want
            assert _analysis(g0, x) == ana
            for k in NEW:
                g0.set_loss(k, 0.03)
                assert _analysis(g0, x) == ana  # information and the closed form never use the loss
                assert _everything(g0, d, x)[0] != want[0]
            g0.set_loss("cauchy", 0.07)
            assert _everything(g0, d, x) == want
            g0.set_loss(None)
            assert g0.loss == ("none", 0.05) and _everything(g0, d, x) == none
            # a rejected set_loss leaves the loss as it was, in the library as well as through the Python checks
            g0.set_loss("huber", 0.04)
            for kind, bad_a in ((7, 0.05), (3, 0.0), (3, float("nan")), (1, 1e-160)):
                assert g0._L.clc_problem_set_loss(g0._h, kind, bad_a) == 1
                assert g0.loss == ("huber", 0.04)
            with pytest.raises(ValueError):
                g0.set_loss("tukey", 0.05)
            assert g0.loss == ("huber", 0.04)


@pytest.mark.parametrize("kind", NEW)
def test_subset_trim_and_group_inherit_the_loss(oracle, kind):
    from camlasercalibratool_b200 import Group, Problem

    p = oracle.generate(80, 300, seed=2, sigma=0.01, exact_m=True, with_edges=True)
    d = Data(p.frame_pose, p.offsets, p.points, p.edge_points)
    x = near_optimum(oracle)
    keep = np.arange(80) % 3 != 1
    with make(d, kind, edges=True, a=0.04) as g:
        with g.subset(keep) as gs:
            assert gs.loss == (kind, 0.04)
            kf = np.nonzero(keep)[0]
            o = d.offsets
            pts = np.concatenate([d.points[o[f]:o[f + 1]] for f in kf])
            fo = np.concatenate([[0], np.cumsum(np.diff(o)[kf])])
            fresh = Data(d.frame_pose[kf], fo, pts, d.edge_points[kf])
            with make(fresh, kind, edges=True, a=0.04) as gf:
                assert _everything(gs, fresh, x) == _everything(gf, fresh, x)
        rows = g.frame_report(x)
        tau = 2.0 * rows["rms_e"]
        with g.trim(x, tau) as gt:
            assert gt.loss == (kind, 0.04)
            nd = gt.download()
            fresh = Data(nd["frame_pose"], nd["offsets"], nd["points"], nd["edge_points"])
            with make(fresh, kind, edges=True, a=0.04) as gf:
                assert _everything(gt, fresh, x) == _everything(gf, fresh, x)
        with Group.from_arrays(d.frame_pose, d.offsets, d.points, d.edge_points, devices=(0,)) as grp:
            grp.set_loss(kind, 0.04)
            c1, H1, g1 = g.eval(x)
            c2, H2, g2 = grp.eval(x)
            assert pack_sums(c1, H1, g1).tobytes() == pack_sums(c2, H2, g2).tobytes()
            assert g.frame_report(x).tobytes() == grp.frame_report(x).tobytes()
            assert np.array_equal(grp.solve(X0)[0], g.solve(X0)[0])


def test_zz_report_headroom():
    print("\nworst |err| / A_k per output group (GAMMA = %.0e): %s" % (X.GAMMA, {k: f"{v:.2e}" for k, v in WORST.items()}))
