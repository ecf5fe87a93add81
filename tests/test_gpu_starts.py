"""One calibration at many poses (clc_eval_poses, clc_solve_lm_starts) on the GPU.

* Every pose's sums lie within GAMMA * A_k of the long-double reference on the adversarial layouts of the sweep kernel's
  partition, both kernel families, every loss kind, with and without edge residuals, with more poses than one tile holds.
* Problems the one-cluster kernel serves return, for pose k, the bytes of eval / solve from poses[k].
* On the sweep kernel every start makes the decisions of solve from that start, to a pose within 1e-12.
* Pose k's bytes depend on poses[k] only: K = 1 equals that row of a larger call, permuting the poses permutes the outputs, two
  calls agree, and a start that stops at once next to long ones changes nothing.
* Noise-free data: the best start reaches the truth; subset, trim and set_loss compose.
"""
import numpy as np
import pytest

import exact_sums as X
import layouts as LY
import loss_reference as LR
import small_layouts as SL

from conftest import pack_sums
from test_gpu_partition import FAMILIES, FAR, X0, env, near_optimum

pytestmark = pytest.mark.gpu

KINDS = ("none", "cauchy", "huber", "soft_l1")
A = 0.05
KT = 32  # kPoseTile (csrc/clc_kernels.cuh)


def random_starts(oracle, K, seed, rot=np.pi, trans=0.5):
    """K start poses (t, q): rotations by up to `rot` about random axes, translations up to `trans` metres (fixed seed)."""
    rng = np.random.default_rng(seed)
    xs = []
    for _ in range(K):
        axis = rng.standard_normal(3)
        axis /= np.linalg.norm(axis)
        ang = rng.uniform(0, rot)
        xs.append(np.concatenate([rng.uniform(-trans, trans, 3), np.sin(ang / 2) * axis, [np.cos(ang / 2)]]))
    return np.array(xs)


def mixed_poses(oracle, K, seed):
    """K poses: near the optimum, far away and in between."""
    rng = np.random.default_rng(seed)
    x0 = oracle.ground_truth()[1]
    out = [near_optimum(oracle), FAR, X0]
    while len(out) < K:
        out.append(oracle.pose_plus(x0, 10.0 ** rng.uniform(-4, -0.5) * rng.standard_normal(6)))
    return np.array(out[:K])


def make(d, kind, edges):
    from camlasercalibratool_b200 import Problem

    g = Problem.from_arrays(d.frame_pose, d.offsets, d.points, d.edge_points if edges else None, use_loss=True, cauchy_a=A)
    g.set_loss(kind, A)
    return g


@pytest.fixture(scope="module")
def grid_full():
    from camlasercalibratool_b200 import Problem

    with Problem.synthetic(600, 1000) as probe:
        return probe.partition(warp_table=False)["grid"]


@pytest.fixture(scope="module")
def lbase(oracle):
    return LY.base_problem(oracle)


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", ["L2_off_by_one", "L3_empty_runs", "L4_giant_frame", "L5_confetti"])
def test_sums_against_long_double(oracle, lbase, grid_full, name, family):
    stage = LY.STAGE_PLANAR if family == "planar" else LY.STAGE_GENERAL
    lay = LY.build(name, lbase, grid_full, 256, stage)
    K = KT + 3  # two tiles
    x = mixed_poses(oracle, K, seed=5)
    checked = (0, 1, 2, KT - 1, KT, K - 1)
    with env(**FAMILIES[family]):
        for kind in KINDS:
            for edges in (False, True):
                with make(lay, kind, edges) as g:
                    assert g.planar == (family == "planar")
                    assert g.dispatch()["eval"] != "one_cluster"
                    cost, H, gr = g.eval_poses(x)
                    for k in checked:
                        val, mag = LR.lm_sums(lay.frame_pose, lay.offsets, lay.points, x[k], kind, A,
                                              lay.edge_points if edges else None)
                        X.assert_within(pack_sums(cost[k], H[k], gr[k]), val, mag, X.GROUPS_LM,
                                        f"{name}/{family}/{kind}/edges={edges}/pose {k}")
                    # K = 1 and K = KT: the bytes of the same rows
                    for sel in ([K - 1], list(range(KT))):
                        c1, H1, g1 = g.eval_poses(x[sel])
                        assert c1.tobytes() == cost[sel].tobytes() and H1.tobytes() == H[sel].tobytes()
                        assert g1.tobytes() == gr[sel].tobytes()


SMALL = ["seam_2048", "seam_2049", "one_point_frames_edges", "edges_total_16384", "one_frame_16384"]


@pytest.mark.parametrize("name", SMALL)
def test_one_cluster_path_is_bytes_equal(oracle, name):
    bases = SL.base_problems(oracle)
    lay = SL.build(name, bases, LY.STAGE_GENERAL)
    edges = lay.edge_points is not None
    x = mixed_poses(oracle, 6, seed=11)
    with env(CLC_SMALL_KERNEL="1", CLC_PLANAR="0"):
        for kind in ("cauchy", "huber"):
            with make(lay, kind, edges) as g:
                d = g.dispatch()
                assert d["eval"] == "one_cluster", d
                cost, H, gr = g.eval_poses(x)
                for k in range(len(x)):
                    c, h, gg = g.eval(x[k])
                    assert np.float64(c).tobytes() == cost[k].tobytes() and h.tobytes() == H[k].tobytes() and gg.tobytes() == gr[k].tobytes()
                if d["solve"] != "one_cluster":
                    continue
                xs, sums, traces, best = g.solve_starts(x, trace_cap=256)
                for k in range(len(x)):
                    xk, sk, tk = g.solve(x[k])
                    assert xk.tobytes() == xs[k].tobytes(), (name, kind, k)
                    assert (sk.termination, sk.num_iterations, sk.final_cost) == (sums[k].termination, sums[k].num_iterations,
                                                                                 sums[k].final_cost)
                    assert [bytes(r) for r in tk] == [bytes(r) for r in traces[k]]


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("kind", ["cauchy", "huber"])
def test_sweep_solves_follow_single_solves(oracle, family, kind):
    from camlasercalibratool_b200 import Problem

    p = oracle.generate(120, 400, seed=4, sigma=0.01)
    x = random_starts(oracle, 6, seed=9, rot=0.5, trans=0.2)
    with env(**FAMILIES[family]), Problem.from_arrays(p.frame_pose, p.offsets, p.points, use_loss=True, cauchy_a=A) as g:
        g.set_loss(kind, A)
        assert g.dispatch()["solve"] != "one_cluster" and g.planar == (family == "planar")
        xs, sums, traces, best = g.solve_starts(x, trace_cap=256)
        for k in range(len(x)):
            xk, sk, tk = g.solve(x[k])
            assert (sk.termination, sk.num_iterations) == (sums[k].termination, sums[k].num_iterations), k
            assert [r.step_is_successful for r in tk] == [r.step_is_successful for r in traces[k]], k
            assert np.abs(xk - xs[k]).max() < 1e-12, (k, np.abs(xk - xs[k]).max())
            if kind == "cauchy":  # the oracle's loss: Cauchy(0.05)
                xo, so, to = oracle.solve(p, x[k])
                assert (sums[k].termination, sums[k].num_iterations) == (so.termination, so.num_iterations), k
                assert [r.step_is_successful for r in traces[k]] == [r.step_is_successful for r in to], k
                assert np.abs(xs[k] - xo).max() < 1e-9, (k, np.abs(xs[k] - xo).max())
        ok = [k for k in range(len(x)) if sums[k].termination != 6]
        assert best == min(ok, key=lambda k: (sums[k].final_cost, k))


def test_independence_permutation_and_repeatability(oracle):
    from camlasercalibratool_b200 import Problem

    p = oracle.generate(200, 400, seed=6, sigma=0.01, with_edges=True)
    x = mixed_poses(oracle, 37, seed=3)
    with Problem.from_arrays(p.frame_pose, p.offsets, p.points, p.edge_points, use_loss=True) as g:
        assert g.dispatch()["eval"] != "one_cluster"
        c, H, gr = g.eval_poses(x)
        c2, H2, gr2 = g.eval_poses(x)
        assert c.tobytes() == c2.tobytes() and H.tobytes() == H2.tobytes() and gr.tobytes() == gr2.tobytes()
        perm = np.random.default_rng(1).permutation(len(x))
        cp, Hp, gp = g.eval_poses(x[perm])
        assert cp.tobytes() == c[perm].tobytes() and Hp.tobytes() == H[perm].tobytes() and gp.tobytes() == gr[perm].tobytes()
        for k in (0, 17, 36):
            c1, H1, g1 = g.eval_poses(x[k:k + 1])
            assert c1.tobytes() == c[k:k + 1].tobytes() and H1.tobytes() == H[k:k + 1].tobytes()
        # a start at the solution stops at once, next to starts that run long
        xsol, s0, _ = g.solve(near_optimum(oracle))
        starts = np.stack([FAR, xsol, X0, near_optimum(oracle, 1e-1)])
        xs, sums, tr, best = g.solve_starts(starts, trace_cap=64)
        assert sums[1].num_iterations <= 2 < max(s.num_iterations for s in sums)
        xs2, sums2, tr2, best2 = g.solve_starts(starts, trace_cap=64)
        assert xs.tobytes() == xs2.tobytes() and best == best2
        for k in range(len(starts)):
            x1, s1, t1, _ = g.solve_starts(starts[k:k + 1], trace_cap=64)
            assert x1.tobytes() == xs[k:k + 1].tobytes(), k
            assert bytes(s1[0])[:-8] == bytes(sums[k])[:-8] or (s1[0].final_cost == sums[k].final_cost
                                                                  and s1[0].num_iterations == sums[k].num_iterations)
            assert [bytes(r) for r in t1[0]] == [bytes(r) for r in tr[k]]
        xr, sr, _, _ = g.solve_starts(starts[::-1].copy(), trace_cap=0)
        assert xr.tobytes() == xs[::-1].tobytes()


@pytest.mark.parametrize("size", [(50, 180), (300, 400)])
def test_noise_free_best_start_reaches_the_truth(oracle, size):
    from camlasercalibratool_b200 import Problem

    p = oracle.generate(*size, seed=2, sigma=0.0)
    x_gt = oracle.ground_truth()[1]
    x = random_starts(oracle, 16, seed=7)
    with Problem.from_arrays(p.frame_pose, p.offsets, p.points, use_loss=True) as g:
        xs, sums, _, best = g.solve_starts(x)
        ok = [k for k in range(len(x)) if sums[k].termination != 6]
        assert best == min(ok, key=lambda k: (sums[k].final_cost, k))
        ang, dt = oracle.pose_error(xs[best], x_gt)
        assert ang < 1e-9 and dt < 1e-9, (ang, dt)


def test_composition_with_subset_trim_and_set_loss(oracle):
    from camlasercalibratool_b200 import Problem

    p = oracle.generate(150, 300, seed=8, sigma=0.01)
    x = mixed_poses(oracle, 5, seed=4)
    with Problem.from_arrays(p.frame_pose, p.offsets, p.points, use_loss=True) as g:
        keep = np.arange(150) % 2 == 0
        with g.subset(keep) as s:
            c, H, gr = s.eval_poses(x)
            for k in range(len(x)):
                ck, Hk, gk = s.eval(x[k])
                assert abs(ck - c[k]) <= 1e-12 * abs(ck) and np.abs(Hk - H[k]).max() <= 1e-12 * np.abs(Hk).max()
        with g.trim(near_optimum(oracle), 0.02) as tr:
            xs, sums, _, best = tr.solve_starts(x[:3])
            for k in range(3):
                xk, sk, _ = tr.solve(x[k])
                assert sk.num_iterations == sums[k].num_iterations and np.abs(xk - xs[k]).max() < 1e-12
        g.set_loss("soft_l1", 0.03)
        c, H, gr = g.eval_poses(x)
        for k in range(len(x)):
            ck, Hk, gk = g.eval(x[k])
            assert abs(ck - c[k]) <= 1e-12 * abs(ck) and np.abs(Hk - H[k]).max() <= 1e-12 * np.abs(Hk).max()


def test_communicator_attached_problem_is_refused(oracle):
    """Multi-pose calls run on a problem without a communicator: CLC_ERR_STATE, before any device work."""
    import ctypes as C

    from camlasercalibratool_b200 import Comm, Problem, comm_unique_id
    from camlasercalibratool_b200._lib import LmSummary

    try:
        comm = Comm(comm_unique_id(), 1, 0, device=0)
    except Exception as exc:  # no NCCL on this machine
        pytest.skip(f"no communicator: {exc}")
    p = oracle.generate(30, 180, seed=1, sigma=0.01)
    x = mixed_poses(oracle, 3, seed=1)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    with Problem.from_arrays(p.frame_pose, p.offsets, p.points) as g:
        g.attach_comm(comm)
        cost = np.zeros(3)
        summ = (LmSummary * 3)()
        best = C.c_int64(-7)
        ms = (C.c_float * 1)()
        xs = x.copy()
        assert g._L.clc_eval_poses(g._h, 3, dp(x), None, None, dp(cost)) == 4
        assert g._L.clc_solve_lm_starts(g._h, 3, dp(xs), None, summ, None, 0, C.byref(best)) == 4
        assert g._L.clc_bench_poses(g._h, 3, dp(x), 1, 0, ms) == 4
        assert np.array_equal(xs, x) and best.value == -7
        g.attach_comm(None)
        c, _, _ = g.eval_poses(x)  # detached: served again
        assert c.tobytes() == np.array([g.eval(x[k])[0] for k in range(3)]).tobytes()
    comm.close()


# ---- at the size the benchmarks run: 10^7 points, K = KT + 1 (two tiles) -----------------------------------------------------
@pytest.mark.parametrize("family", list(FAMILIES))
def test_sums_at_scale(oracle, family):
    """configs[1] (10^4 frames x 10^3 points): every lane adds thousands of points and every warp range holds split frames.  The
    checked poses' sums within GAMMA * A_k of the long-double reference (computed over frame ranges in forked workers) under the
    four loss kinds; every other row equals the bytes of a call with that pose alone."""
    import scale_scenes as SS
    from test_gpu_segments import Data, plane_slack

    from camlasercalibratool_b200 import Problem

    K = KT + 1
    x = mixed_poses(oracle, K, seed=13)
    checked = (0, 1, KT)
    with env(**FAMILIES[family]), Problem.synthetic(10_000, 1_000, seed=SS.SEED, sigma=SS.SIGMA) as g:
        assert g.planar == (family == "planar") and g.dispatch()["eval"] != "one_cluster"
        d = g.download()
        arrays = (d["frame_pose"], d["offsets"], d["points"], None)
        slack = plane_slack(Data(d["frame_pose"], d["offsets"], None, None))
        for kind in KINDS:
            g.set_loss(kind, A)
            cost, H, gr = g.eval_poses(x)
            for k in checked:
                val, mag = SS.spread(arrays, "lm", (x[k], kind, False))
                X.assert_within(pack_sums(cost[k], H[k], gr[k]), val, mag + slack, X.GROUPS_LM, f"scale/{family}/{kind}/pose {k}")
            for k in (2, KT - 1):
                c1, H1, g1 = g.eval_poses(x[k:k + 1])
                assert c1.tobytes() == cost[k:k + 1].tobytes() and H1.tobytes() == H[k:k + 1].tobytes()
                assert g1.tobytes() == gr[k:k + 1].tobytes()
