"""Independent solves over runs of frames (clc_eval_segments, clc_information_segments, clc_solve_lm_segments) on the GPU.

Segment s's results are those of a fresh problem of its frames alone: its sums within GAMMA * A_k of the long-double reference on
its slice, its solve making the decisions of clc_solve_lm on the fresh problem and of the oracle, to a pose within 1e-12 on a
reference-sized rig (1e-9 on segments of a few ragged frames).  A NaN point or moved points in one segment leave every other
segment's outputs bit-identical.
"""
import contextlib
import os

import numpy as np
import pytest

import exact_sums as X

pytestmark = pytest.mark.gpu

FAMILIES = {"general": dict(CLC_PLANAR="0"), "planar": dict(CLC_PLANAR="1", CLC_PLANAR_MIN_POINTS="0")}
MODES = {"loss": (True, False), "no_loss": (False, False), "edges": (True, True)}  # use_loss, edge residuals
IDENT = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
GROUPS = {"all": slice(None)}
MIN_LIVE_FRAMES = 20  # segments with at least this many non-empty frames are held to the 1e-12 pose bound


@contextlib.contextmanager
def env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


class Data:
    def __init__(self, frame_pose, offsets, points, edge_points):
        self.frame_pose, self.offsets, self.points, self.edge_points = frame_pose, np.asarray(offsets, dtype=np.int64), points, edge_points

    def slice(self, a, b):
        o = self.offsets
        ep = None if self.edge_points is None else self.edge_points[a:b]
        return Data(self.frame_pose[a:b], o[a:b + 1] - o[a], self.points[o[a]:o[b]], ep)

    def problem(self, use_loss=True, edges=False):
        from camlasercalibratool_b200 import Problem

        return Problem.from_arrays(self.frame_pose, self.offsets, self.points, self.edge_points if edges else None,
                                   use_loss=use_loss)


def ragged(oracle, n_frames, seed, sigma=0.01):
    """Oracle frames with random point counts: empty frames, one-point frames and frames of a few to 400 points."""
    rng = np.random.default_rng(seed)
    p = oracle.generate(n_frames, 400, seed=seed, sigma=sigma, with_edges=True)
    counts = rng.choice([0, 1, 2, 5, 37, 180, 400], size=n_frames, p=[0.05, 0.1, 0.1, 0.15, 0.2, 0.25, 0.15])
    pts, off = [], [0]
    for f in range(n_frames):
        a = p.offsets[f]
        k = min(int(counts[f]), int(p.offsets[f + 1] - a))
        pts.append(p.points[a:a + k])
        off.append(off[-1] + k)
    return Data(p.frame_pose, off, np.concatenate(pts), p.edge_points)


def seams(part, offsets, n_frames):
    """Segment boundaries on the frames around the warp-range and stage ends of the partition (and one either side), plus empty
    segments, a one-frame segment and a long segment across many warp ranges."""
    per_warp, stage = part["per_warp"], part["stage"]
    P = int(offsets[-1])
    cuts = set()
    for step in (stage, per_warp, per_warp * 12):
        for q in range(step, P, step):
            f = int(np.searchsorted(offsets, q, side="right")) - 1
            for d in (-1, 0, 1):
                if 0 < f + d < n_frames:
                    cuts.add(f + d)
    cuts = sorted(cuts)
    # keep a long segment: drop the cuts inside the middle third
    lo, hi = n_frames // 3, 2 * n_frames // 3
    cuts = [c for c in cuts if not lo < c < hi]
    off = [0] + cuts + [n_frames]
    # empty segments at two seams and a one-frame segment
    off = sorted(off + [cuts[0], cuts[0], cuts[-1]] + ([cuts[1] + 1] if len(cuts) > 1 and cuts[1] + 1 < n_frames else []))
    return np.array(off, dtype=np.int64)


def seg_poses(oracle, W, seed, scale=1e-2):
    rng = np.random.default_rng(seed)
    x0 = oracle.ground_truth()[1]
    return np.stack([oracle.pose_plus(x0, scale * rng.standard_normal(6)) for _ in range(W)])


def plane_slack(sl):
    """The board planes are inputs the library rounds once (frame_plane, |n| = 1), to about one ulp of |n| in every component.
    exact_sums' magnitudes do not carry that term; it matters in a segment of one or two frames whose normal has a tiny component,
    where H_tt[i, j] = s^2 sum w n_i n_j is small.  Adds |dH_ij / dn| |n| = (|n_i| + |n_j|) s^2 sum w <= |n_i| + |n_j| per live frame
    to the six H_tt magnitudes."""
    slack = np.zeros(28)
    live = np.diff(sl.offsets) > 0
    if np.any(live):
        n = np.abs(np.asarray(X.frame_planes(sl.frame_pose[live]), dtype=np.float64)[:, :3])
        for k, (i, j) in zip((0, 1, 2, 6, 7, 11), ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))):
            slack[k] = float(np.sum(n[:, i] + n[:, j]))
    return slack


@pytest.mark.parametrize("family", list(FAMILIES))
def test_sums_against_long_double(oracle, family):
    d = ragged(oracle, 900, seed=3)
    with env(**FAMILIES[family]):
        for mode, (loss, edges) in MODES.items():
            with d.problem(loss, edges) as g:
                assert g.planar == (family == "planar")
                off = seams(g.partition(warp_table=False), d.offsets, len(d.frame_pose))
                W = len(off) - 1
                assert W > 20
                x = seg_poses(oracle, W, seed=W)
                cost, H, gr = g.eval_segments(off, x)
                Hi, b, chi, sv = g.information_segments(off, x)
                for s in range(W):
                    sl = d.slice(off[s], off[s + 1])
                    ep = sl.edge_points if edges else None
                    val, mag = X.lm_sums(sl.frame_pose, sl.offsets, sl.points, x[s], loss, 0.05, ep)
                    mag = mag + plane_slack(sl)
                    X.assert_within(X.pack_lm(cost[s], H[s], gr[s]), val, mag, GROUPS, f"{family}/{mode}/eval segment {s}")
                    val, mag = X.lm_sums(sl.frame_pose, sl.offsets, sl.points, x[s], False, 0.05, None)
                    mag = mag + plane_slack(sl)
                    X.assert_within(X.pack_lm(chi[s] / 2, Hi[s], -b[s]), val, mag, GROUPS, f"{family}/{mode}/information segment {s}")
                    if off[s] == off[s + 1]:
                        assert cost[s] == 0 and not np.any(H[s]) and not np.any(gr[s])
                # two calls: identical bytes
                c2, H2, g2 = g.eval_segments(off, x)
                assert c2.tobytes() == cost.tobytes() and H2.tobytes() == H.tobytes() and g2.tobytes() == gr.tobytes()


def _T(p7):
    from camlasercalibratool_b200 import pose7_to_T

    return pose7_to_T(p7)


def test_distinct_truths_noise_free(oracle):
    """Segment s's boards are seen by a camera moved by M_s: its extrinsic is M_s T_cl; every segment reaches its own."""
    from camlasercalibratool_b200 import T_to_pose7

    W, per = 6, 50
    p = oracle.generate(W * per, 180, seed=5, sigma=0.0)
    rng = np.random.default_rng(5)
    fp = p.frame_pose.copy()
    truths = []
    x_gt = oracle.ground_truth()[1]
    for s in range(W):
        M = _T(oracle.pose_plus(IDENT, np.r_[0.05 * rng.standard_normal(3), 0.1 * rng.standard_normal(3)]))
        for f in range(s * per, (s + 1) * per):
            Tf = _T(np.r_[fp[f, 4:7], fp[f, 0:4]])
            q = T_to_pose7(M @ Tf)
            fp[f] = np.r_[q[3:7], q[0:3]]
        truths.append(T_to_pose7(M @ _T(x_gt)))
    d = Data(fp, p.offsets, p.points, None)
    off = np.arange(0, W * per + 1, per)
    with d.problem() as g:
        x, summ, _ = g.solve_segments(off, np.tile(IDENT, (W, 1)))
    for s in range(W):
        ang, dt = oracle.pose_error(x[s], truths[s])
        assert ang < 1e-9 and dt < 1e-9, (s, ang, dt, summ[s].termination)


def _same_decisions(a, b, ta, tb, what):
    assert (a.termination, a.num_iterations, a.num_successful_steps, a.num_unsuccessful_steps) == \
        (b.termination, b.num_iterations, b.num_successful_steps, b.num_unsuccessful_steps), what
    assert [(t.step_is_valid, t.step_is_successful) for t in ta] == [(t.step_is_valid, t.step_is_successful) for t in tb], what


@pytest.mark.parametrize("family", list(FAMILIES))
def test_solve_matches_fresh_problems_and_oracle(oracle, family):
    d = ragged(oracle, 600, seed=11)
    rng = np.random.default_rng(11)
    inner = np.sort(rng.choice(np.arange(1, 600), size=10, replace=False))
    off = np.r_[0, inner, inner[4], 600].astype(np.int64)  # one empty segment
    off.sort()
    W = len(off) - 1
    x_gt = oracle.ground_truth()[1]
    x0 = np.stack([IDENT if s % 2 == 0 else oracle.pose_plus(x_gt, 1e-2 * rng.standard_normal(6)) for s in range(W)])
    opts = [None, dict(max_num_iterations=3), dict(function_tolerance=1e-3)]
    from camlasercalibratool_b200 import default_options

    with env(**FAMILIES[family]):
        for o in opts:
            options = default_options(**o) if o else None
            with d.problem() as g:
                x, summ, tr = g.solve_segments(off, x0, options, trace_cap=256)
                x_again, summ2, tr2 = g.solve_segments(off, x0, options, trace_cap=256)
                assert x_again.tobytes() == x.tobytes()
                assert [bytes(t) for ts in tr2 for t in ts] == [bytes(t) for ts in tr for t in ts]
            for s in range(W):
                sl = d.slice(off[s], off[s + 1])
                with sl.problem() as f:  # an empty segment: the fresh problem of zero frames
                    xf, sf, tf = f.solve(x0[s], options)
                _same_decisions(summ[s], sf, tr[s], tf, f"{family}/{o}/segment {s} vs fresh")
                live = int(np.sum(np.diff(sl.offsets) > 0))
                if live == 0:
                    # no residual at all: both sides see exactly zero sums, so everything but the timing is equal bit for bit
                    assert x[s].tobytes() == xf.tobytes() and bytes(summ[s])[:-8] == bytes(sf)[:-8]
                    assert [bytes(t) for t in tr[s]] == [bytes(t) for t in tf]
                    continue
                # the fresh problem sums in another order (the one-cluster kernel or another partition).  With enough frames the
                # optimum is well conditioned and the contract's 1e-12 holds; a segment of a few ragged frames (these random cuts
                # make some) amplifies the summation order, so it is held to 1e-9.
                bound = 1e-12 if live >= MIN_LIVE_FRAMES else 1e-9
                assert np.abs(x[s] - xf).max() <= bound, (s, live, np.abs(x[s] - xf).max())
                if sl.offsets[-1] > 0:
                    oo = oracle.default_options(**(o or {}))
                    xo, so, to = oracle.solve(oracle.Problem(sl.frame_pose, sl.offsets, sl.points), x0[s], oo)
                    _same_decisions(summ[s], so, tr[s], to, f"{family}/{o}/segment {s} vs oracle")
            terms = {sm.termination for sm in summ}
            if o and "max_num_iterations" in o:
                assert 5 in terms  # NO_CONVERGENCE at the cap


def test_one_segment_is_solve(oracle):
    p = oracle.generate(50, 180, seed=1, sigma=0.01)
    d = Data(p.frame_pose, p.offsets, p.points, None)
    with d.problem() as g:
        x1, s1, t1 = g.solve(IDENT)
        x, summ, tr = g.solve_segments([0, 50], IDENT[None], trace_cap=256)
    _same_decisions(summ[0], s1, tr[0], t1, "W = 1")
    assert np.abs(x[0] - x1).max() <= 1e-12


@pytest.mark.parametrize("family", list(FAMILIES))
def test_isolation(oracle, family):
    """A NaN point, or moved points, in segment A (including in a stage shared with segment B): every other segment's pose,
    summary and trace are bit-identical to the clean run; segment A ends as the fresh solve of its slice."""
    d = ragged(oracle, 300, seed=21)
    off = np.array([0, 40, 41, 97, 150, 151, 220, 300], dtype=np.int64)
    W = len(off) - 1
    x0 = seg_poses(oracle, W, seed=4)
    A = 3  # frames 97..150
    live = [f for f in range(off[A], off[A + 1]) if d.offsets[f + 1] - d.offsets[f] > 1]
    bad_nan = d.points.copy()
    bad_nan[d.offsets[live[0]], 0] = np.nan  # x only: z stays 0, so the kernel family does not change
    bad_move = d.points.copy()
    bad_move[d.offsets[live[-1]]:d.offsets[live[-1] + 1], :2] *= 1.3
    # the last point of segment A's last non-empty frame: it shares a stage with segment B's first points
    bad_nan_edge = d.points.copy()
    last = max(f for f in range(off[A], off[A + 1]) if d.offsets[f + 1] > d.offsets[f])
    bad_nan_edge[d.offsets[last + 1] - 1, 1] = np.nan
    with env(**FAMILIES[family]):
        with d.problem() as g:
            planar = g.planar
            xc, sc, tc = g.solve_segments(off, x0, trace_cap=256)
            cc, Hc, gc = g.eval_segments(off, x0)
        for pts in (bad_nan, bad_move, bad_nan_edge):
            dd = Data(d.frame_pose, d.offsets, pts, None)
            with dd.problem() as g:
                assert g.planar == planar == (family == "planar")
                x, s, t = g.solve_segments(off, x0, trace_cap=256)
                c, H, gr = g.eval_segments(off, x0)
            for k in range(W):
                if k == A:
                    continue
                assert x[k].tobytes() == xc[k].tobytes()
                assert bytes(s[k])[:-8] == bytes(sc[k])[:-8]  # every field but device_ms, the last one
                assert [bytes(i) for i in t[k]] == [bytes(i) for i in tc[k]]
                assert c[k].tobytes() == cc[k].tobytes() and H[k].tobytes() == Hc[k].tobytes() and gr[k].tobytes() == gc[k].tobytes()
            sl = dd.slice(off[A], off[A + 1])
            with sl.problem() as f:
                xf, sf, tf = f.solve(x0[A])
            _same_decisions(s[A], sf, t[A], tf, f"{family}: segment A vs its fresh problem")
            if sf.termination != 6:
                assert np.abs(x[A] - xf).max() <= 1e-12
            else:
                assert s[A].termination == 6  # FAILURE: a NaN point at the start


def test_source_unchanged_and_composition(oracle):
    d = ragged(oracle, 200, seed=31)
    off = np.array([0, 60, 130, 200])
    x0 = np.tile(IDENT, (3, 1))
    with d.problem() as g:
        before = g.eval(IDENT)
        g.solve_segments(off, x0)
        after = g.eval(IDENT)
        assert all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(before, after))
        keep = np.ones(200, dtype=bool)
        keep[10:20] = False
        with g.subset(keep) as s:
            xs, ss, _ = s.solve_segments([0, 50, 190], np.tile(IDENT, (2, 1)))
            assert all(sm.termination in (1, 2, 3) for sm in ss)
        with g.trim(IDENT, 10.0) as t:
            xt, st, _ = t.solve_segments(off, x0)
            assert all(sm.termination in (1, 2, 3) for sm in st)
