"""Extended-precision per-frame reference for clc_frame_report, with an error magnitude for every field of every frame.

The per-residual terms and magnitudes are those of tests/exact_sums.py (lm_sums_of_blocks), summed per frame instead of over the
problem; the report's own statistics add four: sum e (magnitude |e| + L_e, the rounding of e = m.p + c), sum e^2 (e^2 + 2|e| L_e),
max |e| (|e| + L_e at the largest) and sum w (w + |w'| L_e).  Rows are compared in the "comparable" form (COLUMNS): the sums the
kernel forms before it divides by the frame's point count, so that every field has a bound of the form GAMMA * A.
Test infrastructure only.
"""
from __future__ import annotations

import numpy as np

import exact_sums as X

LD = X.LD
COLUMNS = ["cost", "chi", "sum_e", "sum_e2", "max_abs_e", "sum_w", "edge_e0", "edge_e1"] + [f"H{k}" for k in range(21)] + \
          [f"g{k}" for k in range(6)]
K = len(COLUMNS)
C_COST, C_CHI, C_SE, C_SE2, C_MAX, C_SW, C_EDGE, C_H, C_G = 0, 1, 2, 3, 4, 5, 6, 8, 29
GROUPS = {"cost": [C_COST], "chi": [C_CHI], "stats": [C_SE, C_SE2, C_MAX, C_SW], "edge_e": [C_EDGE, C_EDGE + 1],
          "H_tt": [C_H + k for k in X.GROUPS_LM["H_tt"]], "H_ttheta": [C_H + k for k in X.GROUPS_LM["H_ttheta"]],
          "H_thetatheta": [C_H + k for k in X.GROUPS_LM["H_thetatheta"]], "g_t": [C_G, C_G + 1, C_G + 2],
          "g_theta": [C_G + 3, C_G + 4, C_G + 5]}


def comparable(rows):
    """Report rows (clc_frame_row records, or [N, 36] arrays in its order) -> [N, K] float64 in the COLUMNS form."""
    if rows.dtype.names:
        n = rows["n_points"].astype(np.float64)
        cols = [rows["cost"], rows["chi"], rows["mean_e"] * n, rows["rms_e"] ** 2 * n, rows["max_abs_e"], rows["mean_weight"] * n,
                rows["edge_e"][:, 0], rows["edge_e"][:, 1]]
        return np.column_stack(cols + [rows["H21"], rows["g6"]])
    r = np.asarray(rows, dtype=np.float64)
    n = r[:, 0]
    return np.column_stack([r[:, 1], r[:, 2], r[:, 3] * n, r[:, 4] ** 2 * n, r[:, 5], r[:, 6] * n, r[:, 7], r[:, 8], r[:, 9:36]])


def _terms(plane, p, s2, R, t, use_loss, a2):
    """Per residual, long double: the 28 LM terms and their magnitudes (exact_sums), e, L_e, w and the magnitude of w."""
    n, d = plane[:, :3], plane[:, 3]
    m = n @ R
    c = n @ t + d
    e = np.sum(m * p, axis=-1) + c
    L_e = X._norm(m) * X._norm(p) + X._norm(n) * X._norm(t) + np.abs(d)
    J = np.concatenate([n, X._cross(p, m)], axis=1)
    Jabs = np.concatenate([np.abs(n), np.repeat((X._norm(p) * X._norm(m))[:, None], 3, axis=1)], axis=1)
    if use_loss:
        q = e * e / a2
        w = LD(1) / (LD(1) + q)
        dw = 2 * np.abs(e) * w * w / a2
        lg = np.log1p(q)
        cost = LD(0.5) * s2 * a2 * lg
        cost_mag = 0.5 * s2 * a2 * (lg + LD(X.U_PROD)) + s2 * w * np.abs(e) * L_e
    else:
        w = np.ones_like(e)
        dw = np.zeros_like(e)
        cost = LD(0.5) * s2 * e * e
        cost_mag = cost + s2 * np.abs(e) * L_e
    sw = s2 * w
    val = np.concatenate([J[:, X.IU6[0]] * J[:, X.IU6[1]] * sw[:, None], J * (sw * e)[:, None], cost[:, None]], axis=1)
    Jf = Jabs.astype(np.float64)
    hw = (s2 * (w + dw * L_e)).astype(np.float64)
    mag = np.concatenate([Jf[:, X.IU6[0]] * Jf[:, X.IU6[1]] * hw[:, None], Jf * (sw * L_e).astype(np.float64)[:, None],
                          cost_mag.astype(np.float64)[:, None]], axis=1)
    return val, mag, e, L_e, w, (w + dw * L_e)


def frame_sums(frame_pose, offsets, points, pose7, use_loss=True, cauchy_a=0.05, edge_points=None):
    """(val [N, K] long double, mag [N, K] float64) per frame, in the COLUMNS form.  Empty frames: zeros, magnitude 0."""
    off = np.asarray(offsets, dtype=np.int64)
    counts = np.diff(off)
    N, P = len(counts), int(off[-1])
    val = np.zeros((N, K), dtype=LD)
    mag = np.zeros((N, K))
    planes = X.frame_planes(frame_pose)
    s2f = np.zeros(N, dtype=LD)
    s2f[counts > 0] = LD(1) / counts[counts > 0].astype(LD)
    pose = np.asarray(pose7, dtype=np.float64).astype(LD)
    R, t = X._rot(pose[3:7]), pose[:3]
    a2 = LD(cauchy_a) * LD(cauchy_a)
    f_of = np.repeat(np.arange(N), counts)
    mx = np.full(N, -1.0, dtype=LD)  # max |e| (NaN kept) and the magnitude at it
    for a in range(0, P, X.CHUNK):
        b = min(P, a + X.CHUNK)
        f = f_of[a:b]
        p = np.asarray(points[a:b], dtype=np.float64).astype(LD)
        v, mg, e, L_e, w, wmag = _terms(planes[f], p, s2f[f], R, t, use_loss, a2)
        s2 = s2f[f]
        ev = np.column_stack([v[:, 27], s2 * e * e, e, e * e, w])
        em = np.column_stack([mg[:, 27], (s2 * (e * e + 2 * np.abs(e) * L_e)).astype(np.float64), (np.abs(e) + L_e).astype(np.float64),
                              (e * e + 2 * np.abs(e) * L_e).astype(np.float64), wmag.astype(np.float64)])
        uf, starts = np.unique(f, return_index=True)
        val[uf, C_COST] += np.add.reduceat(ev[:, 0], starts)
        mag[uf, C_COST] += np.add.reduceat(em[:, 0], starts)
        for col, j in ((C_CHI, 1), (C_SE, 2), (C_SE2, 3), (C_SW, 4)):
            val[uf, col] += np.add.reduceat(ev[:, j], starts)
            mag[uf, col] += np.add.reduceat(em[:, j], starts)
        val[uf, C_H:C_H + 27] += np.add.reduceat(v[:, :27], starts, axis=0)
        mag[uf, C_H:C_H + 27] += np.add.reduceat(mg[:, :27], starts, axis=0)
        ae = np.abs(e)
        cm = np.fmax.reduceat(ae, starts)  # the largest finite |e| of the piece
        nan = np.add.reduceat(np.isnan(ae).astype(np.int64), starts) > 0
        cm = np.where(nan, LD(np.nan), cm)
        mx[uf] = np.where(np.isnan(mx[uf]) | np.isnan(cm), LD(np.nan), np.maximum(mx[uf], cm))
        mag[uf, C_MAX] = np.maximum(mag[uf, C_MAX], np.fmax.reduceat((ae + L_e).astype(np.float64), starts))
    live = counts > 0
    val[live, C_MAX] = mx[live]
    if edge_points is not None:
        fl = np.nonzero(live)[0]
        ep = np.asarray(edge_points, dtype=np.float64).reshape(-1, 2, 3)[fl].astype(LD)
        epl = X.edge_planes(np.asarray(frame_pose).reshape(-1, 7)[fl])
        for k in range(2):
            v, mg, e, L_e, _, _ = _terms(epl[:, k], ep[:, k], s2f[fl], R, t, use_loss, a2)
            val[fl, C_COST] += v[:, 27]
            mag[fl, C_COST] += mg[:, 27]
            val[fl, C_H:C_H + 27] += v[:, :27]
            mag[fl, C_H:C_H + 27] += mg[:, :27]
            val[fl, C_EDGE + k] = e
            mag[fl, C_EDGE + k] = (np.abs(e) + L_e).astype(np.float64)
    return val, mag


def ratios(got, val, mag):
    """|got - val| / mag per frame and column (the difference in long double); 0 where both are equal, inf where mag = 0 and
    they differ.  NaN in both counts as equal."""
    g = np.asarray(got, dtype=np.float64).astype(LD)
    err = np.abs(g - val).astype(np.float64)
    both_nan = np.isnan(g) & np.isnan(val)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(mag > 0, err / np.where(mag > 0, mag, 1.0), np.where(err > 0, np.inf, 0.0))
    r[both_nan] = 0.0
    return np.where(np.isnan(r), np.inf, r)


def assert_within(got, val, mag, gamma=X.GAMMA, what=""):
    r = ratios(got, val, mag)
    bad = np.argwhere(r > gamma)
    assert bad.size == 0, (f"{what}: {len(bad)} (frame, field) pairs exceed gamma * A, first "
                           f"{[(int(f), COLUMNS[c], float(r[f, c])) for f, c in bad[:5]]}")
    return {name: float(np.max(r[:, idx])) if len(r) else 0.0 for name, idx in GROUPS.items()}
