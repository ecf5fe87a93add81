"""Per-frame restatement of clc_frame_report in numpy, written apart from tests/frame_oracle.c (vectorised over points, per-frame
sums by bincount), so that a transcription error in one of the two shows up as a disagreement.  Same model as the oracle twin
(oracle/oracle_np.py): PointInPlaneFactor (reference src/LaseCamCalCeres.cpp:43-66), the Ceres Cauchy corrector (:249), the
analysis tail's chi (:318-381).  Rows: [N, 36] in clc_frame_row's order, n_points as a float.  Test infrastructure only.
"""
from __future__ import annotations

import numpy as np

from oracle import oracle_np as ON

ROW = 36
N_POINTS, COST, CHI, MEAN_E, RMS_E, MAX_E, MEAN_W, EDGE_E, H21, G6 = 0, 1, 2, 3, 4, 5, 6, 7, 9, 30
IU6 = np.triu_indices(6)


def _terms(planes, pts, s, pose7, use_loss, cauchy_a):
    """Per residual: raw distance e, r = s e, rho', cost, and the corrected J^T J (upper triangle) and J^T r."""
    R = ON.quat_to_rot(pose7[3:7])
    n = planes[:, :3]
    e = np.einsum("ij,ij->i", n, pts @ R.T + pose7[:3]) + planes[:, 3]
    r = s * e
    J = np.concatenate([s[:, None] * n, s[:, None] * np.cross(pts, n @ R)], axis=1)
    if use_loss:
        b = (cauchy_a * s) ** 2
        q = 1.0 + r * r / b
        inv = 1.0 / q
        w = np.where(inv > np.finfo(float).tiny, inv, np.finfo(float).tiny)  # the corrector's clamp (a NaN becomes DBL_MIN)
        cost = 0.5 * b * np.log(q)
    else:
        w = np.ones_like(r)
        cost = 0.5 * r * r
    sq = np.sqrt(w)
    Jc, rc = J * sq[:, None], r * sq
    return e, r, w, cost, Jc[:, IU6[0]] * Jc[:, IU6[1]], Jc * rc[:, None]


def frame_report(frame_pose, offsets, points, pose7, use_loss=True, cauchy_a=0.05, edge_points=None):
    frame_pose = np.asarray(frame_pose, dtype=np.float64).reshape(-1, 7)
    offsets = np.asarray(offsets, dtype=np.int64)
    points = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    pose7 = np.asarray(pose7, dtype=np.float64)
    N = frame_pose.shape[0]
    counts = np.diff(offsets)
    rows = np.zeros((N, ROW))
    live = counts > 0
    if not np.any(live):
        return rows
    planes = np.zeros((N, 4))
    planes[live] = [ON.frame_plane(frame_pose[f]) for f in np.nonzero(live)[0]]
    f_of = np.repeat(np.arange(N), counts)
    s_f = np.zeros(N)
    s_f[live] = 1.0 / np.sqrt(counts[live].astype(np.float64))
    e, r, w, cost, HH, gg = _terms(planes[f_of], points, s_f[f_of], pose7, use_loss, cauchy_a)

    def per_frame(v):
        return np.bincount(f_of, weights=v, minlength=N)

    rows[:, N_POINTS] = counts
    rows[:, COST] = per_frame(cost)
    rows[:, CHI] = per_frame(r * r)
    rows[live, MEAN_E] = per_frame(e)[live] / counts[live]
    rows[live, RMS_E] = np.sqrt(per_frame(e * e)[live] / counts[live])
    rows[live, MAX_E] = np.maximum.reduceat(np.abs(e), offsets[:-1][live])  # np.maximum keeps a NaN
    rows[live, MEAN_W] = per_frame(w)[live] / counts[live]
    for k in range(21):
        rows[:, H21 + k] = per_frame(HH[:, k])
    for k in range(6):
        rows[:, G6 + k] = per_frame(gg[:, k])
    if edge_points is not None:
        ep = np.asarray(edge_points, dtype=np.float64).reshape(-1, 2, 3)
        fl = np.nonzero(live)[0]
        for k in range(2):
            epl = np.array([ON.edge_planes(frame_pose[f])[k] for f in fl]).reshape(-1, 4)
            ek, _, _, ck, Hk, gk = _terms(epl, ep[fl, k], s_f[fl], pose7, use_loss, cauchy_a)
            rows[fl, EDGE_E + k] = ek
            rows[fl, COST] += ck
            rows[fl, H21:H21 + 21] += Hk
            rows[fl, G6:G6 + 6] += gk
    return rows
