#!/usr/bin/env python3
"""Measures Problem.trim (clc_problem_trim): dropping the points far from their board from a device-resident problem without
re-uploading its points.

For configs[1] (10^4 frames x 10^3 beams) and config 3 (10^5 x 2*10^3) of Problem.synthetic (sigma = 0.01): a seeded 1 % of the
points is moved 0.3 - 1 m off its board inside the laser plane (a beam that runs past the board; z stays 0, so the source can
stay on the planar kernel family) and the edited points are uploaded with from_arrays.  With the source on the general and on the
planar family, two thresholds at the pose the clean problem solves to: tau = 0.2 m (drops exactly the moved points) and
tau = +inf (the mark pass plus a keep-all gather).  Per row:
* the device times of the mark and the gather pass (clc_bench_trim: CUDA events, L2 flushed before each pass, medians);
* the bytes each pass moves -- mark: the source's coordinate streams + the keep mask; gather: the mask + read and write of the
  kept points' streams + 40 B per frame -- and each pass's fraction of the H100 SXM data sheet's 3.35 TB/s;
* the ratio of mark + gather to one cold clc_eval of the source on the same family;
* the host wall time of the whole trim() call;
* at configs[1], the wall time of the host route: download(), the same filter in numpy, from_arrays.
The card's name and power limit are read in the same run.  Prints one JSON line per row.

--accuracy runs the seeded accuracy experiment instead: 500 frames x 180 beams, sigma = 0.01; in 10 % of the frames the first and
last 3 points are moved 0.3 - 1 m behind the board along their beam (ghost returns).  Solve, trim at the solved pose with
tau_f = 3 rms_e_f from the frame report, solve again; the rotation and translation errors against the generator's ground truth
before and after.

    python bench_trim.py [--n 20] [--configs configs[1],config3] [--accuracy] [--out bench_trim.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import time

import numpy as np

CONFIGS = {"configs[1]": (10_000, 1_000), "config3": (100_000, 2_000)}
HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
TAU = 0.2


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as exc:  # the numbers below still stand, without the card's description
        return f"unknown ({exc})", "unknown"


def laser_normals(planes, pose):
    """m = R^T n and c = n.t + d of every frame at pose (host arithmetic: the device's rounding can differ in the last bit)."""
    from oracle import oracle as O

    R = O.quat_to_rot(pose[3:])
    return planes[:, :3] @ R, planes[:, :3] @ pose[:3] + planes[:, 3]


def wall_ms(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def edited_source(Problem, n_frames, beams):
    """The synthetic problem with 1 % of its points moved 0.3 - 1 m off the board inside the laser plane, and the pose its clean
    version solves to."""
    with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as syn:
        x, _, _ = syn.solve(np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]))
        d = syn.download()
    rng = np.random.default_rng(2024)
    P = len(d["points"])
    idx = rng.choice(P, P // 100, replace=False)
    m, _ = laser_normals(d["planes"], x)
    fi = np.searchsorted(d["offsets"], idx, side="right") - 1
    mxy = m[fi, :2]
    shift = rng.uniform(0.3, 1.0, size=len(idx)) * rng.choice([-1.0, 1.0], size=len(idx))
    d["points"][idx, :2] += (shift / np.einsum("ij,ij->i", mxy, mxy))[:, None] * mxy  # e moves by `shift`, z stays 0
    return Problem.from_arrays(d["frame_pose"], d["offsets"], d["points"]), x, len(idx)


def host_route(src, Problem, pose, tau):
    """download -> numpy filter -> from_arrays."""
    def run():
        d = src.download()
        m, c = laser_normals(d["planes"], pose)
        f = np.repeat(np.arange(len(m)), np.diff(d["offsets"]))
        keep = np.abs(np.einsum("ij,ij->i", d["points"], m[f]) + c[f]) <= tau
        ck = np.concatenate([[0], np.cumsum(keep)])
        return Problem.from_arrays(d["frame_pose"], ck[d["offsets"]], d["points"][keep])
    run().close()
    t, p = wall_ms(run)
    p.close()
    return t


def measure(src, family, cfg, tau_name, tau, pose, n, card_info, Problem, want_host):
    N, P, _ = src.sizes()
    src.bench_trim(pose, tau, 2)
    mark, gather = src.bench_trim(pose, tau, n)
    src.trim(pose, tau).close()
    call_ms, t = wall_ms(lambda: src.trim(pose, tau))
    with t:
        K = t.sizes()[1]
    src.bench_eval(pose, 3)
    ev = float(np.median(src.bench_eval(pose, n)))
    stream = 16  # synthetic data is planar: z is known to be 0 and is neither read nor written
    mask = (P + 7) // 8
    mark_bytes = stream * P + mask
    gather_bytes = mask + 2 * stream * K + 40 * N
    m_ms, g_ms = float(np.median(mark)), float(np.median(gather))
    host_ms = host_route(src, Problem, pose, tau) if want_host else None
    return dict(config=cfg, family=family, tau=tau_name, points=P, kept_points=K, dropped_points=P - K, mark_ms=m_ms,
                gather_ms=g_ms, mark_bytes=mark_bytes, gather_bytes=gather_bytes,
                mark_fraction_of_3_35_TBps=mark_bytes / (m_ms * 1e-3) / HBM_PEAK,
                gather_fraction_of_3_35_TBps=gather_bytes / (g_ms * 1e-3) / HBM_PEAK, eval_ms=ev,
                mark_plus_gather_over_eval=(m_ms + g_ms) / ev, trim_call_wall_ms=call_ms, host_route_wall_ms=host_ms,
                card=card_info[0], power_limit=card_info[1], samples=len(mark))


def accuracy(card_info):
    from camlasercalibratool_b200 import Problem
    from oracle import oracle as O

    p = O.generate(500, 180, seed=7, sigma=0.01)
    gt = O.ground_truth()[1]
    rng = np.random.default_rng(99)
    pts = p.points.copy()
    ghost_frames = np.sort(rng.choice(500, 50, replace=False))
    for f in ghost_frames:
        a, b = p.offsets[f], p.offsets[f + 1]
        for j in list(range(a, a + 3)) + list(range(b - 3, b)):
            r = np.linalg.norm(pts[j])
            pts[j] *= (r + rng.uniform(0.3, 1.0)) / r  # farther along the beam: behind the board
    x0 = O.pose_plus(gt, 1e-2 * np.array([1.0, -0.7, 0.4, -1.0, 0.6, 0.3]))
    with Problem.from_arrays(p.frame_pose, p.offsets, pts) as src:
        x1, s1, _ = src.solve(x0)
        rows = src.frame_report(x1)
        tau = 3 * rows["rms_e"]
        with src.trim(x1, tau) as t:
            x2, s2, _ = t.solve(x1)
            dropped = src.sizes()[1] - t.sizes()[1]
    e1, e2 = O.pose_error(x1, gt), O.pose_error(x2, gt)
    return dict(experiment="ghost_returns", frames=500, beams=180, sigma=0.01, ghost_frames=len(ghost_frames),
                ghost_points=6 * len(ghost_frames), dropped_points=int(dropped), rot_err_before_rad=e1[0],
                trans_err_before_m=e1[1], rot_err_after_rad=e2[0], trans_err_after_m=e2[1],
                iterations=(s1.num_iterations, s2.num_iterations), card=card_info[0], power_limit=card_info[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20, help="timed launches per row")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--accuracy", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from camlasercalibratool_b200 import Problem

    info = card()
    results = []

    def emit(r):
        print(json.dumps(r), flush=True)
        results.append(r)

    if a.accuracy:
        emit(accuracy(info))
    else:
        for cfg in a.configs.split(","):
            n_frames, beams = CONFIGS[cfg]
            src, pose, moved = edited_source(Problem, n_frames, beams)
            with src:
                for family in ("general", "planar"):
                    src.set_planar_mode(1 if family == "planar" else 0)
                    for tau_name, tau in (("0.2", TAU), ("inf", np.inf)):
                        r = measure(src, family, cfg, tau_name, tau, pose, a.n, info, Problem, cfg == "configs[1]")
                        r["moved_points"] = moved
                        emit(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
