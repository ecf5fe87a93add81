#!/usr/bin/env python3
"""Measures the segmented solves (clc_*_segments): many independent extrinsics from one device-resident problem.

* fleet: Problem.synthetic with W rigs x 50 frames x 180 beams (sigma 0.01), W = 10^3 and 10^4, every segment from the identity.
  The device time of one solve_segments call (its summaries' device_ms), the largest iteration count over the segments, the time
  per shared iteration (device time / the largest sweep count), and the sequential alternative: a sample of 50 rigs solved as
  problems of their own (the one-cluster kernel, device time of each clc_solve_lm), extrapolated to W.
  The rig with the most iterations is also solved on its own, to show what sets the segmented solve's length.
* windows: configs[1] (10^4 frames x 10^3 beams) cut into 100 windows of 100 frames, general and planar kernel families: the
  device time of one segmented iteration (frame constants + segment sweep + fix-up + two-level reduction; CUDA events, L2 flushed
  before each launch) against one cold clc_eval sweep of the same problem, alternated in one process.  The LM update step (one
  warp per segment) is not in this bracket; the fleet's time per iteration includes it.
The card's name and power limit are read in the same run.  Prints one JSON line per measurement.

    python bench_segments.py [--fleet 1000,10000] [--reps 5] [--n 10] [--out bench_segments.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess

import numpy as np

IDENT = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as exc:  # the numbers below still stand, without the card's description
        return f"unknown ({exc})", "unknown"


def fleet(W, name, power, sample=50):
    from camlasercalibratool_b200 import Problem

    frames, beams = 50, 180
    with Problem.synthetic(W * frames, beams, seed=1, sigma=0.01) as p:
        off = np.arange(0, W * frames + 1, frames)
        x0 = np.tile(IDENT, (W, 1))
        p.solve_segments(off, x0)  # warm-up
        ms = []
        for _ in range(3):
            x, summ, _ = p.solve_segments(off, x0)
            ms.append(summ[0].device_ms)
        its = np.array([s.num_iterations for s in summ])
        iters = int(its.max())
        sweeps = max(s.num_sweeps for s in summ)
        slowest = int(np.argmax(its))
        d = p.download()
    # the sequential alternative: the first `sample` rigs as problems of their own
    seq = []
    for r in range(sample):
        a, b = d["offsets"][r * frames], d["offsets"][(r + 1) * frames]
        with Problem.from_arrays(d["frame_pose"][r * frames:(r + 1) * frames], d["offsets"][r * frames:(r + 1) * frames + 1] - a,
                                 d["points"][a:b]) as q:
            q.solve(IDENT)
            seq.append(q.solve(IDENT)[1].device_ms)
    # the rig that set the segmented solve's length, solved as a problem of its own
    a, b = d["offsets"][slowest * frames], d["offsets"][(slowest + 1) * frames]
    with Problem.from_arrays(d["frame_pose"][slowest * frames:(slowest + 1) * frames],
                             d["offsets"][slowest * frames:(slowest + 1) * frames + 1] - a, d["points"][a:b]) as q:
        _, s_alone, _ = q.solve(IDENT)
    total = float(np.median(ms))
    seq_total = float(np.mean(seq)) * W
    return dict(bench="fleet", rigs=W, frames_per_rig=frames, beams=beams, device_ms=total, device_ms_runs=ms,
                max_iterations=iters, max_sweeps=sweeps, median_iterations=float(np.median(its)),
                iterations_histogram={int(k): int(v) for k, v in zip(*np.unique(its, return_counts=True))},
                slowest_rig=slowest, slowest_rig_alone_iterations=s_alone.num_iterations,
                slowest_rig_alone_termination=s_alone.termination, ms_per_iteration=total / sweeps,
                sequential_rig_ms_median=float(np.median(seq)), sequential_rig_ms_mean=float(np.mean(seq)), sequential_sample=sample,
                sequential_extrapolated_ms=seq_total, speedup=seq_total / total, card=name, power_limit=power)


def windows(reps, n, name, power):
    from camlasercalibratool_b200 import Problem, T_to_pose7

    out = []
    n_frames, beams = 10_000, 1_000
    with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as p:
        pose = T_to_pose7(np.linalg.inv(p.closed_form()[0]))
        off = np.arange(0, n_frames + 1, 100)
        poses = np.tile(pose, (len(off) - 1, 1))
        for family in ("general", "planar"):
            p.set_planar_mode(1 if family == "planar" else 0)
            assert p.planar == (family == "planar")
            p.bench_eval(pose, 3)
            p.bench_segments(off, poses, 3)
            ev, sg = [], []
            for _ in range(reps):
                ev.extend(p.bench_eval(pose, n))
                sg.extend(p.bench_segments(off, poses, n))
            e, s = float(np.median(ev)), float(np.median(sg))
            out.append(dict(bench="windows", n_frames=n_frames, beams=beams, windows=len(off) - 1, family=family, iteration_ms=s,
                            iteration_ms_min=float(np.min(sg)), eval_ms=e, eval_ms_min=float(np.min(ev)), ratio=s / e,
                            card=name, power_limit=power, samples=len(sg)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fleet", default="1000,10000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    results = []
    for r in windows(a.reps, a.n, name, power):
        print(json.dumps(r), flush=True)
        results.append(r)
    for W in [int(w) for w in a.fleet.split(",") if w]:
        r = fleet(W, name, power)
        print(json.dumps(r), flush=True)
        results.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
