#!/usr/bin/env python3
"""Measures the time-offset calls (clc_*_time_offset).

* iteration: configs[1] (10^4 frames x 10^3 beams, Problem.synthetic) and 10^5 x 2*10^3, with a trajectory whose knots are the
  frames' board poses at 30 Hz and scan times jittered inside the intervals.  The device time of one time-offset iteration
  (clc_bench_time_offset: planes and constants, segment sweep, fix-up into 36 sums, two-level reduction; CUDA events, L2 flushed
  before each launch) against one cold clc_eval sweep of the same problem, alternated in one process, for the general and planar
  kernel families.  The LM update (one warp) is not in this bracket.
* reference: the reference's size (50 frames x 180 beams): the device time of a whole solve_time_offset against clc_solve_lm on
  the one-cluster kernel, both from the closed form.
The card's name and power limit are read in the same run.  Prints one JSON line per measurement.

    python bench_time_offset.py [--sizes 10000x1000,100000x2000] [--reps 5] [--n 10] [--out bench_time_offset.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess

import numpy as np


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as exc:  # the numbers below still stand, without the card's description
        return f"unknown ({exc})", "unknown"


def attach(p, n_frames, seed=1):
    """Knots: the frames' board poses at 30 Hz; scan times jittered inside the intervals."""
    fp = np.empty((n_frames, 7))
    from camlasercalibratool_b200 import _lib

    _lib.check(p._L.clc_problem_download(p._h, fp.ctypes.data_as(_lib.c_double_p), None, None, None, None), "download")
    kt = 1.7e9 + np.arange(n_frames) / 30.0
    s = kt + np.random.default_rng(seed).uniform(0.0, 1.0 / 30.0, n_frames)
    s[-1] = kt[-1]
    p.set_trajectory(kt, fp, s)


def iteration(n_frames, beams, reps, n, name, power):
    from camlasercalibratool_b200 import Problem, T_to_pose7

    out = []
    with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as p:
        pose = T_to_pose7(np.linalg.inv(p.closed_form()[0]))
        attach(p, n_frames)
        for family in ("general", "planar"):
            p.set_planar_mode(1 if family == "planar" else 0)
            assert p.planar == (family == "planar")
            p.bench_eval(pose, 3)
            p.bench_time_offset(pose, 0.0, 3)
            ev, to = [], []
            for _ in range(reps):
                ev.extend(p.bench_eval(pose, n))
                to.extend(p.bench_time_offset(pose, 0.0, n))
            e, t = float(np.median(ev)), float(np.median(to))
            out.append(dict(bench="time_offset_iteration", n_frames=n_frames, beams=beams, family=family, iteration_ms=t,
                            iteration_ms_min=float(np.min(to)), eval_ms=e, eval_ms_min=float(np.min(ev)), ratio=t / e,
                            card=name, power_limit=power, samples=len(to)))
    return out


def reference(reps, name, power):
    from camlasercalibratool_b200 import Problem, T_to_pose7

    with Problem.synthetic(50, 180, seed=1, sigma=0.01) as p:
        attach(p, 50)
        x0 = T_to_pose7(np.linalg.inv(p.closed_form()[0]))
        assert p.dispatch()["solve"] == "one_cluster"
        p.solve(x0)
        p.solve_time_offset(x0, 0.0)
        lm, to, it_lm, it_to = [], [], 0, 0
        for _ in range(reps):
            _, s, _ = p.solve(x0)
            lm.append(s.device_ms)
            it_lm = s.num_iterations
            _, _, s2, _ = p.solve_time_offset(x0, 0.0)
            to.append(s2.device_ms)
            it_to = s2.num_iterations
    return dict(bench="time_offset_reference_size", n_frames=50, beams=180, solve_ms=float(np.median(lm)), solve_iterations=it_lm,
                time_offset_solve_ms=float(np.median(to)), time_offset_iterations=it_to, card=name, power_limit=power,
                samples=reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000x1000,100000x2000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    rows = []
    for size in a.sizes.split(","):
        nf, beams = (int(v) for v in size.split("x"))
        rows.extend(iteration(nf, beams, a.reps, a.n, name, power))
    rows.append(reference(a.reps, name, power))
    for r in rows:
        print(json.dumps(r))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
