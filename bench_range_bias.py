#!/usr/bin/env python3
"""Measures the range-bias calls (clc_*_range_bias, clc_problem_range_correct).

* iteration: configs[1] (10^4 frames x 10^3 beams, Problem.synthetic) and 10^5 x 2*10^3.  The device time of one range-bias
  iteration (clc_bench_range_bias: frame constants, kModeRange sweep, fix-up into 45 sums, two-level reduction; CUDA events, L2
  flushed before each launch) against one cold clc_eval sweep of the same problem, alternated in one process, for the general
  and planar kernel families.  The LM update (one warp) is not in this bracket.
* solve: the device time of a whole solve_range_bias against clc_solve_lm, both from the closed form, at the reference's size
  (50 x 180) and at 10^4 x 10^3.
* correct: the wall time of range_corrected (gather copy + in-place correction) as a fraction of 3.35 TB/s over the bytes the
  correction kernel alone moves (read and write of every coordinate stream).
The card's name and power limit are read in the same run.  Prints one JSON line per measurement.

    python bench_range_bias.py [--sizes 10000x1000,100000x2000] [--reps 5] [--n 10] [--out bench_range_bias.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import time

import numpy as np

BIAS = (0.025, 0.005)


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as exc:  # the numbers below still stand, without the card's description
        return f"unknown ({exc})", "unknown"


def iteration(n_frames, beams, reps, n, name, power):
    from camlasercalibratool_b200 import Problem, T_to_pose7

    out = []
    with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as p:
        pose = T_to_pose7(np.linalg.inv(p.closed_form()[0]))
        for family in ("general", "planar"):
            p.set_planar_mode(1 if family == "planar" else 0)
            assert p.planar == (family == "planar")
            p.bench_eval(pose, 3)
            p.bench_range_bias(pose, BIAS, 3)
            ev, rb = [], []
            for _ in range(reps):
                ev.extend(p.bench_eval(pose, n))
                rb.extend(p.bench_range_bias(pose, BIAS, n))
            e, t = float(np.median(ev)), float(np.median(rb))
            out.append(dict(bench="range_bias_iteration", n_frames=n_frames, beams=beams, family=family, iteration_ms=t,
                            iteration_ms_min=float(np.min(rb)), eval_ms=e, eval_ms_min=float(np.min(ev)), ratio=t / e,
                            card=name, power_limit=power, samples=len(rb)))
        p.set_planar_mode(0)
        c0 = time.perf_counter()
        q = p.range_corrected(BIAS)
        wall = time.perf_counter() - c0
        for _ in range(reps - 1):
            q.close()
            c0 = time.perf_counter()
            q = p.range_corrected(BIAS)
            wall = min(wall, time.perf_counter() - c0)
        q.close()
        nbytes = 2 * 3 * 8 * n_frames * beams
        out.append(dict(bench="range_correct", n_frames=n_frames, beams=beams, wall_ms=wall * 1e3,
                        kernel_bytes=nbytes, fraction_of_3_35TBps_if_wall_were_kernel=nbytes / wall / 3.35e12, card=name,
                        power_limit=power, samples=reps))
    return out


def solve(n_frames, beams, reps, name, power):
    from camlasercalibratool_b200 import Problem, T_to_pose7

    with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as p:
        x0 = T_to_pose7(np.linalg.inv(p.closed_form()[0]))
        p.solve(x0)
        p.solve_range_bias(x0)
        lm, rb, it_lm, it_rb = [], [], 0, 0
        for _ in range(reps):
            _, s, _ = p.solve(x0)
            lm.append(s.device_ms)
            it_lm = s.num_iterations
            _, _, s2, _ = p.solve_range_bias(x0)
            rb.append(s2.device_ms)
            it_rb = s2.num_iterations
    return dict(bench="range_bias_solve", n_frames=n_frames, beams=beams, solve_ms=float(np.median(lm)), solve_iterations=it_lm,
                range_bias_solve_ms=float(np.median(rb)), range_bias_iterations=it_rb, card=name, power_limit=power,
                samples=reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000x1000,100000x2000")
    ap.add_argument("--solve-sizes", default="50x180,10000x1000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    rows = []
    for size in a.sizes.split(","):
        nf, beams = (int(v) for v in size.split("x"))
        rows.extend(iteration(nf, beams, a.reps, a.n, name, power))
    for size in a.solve_sizes.split(","):
        nf, beams = (int(v) for v in size.split("x"))
        rows.append(solve(nf, beams, a.reps, name, power))
    for r in rows:
        print(json.dumps(r))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
