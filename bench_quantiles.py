#!/usr/bin/env python3
"""Measures the exact quantiles of the point-to-board distances (Problem.residual_quantiles / frame_quantiles).

For configs[1] (10^4 frames x 10^3 beams, 10^7 points) and config 3 (10^5 x 2*10^3, 2*10^8 points) of Problem.synthetic
(sigma = 0.01, noisy data), on the general and on the planar kernel family, at the pose the problem solves to.  Per row, medians
over --n rounds; within a round the calls alternate, each after an L2 flush (clc_bench_eval / clc_bench_quantiles, CUDA events):
* one eval (the sweep kernel), the yardstick of the ratios;
* one problem-wide call with R = 1 (the median) and with R = 16, from its first pass to the end of its last (the host steps between
  the passes included), and the passes over the point streams it made;
* one per-frame kernel with R = 3 (quartiles);
* the host wall time of what a user would do without them: point_residuals of every point to the host, then np.partition for the
  median.
The card's name and power limit are read in the same run.  Prints one JSON line per row.

    python bench_quantiles.py [--n 10] [--configs configs[1],config3] [--out bench_quantiles.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import time

import numpy as np

CONFIGS = {"configs[1]": (10_000, 1_000), "config3": (100_000, 2_000)}
Q16 = np.linspace(0.0, 1.0, 16)
Q3 = np.array([0.25, 0.5, 0.75])


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as exc:  # the numbers below still stand, without the card's description
        return f"unknown ({exc})", "unknown"


def host_route(p, x):
    t0 = time.perf_counter()
    a = np.abs(p.point_residuals(x))
    a = a[~np.isnan(a)]
    k = max(int(np.ceil(0.5 * a.size)) - 1, 0)
    v = np.partition(a, k)[k]
    return (time.perf_counter() - t0) * 1e3, v


def run(config, family, n):
    from camlasercalibratool_b200 import Problem

    n_frames, beams = CONFIGS[config]
    with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as p:
        if family == "general":
            p.set_planar_mode(0)
        assert p.planar == (family == "planar")
        x, _, _ = p.solve(np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]))
        for q in (0.5, Q16, Q3):  # warm-up of every shape
            p.bench_quantiles(x, q, 1)
        p.bench_eval(x, 2)
        ev, w1, w16, fr3, passes1, passes16 = [], [], [], [], 0, 0
        for _ in range(n):
            ev.append(p.bench_eval(x, 1)[0])
            ms, _, passes1 = p.bench_quantiles(x, 0.5, 1)
            w1.append(ms[0])
            ms, _, passes16 = p.bench_quantiles(x, Q16, 1)
            w16.append(ms[0])
            _, fms, _ = p.bench_quantiles(x, Q3, 1)
            fr3.append(fms[0])
        med, _ = p.residual_quantiles(x, 0.5)
        host_ms, host_med = host_route(p, x)
        assert host_med == med[0], (host_med, med[0])
        name, power = card()
        e = float(np.median(ev))
        return {"config": config, "family": family, "points": n_frames * beams, "frames": n_frames,
                "eval_ms": e, "wide_r1_ms": float(np.median(w1)), "wide_r1_passes": passes1,
                "wide_r16_ms": float(np.median(w16)), "wide_r16_passes": passes16, "frame_r3_ms": float(np.median(fr3)),
                "wide_r1_over_eval": float(np.median(w1)) / e, "wide_r16_over_eval": float(np.median(w16)) / e,
                "frame_r3_over_eval": float(np.median(fr3)) / e, "host_route_ms": host_ms, "rounds": n,
                "card": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rows = []
    for config in args.configs.split(","):
        for family in ("general", "planar"):
            row = run(config, family, args.n)
            print(json.dumps(row), flush=True)
            rows.append(row)
    if args.out:
        with open(args.out, "w") as f:
            for row in rows:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
