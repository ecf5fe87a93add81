#!/usr/bin/env python3
"""Measures one calibration at many poses (clc_eval_poses, clc_solve_lm_starts): a multi-start from K start poses.

* sweeps (sweep kernel): 10^5 frames x 2*10^3 beams and 10^4 x 10^3, general and planar kernel families.  The device time of one
  evaluation of K poses (bench_poses: frame constants, multi-pose sweeps, fix-up, reduction; CUDA events, L2 flushed before each
  launch) for K in {1, 2, 4, 8, 16, 32}, divided by one cold clc_eval sweep (bench_eval), the two alternated in one process.
* reference size (one-cluster kernel): 50 x 180, sigma 0.01, solve_starts from K in {1, 16, 64} random starts (rotations up to
  pi, translations up to 0.5 m, fixed seed): the device time of the call, the largest iteration count, how many starts reach the
  lowest cost, and the sum of the K sequential solve device times from the same starts.
* large problem (sweep kernel): 10^4 x 10^3, the same comparison for K = 16.
The card's name and power limit are read in the same run.  Prints one JSON line per measurement.

    python bench_starts.py [--reps 5] [--n 10] [--out bench_starts.json]
"""
from __future__ import annotations

import argparse
import json

import numpy as np

from bench_segments import card

IDENT = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])


def random_starts(K, seed=1, rot=np.pi, trans=0.5):
    rng = np.random.default_rng(seed)
    xs = []
    for _ in range(K):
        axis = rng.standard_normal(3)
        axis /= np.linalg.norm(axis)
        ang = rng.uniform(0, rot)
        xs.append(np.concatenate([rng.uniform(-trans, trans, 3), np.sin(ang / 2) * axis, [np.cos(ang / 2)]]))
    return np.array(xs)


def sweeps(frames, beams, family, name, power, reps, n, Ks=(1, 2, 4, 8, 16, 32)):
    from camlasercalibratool_b200 import Problem

    rows = []
    with Problem.synthetic(frames, beams, seed=1, sigma=0.01) as p:
        p.set_planar_mode(1 if family == "planar" else 0)
        x = random_starts(max(Ks), seed=2, rot=0.3, trans=0.1)
        for K in Ks:
            p.bench_poses(x[:K], 2)
        p.bench_eval(IDENT, 2)
        ev, po = [], {K: [] for K in Ks}
        for _ in range(reps):  # alternated
            ev.append(float(np.median(p.bench_eval(IDENT, n))))
            for K in Ks:
                po[K].append(float(np.median(p.bench_poses(x[:K], n))))
        e = float(np.median(ev))
        for K in Ks:
            t = float(np.median(po[K]))
            rows.append(dict(bench="starts_sweep", frames=frames, beams=beams, family=family, K=K, eval_ms=e, poses_ms=t,
                             evals_per_iteration=t / e, evals_per_pose=t / e / K, card=name, power_limit=power))
    return rows


def solves(frames, beams, K, name, power, reps):
    from camlasercalibratool_b200 import Problem

    x = random_starts(K, seed=3)
    with Problem.synthetic(frames, beams, seed=1, sigma=0.01) as p:
        path = p.dispatch()["solve"]
        p.solve_starts(x)  # warm-up
        p.solve(x[0])
        call, seq = [], []
        for _ in range(reps):  # alternated
            xs, summ, _, best = p.solve_starts(x)
            call.append(summ[0].device_ms)
            seq.append(sum(p.solve(x[k])[1].device_ms for k in range(K)))
        costs = np.array([s.final_cost for s in summ])
        own = [p.solve(x[k])[1].device_ms for k in range(K)]
        slowest = int(np.argmax([s.num_iterations for s in summ]))
    c, s = float(np.median(call)), float(np.median(seq))
    return [dict(bench="starts_solve", frames=frames, beams=beams, K=K, path=path, device_ms=c,
                 max_iterations=int(max(sm.num_iterations for sm in summ)),
                 starts_at_lowest_cost=int(np.sum(costs <= costs.min() * (1 + 1e-9))), best=int(best),
                 sequential_ms=s, speedup=s / c, slowest_start_own_ms=float(own[slowest]), card=name, power_limit=power)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    rows = []
    for frames, beams in ((100_000, 2_000), (10_000, 1_000)):
        for family in ("general", "planar"):
            rows += sweeps(frames, beams, family, name, power, a.reps, a.n)
    for K in (1, 16, 64):
        rows += solves(50, 180, K, name, power, a.reps)
    rows += solves(10_000, 1_000, 16, name, power, a.reps)
    for r in rows:
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
