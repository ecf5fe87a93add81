#!/usr/bin/env python3
"""Measures the robust losses (Problem.set_loss): none, Cauchy, Huber and soft-L1, alternated in one process on the same problems.

* sweep: device time of one clc_bench_eval launch (CUDA events, L2 flushed before each launch) and its share of the H100 SXM data
  sheet's 3.35 TB/s over streamed_bytes, at 10^4 x 10^3 and 10^5 x 2*10^3 points, for the general and the planar kernel family,
  at the closed-form pose (near the optimum: most points are Huber inliers) and at the identity (most are outliers).
* solve: a full LM solve from the identity at 10^4 x 10^3 (device time, iterations).
* k2: CamLaserCalibration-sized solves (50 x 180) on the one-cluster kernel (device time, iterations).
* loop: a single-block problem (40 x 250) solved by the sweep kernel's looping instantiation (CLC_SMALL_KERNEL=0), the whole
  LM loop in one launch: device time per LM sweep of every kind.
The card's name and power limit are read in the same run.  Prints one JSON line per row.

    python bench_loss.py [--reps 5] [--n 10] [--big 100000x2000] [--out bench_loss.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess

import numpy as np

IDENT = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
KINDS = ("none", "cauchy", "huber", "soft_l1")
HBM_TBS = 3.35  # H100 SXM data sheet


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as exc:  # the numbers below still stand, without the card's description
        return f"unknown ({exc})", "unknown"


def sweep(n_frames, beams, reps, n, name, power):
    from camlasercalibratool_b200 import Problem, T_to_pose7

    out = []
    with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as p:
        near = T_to_pose7(np.linalg.inv(p.closed_form()[0]))
        for family in ("general", "planar"):
            p.set_planar_mode(1 if family == "planar" else 0)
            assert p.planar == (family == "planar")
            nbytes = p.streamed_bytes()
            for pose_name, pose in (("near", near), ("identity", IDENT)):
                ms = {k: [] for k in KINDS}
                for k in KINDS:  # warm-up of every instantiation
                    p.set_loss(k)
                    p.bench_eval(pose, 3)
                for _ in range(reps):  # alternated
                    for k in KINDS:
                        p.set_loss(k)
                        ms[k].extend(p.bench_eval(pose, n))
                for k in KINDS:
                    t = float(np.median(ms[k]))
                    out.append(dict(bench="sweep", kind=k, n_frames=n_frames, beams=beams, family=family, pose=pose_name,
                                    eval_ms=t, eval_ms_min=float(np.min(ms[k])), streamed_bytes=nbytes,
                                    hbm_share=nbytes / (t * 1e-3) / (HBM_TBS * 1e12),
                                    vs_cauchy=t / float(np.median(ms["cauchy"])), samples=len(ms[k]), card=name, power_limit=power))
    return out


def solves(n_frames, beams, reps, what, name, power, env=None):
    from camlasercalibratool_b200 import Problem

    out = []
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})  # knobs are read when the problem is created
    try:
        p = Problem.synthetic(n_frames, beams, seed=1, sigma=0.01)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    with p:
        runs = {k: [] for k in KINDS}
        for k in KINDS:
            p.set_loss(k)
            p.solve(IDENT)  # warm-up
        for _ in range(reps):
            for k in KINDS:
                p.set_loss(k)
                x, s, _ = p.solve(IDENT)
                runs[k].append((s.device_ms, s.num_iterations, s.termination, s.num_sweeps))
        path = p.dispatch()["solve"]
        for k in KINDS:
            ms = [r[0] for r in runs[k]]
            out.append(dict(bench=what, kind=k, n_frames=n_frames, beams=beams, path=path, device_ms=float(np.median(ms)),
                            device_ms_min=float(np.min(ms)), iterations=runs[k][0][1], sweeps=runs[k][0][3],
                            termination=runs[k][0][2], ms_per_sweep=float(np.median(ms)) / runs[k][0][3], samples=len(ms),
                            card=name, power_limit=power))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n", type=int, default=10)
    ap.add_argument("--big", default="100000x2000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    rows = []

    def emit(rs):
        for r in rs:
            print(json.dumps(r), flush=True)
            rows.append(r)

    emit(sweep(10_000, 1_000, a.reps, a.n, name, power))
    if a.big:
        nf, nb = (int(v) for v in a.big.split("x"))
        emit(sweep(nf, nb, a.reps, a.n, name, power))
    emit(solves(10_000, 1_000, a.reps, "solve", name, power))
    emit(solves(50, 180, 4 * a.reps, "k2", name, power))
    emit(solves(40, 250, 4 * a.reps, "loop", name, power, env={"CLC_SMALL_KERNEL": "0"}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
