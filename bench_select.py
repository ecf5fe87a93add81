#!/usr/bin/env python3
"""Measures the greedy D-optimal frame selection (clc_select_frames) on the device against the float64 numpy reference on the host.

Cases: configs[1] (10^4 frames x 10^3 beams) at budgets 100 and 1 000, and 10^5 x 2*10^3 at budget 1 000, on the kernel family
the problem picks.  Per case, in one process: the device time of one report sweep (clc_bench_frame_report) next to one cold
clc_eval (both with the L2 flushed, CUDA events); the device time of the whole selection on the report's device rows
(clc_bench_select: sum, init and scale kernels and every step launch, the host polls between step batches included) and per step;
and the host time of the float64 reference (tests/select_reference.py) on the same rows, per step, over the first --ref-steps
steps (its per-step cost does not fall with the step).  The card's name and power limit are read in the same run.  Prints one
JSON line per case.

    python bench_select.py [--reps 5] [--ref-steps 5] [--out bench_select.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

CASES = [("configs[1]", 10_000, 1_000, 100), ("configs[1]", 10_000, 1_000, 1_000), ("config3", 100_000, 2_000, 1_000)]


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as exc:  # the numbers below still stand, without the card's description
        return f"unknown ({exc})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed selections per case")
    ap.add_argument("--ref-steps", type=int, default=5, help="steps of the host reference that are timed")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
    import select_reference as SR

    from camlasercalibratool_b200 import Problem, T_to_pose7

    name, power = card()
    results = []
    for cfg, n_frames, beams, budget in CASES:
        with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as p:
            T_lc = p.closed_form()[0]
            pose = T_to_pose7(np.linalg.inv(T_lc))  # the closed form's T_cl
            p.bench_eval(pose, 3)
            p.bench_frame_report(pose, 3)
            ev, fr = [], []
            for _ in range(a.reps):
                ev.extend(p.bench_eval(pose, 5))
                fr.extend(p.bench_frame_report(pose, 5))
            p.bench_select(pose, budget, 1)  # warm-up
            sel_ms, n_sel = p.bench_select(pose, budget, a.reps)
            sel = p.select_frames(pose, budget)
            assert len(sel.order) == n_sel
            H21 = p.frame_report(pose)["H21"]
            planar = p.planar
        P = SR.prepare(H21)
        A = P["A0"].copy()
        idx = np.nonzero(P["cand"])[0]
        t0 = time.perf_counter()
        for s in range(a.ref_steps):
            g = SR.gains(A, P["Ht"][idx], np.float64)
            k = int(np.argmax(g))
            A = A + P["Ht"][idx[k]]
            idx = np.delete(idx, k)
        ref_step_ms = (time.perf_counter() - t0) * 1e3 / a.ref_steps
        select_ms = float(np.median(sel_ms))
        step_ms = select_ms / max(n_sel, 1)
        r = dict(config=cfg, n_frames=n_frames, beams=beams, budget=budget, n_selected=int(n_sel), planar=planar,
                 eval_ms=float(np.median(ev)), report_ms=float(np.median(fr)), report_over_eval=float(np.median(fr) / np.median(ev)),
                 select_ms=select_ms, select_ms_min=float(np.min(sel_ms)), step_us=step_ms * 1e3,
                 ref_step_ms=ref_step_ms, ref_select_ms_est=ref_step_ms * n_sel, speedup_per_step=ref_step_ms / step_ms,
                 card=name, power_limit=power, samples=len(sel_ms))
        print(json.dumps(r), flush=True)
        results.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
