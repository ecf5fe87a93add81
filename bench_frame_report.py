#!/usr/bin/env python3
"""Measures the per-frame report (clc_frame_report) against one evaluation (clc_eval) of the same problem.

For configs[1] (10^4 frames x 10^3 beams) and config 3 (10^5 x 2*10^3), on the general and the planar kernel family: the device
time of one report (the per-frame sweep + the split-frame fix-up, CUDA events, L2 flushed before each launch) next to the device
time of one clc_eval sweep, alternated in one process; the bytes the report has to move (24 B general / 16 B planar per point,
40 B per frame of planes and offsets, and the 288-byte report row it writes per frame) over its time, as a fraction of the H100
SXM data sheet's 3.35 TB/s; and, separately, the host wall time of the whole Problem.frame_report call including the copy of the
rows to the host.  The card's name and power limit are read in the same run.  Prints one JSON line per (config, family).

    python bench_frame_report.py [--reps 5] [--n 10] [--out bench_frame_report.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import time

import numpy as np

CONFIGS = {"configs[1]": (10_000, 1_000), "config3": (100_000, 2_000)}
HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
ROW_BYTES = 288     # sizeof(clc_frame_row)


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as exc:  # the numbers below still stand, without the card's description
        return f"unknown ({exc})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="alternating rounds of (eval, report) measurements")
    ap.add_argument("--n", type=int, default=10, help="timed launches per round")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from camlasercalibratool_b200 import Problem, T_to_pose7

    name, power = card()
    results = []
    for cfg in a.configs.split(","):
        n_frames, beams = CONFIGS[cfg]
        with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as p:
            T_lc = p.closed_form()[0]
            pose = T_to_pose7(np.linalg.inv(T_lc))  # the closed form's T_cl: where a solve starts
            for family in ("general", "planar"):
                p.set_planar_mode(1 if family == "planar" else 0)
                assert p.planar == (family == "planar")
                p.bench_eval(pose, 3)
                p.bench_frame_report(pose, 3)
                ev, fr = [], []
                for _ in range(a.reps):
                    ev.extend(p.bench_eval(pose, a.n))
                    fr.extend(p.bench_frame_report(pose, a.n))
                rows = p.frame_report(pose)
                t0 = time.perf_counter()
                rows = p.frame_report(pose)
                wall_ms = (time.perf_counter() - t0) * 1e3
                assert len(rows) == n_frames
                P = n_frames * beams
                nbytes = (16 if family == "planar" else 24) * P + 40 * n_frames + ROW_BYTES * n_frames
                report_ms, eval_ms = float(np.median(fr)), float(np.median(ev))
                r = dict(config=cfg, n_frames=n_frames, beams=beams, family=family, report_ms=report_ms,
                         report_ms_min=float(np.min(fr)), eval_ms=eval_ms, eval_ms_min=float(np.min(ev)),
                         report_over_eval=report_ms / eval_ms, bytes=nbytes, report_TBps=nbytes / report_ms / 1e9,
                         fraction_of_3_35_TBps=nbytes / (report_ms * 1e-3) / HBM_PEAK, call_wall_ms=wall_ms,
                         rows_bytes=ROW_BYTES * n_frames, card=name, power_limit=power, samples=len(fr))
                print(json.dumps(r), flush=True)
                results.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
