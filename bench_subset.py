#!/usr/bin/env python3
"""Measures Problem.subset (clc_problem_subset): dropping frames from a device-resident problem without re-uploading its points.

For configs[1] (10^4 frames x 10^3 beams) and config 3 (10^5 x 2*10^3) of Problem.synthetic (sigma = 0.01), with the source on the
general and on the planar kernel family, and two masks -- drop every tenth frame (keep 90 %) and a seeded random 50 % -- and for
"confetti" (2*10^6 frames x 5 beams) the same masks plus keeping every other frame, whose runs are single 5-point frames:
* the device time of the gather kernel (clc_bench_subset: CUDA events, L2 flushed before each launch, a scratch subset each time);
* the bytes it moves -- read + write of the kept points' coordinate streams, plus 40 B per kept frame -- over that time, as a
  fraction of the H100 SXM data sheet's 3.35 TB/s.  Synthetic data is planar: its z is known to be 0 and is not copied
  (16 B per point each way); the `general_z` rows (configs[1], z drawn off the plane, uploaded with from_arrays) copy and check z too
  (24 B);
* the cold device time of one clc_eval of the subset on the same kernel family, and the ratio of the two;
* the host wall time of the whole subset() call;
* beside it (--recreate, default configs[1]), the wall time of creating the same kept frames from the host: from pageable per-frame
  arrays (Problem.from_frames) and from one pinned flat buffer (Problem.from_arrays).
The card's name and power limit are read in the same run.  Prints one JSON line per row.

    python bench_subset.py [--n 20] [--configs configs[1],config3,confetti] [--recreate configs[1]] [--out bench_subset.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import time

import numpy as np

CONFIGS = {"configs[1]": (10_000, 1_000), "config3": (100_000, 2_000), "confetti": (2_000_000, 5)}
HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as exc:  # the numbers below still stand, without the card's description
        return f"unknown ({exc})", "unknown"


def masks(n_frames, confetti=False):
    m = {"drop_every_10th": np.arange(n_frames) % 10 != 9,
         "random_50": np.random.default_rng(12345).random(n_frames) < 0.5}
    if confetti:  # runs of one 5-point frame: the gather's many-short-runs case
        m["keep_every_other"] = np.arange(n_frames) % 2 == 0
    return m


def wall_ms(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def recreate(sub, pinned_array, Problem):
    """Wall times of creating the subset's frames from host memory: pageable per-frame arrays, one pinned flat buffer."""
    d = sub.download()
    off, pts = d["offsets"], d["points"]
    frames = [pts[off[f]:off[f + 1]] for f in range(len(off) - 1)]
    Problem.from_frames(d["frame_pose"], frames).close()  # warm the pack threads and pinned slots
    t_frames, p = wall_ms(lambda: Problem.from_frames(d["frame_pose"], frames))
    p.close()
    buf = pinned_array(pts.shape)
    buf.array[...] = pts
    Problem.from_arrays(d["frame_pose"], off, buf.array).close()
    t_pinned, p = wall_ms(lambda: Problem.from_arrays(d["frame_pose"], off, buf.array))
    p.close()
    buf.free()
    return t_frames, t_pinned


def measure(src, family, cfg, name, keep, n, z_copied, want_recreate, card_info, Problem, pinned_array):
    pose = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
    src.bench_subset(keep, 2)
    gather = src.bench_subset(keep, n)
    src.subset(keep).close()
    call_ms, sub = wall_ms(lambda: src.subset(keep))
    with sub:
        sub.set_planar_mode(1 if family == "planar" else 0)
        sub.bench_eval(pose, 3)
        ev = sub.bench_eval(pose, n)
        K, P, _ = sub.sizes()
        t_frames, t_pinned = recreate(sub, pinned_array, Problem) if want_recreate else (None, None)
    nbytes = 2 * (24 if z_copied else 16) * P + 40 * K
    g_ms, e_ms = float(np.median(gather)), float(np.median(ev))
    return dict(config=cfg, family=family, mask=name, kept_frames=K, kept_points=P, z_copied=z_copied, gather_ms=g_ms,
                gather_ms_min=float(np.min(gather)), bytes=nbytes, gather_TBps=nbytes / g_ms / 1e9,
                fraction_of_3_35_TBps=nbytes / (g_ms * 1e-3) / HBM_PEAK, subset_eval_ms=e_ms, gather_over_eval=g_ms / e_ms,
                subset_call_wall_ms=call_ms, recreate_from_frames_wall_ms=t_frames, recreate_from_pinned_wall_ms=t_pinned,
                card=card_info[0], power_limit=card_info[1], samples=len(gather))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20, help="timed launches per row")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--recreate", default="configs[1]", help="configs whose rows also time the re-creation from the host")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from camlasercalibratool_b200 import Problem
    from camlasercalibratool_b200.api import pinned_array

    info = card()
    recreate_cfgs = set(a.recreate.split(",")) if a.recreate else set()
    results = []

    def emit(r):
        print(json.dumps(r), flush=True)
        results.append(r)

    for cfg in a.configs.split(","):
        n_frames, beams = CONFIGS[cfg]
        with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as src:
            for family in ("general", "planar"):
                src.set_planar_mode(1 if family == "planar" else 0)
                for name, keep in masks(n_frames, cfg == "confetti").items():
                    emit(measure(src, family, cfg, name, keep, a.n, False, cfg in recreate_cfgs, info, Problem, pinned_array))
        if cfg == "configs[1]":
            # off-plane data: the gather copies z and checks it
            with Problem.synthetic(n_frames, beams, seed=1, sigma=0.01) as syn:
                d = syn.download()
            d["points"][:, 2] = np.random.default_rng(7).normal(size=len(d["points"])) * 0.01
            with Problem.from_arrays(d["frame_pose"], d["offsets"], d["points"]) as src:
                for name, keep in masks(n_frames).items():
                    r = measure(src, "general", cfg, name, keep, a.n, True, False, info, Problem, pinned_array)
                    r["config"] = "configs[1]_general_z"
                    emit(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
