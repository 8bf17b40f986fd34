"""Time K1 (the fused rollout) of RacerSuspension (the rigid-body RACER vehicle) + RacerQuadraticCost against
RacerDubinsElevation + RacerQuadraticCost on flat ground, both VanillaMPPI with the Gaussian sampler at N = 32768, T = 100:
  - rigid:     workloads.racer_rigid_suspension (dt 0.01);
  - dubins:    workloads.racer_elevation without a map, at the same N, T, sampler and cost.
The engines are built and warmed up first, then timed in alternation, `--rounds` rounds of `--steps` solves each. K1 time:
mppib_get_timing's rollout_ms (CUDA events around the rollout launch); the median over all timed solves is reported, with
the spread of the per-round medians. Prints one JSON line with the card's name, power limit and maximum SM clock read in
the same run.
Usage: python tools/racer_rigid_suspension_timing.py [--steps 100] [--rounds 5] [--warmup 30]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mppi_generic_b200 import workloads as W  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=30)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    N, T = 32768, 100
    out = {"gpu": gpu[0] if gpu else "unknown", "N": N, "T": T, "steps": a.steps, "rounds": a.rounds, "cases": []}
    dubins = W.racer_elevation(N, T, use_map=False)
    dubins.sampler.setStdDev([0.3, 0.3])
    cases = {"rigid": W.racer_rigid_suspension(N, T), "dubins": dubins}
    engines = {k: w.make_engine() for k, w in cases.items()}
    for k, e in engines.items():
        for _ in range(a.warmup):
            e.solve(cases[k].x0, cases[k].U0)
        e.enable_timing(True)
    k1 = {k: [] for k in cases}
    for _ in range(a.rounds):
        for k, e in engines.items():
            r = []
            for _ in range(a.steps):
                e.solve(cases[k].x0, cases[k].U0)
                r.append(e.timing()["rollout_ms"])
            k1[k].append(r)
    for k, e in engines.items():
        info = e.launch_info()
        rounds = np.array(k1[k]) * 1e3
        out["cases"].append({"model": k, "grid": info["grid"], "block": info["block"],
                             "k1_us_median": float(np.median(rounds)),
                             "round_medians_us": [round(float(v), 1) for v in np.median(rounds, axis=1)]})
        e.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
