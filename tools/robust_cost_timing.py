"""Time K1 (the fused rollout) and whole solves with the robust costs next to the costs they replace, on the same model,
sizes and launch rules:
  - Autorally at N = 32768, T = 100 (C4's size, the warp-specialised K1): ARStandardCost on track_map_standard against
    ARRobustCost on track_map_robust (workloads.autorally / autorally_robust);
  - the double integrator at C3's size (N = 16384, T = 150), Tube-MPPI (two systems): the circle cost against
    DoubleIntegratorRobustCost (workloads.double_integrator_tube / double_integrator_robust_tube).
K1 time: mppib_get_timing's rollout_ms (CUDA events around the rollout launch), averaged over the timed solves. Solves/s:
host wall clock over `--steps` back-to-back mppib_solve calls, each ending in a stream synchronise. Prints one JSON line
with the card's name, power limit and maximum SM clock read in the same run.
Usage: python tools/robust_cost_timing.py [--steps 300] [--warmup 30]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mppi_generic_b200 as m  # noqa: E402
from mppi_generic_b200 import workloads as W  # noqa: E402


def measure(w, steps, warmup):
    e = w.make_engine()
    info = e.launch_info()
    for _ in range(warmup):
        e.solve(w.x0, w.U0)
    e.enable_timing(True)
    k1 = []
    t0 = time.perf_counter()
    for _ in range(steps):
        e.solve(w.x0, w.U0)
        k1.append(e.timing()["rollout_ms"])
    wall = time.perf_counter() - t0
    e.enable_timing(False)
    t0 = time.perf_counter()
    for _ in range(steps):
        e.solve(w.x0, w.U0)
    wall_untimed = time.perf_counter() - t0
    e.close()
    return {"workload": w.name, "cost": type(w.cost).__name__, "N": w.N, "T": w.T, "D": w.D,
            "grid": info["grid"], "block": info["block"], "k1_us_mean": 1e3 * float(np.mean(k1)),
            "k1_us_median": 1e3 * float(np.median(k1)), "solves_per_s": steps / wall_untimed,
            "solves_per_s_with_events": steps / wall}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    out = {"gpu": gpu[0] if gpu else "unknown", "steps": a.steps, "cases": []}
    for build in (W.autorally, W.autorally_robust):
        out["cases"].append(measure(build(32768, 100), a.steps, a.warmup))
    for build in (W.double_integrator_tube, W.double_integrator_robust_tube):
        out["cases"].append(measure(build(16384, 150), a.steps, a.warmup))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
