"""Time K1 (the fused rollout) of the smooth-MPPI sampler against the Gaussian sampler on the same pair and the same
kernel form, at N = 32768, T = 100:
  - cartpole:  Gaussian and smooth-MPPI, both on the generic kernel;
  - autorally: Gaussian on the generic kernel (MPPIB_FLAG_NO_WARP_SPEC) and smooth-MPPI (which always takes it), next to
               the Gaussian engine's default warp-specialised kernel, so that the price of routing a smooth engine to the
               generic form is visible.
The engines are built and warmed up first, then timed in alternation, `--rounds` rounds of `--steps` solves each. K1 time:
mppib_get_timing's rollout_ms (CUDA events around the rollout launch) of each solve; the median over all timed solves is
reported, with the spread of the per-round medians. Prints one JSON line with the card's name, power limit and maximum SM
clock read in the same run.
Usage: python tools/smooth_mppi_timing.py [--steps 100] [--rounds 5] [--warmup 30]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mppi_generic_b200 import host as H  # noqa: E402
from mppi_generic_b200 import workloads as W  # noqa: E402


def _smooth(w, sd):
    """The workload with a smooth-MPPI sampler whose control samples spread as the Gaussian one's: sigma / dt_s."""
    s = H.SmoothMPPIDistribution(w.dyn.CONTROL_DIM, [v / 0.015 for v in sd], dt=0.015)
    for c in range(w.dyn.CONTROL_DIM):
        s.params.control_cost_coeff[c] = w.sampler.params.control_cost_coeff[c]
    w.sampler = s
    return w


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
    cases = {
        "cartpole gaussian generic": (W.cartpole(N, T), 0),
        "cartpole smooth generic": (_smooth(W.cartpole(N, T), [5.0]), 0),
        "autorally gaussian generic": (W.autorally(N, T), H.FLAG_NO_WARP_SPEC),
        "autorally smooth generic": (_smooth(W.autorally(N, T), [0.3, 0.3]), 0),
        "autorally gaussian warp-specialised": (W.autorally(N, T), 0),
    }
    engines = {k: w.make_engine(flags=f) for k, (w, f) in cases.items()}
    for k, e in engines.items():
        w = cases[k][0]
        for _ in range(a.warmup):
            e.solve(w.x0, w.U0)
    k1 = {k: [] for k in cases}
    for _ in range(a.rounds):
        for k, e in engines.items():
            w = cases[k][0]
            r = []
            for _ in range(a.steps):
                e.enable_timing(True)  # resets the sums: the next read is this solve's
                e.solve(w.x0, w.U0)
                r.append(e.timing()["rollout_ms"])
            e.enable_timing(False)
            k1[k].append(r)
    for k, e in engines.items():
        info = e.launch_info()
        rounds = np.array(k1[k]) * 1e3
        out["cases"].append({"case": k, "grid": info["grid"], "block": info["block"],
                             "k1_us_median": float(np.median(rounds)),
                             "round_medians_us": [round(float(v), 1) for v in np.median(rounds, axis=1)]})
        e.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
