"""Check that an engine gives back every byte of device memory it took, after each buffer that grows or is freed on
demand has done so (csrc/device_resources.cuh: DeviceBuffer::reserve / reset):
  - an RMPPI engine (quadrotor + QuadrotorMapCost, D = 2): solve, init-eval twice with more candidates the second time, the
    cost map replaced by one with four times the cells, a DDP at the horizon that writes the feedback gains, a longer DDP
    that grows its workspace, the feedback gains freed and set again, a solve after each;
  - a Vanilla engine with written-back controls: solve, sampled trajectories twice with more samples the second time,
    the device-side roll-forward of the caller's controls and of the solve's result, the importance weights (a buffer made
    on first use), and an L2 flush set, grown and set to 0, then a solve;
  - a ColoredNoise and an NLN engine (the samplers whose spectrum, plan and log-normal planes the noise source owns): solve,
    new sampler parameters, solve, burn_draws, solve;
  - an Autorally engine: solve, new NN weights, solve, a costmap with four times the texels, solve;
  - a RACER LSTM engine: solve, new LSTM weights, solve, an elevation map with four times the cells, solve.
The free device memory (cudaMemGetInfo) after all six are destroyed is compared with the value before they were created. The
sequence runs twice and the second pass is the one checked: the first also loads the kernels, which stay on the device.
Every call raises on a status other than MPPIB_OK. Prints one JSON line; exits 1 if the second pass leaves more than
`--slack-mib` less free memory than it found (another process on a shared card can move the figure as well).
Usage: python tools/engine_memory_check.py [--slack-mib 2]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mppi_generic_b200 as m  # noqa: E402
from mppi_generic_b200 import workloads as W  # noqa: E402

H = m.host


def exercise():
    w = W.quadrotor_gates(1024, 40)
    e = H.Engine(w.dyn, w.cost, w.sampler, w.N, w.T, 2, flags=H.FLAG_RMPPI)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    e.seed(w.seed, 0)
    gains = (np.random.RandomState(3).randn(w.T, 13, 4) * 0.05).astype(np.float32)
    x0 = np.stack([w.x0[0], w.x0[0] + np.array([0.05, 0.1, 0.02] + [0.0] * 10, np.float32)])
    U = np.tile(w.U0, (2, 1, 1))
    e.set_rmppi(3000.0, gains)
    e.solve(x0, U)
    for K, spc in ((2, 32), (4, 128)):
        cand = np.linspace(x0[0], x0[1], K).astype(np.float32)
        e.init_eval(cand, np.arange(K, dtype=np.int32), spc, U[0], 1)
    w.cost.tex_helper_ = W.quadrotor_track_map(resolution=0.125)[0]
    e.push_cost()
    e.solve(x0, U)
    for T, to_rmppi in ((w.T, True), (3 * w.T, False)):  # hover targets; the second horizon grows the DDP workspace
        e.ddp_feedback(x0[0], np.tile(x0[0], (T, 1)), np.tile(U[0, :1], (T, 1)), to_rmppi=to_rmppi)
        e.solve(x0, U)
    e.set_rmppi(3000.0, None)
    e.solve(x0, U)
    e.set_rmppi(3000.0, gains)
    e.solve(x0, U)
    e.close()

    w = W.quadrotor_gates(1024, 40)
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    U_opt, _ = e.solve(w.x0, w.U0)
    for n in (8, 256):
        idx = np.concatenate([[-1], np.arange(n - 1)]).astype(np.int32)
        e.sample_trajectories(w.x0[0], w.U0[0], idx, U_opt=U_opt[0])
    e.nominal_trajectory(w.x0, U_opt, np.zeros((2, 4), np.float32))
    e.nominal_trajectory(w.x0)
    e.get_weights()
    for nbytes in (1 << 20, 8 << 20, 0):
        e.set_option(H.OPT_L2_FLUSH_BYTES, nbytes)
    e.solve(w.x0, w.U0)
    e.close()

    # N * T a multiple of 8192: an NLN draw re-positions the generator after burn_draws only on such a boundary
    for sampler in (H.ColoredNoiseDistribution(2, [1.0, 1.0], [1.0, 2.0]), H.NLNDistribution(2, [0.5, 0.5])):
        w = W.double_integrator_vanilla(1024, 32)
        w.sampler = sampler
        e = w.make_engine()
        e.solve(w.x0, w.U0)
        sampler.setStdDev([0.8, 0.6])
        if isinstance(sampler, H.ColoredNoiseDistribution):
            sampler.setExponents([0.5, 1.5])
        e.push_params()
        e.solve(w.x0, w.U0)
        e.burn_draws(3)
        e.solve(w.x0, w.U0)
        e.close()

    # the model's weights and maps (csrc/model_params.cuh), each replaced between solves; the maps grow
    w = W.autorally(1024, 40)
    e = w.make_engine()
    e.solve(w.x0, w.U0)
    w.dyn.updateModel([6, 32, 32, 4], W.synthetic_nn_weights(5))
    e.push_params()
    e.solve(w.x0, w.U0)
    ch0, xb, yb, ppm = W.track_map_standard()
    w.cost.loadTrackData(np.kron(ch0, np.ones((2, 2), np.float32)), xb[0], xb[1], yb[0], yb[1], 2 * ppm)
    e.push_params()
    e.solve(w.x0, w.U0)
    e.close()

    w = W.racer_lstm_gaussian(1024, 40)
    hills = lambda n: np.sin(0.3 * np.arange(n * n, dtype=np.float32)).reshape(n, n)  # noqa: E731
    w.dyn.setElevationMap(hills(48), 0.5, (-12.0, -12.0, 0.0))
    e = w.make_engine()
    e.solve(w.x0, w.U0)
    w.dyn.setAllValues(*W.synthetic_lstm_weights(4, 20, 9))
    e.push_params()
    e.solve(w.x0, w.U0)
    w.dyn.setElevationMap(hills(96), 0.25, (-12.0, -12.0, 0.0))
    e.push_params()
    e.solve(w.x0, w.U0)
    e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slack-mib", type=float, default=2.0)
    a = ap.parse_args()
    torch.cuda.init()
    free = [torch.cuda.mem_get_info()[0]]
    for _ in range(2):
        exercise()
        free.append(torch.cuda.mem_get_info()[0])
    out = {"gpu": torch.cuda.get_device_name(0), "free_before": free[0], "free_after_first_pass": free[1],
           "free_after_second_pass": free[2], "second_pass_kept_bytes": free[1] - free[2]}
    out["ok"] = out["second_pass_kept_bytes"] <= a.slack_mib * 2 ** 20
    print(json.dumps(out))
    sys.exit(0 if out["ok"] else 1)


if __name__ == "__main__":
    main()
