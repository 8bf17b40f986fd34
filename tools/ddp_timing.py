"""Time the device DDP feedback solve (mppib_ddp_feedback, csrc/ddp_kernel.cuh) and the CPU restatement of it.

Kernel time: device durations of the ddp_kernel launches, read from torch.profiler's CUDA activity over many calls, in a
pass of their own. (CUDA events cannot bracket the kernel alone: mppib_ddp_feedback launches it on the engine's stream and
synchronises before it returns, so an end event recorded after the call would include the host's return.)
Call time: host wall clock around mppib_ddp_feedback, which ends in a stream synchronise. CPU: tests/ddp_oracle.py (float32
numpy) on the same inputs. Cases: double integrator and Autorally at T = 100 with 1 iteration, quadrotor at T = 500 with
100 iterations. Prints one JSON line with the card's name and power limit read in the same run."""
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
from tests import ddp_oracle as DO  # noqa: E402  (the CPU restatement being timed)

H = m.host


def tracking_case(dyn, dt, x_start, ut):
    """Targets = the open-loop rollout of ut from x_start; the solve starts 0.05 away."""
    mdl = DO.Model(dyn)
    T = ut.shape[0]
    xt = np.zeros((T, mdl.S), np.float32)
    xt[0] = x_start
    for i in range(1, T):
        xt[i] = xt[i - 1] + DO.f(mdl, xt[i - 1], ut[i - 1]) * np.float32(dt)
    x0 = (x_start + 0.05 * np.random.RandomState(7).randn(mdl.S)).astype(np.float32)
    return x0, xt


def case(name, T):
    if name == "quadrotor_tracking":
        dyn = H.QuadrotorDynamics([(-2.5, 2.5)] * 3 + [(0.0, 36.0)])
        dt = 0.01
        x_goal = np.array([6, 4, 3, 0, 0, 0, 0.7071068, 0, 0, 0.7071068, 0, 0, 0], np.float32)
        x0 = np.array([0, -0.5, 0, 0, 0.5, 0, 1, 0, 0, 0, 0, 0, 0], np.float32)
        xt, ut = np.tile(x_goal, (T, 1)), np.tile(dyn.zero_control_, (T, 1))
        Q = np.diag([25, 25, 300, 15, 15, 300, 0, 0, 0, 0, 30, 30, 30]).astype(np.float32)
        Qf = np.diag([250, 250, 3000, 150, 150, 3000, 0, 0, 0, 0, 300, 300, 300]).astype(np.float32)
        R = np.diag([550, 550, 550, 1]).astype(np.float32)
    else:
        k = np.arange(T)
        if name == "di":
            dyn = H.DoubleIntegratorDynamics(1.0)
            xs = np.array([2, 0, 0, 1], np.float32)
            ut = np.stack([np.cos(k * 0.05), np.sin(k * 0.05)], 1).astype(np.float32)
        else:
            dyn = H.NeuralNetModel([(-1.0, 1.0), (-2.0, 2.0)])
            dyn.updateModel([6, 32, 32, 4], W.synthetic_nn_weights(1))
            xs = np.array([0, 0, 0, 0, 4, 0, 0], np.float32)
            ut = np.stack([0.3 * np.sin(k * 0.05), 0.2 + 0.1 * np.cos(k * 0.07)], 1).astype(np.float32)
        dt = 0.02
        x0, xt = tracking_case(dyn, dt, xs, ut)
        S, Cd = dyn.STATE_DIM, dyn.CONTROL_DIM
        Q, Qf, R = np.eye(S, dtype=np.float32), np.eye(S, dtype=np.float32), np.eye(Cd, dtype=np.float32)
    return dyn, dt, x0, xt, ut, Q, Qf, R


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    out = {"gpu": gpu, "cases": []}
    for name, T, iters, reps in (("di", 100, 1, 200), ("autorally", 100, 1, 200), ("quadrotor_tracking", 500, 100, 10)):
        dyn, dt, x0, xt, ut, Q, Qf, R = case(name, T)
        e = H.Engine(dyn, H._standalone_cost(dyn.DYN_ID), H.GaussianDistribution(dyn.CONTROL_DIM), 64, 8)
        e.set_solver(dt, 1.0, 0.0)
        e.set_ddp(Q, Qf, R, iters)
        for _ in range(3):
            e.ddp_feedback(x0, xt, ut)
        t0 = time.perf_counter()
        for _ in range(reps):
            e.ddp_feedback(x0, xt, ut)
        call_us = (time.perf_counter() - t0) / reps * 1e6
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                e.ddp_feedback(x0, xt, ut)
        durs = [ev.device_time for ev in prof.events() if "ddp_kernel" in ev.name]
        e.close()
        t0 = time.perf_counter()
        DO.ddp_run(DO.Model(dyn), dt, x0, xt, ut, Q, Qf, R, iters)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        out["cases"].append({"case": name, "T": T, "iterations": iters, "kernel_us_mean": float(np.mean(durs)),
                             "kernel_us_min": float(np.min(durs)), "kernels": len(durs), "call_us": call_us,
                             "cpu_oracle_ms": cpu_ms})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
