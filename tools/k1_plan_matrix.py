"""Print the rollout kernel's (K1's) launch for one engine per row, or the error text when the engine is refused. Two builds of
the same ABI print the same lines exactly when they choose every K1 launch alike, so a change to the K1 choice is checked
by running it against the parent's build and diffing:

    MPPIB_LIB=OLD.so python tools/k1_plan_matrix.py > old.txt
    python tools/k1_plan_matrix.py > new.txt
    diff old.txt new.txt

A row is one workload at a small size or at its BASELINE size, with no override or with one override set alone (a
descriptor flag or an environment variable read at create time). Each line holds launch_info() (grid, block, shared
memory, TMA, kernels per solve) and whether the engine keeps written-back controls (mppib_get_samples succeeds). Each
engine is created and closed; none solves. Needs a GPU."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mppi_generic_b200 as m  # noqa: E402
from mppi_generic_b200 import workloads as W  # noqa: E402

H = m.host

# (label, builder, flags); the builder takes N and T
WORKLOADS = [
    ("cartpole", W.cartpole, 0),
    ("double_integrator_tube", W.double_integrator_tube, 0),
    ("double_integrator_robust_tube+RMPPI", W.double_integrator_robust_tube, H.FLAG_RMPPI),
    ("autorally", W.autorally, 0),
    ("autorally_robust", W.autorally_robust, 0),
    ("racer_lstm", W.racer_lstm, 0),
    ("racer_lstm_h32", W.racer_lstm_h32, 0),
    ("quadrotor", W.quadrotor, 0),
    ("quadrotor_gates", W.quadrotor_gates, 0),
]
SMALL = (1024, 64)  # (N, T); the BASELINE size is each builder's default

# (label, environment, extra flags)
OVERRIDES = [
    ("default", {}, 0),
    ("MPPIB_NO_TMA", {"MPPIB_NO_TMA": "1"}, 0),
    ("MPPIB_NN_TENSOR", {"MPPIB_NN_TENSOR": "1"}, 0),
    ("MPPIB_NN_FFMA2", {"MPPIB_NN_FFMA2": "1"}, 0),
    ("FLAG_NN_MMA|FLAG_NN_TENSOR", {}, H.FLAG_NN_MMA | H.FLAG_NN_TENSOR),
    ("MPPIB_LSTM_SIMT", {"MPPIB_LSTM_SIMT": "1"}, 0),
    ("MPPIB_NO_WS", {"MPPIB_NO_WS": "1"}, 0),
    ("MPPIB_BX=64", {"MPPIB_BX": "64"}, 0),
    ("MPPIB_SPW=16", {"MPPIB_SPW": "16"}, 0),
    ("MPPIB_SPW=8", {"MPPIB_SPW": "8"}, 0),
    ("MPPIB_SPT=2", {"MPPIB_SPT": "2"}, 0),
    ("MPPIB_WS_PSPW=8", {"MPPIB_WS_PSPW": "8"}, 0),
    ("MPPIB_WS_PSPW=16", {"MPPIB_WS_PSPW": "16"}, 0),
    ("MPPIB_WS_PSPW=32", {"MPPIB_WS_PSPW": "32"}, 0),
    ("MPPIB_STREAM=0", {"MPPIB_STREAM": "0"}, 0),
    ("MPPIB_STREAM=1", {"MPPIB_STREAM": "1"}, 0),
    ("MPPIB_STREAM_READBACK", {"MPPIB_STREAM_READBACK": "1"}, 0),
    ("MPPIB_STREAM_READBACK+FLAG_WRITEBACK_CONTROLS", {"MPPIB_STREAM_READBACK": "1"}, H.FLAG_WRITEBACK_CONTROLS),
]


def row(builder, size, flags, env):
    w = builder() if size is None else builder(*size)
    for k, v in env.items():
        os.environ[k] = v
    try:
        e = w.make_engine(flags=flags)
    except H.MppibError as err:
        return f"N={w.N} T={w.T} refused: {err}"
    finally:
        for k in env:
            del os.environ[k]
    try:
        info = e.launch_info()
        try:
            e.get_samples()
            writeback = True
        except H.MppibError:
            writeback = False
        return (f"N={w.N} T={w.T} grid={info['grid']} block={info['block']} smem_bytes={info['smem_bytes']} "
                f"uses_tma={int(info['uses_tma'])} kernels_per_solve={info['kernels_per_solve']} writeback={int(writeback)}")
    finally:
        e.close()


def main():
    for name, builder, wflags in WORKLOADS:
        for size in (SMALL, None):
            for label, env, flags in OVERRIDES:
                print(f"{name:36s} {label:46s} {row(builder, size, wflags | flags, env)}", flush=True)


if __name__ == "__main__":
    main()
