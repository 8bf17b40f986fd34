"""Snapshot of the library's host twins (include/mppi_b200/host_twins.h) on seeded inputs.

    python tests/golden/make_host_twin_snapshot.py [OUT.npz]     (default: tests/golden/host_twins/snapshot.npz)

Every built-in dynamics model is stepped and rolled forward through each exported entry that takes it: the generic
mppib_host_step / _output_trajectory, and each model's own _step_* / _output_trajectory_* pair. The inputs cover the RACER
LSTM at two network sizes, the RACER models with and without their maps, and controls both inside the deadband and outside
the limits. Every output buffer starts as NaN, so the snapshot also pins which entries a call leaves alone. Return codes are
recorded for every generic entry and every dynamics id (refused and unknown ids included) and for each argument a call
checks. tests/test_host_twin_snapshot.py regenerates the inputs and compares the library against this file bit for bit.
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mppi_generic_b200 import host as H  # noqa: E402

SEED = 20261018
T = 16          # trajectory length
DT = 0.05
NSTEP = 6       # single steps per model
IDS = list(range(8)) + [8, -1, 1000, 1 << 30]  # the built-in ids, then unknown ones
PAD = 32        # buffer length for calls whose dimensions are unknown
f32 = np.float32


def _nan(n: int) -> np.ndarray:
    return np.full(n, np.nan, f32)


def _p(a):
    return None if a is None else a.ctypes.data


def cpu_runs_v3_clones() -> bool:
    """The FNN and LSTM heads are target_clones("arch=x86-64-v3", "default"): the loader picks the x86-64-v3 (AVX2 + FMA)
    clone when the CPU has every x86-64-v3 feature ("abm" is LZCNT in /proc/cpuinfo)."""
    try:
        flags = set(open("/proc/cpuinfo").read().split())
    except OSError:
        return False
    return {"avx", "avx2", "bmi1", "bmi2", "f16c", "fma", "abm", "movbe", "xsave"} <= flags


class Model:
    """One set of inputs for one model: parameters (a ctypes blob), optional network and maps, sample states and controls,
    and a trajectory's x0 / U."""

    def __init__(self, name, dyn_id, S, Cd, O, params, kind, nn=None, lstm=None, elev=None, normals=None):
        self.name, self.dyn_id, self.S, self.C, self.O = name, dyn_id, S, Cd, O
        self.params, self.kind, self.nn, self.lstm, self.elev, self.normals = params, kind, nn, lstm, elev, normals

    @property
    def uses_clones(self) -> bool:
        """Runs the target_clones network code (bits may differ between the AVX2 + FMA and baseline clones)."""
        return self.nn is not None or self.lstm is not None

    def net(self, hidden, cell) -> H.HostLSTM:
        theta, Hd, L1 = self.lstm
        return H.HostLSTM(theta.ctypes.data, Hd, L1, _p(hidden), _p(cell), _p(self.elev))

    def initial_hidden_cell(self):
        theta, Hd, _ = self.lstm
        base = 4 * Hd * Hd + 4 * Hd * H.RACER_LSTM_INPUT_DIM + 4 * Hd
        return theta[base:base + Hd].copy(), theta[base + Hd:base + 2 * Hd].copy()


def _limits(p, lo, hi, db):
    for i, (a, b, d) in enumerate(zip(lo, hi, db)):
        p.lim.rng_lo[i], p.lim.rng_hi[i], p.lim.deadband[i] = a, b, d


def _controls(rng, p, Cd, n):
    """A third of the entries inside the deadband, a third outside the limits, the rest inside the range."""
    lim = p.lim
    lo = np.array([lim.rng_lo[i] for i in range(Cd)], f32)
    hi = np.array([lim.rng_hi[i] for i in range(Cd)], f32)
    db = np.array([lim.deadband[i] for i in range(Cd)], f32)
    which = rng.integers(0, 3, (n, Cd))
    inside_db = rng.uniform(-1, 1, (n, Cd)) * db
    span = hi - lo
    outside = np.where(rng.random((n, Cd)) < 0.5, lo - rng.uniform(0.1, 1.0, (n, Cd)) * span,
                       hi + rng.uniform(0.1, 1.0, (n, Cd)) * span)
    inside = lo + rng.uniform(0, 1, (n, Cd)) * span
    return np.where(which == 0, inside_db, np.where(which == 1, outside, inside)).astype(f32)


def _map_blob(values):
    hdr = H.ElevationMapHeader()
    hdr.height, hdr.width = values.shape[0], values.shape[1]
    hdr.origin[:] = [-5.0, -4.0, 0.0]
    c, s = np.cos(0.2), np.sin(0.2)
    hdr.rotations[:] = [c, -s, 0.0, s, c, 0.0, 0.0, 0.0, 1.0]
    hdr.resolution[:] = [0.5, 0.5, 1.0]
    hdr.use = 1
    return np.concatenate([np.frombuffer(bytes(hdr), np.uint8),
                           np.ascontiguousarray(values, f32).reshape(-1).view(np.uint8)])


def _elevation(rng):
    yy, xx = np.mgrid[0:16, 0:20].astype(f32)
    v = 0.3 * np.sin(0.5 * xx) + 0.2 * np.cos(0.3 * yy) + 0.02 * rng.standard_normal((16, 20))
    v[3, 7] = v[11, 2] = np.nan  # unobserved cells: the models fall back on their own guards
    return _map_blob(v)


def _normals(rng):
    n = np.concatenate([0.15 * rng.standard_normal((16, 20, 2)), np.ones((16, 20, 1))], axis=-1)
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    return _map_blob(np.concatenate([n, np.zeros((16, 20, 1))], axis=-1))


def _racer_state(rng, n, S):
    x = np.zeros((n, S), f32)
    x[:, 0] = rng.choice([0.1, -0.15, 1.5, 4.0, -2.0, 7.0], n) + 0.05 * rng.standard_normal(n)  # every speed band
    x[:, 1] = rng.uniform(-3.1, 3.1, n)
    x[:, 2] = rng.uniform(-7.0, 7.0, n)  # partly off the map
    x[:, 3] = rng.uniform(-6.0, 6.0, n)
    x[:, 4] = rng.uniform(-0.6, 0.6, n)
    x[:, 5] = rng.uniform(-0.05, 0.3, n)
    x[:, 6:8] = 0.1 * rng.standard_normal((n, 2))
    return x


def _lstm_theta(rng, Hd, L1):
    return (0.3 * rng.standard_normal(H.racer_lstm_num_params(Hd, L1))).astype(f32)


def models():
    """Every model's inputs, drawn from SEED."""
    rng = np.random.default_rng(SEED)
    elev, normals = _elevation(rng), _normals(rng)
    out = []

    p = H.CartpoleDynamics(1.0, 0.5, 1.2).params
    _limits(p, [-5.0], [5.0], [0.2])
    out.append(Model("cartpole", H.DYN_CARTPOLE, 4, 1, 4, p, "generic"))
    out[-1].x = rng.standard_normal((NSTEP + 1, 4)).astype(f32)

    p = H.DoubleIntegratorDynamics().params
    _limits(p, [-2.0, -1.5], [2.0, 1.5], [0.1, 0.05])
    out.append(Model("double_integrator", H.DYN_DOUBLE_INTEGRATOR, 4, 2, 4, p, "generic"))
    out[-1].x = (2 * rng.standard_normal((NSTEP + 1, 4))).astype(f32)

    p = H.NeuralNetModel().params
    _limits(p, [-0.99, -0.99], [0.99, 0.65], [0.05, 0.02])
    nn = (0.3 * rng.standard_normal(H.AR_NN_NUM_PARAMS)).astype(f32)
    out.append(Model("autorally", H.DYN_AUTORALLY_NN, 7, 2, 8, p, "generic", nn=nn))
    out[-1].x = (rng.standard_normal((NSTEP + 1, 7)) * [2, 2, 1, 0.2, 3, 0.5, 0.5]).astype(f32)

    p = H.QuadrotorDynamics(mass=1.2).params
    _limits(p, [-2.5, -2.5, -2.5, 0.0], [2.5, 2.5, 2.5, 36.0], [0.05, 0.05, 0.05, 0.5])
    out.append(Model("quadrotor", H.DYN_QUADROTOR, 13, 4, 13, p, "generic"))
    x = rng.standard_normal((NSTEP + 1, 13)).astype(f32)
    q = np.concatenate([np.ones((NSTEP + 1, 1)), 0.2 * rng.standard_normal((NSTEP + 1, 3))], axis=1)
    x[:, 6:10] = q / np.linalg.norm(q, axis=1, keepdims=True)
    x[:, 10:13] *= 0.5
    out[-1].x = x

    for Hd, L1 in ((4, 20), (16, 36)):
        for m_ in (None, elev):
            p = H.RacerDubinsElevationLSTMSteering().params
            _limits(p, [-1.0, -1.0], [1.0, 1.0], [0.05, 0.02])
            name = f"racer_lstm_h{Hd}_l{L1}" + ("_map" if m_ is not None else "")
            out.append(Model(name, H.DYN_RACER_LSTM, 19, 2, 28, p, "lstm", lstm=(_lstm_theta(rng, Hd, L1), Hd, L1),
                             elev=m_))
            x = _racer_state(rng, NSTEP + 1, 19)
            x[:, 8] = 0.5 * rng.standard_normal(NSTEP + 1)
            x[:, 9:19] = rng.uniform(0.01, 0.2, (NSTEP + 1, 10))
            out[-1].x = x

    for m_ in (None, elev):
        p = H.RacerDubinsElevation().params
        _limits(p, [-1.0, -1.0], [1.0, 1.0], [0.05, 0.02])
        out.append(Model("racer_dubins_elevation" + ("_map" if m_ is not None else ""), H.DYN_RACER_DUBINS_ELEVATION, 19,
                         2, 28, p, "dubins", elev=m_))
        x = _racer_state(rng, NSTEP + 1, 19)
        x[:, 8] = 0.5 * rng.standard_normal(NSTEP + 1)
        x[:, 9:19] = rng.uniform(0.01, 0.2, (NSTEP + 1, 10))
        out[-1].x = x

    for tag, e_, n_ in (("", None, None), ("_elev", elev, None), ("_elev_normals", elev, normals)):
        p = H.RacerDubinsElevationSuspension().params
        _limits(p, [-1.0, -1.0], [1.0, 1.0], [0.05, 0.02])
        out.append(Model("racer_suspension_lstm" + tag, H.DYN_RACER_SUSPENSION_LSTM, 24, 2, 28, p, "suspension",
                         lstm=(_lstm_theta(rng, 4, 20), 4, 20), elev=e_, normals=n_))
        x = _racer_state(rng, NSTEP + 1, 24)
        x[:, 8] = rng.uniform(0.2, 0.8, NSTEP + 1)
        x[:, 9:12] = 0.3 * rng.standard_normal((NSTEP + 1, 3))
        x[:, 12] = 0.5 * rng.standard_normal(NSTEP + 1)
        x[:, 13:23] = rng.uniform(0.01, 0.2, (NSTEP + 1, 10))
        x[:, 23] = rng.standard_normal(NSTEP + 1)
        out[-1].x = x

    dyn = H.RacerSuspension()
    p = dyn.params
    _limits(p, [-1.0, -1.0], [1.0, 1.0], [0.05, 0.02])
    out.append(Model("racer_suspension", H.DYN_RACER_SUSPENSION, 14, 2, 26, p, "rigid"))
    x = np.zeros((NSTEP + 1, 14), f32)
    x[:, 0:2] = rng.uniform(-5, 5, (NSTEP + 1, 2))
    x[:, 2] = dyn.restHeight() + 0.05 * rng.standard_normal(NSTEP + 1)
    yaw = rng.uniform(-3, 3, NSTEP + 1)
    q = np.stack([np.cos(yaw / 2), 0.03 * rng.standard_normal(NSTEP + 1), 0.03 * rng.standard_normal(NSTEP + 1),
                  np.sin(yaw / 2)], axis=1)
    x[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    x[:, 7:10] = rng.standard_normal((NSTEP + 1, 3)) * [3.0, 0.5, 0.2]
    x[:, 10:13] = 0.2 * rng.standard_normal((NSTEP + 1, 3))
    x[:, 13] = rng.uniform(-0.4, 0.4, NSTEP + 1)
    out[-1].x = x

    for m in out:
        m.u = _controls(rng, m.params, m.C, NSTEP)
        m.U = _controls(rng, m.params, m.C, T)
        if m.lstm is not None:
            Hd = m.lstm[1]
            m.hc = (0.5 * rng.standard_normal((NSTEP, 2, Hd))).astype(f32)
    return out


def _blob(m):
    return C.addressof(m.params)


def step(L, m, x, u, hidden=None, cell=None, generic=False, y=None):
    """The model's own exported step (the generic mppib_host_step when `generic`): (rc, x_next, xdot, y). The outputs go
    to a copy of `y` (default NaN)."""
    xn, xd = _nan(m.S), _nan(m.S)
    y = _nan(m.O) if y is None else np.array(y, f32)
    x, u = np.ascontiguousarray(x, f32), np.ascontiguousarray(u, f32)
    a = (_p(x), _p(u), C.c_float(DT), _p(xn), _p(xd), _p(y))
    if generic:
        rc = L.mppib_host_step(m.dyn_id, _blob(m), _p(m.nn), *a)
    elif m.kind == "lstm":
        rc = L.mppib_host_step_lstm(_blob(m), C.byref(m.net(hidden, cell)), *a)
    elif m.kind == "dubins":
        rc = L.mppib_host_step_racer_dubins_elevation(_blob(m), _p(m.elev), *a)
    elif m.kind == "suspension":
        rc = L.mppib_host_step_racer_suspension(_blob(m), C.byref(m.net(hidden, cell)), _p(m.normals), *a)
    elif m.kind == "rigid":
        rc = L.mppib_host_step_racer_rigid_suspension(_blob(m), *a)
    else:
        rc = L.mppib_host_step(m.dyn_id, _blob(m), _p(m.nn), *a)
    return rc, xn, xd, y


def trajectory(L, m, generic=False, hidden=None, cell=None):
    """The model's own exported roll-forward of (m.x[0], m.U) (the generic one when `generic`): (rc, states, outputs)."""
    states, outputs = _nan(T * m.S), _nan(T * m.O)
    a = (_p(m.x[0]), _p(m.U), T, C.c_float(DT), _p(states), _p(outputs))
    if generic or m.kind == "generic":
        rc = L.mppib_host_output_trajectory(m.dyn_id, _blob(m), _p(m.nn), *a)
    elif m.kind == "lstm":
        rc = L.mppib_host_output_trajectory_lstm(_blob(m), C.byref(m.net(hidden, cell)), *a)
    elif m.kind == "dubins":
        rc = L.mppib_host_output_trajectory_racer_dubins_elevation(_blob(m), _p(m.elev), *a)
    elif m.kind == "suspension":
        rc = L.mppib_host_output_trajectory_racer_suspension(_blob(m), C.byref(m.net(hidden, cell)), _p(m.normals), *a)
    else:
        rc = L.mppib_host_output_trajectory_racer_rigid_suspension(_blob(m), *a)
    return rc, states.reshape(T, m.S), outputs.reshape(T, m.O)


def _argument_checks(L, m, out):
    """The return code (and what is left in the buffers) with each pointer argument NULL in turn, and with T <= 0."""
    x, u = m.x[0], m.u[0]
    hidden, cell = (m.hc[0][0].copy(), m.hc[0][1].copy()) if m.lstm is not None else (None, None)
    rcs = []

    def call_step(fn, *pre, nulls=()):
        bufs = [_nan(m.S), _nan(m.S), _nan(m.O)]
        args = [_p(x), _p(u), C.c_float(DT)] + [_p(b) for b in bufs]
        for i in nulls:
            args[i] = None
        rcs.append(fn(*pre, *args))
        return bufs

    def call_traj(fn, *pre, nulls=(), steps=T):
        bufs = [_nan(T * m.S), _nan(T * m.O)]
        args = [_p(m.x[0]), _p(m.U), steps, C.c_float(DT)] + [_p(b) for b in bufs]
        for i in nulls:
            args[i] = None
        rcs.append(fn(*pre, *args))
        return bufs

    left = []
    step_nulls, traj_nulls = [(0,), (1,), (3,), (4,), (5,)], [(0,), (1,), (4,), (5,)]
    if m.kind in ("generic", "rigid"):
        for nulls in step_nulls:
            left += call_step(L.mppib_host_step, m.dyn_id, _blob(m), _p(m.nn), nulls=nulls)
        left += call_step(L.mppib_host_step, m.dyn_id, None, _p(m.nn))
        left += call_step(L.mppib_host_step, m.dyn_id, _blob(m), None)  # Autorally without its network
        for nulls in traj_nulls:
            left += call_traj(L.mppib_host_output_trajectory, m.dyn_id, _blob(m), _p(m.nn), nulls=nulls)
        left += call_traj(L.mppib_host_output_trajectory, m.dyn_id, None, _p(m.nn))
        left += call_traj(L.mppib_host_output_trajectory, m.dyn_id, _blob(m), None)
        for steps in (0, -1, 1):
            left += call_traj(L.mppib_host_output_trajectory, m.dyn_id, _blob(m), _p(m.nn), steps=steps)
    if m.kind == "rigid":
        fs, ft = L.mppib_host_step_racer_rigid_suspension, L.mppib_host_output_trajectory_racer_rigid_suspension
        for nulls in step_nulls:
            left += call_step(fs, _blob(m), nulls=nulls)
        left += call_step(fs, None)
        for nulls in traj_nulls:
            left += call_traj(ft, _blob(m), nulls=nulls)
        left += call_traj(ft, None)
        for steps in (0, -1, 1):
            left += call_traj(ft, _blob(m), steps=steps)
        for jac in (True, False):
            for i in range(5):
                xd, y, J = _nan(14), _nan(26), _nan(9)
                args = [_blob(m), _p(x), _p(u), _p(xd), _p(y), _p(J) if jac else None]
                args[i] = None
                rcs.append(L.mppib_host_state_deriv_racer_rigid_suspension(*args))
                left += [xd, y, J]
    if m.kind == "dubins":
        fs, ft = L.mppib_host_step_racer_dubins_elevation, L.mppib_host_output_trajectory_racer_dubins_elevation
        for nulls in step_nulls:
            left += call_step(fs, _blob(m), _p(m.elev), nulls=nulls)
        left += call_step(fs, None, _p(m.elev))
        for nulls in traj_nulls:
            left += call_traj(ft, _blob(m), _p(m.elev), nulls=nulls)
        left += call_traj(ft, None, _p(m.elev))
        for steps in (0, -1, 1):
            left += call_traj(ft, _blob(m), _p(m.elev), steps=steps)
    if m.kind in ("lstm", "suspension"):
        if m.kind == "lstm":
            fs, ft, extra = L.mppib_host_step_lstm, L.mppib_host_output_trajectory_lstm, ()
        else:
            fs, ft = L.mppib_host_step_racer_suspension, L.mppib_host_output_trajectory_racer_suspension
            extra = (_p(m.normals),)
        nets = [m.net(hidden, cell) for _ in range(4)]
        nets[1].theta, nets[2].hidden, nets[3].cell = None, None, None
        for net in nets:
            left += call_step(fs, _blob(m), C.byref(net), *extra)
            left += call_traj(ft, _blob(m), C.byref(net), *extra)
        left += call_step(fs, _blob(m), None, *extra)
        left += call_step(fs, None, C.byref(nets[0]), *extra)
        left += call_traj(ft, _blob(m), None, *extra)
        left += call_traj(ft, None, C.byref(nets[0]), *extra)
        for nulls in step_nulls:
            left += call_step(fs, _blob(m), C.byref(nets[0]), *extra, nulls=nulls)
        for nulls in traj_nulls:
            left += call_traj(ft, _blob(m), C.byref(nets[0]), *extra, nulls=nulls)
        for steps in (0, -1, 1):
            left += call_traj(ft, _blob(m), C.byref(nets[0]), *extra, steps=steps)
        left += [hidden, cell]
    out[f"{m.name}.args.rc"] = np.asarray(rcs, np.int32)
    out[f"{m.name}.args.left"] = np.concatenate([b.ravel() for b in left])


def _generic_entries(L, ms, out):
    """mppib_host_dims / _enforce_constraints / _step / _output_trajectory for every id: return codes and buffers."""
    by_id = {}
    for m in ms:
        by_id.setdefault(m.dyn_id, m)
    zeros = np.zeros(512, np.uint8)
    rcs, left = [], []
    for i in IDS:
        m = by_id.get(i)
        blob = _blob(m) if m else zeros.ctypes.data
        nn = _p(m.nn) if m else None
        S_, C_, O_ = C.c_int(-7), C.c_int(-7), C.c_int(-7)
        rcs.append(L.mppib_host_dims(i, C.byref(S_), C.byref(C_), C.byref(O_)))
        rcs.append(L.mppib_host_dims(i, None, None, None))
        left.append(np.array([S_.value, C_.value, O_.value], f32))
        u = np.concatenate([m.u.ravel() if m else np.zeros(0, f32), _nan(8)])[:8].copy()
        rcs.append(L.mppib_host_enforce_constraints(i, blob, _p(u)))
        left.append(u)
        x = np.concatenate([m.x[0] if m else np.zeros(0, f32), np.ones(PAD, f32)])[:PAD].copy()
        uu = np.concatenate([m.u[0] if m else np.zeros(0, f32), np.ones(4, f32)])[:4].copy()
        xn, xd, y = _nan(PAD), _nan(PAD), _nan(PAD)
        rcs.append(L.mppib_host_step(i, blob, nn, _p(x), _p(uu), C.c_float(DT), _p(xn), _p(xd), _p(y)))
        left += [xn, xd, y]
        U = np.concatenate([m.U.ravel() if m else np.zeros(0, f32), np.ones(4 * T, f32)])[:4 * T].copy()
        st, op = _nan(T * PAD), _nan(T * PAD)
        rcs.append(L.mppib_host_output_trajectory(i, blob, nn, _p(x), _p(U), T, C.c_float(DT), _p(st), _p(op)))
        left += [st, op]
    out["generic.rc"] = np.asarray(rcs, np.int32)
    out["generic.left"] = np.concatenate(left)


def snapshot(L=None):
    """Everything the snapshot records, from the library `L` (default: the one mppi_generic_b200.host loads)."""
    L = L or H.lib()
    ms = models()
    out = {}
    for m in ms:
        # single steps
        res = []
        for k in range(NSTEP):
            if m.lstm is not None:
                h, c = m.hc[k][0].copy(), m.hc[k][1].copy()
                rc, xn, xd, y = step(L, m, m.x[k], m.u[k], h, c)
                res.append((rc, [xn, xd, y, h, c]))
            else:
                rc, xn, xd, y = step(L, m, m.x[k], m.u[k])
                res.append((rc, [xn, xd, y]))
            if m.kind in ("generic", "rigid"):
                rc, xn, xd, y = step(L, m, m.x[k], m.u[k], generic=True)
                res.append((rc, [xn, xd, y]))
        for k in range(NSTEP):
            u = m.u[k].copy()
            res.append((L.mppib_host_enforce_constraints(m.dyn_id, _blob(m), _p(u)), [u]))
        out[f"{m.name}.step.rc"] = np.asarray([r for r, _ in res], np.int32)
        out[f"{m.name}.step.out"] = np.concatenate([b for _, bufs in res for b in bufs])
        # roll-forward; an LSTM net's own hidden / cell must come back untouched
        if m.lstm is not None:
            h, c = m.hc[0][0].copy(), m.hc[0][1].copy()
            rc, st, op = trajectory(L, m, hidden=h, cell=c)
            extra = [h, c]
        else:
            rc, st, op = trajectory(L, m)
            extra = []
        rcs, bufs = [rc], [st.ravel(), op.ravel()] + extra
        if m.kind == "rigid":
            rc, st, op = trajectory(L, m, generic=True)
            rcs.append(rc)
            bufs += [st.ravel(), op.ravel()]
            for k in range(NSTEP):
                xd, y, J = _nan(14), _nan(26), _nan(9)
                for jac in (J, None):
                    rcs.append(L.mppib_host_state_deriv_racer_rigid_suspension(_blob(m), _p(m.x[k]), _p(m.u[k]), _p(xd),
                                                                               _p(y), _p(jac)))
                    bufs += [xd.copy(), y.copy()]
                bufs.append(J)
        out[f"{m.name}.trajectory.rc"] = np.asarray(rcs, np.int32)
        out[f"{m.name}.trajectory.out"] = np.concatenate(bufs)
        _argument_checks(L, m, out)
    _generic_entries(L, ms, out)
    return out


def main(path=None):
    # a directory of its own: tests/golden/*.npz are make_golden.py's vectors
    path = path or os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_twins", "snapshot.npz")
    out = snapshot()
    out["meta.x86_64_v3"] = np.asarray([cpu_runs_v3_clones()], np.int32)
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
