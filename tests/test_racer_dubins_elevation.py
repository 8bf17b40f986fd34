"""RacerDubinsElevation (MPPIB_DYN_RACER_DUBINS_ELEVATION) with RacerQuadraticCost: the host twin and the device model
against the reference's known answers and against the restatement in tests/racer_dubins_elevation_oracle.py, every K1
form, Tube-MPPI, RMPPI, init-eval, sampled trajectories, the device-side roll-forward and DDP feedback."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

import mppi_generic_b200 as m
from mppi_generic_b200 import workloads as W
from tests import ddp_oracle as DO
from tests import racer_dubins_elevation_oracle as RO

H = m.host
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KA = json.load(open(os.path.join(ROOT, "tests", "golden", "racer_dubins_elevation_known_answers.json")))


def _dyn_for(case):
    """The reference test's dynamics: default parameters with the case's overrides, default control ranges."""
    dyn = H.RacerDubinsElevation()
    for k, v in case["params"].items():
        if "[" in k:
            getattr(dyn.params, k[:-3])[int(k[-2])] = v
        else:
            setattr(dyn.params, k, type(getattr(dyn.params, k))(v))
    return dyn


def _state(case):
    x = np.zeros(19, np.float32)
    x[:len(case["state"])] = case["state"]
    return x


def _stale(case):
    """The reference's step tests predate two details of the source they test: they take 0.54 and 0.56 m/s (lines 353,
    385) in the first speed bin, which racer_dubins_elevation.cu:37-39 now ends at linear_brake_slope = 0.2, and they leave
    the brake state uncapped where :42 caps it at 0.25 (lines 516-604). In those cases the source's acceleration differs
    from the test's; every other value still holds."""
    x = case["state"]
    return 0.2 < abs(x[0]) < 0.6 or x[5] > 0.25


def _check_known(case, xn, xd, y, tol):
    for kind, i, want, line in case["expect"]:
        if _stale(case) and (kind == "accel_x" or i == RO.VEL_X):
            continue
        got = {"next_state": xn, "state_der": xd}[kind][i] if kind != "accel_x" else y[RO.O_ACCEL_X]
        assert abs(float(got) - want) <= tol, (case["test"], line, kind, i, float(got), want)


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_ids_and_blob_layout():
    assert H.DYN_RACER_DUBINS_ELEVATION == 5
    dyn = H.RacerDubinsElevation()
    assert dyn.blob() == bytes(H.RacerDubinsElevationLSTMSteering().params)  # the same RacerDubinsElevationParams
    S, Cd, O = C.c_int(), C.c_int(), C.c_int()
    assert H.lib().mppib_host_dims(5, C.byref(S), C.byref(Cd), C.byref(O)) == 0
    assert (S.value, Cd.value, O.value) == (19, 2, 28)


@pytest.mark.parametrize("body", ["host_twin", "host_restated", "device_restated"])
def test_reference_known_answers(body):
    """TestStep / TestStepReverse (racer_dubins_elevation_model_test.cu:305-606, :694-914): first nine states, their
    derivatives and ACCEL_X within the reference's 1e-6 (VEL_X rows of the stale cases aside, see _stale); the uncertainty
    entries start at zero."""
    assert sum(map(_stale, KA["cases"])) == 13  # of 27; their other rows are checked
    for case in KA["cases"]:
        dyn = _dyn_for(case)
        x, u = _state(case), np.asarray(case["control"], np.float32)
        if body == "host_twin":
            xn, xd, y = dyn.step(x, u, case["dt"])
        else:
            xn, xd, y = RO.step(RO.Params(dyn.params), x, u, case["dt"], "host" if body == "host_restated" else "device")
        _check_known(case, xn, xd, y, 1e-6 if body != "device_restated" else 2e-6)


def test_host_twin_equals_host_restatement():
    rng = np.random.RandomState(4)
    dyn = H.RacerDubinsElevation()
    dyn.setControlRanges([(-0.8, 1.0), (-1.0, 1.0)])
    p = RO.Params(dyn.params)
    for _ in range(300):
        x, u = _random_state(rng), rng.uniform(-1, 1, 2).astype(np.float32)
        a = dyn.step(x, u, 0.02)
        b = RO.step(p, x, u, 0.02, "host")
        for v, w in zip(a, b):
            np.testing.assert_allclose(np.nan_to_num(v), np.nan_to_num(w), rtol=2e-6, atol=2e-6)


def test_finite_500_step_trajectories():
    """ComputeStateTrajectoryFiniteTest (racer_dubins_elevation_model_test.cu:1005-1055) through the host twin."""
    dyn = H.RacerDubinsElevation()
    p = dyn.params
    p.c_t[0], p.c_b[0], p.c_v[0], p.c_0, p.wheel_base, p.steering_constant = 3.0, 0.2, 0.2, 0.2, 3.0, 1.0
    for steer, k in ((-0.000735827, 1.0), (-1.0, 0.5)):
        p.steering_constant = k
        x = np.zeros(19, np.float32)
        x[:5] = [0, 1.46919e-6, 0.0140179, 1.09739e-8, steer]
        for _ in range(500):
            xn, xd, _ = dyn.step(x, np.zeros(2, np.float32), 0.02)
            assert np.isfinite(xn).all() and np.isfinite(xd).all() and np.any(xd != 0)
            x = xn


def _random_state(rng):
    """Covers the three speed bins and the +-0.2 band, braking and reverse, steer-rate saturation and |pitch| > pi / 2."""
    x = np.zeros(19, np.float32)
    x[RO.VEL_X] = rng.choice([rng.uniform(-0.2, 0.2), rng.uniform(0.2, 3.0), rng.uniform(3.0, 8.0), rng.uniform(-6, -0.2)])
    x[RO.YAW] = rng.uniform(-math.pi, math.pi)
    x[RO.POS_X], x[RO.POS_Y] = rng.uniform(-20, 20, 2)
    x[RO.STEER_ANGLE] = rng.uniform(-0.6, 0.6)
    x[RO.BRAKE_STATE] = rng.uniform(0, 0.4)
    x[RO.ROLL] = rng.uniform(-0.3, 0.3)
    x[RO.PITCH] = rng.choice([rng.uniform(-0.5, 0.5), rng.uniform(1.6, 3.0) * rng.choice([-1, 1])])
    x[RO.STEER_ANGLE_RATE] = rng.uniform(-2, 2)
    diag = rng.uniform(1e-4, 0.1, 4)
    x[RO.UNC0:RO.UNC0 + 4] = diag
    x[RO.UNC0 + 4:RO.UNC0 + 10] = rng.uniform(-1e-4, 1e-4, 6)
    return x


def test_restatement_float32_against_float64():
    rng = np.random.RandomState(1)
    dyn = H.RacerDubinsElevation()
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    p = RO.Params(dyn.params)
    seen = set()
    for _ in range(400):
        x = _random_state(rng)
        u = np.array([rng.uniform(-1, 1), rng.choice([rng.uniform(-1, 1), rng.choice([-1.0, 1.0]) * 20.0])], np.float32)
        a = RO.step(p, x, u, 0.02, dtype=np.float32)
        b = RO.step(p, x, u, 0.02, dtype=np.float64)
        vx = abs(float(x[0]))
        seen.add(int(vx > 0.2) + int(vx > 3.0))
        seen.add("brake" if u[0] < 0 else "throttle")
        seen.add("reverse" if x[0] < 0 else "forward")
        seen.add("saturated" if abs((u[1] * p.steer_command_angle_scale - x[4]) * p.steering_constant) > p.max_steer_rate
                 else "linear")
        seen.add("steep" if abs(float(x[RO.PITCH])) > math.pi / 2 else "flat")
        for v32, v64 in zip(a, b):
            v32, v64 = np.nan_to_num(v32.astype(np.float64)), np.nan_to_num(v64)
            assert np.all(np.abs(v32 - v64) <= 2e-5 * np.maximum(1.0, np.abs(v64))), np.abs(v32 - v64).max()
    assert {0, 1, 2, "brake", "throttle", "reverse", "forward", "saturated", "linear", "steep", "flat"} <= seen


def test_host_minus_device_is_the_two_documented_differences():
    """Host and device bodies differ in (1) sin / tan / sincos without normalizeAngle and (2) the brake clamp: [0, 1] on
    the device, [0, -control_rngs_[0].x] on the host. With angles inside (-pi, pi] and the throttle's lower limit at -1 they
    agree; with another limit only the brake state differs, and only where the clamp is active."""
    rng = np.random.RandomState(2)
    dyn = H.RacerDubinsElevation()
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    p = RO.Params(dyn.params)
    for _ in range(200):
        x, u = _random_state(rng), rng.uniform(-1, 1, 2).astype(np.float32)
        x[RO.PITCH] = np.clip(x[RO.PITCH], -3.1, 3.1)
        hn, hd, hy = RO.step(p, x, u, 0.02, "host", np.float64)
        dn, dd, dy = RO.step(p, x, u, 0.02, "device", np.float64)
        np.testing.assert_allclose(hn, dn, rtol=1e-12, atol=1e-12)
    # angles outside (-pi, pi]: tan(delta) and sin(pitch) do not change under a 2 pi shift, sincos(yaw) neither
    x = _random_state(rng)
    x[RO.YAW] += 4 * math.pi
    hn, _, _ = RO.step(p, x, np.zeros(2, np.float32), 0.02, "host", np.float64)
    dn, _, _ = RO.step(p, x, np.zeros(2, np.float32), 0.02, "device", np.float64)
    np.testing.assert_allclose(hn[RO.POS_X:RO.POS_Y + 1], dn[RO.POS_X:RO.POS_Y + 1], rtol=1e-9, atol=1e-9)
    # the brake clamp: lower throttle limit -0.5 -> host caps the brake state at 0.5, the device at 1
    dyn.setControlRanges([(-0.5, 1.0), (-1.0, 1.0)])
    p = RO.Params(dyn.params)
    x = np.zeros(19, np.float32)
    x[RO.BRAKE_STATE] = 0.6
    u = np.array([-1.0, 0.0], np.float32)
    hn, _, _ = RO.step(p, x, u, 0.02, "host")
    dn, _, _ = RO.step(p, x, u, 0.02, "device")
    assert hn[RO.BRAKE_STATE] == np.float32(0.5) and dn[RO.BRAKE_STATE] > np.float32(0.5)
    same = np.arange(19) != RO.BRAKE_STATE
    np.testing.assert_allclose(hn[same], dn[same], rtol=1e-6, atol=1e-7)
    tw, _, _ = dyn.step(x, u, 0.02)
    assert tw[RO.BRAKE_STATE] == np.float32(0.5)


def test_gradient_restatement_and_central_differences():
    """computeGrad as restated, against float64 central differences of f in the interior: no clamp active, |vx| away
    from the bin edges. The kinematic rows (VEL_X, YAW, POS_X, POS_Y) agree there."""
    rng = np.random.RandomState(3)
    dyn = H.RacerDubinsElevation()
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    p = RO.Params(dyn.params)
    checked = 0
    for _ in range(400):
        x = _random_state(rng)
        x[RO.PITCH] = rng.uniform(-0.5, 0.5)
        x[RO.BRAKE_STATE] = 0.0
        u = np.array([rng.uniform(0.05, 1.0), rng.uniform(-0.1, 0.1)], np.float32)
        vx = abs(float(x[0]))
        if min(abs(vx - 0.2), abs(vx - 3.0)) < 0.05 or vx < 0.25:
            continue
        sd = (u[1] * p.steer_command_angle_scale - x[4]) * p.steering_constant
        if abs(sd) > p.max_steer_rate - 0.05:
            continue
        acc = p.c_t[int(vx > 3.0) + 1] * u[0] - p.c_v[int(vx > 3.0) + 1] * x[0] + p.c_0
        if abs(acc) > p.clamp_ax - 0.1:
            continue
        A, B = RO.grad(p, x, u, np.float64)
        J = np.zeros((19, 21))
        z = np.concatenate([x, u]).astype(np.float64)
        for j in range(21):
            h = 1e-5 * max(1.0, abs(z[j]))
            zp, zm = z.copy(), z.copy()
            zp[j] += h
            zm[j] -= h
            J[:, j] = (RO.f_ddp(p, zp[:19], zp[19:], np.float64) - RO.f_ddp(p, zm[:19], zm[19:], np.float64)) / (2 * h)
        rows = [RO.VEL_X, RO.YAW, RO.POS_X, RO.POS_Y]
        for r in rows:
            for j in range(21):
                if r == RO.VEL_X and j in (RO.BRAKE_STATE, RO.PITCH):  # brake term off at brake_state 0; pitch: sign below
                    continue
                ref = A[r, j] if j < 19 else B[r, j - 19]
                assert abs(J[r, j] - ref) <= 1e-4 * max(1.0, abs(ref)), (r, j, J[r, j], ref)
        # gravity row: d/dpitch of -g sin(pitch) is -g cos(pitch)
        assert abs(J[RO.VEL_X, RO.PITCH] - A[RO.VEL_X, RO.PITCH]) <= 1e-4 * max(1.0, abs(A[RO.VEL_X, RO.PITCH]))
        checked += 1
    assert checked > 50
    # the quirks as written: A(4,4) clamp, brake-command row on the throttle's lower limit
    x = np.zeros(19, np.float32)
    A, B = RO.grad(p, x, np.array([0.0, 0.0], np.float32))
    assert A[RO.STEER_ANGLE, RO.STEER_ANGLE] == np.float32(-p.steering_constant)
    A, B = RO.grad(p, x, np.array([0.0, 1.6], np.float32))  # steer_dot 4.8: inside the 0.01 margin, still linear
    assert A[RO.STEER_ANGLE, RO.STEER_ANGLE] == np.float32(-p.steering_constant)
    A, B = RO.grad(p, x, np.array([0.0, 1.665], np.float32))  # steer_dot 4.995: within 0.01 of the limit
    assert A[RO.STEER_ANGLE, RO.STEER_ANGLE] == 0
    A, B = RO.grad(p, x, np.array([0.0, 5.0], np.float32))  # saturated steering
    assert A[RO.STEER_ANGLE, RO.STEER_ANGLE] == 0
    x[RO.BRAKE_STATE] = 0.1
    A, B = RO.grad(p, x, np.array([-0.05, 0.0], np.float32))  # brake_dot = (0.05 - 0.1) 6.6 < 0, brake state < 1
    assert B[RO.BRAKE_STATE, 0] == np.float32(-p.brake_delay_constant)
    assert not A[6:].any() and not B[6:].any()


def test_workloads():
    for use_map in (False, True):
        w = W.racer_elevation(256, 20, use_map=use_map)
        assert w.dyn.DYN_ID == 5 and w.D == 1 and w.dyn.tex_helper_.checkTextureUse(0) == use_map
        t = W.racer_elevation_tube(256, 20, use_map=use_map)
        assert t.D == 2 and t.controller == "tube" and t.x0.shape == (2, 19) and t.U0.shape == (2, 20, 2)


def test_engine_rejects_weights_and_takes_the_map():
    """Blob rules without a device: the ids reach the device check (mppib_create fails only for the missing GPU)."""
    w = W.racer_elevation(256, 20)
    try:
        e = w.make_engine()
    except H.MppibError as err:
        assert "no kernel registered" not in str(err)
        pytest.skip("no GPU")
    L = H.lib()
    dummy = np.zeros(16, np.float32)
    assert L.mppib_set_blob(e._h, H.BLOB_LSTM_WEIGHTS, dummy.ctypes.data, dummy.nbytes) != 0
    assert L.mppib_set_blob(e._h, H.BLOB_NN_WEIGHTS, dummy.ctypes.data, dummy.nbytes) != 0
    m_ = w.dyn.tex_helper_.blob()
    assert L.mppib_set_blob(e._h, H.BLOB_ELEVATION_MAP, m_.ctypes.data, m_.nbytes) == 0
    e.close()


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _map_blob(w):
    return w.dyn.tex_helper_.blob() if w.dyn.tex_helper_.checkTextureUse(0) else None


def _restated_rollout(w, x0, controls):
    """Outputs [T][O] and the trajectory cost (sum of RacerQuadraticCost over the T steps, / T) of one sample, controls
    clamped to the model's ranges like enforceConstraints."""
    p = RO.Params(w.dyn.params)
    lo, hi = np.array(p.rng_lo, np.float32), np.array(p.rng_hi, np.float32)
    cp = w.cost.params
    mb = _map_blob(w)
    x = np.asarray(x0, np.float32)
    Y = np.zeros((w.T, 28), np.float32)
    steps = np.zeros(w.T, np.float32)
    for t in range(w.T):
        u = np.minimum(np.maximum(controls[t], lo), hi).astype(np.float32)
        x, _, y = RO.step(p, x, u, w.dt, "device", np.float32, mb)
        Y[t] = y
        f = np.float32
        dv = f(y[0] - f(cp.desired_speed))
        dyaw = RO.normalize_angle(f(y[5] - f(cp.desired_yaw)), np.float32)
        dy = f(y[3] - f(cp.desired_y))
        steps[t] = (f(cp.speed_coeff) * dv * dv + f(cp.yaw_coeff) * dyaw * dyaw + f(cp.lateral_coeff) * dy * dy +
                    f(cp.steer_coeff) * y[8] * y[8])
    run = np.float32(0)
    for v in steps:
        run = np.float32(run + v)
    return Y, run / np.float32(w.T), steps


def _on_discontinuity(w, Y_a, Y_b, t):
    """A speed-bin edge (|vx| at 0.2 / 3), brake enable (throttle command at 0) or an elevation-map texel edge at step t or
    the step before it, on either trajectory."""
    for Y in (Y_a, Y_b):
        for k in (t - 1, t):
            if k < 0:
                continue
            vx = abs(float(Y[k][0]))
            if min(abs(vx - 0.2), abs(vx - 3.0)) < 2e-3:
                return True
            tex = w.dyn.tex_helper_
            if _map_blob(w) is not None:
                res, org = tex.hdr.resolution[0], tex.hdr.origin
                for c, o in ((Y[k][2], org[0]), (Y[k][3], org[1])):
                    # the four wheel contacts lie within 3 m of the base: any of them may sit on an edge
                    for off in np.linspace(-3.0, 3.0, 61):
                        q = (c + off - o) / res - 0.5
                        if abs(q - round(q)) < 2e-3:
                            return True
    return False


def _parity(w, c, controls, x0, dump, idx, tol=1e-4, brake_u=None):
    """Per-sample costs c[idx] within `tol` of the restatement, or, for each outlier, the device's own dump sums to its
    cost and the first step that differs sits on a discontinuity."""
    rel_all = []
    outliers = []
    for n in idx:
        Y, ref, _ = _restated_rollout(w, x0, controls[n])
        rel = abs(float(c[n]) - float(ref)) / max(abs(float(ref)), 1.0)
        rel_all.append(rel)
        if rel > tol:
            outliers.append((n, Y))
    assert len(outliers) <= 0.03 * len(idx), (len(outliers), max(rel_all))
    assert np.median(rel_all) < 1e-5
    if outliers:
        ix = np.array([o[0] for o in outliers])
        outs_dev, costs_dev, _ = dump(ix)
        np.testing.assert_allclose(costs_dev.sum(axis=1), c[ix], rtol=5e-6)
        for k, (n, Y) in enumerate(outliers):
            d = np.abs(np.nan_to_num(outs_dev[k][:, :10]) - np.nan_to_num(Y[:, :10])).max(axis=1)
            bad = np.nonzero(d > 1e-4)[0]
            if bad.size == 0:
                continue
            u0 = controls[n][:, 0]
            near_zero = np.abs(u0[max(0, bad[0] - 1):bad[0] + 1]) < 1e-5
            assert near_zero.any() or _on_discontinuity(w, outs_dev[k], Y, int(bad[0])), (n, int(bad[0]))
    return len(outliers)


def _wide(w, std=(0.6, 0.6)):
    w.sampler.setStdDev(list(std))
    w.sampler.setControlCostCoeff([0.0, 0.0])
    return w


FORMS = [("resident", 0, {}), ("no_tma", H.FLAG_NO_TMA, {}), ("stream", 0, {"MPPIB_STREAM": "1"}),
         ("bx64", 0, {"MPPIB_BX": "64"}), ("bx128", 0, {"MPPIB_BX": "128"})]


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 2], ids=["D1", "D2"])
@pytest.mark.parametrize("use_map", [False, True], ids=["map_off", "map_on"])
@pytest.mark.parametrize("name,flags,env", FORMS, ids=[f[0] for f in FORMS])
def test_k1_forms_match_the_restatement(name, flags, env, use_map, D, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    w = _wide(W.racer_elevation_tube(2048, 40, use_map) if D == 2 else W.racer_elevation(2048, 40, use_map))
    if D == 2:
        w.x0[1, :4] += np.array([0.3, 0.1, 0.5, -0.4], np.float32)
    e = w.make_engine(flags=flags | H.FLAG_WRITEBACK_CONTROLS)
    info = e.launch_info()
    if name == "no_tma":
        assert not info["uses_tma"]
    if name.startswith("bx"):
        assert info["block"] == int(env["MPPIB_BX"])
    e.solve(w.x0, w.U0)
    c, samples = e.get_costs(), e.get_samples()
    for d in range(D):
        idx = np.random.RandomState(d).choice(w.N, 150, replace=False)
        _parity(w, c[d], samples[d], w.x0[d],
                lambda ix, d=d: e.sample_trajectories(w.x0[d], w.U0[d], ix, distribution=d), idx)
    e.close()


@pytest.mark.gpu
def test_device_step_at_the_known_answers():
    """The device step (through the device-side roll-forward, whose step 1 is one model step) at the reference's
    known-answer states: the restated device body within 1e-5, the reference's values within 2e-5 (device sin / tan)."""
    groups = {}
    for case in KA["cases"]:
        groups.setdefault((json.dumps(case["params"], sort_keys=True), case["dt"]), []).append(case)
    for (_, dt), cases in groups.items():
        dyn = _dyn_for(cases[0])
        sampler = H.GaussianDistribution(2, [0.1, 0.1])
        e = H.Engine(dyn, H.RacerQuadraticCost(), sampler, 256, 2, 1)
        e.set_solver(dt, 1.0, 0.0)
        for case in cases:
            x0 = _state(case)[None]
            U = np.tile(np.asarray(case["control"], np.float32), (1, 2, 1))
            _, states, outputs = e.nominal_trajectory(x0, U)
            xn, y = states[0, 1], outputs[0, 1]
            rn, rd, ry = RO.step(RO.Params(dyn.params), x0[0], U[0, 0], dt, "device")
            np.testing.assert_allclose(xn, rn, rtol=1e-5, atol=1e-5)
            _check_known(case, xn, rd, y, 2e-5)
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("use_map", [False, True], ids=["map_off", "map_on"])
def test_sampled_trajectories_sum_to_k1_and_u(use_map):
    w = _wide(W.racer_elevation(2048, 40, use_map))
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    U, _ = e.solve(w.x0, w.U0)
    c, samples = e.get_costs()[0], e.get_samples()[0]
    idx = np.arange(0, w.N, 16)
    outs, costs, _ = e.sample_trajectories(w.x0[0], w.U0[0], idx)
    np.testing.assert_allclose(costs.sum(axis=1), c[idx], rtol=5e-6)
    for k, n in enumerate(idx[:40]):
        Y, _, _ = _restated_rollout(w, w.x0[0], samples[n])
        assert np.abs(outs[k][:, :4] - Y[:, :4]).max() < 2e-3
    cc = c.astype(np.float64)
    wts = np.exp(-(cc - cc.min()) / w.lambda_)
    u64 = np.tensordot(wts / wts.sum(), samples.astype(np.float64), axes=1)
    np.testing.assert_allclose(U[0], u64, atol=2e-4)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("use_map", [False, True], ids=["map_off", "map_on"])
def test_tube_two_systems_agree(use_map):
    """runRolloutKernelOnMultipleSystems (the reference's rollout kernel test): in one D = 2 engine, two systems with the
    same x0 and U roll out the same costs, and the solve returns the same U for both."""
    w = W.racer_elevation_tube(4096, 50, use_map)
    assert np.array_equal(w.x0[0], w.x0[1]) and np.array_equal(w.U0[0], w.U0[1])
    e = w.make_engine()
    U, _ = e.solve(w.x0, w.U0)
    c = e.get_costs()
    e.close()
    np.testing.assert_array_equal(c[0], c[1])
    np.testing.assert_array_equal(U[0], U[1])


def _reroll(w, x0, controls):
    N = controls.shape[0]
    sampler = H.GaussianDistribution(2, [1.0, 1.0])
    e = H.Engine(w.dyn, w.cost, sampler, N + 1, w.T, 1, flags=H.FLAG_WRITEBACK_CONTROLS)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    eps = np.concatenate([np.zeros((1, w.T, 2), np.float32), controls]).astype(np.float32)
    e.set_noise(eps)
    zeros = np.zeros((1, w.T, 2), np.float32)
    e.rollout_only(x0[None], zeros, 0, 0)
    np.testing.assert_array_equal(e.get_samples()[0][1:], controls)
    return e, e.get_costs()[0][1:], lambda ix: e.sample_trajectories(x0, zeros[0], np.asarray(ix) + 1)


@pytest.mark.gpu
@pytest.mark.parametrize("with_gains", [False, True], ids=["no_gains", "gains"])
def test_rmppi_rollouts_match(with_gains):
    w = _wide(W.racer_elevation(1024, 40))
    thr = 200.0
    e = H.Engine(w.dyn, w.cost, w.sampler, w.N, w.T, 2, flags=H.FLAG_RMPPI)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    e.seed(w.seed, 0)
    gains = (np.random.RandomState(3).randn(w.T, 19, 2) * 0.05).astype(np.float32) if with_gains else None
    e.set_rmppi(thr, gains)
    x0 = np.stack([w.x0[0], w.x0[0] + np.array([0.2, 0.05, 0.1, -0.1] + [0.0] * 15, np.float32)])
    U_in = np.tile(w.U0, (2, 1, 1))
    e.draw_noise()
    e.rollout_only(x0, U_in, 1, 0)
    c, applied = e.get_costs(), e.get_samples()
    costs = []
    for d in range(2):
        r, v, dump = _reroll(w, x0[d], applied[d])
        idx = np.random.RandomState(d).choice(w.N, 120, replace=False)
        _parity(w, v, applied[d], x0[d], dump, idx)
        costs.append(v)
        r.close()
    c_nom, c_real = costs
    np.testing.assert_allclose(c[1], c_real, rtol=1e-6, atol=0)
    nom = (np.float32(0.5) * c_nom + np.float32(0.5) * np.maximum(np.minimum(c[1], np.float32(thr)), c_nom)).astype(np.float32)
    np.testing.assert_allclose(c[0], nom, rtol=1e-6, atol=0)
    e.close()


@pytest.mark.gpu
def test_init_eval_matches():
    import oracle
    w = _wide(W.racer_elevation(512, 30))
    e = H.Engine(w.dyn, w.cost, w.sampler, w.N, w.T, 2, flags=H.FLAG_RMPPI)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    e.seed(w.seed, 0)
    e.set_rmppi(200.0, None)
    x0 = np.stack([w.x0[0], w.x0[0] + np.array([0.3, 0.2, 0.1] + [0.0] * 16, np.float32)])
    U_in = np.tile(w.U0, (2, 1, 1))
    e.draw_noise()
    e.rollout_only(x0, U_in, 1, 0)
    K, spc, stride = 3, 64, 2
    cand = np.stack([x0[0], 0.5 * (x0[0] + x0[1]), x0[1]]).astype(np.float32)
    strides = np.array([0, 1, 2], np.int32)
    got = e.init_eval(cand, strides, spc, U_in[0], stride)
    ctl = e.get_noise()[None].copy()
    oracle.set_gaussian_controls(U_in[:1], w.sampler.params, ctl, 2, w.T, w.N, 1, stride, 0)
    ctl = ctl[0, :spc]
    bad = 0
    for k in range(K):
        idx = np.minimum(np.arange(w.T) + strides[k], w.T - 1)
        want = np.array([_restated_rollout(w, cand[k], ctl[n][idx])[1] for n in range(spc)], np.float32)
        rel = np.abs(got[k * spc:(k + 1) * spc] - want) / np.maximum(np.abs(want), 1.0)
        bad += int((rel > 1e-4).sum())
    assert bad <= 0.03 * K * spc, bad
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("use_map", [False, True], ids=["map_off", "map_on"])
def test_device_tail_matches_the_host_twin(use_map):
    """The device-side nominal roll-forward against the host twin: equal up to the two documented body differences,
    which these states do not reach (angles in range, throttle lower limit -1), and the device's fast sin / tan."""
    w = W.racer_elevation_tube(2048, 60, use_map)
    e = w.make_engine()
    U, _ = e.solve(w.x0, w.U0)
    _, st_d, out_d = e.nominal_trajectory(w.x0, U)
    e.close()
    for d in range(2):
        st_h = np.zeros((w.T, 19), np.float32)
        out_h = np.zeros((w.T, 28), np.float32)
        w.dyn.output_trajectory(w.x0[d], U[d], w.T, w.dt, st_h, out_h)
        for a, b in ((st_d[d], st_h), (out_d[d], out_h)):
            nan = np.isnan(b)
            assert np.array_equal(np.isnan(a), nan)
            a, b = np.where(nan, 0.0, a), np.where(nan, 0.0, b)
            scale = np.maximum(np.abs(b).max(axis=0, keepdims=True), 1.0)
            assert (np.abs(a - b) / scale).max() < 1e-4, float((np.abs(a - b) / scale).max())


def _ddp_model(dyn):
    """tests/ddp_oracle.py's solver with this model's f and computeGrad restatement."""
    mdl = DO.Model.__new__(DO.Model)
    mdl.id, mdl.S, mdl.C = dyn.DYN_ID, 19, 2
    mdl.u_lo = np.array([dyn.params.lim.rng_lo[i] for i in range(2)], np.float32)
    mdl.u_hi = np.array([dyn.params.lim.rng_hi[i] for i in range(2)], np.float32)
    mdl.p = RO.Params(dyn.params)
    return mdl


@pytest.fixture
def racer_ddp_oracle(monkeypatch):
    f0, g0 = DO.f, DO.grad
    monkeypatch.setattr(DO, "f", lambda mdl, x, u, dtype=np.float32: RO.f_ddp(mdl.p, x, u, dtype) if mdl.id == 5
                        else f0(mdl, x, u, dtype))
    monkeypatch.setattr(DO, "grad", lambda mdl, x, u, dtype=np.float32: RO.grad(mdl.p, x, u, dtype) if mdl.id == 5
                        else g0(mdl, x, u, dtype))


@pytest.mark.gpu
def test_device_jacobians_match_the_restatement():
    rng = np.random.RandomState(5)
    w = W.racer_elevation(1024, 20, use_map=False)
    e = w.make_engine()
    p = RO.Params(w.dyn.params)
    for _ in range(24):
        x, u = _random_state(rng), rng.uniform(-1, 1, 2).astype(np.float32)
        _, _, _, jac = e.ddp_feedback(x, np.stack([x, x]), np.stack([u, u]), want_jacobians=True)
        A, B = RO.grad(p, x, u)
        ref = np.concatenate([A, B], axis=1)
        assert np.abs(jac[0] - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max())
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [1, 3])
def test_device_ddp_matches_the_restatement(iters, racer_ddp_oracle):
    T, dt = 60, 0.02
    w = W.racer_elevation(1024, T, use_map=False)
    mdl = _ddp_model(w.dyn)
    x0 = w.x0[0].copy()
    ut = np.tile(np.array([0.3, 0.05], np.float32), (T, 1))
    xt = np.zeros((T, 19), np.float32)
    xt[0] = x0
    for i in range(1, T):
        xt[i] = xt[i - 1] + DO.f(mdl, xt[i - 1], ut[i - 1]) * np.float32(dt)
    x0 = (x0 + np.array([0.2, 0.05, 0.1, -0.1] + [0.0] * 15, np.float32)).astype(np.float32)
    Q = np.diag([5, 20, 10, 10, 1, 0.1] + [0.0] * 13).astype(np.float32)
    Qf = (5 * Q).astype(np.float32)
    R = np.diag([1.0, 1.0]).astype(np.float32)
    e = H.Engine(w.dyn, w.cost, w.sampler, 1024, T, 1)
    e.set_solver(dt, 1.0, 0.0)
    e.set_ddp(Q, Qf, R, iters)
    gains, xs, us = e.ddp_feedback(x0, xt, ut)
    e.close()
    ref = DO.ddp_run(mdl, dt, x0, xt, ut, Q, Qf, R, iters)
    per_step = np.maximum(np.abs(ref["gains"]).max(axis=(1, 2)), 1e-6)
    err = np.abs(gains - ref["gains"]).max(axis=(1, 2)) / per_step
    assert err[:-1].max() <= 1e-3, float(err.max())
    assert np.abs(xs - ref["x"]).max() <= 1e-3 * max(1.0, np.abs(ref["x"]).max())
    assert np.abs(us - ref["u"]).max() <= 1e-3 * max(1.0, np.abs(ref["u"]).max())


def _feedback_params():
    p = H.DDPParams(19, 2)
    p.Q = np.diag([20, 30, 5, 5, 1, 0.1] + [0.0] * 13).astype(np.float32)
    p.Q_f = p.Q.copy()
    p.R = np.diag([1.0, 1.0]).astype(np.float32)
    return p


def _disturb(x, rng, dt):
    x = x.copy()
    x[RO.VEL_X] += np.float32(0.3 * math.sqrt(dt) * rng.randn())
    x[RO.YAW] += np.float32(0.05 * math.sqrt(dt) * rng.randn())
    return x


TARGET = 1.4  # m/s: above what a coasting vehicle holds over the map (0.87 m/s), below full throttle's 1.55 m/s


def _closed_loop_workload(w):
    """The closed loops track TARGET with the speed term weighted up, so that holding the target takes throttle."""
    w.cost.params.desired_speed = TARGET
    w.cost.params.speed_coeff = 20.0
    return w


def _coasting_mean_speed(w):
    """Mean speed over the same window with zero control and the same pushes: what a loop that does not track settles at."""
    x = w.x0[0].copy()
    rng = np.random.RandomState(0)
    speeds = []
    for t in range(150):
        x, _, _ = w.dyn.step(x, np.zeros(2, np.float32), w.dt)
        x = _disturb(x, rng, w.dt)
        speeds.append(float(x[0]))
    return float(np.mean(speeds[50:]))


def _check_loop(speeds, yaws, w):
    mean, coast = float(np.mean(speeds[50:])), _coasting_mean_speed(w)
    print(f"closed loop: mean speed {mean:.3f} (coasting {coast:.3f}), range {min(speeds[50:]):.3f} .. "
          f"{max(speeds[50:]):.3f}, max |yaw| {float(np.abs(np.array(yaws[50:])).max()):.3f}")
    assert abs(mean - TARGET) < 0.3, (mean, coast)
    assert abs(mean - TARGET) < 0.5 * abs(coast - TARGET), (mean, coast)
    assert np.abs(np.array(speeds[50:]) - TARGET).max() < 0.4, (min(speeds[50:]), max(speeds[50:]))
    assert np.abs(np.array(yaws[50:])).max() < 0.2, float(np.abs(np.array(yaws[50:])).max())


@pytest.mark.gpu
def test_tube_closed_loop_holds_speed_and_heading():
    """Tube-MPPI with DDP gains over the elevation map, under a random push on speed and heading every step: after 1 s
    the mean speed is within 0.3 m/s of the target and its error less than half a coasting vehicle's, every speed within
    0.4 m/s of it, and the heading within 0.2 rad of 0. On an H100 the Tube loop held a mean of 1.18 m/s and the RMPPI
    loop 1.17 m/s, where coasting gives 0.87 m/s: the hills and the cost's other terms leave a steady offset below the
    target."""
    w = _closed_loop_workload(W.racer_elevation_tube(2048, 50))
    ctrl = m.TubeMPPIController(w.dyn, w.cost, None, w.sampler, w.dt, 3, w.lambda_, w.alpha, w.T, w.N, seed=7,
                                nominal_threshold=20.0)
    ctrl.setFeedbackParams(_feedback_params())
    ctrl.initFeedback()
    x = w.x0[0].copy()
    rng = np.random.RandomState(0)
    speeds, yaws = [], []
    for t in range(150):
        ctrl.computeControl(x, 1)
        ctrl.computeFeedback(x)
        u = ctrl.getCurrentControl(x, 0.0, ctrl.getTargetStateSeq()[0], ctrl.getControlSeq()).astype(np.float32)
        w.dyn.enforceConstraints(x, u)
        x, _, _ = w.dyn.step(x, u, w.dt)
        x = _disturb(x, rng, w.dt)
        ctrl.slideControlSequence(1)
        speeds.append(float(x[0]))
        yaws.append(float(x[1]))
    assert ctrl.getFeedbackEnabled()
    _check_loop(speeds, yaws, w)


@pytest.mark.gpu
def test_rmppi_closed_loop_holds_speed_and_heading():
    """RMPPI with DDP gains, the same scenario and bars as the Tube loop."""
    w = _closed_loop_workload(W.racer_elevation(2048, 50))
    ctrl = H.RobustMPPIController(w.dyn, w.cost, None, w.sampler, w.dt, 1, w.lambda_, w.alpha, 20.0, w.T, w.N, seed=3,
                                  num_candidate_nominal_states=9, eval_samples_per_candidate=64)
    ctrl.setFeedbackParams(_feedback_params())
    ctrl.initFeedback()
    x = w.x0[0].copy()
    rng = np.random.RandomState(1)
    speeds, yaws = [], []
    for t in range(150):
        ctrl.updateImportanceSamplingControl(x, 1)
        ctrl.computeControl(x, 1)
        xn = ctrl.getNominalStateSeq()[0]
        u = (ctrl.getNominalControlSeq()[0] + ctrl.getFeedbackControl(x, xn, 0)).astype(np.float32)
        w.dyn.enforceConstraints(x, u)
        x, _, _ = w.dyn.step(x, u, w.dt)
        x = _disturb(x, rng, w.dt)
        speeds.append(float(x[0]))
        yaws.append(float(x[1]))
    _check_loop(speeds, yaws, w)


# ---- the C++ layer ---------------------------------------------------------------------------------------------------
LIB_DIR = os.path.join(ROOT, "mppi-generic_b200")
CPP_EXE = os.path.join(ROOT, "tests", "cpp", "racer_elevation_example.bin")


def _build_cpp():
    import subprocess
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unused-variable", "-I", os.path.join(ROOT, "include"),
                           "-c", os.path.join(ROOT, "tests", "cpp", "racer_elevation_example.cpp"), "-o", CPP_EXE + ".o"])
    subprocess.check_call(["g++", CPP_EXE + ".o", "-o", CPP_EXE, "-L", LIB_DIR, "-lmppi_b200", "-Wl,-rpath," + LIB_DIR])


def test_cpp_blob_and_grad_match_python():
    """RacerDubinsElevation (C++, built with plain g++ against the reference's include path) and the Python class write
    the same parameter bytes for the same settings, and their host computeGrad agree (and match the restatement)."""
    import subprocess
    _build_cpp()
    out = subprocess.check_output([CPP_EXE, "blob"])
    dyn = H.RacerDubinsElevation()
    dyn.params.c_t[1], dyn.params.wheel_base = 2.75, 0.35
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    n = C.sizeof(H.RacerLSTMDynParams)
    assert out[:n] == dyn.blob()
    J = np.frombuffer(out[n:], np.float32).reshape(19, 21)
    x = np.zeros(19, np.float32)
    x[0], x[1], x[4], x[7] = 1.5, 0.3, 0.1, 0.05
    u = np.array([0.4, 0.1], np.float32)
    A, B = dyn.computeGrad(x, u)
    np.testing.assert_array_equal(J, np.concatenate([A, B], axis=1))
    Ar, Br = RO.grad(RO.Params(dyn.params), x, u)
    np.testing.assert_allclose(np.concatenate([A, B], axis=1), np.concatenate([Ar, Br], axis=1), rtol=1e-6, atol=1e-6)


def test_cpp_example_links_against_the_library():
    """nm: the example's object needs the model's host twins and the controllers' C ABI, and libmppi_b200.so defines
    them; without a device the example stops at the C ABI's NO_DEVICE error (exit code 5)."""
    import subprocess
    _build_cpp()
    und = subprocess.run(["nm", "--undefined-only", CPP_EXE + ".o"], capture_output=True, text=True, check=True).stdout
    lib = subprocess.run(["nm", "-D", "--defined-only", os.path.join(LIB_DIR, "libmppi_b200.so")], capture_output=True,
                         text=True, check=True).stdout
    for sym in ("mppib_host_step_racer_dubins_elevation", "mppib_host_grad_racer_dubins_elevation",
                "mppib_host_output_trajectory_racer_dubins_elevation", "mppib_ddp_feedback", "mppib_create"):
        assert sym in und and sym in lib, sym
    p = subprocess.run([CPP_EXE], capture_output=True, text=True, timeout=900)
    if p.returncode == 5:
        assert "no CUDA device" in p.stdout
    else:
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]


@pytest.mark.gpu
def test_cpp_example_runs_tube_rmppi_and_ddp_on_the_gpu():
    import subprocess
    _build_cpp()
    p = subprocess.run([CPP_EXE], capture_output=True, text=True, timeout=900)
    print(p.stdout)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "racer elevation example rc 0" in p.stdout
