"""RacerSuspension (MPPIB_DYN_RACER_SUSPENSION), the rigid-body RACER vehicle, with RacerQuadraticCost at its output
indices: the blob, the host twin against the restatement in tests/racer_rigid_suspension_oracle.py and the reference's
OmegaJacobian case, closed-form physics, the device step, K1 on Vanilla / Tube / RMPPI and three samplers, the side
rollouts, DDP's refusal, a closed loop and the C++ layer."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import mppi_generic_b200 as m
from mppi_generic_b200 import workloads as W
from tests import racer_rigid_suspension_oracle as RO

H = m.host
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_DIR = ROOT + "/mppi-generic_b200"
CPP_SRC = ROOT + "/tests/cpp/racer_rigid_suspension_example.cpp"
CPP_EXE = ROOT + "/tests/cpp/racer_rigid_suspension_example.bin"


def _rest_state(dyn):
    x = dyn.getZeroState()
    x[RO.P_I_Z] = dyn.restHeight()
    return x


def _random_states(dyn, rng, n):
    """Upright-ish cars near their equilibrium height, moving and turning: every spring loaded (no wheel lift)."""
    x = np.tile(_rest_state(dyn), (n, 1))
    x[:, 0:2] = rng.uniform(-20, 20, (n, 2))
    x[:, RO.P_I_Z] += rng.uniform(-0.04, 0.04, n)
    half = rng.uniform(-0.05, 0.05, (n, 3))
    yaw = rng.uniform(-math.pi, math.pi, n)
    q = np.stack([np.cos(yaw / 2), half[:, 0], half[:, 1], np.sin(yaw / 2)], -1)
    x[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    x[:, 7:9] = rng.uniform(-6, 6, (n, 2))
    x[:, 9] = rng.uniform(-0.3, 0.3, n)
    x[:, 10:13] = rng.uniform(-0.3, 0.3, (n, 3))
    x[:, RO.STEER_ANGLE] = rng.uniform(-0.4, 0.4, n)
    u = rng.uniform(-1, 1, (n, 2)).astype(np.float32)
    return x.astype(np.float32), u


def _away_from_switches(p, x, u, band=1e-3):
    """Samples whose restated derivative is at least `band` (relative) away from the spring clamp and the Stribeck
    saturation, and whose braking samples have |vel_x| >= band."""
    _, _, mg = RO.deriv(p, x, u)
    return (mg["spring"] > band) & (mg["slip"] > band) & (mg["vel_x"] > band)


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_ids_blob_layout_and_defaults():
    assert H.DYN_RACER_SUSPENSION == 7
    assert C.sizeof(H.RacerRigidSuspensionDynParams) == 244
    assert H.RacerRigidSuspensionDynParams.Jxx.offset == 64 + 33 * 4
    S, Cd, O = C.c_int(), C.c_int(), C.c_int()
    assert H.lib().mppib_host_dims(7, C.byref(S), C.byref(Cd), C.byref(O)) == 0
    assert (S.value, Cd.value, O.value) == (14, 2, 26)
    p = H.RacerSuspension().params
    f = np.float32
    assert (f(p.wheel_radius), f(p.mass), f(p.wheel_base), f(p.gravity), f(p.mu), f(p.v_slip)) == \
        (f(0.32), f(1447), f(2.981), f(-9.81), f(0.65), f(0.1))
    assert (f(p.c_t), f(p.c_b), f(p.c_v), f(p.c_0), f(p.steering_constant), f(p.steer_command_angle_scale)) == \
        (f(3), f(10), f(0.2), f(0), f(0.6), f(-2.45))
    # recalcParams (racer_suspension.cuh:113-127) in the reference's types: float expressions, inertias in double
    wb, w, h, m_, g = f(2.981), f(1.5), f(1.5), f(1447), f(-9.81)
    assert list(p.cg_pos_wrt_base_link) == [wb / f(2), 0.0, f(0.2)]
    assert all(f(p.l_0[i]) == f(0.32) + m_ / f(4) * -g / f(14000) for i in range(4))
    assert [list(p.wheel_pos_wrt_base_link[i]) for i in range(4)] == \
        [[wb, w / f(2), 0], [wb, -w / f(2), 0], [0, w / f(2), 0], [0, -w / f(2), 0]]
    assert f(p.Jxx) == f(1.0 / 12 * float(m_) * float(h * h + w * w))
    assert f(p.Jyy) == f(1.0 / 12 * float(m_) * float(h * h + wb * wb))
    assert f(p.Jzz) == f(1.0 / 12 * float(m_) * float(wb * wb + w * w))
    # a changed base field reaches the derived ones only through recalcParams
    p.mass = 1000.0
    assert f(p.l_0[0]) != f(0.32) + f(1000) / f(4) * -g / f(14000)
    p.recalcParams()
    assert f(p.l_0[0]) == f(0.32) + f(1000) / f(4) * -g / f(14000)


def test_host_twin_matches_the_host_restatement():
    """computeStateDeriv, omegaJacobian (as written) and the implicit host step against the float64 restatement, at
    random states away from the switches."""
    dyn = H.RacerSuspension()
    p = RO.params(dyn.params)
    x, u = _random_states(dyn, np.random.RandomState(1), 400)
    keep = _away_from_switches(p, x, u)
    assert keep.sum() > 200
    for xi, ui in zip(x[keep], u[keep]):
        xd, y, J = dyn.computeStateDeriv(xi, ui, omega_jacobian=True)
        rd, ry, _, rJ = RO.deriv(p, xi, ui, jac=True)
        np.testing.assert_allclose(xd, rd, rtol=1e-4, atol=2e-3)
        np.testing.assert_allclose(y, ry, rtol=1e-4, atol=1e-3)
        np.testing.assert_allclose(J, rJ, rtol=1e-4, atol=1e-2)
        xn, xd2, y2 = dyn.step(xi, ui, 0.01)
        rn, _, _ = RO.host_step(p, xi, ui, 0.01)
        np.testing.assert_array_equal(xd2, xd)
        np.testing.assert_array_equal(y2, y)
        np.testing.assert_allclose(xn, rn, rtol=1e-5, atol=2e-5)
        assert abs(np.linalg.norm(xn[3:7].astype(np.float64)) - 1.0) < 1e-6


def test_restatement_float32_against_float64():
    dyn = H.RacerSuspension()
    p = RO.params(dyn.params)
    x, u = _random_states(dyn, np.random.RandomState(2), 300)
    keep = _away_from_switches(p, x, u)
    a, ya, _ = RO.deriv(p, x[keep], u[keep], np.float32)
    b, yb, _ = RO.deriv(p, x[keep], u[keep], np.float64)
    np.testing.assert_allclose(a, b, rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(ya, yb, rtol=1e-4, atol=1e-3)


def test_reference_omega_jacobian_case():
    """racer_suspension_model_test.cu:108-143: the analytic omegaJacobian against forward differences of w_dot, delta
    0.001, abs_tol 2."""
    dyn = H.RacerSuspension()
    x = np.zeros(14, np.float32)
    x[3], x[10], x[11], x[12], x[7] = 1, 0.1, -0.03, 0.02, 2
    u = np.zeros(2, np.float32)
    xd0, _, J = dyn.computeStateDeriv(x, u, omega_jacobian=True)
    for i in range(3):
        x1 = x.copy()
        x1[10 + i] += np.float32(0.001)
        xd1, _ = dyn.computeStateDeriv(x1, u)
        fd = (xd1[10:13] - xd0[10:13]) / np.float32(0.001)
        for r in range(3):
            assert abs(float(J[r, i]) - float(fd[r])) <= 2.0, (r, i, J[r, i], fd[r])


def test_at_rest_at_the_equilibrium_height_nothing_moves():
    dyn = H.RacerSuspension()
    xd, y = dyn.computeStateDeriv(_rest_state(dyn), np.zeros(2, np.float32))
    assert np.abs(xd).max() < 1e-4, xd
    wf = y[19:23]
    np.testing.assert_allclose(wf, 1447 * 9.81 / 4, rtol=1e-5)
    assert y[0] == y[1] == y[2] == 0 and y[23] == y[24] == y[25] == 0


def test_free_fall_and_a_spin_about_a_principal_axis():
    dyn = H.RacerSuspension()
    x = dyn.getZeroState()
    x[RO.P_I_Z] = 30.0
    x[7], x[9] = 1.5, -2.0
    for axis in range(3):
        xs = x.copy()
        xs[10 + axis] = 0.7
        xd, y = dyn.computeStateDeriv(xs, np.array([0.5, 0.3], np.float32))
        assert np.all(y[19:23] == 0)  # every spring slack: no wheel force
        assert xd[9] == np.float32(-9.81) and xd[7] == 0 and xd[8] == 0
        np.testing.assert_array_equal(xd[10:13], 0)  # J w x w = 0 about a principal axis, no torque
        xn, _, _ = dyn.step(xs, np.array([0.5, 0.3], np.float32), 0.01)
        assert xn[10 + axis] == np.float32(0.7)


@pytest.mark.parametrize("u", [0.1, 0.5, 1.0])
def test_throttle_from_equilibrium(u):
    """V_I_X' = c_t u while each wheel's traction m c_t u / 4 stays under mu f_n = mu m g / 4."""
    dyn = H.RacerSuspension()
    assert 1447 * 3.0 * u / 4 < 0.65 * 1447 * 9.81 / 4
    xd, _ = dyn.computeStateDeriv(_rest_state(dyn), np.array([u, 0.0], np.float32))
    np.testing.assert_allclose(xd[7], 3.0 * u, rtol=1e-5)
    assert abs(xd[8]) < 1e-5


def test_steering_lag():
    dyn = H.RacerSuspension()
    x = _rest_state(dyn)
    for delta, cmd in ((0.0, 0.5), (0.2, -0.7), (-0.3, 1.0)):
        x[RO.STEER_ANGLE] = delta
        xd, y = dyn.computeStateDeriv(x, np.array([0.0, cmd], np.float32))
        f = np.float32
        assert xd[13] == f(0.6) * (f(cmd) / f(-2.45) - f(delta))
        assert y[9] == f(delta) and y[10] == xd[13]


def test_mirrored_steering_gives_mirrored_trajectories():
    """Mirroring the steering command about the x-z plane mirrors the host trajectory: y, the quaternion's x and z,
    v_y, w_x, w_z and the steering angle change sign; everything else is equal."""
    dyn = H.RacerSuspension()
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    T = 120
    rng = np.random.RandomState(4)
    u = np.stack([rng.uniform(0.2, 0.8, T), rng.uniform(0.3, 1.0, T)], -1).astype(np.float32)
    um = u * np.array([1, -1], np.float32)
    x0 = _rest_state(dyn)
    x0[7] = 2.0
    sa, oa = np.zeros((T, 14), np.float32), np.zeros((T, 26), np.float32)
    sb, ob = np.zeros_like(sa), np.zeros_like(oa)
    dyn.output_trajectory(x0, u, T, 0.01, sa, oa)
    dyn.output_trajectory(x0, um, T, 0.01, sb, ob)
    sign = np.array([1, -1, 1, 1, -1, 1, -1, 1, -1, 1, -1, 1, -1, -1], np.float32)
    np.testing.assert_allclose(sb, sa * sign, atol=2e-4)
    assert np.abs(sa[:, 1]).max() > 0.05  # it did turn
    np.testing.assert_allclose(ob[:, 4], -oa[:, 4], atol=2e-4)
    np.testing.assert_allclose(ob[:, 6], -oa[:, 6], atol=2e-4)


def test_output_trajectory_is_the_host_step_with_outputs_of_the_state_before():
    dyn = H.RacerSuspension()
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    T = 30
    u = np.tile(np.array([[0.6, 0.4]], np.float32), (T, 1))
    x0 = _rest_state(dyn)
    st, out = np.zeros((T, 14), np.float32), np.zeros((T, 26), np.float32)
    dyn.output_trajectory(x0, u, T, 0.01, st, out)
    assert np.array_equal(out[0, :14], x0) and not out[0, 14:].any()
    x = x0
    for t in range(T - 1):
        xn, _, y = dyn.step(x, u[t], 0.01)
        np.testing.assert_array_equal(st[t + 1], xn)
        np.testing.assert_array_equal(out[t + 1], y)
        x = xn
    # the generic entry points route to the same twin
    st2, out2 = np.zeros_like(st), np.zeros_like(out)
    assert H.lib().mppib_host_output_trajectory(7, C.byref(dyn.params), None, H._ptr(x0), H._ptr(u), T, C.c_float(0.01),
                                                H._ptr(st2), H._ptr(out2)) == 0
    np.testing.assert_array_equal(st2, st)


def test_leash_keeps_the_quaternion_and_leashes_in_the_body_frame():
    dyn = H.RacerSuspension()
    t = _rest_state(dyn)
    t[3:7] = [math.cos(0.25), 0, 0, math.sin(0.25)]  # yaw 0.5
    n = t.copy()
    n[0] += 1.0
    n[4] = 0.3
    n[7] = 2.0
    leash = np.zeros(14, np.float32)
    leash[0], leash[1], leash[7] = 0.5, 0.5, 0.1
    out = dyn.enforceLeash(t, n, leash)
    np.testing.assert_allclose(out[3:7], t[3:7])
    body = np.array([math.cos(0.5), -math.sin(0.5)])  # (1, 0) in the body frame of yaw 0.5
    assert abs(out[0] - t[0] - (min(body[0], 0.5) * math.cos(0.5) - max(min(body[1], 0.5), -0.5) * math.sin(0.5))) < 1e-5
    assert out[7] == np.float32(t[7] + 0.1)


def test_workload():
    w = W.racer_rigid_suspension()
    assert (w.N, w.T, w.D, w.dt) == (32768, 100, 1, 0.01)
    assert w.cost.params.desired_speed == 5.0
    assert w.x0[0, RO.P_I_Z] == np.float32(0.32) + np.float32(0.2)
    xd, _ = w.dyn.computeStateDeriv(w.x0[0], np.zeros(2, np.float32))
    assert np.abs(xd).max() < 1e-4
    assert W.racer_rigid_suspension(D=2).x0.shape == (2, 14)


def _build_cpp():
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unused-variable", "-I", ROOT + "/include", "-c",
                           CPP_SRC, "-o", CPP_EXE + ".o"])
    subprocess.check_call(["g++", CPP_EXE + ".o", "-o", CPP_EXE, "-L", LIB_DIR, "-lmppi_b200", "-Wl,-rpath," + LIB_DIR])


def test_cpp_blob_state_deriv_and_odometry_match_python():
    """RacerSuspension in C++, built with plain g++ against the reference's include path: the same blob bytes, derivative,
    omegaJacobian and host step as the Python class, and stateFromOdometry / velocityFromState / positionFromState round
    trips."""
    _build_cpp()
    out = subprocess.check_output([CPP_EXE, "blob"])
    dyn = H.RacerSuspension()
    n = C.sizeof(H.RacerRigidSuspensionDynParams)
    ref = H.RacerSuspension()
    ref.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    assert out[:n] == ref.blob()
    vals = np.frombuffer(out[n:], np.float32)
    xd_c, J_c, xn_c, rt = vals[:14], vals[14:23].reshape(3, 3), vals[23:37], vals[37:]
    x = np.zeros(14, np.float32)
    x[3], x[10], x[11], x[12], x[7] = 1, 0.1, -0.03, 0.02, 2
    xd, _, J = dyn.computeStateDeriv(x, np.zeros(2, np.float32), omega_jacobian=True)
    np.testing.assert_array_equal(xd_c, xd)
    np.testing.assert_array_equal(J_c, J)
    xn, _, _ = dyn.step(x, np.zeros(2, np.float32), 0.02)
    np.testing.assert_array_equal(xn_c, xn)
    np.testing.assert_allclose(rt, 0, atol=1e-5)  # round-trip errors of the odometry conversions


def test_cpp_example_links_against_the_library():
    _build_cpp()
    und = subprocess.run(["nm", "--undefined-only", CPP_EXE + ".o"], capture_output=True, text=True, check=True).stdout
    lib = subprocess.run(["nm", "-D", "--defined-only", LIB_DIR + "/libmppi_b200.so"], capture_output=True, text=True,
                         check=True).stdout
    for sym in ("mppib_host_step_racer_rigid_suspension", "mppib_host_state_deriv_racer_rigid_suspension", "mppib_create"):
        assert sym in und and sym in lib, sym
    p = subprocess.run([CPP_EXE], capture_output=True, text=True, timeout=900)
    if p.returncode == 5:
        assert "no CUDA device" in p.stdout
    else:
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _device_one_step(e, x, u):
    """One device step through the device-side roll-forward (T = 2): (x_next, y of x)."""
    _, states, outputs = e.nominal_trajectory(x[None], np.tile(u, (1, 2, 1)))
    return states[0, 1], outputs[0, 1]


@pytest.mark.gpu
def test_device_step_matches_the_device_restatement():
    """One explicit device step from each of many random states (one step, so no chatter can compound) against the
    float64 device body."""
    dyn = H.RacerSuspension()
    p = RO.params(dyn.params)
    e = H.Engine(dyn, H.RacerQuadraticCost(), H.GaussianDistribution(2, [0.1, 0.1]), 256, 2, 1)
    e.set_solver(0.01, 1.0, 0.0)
    x, u = _random_states(dyn, np.random.RandomState(5), 300)
    keep = _away_from_switches(p, x, u)
    assert keep.sum() > 150
    for xi, ui in zip(x[keep], u[keep]):
        xn, y = _device_one_step(e, xi, ui)
        rn, _, ry, _ = RO.device_step(p, xi, ui, 0.01)
        np.testing.assert_allclose(xn, rn, rtol=1e-5, atol=2e-5)
        np.testing.assert_allclose(y, ry, rtol=1e-4, atol=1e-3)
    e.close()


@pytest.mark.gpu
def test_reference_cpu_vs_gpu_case():
    """racer_suspension_model_test.cu:145-282 (skipped there): 10 samples, 8 steps, dt 0.02, from (10, 20, 30) in free
    fall, throttle ~ N(0.3, 0.3), steering ~ N(0, 0.8), control ranges [-1, 1]. Host (implicit w) and device (explicit)
    states and outputs within 1.0 and finite."""
    dyn = H.RacerSuspension()
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    x0 = dyn.getZeroState()
    x0[0:3] = [10, 20, 30]
    T = 9  # x_0 .. x_8
    e = H.Engine(dyn, H.RacerQuadraticCost(), H.GaussianDistribution(2, [0.1, 0.1]), 256, T, 1)
    e.set_solver(0.02, 1.0, 0.0)
    rng = np.random.RandomState(15)
    for s in range(10):
        u = np.stack([rng.normal(0.3, 0.3, T), rng.normal(0.0, 0.8, T)], -1).astype(np.float32)
        sh, oh = np.zeros((T, 14), np.float32), np.zeros((T, 26), np.float32)
        dyn.output_trajectory(x0, u, T, 0.02, sh, oh)
        _, sd, od = e.nominal_trajectory(x0[None], u[None])
        assert np.isfinite(oh).all() and np.isfinite(od).all()
        assert np.abs(sh - sd[0]).max() <= 1.0 and np.abs(oh - od[0]).max() <= 1.0
    e.close()


def _near_switch(margin):
    """The restated trajectory passes within 1e-3 (relative) of the spring clamp or the Stribeck saturation, or within
    1e-5 m/s of vel_x = 0 while braking (copysign's sign): there float32 and float64 may take different branches."""
    return (margin["spring"] < 1e-3) | (margin["slip"] < 1e-3) | (margin["vel_x"] < 1e-5)


def _check_costs(p, cp, c, x0, controls, dt, tol=1e-4, n=4096):
    """K1 costs of n random samples within `tol` of the float64 restatement, except samples _near_switch, which are at
    most 2 % of them. Returns the restated costs of all samples when n is None."""
    idx = np.arange(len(c)) if n is None else np.random.RandomState(0).choice(len(c), n, replace=False)
    c, controls = c[idx], controls[idx]
    ref, _, margin = RO.rollout(p, cp, x0, controls, dt)
    rel = np.abs(c.astype(np.float64) - ref) / np.maximum(np.abs(ref), 1.0)
    near = _near_switch(margin)
    bad = rel > tol
    assert not (bad & ~near).any(), (np.nonzero(bad & ~near)[0][:10], rel[bad & ~near][:10])
    assert bad.mean() <= 0.02, bad.mean()
    assert np.median(rel) < 1e-5
    return ref


SAMPLERS = ["gaussian", "colored", "nln"]


@pytest.mark.gpu
@pytest.mark.parametrize("sampler", SAMPLERS)
def test_k1_vanilla_matches_the_restatement(sampler):
    w = W.racer_rigid_suspension(colored=sampler == "colored")
    if sampler == "nln":
        w.sampler = H.NLNDistribution(2, [0.3, 0.3])
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    e.solve(w.x0, w.U0)
    c, samples = e.get_costs()[0], e.get_samples()[0]
    e.close()
    assert np.isfinite(c).all()
    _check_costs(RO.params(w.dyn.params), w.cost.params, c, w.x0[0], samples, w.dt)


@pytest.mark.gpu
def test_k1_tube_matches_the_restatement():
    w = W.racer_rigid_suspension(D=2)
    w.x0[1, 0:2] += [0.3, -0.2]
    w.x0[1, 7] = 0.5
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    e.solve(w.x0, w.U0)
    c, samples = e.get_costs(), e.get_samples()
    e.close()
    for d in range(2):
        _check_costs(RO.params(w.dyn.params), w.cost.params, c[d], w.x0[d], samples[d], w.dt)


@pytest.mark.gpu
def test_k1_rmppi_with_fixed_gains_matches_the_restatement():
    """RMPPI (D = 2, fixed feedback gains through set_rmppi): the real system's written-back controls are the applied
    ones; its costs match the restatement, and the nominal system's are 0.5 c_nom + 0.5 max(min(c_real, thr), c_nom)."""
    w = W.racer_rigid_suspension(D=2)
    thr = 200.0
    e = H.Engine(w.dyn, w.cost, w.sampler, w.N, w.T, 2, flags=H.FLAG_RMPPI)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    e.seed(w.seed, 0)
    gains = np.zeros((w.T, 14, 2), np.float32)
    gains[:, 7, 0] = -0.2  # throttle against V_I_X error
    gains[:, 1, 1] = 0.1  # steering against P_I_Y error
    e.set_rmppi(thr, gains)
    x0 = w.x0.copy()
    x0[1, 1] += 0.2
    x0[1, 7] = 0.3
    e.solve(x0, w.U0)
    c, applied = e.get_costs(), e.get_samples()
    e.close()
    p = RO.params(w.dyn.params)
    idx = np.random.RandomState(1).choice(w.N, 4096, replace=False)
    c_real = _check_costs(p, w.cost.params, c[1][idx], x0[1], applied[1][idx], w.dt, n=None)
    c_nom, _, margin = RO.rollout(p, w.cost.params, x0[0], applied[0][idx], w.dt)
    want = 0.5 * c_nom + 0.5 * np.maximum(np.minimum(c_real, thr), c_nom)
    rel = np.abs(c[0][idx] - want) / np.maximum(np.abs(want), 1.0)
    assert np.median(rel) < 1e-5 and (rel > 1e-4).mean() <= 0.02


@pytest.mark.gpu
def test_sampled_and_nominal_trajectories_match_the_device_body():
    w = W.racer_rigid_suspension(4096, 60)
    p = RO.params(w.dyn.params)
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    U, _ = e.solve(w.x0, w.U0)
    c, samples = e.get_costs()[0], e.get_samples()[0]
    idx = np.arange(0, w.N, 64)
    outs, costs, _ = e.sample_trajectories(w.x0[0], w.U0[0], idx)
    np.testing.assert_allclose(costs.sum(axis=1), c[idx], rtol=5e-6)
    _, Y, margin = RO.rollout(p, w.cost.params, w.x0[0], samples[idx], w.dt)
    clean = ~_near_switch(margin)
    assert clean.sum() > 0.9 * len(idx)
    np.testing.assert_allclose(outs[clean][:, :, :11], Y[clean][:, :, :11], rtol=1e-3, atol=2e-3)
    # the device-side roll-forward of the solve's U: outputs[t + 1] are those of states[t]
    _, st, out = e.nominal_trajectory(w.x0, U)
    x = w.x0[0].astype(np.float64)
    lo, hi = np.array(p["rng_lo"]), np.array(p["rng_hi"])
    for t in range(w.T - 1):
        x, _, y, _ = RO.device_step(p, x, np.clip(U[0, t], lo, hi), w.dt)
        np.testing.assert_allclose(out[0, t + 1, :11], y[:11], rtol=1e-3, atol=2e-3)
        np.testing.assert_allclose(st[0, t + 1], x, rtol=1e-3, atol=2e-3)
    e.close()


@pytest.mark.gpu
def test_ddp_feedback_is_unsupported():
    """No computeGrad in the reference for this class: set_ddp stores the weights, ddp_feedback is refused."""
    w = W.racer_rigid_suspension(1024, 20, D=2)
    e = w.make_engine()
    e.set_ddp(np.eye(14, dtype=np.float32), np.eye(14, dtype=np.float32), np.eye(2, dtype=np.float32), 1)
    with pytest.raises(H.MppibError) as ex:
        e.ddp_feedback(w.x0[0], np.tile(w.x0[0], (20, 1)), np.zeros((20, 2), np.float32))
    assert "status -2" in str(ex.value)
    e.close()


@pytest.mark.gpu
def test_closed_loop_drives_at_the_desired_speed():
    """VanillaMPPI with the host step as the plant, 100 computeControl calls (1 s) from rest: the speed climbs towards
    5 m/s (full throttle gives at most 3 m/s^2), |y|, roll and pitch stay small, |q| stays 1."""
    w = W.racer_rigid_suspension(8192, 100)
    ctrl = m.VanillaMPPIController(w.dyn, w.cost, None, w.sampler, w.dt, 1, w.lambda_, w.alpha, w.T, w.N, seed=3)
    x = w.x0[0].copy()
    speeds = []
    for _ in range(100):
        ctrl.computeControl(x, 1)
        u = ctrl.getControlSeq()[0].astype(np.float32)
        w.dyn.enforceConstraints(x, u)
        x, _, y = w.dyn.step(x, u, w.dt)
        ctrl.slideControlSequence(1)
        assert np.isfinite(x).all()
        assert abs(np.linalg.norm(x[3:7].astype(np.float64)) - 1.0) < 1e-5
        assert abs(x[1]) < 0.3 and abs(y[7]) < 0.05 and abs(y[8]) < 0.05
        speeds.append(float(y[0]))
    print(f"closed loop: speed after 1 s {speeds[-1]:.3f} m/s")
    assert speeds[-1] > 1.5 and speeds[-1] > speeds[50] > speeds[10]


@pytest.mark.gpu
def test_cpp_example_runs_on_the_gpu():
    _build_cpp()
    p = subprocess.run([CPP_EXE], capture_output=True, text=True, timeout=900)
    print(p.stdout)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "racer rigid suspension example rc 0" in p.stdout
