"""DDP feedback (Tube-MPPI / RMPPI ancillary controller): the CPU restatement in tests/ddp_oracle.py against independent
checks, and the device solve (mppib_ddp_feedback, csrc/ddp_kernel.cuh) against the restatement."""
import os
import subprocess

import numpy as np
import pytest

import mppi_generic_b200 as m
from mppi_generic_b200 import workloads as W
from tests import ddp_oracle as DO

H = m.host
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(name):
    if name == "cartpole":
        return H.CartpoleDynamics(1.0, 1.0, 1.0)
    if name == "di":
        return H.DoubleIntegratorDynamics(1.0)
    if name == "quadrotor":
        return H.QuadrotorDynamics()
    d = H.NeuralNetModel([(-1.0, 1.0), (-2.0, 2.0)])
    d.updateModel([6, 32, 32, 4], W.synthetic_nn_weights(1))  # the weights of the Autorally workload and its tests
    return d


def _random_point(name, rng):
    if name == "quadrotor":
        q = rng.randn(4)
        q /= np.linalg.norm(q)
        x = np.concatenate([rng.randn(6), q, rng.randn(3)])
        u = np.concatenate([rng.randn(3), [9.81 + rng.randn()]])
    elif name == "autorally":
        x = rng.randn(7) * [1, 1, 1, 0.3, 2, 0.5, 0.5] + [0, 0, 0, 0, 4, 0, 0]
        u = rng.uniform(-0.9, 0.9, 2)
    else:
        dims = {"cartpole": (4, 1), "di": (4, 2)}[name]
        x, u = rng.randn(dims[0]), rng.randn(dims[1])
    return x.astype(np.float32), u.astype(np.float32)


MODELS = ["cartpole", "di", "quadrotor", "autorally"]


# ---- CPU -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MODELS)
def test_oracle_jacobians_match_central_differences(name):
    mdl = DO.Model(_model(name))
    rng = np.random.RandomState(3)
    for _ in range(20):
        x, u = _random_point(name, rng)
        A, B = DO.grad(mdl, x, u, np.float64)
        J = np.concatenate([A, B], axis=1)
        xu = np.concatenate([x, u]).astype(np.float64)
        num = np.zeros_like(J)
        for j in range(xu.size):
            h = 1e-6 * max(1.0, abs(xu[j]))
            p, q = xu.copy(), xu.copy()
            p[j] += h
            q[j] -= h
            num[:, j] = (DO.f(mdl, p[:mdl.S], p[mdl.S:], np.float64) - DO.f(mdl, q[:mdl.S], q[mdl.S:], np.float64)) / (2 * h)
        scale = max(1.0, np.abs(num).max())
        assert np.abs(J - num).max() <= 1e-3 * scale, (name, np.abs(J - num).max())
        # the float32 form used by the DDP restatement is the same Jacobian
        A32, B32 = DO.grad(mdl, x, u)
        assert np.abs(np.concatenate([A32, B32], axis=1) - J).max() <= 1e-5 * scale


def test_oracle_ddp_equals_lqr_on_the_double_integrator():
    """One DDP iteration on the linear double integrator is the time-varying LQR recursion with the reference's dt
    scaling of the running cost and symmetrisation of Vxx; recomputed here in float64."""
    mdl = DO.Model(_model("di"))
    T, dt = 60, 0.02
    rng = np.random.RandomState(0)
    Q = np.diag([5.0, 5.0, 1.0, 1.0]).astype(np.float32)
    Qf = (10 * np.eye(4)).astype(np.float32)
    R = np.diag([0.5, 2.0]).astype(np.float32)
    xt = np.cumsum(rng.randn(T, 4) * 0.05, axis=0).astype(np.float32)
    ut = (rng.randn(T, 2) * 0.3).astype(np.float32)
    x0 = (xt[0] + [0.2, -0.1, 0.05, 0.0]).astype(np.float32)
    res = DO.ddp_run(mdl, dt, x0, xt, ut, Q, Qf, R, 1)
    Ad = np.eye(4) + dt * np.array([[0, 0, 1, 0], [0, 0, 0, 1], [0, 0, 0, 0], [0, 0, 0, 0]], float)
    Bd = dt * np.array([[0, 0], [0, 0], [1, 0], [0, 1]], float)
    Q64, Qf64, R64 = Q.astype(float), Qf.astype(float), R.astype(float)
    x = np.zeros((T, 4))
    x[0] = x0
    for i in range(1, T):
        x[i] = Ad @ x[i - 1] + Bd @ ut[i - 1]
    Vxx, Vx = Qf64.copy(), Qf64 @ (x[-1] - xt[-1])
    K = np.zeros((T, 2, 4))
    for k in range(T - 2, -1, -1):
        qx = Q64 @ (x[k] - xt[k]) * dt + Ad.T @ Vx
        qu = R64 @ (ut[k] - ut[k]) * dt + Bd.T @ Vx
        qux, qxx, quu = Bd.T @ Vxx @ Ad, Q64 * dt + Ad.T @ Vxx @ Ad, R64 * dt + Bd.T @ Vxx @ Bd
        K[k] = -np.linalg.solve(quu, qux)
        kk = -np.linalg.solve(quu, qu)
        Vxx = qxx + qux.T @ K[k]
        Vxx = 0.5 * (Vxx + Vxx.T)
        Vx = qx + qux.T @ kk
    got = res["gains"].transpose(0, 2, 1)
    np.testing.assert_allclose(got, K, rtol=1e-5, atol=1e-5 * np.abs(K).max())
    assert np.all(got[-1] == 0)


def test_reference_known_answers():
    """tests/feedback_controllers/ddp_test.cu:19-132: the cartpole's f(0, 0) = 0, f is the model step's state_der, and
    the tracking costs' values, gradients and Hessians with identity weights."""
    dyn = _model("cartpole")
    mdl = DO.Model(dyn)
    assert np.all(DO.f(mdl, np.zeros(4), np.zeros(1)) == 0)
    x, u = np.array([1, 2, 3, 4], np.float32), np.array([5], np.float32)
    _, xd, _ = dyn.step(x, u, 0.01)
    np.testing.assert_allclose(DO.f(mdl, x, u), xd, rtol=2e-6, atol=1e-6)
    z4, z1 = np.zeros(4, np.float32), np.zeros(1, np.float32)
    assert DO.tracking_cost(x, u, z4, z1, np.eye(4), np.eye(1)) == 1 + 4 + 9 + 16 + 25
    assert DO.tracking_cost(x, np.zeros(0), z4, np.zeros(0), np.eye(4), np.eye(0)) == 1 + 4 + 9 + 16
    Q, R = np.eye(4, dtype=np.float32), np.eye(1, dtype=np.float32)
    QR = np.eye(5, dtype=np.float32)
    dc, d2c = DO.running_cost_derivatives(x, u, z4, z1, Q, R)
    np.testing.assert_array_equal(dc, QR @ np.array([1, 2, 3, 4, 5], np.float32))  # ComputeCostGradient
    np.testing.assert_array_equal(d2c, QR)  # ComputeCostHessian
    dcf, d2cf = DO.terminal_cost_derivatives(x, z4, Q)
    np.testing.assert_array_equal(dcf, Q @ x)
    np.testing.assert_array_equal(d2cf, Q)


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _engine(dyn, dt, T=8, flags=0, D=1):
    cost = H._standalone_cost(dyn.DYN_ID)
    e = H.Engine(dyn, cost, H.GaussianDistribution(dyn.CONTROL_DIM), 64, T, D, flags=flags)
    e.set_solver(dt, 1.0, 0.0)
    return e


def _scenario(name, T):
    """(dyn, dt, x0, x_target, u_target): track a smooth open-loop trajectory from a perturbed start."""
    dyn = _model(name)
    mdl = DO.Model(dyn)
    rng = np.random.RandomState(7)
    dt = 0.02 if name in ("di", "autorally") else 0.01
    if name == "quadrotor":
        xs = np.array([0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0], np.float32)
        ut = np.tile(np.array([0.0, 0.0, 0.0, 9.81], np.float32), (T, 1))
        ut[:, :3] += (0.2 * np.sin(np.arange(T)[:, None] * 0.05 + np.arange(3))).astype(np.float32)
        ut[:, 3] += 0.5 * np.cos(np.arange(T) * 0.03)
    elif name == "autorally":
        xs = np.array([0, 0, 0, 0, 4, 0, 0], np.float32)
        ut = np.stack([0.3 * np.sin(np.arange(T) * 0.05), 0.2 + 0.1 * np.cos(np.arange(T) * 0.07)], 1).astype(np.float32)
    elif name == "cartpole":
        xs = np.array([0, 0, 0.2, 0], np.float32)
        ut = (2.0 * np.sin(np.arange(T) * 0.05))[:, None].astype(np.float32)
    else:
        xs = np.array([2, 0, 0, 1], np.float32)
        ut = np.stack([np.cos(np.arange(T) * 0.05), np.sin(np.arange(T) * 0.05)], 1).astype(np.float32)
    xt = np.zeros((T, mdl.S), np.float32)
    xt[0] = xs
    for i in range(1, T):
        xt[i] = xt[i - 1] + DO.f(mdl, xt[i - 1], ut[i - 1]) * np.float32(dt)
    x0 = (xs + 0.05 * rng.randn(mdl.S)).astype(np.float32)
    return dyn, dt, x0, xt, ut


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_device_jacobians_match_oracle(name):
    """jac_out of a two-step solve is [A | B] at (x0, u_target[0]) exactly: the device computeGrad against the host twin.
    Bar 1e-4 of the matrix's largest entry (network 1e-3)."""
    dyn = _model(name)
    mdl = DO.Model(dyn)
    e = _engine(dyn, 0.01)
    rng = np.random.RandomState(5)
    tol = 1e-3 if name == "autorally" else 1e-4
    for _ in range(16):
        x, u = _random_point(name, rng)
        xt = np.stack([x, x])
        ut = np.stack([u, u])
        _, _, _, jac = e.ddp_feedback(x, xt, ut, want_jacobians=True)
        A, B = DO.grad(mdl, x, u)
        ref = np.concatenate([A, B], axis=1)
        assert np.abs(jac[0] - ref).max() <= tol * max(1.0, np.abs(ref).max()), (name, np.abs(jac[0] - ref).max())
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [1, 3])
@pytest.mark.parametrize("name", MODELS)
def test_device_ddp_matches_oracle(name, iters):
    """Gains, states and controls of the device solve against the float32 restatement at T = 100. Double integrator:
    1e-5 relative. Nonlinear models: gains within 1e-3 of each step's max |K|, trajectories within 1e-3 of their scale.
    Measured on an H100 (max |dK| / max |K_t|, max |dx|, max |du|; 1 and 3 iterations): cartpole 2.1e-6, 4.8e-7, 4.3e-6;
    double integrator 2.6e-7, 3.6e-7, 2.9e-6; quadrotor 5.7e-7, 1.0e-6, 6.7e-6; Autorally 6.4e-7, 2.4e-7, 3.7e-7."""
    T = 100
    dyn, dt, x0, xt, ut = _scenario(name, T)
    mdl = DO.Model(dyn)
    S, Cd = mdl.S, mdl.C
    rng = np.random.RandomState(9)
    Q = np.diag(rng.uniform(1, 10, S)).astype(np.float32)
    Qf = (5 * Q).astype(np.float32)
    R = np.diag(rng.uniform(0.5, 2, Cd)).astype(np.float32)
    e = _engine(dyn, dt)
    e.set_ddp(Q, Qf, R, iters)
    gains, xs, us = e.ddp_feedback(x0, xt, ut)
    ref = DO.ddp_run(mdl, dt, x0, xt, ut, Q, Qf, R, iters)
    e.close()
    print(f"ddp-vs-oracle {name} iters={iters}: max |dK| / max|K_t| = "
          f"{float((np.abs(gains - ref['gains']).max(axis=(1, 2)) / np.maximum(np.abs(ref['gains']).max(axis=(1, 2)), 1e-6)).max()):.2e}, "
          f"max |dx| = {float(np.abs(xs - ref['x']).max()):.2e}, max |du| = {float(np.abs(us - ref['u']).max()):.2e}")
    if name == "di":
        np.testing.assert_allclose(gains, ref["gains"], rtol=1e-5, atol=1e-5 * np.abs(ref["gains"]).max())
        np.testing.assert_allclose(xs, ref["x"], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(us, ref["u"], rtol=1e-5, atol=1e-5)
        return
    per_step = np.maximum(np.abs(ref["gains"]).max(axis=(1, 2)), 1e-6)
    err = np.abs(gains - ref["gains"]).max(axis=(1, 2)) / per_step
    assert err[:-1].max() <= 1e-3, (name, iters, float(err.max()))
    assert np.all(gains[-1] == 0)
    assert np.abs(xs - ref["x"]).max() <= 1e-3 * max(1.0, np.abs(ref["x"]).max())
    assert np.abs(us - ref["u"]).max() <= 1e-3 * max(1.0, np.abs(ref["u"]).max())


@pytest.mark.gpu
def test_reference_cartpole_tracking():
    """ddp_test.cu:135-244: a VanillaMPPI solve, then 20 DDP iterations from the zero state with Q = Q_f = 100 I track the
    nominal state trajectory within 1e-2 at every step."""
    w = W.cartpole(2048, 100)
    p = w.cost.params
    p.cart_position_coeff, p.pole_angle_coeff, p.cart_velocity_coeff, p.pole_angular_velocity_coeff = 100, 200, 10, 20
    p.terminal_cost_coeff = 0
    w.sampler.setStdDev([5.0])
    dt = 0.01
    fb = H.DDPFeedback(w.dyn, dt, 100)
    params = H.DDPParams(4, 1)
    params.Q = (100 * np.eye(4)).astype(np.float32)
    params.Q_f = params.Q.copy()
    params.num_iterations = 20
    fb.setParams(params)
    fb.initTrackingController()
    ctrl = H.VanillaMPPIController(w.dyn, w.cost, fb, w.sampler, dt, 100, 0.25, 0.001, 100, 2048, seed=1)
    ctrl.computeControl(np.zeros(4, np.float32), 0)
    nominal_state, nominal_control = ctrl.getTargetStateSeq().copy(), ctrl.getControlSeq().copy()
    fb.computeFeedback(np.zeros(4, np.float32), nominal_state, nominal_control)
    d = np.linalg.norm(nominal_state - fb.result_.state_trajectory, axis=1)
    assert d.max() < 1e-2, (int(d.argmax()), float(d.max()))


@pytest.mark.gpu
def test_reference_quadrotor_tracking():
    """ddp_test.cu:246-356: standalone DDPFeedback, T = 500, 100 iterations; the feedback law alone flies the model to
    within 3 of the goal."""
    T, dt = 500, 0.01
    dyn = H.QuadrotorDynamics([(-2.5, 2.5)] * 3 + [(0.0, 36.0)])
    x_goal = np.array([6, 4, 3, 0, 0, 0, 0.7071068, 0, 0, 0.7071068, 0, 0, 0], np.float32)
    p = H.DDPParams(13, 4)
    p.Q = np.diag([25, 25, 300, 15, 15, 300, 0, 0, 0, 0, 30, 30, 30]).astype(np.float32)
    p.Q_f = np.diag([250, 250, 3000, 150, 150, 3000, 0, 0, 0, 0, 300, 300, 300]).astype(np.float32)
    p.R = np.diag([550, 550, 550, 1]).astype(np.float32)
    p.num_iterations = 100
    fb = H.DDPFeedback(dyn, dt, T)
    fb.setParams(p)
    fb.initTrackingController()
    x_real = np.array([0, -0.5, 0, 0, 0.5, 0, 1, 0, 0, 0, 0, 0, 0], np.float32)
    fb.computeFeedback(x_real, np.tile(x_goal, (T, 1)), np.tile(dyn.zero_control_, (T, 1)))
    x = x_real.copy()
    for t in range(T):
        u = fb.k(x, fb.result_.state_trajectory[t], t)
        dyn.enforceConstraints(x, u)
        x, _, _ = dyn.step(x, u, dt)
    fb.close()
    assert np.linalg.norm(x - x_goal) <= 3.0, float(np.linalg.norm(x - x_goal))


def _tube_failure(x) -> bool:  # tests/controllers/tube_mppi_test.cu:10-23
    r2 = float(x[0] ** 2 + x[1] ** 2)
    return r2 < 1.675 ** 2 or r2 > 2.325 ** 2


@pytest.mark.gpu
def test_rmppi_init_feedback_writes_the_engine_gains():
    """RMPPI with initFeedback() on the CORL-2020 double integrator: the gains the kernel writes into the engine are the
    ones mppib_ddp_feedback returns for the same inputs (bit-identical), the next RMPPI rollout matches the oracle's
    rollout with those gains, and explicitly supplied gains are not overwritten afterwards."""
    import oracle
    w = W.double_integrator_tube(2048, 50)
    ctrl = H.RobustMPPIController(w.dyn, w.cost, None, w.sampler, w.dt, 1, w.lambda_, w.alpha, 20.0, w.T, w.N, seed=3,
                                  num_candidate_nominal_states=9, eval_samples_per_candidate=64)
    ctrl.initFeedback()
    x = np.array([2.05, 0.02, 0.0, 1.05], np.float32)
    ctrl.computeControl(x, 1)
    ctrl.updateImportanceSamplingControl(x, 1)
    engine_gains = ctrl.feedback_gains_.copy()
    g2, _, _ = ctrl.engine.ddp_feedback(x, ctrl.nominal_state_trajectory_, ctrl.nominal_control_trajectory_)
    assert np.array_equal(engine_gains, g2)
    assert np.abs(engine_gains).max() > 0
    # the next rollout applies them (rollout only, on the noise the engine drew)
    e = ctrl.engine
    x0 = np.stack([ctrl.nominal_state_, x]).astype(np.float32)
    U_in = np.stack([ctrl.nominal_control_trajectory_, ctrl.nominal_control_trajectory_]).astype(np.float32)
    e.draw_noise()
    e.rollout_only(x0, U_in, 1, 0)
    eps = e.get_noise()
    samples = np.stack([eps, eps]).copy()
    oracle.set_gaussian_controls(U_in, w.sampler.params, samples, 2, w.T, w.N, 2, 1, 0)
    ref = oracle.rmppi_rollout(w.dyn.DYN_ID, w.cost.COST_ID, w.dyn.params, w.cost.params, w.sampler.params, None, None,
                               w.N, w.T, w.dt, w.lambda_, w.alpha, 20.0, x0, U_in, engine_gains, samples, nthreads=8)
    np.testing.assert_allclose(e.get_costs(), ref, rtol=1e-4, atol=1e-5)
    # explicit gains switch the computation off: the next update leaves them in place
    K = np.zeros((w.T, 2, 4), np.float32)
    K[:, 0, 0] = K[:, 1, 1] = -4.0
    ctrl.setFeedbackGains(K)
    ctrl.updateImportanceSamplingControl(x, 1)
    assert not ctrl.getFeedbackEnabled()
    assert np.array_equal(ctrl.feedback_gains_, np.ascontiguousarray(K.transpose(0, 2, 1)))


@pytest.mark.gpu
def test_rmppi_closed_loop_with_ddp_feedback_stays_in_the_tube():
    w = W.double_integrator_tube(2048, 50)
    ctrl = H.RobustMPPIController(w.dyn, w.cost, None, w.sampler, w.dt, 1, w.lambda_, w.alpha, 20.0, w.T, w.N, seed=3,
                                  num_candidate_nominal_states=9, eval_samples_per_candidate=64)
    p = H.DDPParams(4, 2)
    p.Q = np.diag([500, 500, 100, 100]).astype(np.float32)  # examples/double_integrator_CORL2020.cu weights
    p.Q_f = p.Q.copy()
    ctrl.setFeedbackParams(p)
    ctrl.initFeedback()
    x = np.array([2.0, 0.0, 0.0, 1.0], np.float32)
    rng = np.random.RandomState(0)
    radii = []
    for it in range(120):
        ctrl.updateImportanceSamplingControl(x, 1)
        ctrl.computeControl(x, 1)
        xn = ctrl.getNominalStateSeq()[0]
        u = ctrl.getNominalControlSeq()[0] + ctrl.getFeedbackControl(x, xn, 0)
        xnext, _, _ = w.dyn.step(x, u, w.dt)
        xnext[2:] += 0.2 * np.sqrt(w.dt) * rng.randn(2).astype(np.float32)
        x = xnext
        radii.append(float(np.hypot(x[0], x[1])))
    assert 1.6 < min(radii[20:]) and max(radii[20:]) < 2.4


@pytest.mark.gpu
def test_tube_closed_loop_with_ddp_feedback_stays_in_the_tube():
    """The Tube-MPPI circle test under the large disturbance, with computeFeedback / getCurrentControl's DDP feedback in
    place of the fixed PD stand-in."""
    w = W.double_integrator_tube(1024, 50)
    w.sampler.setControlCostCoeff([1.0, 1.0])
    ctrl = m.TubeMPPIController(w.dyn, w.cost, None, w.sampler, 0.02, 3, 4.0, 0.0, w.T, w.N, seed=7,
                                nominal_threshold=20.0)
    p = H.DDPParams(4, 2)
    p.Q = np.diag([500, 500, 100, 100]).astype(np.float32)
    p.Q_f = p.Q.copy()
    ctrl.setFeedbackParams(p)
    ctrl.initFeedback()
    x = np.array([2.0, 0.0, 0.0, 1.0], np.float32)
    rng = np.random.RandomState(0)
    for t in range(300):
        assert not _tube_failure(x), (t, x)
        ctrl.computeControl(x, 1)
        ctrl.computeFeedback(x)
        u = ctrl.getCurrentControl(x, 0.0, ctrl.getTargetStateSeq()[0], ctrl.getControlSeq())
        x, _, _ = w.dyn.step(x, u.astype(np.float32), 0.02)
        x[2:] += rng.randn(2).astype(np.float32) * np.float32(10.0 * 0.02)
        ctrl.slideControlSequence(1)
    assert ctrl.getFeedbackEnabled()


@pytest.mark.gpu
def test_errors():
    w = W.racer_lstm(256, 16)
    e = w.make_engine()
    T = 10
    with pytest.raises(H.MppibError) as ex:
        e.ddp_feedback(w.x0[0], np.zeros((T, 19), np.float32), np.zeros((T, 2), np.float32))
    assert ex.value.status == -2
    e.close()
    dyn = _model("di")
    e = _engine(dyn, 0.02, T=20)
    with pytest.raises(H.MppibError) as ex:  # to_rmppi on a non-RMPPI engine
        e.ddp_feedback(np.zeros(4), np.zeros((20, 4)), np.zeros((20, 2)), to_rmppi=True)
    assert ex.value.status == -1
    e.close()
    e = _engine(dyn, 0.02, T=20, flags=H.FLAG_RMPPI, D=2)
    with pytest.raises(H.MppibError) as ex:  # T differs from the horizon
        e.ddp_feedback(np.zeros(4), np.zeros((10, 4)), np.zeros((10, 2)), to_rmppi=True)
    assert ex.value.status == -1
    with pytest.raises(H.MppibError) as ex:  # non-finite input
        e.ddp_feedback(np.array([np.nan, 0, 0, 0]), np.zeros((20, 4)), np.zeros((20, 2)))
    assert ex.value.status == -1
    e.ddp_feedback(np.zeros(4), np.zeros((20, 4)), np.zeros((20, 2)), to_rmppi=True)
    e.close()


# ---- the C++ host layer ----------------------------------------------------------------------------------------------
CPP_EXE = os.path.join(ROOT, "tests", "cpp", "ddp_feedback_example.bin")


def _build_cpp():
    lib_dir = os.path.join(ROOT, "mppi-generic_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unused-variable", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "ddp_feedback_example.cpp"), "-o", CPP_EXE, "-L", lib_dir,
                           "-lmppi_b200", "-Wl,-rpath," + lib_dir])


def test_cpp_example_compiles_against_the_shim():
    """DDPParams with .diagonal() <<, initFeedback, computeFeedback and getFeedbackControl through the header-only layer,
    built with plain g++; without a device the binary stops at the C ABI's NO_DEVICE error (exit code 5)."""
    _build_cpp()
    p = subprocess.run([CPP_EXE], capture_output=True, text=True, timeout=900)
    if p.returncode == 5:
        assert "no CUDA device" in p.stdout
    else:
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]


@pytest.mark.gpu
def test_cpp_example_runs_on_the_gpu():
    _build_cpp()
    p = subprocess.run([CPP_EXE], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "ddp example rc 0" in p.stdout
