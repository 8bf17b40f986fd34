"""The smooth-MPPI sampler (MPPIB_SAMPLER_SMOOTH_MPPI): its blob and symbols, the float32 restatement in
tests/smooth_mppi_oracle.py against its float64 twin, the C++ layer, and on the GPU the sampled controls, the broadcast
shift and its clamp, K1's costs on every generic form, the rate-mean update, iterations, asynchronous solves, burned
draws, sampled trajectories, the refusals and a closed loop."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from oracle import explain
import mppi_generic_b200 as m
from mppi_generic_b200 import workloads as W
from tests import smooth_mppi_oracle as SO

H = m.host
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_DIR = ROOT + "/mppi-generic_b200"
CPP_SRC = ROOT + "/tests/cpp/smooth_mppi_example.cpp"
CPP_EXE = ROOT + "/tests/cpp/smooth_mppi_example.bin"
NTHREADS = os.cpu_count() or 1


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_blob_layout_matches_the_c_header():
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "mppi_b200.h"', 'int main(void){',
           'printf("%zu %zu %zu %d\\n", sizeof(mppib_smooth_mppi_params), offsetof(mppib_smooth_mppi_params, gaussian), '
           'offsetof(mppib_smooth_mppi_params, dt), (int)MPPIB_SAMPLER_SMOOTH_MPPI);', "return 0;}"]
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write("\n".join(src))
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        size, off_g, off_dt, sid = [int(v) for v in subprocess.check_output([exe]).split()]
    assert C.sizeof(H.SmoothMPPIParams) == size == C.sizeof(H.GaussianParams) + 4
    assert H.SmoothMPPIParams.gaussian.offset == off_g == 0
    assert H.SmoothMPPIParams.dt.offset == off_dt == C.sizeof(H.GaussianParams)
    assert H.SAMPLER_SMOOTH_MPPI == sid == 3
    s = H.SmoothMPPIDistribution(2, [3.0, 4.0])
    assert s.getSamplingDistributionName() == "Smooth-MPPI" and s.dt == pytest.approx(0.015)
    b = H.SmoothMPPIParams.from_buffer_copy(s.blob())
    assert b.dt == np.float32(0.015) and b.gaussian.std_dev[1] == 4.0 and b.gaussian.std_dev_decay == 1.0


def test_rate_mean_symbols_are_declared_and_exported():
    L = H.lib()
    hdr = open(os.path.join(ROOT, "include", "mppi_b200.h")).read()
    for s in ("mppib_get_derivative_mean", "mppib_set_derivative_mean"):
        assert s + "(" in hdr and s in H.ABI_SYMBOLS and hasattr(L, s)


@pytest.mark.parametrize("stride", [0, 1, 3, 9, 10, 12])
def test_shift_is_a_broadcast_of_row_stride_clamped_to_the_horizon(stride):
    rng = np.random.RandomState(stride)
    T, Cd = 10, 2
    dmu = rng.randn(T, Cd).astype(np.float32)
    got = SO.shift(dmu, stride)
    np.testing.assert_array_equal(got, SO.shift64(dmu, stride).astype(np.float32))
    np.testing.assert_array_equal(got, np.broadcast_to(dmu[min(stride, T - 1)], (T, Cd)))
    # a burned draw is the stride-1 shift, idempotent once the rows agree
    np.testing.assert_array_equal(SO.burn(dmu, 1), np.broadcast_to(dmu[1], (T, Cd)))
    np.testing.assert_array_equal(SO.burn(dmu, 3), SO.burn(dmu, 1))


@pytest.mark.parametrize("stride", [0, 1, 5])
def test_rates_controls_and_update_against_the_float64_twin(stride):
    rng = np.random.RandomState(7 + stride)
    N, T, Cd, dt_s, lam = 200, 12, 2, 0.015, 0.5
    eps = rng.randn(N, T, Cd).astype(np.float32)
    dmu_b = np.broadcast_to(rng.randn(Cd).astype(np.float32), (T, Cd))
    mu = rng.randn(T, Cd).astype(np.float32)
    sd = np.array([2.0, 0.5], np.float32)
    pct = 0.1
    v = SO.rates(eps, dmu_b, sd, stride, pct)
    v64 = SO.rates64(eps, dmu_b, sd, stride, pct)
    np.testing.assert_allclose(v, v64, rtol=2e-7, atol=1e-7)
    first_pure = int(np.ceil((1 - pct) * N))
    # the three cases: sample 0 and t < s take the rate mean, the pure-noise rows drop it, the others add it
    np.testing.assert_array_equal(v[0], dmu_b)
    np.testing.assert_array_equal(v[1:, :stride], np.broadcast_to(dmu_b[:stride], v[1:, :stride].shape))
    np.testing.assert_allclose(v[first_pure:, stride:], sd * eps[first_pure:, stride:], rtol=1e-7)
    np.testing.assert_allclose(v[1:first_pure, stride:], sd * eps[1:first_pure, stride:] + dmu_b[0], rtol=1e-6, atol=1e-6)
    u = SO.controls(v, mu, dt_s)
    np.testing.assert_allclose(u, SO.controls64(v, mu, dt_s), rtol=1e-7, atol=1e-7)
    # a pure-noise row keeps mu (the Gaussian sampler's pure-noise rows drop it)
    np.testing.assert_allclose(u[first_pure:, stride:], mu[stride:] + v[first_pure:, stride:] * np.float32(dt_s),
                               rtol=1e-6, atol=1e-7)
    costs = rng.uniform(0, 5, N).astype(np.float32)
    dmu_new, U = SO.update(costs, v, lam, mu, dt_s)
    dmu_new64, U64 = SO.update64(costs, v64, lam, mu, dt_s)
    np.testing.assert_allclose(dmu_new, dmu_new64, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(U, U64, rtol=1e-6, atol=1e-6)
    # the update averages the unconstrained rates: clipping them first gives another mean
    clipped = SO.update64(costs, np.clip(v64, -0.5, 0.5), lam, mu, dt_s)[0]
    assert np.abs(clipped - dmu_new64).max() > 1e-2


def _build_cpp():
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unused-variable", "-I", os.path.join(ROOT, "include"),
                           CPP_SRC, "-o", CPP_EXE, "-L", LIB_DIR, "-lmppi_b200", "-Wl,-rpath," + LIB_DIR])


def test_cpp_example_compiles_and_fails_loudly_without_a_device():
    _build_cpp()
    p = subprocess.run([CPP_EXE], capture_output=True, text=True, timeout=600)
    if p.returncode == 5:
        assert "no CUDA device" in p.stdout
    else:
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]


def _desc(**kw):
    d = H.Desc(H.DYN_CARTPOLE, H.COST_CARTPOLE_QUADRATIC, H.SAMPLER_SMOOTH_MPPI, 256, 16, 1, 0, 0, None, 0, 1)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("kw", [dict(num_distributions=2), dict(world_size=2),
                                dict(dynamics_id=H.DYN_AUTORALLY_NN, cost_id=H.COST_AR_STANDARD, flags=H.FLAG_NN_TENSOR)],
                         ids=["D2", "world2", "nn_tensor_autorally"])
def test_unsupported_engines_are_refused_before_the_device(kw):
    h = C.c_void_p()
    assert H.lib().mppib_create(C.byref(h), C.byref(_desc(**kw))) == -2  # MPPIB_ERR_UNSUPPORTED


def test_nn_tensor_is_ignored_where_there_is_no_tensor_core_kernel(monkeypatch):
    """As for a Gaussian engine, MPPIB_FLAG_NN_TENSOR / MPPIB_NN_TENSOR mean nothing to a model without the wgmma kernel."""
    monkeypatch.setenv("MPPIB_NN_TENSOR", "1")
    L = H.lib()
    h = C.c_void_p()
    rc = L.mppib_create(C.byref(h), C.byref(_desc(flags=H.FLAG_NN_TENSOR)))
    assert rc in (0, -5), rc  # created, or no device on this machine: never refused
    if rc == 0:
        L.mppib_destroy(h)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def _smooth(w, sd, dt_s=0.015, coeff=None):
    """w with its sampler replaced by a smooth-MPPI sampler of rate sigma `sd`."""
    s = H.SmoothMPPIDistribution(w.dyn.CONTROL_DIM, sd, dt=dt_s)
    for c in range(w.dyn.CONTROL_DIM):
        s.params.control_cost_coeff[c] = w.sampler.params.control_cost_coeff[c] if coeff is None else coeff[c]
    w.sampler = s
    return w


def _wide(w):
    w.dyn.setControlRanges([(-1e30, 1e30)] * w.dyn.CONTROL_DIM)
    return w


def _restate(w, e, dmu_prev, stride=1, iteration=0, U=None):
    """(v, u) of the last K1 from its noise, as the restatement forms them."""
    sp = w.sampler.params
    Cd = w.dyn.CONTROL_DIM
    decay = np.float32(np.float32(sp.std_dev_decay) ** iteration)
    sd = np.array([decay * np.float32(sp.std_dev[c]) for c in range(Cd)], np.float32)
    v = SO.rates(e.get_noise(), SO.shift(dmu_prev, stride), sd, stride, sp.pure_noise_trajectories_percentage, w.N)
    return v, SO.controls(v, (w.U0 if U is None else U)[0], w.sampler.dt)


def _oracle_costs(w, u):
    samples = np.ascontiguousarray(u[None], np.float32)
    return oracle.rollout(w.dyn.DYN_ID, w.cost.COST_ID, w.dyn.params, w.cost.params, w.sampler.params, w.dyn.nn_theta,
                          getattr(w.cost, "costmap", None), w.N, w.T, 1, w.dt, w.lambda_, w.alpha, w.x0, w.U0, samples,
                          NTHREADS)[0]


def _rel(a, b):
    return np.abs(a - b) / np.maximum(np.abs(b), 1.0)


def _within_ulp(a, b, n=1):
    return np.abs(a - b) <= n * np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32))


def _cartpole(N=2048, T=100):
    w = _smooth(W.cartpole(N, T), [300.0])
    w.U0 = np.random.RandomState(3).uniform(-1, 1, (1, T, 1)).astype(np.float32)
    return w


@pytest.mark.gpu
def test_first_solve_controls_equal_the_restatement():
    w = _wide(_cartpole())
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    np.testing.assert_array_equal(e.get_derivative_mean(), 0.0)  # defined here: zero at create
    e.solve(w.x0, w.U0)
    _, u = _restate(w, e, np.zeros((w.T, 1), np.float32))
    got = e.get_samples()[0]
    assert _within_ulp(got, u).all(), np.abs(got - u).max()
    np.testing.assert_array_equal(got[0], w.U0[0])  # sample 0 is mu
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("stride", [0, 1, 3, "T-1", "T+2"])
def test_every_step_samples_around_row_stride_of_the_rate_mean(stride):
    w = _wide(_cartpole(1024, 40))
    s = {"T-1": w.T - 1, "T+2": w.T + 2}.get(stride, stride)
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    dmu = (np.arange(w.T, dtype=np.float32) * 10.0 - 100.0)[:, None]
    e.set_derivative_mean(dmu)
    np.testing.assert_array_equal(e.get_derivative_mean(), dmu)
    e.solve(w.x0, w.U0, optimization_stride=s)
    row = dmu[min(s, w.T - 1)]
    expect = SO.fmaf(row, np.float32(w.sampler.dt), w.U0[0])
    np.testing.assert_array_equal(e.get_samples()[0][0], expect)
    _, u = _restate(w, e, dmu, stride=s)
    assert _within_ulp(e.get_samples()[0], u).all()
    e.close()


FORMS = {
    "resident": (H.FLAG_WRITEBACK_CONTROLS, {}),
    "resident_no_writeback": (0, {}),
    "no_tma": (H.FLAG_WRITEBACK_CONTROLS | H.FLAG_NO_TMA, {}),
    "stream": (H.FLAG_WRITEBACK_CONTROLS, {"MPPIB_STREAM": "1"}),
    "stream_no_writeback": (0, {"MPPIB_STREAM": "1"}),
    "stream_readback": (0, {"MPPIB_STREAM": "1", "MPPIB_STREAM_READBACK": "1"}),
}
MODELS = {
    "cartpole": lambda: _cartpole(),
    "double_integrator": lambda: _smooth(W.double_integrator_vanilla(2048, 100), [60.0, 60.0]),
    "quadrotor": lambda: _smooth(W.quadrotor(2048, 100), [30.0, 30.0, 30.0, 100.0]),
}


def _check_costs_and_update(w, e, dmu_prev=None, stride=1, tol=1e-4):
    dmu_prev = np.zeros((w.T, w.dyn.CONTROL_DIM), np.float32) if dmu_prev is None else dmu_prev
    U, _ = e.solve(w.x0, w.U0, optimization_stride=stride)
    v, u = _restate(w, e, dmu_prev, stride=stride)
    costs = e.get_costs()[0]
    ref = _oracle_costs(w, u)
    assert _rel(costs, ref).max() < tol, _rel(costs, ref).max()
    dmu_dev = e.get_derivative_mean()
    dmu64, _ = SO.update64(costs, v.astype(np.float64), w.lambda_, w.U0[0], w.sampler.dt)
    scale = max(1.0, float(np.abs(v).max()))
    assert np.abs(dmu_dev - dmu64).max() < 1e-5 * scale, np.abs(dmu_dev - dmu64).max()
    np.testing.assert_array_equal(U[0], SO.fmaf(dmu_dev, np.float32(w.sampler.dt), w.U0[0]))
    return costs, v, u


@pytest.mark.gpu
@pytest.mark.parametrize("form", sorted(FORMS))
@pytest.mark.parametrize("model", sorted(MODELS))
def test_costs_and_update_match_the_restatement_on_every_form(model, form, monkeypatch):
    flags, env = FORMS[form]
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    w = MODELS[model]()
    e = w.make_engine(flags=flags)
    _check_costs_and_update(w, e)
    # a second solve samples around the first one's rate mean
    dmu1 = e.get_derivative_mean()
    _check_costs_and_update(w, e, dmu_prev=dmu1, stride=2)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("spt", [1, 2])
def test_autorally_runs_the_generic_form(spt, monkeypatch):
    if spt == 2:
        monkeypatch.setenv("MPPIB_SPT", "2")
    w = _smooth(W.autorally(4096, 100), [20.0, 20.0])
    flags = H.FLAG_WRITEBACK_CONTROLS | (H.FLAG_NN_FFMA2 if spt == 2 else 0)
    e = w.make_engine(flags=flags)
    g = W.autorally(4096, 100).make_engine(flags=flags | H.FLAG_NO_WARP_SPEC)
    d = W.autorally(4096, 100).make_engine(flags=flags)
    assert e.launch_info() == g.launch_info()
    if spt == 1:
        assert e.launch_info() != d.launch_info()  # the Gaussian engine runs the warp-specialised kernel
    g.close()
    d.close()
    e.solve(w.x0, w.U0)
    _, u = _restate(w, e, np.zeros((w.T, 2), np.float32))
    assert _within_ulp(e.get_samples()[0], np.clip(u, [-1.0, -2.0], [1.0, 2.0])).all()
    explain.autorally_outliers_explained(w, e, _oracle_costs(w, u), tol=1e-4)
    e.close()


@pytest.mark.gpu
def test_racer_lstm_h32_tensor_core_dynamics():
    w = _smooth(W.racer_lstm(2048, 64, hidden_dim=32, head_hidden=20, colored=False), [20.0, 20.0])
    oracle.set_lstm(w.dyn.lstm_theta, w.dyn.hidden_dim, w.dyn.head_hidden)
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    _check_costs_and_update(w, e, tol=2e-4)  # C5's bar: LSTM steps with tanh_fast (tests/test_gpu_parity.py)
    e.close()


@pytest.mark.gpu
def test_update_averages_the_unconstrained_rates():
    w = _cartpole()
    w.dyn.setControlRanges([(-0.3, 0.3)])
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    costs, v, u = _check_costs_and_update(w, e)
    wts = SO.weights64(costs, w.lambda_)
    constrained_rates = (e.get_samples()[0].astype(np.float64) - w.U0[0]) / np.float64(np.float32(w.sampler.dt))
    other = np.tensordot(wts, constrained_rates, axes=(0, 0))
    assert np.abs(other - e.get_derivative_mean()).max() > 1.0
    e.close()


@pytest.mark.gpu
def test_likelihood_ratio_cost_uses_mu():
    """The likelihood-ratio term takes the mean mu (not mu + dt_s dmu_b), the undecayed sigma and mean 0 on the pure-noise
    rows. The state cost is made small so that the term is most of each cost, and a non-zero rate mean, iteration 1 and
    std_dev_decay 0.5 make each wrong choice a different cost."""
    w = _smooth(W.cartpole(2048, 100), [20.0], coeff=[200.0])
    p = w.cost.params
    p.cart_position_coeff = p.cart_velocity_coeff = p.pole_angle_coeff = p.pole_angular_velocity_coeff = 0.01
    p.control_cost_coeff[0] = 0.0
    p.desired_terminal_state[:] = [0.0, 0.0, 0.0, 0.0]
    w.sampler.params.std_dev_decay = 0.5
    w.sampler.params.pure_noise_trajectories_percentage = 0.1
    # mu of one sign: the shifted mean then changes the term's average over the horizon, not only its steps
    w.U0 = np.random.RandomState(5).uniform(0.5, 2.0, (1, w.T, 1)).astype(np.float32)
    w.alpha = 0.2
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    dmu = (np.linspace(-80.0, 80.0, w.T, dtype=np.float32))[:, None]  # row 1: about -78, so mu + dt_s dmu_b = mu - 1.2
    e.set_derivative_mean(dmu)
    e.solve(w.x0, w.U0, 1, 1)
    _, u = _restate(w, e, dmu, stride=1, iteration=1)
    costs = e.get_costs()[0]
    ref = _oracle_costs(w, u)
    assert _rel(costs, ref).max() < 1e-4, _rel(costs, ref).max()

    def alt(means=None, sd_scale=1.0, coeff=None):
        sp = H.GaussianParams.from_buffer_copy(bytes(w.sampler.params))
        sp.std_dev[0] *= sd_scale
        if coeff is not None:
            sp.control_cost_coeff[0] = coeff
        samples = np.ascontiguousarray(u[None], np.float32)
        return oracle.rollout(w.dyn.DYN_ID, w.cost.COST_ID, w.dyn.params, w.cost.params, sp, None, None, w.N, w.T, 1, w.dt,
                              w.lambda_, w.alpha, w.x0, w.U0 if means is None else means, samples, NTHREADS)[0]

    shifted = SO.fmaf(SO.shift(dmu, 1), np.float32(w.sampler.dt), w.U0[0])[None]
    for name, wrong in (("mean mu + dt_s dmu_b", alt(means=shifted)), ("decayed sigma", alt(sd_scale=0.5)),
                        ("no likelihood-ratio term", alt(coeff=0.0))):
        miss = _rel(costs, wrong)
        assert np.median(miss) > 100 * 1e-4, (name, float(np.median(miss)))
    e.close()


@pytest.mark.gpu
def test_iterations_use_the_decayed_sigma_and_the_first_result():
    w = _wide(_cartpole(2048, 60))
    w.sampler.params.std_dev_decay = 0.5
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    U1, _ = e.solve(w.x0, w.U0, 1, 0)
    dmu1 = e.get_derivative_mean()
    e.solve(w.x0, U1, 1, 1)
    _, u = _restate(w, e, dmu1, stride=1, iteration=1, U=U1)
    assert _within_ulp(e.get_samples()[0], u).all()
    e.close()


@pytest.mark.gpu
def test_two_async_solves_equal_two_blocking_ones():
    w = _cartpole()
    a = w.make_engine()
    U1, _ = a.solve(w.x0, w.U0)
    U2, s2 = a.solve(w.x0, U1)
    dmu = a.get_derivative_mean()
    b = w.make_engine()
    x0, U0 = np.ascontiguousarray(w.x0), np.ascontiguousarray(w.U0)
    b.solve_async(x0, U0)
    b.solve_async(x0, np.ascontiguousarray(U1))  # the second K1 reads the first merge's rate mean on the device
    V2, t2 = b.solve_wait()
    np.testing.assert_array_equal(V2, U2)
    np.testing.assert_array_equal(b.get_derivative_mean(), dmu)
    a.close()
    b.close()


@pytest.mark.gpu
def test_burned_draw_broadcasts_row_one():
    w = _cartpole(1024, 40)
    e = w.make_engine()
    dmu = np.random.RandomState(1).randn(w.T, 1).astype(np.float32)
    e.set_derivative_mean(dmu)
    off = e.rng_offset()
    e.burn_draws(1)
    assert e.rng_offset() == off + w.N * w.T
    np.testing.assert_array_equal(e.get_derivative_mean(), SO.burn(dmu, 1))
    e.close()


@pytest.mark.gpu
def test_sampled_trajectories_sum_to_k1s_costs():
    w = _smooth(W.quadrotor(1024, 100), [30.0, 30.0, 30.0, 100.0])
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    e.solve(w.x0, w.U0)
    idx = np.array([0, 1, 17, 500, 1023], np.int32)
    _, costs, _ = e.sample_trajectories(w.x0[0], w.U0[0], idx)
    np.testing.assert_allclose(costs.sum(axis=1), e.get_costs()[0][idx], rtol=5e-6)
    e.close()


@pytest.mark.gpu
def test_refusals_on_an_engine():
    w = _cartpole(256, 16)
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    L = H.lib()
    with pytest.raises(H.MppibError) as ex:
        e.set_tsallis(1.0, 2.0)
    assert ex.value.status == -2
    g = bytes(w.sampler.params)  # the Gaussian blob's size
    assert L.mppib_set_blob(e._h, H.BLOB_SAMPLER, g, len(g)) == -1
    bad = H.SmoothMPPIParams(w.sampler.params, float("nan"))
    assert L.mppib_set_blob(e._h, H.BLOB_SAMPLER, bytes(bad), C.sizeof(bad)) == -1
    e.solve_async(np.ascontiguousarray(w.x0), np.ascontiguousarray(w.U0))
    buf = np.zeros((w.T, 1), np.float32)
    assert L.mppib_set_derivative_mean(e._h, buf.ctypes.data) == -9  # MPPIB_ERR_STATE while a solve is pending
    e.solve_wait()
    e.close()
    gw = W.cartpole(256, 16)
    ge = gw.make_engine()
    assert L.mppib_get_derivative_mean(ge._h, buf.ctypes.data) == -1
    assert L.mppib_set_derivative_mean(ge._h, buf.ctypes.data) == -1
    ge.close()


def _tube_failure(x) -> bool:  # tests/controllers/tube_mppi_test.cu:10-23
    r2 = float(x[0] ** 2 + x[1] ** 2)
    return r2 < 1.675 ** 2 or r2 > 2.325 ** 2


@pytest.mark.gpu
def test_double_integrator_vanilla_tracks_the_circle():
    """The closed loop of test_gpu_parity's Gaussian case with the smooth sampler: rate sigma 1 / dt_s, so that a
    control sample spreads by 1 as there."""
    w = W.double_integrator_vanilla(1024, 50)
    dt_s = 0.015
    w = _smooth(w, [1.0 / dt_s, 1.0 / dt_s], dt_s=dt_s, coeff=[1.0, 1.0])
    ctrl = m.VanillaMPPIController(w.dyn, w.cost, None, w.sampler, 0.02, 3, 4.0, 0.0, w.T, w.N, seed=11)
    x = np.array([2.0, 0.0, 0.0, 1.0], np.float32)
    rng = np.random.RandomState(0)
    for t in range(500):
        assert not _tube_failure(x), (t, x)
        ctrl.computeControl(x, 1)
        u = ctrl.getControlSeq()[0].copy()
        x, _, _ = w.dyn.step(x, u, 0.02)
        x[2:] += rng.randn(2).astype(np.float32) * np.float32(0.02)
        ctrl.slideControlSequence(1)


@pytest.mark.gpu
def test_cpp_example_runs_on_the_gpu():
    _build_cpp()
    p = subprocess.run([CPP_EXE], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "smooth-MPPI cartpole" in p.stdout
