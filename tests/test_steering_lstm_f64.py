"""The RACER steering LSTM against a float64 network (tests/steering_lstm_f64.py) at every hidden and head width the engine
accepts, on each form that evaluates it: the host twin (CPU), the compile-time SIMT form (H = 4, L1 = 20), the run-time
SIMT form (every other size, the side rollouts, and H = 32 under MPPIB_FLAG_LSTM_SIMT) and the tensor-core form (H = 32,
L1 <= 24).

What the GPU tests observe is the steering subsystem alone: RacerQuadraticCost with only steer_coeff = 1 and no control
cost reads the steer angle, which depends on nothing but the steer states, the steering command and the network — a
closed two-state system around the LSTM, restated in float64. dt = 0.1 lets the network carry the cost (its output enters
as 5 * out * dt^2 on the angle), and the angle / rate limits are raised so the clamps stay slack. Every comparison
asserts |float32 - float64| <= 2 * bound + 4 ulps with the running bound of steering_lstm_f64 (factor fixed beforehand),
and prints the largest error / bound ratio."""
import json
import math
import os

import numpy as np
import pytest

import mppi_generic_b200 as M
from mppi_generic_b200 import workloads as W
from tests import steering_lstm_f64 as R

H = M.host

# (H, L1): the compile-time fast path, the run-time SIMT sizes around it and at the edges of [1, 64]^2, and H = 32 at
# every head width on both sides of the tensor-core form's three n-tiles
SIMT_SIZES = [(1, 1), (4, 19), (4, 21), (7, 5), (8, 20), (31, 24), (33, 24), (64, 1), (64, 64)]
TC_HEADS = [1, 7, 8, 9, 16, 23, 24]
AUTO_SIMT_HEADS = [25, 64]
GRID = [(4, 20)] + SIMT_SIZES + [(32, L1) for L1 in TC_HEADS + AUTO_SIMT_HEADS]
REGIMES = ["synthetic", "x6", "tiny", "init"]
DT, SA0, SR0 = 0.1, 0.3, -0.5


def weights(Hd, L1, regime, seed=2):
    """(lstm block, head) of one weight regime: the synthetic U(-1,1)/sqrt(fan_in) draw; six times it (gates saturate);
    1e-6 times it (FP16-subnormal hi parts on the tensor-core form); or the draw with distinct nonzero initial hidden and
    cell values per unit (the synthetic head already has nonzero b1 and b2)."""
    lstm, head = W.synthetic_lstm_weights(Hd, L1, seed)
    lstm, head = lstm.astype(np.float64), head.astype(np.float64)
    if regime == "x6":
        lstm, head = 6.0 * lstm, 6.0 * head
    elif regime == "tiny":
        lstm, head = 1e-6 * lstm, 1e-6 * head
    elif regime == "init":
        j = np.arange(Hd)
        lstm[-2 * Hd:-Hd] = 0.9 * np.sin(1.7 * j + 0.4)
        lstm[-Hd:] = 1.5 * np.cos(2.3 * j + 0.1)
    return lstm.astype(np.float32), head.astype(np.float32)


def make_dyn(Hd, L1, regime, suspension=False, control_range=1.0):
    cls = H.RacerDubinsElevationSuspension if suspension else H.RacerDubinsElevationLSTMSteering
    dyn = cls(3, 20, (23, 100, 2 * Hd), 4, Hd, (Hd + 4, L1, 1), 11)
    dyn.setControlRanges([(-1.0, 1.0), (-control_range, control_range)])
    dyn.params.max_steer_angle, dyn.params.max_steer_rate = 50.0, 500.0
    dyn.setAllValues(*weights(Hd, L1, regime))
    return dyn


def commands(n, T, scale, seed=5):
    """n command sequences; the first is all zero, the engine's zero-noise sample (the mean, here zero)."""
    c = (np.random.RandomState(seed).uniform(-1.0, 1.0, (n, T)) * scale).astype(np.float32)
    c[0] = 0.0
    return c


# ---- the reference itself ----------------------------------------------------------------------------------------------
def test_known_answer_all_ones():
    """lstm_helper_test.cu forwardCPU: H = 20, 8 inputs, head {28, 3}, every weight, initial hidden and cell 1, input 1."""
    with open(os.path.join(os.path.dirname(__file__), "golden", "reference_known_answers.json")) as f:
        want = json.load(f)["lstm_all_ones_outputs"]["value"]
    Hd, In = 20, 8
    net = R.Blob(np.ones(4 * Hd * Hd + 4 * Hd * In + 6 * Hd + 28 * 3 + 3), Hd, head=[28, 3], input_dim=In)
    h, c, x = net.h0.copy(), net.c0.copy(), np.ones(In)
    for v in want:
        out, h, c = R.forward(net, x, h, c)
        np.testing.assert_allclose(out, [v] * 3, rtol=1e-6)  # EXPECT_FLOAT_EQ: within 4 float32 ulps


def _hand_blob():
    """H = 1, L1 = 1: one distinct nonzero weight per block, each input weight on a different input."""
    v = dict(W_im=0.3, W_fm=-0.7, W_om=1.1, W_cm=0.45, W_ii=(0, 0.8), W_fi=(1, -0.35), W_oi=(2, 0.6), W_ci=(3, -1.3),
             b_i=0.15, b_f=0.9, b_o=-0.25, b_c=0.05, h0=0.55, c0=-0.8, W1h=0.9, W1=(2, 1.7), b1=-0.4, W2=2.2,
             b2=0.65)
    theta = np.zeros(R.num_params(1, 1))
    theta[0:4] = [v["W_im"], v["W_fm"], v["W_om"], v["W_cm"]]
    for q, k in enumerate(("W_ii", "W_fi", "W_oi", "W_ci")):
        theta[4 + 4 * q + v[k][0]] = v[k][1]
    theta[20:24] = [v["b_i"], v["b_f"], v["b_o"], v["b_c"]]
    theta[24], theta[25] = v["h0"], v["c0"]
    theta[26] = v["W1h"]  # W1 [1 x 5] on [h' ; x]: position 0 = h'
    theta[26 + v["W1"][0]] = v["W1"][1]  # position 2 = x[1]
    theta[31], theta[32], theta[33] = v["b1"], v["W2"], v["b2"]
    return theta.astype(np.float32), v


def test_hand_checked_blob():
    """A blob whose every block holds one distinct value, so that any permutation of the layout changes the output; the
    expected output is written out by hand."""
    theta, v = _hand_blob()
    x = np.array([0.2, -0.6, 0.9, 0.35])
    sig = lambda z: 1.0 / (1.0 + math.exp(-z))  # noqa: E731
    h, c = v["h0"], v["c0"]
    i = sig(v["W_ii"][1] * x[0] + v["W_im"] * h + v["b_i"])
    f = sig(v["W_fi"][1] * x[1] + v["W_fm"] * h + v["b_f"])
    o = sig(v["W_oi"][1] * x[2] + v["W_om"] * h + v["b_o"])
    g = math.tanh(v["W_ci"][1] * x[3] + v["W_cm"] * h + v["b_c"])
    c2 = i * g + f * c
    h2 = math.tanh(c2) * o
    a = math.tanh(v["W1h"] * h2 + v["W1"][1] * x[1] + v["b1"])  # head inputs 0 and 2 of [h' ; x]: h' and x[1]
    want = v["W2"] * a + v["b2"]
    net = R.Blob(theta, 1, 1)
    out, hn, cn = R.forward(net, x, net.h0, net.c0)
    f32 = lambda t: float(np.float32(t))  # noqa: E731  the blob holds float32 values
    assert abs(out[0] - want) < 1e-6 and abs(hn[0] - h2) < 1e-6 and abs(cn[0] - c2) < 1e-6
    # and exactly, with the blob's float32 values
    i = sig(f32(0.8) * x[0] + f32(0.3) * f32(0.55) + f32(0.15))
    f = sig(f32(-0.35) * x[1] + f32(-0.7) * f32(0.55) + f32(0.9))
    o = sig(f32(0.6) * x[2] + f32(1.1) * f32(0.55) + f32(-0.25))
    g = math.tanh(f32(-1.3) * x[3] + f32(0.45) * f32(0.55) + f32(0.05))
    c2 = i * g + f * f32(-0.8)
    h2 = math.tanh(c2) * o
    assert abs(cn[0] - c2) < 1e-14 and abs(hn[0] - h2) < 1e-14
    assert abs(out[0] - (f32(2.2) * math.tanh(f32(0.9) * h2 + f32(1.7) * x[1] + f32(-0.4)) + f32(0.65))) < 1e-14
    # the host twin on the same blob, one step from the blob's initial state: the head reads h', so the rate depends on
    # every gate and state block
    dyn = H.RacerDubinsElevationLSTMSteering(3, 20, (23, 100, 2), 4, 1, (5, 1, 1), 11)
    dyn.setAllValues(theta[:R.num_params(1, 1) - 8], theta[R.num_params(1, 1) - 8:])
    hh, cc = dyn.initial_hidden_cell()
    x0 = np.zeros(19, np.float32)
    x0[4], x0[8] = 0.4, -0.7
    xn, _, _, hh, cc = dyn.step(x0, [0.0, 0.3], 0.1, hh, cc)
    r = R.steer_rollout(net, R.SteerParams(dyn.params), x0[4], x0[8], [0.3], 0.1, "host")
    R.check("host twin, hand blob: rate", xn[8], r["rate"][0], r["e_rate"][0])


def _host_rollout(dyn, sa0, sr0, cmds, dt, suspension=False):
    x = np.zeros(24 if suspension else 19, np.float32)
    sa_i, sr_i = (4, 12) if suspension else (4, 8)
    x[sa_i], x[sr_i] = sa0, sr0
    h, c = dyn.initial_hidden_cell()
    sa, sr = [], []
    for u in cmds:
        x, _, _, h, c = dyn.step(x, [0.0, u], dt, h, c)
        sa.append(x[sa_i])
        sr.append(x[sr_i])
    return np.array(sa), np.array(sr)


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("Hd,L1", GRID, ids=[f"H{h}_L{l}" for h, l in GRID])
def test_host_twin_against_float64(Hd, L1, regime):
    """dyn.step (the host twin the controller's tail rolls forward) over 24 steps, its steer angle and rate against the
    float64 subsystem with the host form's bound; two command sequences, the second over a +-1e3 command range."""
    for scale in (1.0, 1e3):
        dyn = make_dyn(Hd, L1, regime, control_range=scale)
        net = R.Blob(dyn.lstm_theta, Hd, L1)
        sp = R.SteerParams(dyn.params)
        cmds = commands(1, 24, scale)[0]
        sa, sr = _host_rollout(dyn, SA0, SR0, cmds, DT)
        r = R.steer_rollout(net, sp, SA0, SR0, cmds, DT, "host")
        R.check(f"host H{Hd} L1 {L1} {regime} x{scale:g}: angle", sa, r["angle"], r["e_angle"])
        R.check(f"host H{Hd} L1 {L1} {regime} x{scale:g}: rate", sr, r["rate"], r["e_rate"])


def test_host_twin_suspension_model():
    """RacerDubinsElevationSuspension's host step shares the steering network and places the rate at index 12."""
    dyn = make_dyn(8, 20, "init", suspension=True)
    net = R.Blob(dyn.lstm_theta, 8, 20)
    cmds = commands(1, 24, 1.0)[0]
    sa, sr = _host_rollout(dyn, SA0, SR0, cmds, DT, suspension=True)
    r = R.steer_rollout(net, R.SteerParams(dyn.params), SA0, SR0, cmds, DT, "host")
    R.check("host suspension: angle", sa, r["angle"], r["e_angle"])
    R.check("host suspension: rate", sr, r["rate"], r["e_rate"])


# ---- GPU ---------------------------------------------------------------------------------------------------------------
STAGING = {"resident": (0, {}), "no_tma": (H.FLAG_NO_TMA, {}), "stream": (0, {"MPPIB_STREAM": "1"})}


class Case:
    """One engine of N = len(cmds) rollouts over chosen steering commands (the noise, on a zero mean and unit standard
    deviation), throttle zero."""

    def __init__(self, dyn, cmds, flags=0):
        self.dyn, self.cmds = dyn, cmds
        self.N, self.T = cmds.shape
        self.S = dyn.STATE_DIM
        self.sa_i, self.sr_i = 4, (12 if self.S == 24 else 8)
        cost = H.RacerQuadraticCost()
        p = cost.params
        p.speed_coeff = p.yaw_coeff = p.lateral_coeff = 0.0
        p.steer_coeff = 1.0
        sampler = H.GaussianDistribution(2, [1.0, 1.0])
        sampler.setControlCostCoeff([0.0, 0.0])
        self.e = H.Engine(dyn, cost, sampler, self.N, self.T, 1, flags=flags | H.FLAG_WRITEBACK_CONTROLS)
        self.e.set_solver(DT, 1.0, 0.0)
        self.x0 = np.zeros(self.S, np.float32)
        self.x0[self.sa_i], self.x0[self.sr_i] = SA0, SR0
        if self.S == 24:
            self.x0[8] = dyn.params.wheel_radius  # CG_POS_Z: the springs start near their rest length
        self.zeros = np.zeros((1, self.T, 2), np.float32)
        self.roll()

    def roll(self):
        eps = np.zeros((self.N, self.T, 2), np.float32)
        eps[:, :, 1] = self.cmds
        self.e.set_noise(eps)
        self.e.rollout_only(self.x0[None], self.zeros, 0, 0)
        np.testing.assert_array_equal(self.e.get_samples()[0][:, :, 1], self.cmds)
        self.costs = self.e.get_costs()[0].copy()
        return self.costs

    def trajectories(self, idx):
        outs, costs, _ = self.e.sample_trajectories(self.x0, self.zeros[0], np.asarray(idx))
        return outs, costs

    def close(self):
        self.e.close()


def _check_costs(name, case, form, idx):
    net = R.Blob(case.dyn.lstm_theta, case.dyn.hidden_dim, case.dyn.head_hidden)
    sp = R.SteerParams(case.dyn.params)
    assert np.all(np.isfinite(case.costs)), name
    want, bound = [], []
    for n in idx:
        r = R.steer_rollout(net, sp, SA0, SR0, case.cmds[n], DT, form)
        want.append(r["cost"])
        bound.append(r["e_cost"])
    return R.check(f"{name}: K1 costs", case.costs[idx], want, bound)


def _check_steps(name, case, idx, k1_simt=True):
    """The side rollouts' per-step steer angle (output 8) and rate (output 9): the run-time SIMT form (AuxDyn), whose
    per-step costs sum to K1's when K1 runs a SIMT form too."""
    net = R.Blob(case.dyn.lstm_theta, case.dyn.hidden_dim, case.dyn.head_hidden)
    sp = R.SteerParams(case.dyn.params)
    outs, costs = case.trajectories(idx)
    if k1_simt:
        np.testing.assert_allclose(costs.sum(axis=1), case.costs[idx], rtol=5e-6)
    for k, n in enumerate(idx):
        r = R.steer_rollout(net, sp, SA0, SR0, case.cmds[n], DT, "simt")
        R.check(f"{name}: side rollout {n} angle", outs[k, :, 8], r["angle"], r["e_angle"])
        R.check(f"{name}: side rollout {n} rate", outs[k, :, 9], r["rate"], r["e_rate"])


def _form(Hd, L1, flags):
    return "tc" if Hd == 32 and L1 <= 24 and not flags & H.FLAG_LSTM_SIMT else "simt"


GPU_SIZES = [(4, 20)] + SIMT_SIZES


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("Hd,L1", GPU_SIZES, ids=[f"H{h}_L{l}" for h, l in GPU_SIZES])
def test_simt_forms_against_float64(Hd, L1, regime):
    """K1 costs (compile-time form at (4, 20), run-time form elsewhere) and the side rollouts' per-step outputs, at an
    even and an odd horizon (the run-time form's hidden state ping-pongs on t & 1)."""
    for T, scale in ((32, 1.0), (33, 1e3)):
        dyn = make_dyn(Hd, L1, regime, control_range=scale)
        case = Case(dyn, commands(96, T, scale))
        name = f"LSTM simt H{Hd} L1 {L1} {regime} T{T} x{scale:g}"
        _check_costs(name, case, "simt", np.arange(0, 96, 3))
        _check_steps(name, case, np.arange(0, 96, 24))
        case.close()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("L1", TC_HEADS)
@pytest.mark.parametrize("simt", [False, True], ids=["tc", "simt_flag"])
def test_hidden_32_forms_against_float64(L1, regime, simt):
    """H = 32 at every head width the tensor-core form takes, on that form and under MPPIB_FLAG_LSTM_SIMT."""
    flags = H.FLAG_LSTM_SIMT if simt else 0
    for scale in (1.0, 1e3):
        dyn = make_dyn(32, L1, regime, control_range=scale)
        case = Case(dyn, commands(96, 32, scale), flags)
        _check_costs(f"LSTM {'simt' if simt else 'tc'} H32 L1 {L1} {regime} x{scale:g}", case, _form(32, L1, flags),
                     np.arange(0, 96, 3))
        if not simt and regime in ("synthetic", "init"):  # the tensor-core form ran: its costs are not the SIMT form's
            other = Case(dyn, case.cmds, H.FLAG_LSTM_SIMT)
            assert not np.array_equal(case.costs, other.costs)
            other.close()
        case.close()


@pytest.mark.gpu
@pytest.mark.parametrize("L1", AUTO_SIMT_HEADS)
def test_wide_heads_take_the_simt_form(L1):
    """At H = 32 and L1 > 24 the engine keeps the SIMT form by itself: costs bit-identical to an engine built with
    MPPIB_FLAG_LSTM_SIMT on the same commands, and within the SIMT bound of the float64 network."""
    cmds = commands(96, 32, 1.0)
    a = Case(make_dyn(32, L1, "init"), cmds)
    b = Case(make_dyn(32, L1, "init"), cmds, H.FLAG_LSTM_SIMT)
    np.testing.assert_array_equal(a.costs, b.costs)
    _check_costs(f"LSTM auto H32 L1 {L1}", a, "simt", np.arange(0, 96, 3))
    a.close()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STAGING))
@pytest.mark.parametrize("Hd,L1", [(4, 20), (7, 5), (32, 20)], ids=["H4_L20", "H7_L5", "H32_L20"])
def test_k1_staging_forms(Hd, L1, name, monkeypatch):
    """Resident TMA, plain loads (MPPIB_FLAG_NO_TMA) and the streaming form (MPPIB_STREAM=1) on each network form."""
    flags, env = STAGING[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    case = Case(make_dyn(Hd, L1, "init"), commands(256, 64, 1.0), flags)
    assert case.e.launch_info()["uses_tma"] == (name != "no_tma")
    _check_costs(f"LSTM {name} H{Hd} L1 {L1}", case, _form(Hd, L1, 0), np.arange(0, 256, 4))
    case.close()


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 15, 17, 1000, 1300])
def test_tensor_core_form_ragged_n(N):
    """The tensor-core form is warp-collective over 16 samples and keeps the rows past N running: ragged N, and a
    partial last block, leave every valid cost within the bound and the solve's U finite."""
    cmds = commands(N, 32, 1.0)
    case = Case(make_dyn(32, 20, "init"), cmds)
    idx = np.unique(np.linspace(0, cmds.shape[0] - 1, min(cmds.shape[0], 48)).astype(int))
    _check_costs(f"LSTM tc ragged N{N}", case, "tc", idx)
    U, _ = case.e.reduce_only()
    assert np.all(np.isfinite(U))
    case.close()


SUSPENSION = [(4, 20, 0), (7, 5, 0), (32, 20, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["synthetic", "init"])
@pytest.mark.parametrize("Hd,L1,flags", SUSPENSION, ids=["H4_L20", "H7_L5", "H32_L20_tc"])
def test_suspension_model_against_float64(Hd, L1, flags, regime):
    """RacerDubinsElevationSuspension: the compile-time form, one run-time size and the tensor-core form at H = 32."""
    case = Case(make_dyn(Hd, L1, regime, suspension=True), commands(96, 32, 1.0), flags)
    name = f"suspension {_form(Hd, L1, flags)} H{Hd} L1 {L1} {regime}"
    _check_costs(name, case, _form(Hd, L1, flags), np.arange(0, 96, 3))
    _check_steps(name, case, np.arange(0, 96, 32), _form(Hd, L1, flags) == "simt")
    case.close()


@pytest.mark.gpu
@pytest.mark.parametrize("edge", ["command", "weight"])
def test_fp16_operand_edge_takes_the_simt_form(edge):
    """Values the tensor-core form's FP16 operands cannot hold: a steering command range of +-1e5 (the command is input 2
    of the network), or one cell-gate weight of 3e4 (2.885 x 3e4 after pre-scaling). The engine keeps the SIMT form there
    (costs bit-identical to MPPIB_FLAG_LSTM_SIMT, finite, within the SIMT bound of the float64 network), and goes back to
    the tensor-core form when the blobs are set back in range."""
    scale = 1e5 if edge == "command" else 1.0
    dyn = make_dyn(32, 20, "init", control_range=scale)
    lstm, head = weights(32, 20, "init")
    wide = lstm.copy()
    if edge == "weight":
        wide[3 * 32 * 32 + 5 * 32 + 7] = 3e4  # W_cm[5][7]
    dyn.setAllValues(wide, head)
    cmds = commands(96, 32, scale)
    if edge == "command":
        assert np.abs(cmds).max() >= 65520.0
    a = Case(dyn, cmds)
    b = Case(dyn, cmds, H.FLAG_LSTM_SIMT)
    np.testing.assert_array_equal(a.costs, b.costs)
    _check_costs(f"LSTM fp16 edge {edge}", a, "simt", np.arange(0, 96, 3))
    # back in range: the tensor-core form again (its costs differ from the SIMT form's), within its bound
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    dyn.setAllValues(lstm, head)
    for c in (a, b):
        c.cmds = commands(96, 32, 1.0)
        c.e.push_params()
        c.roll()
    assert not np.array_equal(a.costs, b.costs)
    _check_costs(f"LSTM fp16 edge {edge}, back in range", a, "tc", np.arange(0, 96, 3))
    a.close()
    b.close()
