"""The Autorally 6-32-32-4 network against a float64 network (tests/autorally_nn_f64.py) on every form that evaluates it:
the host twin (CPU), FFMA2 (plain FP32), mma.sync (FP16 hi / lo split, the default, in the generic, warp-specialised and
side kernels) and wgmma (3xTF32).

The weights are synthetic: the reference's trained Autorally network is a git-LFS stub, so each regime below is a scaled
or reshaped draw of workloads.synthetic_nn_weights, chosen for the arithmetic it exercises:
  * synthetic: the draw itself (the bench's network);
  * x6: six times it, so the tanh layers saturate and the mma.sync form's folded biases b' = b + sum W cancel;
  * tiny: 1e-6 times it, so the FP16 hi parts of the weights are subnormal;
  * mixed: every weight row spans 1e-6 .. 4 in magnitude, so the FP16 subnormal floor sits beside full-precision terms;
  * large: large inputs (vx 20, yaw rate 3, roll 0.5) and wider control ranges.
For each regime, dt and T keep every compared sample's forward speed at 0.5 or above (asserted), since the slip term
atan(vy / |vx|) has a kink at vx = 0.

What the GPU tests observe is the network alone: ARStandardCost with its track and crash terms off on a constant costmap,
only the speed (desired speed away from the trajectories) and slip terms live, and no control cost, on commands chosen
through set_noise. Every comparison asserts |float32 - float64| <= 2 x bound + 4 ulps with the running bound of
autorally_nn_f64 (factor fixed beforehand) and prints the largest error / bound ratio."""
import json
import os

import numpy as np
import pytest

import mppi_generic_b200 as M
from mppi_generic_b200 import workloads as W
from tests import autorally_nn_f64 as R

H = M.host
f16, f32 = np.float16, np.float32
REGIMES = ["synthetic", "x6", "tiny", "mixed", "large"]
DESIRED_SPEED = 10.0


def weights(regime, seed=1):
    th = W.synthetic_nn_weights(seed).astype(np.float64)
    if regime == "x6":
        th = 6.0 * th
    elif regime == "tiny":
        th = 1e-6 * th
    elif regime == "mixed":
        rng = np.random.RandomState(11)
        o = 0
        for a, b in ((6, 32), (32, 32), (32, 4)):
            for j in range(b):  # row j of W: magnitudes 1e-6 .. 4, log-spaced, in a random order, random signs
                mag = np.logspace(-6.0, np.log10(4.0), a)[rng.permutation(a)]
                th[o + j * a:o + (j + 1) * a] = mag * rng.choice([-1.0, 1.0], a) / a
            o += a * b + b
    return th.astype(np.float32)


# regime -> (x0, control ranges, command scale, dt, T)
SCENARIOS = {
    "synthetic": ([0.0, 0.0, 0.0, 0.0, 4.0, 0.0, 0.0], [(-1.0, 1.0), (-2.0, 2.0)], 0.6, 0.02, 100),
    "x6": ([0.0, 0.0, 0.0, 0.0, 4.0, 0.0, 0.0], [(-1.0, 1.0), (-2.0, 2.0)], 0.6, 0.01, 64),
    "tiny": ([0.0, 0.0, 0.0, 0.0, 4.0, 0.0, 0.0], [(-1.0, 1.0), (-2.0, 2.0)], 0.6, 0.02, 100),
    "mixed": ([0.0, 0.0, 0.0, 0.0, 4.0, 0.0, 0.0], [(-1.0, 1.0), (-2.0, 2.0)], 0.6, 0.01, 64),
    "large": ([1.0, -2.0, 0.3, 0.5, 20.0, 0.5, 3.0], [(-5.0, 5.0), (-8.0, 8.0)], 4.0, 0.01, 64),
}


def make_dyn(regime, ranges=None, theta=None):
    dyn = H.NeuralNetModel(ranges or SCENARIOS[regime][1])
    dyn.updateModel([6, 32, 32, 4], weights(regime) if theta is None else theta)
    return dyn


def make_cost(robust=False):
    """ARStandardCost (or ARRobustCost, heading term off) with only the speed and slip terms: no track or crash cost,
    slip and boundary limits out of reach, a constant zero costmap."""
    cost = H.ARRobustCost() if robust else H.ARStandardCost()
    p = cost.params
    if robust:
        p.heading_coeff = 0.0
    p.track_coeff = p.crash_coeff = 0.0
    p.max_slip_ang, p.boundary_threshold = 1e6, 1e6
    p.speed_coeff, p.slip_coeff, p.desired_speed = 4.25, 10.0, DESIRED_SPEED
    cost.setCostmap(np.zeros((8, 8, 4), np.float32), 8, 8)
    return cost


def commands(n, T, scale, seed=5):
    """Noise [n][T][2] on a zero mean with unit standard deviation, i.e. the commands themselves; the first sample is all
    zero, the engine's zero-noise sample."""
    rng = np.random.RandomState(seed)
    eps = (rng.uniform(-1.0, 1.0, (n, T, 2)) * scale).astype(np.float32)
    eps[0] = 0.0
    return eps


def reference(regime, eps, form, dyn=None, x0=None, dt=None, robust=False):
    dyn = dyn or make_dyn(regime)
    sc = SCENARIOS[regime]
    r = R.rollout(R.Net(dyn.nn_theta), R.Params(dyn, make_cost(robust)), sc[0] if x0 is None else x0, eps,
                  sc[3] if dt is None else dt, form)
    assert np.all(r["vx_min"] >= 0.5), (regime, float(r["vx_min"].min()))  # the slip term is smooth along the samples
    return r


# ---- the float64 network itself ------------------------------------------------------------------------------------------
def test_known_answer_all_ones():
    """ar_dynamics_nn_test.cu (computeDynamics): every weight and bias 1, state 0, u = (1, -1) => s_der[3..6] = 33."""
    net = R.Net(np.ones(R.NUM_PARAMS, np.float32))
    out = R.forward(net, np.array([0.0, 0.0, 0.0, 0.0, 1.0, -1.0]))
    np.testing.assert_allclose(out, [33.0] * 4, rtol=1e-6)
    with open(os.path.join(os.path.dirname(__file__), "golden", "reference_known_answers.json")) as f:
        assert "lstm_all_ones_outputs" in json.load(f)  # the same fixture file the LSTM restatement pins


def test_hand_checked_blob():
    """One distinct value per block (W1, b1, W2, b2, W3, b3), each W with a single nonzero entry off its diagonal, so that
    any permutation of the layout, or a transposed block, changes the output; the expected output is written out by hand."""
    th = np.zeros(R.NUM_PARAMS, np.float32)
    th[0 * 6 + 3] = 0.7      # W1[0][3]: neuron 0 reads input 3 (yaw rate)
    th[192:224] = -0.2       # b1
    th[224 + 5 * 32 + 0] = 1.3  # W2[5][0]: neuron 5 reads layer-1 neuron 0
    th[1248:1280] = 0.1      # b2
    th[1280 + 2 * 32 + 5] = -2.5  # W3[2][5]: output 2 reads layer-2 neuron 5
    th[1408:1412] = [0.05, -0.15, 0.25, 0.35]
    x = np.array([0.3, 4.0, -0.2, 0.9, 0.5, -1.0])
    f = lambda v: float(np.float32(v))  # noqa: E731
    a1_0 = np.tanh(f(0.7) * 0.9 + f(-0.2))
    a1_rest = np.tanh(f(-0.2))
    a2_5 = np.tanh(f(1.3) * a1_0 + f(0.1))
    a2_rest = np.tanh(f(0.1))
    want = np.array([f(0.05), f(-0.15), f(-2.5) * a2_5 + f(0.25), f(0.35)])
    got = R.forward(R.Net(th), x)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-14)
    assert a1_rest != a1_0 and a2_rest != a2_5
    # and the host twin's state derivative on the same blob
    dyn = make_dyn("synthetic", theta=th)
    s = np.array([0.0, 0.0, 0.0, 0.3, 4.0, -0.2, 0.9], np.float32)
    _, xd, _ = dyn.step(s, np.array([0.5, -1.0], np.float32), 0.01)
    out, eo = R.net_bound(R.Net(th), np.concatenate([s[3:], [0.5, -1.0]]).astype(np.float32).astype(np.float64), "host")
    R.check("host twin, hand blob", xd[3:], out[0], eo[0])


# ---- bit-level emulations of each device form ----------------------------------------------------------------------------
def _acc(c, s, trunc):
    """One MMA: the incoming FP32 accumulator c plus the exact sum s, rounded to FP32 (to nearest, or towards zero)."""
    v = np.asarray(c, np.float64) + s
    r = v.astype(f32)
    if trunc:
        r = np.where(np.abs(r.astype(np.float64)) > np.abs(v), np.nextafter(r, f32(0)), r).astype(f32)
    return r


def _r(z, s):
    """r = rcp(ex2(z) + 1), ex2 and rcp perturbed by s times their documented error (2 ulp, 1 ulp)."""
    with np.errstate(over="ignore"):
        e = (np.exp2(z.astype(np.float64)) * (1.0 + s * 2.0 ** -22)).astype(f32)
        d = (e + f32(1.0)).astype(f32)
        return ((1.0 / d.astype(np.float64)) * (1.0 + s * 2.0 ** -23)).astype(f32)


def _split16(v):
    hi = v.astype(f16)
    lo = (v - hi.astype(f32)).astype(f16)
    return hi.astype(np.float64), lo.astype(np.float64)


def mma_net(net, variant="three", trunc=False, s=0.0):
    """nn_mma.cuh forward_frag on float32 inputs [B][6]: folded weights, FP16 split operands, products exact, one FP32
    rounding per MMA in its issue order. variant "two" drops the a_hi w_lo product, "single" keeps a_hi w_hi alone."""
    W1, b1, W2, b2, W3, b3 = (np.asarray(v, f32) for v in (net.mW1, net.mb1, net.mW2, net.mb2, net.mW3, net.mb3))

    def products(ah, al, wh, wl):
        p = [ah @ wh.T, al @ wh.T, ah @ wl.T]
        return p if variant == "three" else (p[:2] if variant == "two" else p[:1])

    def f(x):
        xh, xl = _split16(np.asarray(x, f32))
        wh, wl = _split16(W1)
        c = np.broadcast_to(b1, (x.shape[0], 32)).astype(f32)
        p = products(xh, xl, wh, wl)
        c = _acc(c, sum(p[:2]), trunc)  # the k16 MMA: a_hi w_hi + a_lo w_hi
        if len(p) > 2:
            c = _acc(c, p[2], trunc)    # the k8 MMA: a_hi w_lo
        r1 = _r(c, s)
        rh, rl = _split16(r1)
        wh, wl = _split16(W2)
        c = np.broadcast_to(b2, (x.shape[0], 32)).astype(f32)
        for j in range(2):
            J = slice(16 * j, 16 * j + 16)
            for q in products(rh[:, J], rl[:, J], wh[:, J], wl[:, J]):
                c = _acc(c, q, trunc)
        r2 = _r(c, s)
        rh, rl = _split16(r2)
        wh, wl = _split16(W3)
        o = np.broadcast_to(b3, (x.shape[0], 4)).astype(f32)
        o2 = np.zeros((x.shape[0], 4), f32)
        p0 = products(rh[:, :16], rl[:, :16], wh[:, :16], wl[:, :16])
        p1 = products(rh[:, 16:], rl[:, 16:], wh[:, 16:], wl[:, 16:])
        for a, b in zip(p0, p1):
            o = _acc(o, a, trunc)
            o2 = _acc(o2, b, trunc)
        return (o + o2).astype(f32)
    return f


def ffma2_net(net, s=0.0):
    """AutorallyNNDynamics::layer: k-ascending FMA chains from zero, the bias last, tanh_fast on each hidden value."""
    Ws = [np.asarray(w, f32).astype(np.float64) for w in (net.W1, net.W2, net.W3)]
    bs = [np.asarray(b, f32) for b in (net.b1, net.b2, net.b3)]

    def tanh_fast(z):
        t = _r((z * f32(R.K_TANH)).astype(f32), s)
        return (1.0 - 2.0 * t.astype(np.float64)).astype(f32)

    def f(x):
        a = np.asarray(x, f32)
        for i in range(3):
            acc = np.zeros((a.shape[0], Ws[i].shape[0]), f32)
            for k in range(Ws[i].shape[1]):
                acc = (a[:, k:k + 1].astype(np.float64) * Ws[i][:, k] + acc).astype(f32)
            a = (acc + bs[i]).astype(f32)
            if i < 2:
                a = tanh_fast(a)
        return a
    return f


def _rna_tf32(v):
    b = np.asarray(v, f32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(f32)


def _trunc_tf32(v):
    return (np.asarray(v, f32).view(np.uint32) & np.uint32(0xFFFFE000)).view(f32)


def wgmma_net(net, trunc=False, s=0.0):
    """rollout_kernel_nn_tc.cuh: hi = rna_tf32(v), lo = v - hi read truncated to TF32, three products per K block of 8,
    the bias as a K column against a constant one, tanh = 1 - 2 r."""
    f = np.float64
    layers = [(np.asarray(net.tW1, f32), np.asarray(net.tb1, f32), True, False),
              (np.asarray(net.tW2, f32), np.asarray(net.tb2, f32), True, True),
              (np.asarray(net.W3, f32), np.asarray(net.b3, f32), False, True)]

    def parts(v):
        hi = _rna_tf32(v)
        return hi.astype(f), _trunc_tf32((v - hi).astype(f32)).astype(f)

    def f_(x):
        a = np.asarray(x, f32)
        B = a.shape[0]
        for Wl, bl, act, bias_block in layers:
            if not bias_block:  # layer 1: K = 8 = 6 inputs, the bias column, a zero
                A = np.concatenate([a, np.ones((B, 1), f32), np.zeros((B, 1), f32)], 1)
                Wb = np.concatenate([Wl, bl[:, None], np.zeros((Wl.shape[0], 1), f32)], 1)
                ah, al = parts(A)
                wh, wl = parts(Wb)
                c = _acc(np.zeros((B, Wl.shape[0]), f32), ah @ wh.T, trunc)
                c = _acc(c, al @ wh.T, trunc)
                c = _acc(c, ah @ wl.T, trunc)
            else:
                ah, al = parts(a)
                wh, wl = parts(Wl)
                c = np.zeros((B, Wl.shape[0]), f32)
                for kb in range(4):
                    K = slice(8 * kb, 8 * kb + 8)
                    c = _acc(c, ah[:, K] @ wh[:, K].T, trunc)
                    c = _acc(c, al[:, K] @ wh[:, K].T, trunc)
                    c = _acc(c, ah[:, K] @ wl[:, K].T, trunc)
                bh, bl_ = parts(bl)
                c = _acc(c, np.broadcast_to(bh, c.shape), trunc)
                c = _acc(c, np.broadcast_to(bl_, c.shape), trunc)
            a = (1.0 - 2.0 * _r(c, s).astype(f)).astype(f32) if act else c
        return a
    return f_


def host_net(dyn):
    """The host twin's network, read through its state derivative at yaw 0."""
    def f(x):
        out = np.empty((x.shape[0], 4), f32)
        for b in range(x.shape[0]):
            s = np.array([0.0, 0.0, 0.0, *x[b, :4]], f32)
            _, xd, _ = dyn.step(s, x[b, 4:], 0.01)
            out[b] = xd[3:]
        return out
    return f


def roll32(net32, cp, x0, eps, dt):
    """A float32 rollout with the network `net32`: kinematics, Euler update and cost as the kernels compute them."""
    dt = f32(dt)
    B, T, _ = eps.shape
    x = np.tile(np.asarray(x0, f32), (B, 1))
    run = np.zeros(B, f32)
    states = np.zeros((B, T, 7), f32)
    for t in range(T):
        u = np.clip(eps[:, t], cp.lo.astype(f32), cp.hi.astype(f32)).astype(f32)
        cs, sn = np.cos(x[:, 2]), np.sin(x[:, 2])
        xd = np.zeros((B, 7), f32)
        xd[:, 0] = cs * x[:, 4] - sn * x[:, 5]
        xd[:, 1] = sn * x[:, 4] + cs * x[:, 5]
        xd[:, 2] = -x[:, 6]
        xd[:, 3:] = net32(np.concatenate([x[:, 3:], u], 1))
        x = (x + xd * dt).astype(f32)
        states[:, t] = x
        e = x[:, 4] - f32(cp.desired)
        slip = -np.arctan(x[:, 5] / np.abs(x[:, 4]))
        c = (f32(cp.speed) * (e * e) + f32(cp.slip) * (slip * slip)).astype(f32)
        run = (run + c).astype(f32)
    return states, (run / f32(T)).astype(f32)


EMULATIONS = {
    "ffma2": lambda net, s: ffma2_net(net, s),
    "mma": lambda net, s: mma_net(net, "three", trunc=s != 0.0, s=s),
    "wgmma": lambda net, s: wgmma_net(net, trunc=s != 0.0, s=s),
}


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("form", list(EMULATIONS))
def test_emulated_forms_lie_within_the_bound(form, regime):
    """Each device form emulated bit for bit on the CPU, with round-to-nearest MMAs and exact-rounded ex2 / rcp, and with
    truncating MMAs and ex2 / rcp pushed to either end of their documented error: per-step states and costs within the
    form's bound."""
    x0, _, scale, dt, T = SCENARIOS[regime]
    T = min(T, 48)
    eps = commands(12, T, scale)
    dyn = make_dyn(regime)
    net = R.Net(dyn.nn_theta)
    cp = R.Params(dyn, make_cost())
    r = reference(regime, eps, form, dyn, dt=dt)
    for s in (0.0, 1.0, -1.0):
        states, cost = roll32(EMULATIONS[form](net, s), cp, x0, eps, dt)
        R.check(f"emulated {form} {regime} s{s:+g}: states", states, r["states"], r["e_states"])
        R.check(f"emulated {form} {regime} s{s:+g}: costs", cost, r["cost"], r["e_cost"])


@pytest.mark.parametrize("variant", ["two", "single"])
def test_subtly_wrong_splits_exceed_the_bound(variant):
    """The bound would catch a subtly wrong kernel: at the synthetic regime, a two-product split that drops a_hi w_lo, and
    a single FP16 product, leave the mma.sync bound somewhere along the rollout."""
    x0, _, scale, dt, T = SCENARIOS["synthetic"]
    eps = commands(12, T, scale)
    dyn = make_dyn("synthetic")
    net = R.Net(dyn.nn_theta)
    r = reference("synthetic", eps, "mma", dyn)
    states, cost = roll32(mma_net(net, variant), R.Params(dyn, make_cost()), x0, eps, dt)
    err = np.abs(states - r["states"])
    over = err > 2.0 * r["e_states"] + R.ulps(r["states"])
    assert over.any(), (variant, float((err / (r["e_states"] + R.ulps(r["states"]))).max()))


def test_cost_bound_is_below_the_references_bar():
    """The mma.sync form's cost bound at the synthetic regime (the bench's network, dt 0.02, T 100) is below the reference's
    1e-4 per-trajectory bar, relative to max(|cost|, 1) (rollout_kernel_tests.cu:258): up to 2.6e-5 here (FFMA2 1.9e-5,
    wgmma 2.5e-5), so the bound is a sharper bar than the reference's."""
    x0, _, scale, dt, T = SCENARIOS["synthetic"]
    eps = commands(32, T, scale)
    for form in ("mma", "ffma2", "wgmma"):
        r = reference("synthetic", eps, form)
        rel = r["e_cost"] / np.maximum(np.abs(r["cost"]), 1.0)
        print(f"{form}: cost bound / max(|cost|, 1) up to {rel.max():.3g}")
        assert rel.max() < 1e-4, (form, rel.max())


@pytest.mark.parametrize("regime", REGIMES)
def test_host_twin_against_float64(regime):
    """NeuralNetModel.step, the host twin the controller's roll-forward uses, over the scenario's horizon on clamped
    commands: every state within the host form's bound."""
    x0, _, scale, dt, T = SCENARIOS[regime]
    eps = commands(4, T, scale)
    dyn = make_dyn(regime)
    r = reference(regime, eps, "host", dyn)
    cp = R.Params(dyn, make_cost())
    for b in range(eps.shape[0]):
        x = np.asarray(x0, f32)
        got = np.zeros((T, 7), f32)
        for t in range(T):
            u = np.clip(eps[b, t], cp.lo, cp.hi).astype(f32)
            x, _, _ = dyn.step(x, u, dt)
            got[t] = x
        R.check(f"host {regime} sample {b}", got, r["states"][b], r["e_states"][b])


# ---- GPU ---------------------------------------------------------------------------------------------------------------
class Case:
    """One engine of N = len(eps) rollouts over chosen commands (the noise, on a zero mean and unit standard deviation),
    K1 run once through rollout_only; `x0` [D][7]."""

    def __init__(self, dyn, eps, x0, dt, flags=0, cost=None):
        self.dyn, self.eps, self.x0, self.dt = dyn, eps, np.asarray(x0, f32).reshape(-1, 7), dt
        self.N, self.T, _ = eps.shape
        self.D = self.x0.shape[0]
        sampler = H.GaussianDistribution(2, [1.0, 1.0])
        sampler.setControlCostCoeff([0.0, 0.0])
        self.e = H.Engine(dyn, cost or make_cost(), sampler, self.N, self.T, self.D, flags=flags | H.FLAG_WRITEBACK_CONTROLS)
        self.e.set_solver(dt, 1.0, 0.0)
        self.roll()

    def roll(self):
        self.e.set_noise(self.eps)
        self.e.rollout_only(self.x0, np.zeros((self.D, self.T, 2), f32), 0, 0)  # stride 0: every step takes the noise
        cp = R.Params(self.dyn, make_cost())
        want = np.clip(self.eps, cp.lo.astype(f32), cp.hi.astype(f32))
        np.testing.assert_array_equal(self.e.get_samples()[0], want)  # the controls are the chosen commands
        self.costs = self.e.get_costs().copy()
        return self.costs

    def close(self):
        self.e.close()


def _idx(N, n=48):
    return np.unique(np.linspace(0, N - 1, min(N, n)).astype(int))


def _check_costs(name, case, form, regime, idx=None, d=0, robust=False):
    idx = _idx(case.N) if idx is None else idx
    assert np.all(np.isfinite(case.costs)), name
    r = reference(regime, case.eps[idx], form, case.dyn, x0=case.x0[d], dt=case.dt, robust=robust)
    return R.check(f"{name}: K1 costs", case.costs[d, idx], r["cost"], r["e_cost"])


MAIN_FORMS = {"mma": 0, "ffma2": H.FLAG_NN_FFMA2, "wgmma": H.FLAG_NN_TENSOR}
BX = 64  # MPPIB_BX: samples per CTA, so that each form's block width is known


def _block(form, pspw=None, spw=None, spt=1):
    """The block width of each K1 form at BX samples per CTA: the warp-specialised kernel's 32 / pspw producers and one
    consumer per 32 samples; the generic kernel's 32 / spw lanes per sample (or one thread per spt samples); the wgmma
    kernel's 128 rows."""
    if form == "wgmma":
        return 128
    if pspw:
        return (32 // pspw + 1) * BX
    if spw:
        return BX * 32 // spw
    return BX // spt


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("form", list(MAIN_FORMS))
def test_forms_against_float64(form, regime, monkeypatch):
    """K1 per-sample costs of the default form (warp-specialised mma.sync), FFMA2 and wgmma in every regime."""
    monkeypatch.setenv("MPPIB_BX", str(BX))
    x0, _, scale, dt, T = SCENARIOS[regime]
    case = Case(make_dyn(regime), commands(512, T, scale), x0, dt, MAIN_FORMS[form])
    assert case.e.launch_info()["block"] == _block(form, pspw=8 if form == "mma" else None)
    _check_costs(f"{form} {regime}", case, form, regime)
    case.close()


# name -> (flags, environment, block width, bound)
VARIANTS = {
    "generic_spw32": (0, {"MPPIB_SPW": "32"}, _block("mma", spw=32), "mma"),
    "generic_spw16": (0, {"MPPIB_SPW": "16"}, _block("mma", spw=16), "mma"),
    "generic_spw8": (0, {"MPPIB_SPW": "8"}, _block("mma", spw=8), "mma"),
    "ws_pspw32": (0, {"MPPIB_WS_PSPW": "32"}, _block("mma", pspw=32), "mma"),
    "ws_pspw16": (0, {"MPPIB_WS_PSPW": "16"}, _block("mma", pspw=16), "mma"),
    "ws_pspw8": (0, {"MPPIB_WS_PSPW": "8"}, _block("mma", pspw=8), "mma"),
    "ws_pspw16_stream": (0, {"MPPIB_WS_PSPW": "16", "MPPIB_STREAM": "1"}, _block("mma", pspw=16), "mma"),
    "ws_pspw8_no_tma": (H.FLAG_NO_TMA, {"MPPIB_WS_PSPW": "8"}, _block("mma", pspw=8), "mma"),
    "ffma2_spt2": (H.FLAG_NN_FFMA2, {"MPPIB_SPT": "2"}, _block("ffma2", spt=2), "ffma2"),
    "ffma2_no_tma": (H.FLAG_NN_FFMA2 | H.FLAG_NO_TMA, {}, _block("ffma2"), "ffma2"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["synthetic", "x6", "mixed"])
@pytest.mark.parametrize("name", list(VARIANTS))
def test_kernel_variants_against_float64(name, regime, monkeypatch):
    """The generic kernel at 32 / 16 / 8 samples per warp, the warp-specialised kernel at 32 / 16 / 8 samples per producer
    (resident, streaming, without TMA), and FFMA2 at two samples per thread: the intended kernel ran (its block width, its
    staging), and its costs are within the bound of its network form."""
    flags, env, block, form = VARIANTS[name]
    monkeypatch.setenv("MPPIB_BX", str(BX))
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    x0, _, scale, dt, T = SCENARIOS[regime]
    case = Case(make_dyn(regime), commands(300, T, scale), x0, dt, flags)
    info = case.e.launch_info()
    assert info["block"] == block, info
    assert info["uses_tma"] == (not flags & H.FLAG_NO_TMA), info
    _check_costs(f"{name} {regime}", case, form, regime)
    case.close()


SHAPES = [(1037, 100), (677, 64), (20, 64), (1037, 1), (677, 33), (300, 7)]


@pytest.mark.gpu
@pytest.mark.parametrize("form", list(MAIN_FORMS))
@pytest.mark.parametrize("N,T", SHAPES, ids=[f"N{n}_T{t}" for n, t in SHAPES])
def test_shapes_against_float64(N, T, form):
    """Ragged N (1037, 677), N < 32, T = 1, and odd T (33, 7: the warp-specialised kernel's one-step last group, T * C not
    a multiple of 4, so plain-load staging); every valid sample's cost within the bound and the solve's U finite."""
    x0, _, scale, dt, _ = SCENARIOS["synthetic"]
    case = Case(make_dyn("synthetic"), commands(N, T, scale), x0, dt, MAIN_FORMS[form])
    _check_costs(f"{form} N{N} T{T}", case, form, "synthetic")
    U, _ = case.e.reduce_only()
    assert np.all(np.isfinite(U))
    case.close()


@pytest.mark.gpu
def test_bench_size_against_float64():
    """The default form at the bench's C4 size, 32768 x 100, on 64 samples spread over the population."""
    x0, _, scale, dt, T = SCENARIOS["synthetic"]
    case = Case(make_dyn("synthetic"), commands(32768, T, scale), x0, dt)
    _check_costs("mma C4 32768 x 100", case, "mma", "synthetic", idx=_idx(32768, 64))
    case.close()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["synthetic", "large"])
def test_two_distributions_against_float64(regime):
    """D = 2 (Tube-MPPI's two systems in one thread, the generic kernel on the default form): each distribution from its
    own start state."""
    x0, _, scale, dt, T = SCENARIOS[regime]
    x1 = np.array(x0, f32) + np.array([0.5, -0.3, 0.2, -0.1, 0.5, 0.1, -0.4], f32)
    case = Case(make_dyn(regime), commands(300, T, scale), [x0, x1], dt)
    for d in range(2):
        _check_costs(f"D2 {regime} distribution {d}", case, "mma", regime, d=d)
    case.close()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["synthetic", "x6", "large"])
@pytest.mark.parametrize("form", ["mma", "ffma2"])
def test_side_rollouts_against_float64(form, regime):
    """sample_trajectories and nominal_trajectory (their one-lane-per-rollout instantiation of the form's network): every
    state output of every step within the bound, x, y and yaw included."""
    x0, _, scale, dt, T = SCENARIOS[regime]
    dyn = make_dyn(regime)
    case = Case(dyn, commands(256, T, scale), x0, dt, MAIN_FORMS[form])
    idx = np.array([0, 1, 77, 255])
    outs, costs, _ = case.e.sample_trajectories(case.x0[0], np.zeros((T, 2), f32), idx)
    r = reference(regime, case.eps[idx], form, dyn, x0=x0, dt=dt)
    R.check(f"{form} {regime}: sampled trajectories", outs[:, :, :7], r["states"], r["e_states"])
    R.check(f"{form} {regime}: sampled step costs", costs.astype(np.float64).sum(axis=1), r["cost"],
            r["e_cost"])
    # the roll-forward: states[0] = x0, then T - 1 steps under U[0 .. T - 2]
    Us = case.eps[77][None]
    _, states, outputs = case.e.nominal_trajectory(case.x0, Us)
    r = reference(regime, Us[:, :-1], form, dyn, x0=x0, dt=dt)
    np.testing.assert_array_equal(states[0, 0], case.x0[0])
    R.check(f"{form} {regime}: nominal states", states[0, 1:], r["states"][0], r["e_states"][0])
    R.check(f"{form} {regime}: nominal outputs", outputs[0, 1:, :7], r["states"][0], r["e_states"][0])
    case.close()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_ddp_jacobians_against_float64(regime):
    """[A | B] from ddp_feedback(want_jacobians=True) at 16 points against the exact Jacobian of the float64 network, under
    the derived bound of computeGrad's FP32 evaluation."""
    dyn = make_dyn(regime)
    net = R.Net(dyn.nn_theta)
    e = H.Engine(dyn, H._standalone_cost(dyn.DYN_ID), H.GaussianDistribution(2), 64, 8, 1)
    e.set_solver(0.01, 1.0, 0.0)
    rng = np.random.RandomState(5)
    x0, ranges = SCENARIOS[regime][0], SCENARIOS[regime][1]
    for _ in range(16):
        x = (np.asarray(x0) + rng.randn(7) * [1, 1, 1, 0.3, 2, 0.5, 0.5]).astype(f32)
        u = np.array([rng.uniform(*ranges[0]), rng.uniform(*ranges[1])], f32) * f32(0.9)
        _, _, _, jac = e.ddp_feedback(x, np.stack([x, x]), np.stack([u, u]), want_jacobians=True)
        A, E = R.jacobian_bound(net, x, u)
        R.check(f"DDP Jacobian {regime}", jac[0], A, E)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("edge", ["weight", "command"])
def test_fp16_operand_edge_keeps_the_ffma2_form(edge):
    """Values the mma.sync form's FP16 operands cannot hold: one W2 entry of 12000 (-69240 once load_weights scales it by
    -4 log2 e), or a steering control range of +-7e4 with commands that reach it. The engine keeps the FFMA2 form there,
    even under MPPIB_FLAG_NN_MMA: the same launch as MPPIB_FLAG_NN_FFMA2, bit-identical costs, finite and within the
    FFMA2 bound; and it goes back to the mma.sync form once the blobs are set back in range."""
    x0, ranges, scale, dt, T = SCENARIOS["synthetic"]
    theta = weights("synthetic")
    if edge == "weight":
        wide = theta.copy()
        wide[224 + 9 * 32 + 17] = 12000.0  # W2[9][17]
        dyn, eps = make_dyn("synthetic", theta=wide), commands(96, T, scale)
    else:
        dyn = make_dyn("synthetic", ranges=[(-7e4, 7e4), ranges[1]])
        eps = commands(96, T, scale)
        eps[1:, :, 0] *= 7e4 / scale * 1.25
        assert np.abs(np.clip(eps[:, :, 0], -7e4, 7e4)).max() == 7e4
    cases = [Case(dyn, eps, x0, dt, flags) for flags in (0, H.FLAG_NN_MMA, H.FLAG_NN_FFMA2)]
    for c in cases[:2]:
        assert c.e.launch_info() == cases[2].e.launch_info()
        np.testing.assert_array_equal(c.costs, cases[2].costs)
    _check_costs(f"fp16 edge {edge}", cases[0], "ffma2", "synthetic")
    # back in range: the mma.sync form again, within its bound
    dyn.updateModel([6, 32, 32, 4], theta)
    dyn.setControlRanges(ranges)
    fresh = Case(dyn, commands(96, T, scale), x0, dt)
    for c in cases:
        c.eps = fresh.eps
        c.e.push_params()
        c.roll()
    assert cases[0].e.launch_info() == fresh.e.launch_info() != cases[2].e.launch_info()
    np.testing.assert_array_equal(cases[0].costs, fresh.costs)
    assert not np.array_equal(cases[0].costs, cases[2].costs)
    _check_costs(f"fp16 edge {edge}, back in range", cases[0], "mma", "synthetic")
    for c in cases + [fresh]:
        c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["synthetic", "x6", "large"])
@pytest.mark.parametrize("form", ["mma", "ffma2"])
def test_robust_cost_against_float64(form, regime, monkeypatch):
    """ARRobustCost's warp-specialised kernel (default form) and its FFMA2 form, the penalties made continuous: crash and
    heading coefficients zero, slip and boundary thresholds out of reach, so the cost is slip_coeff |slip| + speed_coeff
    |vx - desired|."""
    monkeypatch.setenv("MPPIB_BX", str(BX))
    x0, _, scale, dt, T = SCENARIOS[regime]
    case = Case(make_dyn(regime), commands(300, T, scale), x0, dt, MAIN_FORMS[form], cost=make_cost(robust=True))
    assert case.e.launch_info()["block"] == _block(form, pspw=8 if form == "mma" else None)
    _check_costs(f"ARRobustCost {form} {regime}", case, form, regime, robust=True)
    case.close()


@pytest.mark.gpu
@pytest.mark.parametrize("form", list(MAIN_FORMS))
def test_all_ones_known_answer_on_each_form(form):
    """ar_dynamics_nn_test.cu's known answer on the device: every weight 1, state 0, u = (1, -1) => s_der[3..6] = 33, read
    through one step of dt = 0.01 (vx = vy = 0.33), on a control range of +-2 so that the mma.sync form keeps its FP16
    operands. And with the +-FLT_MAX default range, which the mma.sync form cannot split, the default engine takes the
    FFMA2 launch and its costs."""
    theta = np.ones(R.NUM_PARAMS, np.float32)
    eps = np.tile(np.array([1.0, -1.0], f32), (64, 1, 1))
    eps[0] = 0.0
    x0 = np.zeros(7, f32)
    case = Case(make_dyn("synthetic", ranges=[(-2.0, 2.0)] * 2, theta=theta), eps, x0, 0.01, MAIN_FORMS[form])
    want = 4.25 * (0.33 - DESIRED_SPEED) ** 2 + 10.0 * np.arctan(1.0) ** 2
    np.testing.assert_allclose(case.costs[0, 1:], want, rtol=2e-6)
    case.close()
    if form == "mma":
        wide = [Case(make_dyn("synthetic", ranges=[(-H.FLT_MAX, H.FLT_MAX)] * 2, theta=theta), eps, x0, 0.01, flags)
                for flags in (0, H.FLAG_NN_FFMA2)]
        assert wide[0].e.launch_info() == wide[1].e.launch_info()
        np.testing.assert_array_equal(wide[0].costs, wide[1].costs)
        np.testing.assert_allclose(wide[0].costs[0, 1:], want, rtol=2e-6)
        for c in wide:
            c.close()
