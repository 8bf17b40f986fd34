"""Float64 restatement of the RACER steering network and of the closed steering subsystem around it, with a running
first-order bound on how far a correct float32 evaluation of each device form may sit from it.

Semantics (written from the reference, not from oracle/mppi_oracle.cpp):
  * packed blob, LSTMHelper (lstm_helper.cu:72-88): W_im W_fm W_om W_cm [H x H] | W_ii W_fi W_oi W_ci [H x I] |
    b_i b_f b_o b_c [H] | initial hidden [H] | initial cell [H]; then the FNN head, per layer W [out x in] row-major
    then b (fnn_helper.cu:176-183);
  * one step, LSTMHelper::forward (lstm_helper.cu:341-463): i, f, o = sigmoid, g = tanh of W_*i x + W_*m h + b;
    c' = i g + f c; h' = tanh(c') o; the head runs on [h' ; x] with tanh on every layer but the last;
  * computeLSTMSteering (racer_dubins_elevation_lstm_steering.cu:131-166): the parametric steer-rate derivative, clamped
    to the rate limit, the inputs (0.2 angle, 0.2 rate, command, 0.2 derivative), then 5 * output on the derivative.

Error model. Every value v carries e(v) >= |float32 form - float64 value| to first order; `u` is 2^-24.
  * a float32 dot product of n terms (any order, fma or not): gamma_n * sum |w x| (Higham, Thm. 3.1);
  * SIMT forms' activations: tanh_fast's documented absolute error < 2e-7 (plugins/dynamics.cuh), so sigmoid_dev
    = (1 + tanh_fast(v / 2)) / 2 is within 1e-7 + u / 2; the host twin documents the same 2e-7 for its exp-based
    activations (host_twins.cpp);
  * tensor-core form (plugins/lstm_mma.cuh): each operand v is split as hi + lo in FP16 with |v - hi - lo| <=
    2^-22 |v| + 2^-25 (the FP16 subnormal floor) and |lo| <= 2^-11 |v| + 2^-25; a product keeps hi.hi, lo.hi, hi.lo and
    drops lo.lo. Each m16n8k16 MMA adds 16 exact FP16 products to an FP32 accumulator; we take (k + 2) * 2^-23 of the
    magnitude of everything it sums as its error (alignment to the largest term with truncation, then truncation of the
    sum). Activations: ex2.approx.f32 within 2 ulp (2^-22 relative) and rcp.approx.f32 within 1 ulp (2^-23 relative),
    the PTX ISA's figures, so r = 1 / (1 + 2^z) is within (2^-22 + 2^-23 + 2^-24) r plus the argument's error;
  * within a step the bound flows through c' = i g + f c, h' = o tanh(c') and the head with float64 derivative
    magnitudes; from step to step the state's bound goes through the magnitude of the exact step's Jacobian (|J| e),
    so it is valid for any sign pattern of the rounding errors.
"""
import math

import numpy as np

I = 4
U = 2.0 ** -24
F32 = lambda v: float(np.float32(v))  # noqa: E731  a float32 constant of the kernels, exactly in float64
FIFTH = F32(0.2)

SIMT_TANH = 2e-7
SIMT_SIG = 1e-7 + U / 2
TC_ACT_REL = 2.0 ** -22 + 2.0 ** -23 + 2.0 ** -24
LOG2E = F32(1.4426950408889634)
SPLIT_REL, SPLIT_FLOOR, LO_REL = 2.0 ** -22, 2.0 ** -25, 2.0 ** -11
MMA_UNIT = 2.0 ** -23


def gamma(n):
    return n * U / (1.0 - n * U)


def num_params(H, L1):
    return 4 * H * H + 4 * H * I + 6 * H + L1 * (H + I) + L1 + L1 + 1


class Blob:
    """The packed blob of a steering network (head {H + 4, L1, 1}) or, with `head`, of any LSTMHelper with an FNN head
    `head` = [H + input_dim, ..., out]."""

    def __init__(self, theta, H, L1=None, head=None, input_dim=I):
        t = np.asarray(theta, np.float32).astype(np.float64)
        self.H, self.I = H, input_dim
        self.layers = list(head) if head is not None else [H + input_dim, L1, 1]
        assert self.layers[0] == H + input_dim
        HH, IH = H * H, H * input_dim
        self.Wm = t[:4 * HH].reshape(4, H, H)                       # i, f, o, c
        self.Wi = t[4 * HH:4 * HH + 4 * IH].reshape(4, H, input_dim)
        o = 4 * HH + 4 * IH
        self.b = t[o:o + 4 * H].reshape(4, H)
        self.h0, self.c0 = t[o + 4 * H:o + 5 * H], t[o + 5 * H:o + 6 * H]
        o += 6 * H
        self.W, self.B = [], []
        for a, b in zip(self.layers[:-1], self.layers[1:]):
            self.W.append(t[o:o + a * b].reshape(b, a))
            self.B.append(t[o + a * b:o + a * b + b])
            o += a * b + b
        assert o == t.size, (o, t.size)


def _sig(v):
    return 0.5 * (1.0 + np.tanh(0.5 * v))


def forward(net, x, h, c):
    """One exact step: (output vector, h', c')."""
    z = net.Wi @ x + net.Wm @ h + net.b
    i, f, o, g = _sig(z[0]), _sig(z[1]), _sig(z[2]), np.tanh(z[3])
    c2 = i * g + f * c
    h2 = np.tanh(c2) * o
    a = np.concatenate([h2, x])
    for k, (W, B) in enumerate(zip(net.W, net.B)):
        a = W @ a + B
        if k < len(net.W) - 1:
            a = np.tanh(a)
    return a, h2, c2


# ---- error bounds ------------------------------------------------------------------------------------------------------
def _split(v):
    """|v - hi - lo| of the FP16 hi / lo split, and |lo|."""
    v = np.abs(v)
    return SPLIT_REL * v + SPLIT_FLOOR, LO_REL * v + SPLIT_FLOOR


def _tc_dot(W, a, ea, bias, n_mma):
    """Error of the tensor-core products W @ a + bias (W already pre-scaled, rounded to float32 at load), with `ea` the
    propagated error of a: split errors of both operands, the dropped lo.lo, the FP32 accumulation of n_mma MMAs, and
    the pre-scaling's rounding of W and bias."""
    dW, lW = _split(W)
    dW = dW + U * np.abs(W)
    da, la = _split(a)
    absW, absa = np.abs(W), np.abs(a)
    mag = absW @ absa + np.abs(bias)
    e = dW @ absa + absW @ da + lW @ la + absW @ ea
    return e + n_mma * 18 * MMA_UNIT * mag + U * np.abs(bias)


def step_bound(net, x, ex, h, eh, c, ec, form):
    """One step of the network with the errors of its float32 state (eh, ec) and inputs (ex): returns
    (out, e_out, h', e_h', c', e_c') for `form` in {"simt", "host", "tc"} (the compile-time and run-time SIMT forms share
    one bound: the same operations, the same counts)."""
    H = net.H
    z = net.Wi @ x + net.Wm @ h + net.b
    s = np.array([_sig(z[0]), _sig(z[1]), _sig(z[2]), np.tanh(z[3])])
    dsig = s[:3] * (1.0 - s[:3])
    dtanh = 1.0 - s[3] ** 2
    if form == "tc":
        # pre-activations in pre-scaled units (sc = -log2 e for sigmoids, 2 log2 e for tanh), 9 MMAs per gate tile
        ez = np.empty((4, H))
        for q in range(4):
            sc = 2.0 * LOG2E if q == 3 else -LOG2E
            Wq = np.concatenate([net.Wm[q], net.Wi[q]], axis=1) * sc
            ez[q] = _tc_dot(Wq, np.concatenate([h, x]), np.concatenate([eh, ex]), net.b[q] * sc, 9) / abs(sc)
        e_s = np.empty((4, H))
        e_s[:3] = TC_ACT_REL * s[:3] + dsig * ez[:3]
        rc = _sig(-2.0 * z[3])
        e_s[3] = 2.0 * TC_ACT_REL * rc + U * np.abs(s[3]) + dtanh * ez[3]
    else:
        n = I + H + 1
        mag = np.abs(net.Wi) @ np.abs(x) + np.abs(net.Wm) @ np.abs(h) + np.abs(net.b)
        ez = gamma(n) * mag + np.abs(net.Wi) @ ex + np.abs(net.Wm) @ eh
        sig_act = SIMT_SIG if form == "simt" else SIMT_TANH + U
        e_s = np.empty((4, H))
        e_s[:3] = sig_act + dsig * ez[:3]
        e_s[3] = SIMT_TANH + dtanh * ez[3]
    i, f, o, g = s
    c2 = i * g + f * c
    ec2 = np.abs(i) * e_s[3] + np.abs(g) * e_s[0] + np.abs(f) * ec + np.abs(c) * e_s[1] + gamma(2) * (
        np.abs(i * g) + np.abs(f * c))
    th = np.tanh(c2)
    if form == "tc":  # tanh(c') = 1 - 2 r with r = 1 / (1 + 2^(2 log2 e c')), the argument rounded
        eth = 2.0 * TC_ACT_REL * _sig(-2.0 * c2) + U * np.abs(th) + (1.0 - th ** 2) * (ec2 + U * np.abs(c2))
    else:
        eth = SIMT_TANH + (1.0 - th ** 2) * ec2
    h2 = th * o
    eh2 = np.abs(o) * eth + np.abs(th) * e_s[2] + U * np.abs(h2)
    a, ea = np.concatenate([h2, x]), np.concatenate([eh2, ex])
    last = len(net.W) - 1
    for k, (W, B) in enumerate(zip(net.W, net.B)):
        z1 = W @ a + B
        if form == "tc":
            assert len(net.W) == 2 and W.shape[0] <= 24
            if k == 0:  # layer 1: 9 MMAs per n-tile, weights and bias pre-scaled by 2 log2 e; hands on r = (1 - tanh) / 2
                sc = 2.0 * LOG2E
                ez1 = _tc_dot(W * sc, a, ea, B * sc, 9) / sc
                r = _sig(-2.0 * z1)
                er = TC_ACT_REL * r + r * (1.0 - r) * 2.0 * ez1
                a, ea = r, er
                continue
            # layer 2 on r: W' = -2 W, b' = b + sum W (summed in double, rounded once); two chains of 3 MMAs, then added
            b2 = B + W.sum(axis=1)
            e1 = _tc_dot(-2.0 * W, a, ea, b2, 6) + U * np.abs(b2)
            z1 = -2.0 * W @ a + b2
            return z1, e1 + U * np.abs(z1), h2, eh2, c2, ec2
        n = W.shape[1] + 1
        ez1 = gamma(n) * (np.abs(W) @ np.abs(a) + np.abs(B)) + np.abs(W) @ ea
        if k < last:
            z1t = np.tanh(z1)
            ea = SIMT_TANH + (1.0 - z1t ** 2) * ez1
            a = z1t
        else:
            a, ea = z1, ez1
    return a, ea, h2, eh2, c2, ec2


# ---- the closed steering subsystem ---------------------------------------------------------------------------------------
class SteerParams:
    """The float32 constants the steering step reads, as float64."""

    def __init__(self, p):
        self.scmd, self.ks = F32(p.steer_command_angle_scale), F32(p.steering_constant)
        self.ka, self.kd = F32(p.steer_accel_constant), F32(p.steer_accel_drag_constant)
        self.max_rate, self.max_angle = F32(p.max_steer_rate), F32(p.max_steer_angle)
        self.lo, self.hi = F32(p.lim.rng_lo[1]), F32(p.lim.rng_hi[1])


def _clamp(v, a):
    return min(max(v, -a), a)


def _exact_steps(net, sp, S, u, dt):
    """The exact step of a batch of subsystem states S [B][2 + 2H] = (angle, rate, h, c) under command u: (S', out)."""
    H = net.H
    sa, sr, h, c = S[:, 0], S[:, 1], S[:, 2:2 + H], S[:, 2 + H:]
    pa = (u * sp.scmd - sa) * sp.ks
    sd0 = np.clip((pa - sr) * sp.ka - sr * sp.kd, -sp.max_rate, sp.max_rate)
    x = np.stack([sa * FIFTH, sr * FIFTH, np.full_like(sa, u), sd0 * FIFTH], axis=1)
    z = np.einsum("qij,bj->qbi", net.Wi, x) + np.einsum("qij,bj->qbi", net.Wm, h) + net.b[:, None, :]
    c2 = _sig(z[0]) * np.tanh(z[3]) + _sig(z[1]) * c
    h2 = np.tanh(c2) * _sig(z[2])
    a = np.concatenate([h2, x], axis=1)
    for k, (W, B) in enumerate(zip(net.W, net.B)):
        a = a @ W.T + B
        if k < len(net.W) - 1:
            a = np.tanh(a)
    out = a[:, 0]
    sa2 = np.clip(sa + sr * dt, -sp.max_angle, sp.max_angle)
    sr2 = sr + (sd0 + 5.0 * out) * dt
    return np.concatenate([sa2[:, None], sr2[:, None], h2, c2], axis=1), out


def steer_rollout(net, sp, sa0, sr0, commands, dt, form):
    """The steering states of one sample over len(commands) steps from (sa0, sr0) with the network's initial state,
    exact, with their bounds. Returns dict of arrays [T]: angle, e_angle, rate, e_rate (after each step), cost and e_cost
    (the engine's convention for RacerQuadraticCost with only steer_coeff = 1: sum of angle^2, then / T), and out, e_out
    (the network output per step).

    The bound of the state e = (angle, rate, h, c) is carried as e' = |J| e + d: d is the step's own rounding (the
    operation bounds above with exact inputs) and J the exact step's Jacobian (central differences in float64), so
    what a step does to an incoming error keeps its signs within the step: the rate's own decay through the parametric
    derivative, 1 - dt (steer_accel_constant + drag), contracts it instead of adding the two paths' magnitudes."""
    dt = F32(dt)
    T = len(commands)
    Hd = net.H
    n = 2 + 2 * Hd
    S = np.concatenate([[F32(sa0), F32(sr0)], net.h0, net.c0])
    e = np.zeros(n)
    res = {k: np.zeros(T) for k in ("angle", "e_angle", "rate", "e_rate", "out", "e_out")}
    run, erun = 0.0, 0.0
    zh, zc = np.zeros(Hd), np.zeros(Hd)
    for t in range(T):
        u = min(max(F32(commands[t]), sp.lo), sp.hi)
        sa, sr, h, c = S[0], S[1], S[2:2 + Hd], S[2 + Hd:]
        # the step's own rounding, from exact inputs
        pa = (u * sp.scmd - sa) * sp.ks
        epa = gamma(3) * abs(sp.ks) * (abs(u * sp.scmd) + abs(sa))
        sd0 = _clamp((pa - sr) * sp.ka - sr * sp.kd, sp.max_rate)
        esd0 = abs(sp.ka) * epa + gamma(4) * (abs(sp.ka) * (abs(pa) + abs(sr)) + abs(sp.kd * sr))
        x = np.array([sa * FIFTH, sr * FIFTH, u, sd0 * FIFTH])
        ex = np.array([U * abs(x[0]), U * abs(x[1]), 0.0, FIFTH * esd0 + U * abs(x[3])])
        out, eout, _, dh, _, dc = step_bound(net, x, ex, h, zh, c, zc, form)
        out, eout = float(out[0]), float(eout[0])
        sd = sd0 + 5.0 * out
        esd = esd0 + 5.0 * eout + gamma(1) * abs(sd)
        d = np.concatenate([[gamma(2) * (abs(sa) + abs(sr * dt)), dt * esd + gamma(2) * (abs(sr) + abs(sd * dt))], dh, dc])
        # the exact step's Jacobian
        step = 1e-6 * np.maximum(1.0, np.abs(S))
        P = np.concatenate([S + np.diag(step), S - np.diag(step), S[None]])
        Sn, outs = _exact_steps(net, sp, P, u, dt)
        J = (Sn[:n] - Sn[n:2 * n]).T / (2.0 * step)
        Jout = (outs[:n] - outs[n:2 * n]) / (2.0 * step)
        eout = eout + np.abs(Jout) @ e
        e = np.abs(J) @ e + d
        S = Sn[-1]
        res["angle"][t], res["e_angle"][t], res["rate"][t], res["e_rate"][t] = S[0], e[0], S[1], e[1]
        res["out"][t], res["e_out"][t] = outs[-1], eout
        run += S[0] * S[0]
        erun += 2.0 * abs(S[0]) * e[0] + gamma(2) * abs(run)
    res["cost"] = run / T
    res["e_cost"] = erun / T + U * abs(run / T)
    return res


def ulps(v, k=4):
    """k float32 ulps of |v|."""
    v = np.abs(np.asarray(v, np.float64))
    return k * np.spacing(v.astype(np.float32)).astype(np.float64)


def check(name, got, want, bound):
    """|got - want| <= 2 bound + 4 ulps everywhere; returns the largest error / bound ratio and prints it."""
    got = np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    bound = np.asarray(bound, np.float64)
    assert np.all(np.isfinite(got)), f"{name}: non-finite result"
    err = np.abs(got - want)
    ratio = float(np.max(err / (bound + ulps(want))))
    print(f"{name}: max |err| / bound = {ratio:.3g}")
    worst = int(np.argmax(err - 2.0 * bound - ulps(want)))
    assert np.all(err <= 2.0 * bound + ulps(want)), (name, worst, float(err.flat[worst]), float(bound.flat[worst]))
    return ratio
