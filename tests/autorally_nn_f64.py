"""Float64 restatement of the Autorally NeuralNetModel<7,2,3> + ARStandardCost rollout, with a running first-order bound on
how far a correct float32 evaluation of each form of its 6-32-32-4 network may sit from it.

Semantics (written from the reference, not from oracle/mppi_oracle.cpp):
  * packed blob (fnn_helper.cu:176-183): per layer W [out x in] row-major, then b; layers 6-32-32-4, 1412 floats;
  * FNNHelper::forward (fnn_helper.cu:419-484): tanh on every layer but the last, exact tanh here;
  * NeuralNetModel::computeDynamics (ar_nn_model.cu:90-128): kinematics for states 0-2 (x' = cos(yaw) vx - sin(yaw) vy,
    y' = sin(yaw) vx + cos(yaw) vy, yaw' = -yaw rate), the network on (roll, vx, vy, yaw rate, u0, u1) for states 3-6;
  * Dynamics::updateState (dynamics.cu:118-129): explicit Euler; the cost reads the state after the step;
  * control sampling (gaussian.cu) u = mean + std_dev * eps, then enforceConstraints (dynamics.cu:97-116) clamps it;
  * ARStandardCost (ar_standard_cost.cu:284-413) with only the speed and slip terms live: speed_coeff (vx - desired)^2
    and slip_coeff atan(vy / |vx|)^2; the rollout loop's running cost divided by T (mppi_common.cu:843-853).

Error model. Every value v carries e(v) >= |float32 form - float64 value| to first order; `u` is 2^-24. The constants and
the FP16 split model are those of tests/steering_lstm_f64.py.
  * "ffma2" (AutorallyNNDynamics, plugins/dynamics.cuh) and "host" (fnn_6_32_32_4, host_twins.cpp): a float32 dot product
    of n terms in any order is within gamma_n * sum |w x| (Higham, Thm. 3.1); tanh_fast and the host twin's tanh8 are both
    documented within 2e-7 absolute (the host twin's gets one more rounding, u |t|);
  * "mma" (plugins/nn_mma.cuh): the folded network of load_weights, W1' = k W1, b1' = k b1 (k = 2 log2 e), W2' = -2k W2,
    b2' = k (b2 + sum W2) (the sum in double, rounded once, then scaled), W3' = -2 W3, b3' = b3 + sum W3; every operand v is
    split in FP16 with |v - hi - lo| <= 2^-22 |v| + 2^-25 and |lo| <= 2^-11 |v| + 2^-25, and the lo.lo product is dropped.
    An m16n8kK MMA, taken in the kernel's issue order, aligns its terms to the largest and truncates the others: it adds
    (K + 1) 2^-23 of the largest magnitude it sums, the incoming accumulator included (it starts at b', which is where
    the fold's cancellation shows once tanh saturates), plus 2^-23 of its result. Activations are handed on as
    r = 1 / (2^z + 1) with ex2.approx within 2 ulp and rcp.approx within 1 ulp; layer 3's two accumulators are added at
    the end;
  * "wgmma" (rollout_kernel_nn_tc.cuh): each operand is split hi = rna_tf32(v) (|v - hi| <= 2^-11 |v|), lo = v - hi, exact in
    FP32 but read by the tensor cores as TF32 (taken as truncation, 2^-10 |lo|); the lo.lo product is dropped; the biases
    are a split K column against a constant one; tanh = 1 - 2 r explicitly; an m64nNk8 wgmma is an MMA of depth 8 in the
    sense above;
  * around the network (all forms): sincos at 1.5 ulp, the Euler update's two roundings, the cost terms' float32
    roundings with atanf at 2 ulp, and gamma_T on the running sum;
  * from step to step the state's bound goes through the magnitude of the exact step's Jacobian, |J| e, with J by central
    differences in float64, so it is valid for any sign pattern of the rounding errors (as in steering_lstm_f64.py).
"""
import math

import numpy as np

from tests.steering_lstm_f64 import (F32, LO_REL, MMA_UNIT, SIMT_TANH, SPLIT_FLOOR, SPLIT_REL, TC_ACT_REL, U, check,  # noqa: F401
                                     gamma, ulps)

K_TANH = F32(2.8853900817779268)  # kTanhScale of nn_mma.cuh and rollout_kernel_nn_tc.cuh, as the float the kernels use
LN2 = math.log(2.0)
SINCOS = 3.0 * U   # 1.5 ulp of |v|: an ulp is at most 2^-23 |v|
ATAN = 4.0 * U     # atanf, 2 ulp
TF32_HI, TF32_LO = 2.0 ** -11, 2.0 ** -10
HOST_TANH = SIMT_TANH + U
NUM_PARAMS = 1412


class Net:
    """The packed 1412-float blob of the 6-32-32-4 network, as float64."""

    def __init__(self, theta):
        t = np.asarray(theta, np.float32).astype(np.float64)
        assert t.size == NUM_PARAMS
        self.W1, self.b1 = t[:192].reshape(32, 6), t[192:224]
        self.W2, self.b2 = t[224:1248].reshape(32, 32), t[1248:1280]
        self.W3, self.b3 = t[1280:1408].reshape(4, 32), t[1408:1412]
        f32 = np.float32
        # load_weights of nn_mma.cuh, as the float32 values the kernel builds (tests/test_nn_mma_scheme.py: _folded)
        W1f, W2f, W3f = (w.astype(f32) for w in (self.W1, self.W2, self.W3))
        self.mW1 = (W1f * f32(K_TANH)).astype(np.float64)
        self.mb1 = (self.b1.astype(f32) * f32(K_TANH)).astype(np.float64)
        self.mW2 = (W2f * f32(-2.0 * K_TANH)).astype(np.float64)
        self.mb2 = ((self.b2 + self.W2.sum(1)).astype(f32) * f32(K_TANH)).astype(np.float64)
        self.mW3 = (W3f * f32(-2.0)).astype(np.float64)
        self.mb3 = (self.b3 + self.W3.sum(1)).astype(f32).astype(np.float64)
        # rollout_kernel_nn_tc.cuh: the tanh layers pre-scaled by k, float32 products
        self.tW1 = (W1f * f32(K_TANH)).astype(np.float64)
        self.tb1 = self.mb1
        self.tW2 = (W2f * f32(K_TANH)).astype(np.float64)
        self.tb2 = (self.b2.astype(f32) * f32(K_TANH)).astype(np.float64)


def forward(net, x):
    """The exact network on inputs x [..., 6]: outputs [..., 4]."""
    a = np.tanh(x @ net.W1.T + net.b1)
    a = np.tanh(a @ net.W2.T + net.b2)
    return a @ net.W3.T + net.b3


# ---- the network's own error, per form, for a batch of exact inputs x [B][6] ---------------------------------------------
def _split(v):
    v = np.abs(v)
    return SPLIT_REL * v + SPLIT_FLOOR, LO_REL * v + SPLIT_FLOOR


def _chain(W, a, c0, tiles, K, per_tile):
    """FP32 accumulation error of MMAs of depth K run in issue order: for each k-tile (a slice of the inputs), `per_tile`
    MMAs, the first adding the tile's products to the running accumulator (which starts at c0), the others the tile's lo
    corrections. An MMA aligns its terms to the largest, truncating each of the others by less than an ulp of it, then
    rounds its sum: (K + 1) 2^-23 of the largest magnitude it sums plus 2^-23 of its result. Returns (error, sum)."""
    P = a[:, None, :] * W[None, :, :]                                       # [B][out][in] exact products
    part = np.broadcast_to(c0, P.shape[:2]).astype(np.float64)
    e = np.zeros(P.shape[:2])
    for sl in tiles:
        pm = np.abs(P[:, :, sl]).max(axis=2)
        e += (K + 1) * MMA_UNIT * np.maximum(np.abs(part), pm)
        part = part + P[:, :, sl].sum(axis=2)
        e += MMA_UNIT * np.abs(part)
        e += (per_tile - 1) * ((K + 1) * MMA_UNIT * np.maximum(np.abs(part), pm) + MMA_UNIT * np.abs(part))
    return e, part


def _mma_dot(W, a, ea, b, acc_err, rounded_w=True):
    """Error of bias + W @ a on the mma.sync form, in the units of W (pre-scaled): the split errors of both operands, the
    dropped lo.lo, the propagated error of a, the FP32 accumulation `acc_err` (_chain), and the float32 rounding of the
    pre-scaled weights and bias."""
    aW, ab = np.abs(W), np.abs(b)
    dW, lW = _split(W)
    if rounded_w:
        dW = dW + U * aW
    da, la = _split(a)
    aa = np.abs(a)
    return da @ aW.T + aa @ dW.T + la @ lW.T + np.abs(ea) @ aW.T + acc_err + 2.0 * U * ab


def _wg_dot(W, a, ea, b, acc_err):
    """The same for the wgmma form: TF32 hi (rna) / lo (read truncated) parts, the dropped lo.lo, bias as a split K column
    against an exact one."""
    aW, ab, aa = np.abs(W), np.abs(b), np.abs(a)
    lo_err = TF32_LO * TF32_HI                                   # lo read as TF32: 2^-10 of |lo| <= 2^-11 |v|
    prod = (2.0 * lo_err + TF32_HI * TF32_HI) * (1.0 + TF32_HI)  # a_lo w_hi, a_hi w_lo truncations, dropped lo.lo
    return prod * (aa @ aW.T) + (lo_err + U) * ab + U * (aa @ aW.T) + np.abs(ea) @ aW.T + acc_err


def net_bound(net, x, form):
    """(out [B][4], e_out [B][4]): the exact network on exact inputs x [B][6] and the bound of its float32 evaluation on
    `form` in {"ffma2", "host", "mma", "wgmma"}."""
    x = np.atleast_2d(x)
    z1 = x @ net.W1.T + net.b1
    a1 = np.tanh(z1)
    z2 = a1 @ net.W2.T + net.b2
    a2 = np.tanh(z2)
    out = a2 @ net.W3.T + net.b3
    zx = np.zeros_like(x)
    if form in ("ffma2", "host"):
        act = SIMT_TANH if form == "ffma2" else HOST_TANH
        ez1 = gamma(7) * (np.abs(x) @ np.abs(net.W1).T + np.abs(net.b1))
        ea1 = act + (1.0 - a1 ** 2) * ez1
        ez2 = gamma(33) * (np.abs(a1) @ np.abs(net.W2).T + np.abs(net.b2)) + ea1 @ np.abs(net.W2).T
        ea2 = act + (1.0 - a2 ** 2) * ez2
        eo = gamma(33) * (np.abs(a2) @ np.abs(net.W3).T + np.abs(net.b3)) + ea2 @ np.abs(net.W3).T
        return out, eo
    if form == "mma":
        K16, K8, H0, H1 = slice(0, 16), slice(0, 8), slice(0, 16), slice(16, 32)
        # layer 1: one k16 MMA ([a_hi | a_lo] x [w_hi ; w_hi]) and one k8 (a_hi x w_lo), from the bias
        e16, part = _chain(net.mW1, x, net.mb1, [K16], 16, 1)
        acc1 = e16 + _chain(net.mW1, x, part, [K8], 8, 1)[0] - MMA_UNIT * np.abs(part)  # the k8 MMA adds only lo terms
        ez1 = _mma_dot(net.mW1, x, zx, net.mb1, acc1)
        r1 = 0.5 * (1.0 - a1)                                       # 1 / (2^(k z1) + 1)
        er1 = TC_ACT_REL * r1 + LN2 * r1 * (1.0 - r1) * ez1
        # layer 2 on r1: two k-tiles of three k16 MMAs
        ez2 = _mma_dot(net.mW2, r1, er1, net.mb2, _chain(net.mW2, r1, net.mb2, [H0, H1], 16, 3)[0]) + U * np.abs(net.mb2)
        r2 = 0.5 * (1.0 - a2)
        er2 = TC_ACT_REL * r2 + LN2 * r2 * (1.0 - r2) * ez2
        # layer 3 on r2: two chains of three k16 MMAs (one from the bias over inputs 0-15, one from zero over 16-31), then
        # one add
        acc3 = (_chain(net.mW3[:, H0], r2[:, H0], net.mb3, [slice(0, 16)], 16, 3)[0] +
                _chain(net.mW3[:, H1], r2[:, H1], 0.0, [slice(0, 16)], 16, 3)[0])
        eo = _mma_dot(net.mW3, r2, er2, net.mb3, acc3, rounded_w=False) + U * np.abs(net.mb3) + U * np.abs(out)
        return out, eo
    if form == "wgmma":
        blocks = [slice(8 * k, 8 * k + 8) for k in range(4)]
        # layer 1: one K block of 8 (6 inputs, the bias column, a zero), three m64n32k8 wgmmas from zero
        x1 = np.concatenate([x, np.ones((x.shape[0], 1))], axis=1)
        W1b = np.concatenate([net.tW1, net.tb1[:, None]], axis=1)
        ez1 = _wg_dot(net.tW1, x, zx, net.tb1, _chain(W1b, x1, 0.0, [slice(0, 7)], 8, 3)[0])
        # tanh = 1 - 2 r, r = 1 / (2^z' + 1) with z' = k z
        r1 = 0.5 * (1.0 - a1)
        ea1 = 2.0 * TC_ACT_REL * r1 + U * np.abs(a1) + (1.0 - a1 ** 2) / K_TANH * ez1
        # layers 2 and 3: four K blocks of three wgmmas from zero, then the bias block of two
        def acc(W, a, b):
            Wb = np.concatenate([W, b[:, None]], axis=1)
            ab = np.concatenate([a, np.ones((a.shape[0], 1))], axis=1)
            e, part = _chain(Wb, ab, 0.0, blocks, 8, 3)
            return e + _chain(Wb, ab, part, [slice(32, 33)], 8, 2)[0]
        ez2 = _wg_dot(net.tW2, a1, ea1, net.tb2, acc(net.tW2, a1, net.tb2))
        r2 = 0.5 * (1.0 - a2)
        ea2 = 2.0 * TC_ACT_REL * r2 + U * np.abs(a2) + (1.0 - a2 ** 2) / K_TANH * ez2
        eo = _wg_dot(net.W3, a2, ea2, net.b3, acc(net.W3, a2, net.b3))
        return out, eo
    raise ValueError(form)


# ---- the rollout ---------------------------------------------------------------------------------------------------------
class Params:
    """The float32 constants a rollout reads, as float64: control limits, the speed and slip terms of ARStandardCost or,
    with `robust`, of ARRobustCost (ar_robust_cost.cu:13-132: slip_coeff |atan(vy / |vx|)| + speed_coeff |vx - desired|,
    its penalties, track and heading terms off)."""

    def __init__(self, dyn, cost):
        lim = dyn.params.lim
        self.lo = np.array([F32(lim.rng_lo[i]) for i in range(2)])
        self.hi = np.array([F32(lim.rng_hi[i]) for i in range(2)])
        p = cost.params
        self.speed, self.desired, self.slip = F32(p.speed_coeff), F32(p.desired_speed), F32(p.slip_coeff)
        self.robust = hasattr(p, "heading_coeff")
        assert p.l1_cost == 0 and F32(p.track_coeff) == 0.0 and F32(p.crash_coeff) == 0.0
        assert not self.robust or (F32(p.heading_coeff) == 0.0 and self.desired != -1.0)


def _deriv(net, S, u):
    """The exact state derivative of a batch S [B][7] under controls u [B][2]."""
    yaw, vx, vy = S[:, 2], S[:, 4], S[:, 5]
    cs, sn = np.cos(yaw), np.sin(yaw)
    x6 = np.concatenate([S[:, 3:7], u], axis=1)
    return np.concatenate([(cs * vx - sn * vy)[:, None], (sn * vx + cs * vy)[:, None], -S[:, 6:7], forward(net, x6)],
                          axis=1)


def step_cost(cp, S):
    """The exact running cost of states S [B][7] (after the step), and its gradient [B][7]."""
    vx, vy = S[:, 4], S[:, 5]
    ratio = vy / np.abs(vx)
    slip = -np.arctan(ratio)
    den = vx ** 2 + vy ** 2
    dslip = np.sign(vx) * vy / den, -np.abs(vx) / den                       # d slip / d vx, d slip / d vy
    g = np.zeros_like(S)
    if cp.robust:  # abs is 1-Lipschitz, so the magnitude of its one-sided derivative bounds it at the kink too
        c = cp.slip * np.abs(slip) + cp.speed * np.abs(vx - cp.desired)
        g[:, 4] = cp.speed * np.sign(vx - cp.desired) + cp.slip * np.sign(slip) * dslip[0]
        g[:, 5] = cp.slip * np.sign(slip) * dslip[1]
        return c, g
    c = cp.speed * (vx - cp.desired) ** 2 + cp.slip * slip ** 2
    g[:, 4] = 2.0 * cp.speed * (vx - cp.desired) + 2.0 * cp.slip * slip * dslip[0]
    g[:, 5] = 2.0 * cp.slip * slip * dslip[1]
    return c, g


def _cost_own(cp, S):
    """The float32 rounding of one step's cost at exact states S (speed: subtract, square, scale; slip: divide, atanf,
    square, scale; one add)."""
    vx, vy = S[:, 4], S[:, 5]
    ratio = vy / np.abs(vx)
    slip = -np.arctan(ratio)
    e_slip = ATAN * np.abs(slip) + U * np.abs(ratio) / (1.0 + ratio ** 2)
    if cp.robust:  # slip_coeff |slip| + 0; 0 + speed_coeff |vx - desired| + 0 x heading; their sum
        sp, st = cp.speed * np.abs(vx - cp.desired), cp.slip * np.abs(slip)
        return gamma(2) * sp + cp.slip * e_slip + U * st + gamma(3) * (sp + st)
    sp = cp.speed * (vx - cp.desired) ** 2
    st = cp.slip * slip ** 2
    return gamma(3) * sp + 2.0 * cp.slip * np.abs(slip) * e_slip + gamma(2) * st + U * (sp + st)


def rollout(net, cp, x0, eps, dt, form):
    """Exact rollouts of B samples from x0 [7] under noise eps [B][T][2] (mean 0, std_dev 1), with their bounds on `form`.
    Returns a dict: states [B][T][7] and e_states (after each step), step costs c [B][T], cost [B] (the running sum / T)
    and e_cost [B], and vx_min [B] (the smallest forward speed, for the slip term's precondition)."""
    dt = F32(dt)
    eps = np.asarray(eps, np.float32).astype(np.float64)
    B, T, _ = eps.shape
    S = np.tile(np.asarray(x0, np.float32).astype(np.float64), (B, 1))
    e = np.zeros((B, 7))
    states, e_states, costs = np.zeros((B, T, 7)), np.zeros((B, T, 7)), np.zeros((B, T))
    run, erun, asum = np.zeros(B), np.zeros(B), np.zeros(B)
    hstep = 1e-6
    for t in range(T):
        u = np.clip(eps[:, t], cp.lo, cp.hi)
        # the step's own rounding, from the exact state
        yaw, vx, vy = S[:, 2], S[:, 4], S[:, 5]
        cs, sn = np.cos(yaw), np.sin(yaw)
        x6 = np.concatenate([S[:, 3:7], u], axis=1)
        out, eo = net_bound(net, x6, form)
        kin = np.abs(cs * vx) + np.abs(sn * vy), np.abs(sn * vx) + np.abs(cs * vy)
        xd = _deriv(net, S, u)
        ed = np.zeros((B, 7))
        ed[:, 0] = (SINCOS + gamma(2)) * kin[0]
        ed[:, 1] = (SINCOS + gamma(2)) * kin[1]
        ed[:, 3:] = eo
        d = dt * ed + gamma(2) * (np.abs(S) + np.abs(xd * dt))
        # the exact step's Jacobian by central differences
        hs = hstep * np.maximum(1.0, np.abs(S))                                 # [B][7]
        P = np.concatenate([S[:, None, :] + hs[:, :, None] * np.eye(7), S[:, None, :] - hs[:, :, None] * np.eye(7)], 1)
        uP = np.repeat(u[:, None, :], 14, axis=1).reshape(-1, 2)
        Pn = (P.reshape(-1, 7) + _deriv(net, P.reshape(-1, 7), uP) * dt).reshape(B, 14, 7)
        J = (Pn[:, :7] - Pn[:, 7:]).transpose(0, 2, 1) / (2.0 * hs[:, None, :])  # J[b][i][j] = d S'_i / d S_j
        e = np.einsum("bij,bj->bi", np.abs(J), e) + d
        S = S + xd * dt
        c, g = step_cost(cp, S)
        states[:, t], e_states[:, t], costs[:, t] = S, e, c
        run += c
        asum += np.abs(c)
        erun += np.einsum("bj,bj->b", np.abs(g), e) + _cost_own(cp, S)
    cost = run / T
    e_cost = (erun + gamma(T) * asum) / T + U * np.abs(cost)
    return {"states": states, "e_states": e_states, "c": costs, "cost": cost, "e_cost": e_cost,
            "vx_min": states[:, :, 4].min(axis=1)}


def jacobian_bound(net, x, u):
    """([A | B] [7][9], bound [7][9]): the exact Jacobian of the state derivative at (x, u) and the bound of the device's
    NeuralNetModel::computeGrad (AutorallyNNDynamics::computeGrad: FP32 FMA chains, tanhf within 2 ulp, sincosf within
    1.5 ulp, the back-propagation W3 diag(d2) W2 diag(d1) W1 in its loop order)."""
    x = np.asarray(x, np.float32).astype(np.float64)
    u = np.asarray(u, np.float32).astype(np.float64)
    inp = np.concatenate([x[3:], u])
    A, E = np.zeros((7, 9)), np.zeros((7, 9))
    sn, cs = math.sin(x[2]), math.cos(x[2])
    es, ec = SINCOS * abs(sn), SINCOS * abs(cs)
    A[0, 2], E[0, 2] = -sn * x[4] - cs * x[5], es * abs(x[4]) + ec * abs(x[5]) + gamma(2) * (abs(sn * x[4]) + abs(cs * x[5]))
    A[0, 4], E[0, 4] = cs, ec
    A[0, 5], E[0, 5] = -sn, es
    A[1, 2], E[1, 2] = cs * x[4] - sn * x[5], ec * abs(x[4]) + es * abs(x[5]) + gamma(2) * (abs(cs * x[4]) + abs(sn * x[5]))
    A[1, 4], E[1, 4] = sn, es
    A[1, 5], E[1, 5] = cs, ec
    A[2, 6] = -1.0
    aW1, aW2, aW3 = np.abs(net.W1), np.abs(net.W2), np.abs(net.W3)
    a1 = np.tanh(net.W1 @ inp + net.b1)
    ea1 = 4.0 * U * np.abs(a1) + (1.0 - a1 ** 2) * gamma(7) * (aW1 @ np.abs(inp) + np.abs(net.b1))
    d1 = 1.0 - a1 ** 2
    ed1 = 2.0 * np.abs(a1) * ea1 + gamma(2) * (1.0 + a1 ** 2)
    a2 = np.tanh(net.W2 @ a1 + net.b2)
    ez2 = gamma(33) * (aW2 @ np.abs(a1) + np.abs(net.b2)) + aW2 @ ea1
    ea2 = 4.0 * U * np.abs(a2) + (1.0 - a2 ** 2) * ez2
    d2 = 1.0 - a2 ** 2
    ed2 = 2.0 * np.abs(a2) * ea2 + gamma(2) * (1.0 + a2 ** 2)
    g = (net.W3 * d2) @ net.W2                                              # [4][32]: g_ij before the d1 factor
    eg = gamma(34) * (np.abs(net.W3 * d2) @ aW2) + (aW3 * ed2) @ aW2
    gd = g * d1
    egd = np.abs(g) * ed1 + eg * d1 + U * np.abs(gd)
    J = gd @ net.W1                                                        # [4][6]
    eJ = gamma(33) * (np.abs(gd) @ aW1) + egd @ aW1
    A[3:, 3:] = J
    E[3:, 3:] = eJ
    return A, E
