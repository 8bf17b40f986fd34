"""The softmin reduction — K1's block partials (beta_b, eta_b, sum w^2_b, V_b), K2's merge, the read-back weights and the Tsallis
weights — against a float64 softmin, beta = min c, w = exp(-(c - beta) / lambda), eta = sum w, U = sum w u / eta, sum w^2.

Part 1 chooses the costs: tests/plugins/softmin_probe_pair.cu is an out-of-tree pair whose trajectory cost is, bit for bit,
the value the test puts into the noise (see that file for the recipe), so the cases the in-tree models never produce can be
set up exactly: a block whose every sample costs +inf, scattered +inf, spreads where expf underflows inside a block or
between blocks, ties of the minimum across blocks, costs of 1e16 a few ulps apart, negative costs, extreme lambda, a ragged
last block and the record limit of K2. Each case runs through every form of the generic K1 the probe is built for.

Part 2 takes the costs the real pairs make: every K1 instantiation tools/k1_plan_matrix.py can select, solved with the
controls written back and checked against the float64 softmin of its own costs and controls; then the same seed without
write-back (the instantiation the benchmark runs) must give bit-identical costs, U and statistics.

Error budget of a device weight (derived, not fitted): w_n = s_b * w_nb with w_nb = expf(-lambda_f (c_n - beta_b)) in K1 and
s_b = expf(-lambda_f (beta_b - beta)) in K2, lambda_f = 1/lambda narrowed to float. Each argument carries the narrowing of
lambda_f, the rounding of the difference and of the product (3 a u, a = |argument|, u = 2^-24) and each expf 2 ulp (4 u), so
the relative error of w_n is at most delta_n = 3 a_n u + 8 u with a_n = (c_n - beta) / lambda, plus 2^-148 absolute where
the float result is subnormal. As in test_gpu_parity._check_solve, U then moves by at most
sum_n |dw_n| |u_n - U| / eta, plus the float accumulation of V (one fma per row of a block, one per record of K2) and of eta."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

import mppi_generic_b200 as m
from mppi_generic_b200 import workloads as W

H = m.host
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLUGIN = os.path.join(ROOT, "tests", "plugins", "libmppi_plugin_softmin_probe.so")
PROBE_ID = H.USER_ID_BASE + 1
U32 = 2.0 ** -24  # unit roundoff of float32
SUB = 2.0 ** -148  # two ulps of the smallest subnormal: expf's absolute error where its result is subnormal
F32_MAX = np.float32(H.FLT_MAX)


class ProbeDynParams(C.Structure):
    _fields_ = [("lim", H.ControlLimits)]


class ProbeCostParams(C.Structure):
    _fields_ = [("control_cost_coeff", C.c_float * H.MAX_C), ("discount", C.c_float), ("horizon", C.c_float),
                ("inf_at", C.c_float), ("zero_cost", C.c_float)]


def _plugin():
    """Load the probe pair; build it first if it is missing, rebuild once if the library's layout fingerprint refuses it
    (a plugin must come from the same source revision as libmppi_b200.so)."""
    build = ["bash", os.path.join(ROOT, "tests", "plugins", "build.sh")]
    if not os.path.exists(PLUGIN):
        subprocess.check_call(build)
    try:
        H.load_plugin(PLUGIN)
    except H.MppibError as ex:
        if "another revision" not in str(ex):
            raise
        subprocess.check_call(build)
        H.load_plugin(PLUGIN)


# ---- float64 reference and its error budget ---------------------------------------------------------------------------------
def _softmin64(c, u, lam):
    """float64 softmin of costs c [n] (float32, +inf allowed) and controls u [n][T][C]."""
    c = c.astype(np.float64)
    beta = c.min()
    a = np.where(c == np.inf, np.inf, (c - beta) / lam)
    w = np.exp(-a)
    uu = u.reshape(u.shape[0], -1).astype(np.float64)
    eta = w.sum()
    return beta, a, w, eta, (w @ uu) / eta, (w * w).sum()


def _check_softmin(U, stats, c, u, lam, rows_per_block, nrec, eta_levels, what):
    """U [T][C] and stats (baseline, normaliser, sum w^2) of one distribution against the float64 softmin of (c, u).
    rows_per_block: rows of a block's sequential weighted sum; nrec: records K2 merges; eta_levels: float additions on the way
    to a block's eta_b (per-thread, warp tree, per-warp partials)."""
    beta, a, w, eta, Uref, w2 = _softmin64(c, u, lam)
    assert stats[0] == np.float32(beta), (what, stats[0], beta)
    fin = np.isfinite(a)
    delta = np.where(fin, (3.0 * np.where(fin, a, 0.0) + 8.0) * U32, 0.0)
    dw = delta * w + np.where(fin, SUB, 0.0)
    k_eta = eta_levels + 2  # + the double merge narrowed to float
    assert abs(stats[1] - eta) <= dw.sum() + k_eta * U32 * eta, (what, stats[1], eta)
    assert abs(stats[2] - w2) <= (2.0 * dw * w).sum() + (k_eta + 1) * U32 * w2, (what, stats[2], w2)
    uu = u.reshape(u.shape[0], -1).astype(np.float64)
    Uf = U.reshape(-1).astype(np.float64)
    k_acc = rows_per_block + nrec // 16 + 4 + 16 + 2  # fma chain of a block, K2's per-warp chain and 4 + 16 partial sums, / eta
    bound = (dw @ np.abs(uu - Uref[None])) / eta + k_acc * U32 * ((w @ np.abs(uu)) / eta) + k_eta * U32 * np.abs(Uref)
    err = np.abs(Uf - Uref)
    assert np.all(err <= bound), (what, float((err / np.maximum(bound, 1e-300)).max()), int(np.argmax(err - bound)))


def _check_weights(wdev, c, lam, what):
    """get_weights(): expf(-lambda_f (c - beta)) against the global baseline, one expf (3 a u + 4 u)."""
    beta, a, w, *_ = _softmin64(c, np.zeros((c.size, 1, 1), np.float32), lam)
    fin = np.isfinite(a)
    bound = np.where(fin, (3.0 * np.where(fin, a, 0.0) + 4.0) * U32 * w + SUB, 0.0)
    assert np.all(np.abs(wdev.astype(np.float64) - w) <= bound), what


# ---- the probe pair ---------------------------------------------------------------------------------------------------------
# name -> (environment read when the engine is created, descriptor flags, num_distributions)
FORMS = {
    "resident": ({}, 0, 1),
    "no_tma": ({}, H.FLAG_NO_TMA, 1),
    "stream": ({"MPPIB_STREAM": "1"}, 0, 1),
    "stream_readback": ({"MPPIB_STREAM": "1", "MPPIB_STREAM_READBACK": "1"}, 0, 1),
    "spt2": ({"MPPIB_SPT": "2"}, 0, 1),
    "D2": ({}, 0, 2),
    "bx32": ({"MPPIB_BX": "32"}, 0, 1),
    "bx64": ({"MPPIB_BX": "64"}, 0, 1),
    "bx128": ({"MPPIB_BX": "128"}, 0, 1),
}


class Probe:
    """An engine of the probe pair in one K1 form, and the noise that gives each sample a chosen cost."""

    def __init__(self, N, T, form="resident", lam=1.0, flags=0):
        _plugin()
        env, fflags, D = FORMS[form]
        self.N, self.T, self.D, self.lam, self.form = N, T, D, lam, form
        dyn = H.UserDynamics(PROBE_ID, 1, 2, 1, ProbeDynParams())  # ControlLimits defaults: +-FLT_MAX, no deadband
        self.cp = ProbeCostParams()
        self.cp.discount, self.cp.horizon, self.cp.inf_at = 1.0, float(T), float(F32_MAX)
        for k, v in env.items():
            os.environ[k] = v
        try:
            self.e = H.Engine(dyn, H.UserCost(PROBE_ID, self.cp), H.GaussianDistribution(2, [1.0, 1.0]), N, T, D,
                              flags=fflags | flags)
        finally:
            for k in env:
                del os.environ[k]
        self.e.set_solver(1.0, lam, 0.0)
        info = self.e.launch_info()
        spt = 2 if form == "spt2" else 1
        self.bx = info["block"] * spt
        self.nrec = info["grid"]
        assert self.nrec == -(-N // self.bx)
        if form.startswith("bx"):
            assert self.bx == int(form[2:])
        # float additions on the way to eta_b: the thread's SPT samples, the 5-level warp tree, the per-warp partials
        self.eta_levels = spt + 5 + info["block"] // 32

    def close(self):
        self.e.close()

    def run(self, costs, stride=1, seed=0):
        """Give sample n the cost costs[n] (float32; +inf allowed) and solve. Sample 0 is noise-free, so its cost goes
        through zero_cost, which every sample whose chosen cost is 0 shares. Returns (U, stats, device costs,
        expected costs, controls [N][T][C])."""
        N, T = self.N, self.T
        c = np.asarray(costs, np.float32)
        assert c.shape == (N,)
        assert np.all((c[1:] != 0) | (c[1:] == c[0])), "a chosen cost of 0 is sample 0's cost"
        t0 = T - 1
        assert t0 >= stride, "the cost step must not use the mean"
        self.cp.zero_cost = float(c[0]) if np.isfinite(c[0]) else 0.0
        assert np.isfinite(c[0]), "sample 0's cost goes through zero_cost, which is finite"
        self.e.push_cost()
        rng = np.random.default_rng(seed)
        eps = np.zeros((N, T, 2), np.float32)
        eps[:, t0, 0] = c
        eps[:, :, 1] = rng.standard_normal((N, T)).astype(np.float32)
        self.e.set_noise(eps)
        x0 = np.zeros((self.D, 1), np.float32)
        U0 = np.zeros((self.D, T, 2), np.float32)
        self.e.rollout_only(x0, U0, stride, 0)
        U, stats = self.e.reduce_only()
        # the controls the rollout applied: eps (mean 0, sigma 1), clamped to +-FLT_MAX; the mean (0) for sample 0 and t < stride
        u = np.clip(eps, -F32_MAX, F32_MAX)
        u[0] = 0.0
        u[:, :stride] = 0.0
        # the cost the engine computes: running 0 / T + (T * x) / T in float32, x = the clamped control or zero_cost
        Tf = np.float32(T)
        x = np.where(u[:, t0, 0] == 0.0, np.float32(self.cp.zero_cost), u[:, t0, 0])
        with np.errstate(over="ignore"):
            expect = np.float32(0.0) / Tf + (Tf * x) / Tf
        expect = np.where(u[:, t0, 0] >= F32_MAX, np.float32(np.inf), expect).astype(np.float32)
        return U, stats, self.e.get_costs(), expect, u

    def check(self, costs, stride=1, seed=0):
        U, stats, dev, expect, u = self.run(costs, stride, seed)
        for d in range(self.D):
            # bit-exact: the test chose these costs
            np.testing.assert_array_equal(dev[d], expect, err_msg=f"{self.form} d={d}: device costs")
            _check_softmin(U[d], stats[d], expect, u, self.lam, self.bx, self.nrec, self.eta_levels, f"{self.form} d={d}")
        wd = self.e.get_weights()
        for d in range(self.D):
            _check_weights(wd[d], expect, self.lam, f"{self.form} d={d}: get_weights")
        return U, stats, expect


def _blocks(N, bx):
    return [(b, min(b + bx, N)) for b in range(0, N, bx)]


# each case: (N, T, lambda) and a function (rng, N, bx, lambda) -> costs [N] float32
def _uniform(rng, N, lo, hi):
    return rng.uniform(lo, hi, N).astype(np.float32)


def _case_inf_block(rng, N, bx, lam):
    c = _uniform(rng, N, 1.0, 1.0 + 5.0 * lam)
    c[bx:2 * bx] = np.inf  # block 1: every sample +inf
    return c


def _case_inf_last_block(rng, N, bx, lam):
    c = _uniform(rng, N, 1.0, 1.0 + 5.0 * lam)
    c[(N - 1) // bx * bx:] = np.inf  # the ragged last block, all +inf
    return c


def _case_scattered_inf(rng, N, bx, lam):
    c = _uniform(rng, N, 1.0, 1.0 + 5.0 * lam)
    c[1:][rng.random(N - 1) < 0.2] = np.inf
    return c


def _spread_within(s):
    def f(rng, N, bx, lam):  # every block spans [1, 1 + s lambda], both ends present
        c = _uniform(rng, N, 1.0, 1.0 + s * lam)
        for lo, hi in _blocks(N, bx):
            c[lo] = np.float32(1.0 + s * lam) if lo else c[lo]
            c[hi - 1] = np.float32(1.0) if hi - 1 else c[hi - 1]
        return c
    return f


def _spread_between(s):
    def f(rng, N, bx, lam):  # block k sits at k / (nblocks - 1) * s lambda, one lambda wide
        blocks = _blocks(N, bx)
        c = np.empty(N, np.float32)
        for k, (lo, hi) in enumerate(blocks):
            off = (len(blocks) - 1 - k) / max(len(blocks) - 1, 1) * s * lam
            c[lo:hi] = (1.0 + off + rng.uniform(0.0, lam, hi - lo)).astype(np.float32)
        return c
    return f


def _case_ties(rng, N, bx, lam):
    c = _uniform(rng, N, 3.0, 3.0 + 5.0 * lam)
    for lo, hi in _blocks(N, bx)[::2]:  # every other block holds the minimum, once or twice
        c[rng.integers(max(lo, 1), hi, 2)] = np.float32(3.0)
    return c


def _case_near_1e16(rng, N, bx, lam):
    # 1e16 + k ulps, k = 0..7: consecutive positive floats have consecutive bit patterns
    bits = np.float32(1e16).view(np.int32) + rng.integers(0, 8, N).astype(np.int32)
    return bits.view(np.float32)


def _case_negative(rng, N, bx, lam):
    return _uniform(rng, N, -50.0 * lam, -40.0 * lam)


def _case_mixed_sign(rng, N, bx, lam):
    return _uniform(rng, N, -3.0 * lam, 3.0 * lam)


ULP_1E16 = float(np.spacing(np.float32(1e16)))  # 2^30
CASES = {
    "inf_block": (1037, 64, 1.0, _case_inf_block),
    "inf_last_block": (1037, 64, 1.0, _case_inf_last_block),
    "scattered_inf": (1037, 64, 1.0, _case_scattered_inf),
    "spread_within_10": (1037, 64, 1.0, _spread_within(10.0)),
    "spread_within_100": (1037, 64, 1.0, _spread_within(100.0)),
    "spread_within_1e4": (1037, 64, 1.0, _spread_within(1e4)),
    "spread_between_10": (1037, 64, 1.0, _spread_between(10.0)),
    "spread_between_100": (1037, 64, 1.0, _spread_between(100.0)),
    "spread_between_1e4": (1037, 64, 1.0, _spread_between(1e4)),
    "ties": (1037, 64, 1.0, _case_ties),
    "near_1e16_lambda_ulp": (1037, 64, ULP_1E16, _case_near_1e16),
    "near_1e16_lambda_1": (1037, 64, 1.0, _case_near_1e16),
    "negative": (1037, 64, 1.0, _case_negative),
    "mixed_sign": (1037, 64, 1.0, _case_mixed_sign),
    "lambda_1e-3": (1037, 64, 1e-3, _spread_within(10.0)),
    "lambda_1e6": (1037, 64, 1e6, _spread_between(10.0)),
    "ragged_last_block_min": (1025, 64, 1.0, None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("case", list(CASES))
def test_probe_costs_softmin_matches_float64(form, case):
    N, T, lam, gen = CASES[case]
    p = Probe(N, T, form, lam)
    try:
        rng = np.random.default_rng(zlib.crc32(case.encode()))
        if gen is None:  # one sample in the last block, and it is the minimum
            c = _uniform(rng, N, 2.0, 7.0)
            c[N - 1] = np.float32(1.0)
        else:
            c = gen(rng, N, p.bx, lam)
        U, stats, expect = p.check(c)
        if case.startswith("inf") or case == "scattered_inf":
            assert np.isinf(expect).any() and np.all(np.isfinite(U))
    finally:
        p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["resident", "stream", "spt2", "D2"])
def test_probe_all_infinite_costs_give_nan_control(form):
    """Every sample but the noise-free one costs +inf, and sample 0 too: the reference's global baseline is +inf and its
    weights expf(-(inf - inf)) are NaN, so U is NaN. Here every record is empty: U = 0 / 0 = NaN, baseline +inf, and the
    normaliser and sum w^2 of the empty merge are 0."""
    N, T = 1037, 64
    p = Probe(N, T, form)
    try:
        p.cp.inf_at = 0.0  # every state >= 0 costs +inf, sample 0's included
        c = np.full(N, np.float32(5.0))
        c[1:] = np.inf
        U, stats, dev, expect, u = p.run(c)
        assert np.all(np.isinf(dev)) and np.all(dev > 0)
        assert np.all(np.isnan(U))
        for d in range(p.D):
            assert stats[d][0] == np.inf and stats[d][1] == 0.0 and stats[d][2] == 0.0
    finally:
        p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 17, 100])  # T*C = 2, 34, 200
def test_probe_merge_at_the_record_limit(T):
    """N = 4096 * 32 at BX = 32: K2 merges exactly kCombineMaxRecords = 4096 records (all 8 header slots per thread), with
    one all-+inf block, ties of the minimum in the first and the last record, and a spread of 20 lambda; then a record count
    that is not a multiple of 64 (the tail of K2's 4-way unrolled column loop), and 4097 records, which are refused."""
    stride = 0 if T == 1 else 1
    for N in (4096 * 32, 4059 * 32 + 5):
        p = Probe(N, T, "bx32")
        try:
            assert p.nrec == -(-N // 32)
            rng = np.random.default_rng(T + N)
            c = _uniform(rng, N, 2.0, 22.0)
            c[32 * 100:32 * 101] = np.inf
            c[rng.integers(1, N, 64)] = np.inf
            c[5] = c[N - 3] = np.float32(2.0) - np.float32(2.0 ** -22)
            p.check(c, stride=stride)
        finally:
            p.close()
    with pytest.raises(H.MppibError, match="exceed"):
        Probe(4097 * 32, T, "bx32")


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["resident", "stream", "no_tma"])
@pytest.mark.parametrize("gamma,r", [(3.0, 1.5), (3.0, 2.0), (0.5, 3.0)])
def test_probe_tsallis_weights_at_their_cutoff(form, gamma, r):
    """Tsallis weights w = (1 - (c - beta) / gamma)^(1 / (r - 1)) for c - beta < gamma, else 0, with costs exactly at the
    cutoff, one ulp inside and outside it, and +inf. Device: expf(logf(1 - fl(c - beta) / gamma) / (r - 1)) in float; its
    error in the exponent is |q| (3 u x / (1 - x) + 2 u |log(1 - x)|) + 2 u |q log(1 - x)|, q = 1 / (r - 1), x = (c - beta)
    / gamma, and expf adds 4 u."""
    N, T = 1037, 64
    p = Probe(N, T, form, flags=H.FLAG_WRITEBACK_CONTROLS)
    try:
        p.e.set_tsallis(gamma, r)
        rng = np.random.default_rng(11)
        g32 = np.float32(gamma)
        beta = np.float32(1.0)
        c = (beta + rng.uniform(0.0, 1.5 * gamma, N)).astype(np.float32)
        c[0] = beta
        edge = np.float32(beta + g32)  # beta + gamma is exact for these (gamma, beta)
        assert np.float32(edge - beta) == g32
        c[1:40:3] = edge
        c[2:40:3] = np.nextafter(edge, np.float32(0))
        c[3:40:3] = np.nextafter(edge, np.float32(np.inf))
        c[40:60] = np.inf
        U, stats, dev, expect, u = p.run(c)
        np.testing.assert_array_equal(dev[0], expect)
        # the device's cutoff decision is a float comparison of fl(c - beta) with gamma: emulate it exactly
        cd32 = expect - np.float32(expect.min())
        inside = cd32 < g32
        assert not inside[1:40:3].any() and inside[2:40:3].all() and not inside[3:40:3].any()
        x = np.where(inside, (expect.astype(np.float64) - float(expect.min())) / gamma, 0.0)
        q = 1.0 / (r - 1.0)
        L = np.log1p(-x)
        w = np.where(inside, np.exp(q * L), 0.0)
        E = abs(q) * (3 * U32 * x / np.maximum(1.0 - x, 1e-300) + 2 * U32 * np.abs(L)) + 2 * U32 * np.abs(q * L) + 4 * U32
        dw = np.where(inside, np.expm1(E) * w + SUB, 0.0)
        eta = w.sum()
        assert stats[0][0] == expect.min()
        assert abs(stats[0][1] - eta) <= dw.sum() + U32 * eta
        assert abs(stats[0][2] - (w * w).sum()) <= (2 * dw * w).sum() + U32 * (w * w).sum()
        uu = u.reshape(N, -1).astype(np.float64)
        Uref = (w @ uu) / eta
        k_acc = N // 16 + 16 + 2
        bound = (dw @ np.abs(uu - Uref[None])) / eta + k_acc * U32 * (w @ np.abs(uu)) / eta + 2 * U32 * np.abs(Uref)
        assert np.all(np.abs(U[0].reshape(-1) - Uref) <= bound)
    finally:
        p.close()


# ---- every K1 instantiation of the real pairs, against float64 from its own outputs ---------------------------------------------
# (label, workload builder, environment, descriptor flags, T); the labels follow tools/k1_plan_matrix.py's overrides
K1_FORMS = [
    ("cartpole", W.cartpole, {}, 0, 38),  # C = 1: the host-API normal draw needs an even N * T * C
    ("cartpole NO_TMA", W.cartpole, {"MPPIB_NO_TMA": "1"}, 0, 64),
    ("cartpole STREAM=1", W.cartpole, {"MPPIB_STREAM": "1"}, 0, 64),
    ("cartpole STREAM_READBACK", W.cartpole, {"MPPIB_STREAM": "1", "MPPIB_STREAM_READBACK": "1"}, 0, 64),
    ("cartpole BX=64", W.cartpole, {"MPPIB_BX": "64"}, 0, 64),
    ("double_integrator_tube D=2", W.double_integrator_tube, {}, 0, 37),
    ("double_integrator_tube D=2 STREAM=1", W.double_integrator_tube, {"MPPIB_STREAM": "1"}, 0, 64),
    ("double_integrator_robust_tube RMPPI", W.double_integrator_robust_tube, {}, H.FLAG_RMPPI, 37),
    ("autorally ws", W.autorally, {}, 0, 64),
    ("autorally ws PSPW=8", W.autorally, {"MPPIB_WS_PSPW": "8"}, 0, 37),
    ("autorally ws PSPW=16", W.autorally, {"MPPIB_WS_PSPW": "16"}, 0, 64),
    ("autorally ws PSPW=32", W.autorally, {"MPPIB_WS_PSPW": "32"}, 0, 64),
    ("autorally ws STREAM=1", W.autorally, {"MPPIB_STREAM": "1"}, 0, 64),
    ("autorally ws PSPW=32 STREAM=1", W.autorally, {"MPPIB_STREAM": "1", "MPPIB_WS_PSPW": "32"}, 0, 37),
    ("autorally_robust ws", W.autorally_robust, {}, 0, 64),
    ("autorally mma SPW=32", W.autorally, {"MPPIB_NO_WS": "1"}, 0, 64),
    ("autorally mma SPW=16", W.autorally, {"MPPIB_SPW": "16"}, 0, 37),
    ("autorally mma SPW=8", W.autorally, {"MPPIB_SPW": "8"}, 0, 64),
    ("autorally FFMA2", W.autorally, {"MPPIB_NN_FFMA2": "1"}, 0, 64),
    ("autorally FFMA2 SPT=2", W.autorally, {"MPPIB_NN_FFMA2": "1", "MPPIB_SPT": "2"}, 0, 37),
    ("autorally wgmma", W.autorally, {"MPPIB_NN_TENSOR": "1"}, 0, 64),
    ("racer_lstm_h32 tensor-core", W.racer_lstm_h32, {}, 0, 37),
    ("racer_lstm_h32 SIMT", W.racer_lstm_h32, {"MPPIB_LSTM_SIMT": "1"}, 0, 64),
    ("racer_lstm", W.racer_lstm, {}, 0, 37),
    ("racer_suspension", W.racer_suspension, {}, 0, 64),
    ("quadrotor", W.quadrotor, {}, 0, 37),
    ("quadrotor_gates", W.quadrotor_gates, {}, 0, 64),
]


def _k1_engine(builder, env, flags, T, N=1037):
    w = builder(N, T)
    for k, v in env.items():
        os.environ[k] = v
    try:
        return w, w.make_engine(flags=flags)
    finally:
        for k in env:
            del os.environ[k]


@pytest.mark.gpu
@pytest.mark.parametrize("label,builder,env,flags,T", K1_FORMS, ids=[f[0] for f in K1_FORMS])
def test_k1_form_softmin_matches_float64_of_its_own_outputs(label, builder, env, flags, T):
    w, e = _k1_engine(builder, env, flags | H.FLAG_WRITEBACK_CONTROLS, T)
    try:
        info = e.launch_info()
        U, stats = e.solve(w.x0, w.U0, w.optimization_stride, 0)
        costs, samples, wts = e.get_costs(), e.get_samples(), e.get_weights()
        # rows of a block's sequential weighted sum: at most the block's samples (the warp-specialised streaming form splits
        # them into slices, which only shortens the chain)
        bx = -(-e.n_local // info["grid"])
        for d in range(w.D):
            assert np.all(np.isfinite(costs[d])), label
            _check_softmin(U[d], stats[d], costs[d], samples[d], w.lambda_, bx, info["grid"], 2 + 5 + info["block"] // 32,
                           f"{label} d={d}")
            _check_weights(wts[d], costs[d], w.lambda_, f"{label} d={d}: get_weights")
    finally:
        e.close()
    # the same seed without write-back: the instantiation the benchmark runs computes the same numbers
    w2, e2 = _k1_engine(builder, env, flags, T)
    try:
        U2, stats2 = e2.solve(w2.x0, w2.U0, w2.optimization_stride, 0)
        np.testing.assert_array_equal(e2.get_costs(), costs, err_msg=label)
        np.testing.assert_array_equal(U2, U, err_msg=label)
        assert stats2 == stats, label
    finally:
        e2.close()
