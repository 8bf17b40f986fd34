"""The three rollouts that run beside the solve, through the C ABI: init-eval (mppib_init_eval), sampled trajectories
(mppib_sample_trajectories) and the device-side roll-forward (mppib_nominal_trajectory).

- Every refusal of the three entry points that one GPU can reach, with its status and message. Not reached here:
  init-eval's refusal of a rank of several, which needs an engine that has joined a communicator of two ranks.
- A refused negative stride draws no noise and runs no kernel: the next init-eval and the next solve are bit-identical
  to a fresh engine's on the same seed.
- Scratch that grows and then shrinks between calls leaves every result bit-identical to a fresh engine's on the same
  inputs."""
import ctypes as C

import numpy as np
import pytest

import mppi_generic_b200 as m
from mppi_generic_b200 import workloads as W

H = m.host
INVALID, UNSUPPORTED, STATE = -1, -2, -9
N, T = 1024, 32  # N * T * C a multiple of 8192, so burn_draws positions the generator like the draws it skips

pytestmark = pytest.mark.gpu


def _refused(status, message, call):
    with pytest.raises(H.MppibError) as ex:
        call()
    assert ex.value.status == status, str(ex.value)
    assert str(ex.value).endswith(": " + message), str(ex.value)


def _raw(name, *args):
    H._check(getattr(H.lib(), name)(*args))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _candidates(K, seed):
    rng = np.random.RandomState(seed)
    cand = (0.1 * rng.randn(K, 4)).astype(np.float32)
    strides = rng.randint(0, T + 4, size=K).astype(np.int32)  # a stride past the horizon holds its last control
    U_nom = (0.5 * rng.randn(T, 1)).astype(np.float32)
    return cand, strides, U_nom


# ---- refusals ----------------------------------------------------------------------------------------------------------
def test_init_eval_refusals():
    w = W.cartpole(N, T)
    e = w.make_engine()
    K, spc = 3, 16
    cand, strides, U_nom = _candidates(K, 1)
    costs = np.empty(K * spc, np.float32)

    def call(h=e._h, c=cand, s=strides, k=K, n=spc, u=U_nom, out=costs):
        return lambda: _raw("mppib_init_eval", h, _p(c), _p(s), k, n, _p(u), 1, _p(out))

    _refused(INVALID, "null engine", call(h=None))
    for kw in ({"c": None}, {"s": None}, {"u": None}, {"out": None}, {"k": 0}, {"n": 0}, {"n": -1}):
        _refused(INVALID, "bad argument", call(**kw))
    too_many = "(number of candidates) * (samples per candidate) cannot exceed NUM_ROLLOUTS"
    _refused(INVALID, too_many, call(n=N + 1))
    _refused(INVALID, too_many, call(k=2, n=N // 2 + 1))
    before = e.rng_offset()
    bad = strides.copy()
    bad[2] = -1
    _refused(INVALID, "stride -1 (candidate 2) is negative", call(s=bad))
    bad[1] = -40
    _refused(INVALID, "stride -40 (candidate 1) is negative", call(s=bad))
    assert e.rng_offset() == before  # no noise was drawn
    e.close()

    e = H.Engine(w.dyn, w.cost, w.sampler, N, T, rank=0, world_size=2)
    _refused(STATE, "world_size > 1 but mppib_comm_init was not called", call(h=e._h))
    e.close()


def test_sample_trajectories_refusals():
    w = W.cartpole(N, T)
    x0, U0 = _f32(w.x0[0]), _f32(w.U0[0])
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    U_opt = _f32(w.U0[0] + 0.1)
    idx = np.array([-1, 0, 5], np.int32)
    n = idx.size
    outputs = np.empty((n, T, w.dyn.OUTPUT_DIM), np.float32)
    costs = np.empty((n, T + 1), np.float32)
    crash = np.empty((n, T), np.int32)

    def call(h=e._h, x=x0, u=U0, d=0, i=idx, k=n, opt=U_opt, out=outputs, c=costs, cr=crash):
        return lambda: _raw("mppib_sample_trajectories", h, _p(x), _p(u), d, _p(i), k, _p(opt), _p(out), _p(c), _p(cr))

    _refused(INVALID, "null engine", call(h=None))
    _refused(STATE, "no solve has been run yet", call())
    e.solve(w.x0, w.U0)
    for kw in ({"x": None}, {"u": None}, {"i": None}, {"k": 0}, {"out": None}, {"c": None}, {"cr": None}):
        _refused(INVALID, "bad argument", call(**kw))
    _refused(INVALID, "distribution 1 out of range [0, 1)", call(d=1))
    _refused(INVALID, "distribution -1 out of range [0, 1)", call(d=-1))
    e.solve_async(_f32(w.x0), _f32(w.U0))
    _refused(STATE, "a solve is in flight (mppib_solve_wait first)", call())
    e.solve_wait()
    _refused(INVALID, f"sample index {N} (entry 1) outside [-1, {N})", call(i=np.array([0, N, 1], np.int32)))
    _refused(INVALID, f"sample index -2 (entry 0) outside [-1, {N})", call(i=np.array([-2, 0, 1], np.int32)))
    _refused(INVALID, "index -1 needs U_opt", call(opt=None))
    _refused(INVALID, "x0[2] is not finite", call(x=np.array([0.0, 0.0, np.inf, 0.0], np.float32)))
    call(opt=None, i=np.array([0, 1, 2], np.int32))()  # U_opt is needed only for index -1
    e.close()

    e = w.make_engine()
    e.solve(w.x0, w.U0)
    _refused(STATE, "sampled trajectories re-roll the written-back controls: create the engine with "
                    "MPPIB_FLAG_WRITEBACK_CONTROLS", call(h=e._h))
    e.close()

    wt = W.double_integrator_tube(N, T)
    e = wt.make_engine(flags=H.FLAG_RMPPI)
    _refused(UNSUPPORTED, "sampled trajectories are built for the Vanilla / Tube / Colored rollouts",
             call(h=e._h, x=_f32(wt.x0[0]), u=_f32(wt.U0[0]), opt=_f32(wt.U0[0])))
    e.close()


def test_nominal_trajectory_refusals():
    w = W.double_integrator_tube(N, T)
    x0, U = _f32(w.x0), _f32(w.U0)
    e = w.make_engine()
    Us = np.empty((2, T, 2), np.float32)
    states = np.empty((2, T, 4), np.float32)
    outputs = np.empty((2, T, w.dyn.OUTPUT_DIM), np.float32)

    def call(h=e._h, x=x0, u=U, hist=None, us=Us, st=states, out=outputs):
        return lambda: _raw("mppib_nominal_trajectory", h, _p(x), _p(u), _p(hist), _p(us), _p(st), _p(out))

    _refused(INVALID, "null engine", call(h=None))
    for kw in ({"x": None}, {"st": None}, {"out": None}):
        _refused(INVALID, "null argument", call(**kw))
    _refused(STATE, "U == NULL rolls out the last solve's result, and no solve has been run yet", call(u=None))
    bad = x0.copy()
    bad[1, 0] = np.nan
    _refused(INVALID, "x0[4] is not finite", call(x=bad))
    call(us=None)()  # U_smoothed is optional
    e.close()

    w1 = W.cartpole(N, 1)
    e = w1.make_engine()
    _refused(INVALID, "needs at least two time steps",
             call(h=e._h, x=_f32(w1.x0), u=_f32(w1.U0), us=None, st=np.empty((1, 1, 4), np.float32),
                  out=np.empty((1, 1, w1.dyn.OUTPUT_DIM), np.float32)))
    e.close()


# ---- the generator after a refusal ---------------------------------------------------------------------------------------
def test_refused_negative_stride_moves_nothing():
    w = W.cartpole(N, T)
    cand, strides, U_nom = _candidates(4, 2)
    bad = strides.copy()
    bad[3] = -5
    runs = []
    for refuse_first in (True, False):
        e = w.make_engine()
        if refuse_first:
            with pytest.raises(H.MppibError):
                e.init_eval(cand, bad, 64, U_nom, 2)
        costs = e.init_eval(cand, strides, 64, U_nom, 2)
        U, stats = e.solve(w.x0, w.U0)
        runs.append((costs, U, np.array(stats), e.get_costs(), e.rng_offset()))
        e.close()
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


# ---- scratch that grows, then shrinks ----------------------------------------------------------------------------------
def test_init_eval_grow_then_shrink_matches_fresh_engines():
    w = W.cartpole(N, T)
    e = w.make_engine()
    for i, (K, spc) in enumerate(((2, 16), (9, 100), (3, 8))):
        cand, strides, U_nom = _candidates(K, 10 + i)
        got = e.init_eval(cand, strides, spc, U_nom, 3)
        f = w.make_engine()
        f.burn_draws(i)  # the draws e's earlier calls made
        want = f.init_eval(cand, strides, spc, U_nom, 3)
        assert e.rng_offset() == f.rng_offset()
        assert np.array_equal(got, want), (K, spc)
        f.close()
    e.close()


def test_sample_trajectories_grow_then_shrink_matches_fresh_engines():
    w = W.cartpole(N, T)
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    U_opt, _ = e.solve(w.x0, w.U0)
    rng = np.random.RandomState(4)
    for n in (6, 300, 4):
        idx = np.concatenate([[-1], rng.randint(0, N, size=n - 1)]).astype(np.int32)
        got = e.sample_trajectories(w.x0[0], w.U0[0], idx, U_opt=U_opt[0])
        f = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
        f.solve(w.x0, w.U0)
        want = f.sample_trajectories(w.x0[0], w.U0[0], idx, U_opt=U_opt[0])
        for a, b in zip(got, want):
            assert np.array_equal(a, b), n
        f.close()
    e.close()


@pytest.mark.parametrize("name", ["cartpole", "double_integrator_tube"])
def test_nominal_trajectory_sources_match_fresh_engines(name):
    """The caller's U, then the last solve's result record, then U again: each call as a fresh engine's first."""
    w = {"cartpole": W.cartpole, "double_integrator_tube": W.double_integrator_tube}[name](N, T)
    x0 = _f32(w.x0)
    rng = np.random.RandomState(5)
    hist = (0.1 * rng.standard_normal((2, w.dyn.CONTROL_DIM))).astype(np.float32)
    U_own = (0.3 * rng.standard_normal(w.U0.shape)).astype(np.float32)
    e = w.make_engine()
    e.solve(x0, w.U0)
    for U, h in ((U_own, hist), (None, hist), (None, None), (U_own, None)):
        got = e.nominal_trajectory(x0, U, h)
        f = w.make_engine()
        f.solve(x0, w.U0)
        want = f.nominal_trajectory(x0, U, h)
        for a, b in zip(got, want):
            assert np.array_equal(a, b, equal_nan=True), (U is None, h is None)
        f.close()
    e.close()
