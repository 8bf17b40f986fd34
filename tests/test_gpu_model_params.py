"""The model's blobs through the C ABI (mppib_set_blob): every refusal of a malformed or misplaced blob with its status and
message, the guard against replacing a blob that kernels of a pending solve read, each "not set" refusal of a solve and of
mppib_ddp_feedback, and blobs replaced between solves, which must give what a fresh engine given them from the start gives.
The cost texture's and the costmap's own validations are in test_quadrotor_map_cost.py and test_robust_costs.py."""
import ctypes as C

import numpy as np
import pytest

import mppi_generic_b200 as m
from mppi_generic_b200 import workloads as W

H = m.host
INVALID, STATE = -1, -9


def _blobs(w):
    """(kind, bytes) of every blob H.Engine.push_params would give this workload, in its order."""
    out = [(H.BLOB_DYN, w.dyn.blob()), (H.BLOB_COST, w.cost.blob()), (H.BLOB_SAMPLER, w.sampler.blob())]
    if w.dyn.DYN_ID == H.DYN_AUTORALLY_NN:
        out.append((H.BLOB_NN_WEIGHTS, np.ascontiguousarray(w.dyn.nn_theta, np.float32).tobytes()))
    if w.dyn.DYN_ID == H.DYN_RACER_LSTM:
        out.append((H.BLOB_LSTM_WEIGHTS, np.ascontiguousarray(w.dyn.lstm_theta, np.float32).tobytes()))
    if w.cost.COST_ID in (H.COST_AR_STANDARD, H.COST_AR_ROBUST):
        out.append((H.BLOB_COSTMAP, np.ascontiguousarray(w.cost.costmap, np.float32).tobytes()))
    return out


def _set(h, which, data, nbytes=None):
    buf = C.create_string_buffer(bytes(data), max(len(data), 1))
    return H.lib().mppib_set_blob(h, which, buf, len(data) if nbytes is None else nbytes)


def _err():
    return (H.lib().mppib_last_error() or b"").decode()


class _Bare:
    """An engine made through mppib_create with no blob set (H.Engine pushes every blob)."""

    def __init__(self, w, skip=()):
        self.w = w
        self.h = C.c_void_p()
        d = H.Desc(w.dyn.DYN_ID, w.cost.COST_ID, w.sampler.SAMPLER_ID, w.N, w.T, w.D, 0, 0, None, 0, 1)
        for i, v in enumerate(w.dyn.model_dims()):
            d.model_dims[i] = v
        assert H.lib().mppib_create(C.byref(self.h), C.byref(d)) == 0, _err()
        for which, data in _blobs(w):
            if which not in skip:
                assert _set(self.h, which, data) == 0, _err()

    def solve(self):
        x0 = np.ascontiguousarray(self.w.x0, np.float32)
        U = np.ascontiguousarray(self.w.U0, np.float32)
        U_out = np.empty_like(U)
        stats = (H.SolveStats * self.w.D)()
        return H.lib().mppib_solve(self.h, x0.ctypes.data, U.ctypes.data, 1, 0, U_out.ctypes.data, stats)

    def ddp(self):
        S, Cd, T = self.w.dyn.STATE_DIM, self.w.dyn.CONTROL_DIM, self.w.T
        x0 = np.ascontiguousarray(self.w.x0[0], np.float32)
        xt, ut = np.zeros((T, S), np.float32), np.zeros((T, Cd), np.float32)
        g, xs, us = np.empty((T, S, Cd), np.float32), np.empty((T, S), np.float32), np.empty((T, Cd), np.float32)
        return H.lib().mppib_ddp_feedback(self.h, T, x0.ctypes.data, xt.ctypes.data, ut.ctypes.data, 0, g.ctypes.data,
                                          xs.ctypes.data, us.ctypes.data, None)

    def close(self):
        H.lib().mppib_destroy(self.h)


def _hills(w=48, h=40, res=0.5, origin=(-6.0, -10.0, 0.0), seed=5):
    rng = np.random.default_rng(seed)
    j, i = np.meshgrid(np.arange(w), np.arange(h))
    x, y = (j + 0.5) * res + origin[0], (i + 0.5) * res + origin[1]
    z = 0.6 * np.sin(0.21 * x) * np.cos(0.17 * y) + 0.02 * rng.standard_normal(x.shape)
    return z.astype(np.float32), res, origin


def _racer(seed=2, cells=(48, 40)):
    w = W.racer_lstm_gaussian(1024, 40)
    w.dyn.setAllValues(*W.synthetic_lstm_weights(4, 20, seed))
    vals, res, origin = _hills(*cells)
    w.dyn.setElevationMap(vals, res, origin)
    return w


def _expect(rc, status, text):
    assert rc == status, (rc, _err())
    assert text in _err(), _err()


@pytest.mark.gpu
def test_parameter_and_weight_refusals():
    ar, racer, cart = W.autorally(512, 20), _racer(), W.cartpole(512, 20)
    a, r, c = _Bare(ar), _Bare(racer), _Bare(cart)
    try:
        _expect(_set(a.h, H.BLOB_DYN, ar.dyn.blob()[:-4]), INVALID, "dynamics params: got")
        _expect(_set(a.h, H.BLOB_COST, ar.cost.blob() + b"\0" * 4), INVALID, "cost params: got")
        nn = np.ascontiguousarray(ar.dyn.nn_theta, np.float32)
        _expect(_set(a.h, H.BLOB_NN_WEIGHTS, nn[:-1].tobytes()), INVALID, "NN weights: got")
        bad = nn.copy()
        bad[7] = np.inf
        _expect(_set(a.h, H.BLOB_NN_WEIGHTS, bad.tobytes()), INVALID, "NN weight 7 is not finite")
        lstm = np.ascontiguousarray(racer.dyn.lstm_theta, np.float32)
        _expect(_set(r.h, H.BLOB_LSTM_WEIGHTS, lstm[:-1].tobytes()), INVALID, "LSTM weights: got")
        bad = lstm.copy()
        bad[5] = np.nan
        _expect(_set(r.h, H.BLOB_LSTM_WEIGHTS, bad.tobytes()), INVALID, "LSTM weight 5 is not finite")
        # blobs given to a model that takes none
        _expect(_set(c.h, H.BLOB_NN_WEIGHTS, nn.tobytes()), INVALID, "NN weights given to a non-NN dynamics")
        _expect(_set(a.h, H.BLOB_LSTM_WEIGHTS, lstm.tobytes()), INVALID, "LSTM weights given to a dynamics without an LSTM")
        emap = racer.dyn.getTextureHelper().blob()
        _expect(_set(a.h, H.BLOB_ELEVATION_MAP, emap.tobytes()), INVALID, "elevation map given to a dynamics without one")
        _expect(_set(a.h, 99, b"\0" * 16), INVALID, "unknown blob kind 99")
        # the refused blobs left what was set before: both engines still solve
        assert a.solve() == 0, _err()
        assert r.solve() == 0, _err()
    finally:
        for e in (a, r, c):
            e.close()


@pytest.mark.gpu
def test_elevation_map_header_refusals():
    racer = _racer()
    r = _Bare(racer)
    good = racer.dyn.getTextureHelper().blob()
    hdr_bytes = C.sizeof(H.ElevationMapHeader)

    def patched(field, index, value):
        hd = H.ElevationMapHeader.from_buffer_copy(good[:hdr_bytes].tobytes())
        if index is None:
            setattr(hd, field, value)
        else:
            getattr(hd, field)[index] = value
        return bytes(hd) + good[hdr_bytes:].tobytes()

    try:
        _expect(_set(r.h, H.BLOB_ELEVATION_MAP, good[:16].tobytes()), INVALID, "elevation map: 16 bytes is smaller than")
        _expect(_set(r.h, H.BLOB_ELEVATION_MAP, patched("width", None, 1)), INVALID, "elevation map: extent 1 x")
        _expect(_set(r.h, H.BLOB_ELEVATION_MAP, patched("height", None, 16385)), INVALID, "need 2 .. 16384 cells")
        _expect(_set(r.h, H.BLOB_ELEVATION_MAP, good[:-4].tobytes()), INVALID, "elevation map: got")
        _expect(_set(r.h, H.BLOB_ELEVATION_MAP, patched("origin", 2, np.nan)), INVALID,
                "origin / resolution component 2 is not usable")
        _expect(_set(r.h, H.BLOB_ELEVATION_MAP, patched("resolution", 1, 0.0)), INVALID,
                "origin / resolution component 1 is not usable")
        _expect(_set(r.h, H.BLOB_ELEVATION_MAP, patched("rotations", 4, np.inf)), INVALID, "rotation entry 4 is not finite")
        assert _set(r.h, H.BLOB_ELEVATION_MAP, good.tobytes()) == 0, _err()
    finally:
        r.close()


@pytest.mark.gpu
def test_costmap_before_cost_params_is_refused():
    ar = W.autorally(512, 20)
    a = _Bare(ar, skip=(H.BLOB_COST, H.BLOB_COSTMAP))
    try:
        costmap = np.ascontiguousarray(ar.cost.costmap, np.float32).tobytes()
        _expect(_set(a.h, H.BLOB_COSTMAP, costmap), STATE, "set MPPIB_BLOB_COST_PARAMS (map_width/map_height) before")
        assert _set(a.h, H.BLOB_COST, ar.cost.blob()) == 0, _err()
        assert _set(a.h, H.BLOB_COSTMAP, costmap) == 0, _err()
    finally:
        a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["autorally", "racer", "quadrotor_map"])
def test_blobs_kernels_read_are_refused_while_a_solve_is_pending(case):
    if case == "autorally":
        w = W.autorally(1024, 20)
        kinds = _blobs(w)[3:]
        assert [k for k, _ in kinds] == [H.BLOB_NN_WEIGHTS, H.BLOB_COSTMAP]
    elif case == "racer":
        w = _racer()
        kinds = [_blobs(w)[3], (H.BLOB_ELEVATION_MAP, w.dyn.getTextureHelper().blob().tobytes())]
        assert kinds[0][0] == H.BLOB_LSTM_WEIGHTS
    else:
        w = W.quadrotor_gates(1024, 20)
        kinds = [(H.BLOB_COST_TEXTURE, w.cost.tex_helper_.blob().tobytes())]
    e = w.make_engine()
    try:
        e.solve_async(np.ascontiguousarray(w.x0, np.float32), np.ascontiguousarray(w.U0, np.float32))
        for which, data in kinds:
            _expect(_set(e._h, which, data), STATE, f"mppib_set_blob({which}) while a solve is pending")
        assert _set(e._h, H.BLOB_DYN, w.dyn.blob()) == 0, _err()  # a host copy: the next launch takes it
        e.solve_wait()
        for which, data in kinds:
            assert _set(e._h, which, data) == 0, _err()
    finally:
        e.close()


@pytest.mark.gpu
def test_solve_refuses_each_missing_blob():
    parts = "dynamics / cost / sampler parameter blobs must be set before solving"
    cases = [(W.cartpole(512, 20), H.BLOB_DYN, parts), (W.cartpole(512, 20), H.BLOB_COST, parts),
             (W.cartpole(512, 20), H.BLOB_SAMPLER, parts),
             (W.autorally(512, 20), H.BLOB_NN_WEIGHTS, "MPPIB_BLOB_NN_WEIGHTS not set"),
             (W.autorally(512, 20), H.BLOB_COSTMAP, "MPPIB_BLOB_COSTMAP not set"),
             (_racer(), H.BLOB_LSTM_WEIGHTS, "MPPIB_BLOB_LSTM_WEIGHTS not set")]
    for w, missing, text in cases:
        e = _Bare(w, skip=(missing,))
        try:
            _expect(e.solve(), STATE, text)
        finally:
            e.close()
    e = _Bare(_racer())  # no elevation map: flat ground
    try:
        assert e.solve() == 0, _err()
    finally:
        e.close()


@pytest.mark.gpu
def test_ddp_feedback_refuses_each_missing_blob():
    w = W.autorally(512, 20)
    e = _Bare(w, skip=(H.BLOB_DYN, H.BLOB_NN_WEIGHTS))
    try:
        _expect(e.ddp(), STATE, "dynamics parameters were not set")
        assert _set(e.h, H.BLOB_DYN, w.dyn.blob()) == 0, _err()
        _expect(e.ddp(), STATE, "network weights were not set")
        assert _set(e.h, H.BLOB_NN_WEIGHTS, np.ascontiguousarray(w.dyn.nn_theta, np.float32).tobytes()) == 0, _err()
        assert e.ddp() == 0, _err()
    finally:
        e.close()


def _same_as_fresh(w_old, w_new, replace):
    """Solve on w_old's engine, replace the blobs `replace` with w_new's, re-seed and solve again: U, stats and per-sample
    costs bit-identical to a fresh engine of w_new on the same seed."""
    e = w_old.make_engine()
    e.solve(w_old.x0, w_old.U0)
    for which, data in replace:
        assert _set(e._h, which, data) == 0, _err()
    e.seed(w_new.seed, 0)
    U, stats = e.solve(w_new.x0, w_new.U0)
    costs = e.get_costs()
    e.close()
    f = w_new.make_engine()
    U_f, stats_f = f.solve(w_new.x0, w_new.U0)
    costs_f = f.get_costs()
    f.close()
    np.testing.assert_array_equal(U, U_f)
    assert stats == stats_f
    np.testing.assert_array_equal(costs, costs_f)
    return U


@pytest.mark.gpu
def test_replaced_nn_weights_and_costmap_match_a_fresh_engine():
    old, new = W.autorally(4096, 40), W.autorally(4096, 40)
    new.dyn.updateModel([6, 32, 32, 4], W.synthetic_nn_weights(5))
    ch0, xb, yb, ppm = W.track_map_standard()
    new.cost.loadTrackData(0.5 * ch0 + 1.0, xb[0], xb[1], yb[0], yb[1], ppm)
    U = _same_as_fresh(old, new, _blobs(new)[3:])
    e = old.make_engine()
    U_old, _ = e.solve(old.x0, old.U0)
    e.close()
    assert not np.array_equal(U, U_old), "the replacement must change the solve"


@pytest.mark.gpu
def test_replaced_lstm_weights_and_elevation_map_match_a_fresh_engine():
    old, new = _racer(2, (48, 40)), _racer(9, (96, 80))  # the new map has four times the cells
    replace = [_blobs(new)[3], (H.BLOB_ELEVATION_MAP, new.dyn.getTextureHelper().blob().tobytes())]
    U = _same_as_fresh(old, new, replace)
    e = old.make_engine()
    U_old, _ = e.solve(old.x0, old.U0)
    e.close()
    assert not np.array_equal(U, U_old), "the replacement must change the solve"
