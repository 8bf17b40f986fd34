"""The rollout kernel's owner (csrc/rollout.cuh), through the C ABI: the written-back controls, the importance weights
and the L2 flush.

- An engine keeps written-back controls under MPPIB_FLAG_WRITEBACK_CONTROLS, RMPPI or the generic streaming form's
  read-back (MPPIB_STREAM_READBACK), and under nothing else: mppib_get_samples and the Tsallis weights follow that one fact.
- mppib_get_weights is refused before the first solve; its buffer, made by the first call, gives the same weights on
  every later call as a fresh engine's first.
- An L2 flush set, cleared and set larger between solves changes no result."""
import ctypes as C

import numpy as np
import pytest

import mppi_generic_b200 as m
from mppi_generic_b200 import workloads as W

H = m.host
INVALID, STATE = -1, -9
N, T = 1024, 32

pytestmark = pytest.mark.gpu


def _refused(status, message, call):
    with pytest.raises(H.MppibError) as ex:
        call()
    assert ex.value.status == status, str(ex.value)
    assert str(ex.value).endswith(": " + message), str(ex.value)


def _raw(name, *args):
    H._check(getattr(H.lib(), name)(*args))


def _streaming_engine(monkeypatch, w, readback):
    """Cartpole in the generic kernel's streaming form (T * C spans more 32-float slabs than its ring holds)."""
    monkeypatch.setenv("MPPIB_STREAM", "1")
    if readback:
        monkeypatch.setenv("MPPIB_STREAM_READBACK", "1")
    e = w.make_engine()  # the overrides are read at create only
    monkeypatch.delenv("MPPIB_STREAM")
    monkeypatch.delenv("MPPIB_STREAM_READBACK", raising=False)
    return e


# ---- written-back controls ---------------------------------------------------------------------------------------------
def test_samples_refused_without_write_back(monkeypatch):
    no_controls = "engine was created without MPPIB_FLAG_WRITEBACK_CONTROLS"
    tsallis = "Tsallis weights reduce the written-back controls: create the engine with MPPIB_FLAG_WRITEBACK_CONTROLS"
    out = np.empty((1, N, 128, 1), np.float32)
    for e in (W.cartpole(N, T).make_engine(), _streaming_engine(monkeypatch, W.cartpole(N, 128), readback=False)):
        _refused(INVALID, "null argument", lambda: _raw("mppib_get_samples", e._h, None))
        _refused(STATE, no_controls, lambda: _raw("mppib_get_samples", e._h, out.ctypes.data_as(C.c_void_p)))
        _refused(STATE, tsallis, lambda: e.set_tsallis(0.5, 2.0))
        e.set_tsallis(0.0, 0.0)  # plain weights need no controls
        e.close()


@pytest.mark.parametrize("kind", ["flag", "rmppi", "stream_readback"])
def test_samples_kept_by_each_kind_of_engine(monkeypatch, kind):
    if kind == "flag":
        w = W.cartpole(N, T)
        e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    elif kind == "rmppi":
        w = W.double_integrator_tube(N, T)
        e = w.make_engine(flags=H.FLAG_RMPPI)
    else:
        w = W.cartpole(N, 128)
        e = _streaming_engine(monkeypatch, w, readback=True)  # test_samples_refused_without_write_back: not without it
    assert e.get_samples().shape == (w.D, N, w.T, w.dyn.CONTROL_DIM)  # before a solve: the buffer exists
    U, _ = e.solve(w.x0, w.U0)
    s = e.get_samples()
    assert s.shape == (w.D, N, w.T, w.dyn.CONTROL_DIM)
    assert np.isfinite(s).all() and np.any(s != 0)
    if kind == "stream_readback":
        e.set_tsallis(0.5, 2.0)
        U_t, _ = e.solve(w.x0, w.U0)
        assert np.isfinite(U_t).all()
    e.close()


# ---- the importance weights --------------------------------------------------------------------------------------------
def test_weights_match_a_fresh_engine():
    w = W.cartpole(N, T)
    e = w.make_engine()
    out = np.empty((1, N), np.float32)
    _refused(INVALID, "null argument", lambda: _raw("mppib_get_weights", e._h, None))
    _refused(STATE, "no solve has been run yet", lambda: _raw("mppib_get_weights", e._h, out.ctypes.data_as(C.c_void_p)))
    for solves in (1, 2):
        e.solve(w.x0, w.U0)
        got = [e.get_weights(), e.get_weights()]
        f = w.make_engine()
        for _ in range(solves):
            f.solve(w.x0, w.U0)
        want = f.get_weights()
        f.close()
        for g in got:
            assert np.array_equal(g, want), solves
        assert np.isfinite(want).all() and want.max() > 0
    e.close()


# ---- the L2 flush ------------------------------------------------------------------------------------------------------
def test_l2_flush_changes_no_result():
    w = W.cartpole(N, T)
    e = w.make_engine()
    f = w.make_engine()  # never flushes
    for nbytes in (1 << 20, 0, 16 << 20):
        e.set_option(H.OPT_L2_FLUSH_BYTES, nbytes)
        got = e.solve(w.x0, w.U0)
        want = f.solve(w.x0, w.U0)
        assert np.array_equal(got[0], want[0]), nbytes
        assert np.array_equal(np.array(got[1]), np.array(want[1])), nbytes
        assert np.array_equal(e.get_costs(), f.get_costs()), nbytes
    e.close()
    f.close()
