"""The host twins (host_twins.h) against the snapshot in tests/golden/host_twins/snapshot.npz, bit for bit, and each
model's roll-forward against T - 1 calls of its own exported step. CPU only."""
import ctypes as C
import os

import numpy as np
import pytest

from mppi_generic_b200 import host as H
from tests.golden import make_host_twin_snapshot as snap

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "host_twins", "snapshot.npz")


@pytest.fixture(scope="module")
def stored():
    return dict(np.load(FIXTURE))


@pytest.fixture(scope="module")
def current():
    return snap.snapshot(H.lib())


def _network_clone_differs(stored) -> bool:
    """The FNN and LSTM heads run an AVX2 + FMA clone on an x86-64-v3 CPU and a baseline one elsewhere: when this CPU picks
    another clone than the one the snapshot was made with, those models may differ by rounding."""
    return bool(stored["meta.x86_64_v3"][0]) != snap.cpu_runs_v3_clones()


def test_snapshot_covers_every_model(stored, current):
    assert {m.dyn_id for m in snap.models()} == set(range(8))
    assert set(current) == set(stored) - {"meta.x86_64_v3"}


@pytest.mark.parametrize("model", [m.name for m in snap.models()] + ["generic"])
def test_host_twins_match_snapshot(stored, current, model):
    clones = {m.name for m in snap.models() if m.uses_clones} | {"generic"}  # the generic entries step Autorally too
    keys = sorted(k for k in stored if k.split(".")[0] == model)
    assert keys, model
    for k in keys:
        want, got = stored[k], current[k]
        assert got.dtype == want.dtype and got.shape == want.shape, k
        if got.dtype == np.int32:
            np.testing.assert_array_equal(got, want, err_msg=k)
        elif model in clones and _network_clone_differs(stored):
            np.testing.assert_allclose(got, want, rtol=1e-6, equal_nan=True, err_msg=k)
        else:
            bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
            assert bad.size == 0, f"{k}: {bad.size} values differ, first at {bad[0]}: {got[bad[0]]!r} != {want[bad[0]]!r}"


@pytest.mark.parametrize("model", snap.models(), ids=lambda m: m.name)
def test_roll_is_its_own_step_repeated(model):
    """outputs[0] is x0 on the first min(S, O) entries and 0 after; then each step enforces u_t and calls the model's own
    exported step; an LSTM starts from the initial state stored in its weight blob."""
    L, m = H.lib(), model
    rc, states, outputs = snap.trajectory(L, m)
    assert rc == 0
    y0 = np.zeros(m.O, np.float32)
    y0[:min(m.S, m.O)] = m.x[0][:min(m.S, m.O)]
    assert states[0].tobytes() == m.x[0].tobytes()
    assert outputs[0].tobytes() == y0.tobytes()
    h, c = m.initial_hidden_cell() if m.lstm is not None else (None, None)
    x, y = m.x[0].copy(), y0
    for t in range(snap.T - 1):
        u = m.U[t].copy()
        assert L.mppib_host_enforce_constraints(m.dyn_id, C.addressof(m.params), u.ctypes.data) == 0
        # one output buffer for the whole roll: what a step leaves alone (Autorally's eighth output) keeps its value
        rc, xn, xd, y = snap.step(L, m, x, u, h, c, y=y)
        assert rc == 0
        assert states[t + 1].tobytes() == xn.tobytes(), t
        assert outputs[t + 1].tobytes() == y.tobytes(), t
        x = xn
