"""Two rules of the engine's state, each kept by one owner.

Stage timing counts a solve only if it was enqueued while timing was on: turning timing on while an untimed solve is in
flight neither reads events that solve never recorded (the failed query would be left behind as the thread's last CUDA
error and reported by the next solve) nor adds an earlier solve's stale sample.

RMPPI's feedback gains count as set only while the buffer holds a whole trajectory: a DDP solve whose LDLT fails leaves
them as they were, so the next rollout gives what it gave before the call, with the gains set earlier or with none."""
import numpy as np
import pytest

import mppi_generic_b200 as m
from mppi_generic_b200 import workloads as W

H = m.host
INVALID, STATE = -1, -9

pytestmark = pytest.mark.gpu


def _cartpole_engine():
    w = W.cartpole(1024, 32)
    return w.make_engine(), np.ascontiguousarray(w.x0, np.float32), np.ascontiguousarray(w.U0, np.float32)


def test_timing_turned_on_during_an_untimed_solve():
    e, x0, U = _cartpole_engine()
    e.solve_async(x0, U)
    e.enable_timing(True)
    e.solve_wait()
    with pytest.raises(H.MppibError) as ex:
        e.timing()
    assert ex.value.status == STATE
    e.solve(x0, U)
    assert e.timing()["samples"] == 1
    e.close()


def test_timing_turned_off_and_on_during_an_untimed_solve():
    e, x0, U = _cartpole_engine()
    e.enable_timing(True)
    e.solve(x0, U)
    assert e.timing()["samples"] == 1
    e.enable_timing(False)
    e.solve_async(x0, U)
    e.enable_timing(True)
    e.solve_wait()
    with pytest.raises(H.MppibError) as ex:
        e.timing()
    assert ex.value.status == STATE
    e.close()


T = 30
X0 = np.array([[2.0, 0.0, 0.0, 1.0], [2.05, 0.02, 0.0, 1.05]], np.float32)  # nominal, real


def _rmppi_engine(gains):
    w = W.double_integrator_tube(1024, T)
    e = w.make_engine(flags=H.FLAG_RMPPI)
    if gains is not None:
        e.set_rmppi(20.0, gains)
    return e


def _failed_ddp(e):
    """R = 0 and Q_f = 0: the last step's Q_uu = R dt + B' Vxx B is zero, and the LDLT refuses a zero pivot."""
    e.set_ddp(np.eye(4, dtype=np.float32), np.zeros((4, 4), np.float32), np.zeros((2, 2), np.float32))
    xt = np.tile(X0[0], (T, 1))
    ut = np.zeros((T, 2), np.float32)
    with pytest.raises(H.MppibError) as ex:
        e.ddp_feedback(X0[1], xt, ut, to_rmppi=True)
    assert ex.value.status == INVALID


def _rollout_costs(e):
    U = np.zeros((2, T, 2), np.float32)
    U[:, :, 0] = 0.3
    e.draw_noise()
    e.rollout_only(X0, U, 1, 0)
    return e.get_costs()


@pytest.mark.parametrize("with_gains", [True, False], ids=["gains_set", "no_gains"])
def test_failed_ddp_leaves_the_rmppi_gains_as_they_were(with_gains):
    G = None
    if with_gains:
        G = np.zeros((T, 4, 2), np.float32)  # [t][s][c]: u_c -= 2 (x_c - x_nom_c) on the positions
        G[:, 0, 0] = G[:, 1, 1] = -2.0
    plain, tried = _rmppi_engine(G), _rmppi_engine(G)
    _failed_ddp(tried)
    expected = _rollout_costs(plain)
    assert np.array_equal(_rollout_costs(tried), expected)
    if with_gains:  # the gains act on this rollout: without them the costs differ
        none = _rmppi_engine(None)
        assert not np.array_equal(_rollout_costs(none), expected)
        none.close()
    plain.close()
    tried.close()
