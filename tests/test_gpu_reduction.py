"""Timing mode (mppib_enable_timing) records an event between every stage of a solve, so K2 starts only after K1 has
finished instead of under it (programmatic dependent launch). The merge must compute the same thing either way: U, the
statistics and the per-sample costs of a timed solve are bit-identical to those of an untimed engine on the same seed, and
the stage averages describe the solves that were timed."""
import numpy as np
import pytest

from mppi_generic_b200 import workloads as W

pytestmark = pytest.mark.gpu

CASES = {
    "cartpole": lambda: W.cartpole(4096, 100),  # D = 1
    "double_integrator_tube": lambda: W.double_integrator_tube(4096, 100),  # D = 2
}
SOLVES = 3


@pytest.mark.parametrize("name", sorted(CASES))
def test_timed_solve_matches_untimed(name):
    w = CASES[name]()
    plain, timed = w.make_engine(), w.make_engine()
    timed.enable_timing(True)
    U_in = w.U0
    for _ in range(SOLVES):
        U_p, stats_p = plain.solve(w.x0, U_in)
        U_t, stats_t = timed.solve(w.x0, U_in)
        assert np.array_equal(U_t, U_p)
        assert np.array_equal(np.array(stats_t), np.array(stats_p))
        assert np.array_equal(timed.get_costs(), plain.get_costs())
        U_in = U_p
    t = timed.timing()
    assert t["samples"] == SOLVES
    stages = (t["noise_ms"], t["rollout_ms"], t["reduce_ms"])
    assert all(v > 0.0 for v in stages + (t["total_ms"],)), t
    assert all(v <= t["total_ms"] for v in stages), t
    plain.close()
    timed.close()
