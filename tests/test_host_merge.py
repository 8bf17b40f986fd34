"""The host twin of the softmin merge (mppib_host_merge_records, the CPU copy of K2 / KX's arithmetic) against a float64 softmin
of the samples the records summarise. A record is [beta, eta, sum w^2, pad, V[TC]] with V = sum_n w_n u_n against the record's
own baseline; a record whose every cost is +inf is empty, (+inf, 0, 0, 0, 0...). No GPU needed."""
import numpy as np
import pytest

import mppi_generic_b200 as m

U32 = 2.0 ** -24  # unit roundoff of float32


def _record(c: np.ndarray, u: np.ndarray, lam_inv: float) -> np.ndarray:
    """float64 record of samples c [n], u [n][TC] against their own minimum, rounded to float32 like a device record."""
    TC = u.shape[1]
    r = np.zeros(4 + TC)
    beta = c.min()
    if beta == np.inf:
        r[0] = np.inf  # empty: eta = sum w^2 = V = 0
        return r.astype(np.float32)
    w = np.where(c == np.inf, 0.0, np.exp(-lam_inv * (c - beta)))
    r[0], r[1], r[2] = beta, w.sum(), (w * w).sum()
    r[4:] = w @ u
    return r.astype(np.float32)


def _shards(rng, n_ranks, n, TC, spread, empty=()):
    costs = [rng.uniform(0.0, spread, n).astype(np.float32) for _ in range(n_ranks)]
    for k in empty:
        costs[k][:] = np.inf
    us = [rng.standard_normal((n, TC)).astype(np.float32) for _ in range(n_ranks)]
    return costs, us


def _float64_softmin(costs, us, lam_inv):
    c = np.concatenate(costs).astype(np.float64)
    u = np.concatenate(us).astype(np.float64)
    beta = c.min()
    w = np.where(c == np.inf, 0.0, np.exp(-lam_inv * (c - beta)))
    return beta, w, u


@pytest.mark.parametrize("n_ranks,empty", [(1, ()), (2, ()), (8, ()), (2, (1,)), (8, (0, 3, 7)), (3, (0,))])
@pytest.mark.parametrize("lam", [1.0, 1e-3, 1e3])
def test_host_merge_matches_float64_softmin(n_ranks, empty, lam):
    """Ordinary records, and records of ranks whose every sample costs +inf among finite ones: the merged U, baseline,
    normaliser and sum w^2 are the float64 softmin of all samples, the empty ranks weighing nothing."""
    rng = np.random.default_rng(100 + n_ranks + 7 * len(empty))
    n, TC = 64, 10
    lam_inv = float(np.float32(1.0 / lam))
    costs, us = _shards(rng, n_ranks, n, TC, spread=5.0 * lam, empty=empty)
    recs = np.stack([_record(c.astype(np.float64), u.astype(np.float64), lam_inv) for c, u in zip(costs, us)])[:, None, :]
    out = m.host.merge_records(recs, lam, normalize=True)
    beta, w, u = _float64_softmin(costs, us, lam_inv)
    eta = w.sum()
    U = (w @ u) / eta
    assert out[0, 0] == np.float32(beta)
    # error budget: each record field rounded to float (1 u); s_b = expf of a float product of a rounded difference
    # (3 a_b u + 2 ulp, a_b = lambda^-1 (beta_b - beta) <= 5); float fma accumulation over the records (n_ranks u)
    a_max = 5.0 + 1.0
    delta = (3.0 * a_max + 6.0) * U32
    assert abs(out[0, 1] - eta) <= (delta + 2 * U32) * eta
    assert abs(out[0, 2] - (w * w).sum()) <= (2 * delta + 2 * U32) * (w * w).sum()
    acc = (w @ np.abs(u)) / eta
    bound = 2.0 * delta * np.abs(u - U[None]).max(0) + (n_ranks + 4) * U32 * acc + U32 * np.abs(U)
    assert np.all(np.abs(out[0, 4:] - U) <= bound), (np.abs(out[0, 4:] - U) / bound).max()


def test_host_merge_of_empty_records_is_empty_and_normalised_nan():
    """Merging only empty records (every cost +inf on every rank): un-normalised, the result is again an empty record,
    so a later merge can still drop it; normalised, U = 0 / 0 = NaN, as the reference's one global baseline of +inf gives."""
    TC = 6
    empty = np.zeros((3, 1, 4 + TC), np.float32)
    empty[:, :, 0] = np.inf
    rec = m.host.merge_records(empty, 1.0, normalize=False)
    assert rec[0, 0] == np.inf
    assert np.all(rec[0, 1:] == 0.0)
    out = m.host.merge_records(empty, 1.0, normalize=True)
    assert out[0, 0] == np.inf and out[0, 1] == 0.0 and out[0, 2] == 0.0
    assert np.all(np.isnan(out[0, 4:]))


def test_host_merge_two_level_with_empty_rank_equals_flat_merge():
    """Blocks -> rank records -> world record, with one rank all +inf: the two-level merge (what K2 then KX do) gives the
    same result as merging every block record at once."""
    rng = np.random.default_rng(5)
    TC, lam = 8, 0.5
    lam_inv = float(np.float32(1.0 / lam))
    blocks = []
    for r in range(3):
        for b in range(4):
            c = rng.uniform(0.0, 3.0, 32)
            if r == 1:
                c[:] = np.inf
            blocks.append(_record(c, rng.standard_normal((32, TC)), lam_inv))
    blocks = np.stack(blocks)[:, None, :]
    ranks = np.stack([m.host.merge_records(blocks[4 * r:4 * r + 4], lam, normalize=False) for r in range(3)])
    assert ranks[1, 0, 0] == np.inf and np.all(ranks[1, 0, 1:] == 0.0)
    two = m.host.merge_records(ranks, lam, normalize=True)
    flat = m.host.merge_records(blocks, lam, normalize=True)
    assert np.all(np.isfinite(two))
    np.testing.assert_allclose(two, flat, rtol=1e-5, atol=1e-6)


def test_host_merge_keeps_nan_costs_nan():
    """A record that carries a NaN (a NaN cost) still makes the result NaN: only +inf costs are dropped."""
    TC = 4
    recs = np.zeros((2, 1, 4 + TC), np.float32)
    recs[0, 0, :4] = (0.0, 1.0, 1.0, 0.0)
    recs[0, 0, 4:] = 1.0
    recs[1, 0, :4] = (0.5, np.nan, np.nan, 0.0)
    recs[1, 0, 4:] = np.nan
    out = m.host.merge_records(recs, 1.0, normalize=True)
    assert np.isnan(out[0, 1]) and np.all(np.isnan(out[0, 4:]))
