"""DoubleIntegratorRobustCost and ARRobustCost (cost_functions/double_integrator/double_integrator_robust_cost.cu,
cost_functions/autorally/ar_robust_cost.cu): the C ABI, the host twins against the reference's known answers, the device
bodies against the float32 restatement in tests/robust_cost_oracle.py in every K1 form that runs them, and the reference's
RMPPITest.RobustMPPILargeVarianceRobustCost closed loop."""
import ctypes as C
import math
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import mppi_generic_b200 as m
import oracle
from mppi_generic_b200 import workloads as W
from tests import robust_cost_oracle as RO

H = m.host
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- C ABI ---------------------------------------------------------------------------------------------------------
def test_cost_ids_and_robust_blob_layout():
    assert (H.COST_DI_ROBUST, H.COST_AR_ROBUST) == (5, 6)
    std, rob = H.ARStandardCostParams, H.ARRobustCostParams
    for name, _ in std._fields_:
        assert getattr(rob, name).offset == getattr(std, name).offset, name
    assert rob.heading_coeff.offset == C.sizeof(std) and C.sizeof(rob) == C.sizeof(std) + 4


def test_reference_defaults():
    p = H.ARRobustCost().params  # ar_robust_cost.cuh:11-28
    assert (p.desired_speed, p.max_slip_ang, p.track_coeff, p.slip_coeff, p.speed_coeff) == (-1.0, 1.5, 33.0, 0.0, 20.0)
    assert (p.crash_coeff, p.boundary_threshold, p.track_slop, p.heading_coeff) == (125000.0, 0.75, 0.0, 0.0)
    assert (p.front_d, p.back_d, p.discount) == (0.5, -0.5, 1.0)
    d = H.DoubleIntegratorRobustCost().params  # DoubleIntegratorCircleCostParams
    assert (d.crash_cost, d.velocity_desired, d.velocity_cost) == (1000.0, 2.0, 1.0)


@pytest.mark.parametrize("dyn,cost", [(H.DYN_DOUBLE_INTEGRATOR, H.COST_DI_ROBUST), (H.DYN_AUTORALLY_NN, H.COST_AR_ROBUST)])
@pytest.mark.parametrize("D,flags", [(1, 0), (2, 0), (2, H.FLAG_RMPPI)])
def test_create_reaches_the_device_check(dyn, cost, D, flags):
    """A registered pair: without a GPU mppib_create stops at NO_DEVICE (-5), not at INVALID_ARG / UNSUPPORTED."""
    L = H.lib()
    h = C.c_void_p()
    d = H.Desc(dyn, cost, 0, 256, 20, D, 0, flags, None, 0, 1)
    rc = L.mppib_create(C.byref(h), C.byref(d))
    if rc == 0:
        L.mppib_destroy(h)
    else:
        assert rc == -5, (rc, L.mppib_last_error())


def test_tensor_core_kernel_refuses_the_robust_cost():
    """MPPIB_FLAG_NN_TENSOR is built for ARStandardCost only: ARRobustCost is refused before any device work, never run on
    another kernel."""
    L = H.lib()
    h = C.c_void_p()
    d = H.Desc(H.DYN_AUTORALLY_NN, H.COST_AR_ROBUST, 0, 256, 20, 1, 0, H.FLAG_NN_TENSOR, None, 0, 1)
    assert L.mppib_create(C.byref(h), C.byref(d)) == -2
    assert b"ARRobustCost" in L.mppib_last_error()


def test_host_state_cost_is_only_for_the_robust_costs():
    L = H.lib()
    out = C.c_float()
    p = H.CartpoleQuadraticCost().params
    y = np.zeros(4, np.float32)
    assert L.mppib_host_state_cost(H.COST_CARTPOLE_QUADRATIC, C.byref(p), None, H._ptr(y), 0, None, C.byref(out)) == -2
    rp = H.ARRobustCost().params
    assert L.mppib_host_state_cost(H.COST_AR_ROBUST, C.byref(rp), None, H._ptr(np.zeros(8, np.float32)), 0, None,
                                   C.byref(out)) == -1  # no map


# ---- host twins and the float32 restatement: reference known answers ---------------------------------------------
def test_ar_robust_stabilizing_cost_known_answers():
    """autorally_robust_cost_test.cu:119-153."""
    cost = H.ARRobustCost()
    p = cost.params
    p.max_slip_ang, p.crash_coeff, p.slip_coeff = 1.25, 10000.0, 10.0
    s = np.zeros(7, np.float32)
    s[4], s[5] = 0.24, 0.0
    cases = [((0.24, 0.0, 0.0), 0.0), ((1.0, 1.0, 0.0), 0.785398 * 10), ((1.0, 10.0, 0.0), 1.4711 * 10 + 1e4),
             ((1.0, 10.0, 1.5), 1.4711 * 10 + 1e4)]
    for (vx, vy, roll), want in cases:
        s[3], s[4], s[5] = roll, vx, vy
        assert cost.getStabilizingCost(s) == pytest.approx(want, rel=4e-6, abs=1e-6)
        assert float(RO.ar_stabilizing_cost(p, s)) == pytest.approx(want, rel=4e-6, abs=1e-6)
    s[3] = 1.6  # past pi/2: the roll penalty replaces the slip penalty
    assert cost.getStabilizingCost(s) == pytest.approx(1.4711 * 10 + 1e4, rel=4e-6)
    s[3], s[4] = 0.0, 0.0005  # |vx| < 0.001: no slip
    assert cost.getStabilizingCost(s) == 0.0


# normalised distance from the centre line r = 2 of the default track (half-width 0.125), with the velocity terms off:
# (radius, device value (steep boundary 0.5, steep cost 500), host value (0.75, 100)) for crash_cost 1000
DI_REGIONS = [
    (2.0, 0.0, 0.0),                  # centre
    (2.05, 400.0, 0.4 / 0.75 * 100),  # shallow band on both sides (norm 0.4)
    (2.1, 800.0, 280.0),              # norm 0.8: device steep band; host steep band starts at 0.75
    (1.9375, 500.0, 0.5 / 0.75 * 100),  # inner side, norm 0.5: the device's band edge (shallow branch, = steep cost)
    (2.2, 1000.0, 1000.0),            # beyond the outer radius
    (1.7, 1000.0, 1000.0),            # inside the inner radius
]


@pytest.mark.parametrize("r,dev,host", DI_REGIONS)
def test_di_robust_cost_regions_host_and_device_constants(r, dev, host):
    cost = H.DoubleIntegratorRobustCost()
    cost.params.velocity_cost = 0.0
    y = np.array([r, 0.0, 0.0, 0.0], np.float32)
    assert cost.computeStateCost(y) == pytest.approx(host, rel=2e-5, abs=2e-4)
    assert float(RO.di_robust_cost(cost.params, y, device=False)) == pytest.approx(host, rel=2e-5, abs=2e-4)
    assert float(RO.di_robust_cost(cost.params, y, device=True)) == pytest.approx(dev, rel=2e-5, abs=2e-4)


def test_di_robust_velocity_and_angular_momentum_terms():
    cost = H.DoubleIntegratorRobustCost()
    y = np.array([2.0, 0.0, 0.0, 3.0], np.float32)  # centre; speed 3 (desired 2), momentum 6 (desired 4): 1 + 4
    assert cost.computeStateCost(y) == pytest.approx(5.0, rel=1e-6)
    assert float(RO.di_robust_cost(cost.params, y)) == pytest.approx(5.0, rel=1e-6)
    y = np.array([0.0, 2.05, -1.0, 0.0], np.float32)  # norm 0.4; speed 1, momentum 2.05
    want_vel = 1.0 + (2.05 - 4.0) ** 2
    assert cost.computeStateCost(y) == pytest.approx(0.4 / 0.75 * 100 + want_vel, rel=2e-5)
    assert float(RO.di_robust_cost(cost.params, y)) == pytest.approx(400.0 + want_vel, rel=2e-5)


def _ar_robust_f64(p, tex, y):
    """Float64 restatement of the costmap and stabilizing costs (point-sampled texel, accurate sin / cos)."""
    y = np.asarray(y, np.float64)
    cs, sn = np.cos(y[:, 2]), np.sin(y[:, 2])

    def lookup(x, yy):
        u, v = RO.texel_coords(p, x, yy)
        cx = np.clip(np.floor(u), 0, p.map_width - 1).astype(int)
        cy = np.clip(np.floor(v), 0, p.map_height - 1).astype(int)
        return tex[cy, cx].astype(np.float64)

    f, b = lookup(y[:, 0] + p.front_d * cs, y[:, 1] + p.front_d * sn), lookup(y[:, 0] + p.back_d * cs, y[:, 1] + p.back_d * sn)
    cv = np.minimum(1.0, np.maximum(f[:, 0], b[:, 0]))
    cost = np.where(cv >= p.boundary_threshold, (cv - p.boundary_threshold) / (1 - p.boundary_threshold) * p.crash_coeff, 0)
    cost += np.where(f[:, 1] > p.track_slop, p.track_coeff * f[:, 1], 0)
    cost += p.speed_coeff * np.abs(y[:, 4] - (f[:, 2] if p.desired_speed == -1 else p.desired_speed))
    cost += p.heading_coeff * np.abs(np.sin(y[:, 2]) + f[:, 3])
    slip = np.where(np.abs(y[:, 4]) < 0.001, 0.0, np.abs(np.arctan(y[:, 5] / np.abs(y[:, 4]))))
    pen = np.where(slip >= 0.75 * p.max_slip_ang, (np.minimum(1, slip / p.max_slip_ang) - 0.75) / 0.25 * p.crash_coeff, 0)
    pen = np.where(np.abs(y[:, 3]) >= math.pi / 2, p.crash_coeff, pen)
    return cost + p.slip_coeff * slip + pen


@pytest.mark.parametrize("desired_speed", [10.0, -1.0])
def test_ar_robust_device_form_against_float64(desired_speed):
    w = W.autorally_robust(64, 10)
    p, tex = w.cost.params, w.cost.costmap
    p.desired_speed, p.slip_coeff, p.track_slop = desired_speed, 10.0, 0.5
    rng = np.random.RandomState(5)
    y = np.zeros((4000, 8), np.float32)
    y[:, 0] = rng.uniform(-24, 44, 4000)
    y[:, 1] = rng.uniform(-49, 4, 4000)
    y[:, 2] = rng.uniform(-math.pi, math.pi, 4000)
    y[:, 3] = rng.uniform(-2, 2, 4000)
    y[:, 4] = rng.uniform(-5, 5, 4000)
    y[:, 5] = rng.uniform(-5, 5, 4000)
    keep = ~RO.ar_on_discontinuity(p, y, texel_tol=1e-3) & ~RO.ar_track_slop_crossing(p, tex, y)
    assert keep.mean() > 0.9
    got = RO.ar_robust_cost(p, tex, y[keep])
    want = _ar_robust_f64(p, tex, y[keep])
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-3)
    # the host twin (nearest texel by std::round of the half-texel-shifted coordinate: the same texel away from edges)
    for k in np.nonzero(keep)[0][:200]:
        assert w.cost.computeStateCost(y[k]) == pytest.approx(float(_ar_robust_f64(p, tex, y[k:k + 1])[0]), rel=1e-5,
                                                               abs=1e-3)


def test_track_map_robust_matches_the_fixture_recipe():
    """generateTestMaps.py:76-109, element by element on a sample of the script's (i, j) loop."""
    tex, xb, yb, ppm = W.track_map_robust()
    assert tex.shape == (1100, 1400, 4) and (xb, yb, ppm) == ((-25.0, 45.0), (-50.0, 5.0), 20.0)
    flat = tex.reshape(-1, 4)
    for i, j in [(0, 0), (1, 1099), (700, 300), (1399, 1099), (1285, 1060), (400, 500), (20, 801)]:
        x, y = j / 20.0, i / 20.0
        c0 = 1.0 if (x > 50 or x < 15) else (0.6 if (x > 40 or x < 25) else 0.0)
        want = np.array([c0, abs(55 / 2.0 - y) + x / 70, x, math.atan2(y, x)], np.float32)
        np.testing.assert_array_equal(flat[i * 1100 + j], want)


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _held_state_cost(w, x0, flags=0):
    """The device cost of one state: a zero network (or the double integrator) and dt -> 0 hold the state, T = 1."""
    w.x0[0] = x0
    w.dt = 1e-12
    e = w.make_engine(flags=flags)
    e.set_noise(np.zeros((w.N, w.T, w.dyn.CONTROL_DIM), np.float32))
    e.rollout_only(w.x0, w.U0)
    c = e.get_costs()[0]
    e.close()
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [0, H.FLAG_NO_WARP_SPEC, H.FLAG_NN_FFMA2], ids=["warp_spec", "generic", "ffma2"])
def test_ar_robust_costmap_known_answers_on_device(flags):
    """autorally_robust_cost_test.cu:179-233 on track_map_robust: 11349.729, and 11629.229 with desired_speed = -1. The
    fixture's slip_coeff is 0 and the state's slip angle under the penalty threshold, so the state cost is the costmap
    cost."""
    x0 = [3.0, 0.0, math.pi / 2, 0.0, 2.0, 1.0, 0.0]  # yaw rate 0 so that the state does not move
    for desired_speed, want in ((10.0, 11349.729), (-1.0, 11629.229)):
        w = W.autorally_robust(32, 1)
        w.dyn.updateModel([6, 32, 32, 4], np.zeros(1412, np.float32))
        p = w.cost.params
        p.boundary_threshold, p.crash_coeff, p.track_slop = 0.0, 10000.0, 0.0
        p.desired_speed, p.speed_coeff, p.heading_coeff = desired_speed, 10.0, 20.0
        c = _held_state_cost(w, x0, flags)
        assert np.all(c == c[0])
        assert float(c[0]) == pytest.approx(want, rel=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("r,dev,host", DI_REGIONS)
def test_di_robust_cost_device_constants_on_device(r, dev, host):
    w = W.double_integrator_vanilla(32, 1)
    w.cost = H.DoubleIntegratorRobustCost()
    w.cost.params.velocity_cost = 0.0
    c = _held_state_cost(w, [r, 0.0, 0.0, 0.0])
    assert float(c[0]) == pytest.approx(dev, rel=2e-5, abs=2e-4)


@pytest.mark.gpu
def test_costmap_blob_only_for_map_costs():
    w = W.autorally_robust(256, 10)
    e = w.make_engine()  # uploads the costmap: accepted
    e.close()
    d = W.double_integrator_vanilla(256, 10)
    d.cost = H.DoubleIntegratorRobustCost()
    e = d.make_engine()
    m_ = np.zeros((2, 2, 4), np.float32)
    assert H.lib().mppib_set_blob(e._h, H.BLOB_COSTMAP, H._ptr(m_), m_.nbytes) == -1
    e.close()


def _ar_oracle_costs(w, samples, idx, x0=None):
    """Per-sample trajectory costs of rollouts `idx` from state x0 (default w.x0[0]): the oracle's CPU rollout of the
    device's constrained controls (states only; ARStandardCost's prefix of the blob) and the robust cost restated on its
    outputs."""
    x0 = w.x0[0] if x0 is None else x0
    std = H.ARStandardCostParams.from_buffer_copy(bytes(w.cost.params)[:C.sizeof(H.ARStandardCostParams)])
    out = np.empty(len(idx), np.float32)
    outs = []
    for k, n in enumerate(idx):
        o_ref, _, _ = oracle.sampled_trajectory(w.dyn.DYN_ID, H.COST_AR_STANDARD, w.dyn.params, std, w.sampler.params,
                                                w.dyn.nn_theta, w.cost.costmap, len(samples), w.T, 0, int(n), False, w.dt,
                                                w.lambda_, w.alpha, x0, w.U0[0], samples[n])
        run = np.float32(0)
        for c in RO.ar_robust_cost(w.cost.params, w.cost.costmap, o_ref):
            run = np.float32(run + c)
        out[k] = run / np.float32(w.T)
        outs.append(o_ref)
    return out, outs


def _ar_parity_proof(w, c, samples, x0, dump, idx=None, tol=1e-4):
    """Device per-sample costs c[idx] of the rollouts of `samples` from x0 within `tol` relative of the restatement, or a
    proven discontinuity: for each sample outside, the device's own dump of the rollout (dump(indices) -> (outputs [n][T][O],
    costs [n][T + 1])) sums to its cost and follows the oracle's states, every step whose cost differs sits on a
    discontinuity, and so does the step where the oracle's own trajectory first departs from the device's."""
    idx = np.arange(len(c)) if idx is None else idx
    ref, outs = _ar_oracle_costs(w, samples, idx, x0)
    rel = np.abs(c[idx] - ref) / np.maximum(np.abs(ref), 1.0)
    bad = np.nonzero(rel > tol)[0]
    assert bad.size <= 0.03 * idx.size, (bad.size, idx.size, float(rel.max()))
    assert np.median(rel) < 1e-5
    if bad.size:
        outs_dev, costs_dev = dump(idx[bad])
        np.testing.assert_allclose(costs_dev.sum(axis=1), c[idx[bad]], rtol=5e-6)
        for k, b in enumerate(bad):
            o_dev = outs_dev[k]
            assert np.abs(o_dev[:, :7] - outs[b][:, :7]).max() < 2e-3
            step = RO.ar_robust_cost(w.cost.params, w.cost.costmap, o_dev)
            dev = costs_dev[k][:w.T] * w.T
            off = np.abs(step - dev) > 1e-5 * np.maximum(1.0, np.abs(step))
            jumps = RO.ar_on_discontinuity(w.cost.params, o_dev) | RO.ar_on_discontinuity(w.cost.params, outs[b]) | \
                RO.ar_track_slop_crossing(w.cost.params, w.cost.costmap, o_dev)
            assert np.all(jumps[off]), f"sample {idx[b]}: steps {np.nonzero(off & ~jumps)[0]} differ off any discontinuity"
            ref_steps = RO.ar_robust_cost(w.cost.params, w.cost.costmap, outs[b])
            parted = np.nonzero(np.abs(ref_steps - dev) > 1e-3 * np.maximum(1.0, np.abs(ref_steps)))[0]
            assert parted.size == 0 or jumps[parted[0]], f"sample {idx[b]}: first departure off any discontinuity"
    return bad.size


def _check_ar_parity(w, e, max_check=None, tol=1e-4):
    """One solve of a single-system engine, its costs proven against the restatement (_ar_parity_proof)."""
    U, stats = e.solve(w.x0, w.U0)
    c = e.get_costs()[0]
    samples = e.get_samples()[0]
    idx = None if max_check is None else np.random.RandomState(0).choice(w.N, max_check, replace=False)
    _ar_parity_proof(w, c, samples, w.x0[0], lambda ix: e.sample_trajectories(w.x0[0], w.U0[0], ix)[:2], idx, tol)
    return U, stats, c


def _one_thread_per_sample(e, N):
    """launch_info of the generic K1 (one thread per sample), not the warp-specialised form (3 or 5 warps per 32 samples)."""
    info = e.launch_info()
    return info["grid"] == (N + info["block"] - 1) // info["block"]


@pytest.mark.gpu
@pytest.mark.parametrize("stream", [0, 1])
@pytest.mark.parametrize("pspw", [8, 16, 32])
@pytest.mark.parametrize("N,T", [(1000, 100), (64 * 5 + 7, 37)])
def test_ar_robust_warp_specialised_matches_oracle(N, T, pspw, stream, monkeypatch):
    monkeypatch.setenv("MPPIB_BX", "64")
    monkeypatch.setenv("MPPIB_WS_PSPW", str(pspw))
    monkeypatch.setenv("MPPIB_STREAM", str(stream))
    w = W.autorally_robust(N, T)
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    info = e.launch_info()
    assert info["block"] == (32 // pspw + 1) * 64 and info["grid"] == (N + 63) // 64
    nchunks = (2 * T + 31) // 32
    ring = 3 if stream else nchunks
    assert info["smem_bytes"] >= ring * 64 * 128
    if stream and nchunks > 3:
        r = W.autorally_robust(N, T)
        monkeypatch.setenv("MPPIB_STREAM", "0")
        res = r.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
        assert res.launch_info()["smem_bytes"] - info["smem_bytes"] == (nchunks - 3) * 64 * 128
        res.close()
    _check_ar_parity(w, e)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [H.FLAG_NO_WARP_SPEC, H.FLAG_NN_FFMA2], ids=["generic", "ffma2"])
def test_ar_robust_generic_kernels_match_oracle(flags):
    w = W.autorally_robust(1000, 37)
    e = w.make_engine(flags=flags | H.FLAG_WRITEBACK_CONTROLS)
    info = e.launch_info()
    assert info["grid"] == (1000 + info["block"] - 1) // info["block"]  # one thread per sample: not the warp-specialised form
    _check_ar_parity(w, e)
    e.close()


@pytest.mark.gpu
def test_ar_robust_warp_specialised_equals_generic():
    w = W.autorally_robust(4096, 100)
    a = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    b = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS | H.FLAG_NO_WARP_SPEC)
    assert a.launch_info()["block"] != b.launch_info()["block"]
    Ua, sa = a.solve(w.x0, w.U0)
    Ub, sb = b.solve(w.x0, w.U0)
    np.testing.assert_array_equal(a.get_noise(), b.get_noise())
    np.testing.assert_array_equal(a.get_samples(), b.get_samples())
    ca, cb = a.get_costs(), b.get_costs()
    rel = np.abs(ca - cb) / np.maximum(np.abs(cb), 1.0)
    assert rel.max() < 1e-6 and np.mean(ca != cb) < 0.01, (rel.max(), np.mean(ca != cb))
    np.testing.assert_allclose(Ua, Ub, rtol=0, atol=1e-6)
    np.testing.assert_allclose(np.asarray(sa), np.asarray(sb), rtol=1e-6)
    a.close()
    b.close()


@pytest.mark.gpu
def test_ar_robust_c4_in_one_wave_matches_oracle():
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    w = W.autorally_robust(32768, 100)
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    info = e.launch_info()
    block_rows = info["block"] // 3
    assert info["grid"] == (w.N + block_rows - 1) // block_rows and info["grid"] <= sms, (info, sms)
    _check_ar_parity(w, e, max_check=2048)
    e.close()


@pytest.mark.gpu
def test_ar_robust_tube_matches_oracle():
    """Tube-MPPI (two systems) with ARRobustCost on the generic K1: each system's costs within 1e-4 of the restatement or
    proven discontinuities, dumped per system (mppib_sample_trajectories, `distribution`)."""
    w = W.autorally_robust(1024, 40)
    w.D = 2
    w.x0 = np.stack([w.x0[0], w.x0[0] + np.array([0.1, 0.05, 0.02, 0, 0.1, 0, 0], np.float32)])
    w.U0 = np.zeros((2, w.T, 2), np.float32)
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    assert _one_thread_per_sample(e, w.N)
    e.solve(w.x0, w.U0)
    c, samples = e.get_costs(), e.get_samples()
    for d in range(2):
        _ar_parity_proof(w, c[d], samples[d], w.x0[d],
                         lambda ix, d=d: e.sample_trajectories(w.x0[d], w.U0[d], ix, distribution=d)[:2])
    e.close()


def _reroll(w, x0, controls):
    """A single-system generic-K1 engine that rolls out exactly `controls` [N][T][C] from x0: noise = the controls, sampler
    sigma 1, mean 0, no optimisation stride, so that u = fmaf(1, eps, 0) = eps. Rollout 0 is the sampler's zero-noise
    rollout, so the controls go to rollouts 1 .. N. Returns (engine, costs [N], dump(indices))."""
    N = controls.shape[0]
    sampler = H.GaussianDistribution(2, [1.0, 1.0])
    e = H.Engine(w.dyn, w.cost, sampler, N + 1, w.T, 1, flags=H.FLAG_WRITEBACK_CONTROLS | H.FLAG_NO_WARP_SPEC)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    assert _one_thread_per_sample(e, N + 1)
    eps = np.concatenate([np.zeros((1, w.T, 2), np.float32), controls]).astype(np.float32)
    e.set_noise(eps)
    zeros = np.zeros((1, w.T, 2), np.float32)
    e.rollout_only(x0[None], zeros, 0, 0)
    np.testing.assert_array_equal(e.get_samples()[0][1:], controls)
    return e, e.get_costs()[0][1:], lambda ix: e.sample_trajectories(x0, zeros[0], np.asarray(ix) + 1)[:2]


@pytest.mark.gpu
@pytest.mark.parametrize("with_gains", [False, True])
def test_ar_robust_rmppi_rollout_matches_oracle(with_gains):
    """RMPPI K1 (rmppi_kernels.cu:665-866) with ARRobustCost, no likelihood-ratio or feedback cost (the sampler's
    control_cost_coeff is 0). The engine writes back each system's applied controls:
      - the nominal system's are the constrained sampled controls; the real system's add K_t (x_real - x_nom) before the
        constraints, checked on the oracle's states of both systems;
      - a single-system re-roll of each system's applied controls (_reroll) gives the same per-sample costs as the RMPPI
        kernel's real cost, and its costs are proven against the restatement with the per-step dumps of _ar_parity_proof;
      - the nominal cost is 0.5 c_nom + 0.5 max(min(c_real, threshold), c_nom)."""
    w = W.autorally_robust(512, 40)
    thr = 2000.0
    e = H.Engine(w.dyn, w.cost, w.sampler, w.N, w.T, 2, flags=H.FLAG_RMPPI)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    e.seed(w.seed, 0)
    assert _one_thread_per_sample(e, w.N)
    gains = (np.random.RandomState(3).randn(w.T, 7, 2) * 0.05).astype(np.float32) if with_gains else None
    e.set_rmppi(thr, gains)
    x0 = np.stack([w.x0[0], w.x0[0] + np.array([0.05, 0.02, 0.01, 0, 0.1, 0, 0], np.float32)])
    U_in = np.zeros((2, w.T, 2), np.float32)
    e.draw_noise()
    e.rollout_only(x0, U_in, 1, 0)
    c, applied = e.get_costs(), e.get_samples()
    sampled = np.stack([e.get_noise(), e.get_noise()]).copy()
    oracle.set_gaussian_controls(U_in, w.sampler.params, sampled, 2, w.T, w.N, 2, 1, 0)
    lim = w.dyn.params.lim
    lo, hi = np.array(lim.rng_lo[:2], np.float64), np.array(lim.rng_hi[:2], np.float64)
    np.testing.assert_allclose(applied[0], np.clip(sampled[0], lo, hi), rtol=0, atol=1e-6)
    std = H.ARStandardCostParams.from_buffer_copy(bytes(w.cost.params)[:C.sizeof(H.ARStandardCostParams)])
    fb = np.zeros((w.N, w.T, 2))
    if with_gains:
        for n in range(w.N):
            traj = []
            for d in range(2):
                o, _, _ = oracle.sampled_trajectory(w.dyn.DYN_ID, H.COST_AR_STANDARD, w.dyn.params, std, w.sampler.params,
                                                    w.dyn.nn_theta, w.cost.costmap, w.N, w.T, 0, n, False, w.dt, w.lambda_,
                                                    w.alpha, x0[d], U_in[d], applied[d][n])
                traj.append(np.concatenate([x0[d][None], o[:-1, :7]]).astype(np.float64))  # state before step t
            fb[n] = np.einsum("tsc,ts->tc", gains.astype(np.float64), traj[1] - traj[0])
        assert np.abs(fb).max() > 1e-3  # the feedback acts on the real system
    np.testing.assert_allclose(applied[1], np.clip(sampled[1] + fb, lo, hi), rtol=0, atol=1e-4)
    costs = []
    for d in range(2):
        r, v, dump = _reroll(w, x0[d], applied[d])
        _ar_parity_proof(w, v, applied[d], x0[d], dump)
        costs.append(v)
        r.close()
    c_nom, c_real = costs
    np.testing.assert_allclose(c[1], c_real, rtol=1e-6, atol=0)
    nom = (np.float32(0.5) * c_nom + np.float32(0.5) * np.maximum(np.minimum(c[1], np.float32(thr)), c_nom)).astype(np.float32)
    np.testing.assert_allclose(c[0], nom, rtol=1e-6, atol=0)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 2])
def test_di_robust_rollout_matches_oracle(D):
    w = W.double_integrator_robust_tube(4096, 100) if D == 2 else W.double_integrator_vanilla(4096, 100)
    if D == 1:
        w.cost = H.DoubleIntegratorRobustCost()
    w.x0 = w.x0 + np.array([[0.02, 0.01, 0.0, 0.1]], np.float32)[:, :] * np.arange(1, D + 1)[:, None]
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    U, stats = e.solve(w.x0, w.U0)
    c, samples = e.get_costs(), e.get_samples()
    for d in range(D):
        ref = RO.di_rollout(w.cost.params, w.x0[d], samples[d], w.dt)
        np.testing.assert_allclose(c[d], ref, rtol=1e-4, atol=1e-5)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("with_gains", [False, True])
def test_di_robust_rmppi_rollout_matches_oracle(with_gains):
    w = W.double_integrator_robust_tube(2048, 50)
    e = w.make_engine(flags=H.FLAG_RMPPI)
    rng = np.random.RandomState(1)
    gains = (rng.randn(w.T, 4, 2) * 2.0).astype(np.float32) if with_gains else None
    e.set_rmppi(10.0, gains)
    x0 = np.array([[2.0, 0.0, 0.0, 1.0], [2.05, 0.03, 0.1, 0.9]], np.float32)
    U_in = (rng.randn(2, w.T, 2) * 0.3).astype(np.float32)
    e.draw_noise()
    e.rollout_only(x0, U_in, 1, 0)
    eps = e.get_noise()
    samples = np.stack([eps, eps]).copy()
    oracle.set_gaussian_controls(U_in, w.sampler.params, samples, 2, w.T, w.N, 2, 1, 0)
    ref = RO.di_rmppi_rollout(w.cost.params, x0, samples, gains, w.dt, 10.0)
    np.testing.assert_allclose(e.get_costs(), ref, rtol=1e-4, atol=1e-5)
    # init-eval (initEvalKernel, rmppi_kernels.cu:230-356): candidate k's samples take the sampled controls of distribution 0
    # from step min(t + stride_k, T - 1), on the noise the call draws
    K, spc, stride = 3, 64, 2
    cand = np.stack([x0[0], 0.5 * (x0[0] + x0[1]), x0[1]]).astype(np.float32)
    strides = np.array([0, 1, 2], np.int32)
    got = e.init_eval(cand, strides, spc, U_in[0], stride)
    ctl = e.get_noise()[None].copy()
    oracle.set_gaussian_controls(U_in[:1], w.sampler.params, ctl, 2, w.T, w.N, 1, stride, 0)
    ctl = ctl[0, :spc]
    for k in range(K):
        idx = np.minimum(np.arange(w.T) + strides[k], w.T - 1)
        want = RO.di_rollout(w.cost.params, cand[k], ctl[:, idx], w.dt)
        np.testing.assert_allclose(got[k * spc:(k + 1) * spc], want, rtol=1e-4, atol=1e-5)
    e.close()


def _tube_failure(x):
    r2 = float(x[0]) ** 2 + float(x[1]) ** 2
    return r2 < 1.675 ** 2 or r2 > 2.325 ** 2


@pytest.mark.gpu
def test_rmppi_large_variance_robust_cost_stays_in_the_tube():
    """RMPPITest.RobustMPPILargeVarianceRobustCost (tests/controllers/rmppi_test.cu:714-900): system_noise 100, robust cost
    with crash_cost 100, sigma 1, 3 iterations, lambda 2, alpha 0, T 50, N 1024, value-function threshold 10, DDP with
    Q = diag(500, 500, 100, 100), Q_f = I, R = I, x0 = (2, 0, 0, 1), 5000 steps: never outside r in [1.675, 2.325]."""
    dyn = H.DoubleIntegratorDynamics(100.0)
    cost = H.DoubleIntegratorRobustCost()
    cost.params.velocity_desired, cost.params.crash_cost = 2.0, 100.0
    sampler = H.GaussianDistribution(2, [1.0, 1.0])
    dt, T, N = 0.02, 50, 1024
    ctrl = H.RobustMPPIController(dyn, cost, None, sampler, dt, 3, 2.0, 0.0, 10.0, T, N, seed=11)
    p = H.DDPParams(4, 2)
    p.Q = np.diag([500, 500, 100, 100]).astype(np.float32)
    p.Q_f = np.eye(4, dtype=np.float32)
    p.R = np.eye(2, dtype=np.float32)
    ctrl.setFeedbackParams(p)
    ctrl.initFeedback()
    x = np.array([2.0, 0.0, 0.0, 1.0], np.float32)
    rng = np.random.RandomState(7)
    for t in range(5000):
        assert not _tube_failure(x), f"tube failure at step {t}: {x}"
        ctrl.updateImportanceSamplingControl(x, 1)
        ctrl.computeControl(x, 1)
        u = ctrl.getControlSeq()[0] + ctrl.getFeedbackControl(x, ctrl.getTargetStateSeq()[0], 0)
        x, _, _ = dyn.step(x, u, dt)
        x[2:] += (rng.randn(2) * math.sqrt(100.0)).astype(np.float32) * np.float32(dt)  # computeStateDisturbance
        ctrl.slideControlSequence(1)


# ---- C++ header layer ----------------------------------------------------------------------------------------------
CORL_EXE = os.path.join(ROOT, "tests", "cpp", "corl2020_example.bin")


def _build_corl():
    lib_dir = os.path.join(ROOT, "mppi-generic_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unused-variable", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "corl2020_example.cpp"), "-o", CORL_EXE, "-L", lib_dir,
                           "-lmppi_b200", "-Wl,-rpath," + lib_dir])


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_cpp_robust_cost_headers_compile_and_answer_on_the_host():
    """The reference's include paths, the robust costs' host methods and RobustMPPIController::computeDF, built with plain
    g++ against the shim; the host known answers of autorally_robust_cost_test.cu:119-153 and the DI host constants."""
    tmp = tempfile.mkdtemp()
    src = os.path.join(tmp, "robust_cost_host.bin")
    code = r"""
#include <mppi/controllers/R-MPPI/robust_mppi_controller.cuh>
#include <mppi/cost_functions/autorally/ar_robust_cost.cuh>
#include <mppi/cost_functions/double_integrator/double_integrator_robust_cost.cuh>
#include <mppi/dynamics/double_integrator/di_dynamics.cuh>
#include <mppi/feedback_controllers/DDP/ddp.cuh>
#include <cstdio>
using RM = RobustMPPIController<DoubleIntegratorDynamics, DoubleIntegratorRobustCost,
                                DDPFeedback<DoubleIntegratorDynamics, 50>, 50, 1024>;
float (RM::*df)() = &RM::computeDF;
int main()
{
  ARRobustCost cost;
  ARRobustCostParams p;
  p.max_slip_ang = 1.25;
  p.crash_coeff = 10000;
  p.slip_coeff = 10;
  cost.setParams(p);
  float s[7] = { 0, 0, 0, 0, 1.0f, 10.0f, 0 };
  DoubleIntegratorRobustCost di;
  DoubleIntegratorDynamics::state_array x;
  x << 2.1f, 0, 0, 0;
  auto dp = di.getParams();
  dp.velocity_cost = 0;
  di.setParams(dp);
  std::vector<float> ch0(4 * 4, 0.0f), ch1(16, 1.0f), ch2(16, 3.0f), ch3(16, 0.25f);
  ARRobustCost rc;
  rc.setTrackData(ch0.data(), ch1.data(), ch2.data(), ch3.data(), 0, 2, 0, 2, 2);
  auto rp = rc.getParams();
  rp.heading_coeff = 2;
  rc.setParams(rp);
  float y[8] = { 1.0f, 1.0f, 0.0f, 0.0f, 5.0f, 0.0f, 0.0f, 0.0f };
  printf("%.6f %.6f %.6f %.6f %.6f %d %d\n", cost.getStabilizingCost(s), di.computeStateCost(x), di.getLipshitzConstantCost(),
         rc.getCostmapCost(y), rc.computeStateCost(y), (int)ARRobustCost::COST_ID, (int)sizeof(rc.blob()));
  return df != nullptr ? 0 : 1;
}
"""
    cpp = src[:-4] + ".cpp"
    with open(cpp, "w") as f:
        f.write(code)
    lib_dir = os.path.join(ROOT, "mppi-generic_b200")
    try:
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), cpp, "-o", src,
                               "-L", lib_dir, "-lmppi_b200", "-Wl,-rpath," + lib_dir])
        out = subprocess.run([src], capture_output=True, text=True, check=True).stdout.split()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    vals = [float(v) for v in out[:5]]
    assert vals[0] == pytest.approx(1.4711 * 10 + 1e4, rel=4e-6)
    assert vals[1] == pytest.approx(280.0, rel=2e-5)  # host constants: (0.8 - 0.75) / 0.25 * 900 + 100
    assert vals[2] == 1000.0
    # map: track 1 (coeff 33), speed 20 |5 - 3| (desired_speed -1: the map's .z), heading 2 |sin 0 + 0.25|
    assert vals[3] == pytest.approx(33.0 + 40.0 + 0.5, rel=1e-6)
    assert vals[4] == pytest.approx(vals[3], rel=1e-6)
    assert int(out[5]) == 6 and int(out[6]) == C.sizeof(H.ARRobustCostParams)


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_cpp_corl2020_example_compiles_against_the_shim():
    """examples/double_integrator_CORL2020.cu ported, built with plain g++. Only the device probe runs here: without a device
    the binary stops at NO_DEVICE (exit code 5); the experiment itself is the GPU test below."""
    _build_corl()
    p = subprocess.run([CORL_EXE, "--probe"], capture_output=True, text=True, timeout=120)
    if p.returncode == 5:
        assert "no CUDA device" in p.stdout
    else:
        assert p.returncode == 0 and "CUDA device present" in p.stdout, p.stdout[-2000:] + p.stderr[-2000:]


@pytest.mark.gpu
def test_cpp_corl2020_example_rmppi_runs_stay_in_the_tube():
    _build_corl()
    p = subprocess.run([CORL_EXE], capture_output=True, text=True, timeout=1800)
    print(p.stdout)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "run rmppi_rc: tube_failures 0" in p.stdout and "run rmppi_sc: tube_failures 0" in p.stdout
