"""The streaming form of the warp-specialised Autorally K1 (rollout_kernel_ar_ws.cuh, STREAM: noise slabs through a
three-buffer ring, constrained controls formed by each reader, the epilogue's weighted sum from a second read of eps)
against the generic one-thread-per-sample kernel on the same noise, with the criteria of
test_gpu_parity.py::test_autorally_warp_specialised_equals_generic."""
import numpy as np
import pytest

import mppi_generic_b200 as m
from mppi_generic_b200 import workloads as W

H = m.host
pytestmark = pytest.mark.gpu

RING = 3  # ar_ws::kNoiseRing
BX = 64


@pytest.mark.parametrize("pspw", [16, 8, 32])
@pytest.mark.parametrize("N,T", [
    (1000, 100),     # ragged N; 7 slabs through the 3-buffer ring (TMA)
    (BX * 5 + 7, 37),  # odd T: T*C not a multiple of 4, the ring filled by plain loads, a one-step last group
    (700, 250),      # 16 slabs: every buffer refilled four or five times
])
def test_autorally_ws_streaming_equals_generic(N, T, pspw, monkeypatch):
    monkeypatch.setenv("MPPIB_BX", str(BX))
    monkeypatch.setenv("MPPIB_WS_PSPW", str(pspw))
    w = W.autorally(N, T)
    nchunks = (2 * T + 31) // 32
    monkeypatch.setenv("MPPIB_STREAM", "0")
    r = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    resident = r.launch_info()
    r.close()
    monkeypatch.setenv("MPPIB_STREAM", "1")
    a = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    b = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS | H.FLAG_NO_WARP_SPEC)
    info = a.launch_info()
    # 32 / pspw producer warps and one consumer warp per 32 samples; BX-row slabs, RING of them instead of the whole horizon
    assert info["block"] == (32 // pspw + 1) * BX and info["grid"] == (N + BX - 1) // BX
    assert resident["smem_bytes"] - info["smem_bytes"] == (nchunks - RING) * BX * 128
    Ua, sa = a.solve(w.x0, w.U0)
    Ub, sb = b.solve(w.x0, w.U0)
    np.testing.assert_array_equal(a.get_noise(), b.get_noise())
    np.testing.assert_array_equal(a.get_samples(), b.get_samples())  # constrained controls: identical bits
    ca, cb = a.get_costs(), b.get_costs()
    rel = np.abs(ca - cb) / np.maximum(np.abs(cb), 1.0)
    assert rel.max() < 1e-6 and np.mean(ca != cb) < 0.01, (rel.max(), np.mean(ca != cb))
    np.testing.assert_allclose(Ua, Ub, rtol=0, atol=1e-6)
    np.testing.assert_allclose(np.asarray(sa), np.asarray(sb), rtol=1e-6)
    a.close()
    b.close()


def test_autorally_c4_runs_streaming_in_one_wave():
    """C4 (N = 32768, T = 100): the resident 256-sample tile does not fit an SM's shared memory, so the engine takes the
    streaming form at one CTA per SM instead of the two waves of narrow CTAs the resident form would need."""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    w = W.by_name("autorally")
    e = w.make_engine()
    info = e.launch_info()
    e.close()
    block_rows = info["block"] // 3  # 16 samples per producer warp: two producers and a consumer per 32 samples
    assert info["grid"] == (w.N + block_rows - 1) // block_rows
    assert info["grid"] <= sms, (info, sms)  # one CTA per SM: one wave
    assert info["smem_bytes"] < ((2 * w.T + 31) // 32) * block_rows * 128  # less than the resident tile alone
