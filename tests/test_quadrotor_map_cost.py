"""QuadrotorMapCost (cost_functions/quadrotor/quadrotor_map_cost.cu): the C ABI, the host twins against the reference's
known answer and hand-derived values of every term, the host / device body split, the waypoint and gate updates of both
mirrors, the device body in every K1 form the pair reaches against the float32 restatement in
tests/quadrotor_map_cost_oracle.py, DDP feedback on a map-cost engine, a closed loop through the gate course, and the
pre-built controller of the instantiation library."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

import mppi_generic_b200 as m
import oracle
from mppi_generic_b200 import workloads as W
from tests import quadrotor_map_cost_oracle as QO

H = m.host
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_DIR = os.path.join(ROOT, "mppi-generic_b200")


def _state(pos=(0, 0, 0), vel=(0, 0, 0), q=(1, 0, 0, 0), w=(0, 0, 0)):
    return np.array(list(pos) + list(vel) + list(q) + list(w), np.float32)


def _quat(roll, pitch, yaw=0.0):
    """Euler2QuatNWU (math_utils.h:240-257)."""
    cr, sr = math.cos(roll / 2), math.sin(roll / 2)
    cp, sp = math.cos(pitch / 2), math.sin(pitch / 2)
    cy, sy = math.cos(yaw / 2), math.sin(yaw / 2)
    return (cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy,
            cr * cp * sy - sr * sp * cy)


# ---- C ABI ---------------------------------------------------------------------------------------------------------
def test_ids_and_blob_layout():
    assert H.COST_QUADROTOR_MAP == 7 and H.BLOB_COST_TEXTURE == 7
    assert (H.COST_QUADROTOR_QUADRATIC, H.COST_DI_ROBUST, H.COST_AR_ROBUST) == (4, 5, 6)
    assert H.BLOB_ELEVATION_MAP == 6
    fields = [f for f, _ in H.QuadrotorMapCostParams._fields_]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "mppi_b200.h"', 'int main(void){',
           'printf("%zu\\n", sizeof(mppib_quadrotor_map_cost_params));',
           'printf("%d %d\\n", (int)MPPIB_COST_QUADROTOR_MAP, (int)MPPIB_BLOB_COST_TEXTURE);']
    src += [f'printf("%zu\\n", offsetof(mppib_quadrotor_map_cost_params, {f}));' for f in fields]
    src.append("return 0;}")
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write("\n".join(src))
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = subprocess.check_output([exe]).split()
    assert int(out[0]) == C.sizeof(H.QuadrotorMapCostParams) == 44 * 4
    assert (int(out[1]), int(out[2])) == (7, 7)
    for f, v in zip(fields, out[3:]):
        assert getattr(H.QuadrotorMapCostParams, f).offset == int(v), f


def test_reference_defaults():
    p = H.QuadrotorMapCost().params  # quadrotor_map_cost.cuh:14-60
    assert list(p.control_cost_coeff) == [1, 1, 1, 1] and p.discount == 1
    assert (p.attitude_coeff, p.crash_coeff, p.dist_to_waypoint_coeff, p.heading_coeff, p.heading_power) == \
        (10, 1000, 0, 5, 1)
    assert (p.height_coeff, p.track_coeff, p.speed_coeff, p.track_slop, p.gate_pass_cost) == (5, 10, 5, 0, -150)
    assert (p.desired_speed, p.min_dist_to_gate_side, p.track_boundary_cost) == (5, 0.5, 2.5)
    assert p.gate_margin == pytest.approx(0.5) and p.gate_width == pytest.approx(2.15)
    assert all(math.isnan(v) for v in p.end_waypoint) and list(p.curr_waypoint) == [0, 0, 0, 0]


@pytest.mark.parametrize("D,flags", [(1, 0), (2, 0), (2, H.FLAG_RMPPI)])
def test_create_reaches_the_device_check(D, flags):
    L = H.lib()
    h = C.c_void_p()
    d = H.Desc(H.DYN_QUADROTOR, H.COST_QUADROTOR_MAP, 0, 256, 20, D, 0, flags, None, 0, 1)
    rc = L.mppib_create(C.byref(h), C.byref(d))
    if rc == 0:
        L.mppib_destroy(h)
    else:
        assert rc == -5, (rc, L.mppib_last_error())


def test_host_terms_reject_bad_arguments():
    L = H.lib()
    out = C.c_float()
    p = H.QuadrotorMapCost().params
    s = _state()
    assert L.mppib_host_quadrotor_map_term(C.byref(p), 6, H._ptr(s), C.byref(out)) == -1
    assert L.mppib_host_quadrotor_map_term(None, 0, H._ptr(s), C.byref(out)) == -1
    assert L.mppib_host_quadrotor_map_update_waypoint(None, 0, 0, 0, 0) == -1


# ---- host twins: known answer and hand-derived terms ----------------------------------------------------------------
def test_reference_known_answer_speed_cost():
    """QuadrotorMapCost.checkSpeedCost (quadrotor_map_cost_test.cu:34-52): velocity (3, 4), speed_coeff = desired_speed
    = 10 -> 250, through the host twin, the Python class and the restatement (the C++ class: test_cpp_example)."""
    cost = H.QuadrotorMapCost()
    cost.params.speed_coeff = cost.params.desired_speed = 10.0
    s = _state(vel=(3, 4, 0))
    assert cost.computeSpeedCost(s) == 250.0
    assert float(QO.speed_cost(cost.params, s[None])[0]) == 250.0


def test_height_cost_midpoint_and_step():
    cost = H.QuadrotorMapCost()
    p = cost.params
    cost.updateWaypoint(0, 0, 1, 0)
    cost.updateWaypoint(4, 0, 3, 0)  # prev z = 1, curr z = 3
    # midpoint: d1 = d2 = 2 -> w = 2 / 4.001, height = (1 - w) (1 + 3) = 2.0005; at z = 2.0005 the cost is ~0
    w = 2 / 4.001
    interp = (1 - w) * 1 + (1 - w) * 3
    s = _state(pos=(2, 0, interp))
    assert cost.computeHeightCost(s) == pytest.approx(0.0, abs=1e-5)
    s = _state(pos=(2, 0, interp + 1.0))  # squared difference 1 < gate_width: height_coeff * 1
    assert cost.computeHeightCost(s) == pytest.approx(5.0, rel=1e-5)
    s = _state(pos=(2, 0, interp + 1.5))  # squared difference 2.25 > 2.15: + 400
    assert cost.computeHeightCost(s) == pytest.approx(5.0 * 2.25 + 400, rel=1e-5)
    for z in (interp + 1.0, interp + 1.5, interp - 1.5):
        s = _state(pos=(2, 0, z))
        assert float(QO.height_cost(p, s[None])[0]) == pytest.approx(cost.computeHeightCost(s), rel=1e-6)


@pytest.mark.parametrize("comp,fires", [(-0.25, True), (-0.5, True), (-0.55, False), (0.0, False), (-1e-3, True),
                                        (0.5, False), (1.0, False), (1.001, True), (1.5, True), (1.55, False)])
def test_gate_side_band_edges(comp, fires):
    """Gate corners at (0, +-2.15) (waypoint at the origin, heading pi/2): the right corner (0, -2.15) is comp 0, the left
    (0, 2.15) comp 1. On the gate line (perpendicular distance 0) the term fires in [-0.5, 0) and (1, 1.5]."""
    cost = H.QuadrotorMapCost()
    cost.updateWaypoint(0, 0, 0, math.pi / 2)
    p = cost.params
    right_y, left_y = p.curr_gate_right[1], p.curr_gate_left[1]
    y = right_y + comp * (left_y - right_y)
    s = _state(pos=(p.curr_gate_right[0], y, 0))
    _, c = QO.gate_side_comp(p, s[None])
    got = cost.computeGateSideCost(s)
    if fires:
        assert got == pytest.approx(1000 * abs(float(c[0])), rel=1e-6) and got > 0
    else:
        assert got == 0.0
    assert float(QO.gate_side_cost(p, s[None])[0]) == got


def test_gate_side_needs_the_gate_line():
    cost = H.QuadrotorMapCost()
    cost.updateWaypoint(0, 0, 0, math.pi / 2)
    s = _state(pos=(1.0, -2.5, 0))  # along-gate component in the band, but 1 m off the gate line
    assert cost.computeGateSideCost(s) == 0.0


def test_heading_cost_at_the_waypoint_and_away():
    cost = H.QuadrotorMapCost()
    cost.updateWaypoint(5, 0, 0, math.pi / 2)
    assert cost.computeHeadingCost(_state(pos=(5, 0.1, 0), vel=(0, 3, 0))) == 0.0  # within gate_margin: no term
    assert cost.computeHeadingCost(_state(pos=(0, 0, 0), vel=(2, 0, 0))) == pytest.approx(0.0, abs=1e-6)  # pointing at it
    # flying along +y, the waypoint along +x: pi/2 off; heading_power 2 squares it
    assert cost.computeHeadingCost(_state(vel=(0, 2, 0))) == pytest.approx(5 * math.pi / 2, rel=1e-6)
    cost.params.heading_power = 2.0
    assert cost.computeHeadingCost(_state(vel=(0, 2, 0))) == pytest.approx(5 * (math.pi / 2) ** 2, rel=1e-5)
    # the yaw is the world-frame velocity's: a body yawed by pi/2 flying body-x moves along world +y
    s = _state(vel=(2, 0, 0), q=_quat(0, 0, math.pi / 2))
    assert cost.computeHeadingCost(s) == pytest.approx(5 * (math.pi / 2) ** 2, rel=1e-5)


def test_stabilizing_cost_at_known_roll_and_pitch():
    cost = H.QuadrotorMapCost()
    for roll, pitch in ((0.3, 0.0), (0.0, -0.4), (0.2, 0.25)):
        s = _state(q=_quat(roll, pitch, 0.7))
        assert cost.computeStabilizingCost(s) == pytest.approx(10 * (roll ** 2 + pitch ** 2), rel=1e-5)
        assert float(QO.stabilizing_cost(cost.params, s[None])[0]) == pytest.approx(cost.computeStabilizingCost(s),
                                                                                     rel=2e-6)


def test_gate_pass_inside_and_outside_the_margin():
    cost = H.QuadrotorMapCost()
    cost.params.speed_coeff = cost.params.heading_coeff = cost.params.height_coeff = 0.0
    cost.updateWaypoint(3, 0, 2, math.pi / 2)
    assert cost.computeStateCost(_state(pos=(3, 0.4, 2))) == pytest.approx(-150.0)
    assert cost.computeStateCost(_state(pos=(3, 0.6, 2))) == pytest.approx(0.0)
    assert cost.distToWaypoint(_state(pos=(3, 0.6, 2)), cost.params.curr_waypoint) == pytest.approx(0.6)


def _random_states(n, seed=3, span=8.0):
    rng = np.random.RandomState(seed)
    y = np.zeros((n, 13), np.float32)
    y[:, 0] = rng.uniform(-span, span, n)
    y[:, 1] = rng.uniform(-span, span, n)
    y[:, 2] = rng.uniform(0, 4, n)
    y[:, 3:6] = rng.uniform(-5, 5, (n, 3))
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q *= np.sign(q[:, :1])
    y[:, 6:10] = q
    y[:, 10:13] = rng.uniform(-1, 1, (n, 3))
    return y


def _course_cost(with_map=True):
    w = W.quadrotor_gates(64, 10, use_map=with_map)
    w.cost.params.dist_to_waypoint_coeff = 0.7
    return w.cost


def test_host_minus_device_is_costmap_crash_and_waypoint():
    cost = _course_cost()
    p, tex = cost.params, cost.tex_helper_
    y = _random_states(3000)
    host = np.array([cost.computeStateCost(s) for s in y], np.float32)
    np.testing.assert_allclose(host, QO.host_cost(p, y), rtol=2e-5, atol=2e-3)
    dev, crash = QO.device_cost(p, tex.hdr, tex.values, y)
    want = QO.costmap_cost(p, tex.hdr, tex.values, y) + crash * np.float32(p.crash_coeff) - QO.waypoint_cost(p, y)
    np.testing.assert_allclose(dev - host, want, rtol=1e-5, atol=1e-2)


def test_restatement_against_float64():
    cost = _course_cost()
    p, tex = cost.params, cost.tex_helper_
    y = _random_states(4000, seed=9)
    keep = ~QO.on_discontinuity(p, tex.hdr, tex.values, y)
    assert keep.mean() > 0.9
    y = y[keep]
    got, _ = QO.device_cost(p, tex.hdr, tex.values, y)
    d = y.astype(np.float64)
    cw, pw = np.array(list(p.curr_waypoint), np.float64), np.array(list(p.prev_waypoint), np.float64)
    dist = np.linalg.norm(d[:, :3] - cw[:3], axis=1)
    d1, d2 = np.hypot(d[:, 0] - pw[0], d[:, 1] - pw[1]), np.hypot(d[:, 0] - cw[0], d[:, 1] - cw[1])
    hi = (1 - d1 / (d1 + d2 + 0.001)) * pw[2] + (1 - d2 / (d1 + d2 + 0.001)) * cw[2]
    hd = (d[:, 2] - hi) ** 2
    c = p.height_coeff * hd + np.where(hd > p.gate_width, 400, 0)
    q0, q1, q2, q3 = d[:, 6], d[:, 7], d[:, 8], d[:, 9]
    R = np.array([[q0 ** 2 + q1 ** 2 - q2 ** 2 - q3 ** 2, 2 * (q1 * q2 - q0 * q3), 2 * (q1 * q3 + q0 * q2)],
                  [2 * (q1 * q2 + q0 * q3), q0 ** 2 - q1 ** 2 + q2 ** 2 - q3 ** 2, 2 * (q2 * q3 - q0 * q1)]])
    wv = np.einsum("ijn,nj->ni", R, d[:, 3:6])
    ang = np.arctan2(wv[:, 1], wv[:, 0]) - np.arctan2(cw[1] - d[:, 1], cw[0] - d[:, 0])
    ang = (ang + np.pi) % (2 * np.pi) - np.pi
    c += np.where(dist > p.gate_margin, p.heading_coeff * np.abs(ang) ** p.heading_power, 0)
    c += p.speed_coeff * (np.hypot(d[:, 3], d[:, 4]) - p.desired_speed) ** 2
    roll = np.arctan2(2 * q3 * q2 + 2 * q0 * q1, q0 ** 2 + q3 ** 2 - q2 ** 2 - q1 ** 2)
    pitch = -np.arcsin(np.clip(-2 * q0 * q2 + 2 * q1 * q3, -1, 1))
    c += p.attitude_coeff * (roll ** 2 + pitch ** 2)
    c += np.where(dist < p.gate_margin, p.gate_pass_cost, 0)
    L, Rr = np.array(list(p.curr_gate_left)), np.array(list(p.curr_gate_right))
    g = (L - Rr)[:2]
    r = d[:, :2] - Rr[:2]
    perp, comp = r[:, 0] * g[1] - r[:, 1] * g[0], (r @ g) / (g @ g)
    gate = np.where((np.abs(perp) < p.min_dist_to_gate_side) & (((comp < 0) & (comp >= -0.5)) | ((comp > 1) & (comp <= 1.5))),
                    p.crash_coeff * np.abs(comp), 0)
    c += gate + np.where(gate != 0, p.crash_coeff, 0)
    hdr, vals = tex.hdr, tex.values.astype(np.float64)
    u = (d[:, 0] - hdr.origin[0]) / hdr.resolution[0] / hdr.width
    v = (d[:, 1] - hdr.origin[1]) / hdr.resolution[1] / hdr.height
    c += np.where((u < 0) | (u > 1) | (v < 0) | (v > 1), p.crash_coeff, 0)
    qx, qy = np.clip(u * hdr.width - 0.5, 0, hdr.width - 1), np.clip(v * hdr.height - 0.5, 0, hdr.height - 1)
    x0, y0 = np.minimum(np.floor(qx).astype(int), hdr.width - 2), np.minimum(np.floor(qy).astype(int), hdr.height - 2)
    fx, fy = qx - x0, qy - y0
    t = (vals[y0, x0] * (1 - fx) + vals[y0, x0 + 1] * fx) * (1 - fy) + (vals[y0 + 1, x0] * (1 - fx) + vals[y0 + 1, x0 + 1] * fx) * fy
    c += np.where(t > p.track_slop, p.track_coeff * t, 0) + np.where(t > p.track_boundary_cost, p.crash_coeff, 0)
    np.testing.assert_allclose(got, c, rtol=2e-5, atol=2e-3)


# ---- waypoint / gate updates ------------------------------------------------------------------------------------------
def test_update_waypoint_shifts_and_derives_the_gate():
    cost = H.QuadrotorMapCost()
    p = cost.params
    assert p.updateWaypoint(1, 2, 3, 0.5)
    assert p.updateWaypoint(4, 5, 6, 1.0)
    assert list(p.prev_waypoint) == pytest.approx([1, 2, 3, 0.5]) and list(p.curr_waypoint) == pytest.approx([4, 5, 6, 1.0])
    gw = np.float32(2.15)
    c, s = np.float32(math.cos(1.0)), np.float32(math.sin(1.0))
    assert list(p.curr_gate_left) == pytest.approx([4 + c * gw, 5 + s * gw, 6], rel=1e-6)
    assert list(p.curr_gate_right) == pytest.approx([4 - c * gw, 5 - s * gw, 6], rel=1e-6)
    assert list(p.prev_gate_left) == pytest.approx([1 + math.cos(0.5) * gw, 2 + math.sin(0.5) * gw, 3], rel=1e-6)
    before = bytes(p)
    assert not p.updateWaypoint(4, 5, 6, 1.0) and bytes(p) == before  # unchanged: nothing moves
    assert p.updateGateBoundaries(0, 1, 2, 3, 4, 5)
    assert list(p.prev_gate_left) == pytest.approx([4 + c * gw, 5 + s * gw, 6], rel=1e-6)
    assert not p.updateGateBoundaries(0, 1, 2, 3, 4, 5)


def test_cost_update_overloads_and_size_message(capfd):
    cost = H.QuadrotorMapCost()
    cost.updateWaypoint((1, 2, 3, 0.25))
    a = bytes(cost.params)
    other = H.QuadrotorMapCost()
    other.updateWaypoint(1, 2, 3, 0.25)
    assert bytes(other.params) == a
    cost.updateGateBoundaries([1, 2, 3, 4, 5])
    assert "You need 1 more floats in the call to updateGateBoundaries" in capfd.readouterr().err
    assert bytes(cost.params) == a
    cost.updateGateBoundaries((1, 2, 3), (4, 5, 6))
    other.updateGateBoundaries(1, 2, 3, 4, 5, 6)
    assert bytes(cost.params) == bytes(other.params)
    assert cost.params_pushes == 0  # no engine bound: nothing to push


CPP_BLOB_SRC = r'''
#include <mppi/cost_functions/quadrotor/quadrotor_map_cost.cuh>
#include <cstdio>
int main()
{
  QuadrotorMapCost cost;
  cost.updateWaypoint(0.0f, 0.0f, 2.0f, 0.0f);
  cost.updateWaypoint(float4{ 6.0f, 0.0f, 2.0f, 1.5707964f });
  cost.updateWaypoint(12.0f, 2.0f, 2.5f, 1.2707963f);
  cost.updateGateBoundaries(std::vector<float>{ 1.0f, 2.0f });
  cost.updateGateBoundaries(float3{ 11.0f, 4.0f, 2.5f }, float3{ 13.0f, 0.0f, 2.5f });
  mppib_quadrotor_map_cost_params b = cost.blob();
  fwrite(&b, sizeof(b), 1, stdout);
  float s[13] = { 3, 4, 1, 3, 4, 0, 1, 0, 0, 0, 0, 0, 0 };
  auto p = cost.getParams();
  p.speed_coeff = p.desired_speed = 10;
  cost.setParams(p);
  QuadrotorMapCost::output_array y;
  for (int i = 0; i < 13; i++)
    y[i] = s[i];
  float r[2] = { cost.computeSpeedCost(s), cost.computeStateCost(y) };
  fwrite(r, sizeof(r), 1, stdout);
  return 0;
}
'''


def test_cpp_and_python_blobs_are_byte_identical():
    """The same sequence of calls in the C++ class and the Python class writes the same bytes; the C++ class gives the
    reference's known answer (250) and the host body the Python class gives."""
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "t.cpp"), os.path.join(d, "t")
        open(src, "w").write(CPP_BLOB_SRC)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", LIB_DIR,
                               "-l:libmppi_b200.so", "-Wl,-rpath," + LIB_DIR])
        out = subprocess.check_output([exe])
    cost = H.QuadrotorMapCost()
    cost.updateWaypoint(0.0, 0.0, 2.0, 0.0)
    cost.updateWaypoint((6.0, 0.0, 2.0, 1.5707964))
    cost.updateWaypoint(12.0, 2.0, 2.5, 1.2707963)
    cost.updateGateBoundaries([1.0, 2.0])
    cost.updateGateBoundaries((11.0, 4.0, 2.5), (13.0, 0.0, 2.5))
    n = C.sizeof(H.QuadrotorMapCostParams)
    assert out[:n] == bytes(cost.params)
    speed, state = np.frombuffer(out[n:], np.float32)
    assert speed == 250.0
    cost.params.speed_coeff = cost.params.desired_speed = 10.0
    assert state == np.float32(cost.computeStateCost(np.array([3, 4, 1, 3, 4, 0, 1, 0, 0, 0, 0, 0, 0], np.float32)))


# ---- the gate-course workload and the instantiation library (blob validation needs an engine: GPU section) -----------
def test_workload_course_and_map():
    w = W.quadrotor_gates(64, 10)
    p, tex = w.cost.params, w.cost.tex_helper_
    assert list(p.prev_waypoint) == [0, 0, 2, 0] and list(p.curr_waypoint)[:3] == [6, 0, 2]
    assert tex.checkTextureUse(0) and tex.values.shape == (76, 112)
    # the map is low on the course and crosses both thresholds away from it
    on = QO.bilinear(tex.hdr, tex.values, *QO.tex_coords(tex.hdr, np.array([[3, 0, 2] + [0] * 10], np.float32)))
    assert on[0] < 0.15  # half a cell off the line at most, plus the noise
    assert tex.values.max() > p.track_boundary_cost
    assert W.advance_quadrotor_gate(w, np.array([6.2, 0.1, 2.0])) and w.extra["gate"] == 1
    assert list(p.curr_waypoint)[:3] == [12, 2, 2.5] and list(p.prev_waypoint)[:3] == [6, 0, 2]
    assert not W.advance_quadrotor_gate(w, np.array([7.0, 0.0, 2.0]))


def test_instantiation_library_has_the_map_cost_controller():
    """<mppi/instantiations/quadrotor_mppi/quadrotor_mppi.cuh> with MPPIB_USE_INSTANTIATION_LIBRARY: the map-cost controller
    is an undefined symbol of the user's object and a defined one of libmppi_b200_controllers.so; the example exits 5
    without a device (0 with one: test_cpp_example_flies_the_gates_on_the_gpu)."""
    exe = _build_cpp_example()
    needle = "VanillaMPPIController<QuadrotorDynamics, QuadrotorMapCost, DDPFeedback<QuadrotorDynamics, 100>, 100, 512"
    und = subprocess.run(["nm", "-C", "--undefined-only", exe + ".o"], capture_output=True, text=True, check=True).stdout
    assert any(needle in ln and "::computeControl(" in ln for ln in und.splitlines())
    lib = os.path.join(LIB_DIR, "libmppi_b200_controllers.so")
    defined = subprocess.run(["nm", "-DC", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    assert any(needle in ln and "::computeControl(" in ln for ln in defined.splitlines())
    p = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    if p.returncode == 5:
        assert "no CUDA device" in p.stdout
    else:
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]


def _build_cpp_example():
    subprocess.check_call(["bash", os.path.join(ROOT, "src", "controllers", "build.sh")])
    exe = os.path.join(ROOT, "tests", "cpp", "quadrotor_map_example.bin")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DMPPIB_USE_INSTANTIATION_LIBRARY", "-I", os.path.join(ROOT, "include"),
                           "-c", os.path.join(ROOT, "tests", "cpp", "quadrotor_map_example.cpp"), "-o", exe + ".o"])
    subprocess.check_call(["g++", exe + ".o", "-o", exe, "-L", LIB_DIR, "-l:libmppi_b200_controllers.so",
                           "-l:libmppi_b200.so", "-Wl,-rpath," + LIB_DIR])
    return exe


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _wide_sampler(w, std=(1.5, 1.5, 1.5, 6.0)):
    """Noise wide enough that the samples leave the map, cross both map thresholds and hit gate sides. The sampler's
    control cost (the likelihood-ratio term K1 adds to each step) is off, so that a trajectory's cost is the state cost's."""
    w.sampler.setStdDev(list(std))
    w.sampler.setControlCostCoeff([0.0, 0.0, 0.0, 0.0])
    return w


def _oracle_states(w, samples, idx, x0):
    """State trajectories [T][13] of rollouts `idx` by the oracle's CPU rollout of the device's constrained controls (the
    quadratic-cost pair: the states do not depend on the cost)."""
    qc = H.QuadrotorQuadraticCost()
    outs = []
    for n in idx:
        o, _, _ = oracle.sampled_trajectory(w.dyn.DYN_ID, H.COST_QUADROTOR_QUADRATIC, w.dyn.params, qc.params,
                                            w.sampler.params, None, None, len(samples), w.T, 0, int(n), False, w.dt,
                                            w.lambda_, w.alpha, x0, w.U0[0], samples[n])
        outs.append(np.asarray(o, np.float32))
    return outs


def _restated_cost(w, Y):
    tex = w.cost.tex_helper_
    hdr = tex.hdr if tex.checkTextureUse(0) else None
    c, flags = QO.trajectory_costs(w.cost.params, hdr, tex.values if hdr is not None else None, Y)
    run = np.float32(0)
    for v in c:
        run = np.float32(run + v)
    return run / np.float32(w.T), c, flags


def _parity(w, c, samples, x0, dump, idx, tol=1e-4):
    """Device per-sample costs c[idx] within `tol` of the restatement on the oracle's states, or, for each outlier, the
    device's own per-step dump sums to its cost and the first step that differs sits on one of the cost's
    discontinuities (or the crash flag)."""
    outs = _oracle_states(w, samples, idx, x0)
    ref = np.array([_restated_cost(w, o)[0] for o in outs], np.float32)
    rel = np.abs(c[idx] - ref) / np.maximum(np.abs(ref), 1.0)
    bad = np.nonzero(rel > tol)[0]
    assert bad.size <= 0.03 * len(idx), (bad.size, len(idx), float(rel.max()))
    assert np.median(rel) < 1e-5
    tex = w.cost.tex_helper_
    hdr = tex.hdr if tex.checkTextureUse(0) else None
    if bad.size:
        outs_dev, costs_dev = dump(np.asarray(idx)[bad])[:2]
        np.testing.assert_allclose(costs_dev.sum(axis=1), c[np.asarray(idx)[bad]], rtol=5e-6)
        for k, b in enumerate(bad):
            o_dev = np.asarray(outs_dev[k], np.float32)
            step = _restated_cost(w, o_dev)[1]
            dev = costs_dev[k][:w.T] * w.T
            off = np.nonzero(np.abs(step - dev) > 1e-4 * np.maximum(1.0, np.abs(step)))[0]
            ref_steps = _restated_cost(w, outs[b])[1]
            parted = np.nonzero(np.abs(ref_steps - dev) > 1e-4 * np.maximum(1.0, np.abs(ref_steps)))[0]
            first = min([v[0] for v in (off, parted) if v.size] or [None]) if (off.size or parted.size) else None
            if first is None:
                continue
            jumps = QO.on_discontinuity(w.cost.params, hdr, tex.values if hdr is not None else None,
                                        np.stack([o_dev[first], outs[b][first]]))
            assert jumps.any(), f"sample {idx[b]}: first differing step {first} is off every discontinuity"
    return int(bad.size)


def _solve_and_check(w, e, x0=None):
    x0 = w.x0[0] if x0 is None else x0
    e.solve(w.x0, w.U0)
    c = e.get_costs()[0]
    samples = e.get_samples()[0]
    idx = np.random.RandomState(0).choice(w.N, min(w.N, 300), replace=False)
    return _parity(w, c, samples, x0, lambda ix: e.sample_trajectories(x0, w.U0[0], ix), idx)


def _excursions(w, e):
    """The samples of the last solve really reach the map edge, both thresholds and a gate side (map-on case)."""
    samples = e.get_samples()[0]
    idx = np.arange(0, w.N, max(1, w.N // 200))
    Y = np.concatenate(_oracle_states(w, samples, idx, w.x0[0]))
    p, tex = w.cost.params, w.cost.tex_helper_
    u, v = QO.tex_coords(tex.hdr, Y)
    t = QO.bilinear(tex.hdr, tex.values, u, v)
    assert ((u < 0) | (u > 1) | (v < 0) | (v > 1)).any()
    assert (t > p.track_slop).any() and (t < p.track_boundary_cost).any() and (t > p.track_boundary_cost).any()


FORMS = [("resident", 0, {}), ("no_tma", H.FLAG_NO_TMA, {}), ("stream", 0, {"MPPIB_STREAM": "1"}),
         ("bx64", 0, {"MPPIB_BX": "64"}), ("bx128", 0, {"MPPIB_BX": "128"})]


@pytest.mark.gpu
@pytest.mark.parametrize("use_map", [False, True], ids=["map_off", "map_on"])
@pytest.mark.parametrize("name,flags,env", FORMS, ids=[f[0] for f in FORMS])
def test_k1_forms_match_the_restatement(name, flags, env, use_map, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    w = _wide_sampler(W.quadrotor_gates(4096, 60, use_map=use_map))
    w.x0[0, 3] = 2.0
    if use_map:  # 1 m inside the map's x edge and 5 m off the course: samples leave the map and cross both thresholds
        w.x0[0, :4] = [-3.0, -4.0, 2.0, -2.0]
    e = w.make_engine(flags=flags | H.FLAG_WRITEBACK_CONTROLS)
    info = e.launch_info()
    if name == "no_tma":
        assert not info["uses_tma"]
    if name.startswith("bx"):
        assert info["block"] == int(env["MPPIB_BX"])
    if name == "stream":  # the 2-slab ring at 64 samples per CTA: less shared memory than the resident tile at 64
        monkeypatch.setenv("MPPIB_STREAM", "0")
        monkeypatch.setenv("MPPIB_BX", "64")
        res = w.make_engine(flags=flags | H.FLAG_WRITEBACK_CONTROLS)
        assert info["block"] == 64 and info["smem_bytes"] < res.launch_info()["smem_bytes"]
        res.close()
    _solve_and_check(w, e)
    if use_map:
        _excursions(w, e)
    e.close()


@pytest.mark.gpu
def test_sampled_trajectories_match_and_sum_to_k1():
    w = _wide_sampler(W.quadrotor_gates(2048, 50))
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    U, _ = e.solve(w.x0, w.U0)
    c = e.get_costs()[0]
    samples = e.get_samples()[0]
    idx = np.arange(0, w.N, 16)
    outs, costs, crash = e.sample_trajectories(w.x0[0], w.U0[0], idx)
    np.testing.assert_allclose(costs.sum(axis=1), c[idx], rtol=5e-6)
    ref = _oracle_states(w, samples, idx, w.x0[0])
    crashed = 0
    for k in range(len(idx)):
        o = np.asarray(outs[k], np.float32)
        _, step, flags = _restated_cost(w, o)
        np.testing.assert_array_equal(np.asarray(crash[k])[:w.T], flags)
        crashed += flags.any()
        ok = np.abs(step - costs[k][:w.T] * w.T) <= 1e-4 * np.maximum(1.0, np.abs(step))
        assert ok.all() or QO.on_discontinuity(w.cost.params, w.cost.tex_helper_.hdr, w.cost.tex_helper_.values,
                                               o[~ok]).all()
        assert np.abs(o[:, :3] - ref[k][:, :3]).max() < 2e-3
    # U: the importance-weighted mean of the samples, recomputed in float64 from K1's costs
    lam = w.lambda_
    cc = c.astype(np.float64)
    wts = np.exp(-(cc - cc.min()) / lam)
    u64 = np.tensordot(wts / wts.sum(), samples.astype(np.float64), axes=1)
    np.testing.assert_allclose(U[0], u64, atol=2e-4)


@pytest.mark.gpu
def test_tube_two_systems_match():
    """Tube-MPPI (D = 2): each system's costs against the restatement, dumped per system."""
    w = _wide_sampler(W.quadrotor_gates(2048, 50))
    w.D = 2
    w.x0 = np.stack([w.x0[0], w.x0[0] + np.array([0.1, 0.3, 0.0] + [0.0] * 10, np.float32)])
    w.U0 = np.tile(w.U0, (2, 1, 1))
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    e.solve(w.x0, w.U0)
    c, samples = e.get_costs(), e.get_samples()
    for d in range(2):
        idx = np.random.RandomState(d).choice(w.N, 200, replace=False)
        _parity(w, c[d], samples[d], w.x0[d],
                lambda ix, d=d: e.sample_trajectories(w.x0[d], w.U0[d], ix, distribution=d), idx)
    e.close()


def _reroll(w, x0, controls):
    """A single-system engine that rolls out exactly `controls` [N][T][C] from x0: noise = the controls, sigma 1, mean 0,
    so u = eps. Rollout 0 is the sampler's zero-noise rollout, so the controls go to rollouts 1 .. N."""
    N = controls.shape[0]
    sampler = H.GaussianDistribution(4, [1.0, 1.0, 1.0, 1.0])
    e = H.Engine(w.dyn, w.cost, sampler, N + 1, w.T, 1, flags=H.FLAG_WRITEBACK_CONTROLS)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    eps = np.concatenate([np.zeros((1, w.T, 4), np.float32), controls]).astype(np.float32)
    e.set_noise(eps)
    zeros = np.zeros((1, w.T, 4), np.float32)
    e.rollout_only(x0[None], zeros, 0, 0)
    np.testing.assert_array_equal(e.get_samples()[0][1:], controls)
    return e, e.get_costs()[0][1:], lambda ix: e.sample_trajectories(x0, zeros[0], np.asarray(ix) + 1)


@pytest.mark.gpu
@pytest.mark.parametrize("with_gains", [False, True], ids=["no_gains", "gains"])
def test_rmppi_rollouts_match(with_gains):
    """RMPPI: each system's applied controls, re-rolled in a single-system engine, give the RMPPI kernel's real cost to
    1e-6; the re-rolls match the restatement; the nominal cost is 0.5 c_nom + 0.5 max(min(c_real, threshold), c_nom)."""
    w = _wide_sampler(W.quadrotor_gates(1024, 40))
    thr = 3000.0
    e = H.Engine(w.dyn, w.cost, w.sampler, w.N, w.T, 2, flags=H.FLAG_RMPPI)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    e.seed(w.seed, 0)
    gains = (np.random.RandomState(3).randn(w.T, 13, 4) * 0.05).astype(np.float32) if with_gains else None
    e.set_rmppi(thr, gains)
    x0 = np.stack([w.x0[0], w.x0[0] + np.array([0.05, 0.1, 0.02] + [0.0] * 10, np.float32)])
    U_in = np.tile(w.U0, (2, 1, 1))
    e.draw_noise()
    e.rollout_only(x0, U_in, 1, 0)
    c, applied = e.get_costs(), e.get_samples()
    costs = []
    for d in range(2):
        r, v, dump = _reroll(w, x0[d], applied[d])
        idx = np.random.RandomState(d).choice(w.N, 150, replace=False)
        _parity(w, v, applied[d], x0[d], dump, idx)
        costs.append(v)
        r.close()
    c_nom, c_real = costs
    np.testing.assert_allclose(c[1], c_real, rtol=1e-6, atol=0)
    nom = (np.float32(0.5) * c_nom + np.float32(0.5) * np.maximum(np.minimum(c[1], np.float32(thr)), c_nom)).astype(np.float32)
    np.testing.assert_allclose(c[0], nom, rtol=1e-6, atol=0)
    e.close()


@pytest.mark.gpu
def test_init_eval_matches():
    """init-eval (rmppi_kernels.cu:230-356): candidate k's samples take the sampled controls of distribution 0 from step
    min(t + stride_k, T - 1), on the noise the call draws."""
    w = W.quadrotor_gates(512, 30)
    w.sampler.setControlCostCoeff([0.0, 0.0, 0.0, 0.0])
    e = H.Engine(w.dyn, w.cost, w.sampler, w.N, w.T, 2, flags=H.FLAG_RMPPI)
    e.set_solver(w.dt, w.lambda_, w.alpha)
    e.seed(w.seed, 0)
    e.set_rmppi(3000.0, None)
    x0 = np.stack([w.x0[0], w.x0[0] + np.array([0.3, 0.2, 0.1] + [0.0] * 10, np.float32)])
    U_in = np.tile(w.U0, (2, 1, 1))
    e.draw_noise()
    e.rollout_only(x0, U_in, 1, 0)
    K, spc, stride = 3, 64, 2
    cand = np.stack([x0[0], 0.5 * (x0[0] + x0[1]), x0[1]]).astype(np.float32)
    strides = np.array([0, 1, 2], np.int32)
    got = e.init_eval(cand, strides, spc, U_in[0], stride)
    ctl = e.get_noise()[None].copy()
    oracle.set_gaussian_controls(U_in[:1], w.sampler.params, ctl, 4, w.T, w.N, 1, stride, 0)
    ctl = ctl[0, :spc]
    bad = 0
    for k in range(K):
        idx = np.minimum(np.arange(w.T) + strides[k], w.T - 1)
        ctl_k = ctl[:, idx]
        outs = _oracle_states(w, ctl_k, range(spc), cand[k])
        want = np.array([_restated_cost(w, o)[0] for o in outs], np.float32)
        rel = np.abs(got[k * spc:(k + 1) * spc] - want) / np.maximum(np.abs(want), 1.0)
        bad += int((rel > 1e-4).sum())
    assert bad <= 0.03 * K * spc, bad
    e.close()


@pytest.mark.gpu
def test_cost_texture_blob_validation():
    w = W.quadrotor_gates(256, 10)
    e = w.make_engine()  # pushes the map: accepted
    L = H.lib()
    m_ = w.cost.tex_helper_.blob()
    assert L.mppib_set_blob(e._h, H.BLOB_COST_TEXTURE, m_.ctypes.data, 16) == -1  # shorter than the header
    bad = m_.copy()
    bad[:4] = np.frombuffer(np.int32(1).tobytes(), np.uint8)  # width 1
    assert L.mppib_set_blob(e._h, H.BLOB_COST_TEXTURE, bad.ctypes.data, bad.nbytes) == -1
    assert b"cost texture" in L.mppib_last_error()
    assert L.mppib_set_blob(e._h, H.BLOB_COST_TEXTURE, m_.ctypes.data, m_.nbytes - 4) == -1
    assert L.mppib_set_blob(e._h, H.BLOB_ELEVATION_MAP, m_.ctypes.data, m_.nbytes) == -1  # the dynamics' map id
    e.close()
    q = W.quadrotor(256, 10).make_engine()  # the quadratic cost has no texture
    assert L.mppib_set_blob(q._h, H.BLOB_COST_TEXTURE, m_.ctypes.data, m_.nbytes) == -1
    assert b"cost without one" in L.mppib_last_error()
    q.close()


@pytest.mark.gpu
def test_update_waypoint_pushes_only_on_change():
    w = W.quadrotor_gates(256, 10)
    e = w.make_engine()
    n0 = w.cost.params_pushes
    w.cost.updateWaypoint(tuple(w.cost.params.curr_waypoint))
    assert w.cost.params_pushes == n0
    w.cost.updateWaypoint(12.0, 2.0, 2.5, 1.0)
    assert w.cost.params_pushes == n0 + 1
    e.close()


@pytest.mark.gpu
def test_ddp_gains_do_not_depend_on_the_mppi_cost():
    """DDP tracks its own quadratic costs: a map-cost engine and a quadratic-cost engine give the same gains."""
    wm, wq = W.quadrotor_gates(256, 50), W.quadrotor(256, 50)
    gains = []
    for w in (wm, wq):
        e = w.make_engine()
        traj_x = np.tile(w.x0[0], (w.T, 1)).astype(np.float32)
        traj_u = np.asarray(w.U0[0], np.float32)
        gains.append(np.asarray(e.ddp_feedback(w.x0[0], traj_x, traj_u)[0]))
        e.close()
    np.testing.assert_array_equal(gains[0], gains[1])


@pytest.mark.gpu
def test_closed_loop_flies_two_gates():
    """VanillaMPPIController on quadrotor_gates: through the first two gates (the flight crosses each gate's plane) with no
    gate-side hit, i.e. no crash flag, on any flown state. Prints where each gate was crossed."""
    w = W.quadrotor_gates(512, 100)
    ctrl = H.VanillaMPPIController(w.dyn, w.cost, None, w.sampler, w.dt, 1, w.lambda_, w.alpha, w.T, w.N,
                                   init_control_traj=w.U0[0], seed=w.seed)
    x = w.x0[0].copy()
    flown = []
    for it in range(700):
        ctrl.computeControl(x, 1)
        u = np.asarray(ctrl.getControlSeq()[0], np.float32).copy()
        w.dyn.enforceConstraints(x, u)
        x, _, _ = w.dyn.step(x, u, w.dt)
        flown.append(x.copy())
        ctrl.slideControlSequence(1)
        if W.advance_quadrotor_gate(w, x, radius=0.0):
            print(f"waypoint moved to gate {w.extra['gate']} at step {it}: {x[:3]}")
        if it % 50 == 0:
            print(f"step {it}: position {x[:3]}, velocity {x[3:6]}")
        if w.extra["gate"] >= 2:
            break
    Y = np.array(flown, np.float32)
    gates = W.quadrotor_gate_course()
    assert w.extra["gate"] == 2, (w.extra, Y[-1, :3])
    for g in range(2):
        gx, gy, gz, hd = gates[g]
        side = (Y[:, 0] - gx) * -math.sin(hd) + (Y[:, 1] - gy) * math.cos(hd)
        k = int(np.nonzero(side < 0)[0][0])
        along = (Y[k, 0] - gx) * math.cos(hd) + (Y[k, 1] - gy) * math.sin(hd)
        print(f"gate {g}: crossed at step {k}, {along:+.2f} m from the centre along the gate (half-width "
              f"{w.cost.params.gate_width:.2f} m), height {Y[k, 2]:.2f} m (gate {gz} m)")
        assert abs(along) < w.cost.params.gate_width
    for g in range(3):
        cost = H.QuadrotorMapCost()
        cost.updateWaypoint(gates[g])
        assert not np.any(QO.gate_side_cost(cost.params, Y) != 0), g


@pytest.mark.gpu
def test_cpp_example_flies_the_gates_on_the_gpu():
    exe = _build_cpp_example()
    p = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    print(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
