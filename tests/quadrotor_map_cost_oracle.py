"""Float32 numpy restatement of QuadrotorMapCost (cost_functions/quadrotor/quadrotor_map_cost.cu): the device body
(:92-144, what every rollout runs) and the host body (:63-90, what computeStateCost returns on the CPU), term by term,
vectorised over states y [n][13] (POS 0-2, VEL 3-5, QUAT_W..Z 6-9, ANG_VEL 10-12). Double where the reference computes in
double (the height interpolation). The map is a TwoDTextureHelper<float> map 0 as (header, values [height][width]) with
the host's bilinear formula, which the device evaluates too (csrc/plugins/texture_map.cuh).

Written from the reference's source, not from this project's kernels, so that the tests compare two independent
statements of the same formulas."""
import numpy as np

f32 = np.float32


def _p(p, name):
    return np.asarray(list(getattr(p, name)), np.float32)


def dist_to_waypoint(y, w):
    y = np.asarray(y, np.float32)
    w = np.asarray(w, np.float32)
    return np.sqrt((y[:, 0] - w[0]) ** 2 + (y[:, 1] - w[1]) ** 2 + (y[:, 2] - w[2]) ** 2).astype(np.float32)


def tex_coords(hdr, y):
    """TextureHelper::worldPoseToTexCoord (texture_helper.cu:94-134): normalised (u, v) of each state's position."""
    o = np.asarray(list(hdr.origin), np.float32)
    r = np.asarray(list(hdr.rotations), np.float32)
    res = np.asarray(list(hdr.resolution), np.float32)
    d = (np.asarray(y, np.float32)[:, :3] - o).astype(np.float32)
    mx = r[0] * d[:, 0] + r[1] * d[:, 1] + r[2] * d[:, 2]
    my = r[3] * d[:, 0] + r[4] * d[:, 1] + r[5] * d[:, 2]
    return (mx / res[0] / f32(hdr.width)).astype(np.float32), (my / res[1] / f32(hdr.height)).astype(np.float32)


def bilinear(hdr, values, u, v):
    """TwoDTextureHelper::queryTextureCPU (two_d_texture_helper.cu:151-243): clamp, bilinear, value at the cell centre."""
    w, h = hdr.width, hdr.height
    qx = np.clip((u * f32(w) - f32(0.5)).astype(np.float32), 0, w - 1)
    qy = np.clip((v * f32(h) - f32(0.5)).astype(np.float32), 0, h - 1)
    x0 = np.minimum(np.floor(qx).astype(int), w - 2)
    y0 = np.minimum(np.floor(qy).astype(int), h - 2)
    fx1, fx0 = (x0 + 1 - qx).astype(np.float32), (qx - x0).astype(np.float32)
    fy1, fy0 = (y0 + 1 - qy).astype(np.float32), (qy - y0).astype(np.float32)
    lo = values[y0, x0] * fx1 + values[y0, x0 + 1] * fx0
    hi = values[y0 + 1, x0] * fx1 + values[y0 + 1, x0 + 1] * fx0
    return (lo * fy1 + hi * fy0).astype(np.float32)


def costmap_cost(p, hdr, values, y):
    """:359-395. 0 without a map; outside [0, 1] adds crash_coeff, the clamped map is still read."""
    n = len(y)
    if hdr is None or values is None or not hdr.use:
        return np.zeros(n, np.float32)
    u, v = tex_coords(hdr, y)
    cost = np.where((u < 0) | (u > 1) | (v < 0) | (v > 1), f32(p.crash_coeff), f32(0)).astype(np.float32)
    t = bilinear(hdr, values, u, v)
    cost = cost + np.where(t > f32(p.track_slop), f32(p.track_coeff) * t, f32(0))
    cost = cost + np.where(t > f32(p.track_boundary_cost), f32(p.crash_coeff), f32(0))
    return cost.astype(np.float32)


def gate_side_comp(p, y):
    """(cross product with the gate vector, along-gate component from the right corner) of :264-323."""
    y = np.asarray(y, np.float32)
    L, R = _p(p, "curr_gate_left"), _p(p, "curr_gate_right")
    gx, gy = L[0] - R[0], L[1] - R[1]
    rx, ry = y[:, 0] - R[0], y[:, 1] - R[1]
    with np.errstate(invalid="ignore", divide="ignore"):
        comp = ((rx * gx + ry * gy) / f32(gx * gx + gy * gy)).astype(np.float32)
    return (rx * gy - ry * gx).astype(np.float32), comp


def gate_side_cost(p, y):
    perp, comp = gate_side_comp(p, y)
    with np.errstate(invalid="ignore"):
        fire = (np.abs(perp) < f32(p.min_dist_to_gate_side)) & (((comp < 0) & (comp >= -0.5)) | ((comp > 1) & (comp <= 1.5)))
    return np.where(fire, f32(p.crash_coeff) * np.abs(comp), f32(0)).astype(np.float32)


def height_diff(p, y):
    y = np.asarray(y, np.float32)
    pw, cw = _p(p, "prev_waypoint"), _p(p, "curr_waypoint")
    d1 = np.sqrt((y[:, 0] - pw[0]) ** 2 + (y[:, 1] - pw[1]) ** 2).astype(np.float32)
    d2 = np.sqrt((y[:, 0] - cw[0]) ** 2 + (y[:, 1] - cw[1]) ** 2).astype(np.float32)
    den = (d1 + d2).astype(np.float64) + 0.001
    w1 = (d1.astype(np.float64) / den).astype(np.float32)
    w2 = (d2.astype(np.float64) / den).astype(np.float32)
    hi = ((1.0 - w1.astype(np.float64)) * float(pw[2]) + (1.0 - w2.astype(np.float64)) * float(cw[2])).astype(np.float32)
    return (np.abs(y[:, 2] - hi) ** 2).astype(np.float32)


def height_cost(p, y):
    """:325-357: height_coeff * squared difference, +400 when the squared difference exceeds gate_width."""
    hd = height_diff(p, y)
    return (f32(p.height_coeff) * hd + np.where(hd > f32(p.gate_width), f32(400), f32(0))).astype(np.float32)


def _normalize_angle(a):
    r = np.fmod((a + f32(np.pi)).astype(np.float32), f32(2 * np.pi)).astype(np.float32)
    return np.where(r <= 0, r + f32(np.pi), r - f32(np.pi)).astype(np.float32)


def heading_cost(p, y):
    """:210-238: yaw of Quat2DCM(q) v against the bearing to the waypoint, outside gate_margin."""
    y = np.asarray(y, np.float32)
    q0, q1, q2, q3 = y[:, 6], y[:, 7], y[:, 8], y[:, 9]
    vx, vy, vz = y[:, 3], y[:, 4], y[:, 5]
    R00 = q0 * q0 + q1 * q1 - q2 * q2 - q3 * q3
    R01, R02 = 2 * (q1 * q2 - q0 * q3), 2 * (q1 * q3 + q0 * q2)
    R10, R11, R12 = 2 * (q1 * q2 + q0 * q3), q0 * q0 - q1 * q1 + q2 * q2 - q3 * q3, 2 * (q2 * q3 - q0 * q1)
    yaw = np.arctan2(R10 * vx + R11 * vy + R12 * vz, R00 * vx + R01 * vy + R02 * vz).astype(np.float32)
    cw = _p(p, "curr_waypoint")
    wh = np.arctan2(cw[1] - y[:, 1], cw[0] - y[:, 0]).astype(np.float32)
    c = f32(p.heading_coeff) * np.power(np.abs(_normalize_angle((yaw - wh).astype(np.float32))), f32(p.heading_power))
    return np.where(dist_to_waypoint(y, cw) > f32(p.gate_margin), c, f32(0)).astype(np.float32)


def speed_cost(p, y):
    y = np.asarray(y, np.float32)
    s = np.sqrt(y[:, 3] * y[:, 3] + y[:, 4] * y[:, 4]).astype(np.float32)
    return (f32(p.speed_coeff) * (s - f32(p.desired_speed)) ** 2).astype(np.float32)


def roll_pitch(y):
    """Quat2EulerNWU (math_utils.h:263-270), roll and pitch."""
    y = np.asarray(y, np.float32)
    q0, q1, q2, q3 = y[:, 6], y[:, 7], y[:, 8], y[:, 9]
    roll = np.arctan2(2 * q3 * q2 + 2 * q0 * q1, q0 * q0 + q3 * q3 - q2 * q2 - q1 * q1).astype(np.float32)
    pitch = -np.arcsin(np.clip(-2 * q0 * q2 + 2 * q1 * q3, -1, 1)).astype(np.float32)
    return roll, pitch


def stabilizing_cost(p, y):
    r, pt = roll_pitch(y)
    return (f32(p.attitude_coeff) * (r * r + pt * pt)).astype(np.float32)


def waypoint_cost(p, y):
    d = dist_to_waypoint(y, _p(p, "curr_waypoint"))
    return (f32(p.dist_to_waypoint_coeff) * d * d).astype(np.float32)


def gate_pass(p, y):
    return np.where(dist_to_waypoint(y, _p(p, "curr_waypoint")) < f32(p.gate_margin), f32(p.gate_pass_cost),
                    f32(0)).astype(np.float32)


def host_cost(p, y):
    """:63-90: no costmap term, no crash flag, the waypoint term added."""
    c = gate_side_cost(p, y)
    for term in (height_cost, heading_cost, speed_cost, stabilizing_cost, waypoint_cost):
        c = (c + term(p, y)).astype(np.float32)
    return (c + gate_pass(p, y)).astype(np.float32)


def device_cost(p, hdr, values, y, crash=None):
    """:92-144 for states y with the crash flag each one enters with (default 0). Returns (cost, crash flag after)."""
    y = np.asarray(y, np.float32)
    crash = np.zeros(len(y), np.int32) if crash is None else np.asarray(crash, np.int32).copy()
    gate = gate_side_cost(p, y)
    c = costmap_cost(p, hdr, values, y) + gate
    for term in (height_cost, heading_cost, speed_cost, stabilizing_cost):
        c = (c + term(p, y)).astype(np.float32)
    crash = np.where(gate != 0, 1, crash).astype(np.int32)
    c = (c + gate_pass(p, y)).astype(np.float32)
    return (c + crash.astype(np.float32) * f32(p.crash_coeff)).astype(np.float32), crash


def trajectory_costs(p, hdr, values, Y):
    """Per-step device costs and crash flags of one trajectory Y [T][13] (the crash flag is sticky along it)."""
    Y = np.asarray(Y, np.float32)
    costs = np.empty(len(Y), np.float32)
    flags = np.empty(len(Y), np.int32)
    crash = np.zeros(1, np.int32)
    for t in range(len(Y)):
        c, crash = device_cost(p, hdr, values, Y[t:t + 1], crash)
        costs[t], flags[t] = c[0], crash[0]
    return costs, flags


def on_discontinuity(p, hdr, values, y, tol=2e-3):
    """States within `tol` (relative) of one of this cost's discontinuities: gate_margin, the gate band edges (0, -0.5, 1,
    1.5) and the perpendicular threshold, the +400 step, the two map thresholds, the map edge (0 and 1)."""
    y = np.asarray(y, np.float32)
    d = dist_to_waypoint(y, _p(p, "curr_waypoint"))
    near = np.abs(d - p.gate_margin) < tol * max(1.0, p.gate_margin)
    perp, comp = gate_side_comp(p, y)
    with np.errstate(invalid="ignore"):
        for edge in (0.0, -0.5, 1.0, 1.5):
            near |= np.abs(comp - edge) < tol
        near |= np.abs(np.abs(perp) - p.min_dist_to_gate_side) < tol * max(1.0, p.min_dist_to_gate_side)
    near |= np.abs(height_diff(p, y) - p.gate_width) < tol * max(1.0, p.gate_width)
    if hdr is not None and values is not None and hdr.use:
        u, v = tex_coords(hdr, y)
        for c in (u, v):
            near |= (np.abs(c) < tol) | (np.abs(c - 1) < tol)
        t = bilinear(hdr, values, u, v)
        near |= np.abs(t - p.track_slop) < tol * max(1.0, abs(p.track_slop))
        near |= np.abs(t - p.track_boundary_cost) < tol * max(1.0, abs(p.track_boundary_cost))
    return near
