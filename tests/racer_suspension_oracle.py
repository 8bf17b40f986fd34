"""CPU restatement of RacerDubinsElevationSuspension (dynamics/racer_dubins/racer_dubins_elevation_suspension_lstm.{cuh,cu}),
the yardstick of the device model (csrc/plugins/dynamics.cuh: RacerSuspensionLSTMDynamics and its tensor-core form) and of
its host twin (csrc/host_twins.cpp: racer_suspension_step).

  step(p, net, x, u, dt, h, c, body="device")  the device step, :343-391: the parametric derivatives, the LSTM steering,
                                               computeSimpleSuspensionStep (:200-340), updateState (:394-418, brake in
                                               [0, 1]), the uncertainty propagation and setOutputs (:438-525).
  step(..., body="host")                       the host step, :168-197: the same with sincosf / sinf / tanf of raw angles
                                               (:60-166) and the brake clamped to [0, -control_rngs_[0].x] (:421-435).

The parametric rows and the uncertainty propagation are tests/racer_dubins_elevation_oracle.py's, run on the 19-state
view of this model's state (the layouts differ only in where the steering rate and the uncertainty entries sit). The
network is the CPU oracle's (oracle.binding.lstm_forward), the elevation query the oracle's (oracle.elevation_at_world_pose);
the float4 query is restated here. On the device the divisions by mass, I_xx, I_yy and the normal's z are a product with
the reciprocal; "device" restates that too. `dtype` float32 is the restatement, float64 its precision check (the network
and the elevation query stay float32). Test infrastructure only."""
import math

import numpy as np

from tests import racer_dubins_elevation_oracle as RO

(VEL_X, YAW, POS_X, POS_Y, STEER_ANGLE, BRAKE_STATE, ROLL, PITCH, CG_POS_Z, CG_VEL_I_Z, ROLL_RATE, PITCH_RATE,
 STEER_ANGLE_RATE) = range(13)
UNC0, FILLER_1 = 13, 23
S, C, O = 24, 2, 28
O_POS_I_Z, O_WF_UP, O_WF_FWD, O_WF_SIDE = 4, 10, 11, 12
# wheel body positions FL, FR, BL, BR (:74-77; the rear labels carry swapped y signs)
WHEELS = ((2.981, 0.737), (2.981, -0.737), (0.0, -0.737), (0.0, 0.737))

Params = RO.Params


class Net:
    """The steering network: MPPIB_BLOB_LSTM_WEIGHTS and its (H, L1)."""

    def __init__(self, theta, H, L1):
        self.theta, self.H, self.L1 = np.asarray(theta, np.float32), H, L1
        self.block = 4 * H * H + 4 * H * 4 + 6 * H

    def initial(self):
        b = self.block - 2 * self.H
        return self.theta[b:b + self.H].copy(), self.theta[b + self.H:b + 2 * self.H].copy()

    def __call__(self, inp, h, c):
        from oracle import binding
        out, h, c = binding.lstm_forward(self.theta[:self.block], 4, self.H, self.theta[self.block:],
                                         [self.H + 4, self.L1, 1], np.asarray(inp, np.float32), h, c)
        return np.float32(out[0]), h, c


def _header(blob):
    b = np.ascontiguousarray(blob, np.uint8)
    ints = b[:8].view(np.int32)
    fl = b[8:68].view(np.float32)
    use = int(b[68:72].view(np.int32)[0])
    return int(ints[0]), int(ints[1]), fl[0:3], fl[3:12], fl[12:15], use, b[72:]


def map_use(blob):
    return blob is not None and _header(blob)[5] != 0


def normals_at_world_pose(blob, wx, wy, wz):
    """TwoDTextureHelper<float4>::queryTextureAtWorldPose, host formula (two_d_texture_helper.cu:151-243 per channel), in
    float32."""
    f = np.float32
    w, h, org, rot, res, _, data = _header(blob)
    vals = data.view(np.float32).reshape(h, w, 4)
    dx, dy, dz = f(f(wx) - org[0]), f(f(wy) - org[1]), f(f(wz) - org[2])
    mx = f(f(f(rot[0] * dx) + f(rot[1] * dy)) + f(rot[2] * dz))
    my = f(f(f(rot[3] * dx) + f(rot[4] * dy)) + f(rot[5] * dz))
    qx = f(f(f(f(mx / res[0]) / f(w)) * f(w)) - f(0.5))
    qy = f(f(f(f(my / res[1]) / f(h)) * f(h)) - f(0.5))
    qx = f(w - 1) if qx > w - 1 else (f(0) if qx <= 0 else qx)
    qy = f(h - 1) if qy > h - 1 else (f(0) if qy <= 0 else qy)
    if math.isnan(qx) or math.isnan(qy):
        return np.full(4, np.nan, np.float32)
    x0, y0 = min(int(math.floor(qx)), w - 2), min(int(math.floor(qy)), h - 2)
    fx1, fx0, fy1, fy0 = f(f(x0 + 1) - qx), f(qx - f(x0)), f(f(y0 + 1) - qy), f(qy - f(y0))
    q11, q12, q21, q22 = vals[y0, x0], vals[y0, x0 + 1], vals[y0 + 1, x0], vals[y0 + 1, x0 + 1]
    lo = (q11 * fx1 + q12 * fx0).astype(np.float32)
    hi = (q21 * fx1 + q22 * fx0).astype(np.float32)
    return (lo * fy1 + hi * fy0).astype(np.float32)


def _height(elev_blob, wx, wy, wz):
    import oracle
    return oracle.elevation_at_world_pose(elev_blob, float(wx), float(wy), float(wz))


def suspension(p, x, xd, body, dtype, elev_blob=None, normals_blob=None):
    """computeSimpleSuspensionStep: xd's ROLL, PITCH, CG_POS_Z, CG_VEL_I_Z, ROLL_RATE, PITCH_RATE; returns the maxima
    (up, |fwd|, |side|) over the four wheels, summed in wheel order."""
    f = dtype
    dev = body == "device"
    nrm = (lambda a: RO.normalize_angle(a, dtype)) if dev else (lambda a: a)
    roll, pitch, yaw = x[ROLL], x[PITCH], x[YAW]
    sr, cr = f(np.sin(nrm(roll))), f(np.cos(nrm(roll)))
    sp, cp = f(np.sin(nrm(pitch))), f(np.cos(nrm(pitch)))
    sy, cy = f(np.sin(nrm(yaw))), f(np.cos(nrm(yaw)))
    M00, M01, M10, M11, M20, M21 = cp * cy, sr * sp * cy - cr * sy, cp * sy, sr * sp * sy + cr * cy, -sp, sr * cp
    xd[ROLL], xd[PITCH], xd[CG_POS_Z] = x[ROLL_RATE], x[PITCH_RATE], x[CG_VEL_I_Z]
    k, c_d, r = f(p.spring_k), f(p.drag_c), f(p.wheel_radius)
    if dev:
        inv_m, inv_xx, inv_yy = f(1) / f(p.mass), f(1) / f(p.I_xx), f(1) / f(p.I_yy)
    acc = [f(0), f(0), f(0)]
    up = fwd = side = None
    height, n = f(0), np.array([0, 0, 1, 0], dtype)
    for i, (bx, by) in enumerate(WHEELS):
        bx, by = f(bx), f(by)
        cgx, cgy = f(bx - f(p.c_g[0])), f(by - f(p.c_g[1]))
        wx, wy, wz = M00 * bx + M01 * by + x[POS_X], M10 * bx + M11 * by + x[POS_Y], M20 * bx + M21 * by
        if map_use(elev_blob):
            height = f(_height(elev_blob, wx, wy, wz))
            if not np.isfinite(height):
                height = f(x[CG_POS_Z] - r)
        if map_use(normals_blob):
            n = normals_at_world_pose(normals_blob, wx, wy, wz).astype(dtype)
            if not np.isfinite(n[:3]).all():
                n = np.array([0, 0, 1, 0], dtype)
        wyaw = f(yaw + f(4.0 / -9.1)) if i < 2 else yaw  # S_INDEX(STEER_ANGLE) / -9.1 (:123-126, :260, :264)
        swy, cwy = f(np.sin(wyaw)), f(np.cos(wyaw))
        pos_z = f(x[CG_POS_Z] + roll * cgy - pitch * cgx - r)
        vel_z = f(x[CG_VEL_I_Z] + x[ROLL_RATE] * cgy - x[PITCH_RATE] * cgx)
        h_dot = f(-(x[VEL_X] * cwy * n[0] + x[VEL_X] * swy * n[1]))
        F = f(-k * (pos_z - height) - c_d * (vel_z - h_dot))
        q = f(F * (f(1) / n[2])) if dev else f(F / n[2])
        fw = abs(f(q * (n[0] * cwy + n[1] * swy + n[2] * (-pitch))))
        sd = abs(f(q * (-n[0] * swy + n[1] * cwy + n[2] * roll)))
        up, fwd, side = (F, fw, sd) if i == 0 else (max(up, F), max(fwd, fw), max(side, sd))
        if dev:
            acc[0] = f(acc[0] + F * inv_m)
            acc[1] = f(acc[1] + f(F * cgy) * inv_xx)
            acc[2] = f(acc[2] + f(-F * cgx) * inv_yy)
        else:
            acc[0] = f(acc[0] + F / f(p.mass))
            acc[1] = f(acc[1] + f(F * cgy) / f(p.I_xx))
            acc[2] = f(acc[2] + f(-F * cgx) / f(p.I_yy))
    xd[CG_VEL_I_Z], xd[ROLL_RATE], xd[PITCH_RATE] = acc
    return up, fwd, side


def _view19(x):
    return np.concatenate([x[:8], x[STEER_ANGLE_RATE:STEER_ANGLE_RATE + 1], x[UNC0:UNC0 + 10]])


def step(p, net, x, u, dt, h, c, body="device", dtype=np.float32, elev_blob=None, normals_blob=None):
    """Returns (next_state, state_der, output, h, c) of one step."""
    f = dtype
    x = np.asarray(x, dtype)
    u = np.asarray(u, dtype)
    dt = f(dt)
    # parametric rows and the uncertainty propagation on the 19-state view (its steering rows are replaced below)
    xn19, xd19, _ = RO.step(p, _view19(x), u, dt, body, dtype)
    xd = np.zeros(S, dtype)
    xd[:6] = xd19[:6]
    # computeLSTMSteering (lstm_steering.cu:66-88 host, :131-166 device)
    pa = f((u[1] * f(p.steer_command_angle_scale) - x[STEER_ANGLE]) * f(p.steering_constant))
    sr = f((pa - x[STEER_ANGLE_RATE]) * f(p.steer_accel_constant) - x[STEER_ANGLE_RATE] * f(p.steer_accel_drag_constant))
    xd[STEER_ANGLE_RATE] = max(min(sr, f(p.max_steer_rate)), f(-p.max_steer_rate))
    inp = np.array([x[STEER_ANGLE] * f(0.2), x[STEER_ANGLE_RATE] * f(0.2), u[1], xd[STEER_ANGLE_RATE] * f(0.2)], np.float32)
    out, h, c = net(inp, h, c)
    xd[STEER_ANGLE_RATE] = f(xd[STEER_ANGLE_RATE] + f(out) * f(5.0))
    xd[STEER_ANGLE] = x[STEER_ANGLE_RATE]
    up, fwd, side = suspension(p, x, xd, body, dtype, elev_blob, normals_blob)
    xn = np.zeros(S, dtype)
    xn[:STEER_ANGLE_RATE] = x[:STEER_ANGLE_RATE] + xd[:STEER_ANGLE_RATE] * dt
    xn[YAW] = RO.normalize_angle(xn[YAW], dtype)
    xn[STEER_ANGLE] = max(min(xn[STEER_ANGLE], f(p.max_steer_angle)), f(-p.max_steer_angle))
    xn[STEER_ANGLE_RATE] = x[STEER_ANGLE_RATE] + xd[STEER_ANGLE_RATE] * dt
    xn[BRAKE_STATE] = min(max(xn[BRAKE_STATE], f(0)), f(1) if body == "device" else f(-p.rng_lo[0]))
    xn[UNC0:UNC0 + 10] = xn19[9:19]
    xn[FILLER_1] = x[FILLER_1]
    y = np.zeros(O, dtype)
    y[0], y[2], y[3], y[5] = xn[VEL_X], xn[POS_X], xn[POS_Y], xn[YAW]
    y[O_POS_I_Z] = f(xn[CG_POS_Z] - xn[PITCH] * f(-p.c_g[0]))
    y[6], y[7], y[8], y[9] = xn[ROLL], xn[PITCH], xn[STEER_ANGLE], xn[STEER_ANGLE_RATE]
    y[O_WF_UP], y[O_WF_FWD], y[O_WF_SIDE] = up, fwd, side
    y[RO.O_ACCEL_X], y[15], y[16] = xd[VEL_X], xd[YAW], abs(xn[VEL_X])
    y[17:27] = xn[UNC0:UNC0 + 10]
    return xn, xd, y, h, c
