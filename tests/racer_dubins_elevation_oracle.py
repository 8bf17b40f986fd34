"""CPU restatement of RacerDubinsElevation (dynamics/racer_dubins/racer_dubins_elevation.{cuh,cu}), the yardstick of the
device model (csrc/plugins/dynamics.cuh: RacerDubinsElevationDynamics) and of its host twin (csrc/host_twins.cpp).

  step(p, x, u, dt, body="device")   the device body: racer_dubins_elevation.cu:835-878 with the delay derivative of
                                     racer_dubins.cu:281-293, the steering derivative of :296-304, the acceleration of
                                     racer_dubins_elevation.cu:759-797 and updateState of :800-832 (brake in [0, 1]).
  step(p, x, u, dt, body="host")     the host body: racer_dubins_elevation.cu:32-67,229-255 and RacerDubinsImpl::updateState
                                     (racer_dubins.cu:43-59): sin / tan / sincos without normalizeAngle, brake in
                                     [0, -control_rngs_[0].x].
  grad(p, x, u)                      computeGrad, racer_dubins_elevation.cu:257-334, as written.

Both bodies then run computeUncertaintyPropagation (:662-741) and the static settling; the settling is the CPU oracle's
(oracle/mppi_oracle.cpp: orc_static_settling) when a map is given, flat ground (roll = pitch = height = 0) otherwise. The
restatement lives here, next to the other plugin restatements of tests/, rather than in oracle/mppi_oracle.cpp: the oracle
is a yardstick of the existing pairs and stays as it is. `dtype` selects
float32 (the restatement) or float64 (its precision check). Test infrastructure only."""
import math

import numpy as np

VEL_X, YAW, POS_X, POS_Y, STEER_ANGLE, BRAKE_STATE, ROLL, PITCH, STEER_ANGLE_RATE = range(9)
# covariance entries from index 9: POS_X, POS_Y, YAW, VEL_X, POS_X_Y, POS_X_YAW, POS_X_VEL_X, POS_Y_YAW, POS_Y_VEL_X,
# YAW_VEL_X (racer_dubins_elevation.cuh:29-38)
UNC0 = 9
S, C, O = 19, 2, 28
O_ACCEL_X = 13


class Params:
    """The fields of mppib_racer_dubins_elevation_dyn_params as Python floats."""

    def __init__(self, blob):
        for name, _ in blob._fields_:
            if name == "lim":
                self.rng_lo = [blob.lim.rng_lo[i] for i in range(C)]
                self.rng_hi = [blob.lim.rng_hi[i] for i in range(C)]
            else:
                v = getattr(blob, name)
                setattr(self, name, list(v) if hasattr(v, "__len__") else v)


def normalize_angle(a, dtype):
    """angle_utils::normalizeAngle: (a + pi) mod 2 pi shifted back into (-pi, pi]."""
    pi = dtype(math.pi)
    r = dtype(math.fmod(float(dtype(a + pi)), float(dtype(2 * pi))))
    return dtype(r + pi) if r <= 0 else dtype(r - pi)


def _index(vx):
    return int(0.2 < abs(vx) <= 3.0) + int(abs(vx) > 3.0) * 2


def step(p: Params, x, u, dt, body="device", dtype=np.float32, map_blob=None):
    """Returns (next_state, state_der, output) of one step."""
    f = dtype
    x = np.asarray(x, dtype)
    u = np.asarray(u, dtype)
    dt = f(dt)
    xd = np.zeros(S, dtype)
    xn = np.zeros(S, dtype)
    dev = body == "device"
    nrm = (lambda a: normalize_angle(a, dtype)) if dev else (lambda a: a)
    vx = x[VEL_X]
    idx = _index(vx)
    enable_brake = u[0] < 0
    # delay, racer_dubins.cu:281-293 (host :306-319, the same)
    err = f(enable_brake * -u[0] - x[BRAKE_STATE])
    xd[BRAKE_STATE] = min(max(f((err > 0) * err * f(p.brake_delay_constant) + (err < 0) * err * f(p.brake_delay_constant_neg)),
                              f(-p.max_brake_rate_neg)), f(p.max_brake_rate_pos))
    # steering, racer_dubins.cu:296-304 (host :321-330, the same)
    xd[STEER_ANGLE] = max(min(f((u[1] * f(p.steer_command_angle_scale) - x[STEER_ANGLE]) * f(p.steering_constant)),
                              f(p.max_steer_rate)), f(-p.max_steer_rate))
    # acceleration
    brake_state = min(max(x[BRAKE_STATE], f(0)), f(0.25))
    c_t, c_b, c_v = f(p.c_t[idx]), f(p.c_b[idx]), f(p.c_v[idx])
    throttle = c_t * u[0]
    brake = c_b * brake_state * (f(-1) if vx >= 0 else f(1))
    if abs(vx) <= 0.2:
        throttle = c_t * max(f(u[0] - f(p.low_min_throttle)), f(0))
        brake = c_b * brake_state * -vx
    a = f((not enable_brake) * throttle * f(p.gear_sign) + brake - c_v * vx + f(p.c_0))
    a = min(max(a, f(-p.clamp_ax)), f(p.clamp_ax))
    if abs(x[PITCH]) < f(math.pi / 2):
        a = f(a - f(p.gravity) * f(np.sin(nrm(x[PITCH]))))
    xd[VEL_X] = a
    delta = f(x[STEER_ANGLE] / f(p.steer_angle_scale))
    xd[YAW] = f((vx / f(p.wheel_base)) * f(np.tan(nrm(delta))))
    yaw = nrm(x[YAW])
    sy, cy = f(np.sin(yaw)), f(np.cos(yaw))
    xd[POS_X] = vx * cy
    xd[POS_Y] = vx * sy
    # updateState
    xn[:6] = x[:6] + xd[:6] * dt
    xn[YAW] = normalize_angle(xn[YAW], dtype)
    xn[STEER_ANGLE] = max(min(xn[STEER_ANGLE], f(p.max_steer_angle)), f(-p.max_steer_angle))
    xn[STEER_ANGLE_RATE] = xd[STEER_ANGLE]
    brake_hi = f(1) if dev else f(-p.rng_lo[0])
    xn[BRAKE_STATE] = min(max(xn[BRAKE_STATE], f(0)), brake_hi)
    _uncertainty(p, x, xd, xn, dt, idx, brake_state, delta, sy, cy, dtype)
    roll, pitch, height = f(0), f(0), f(0)
    if map_blob is not None:
        roll, pitch, height = _settle(map_blob, xn[YAW], xn[POS_X], xn[POS_Y], x[ROLL], x[PITCH], dtype)
    xn[ROLL], xn[PITCH] = roll, pitch
    y = np.zeros(O, dtype)
    y[0], y[2], y[3], y[4], y[5] = xn[VEL_X], xn[POS_X], xn[POS_Y], height, xn[YAW]
    y[6], y[7], y[8], y[9] = xn[ROLL], xn[PITCH], xn[STEER_ANGLE], xn[STEER_ANGLE_RATE]
    y[10:13] = np.nan
    y[O_ACCEL_X], y[15], y[16] = xd[VEL_X], xd[YAW], abs(xn[VEL_X])
    y[17:27] = xn[UNC0:UNC0 + 10]
    return xn, xd, y


def _uncertainty(p, x, xd, xn, dt, idx, brake_state, delta, sy, cy, dtype):
    """computeUncertaintyPropagation (racer_dubins_elevation.cu:662-741) over (VEL_X, YAW, POS_X, POS_Y)."""
    f = dtype
    vx = x[VEL_X]
    tan_d, cos2 = f(np.tan(delta)), f(np.cos(delta)) ** 2
    wb = f(p.wheel_base)
    A = np.zeros((4, 4), dtype)
    A[0, 0] = -f(p.c_v[idx]) - f(p.K_vel_x) - (f(1) if idx == 0 else f(0)) * f(p.c_b[0]) * brake_state
    A[0, 2], A[0, 3] = -f(p.K_x) * cy, -f(p.K_x) * sy
    A[1, 0] = tan_d / wb
    A[1, 1] = -abs(vx) * f(p.K_yaw) / (wb * cos2)
    A[1, 2] = vx * f(p.K_y) * sy / (wb * cos2)
    A[1, 3] = -vx * f(p.K_y) * cy / (wb * cos2)
    A[2, 0], A[2, 1] = cy, -sy * vx
    A[3, 0], A[3, 1] = sy, cy * vx
    s = x[UNC0:UNC0 + 10]
    Sg = np.array([[s[3], s[9], s[6], s[8]],
                   [s[9], s[2], s[5], s[7]],
                   [s[6], s[5], s[0], s[4]],
                   [s[8], s[7], s[4], s[1]]], dtype)
    Ad = (np.eye(4, dtype=dtype) + A * dt).astype(dtype)
    Sg = (Ad @ Sg @ Ad.T).astype(dtype)
    abs_vx = abs(vx)
    side = abs_vx * abs_vx * tan_d / wb + f(p.gravity) * f(np.sin(x[ROLL]))
    q11 = abs(f(p.Q_y_f) * abs(side) * max(f(abs_vx - 2), f(0)))
    Q = np.zeros((4, 4), dtype)
    Q[0, 0] = f(p.Q_x_acc) * abs(xd[VEL_X]) + f(p.Q_x_v[idx]) * abs_vx
    Q[1, 1] = abs_vx * (f(p.Q_omega_steering) * abs(delta) + f(p.Q_omega_v))
    Q[2, 2] = q11 * sy * sy
    Q[2, 3] = Q[3, 2] = -q11 * sy * cy
    Q[3, 3] = q11 * cy * cy
    Sg = Sg + Q * dt
    xn[UNC0:UNC0 + 10] = [Sg[2, 2], Sg[3, 3], Sg[1, 1], Sg[0, 0], Sg[3, 2], Sg[2, 1], Sg[2, 0], Sg[3, 1], Sg[3, 0],
                          Sg[1, 0]]


def _settle(map_blob, yaw, px, py, roll, pitch, dtype):
    """RACER::computeStaticSettling through the CPU oracle's own restatement (oracle/mppi_oracle.cpp: orc_static_settling),
    not the library under test."""
    import oracle
    r, p_, h = oracle.static_settling(map_blob, float(yaw), float(px), float(py), float(roll), float(pitch))
    return dtype(r), dtype(p_), dtype(h)


def grad(p: Params, x, u, dtype=np.float32):
    """computeGrad (racer_dubins_elevation.cu:257-334) as written; A [19][19], B [19][2]. The reference (and the host
    twin) evaluate 1 / cos^2 in double; the device and this restatement in float."""
    f = dtype
    x, u = np.asarray(x, dtype), np.asarray(u, dtype)
    A = np.zeros((S, S), dtype)
    B = np.zeros((S, C), dtype)
    eps = f(0.01)
    enable_brake = u[0] < 0
    vx = x[VEL_X]
    idx = _index(vx)
    A[VEL_X, VEL_X] = -f(p.c_v[idx])
    if abs(vx) < 0.2:
        A[VEL_X, BRAKE_STATE] = f(p.c_b[idx]) * -vx
    else:
        A[VEL_X, BRAKE_STATE] = f(p.c_b[idx]) * (f(-1) if vx >= 0 else f(1))
    delta = f(x[STEER_ANGLE] / f(p.steer_angle_scale))
    wb = f(p.wheel_base)
    A[YAW, VEL_X] = (f(1) / wb) * f(np.tan(delta))
    A[YAW, STEER_ANGLE] = (vx / wb) * (f(1) / f(np.cos(delta)) ** 2) / f(p.steer_angle_scale)
    sy, cy = f(np.sin(x[YAW])), f(np.cos(x[YAW]))
    A[POS_X, VEL_X], A[POS_X, YAW] = cy, -sy * vx
    A[POS_Y, VEL_X], A[POS_Y, YAW] = sy, cy * vx
    steer_dot = f((u[1] * f(p.steer_command_angle_scale) - x[STEER_ANGLE]) * f(p.steering_constant))
    a44 = f(0) if (steer_dot - eps < -p.max_steer_rate or steer_dot + eps > p.max_steer_rate) else -f(p.steering_constant)
    A[STEER_ANGLE, STEER_ANGLE] = max(min(a44, f(p.max_steer_rate)), f(-p.max_steer_rate))
    A[VEL_X, PITCH] = -f(p.gravity) * f(np.cos(x[PITCH]))
    brake_dot = f((enable_brake * -u[0] - x[BRAKE_STATE]) * f(p.brake_delay_constant))
    if brake_dot - eps < -p.max_brake_rate_neg or brake_dot + eps > p.max_brake_rate_pos:
        A[BRAKE_STATE, BRAKE_STATE] = 0
    else:
        A[BRAKE_STATE, BRAKE_STATE] = -f(p.brake_delay_constant)
    B[STEER_ANGLE, 1] = f(p.steer_command_angle_scale) * f(p.steering_constant)
    B[VEL_X, 0] = f(p.c_t[idx]) * f(p.gear_sign) * f(not enable_brake)
    if (x[BRAKE_STATE] < -p.rng_lo[0] and brake_dot < 0) or (x[BRAKE_STATE] > 0 and brake_dot > 0):
        B[BRAKE_STATE, 0] = -f(p.brake_delay_constant) * f(enable_brake)
    return A, B


def f_ddp(p: Params, x, u, dtype=np.float32):
    """f(x, u) of DDP: the step's six derivative rows, the rest zero (plugins/dynamics.cuh: computeDynamics)."""
    _, xd, _ = step(p, x, u, 0.01, "device", dtype)
    return xd
