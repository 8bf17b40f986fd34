"""A numpy restatement of RacerSuspension (dynamics/racer_suspension/racer_suspension.cu), the rigid-body RACER vehicle,
in float32 or float64, vectorised over samples: x [..., 14], u [..., 2].

  deriv        computeStateDeriv (:93-298) on the plane z = 0 with normal (0, 0, 1), outputs of x, and optionally the 3x3
               omegaJacobian as written (f_r_B_i_Jac = f_r_C_i_Jac, :215)
  host_step    the host step (:31-45): the body rates by (I - dt J)^-1 dt w_dot, the rest explicit, then q / |q|
  device_step  the device step (:300-306, :55-75): explicit Euler on all 14 states, then q / |q|
  rollout      a K1 rollout through device_step with RacerQuadraticCost at this model's output indices, and for each sample
               how close its trajectory came to the body's three switches

The one deviation from the reference: outputs 1 and 2 hold the base link's body y / z velocity (the reference writes all
three components into output 0). Outputs 23..25 are 0.
"""
import numpy as np

S, C, O = 14, 2, 26
P_I_Z, Q_W, V_I_X, OMEGA_B_X, STEER_ANGLE = 2, 3, 7, 10, 13
O_VEL_X, O_POS_Y, O_YAW, O_ROLL, O_PITCH, O_STEER = 0, 4, 6, 7, 8, 9


def params(blob):
    """The blob's fields (host.RacerRigidSuspensionDynParams) as Python floats / lists."""
    b = blob
    return {
        "rng_lo": [b.lim.rng_lo[i] for i in range(2)], "rng_hi": [b.lim.rng_hi[i] for i in range(2)],
        "mass": b.mass, "wheel_base": b.wheel_base, "width": b.width, "gravity": b.gravity,
        "k_s": list(b.k_s), "c_s": list(b.c_s), "l_0": list(b.l_0), "cg": list(b.cg_pos_wrt_base_link),
        "wheel_pos": [list(b.wheel_pos_wrt_base_link[i]) for i in range(4)], "J": [b.Jxx, b.Jyy, b.Jzz],
        "mu": b.mu, "v_slip": b.v_slip, "c_t": b.c_t, "c_b": b.c_b, "c_v": b.c_v, "c_0": b.c_0,
        "steering_constant": b.steering_constant, "steer_command_angle_scale": b.steer_command_angle_scale,
    }


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def _rot(q, f):
    """Eigen's Quaternion::toRotationMatrix, [..., 3, 3]."""
    w, x, y, z = (q[..., i] for i in range(4))
    two = f(2)
    tx, ty, tz = two * x, two * y, two * z
    twx, twy, twz, txx, txy, txz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    one = f(1)
    return np.stack([np.stack([one - (tyy + tzz), txy - twz, txz + twy], -1),
                     np.stack([txy + twz, one - (txx + tzz), tyz - twx], -1),
                     np.stack([txz - twy, tyz + twx, one - (txx + tyy)], -1)], -2)


def _mv(R, v):
    return np.einsum("...ij,...j->...i", R, v)


def _mtv(R, v):
    return np.einsum("...ji,...j->...i", R, v)


def deriv(p, x, u, dtype=np.float64, jac=False):
    """(xdot, y[, omegaJacobian [..., 3, 3]]) and a dict of switch margins (see rollout)."""
    f = dtype
    x, u = np.asarray(x).astype(f), np.asarray(u).astype(f)
    R = _rot(x[..., 3:7], f)
    pI, v, w = x[..., 0:3], x[..., 7:10], x[..., 10:13]
    tan_delta = np.tan(x[..., STEER_ANGLE])
    vb = _mtv(R, v)
    throttle, brake = np.maximum(f(0), u[..., 0]), np.maximum(f(0), -u[..., 0])
    acc = f(p["c_t"]) * throttle - np.copysign(f(p["c_b"]) * brake, vb[..., 0]) - f(p["c_v"]) * vb[..., 0] + f(p["c_0"])
    prop = f(p["mass"]) * acc
    mu_, v_slip = f(p["mu"]), f(p["v_slip"])
    f_B = np.zeros(x.shape[:-1] + (3,), f)
    tau_B = np.zeros_like(f_B)
    tau_jac = np.zeros(x.shape[:-1] + (3, 3), f)
    y = np.zeros(x.shape[:-1] + (O,), f)
    weight = f(p["mass"]) / f(4) * -f(p["gravity"])
    margin = {"spring": np.full(x.shape[:-1], np.inf), "slip": np.full(x.shape[:-1], np.inf)}
    n = R[..., 2, :]  # R^T (0, 0, 1)
    eye = np.eye(3, dtype=f)
    for i in range(4):
        pb = (np.array(p["wheel_pos"][i], f) - np.array(p["cg"], f)).astype(f)
        pw = pI + _mv(R, np.broadcast_to(pb, pI.shape))
        pdot = v + _mv(R, _cross(w, np.broadcast_to(pb, w.shape)))
        pdot_jac = np.stack([_mv(R, np.broadcast_to(_cross(eye[k], pb), pI.shape)) for k in range(3)], -1)
        f_k = -f(p["k_s"][i]) * (pw[..., 2] - f(p["l_0"][i])) - f(p["c_s"][i]) * pdot[..., 2]
        margin["spring"] = np.minimum(margin["spring"], np.abs(f_k.astype(np.float64)) / float(weight))
        lift = f_k < 0
        f_k_jac = -f(p["c_s"][i]) * pdot_jac[..., 2, :]
        f_k = np.where(lift, f(0), f_k)
        f_k_jac = np.where(lift[..., None], f(0), f_k_jac)
        if i == 0:
            delta = np.arctan(f(p["wheel_base"]) * tan_delta / (f(p["wheel_base"]) - tan_delta * f(p["width"]) / f(2)))
        elif i == 1:
            delta = np.arctan(f(p["wheel_base"]) * tan_delta / (f(p["wheel_base"]) + tan_delta * f(p["width"]) / f(2)))
        else:
            delta = np.zeros_like(tan_delta)
        wd = np.stack([np.cos(delta), np.sin(delta), np.zeros_like(delta)], -1)
        s = _cross(n, wd)
        s = s / np.sqrt(np.sum(s * s, -1, keepdims=True))
        t = _cross(s, n)
        pdc = np.concatenate([pdot[..., :2], np.zeros_like(pdot[..., 2:])], -1)
        v_s = np.sum(s * _mtv(R, pdc), -1)
        margin["slip"] = np.minimum(margin["slip"], np.abs(np.abs(v_s.astype(np.float64)) - float(v_slip)) / float(v_slip))
        pdc_jac = np.concatenate([pdot_jac[..., :2, :], np.zeros_like(pdot_jac[..., 2:, :])], -2)
        v_s_jac = np.einsum("...j,...jk->...k", s, np.einsum("...ji,...jk->...ik", R, pdc_jac))
        mu_s = v_s / v_slip * mu_
        sat_hi, sat_lo = mu_s > mu_, mu_s < -mu_
        dmu = np.where(sat_hi | sat_lo, f(0), mu_ / v_slip)
        mu_s = np.where(sat_hi, mu_, np.where(sat_lo, -mu_, mu_s))
        f_n = f_k
        f_s = -mu_s * f_n
        f_t = np.maximum(-mu_ * f_n, np.minimum(prop / f(4), mu_ * f_n))
        ft_jac = np.where((prop / f(4) > mu_ * f_n)[..., None], mu_ * f_k_jac,
                          np.where((prop / f(4) < -mu_ * f_n)[..., None], -mu_ * f_k_jac, f(0)))
        fs_jac = (-f_n * dmu)[..., None] * v_s_jac - mu_s[..., None] * f_k_jac
        fc_jac = np.stack([ft_jac, fs_jac, f_k_jac], -2)  # rows t, s, n
        force = t * f_t[..., None] + s * f_s[..., None] + n * f_n[..., None]
        dc = np.stack([pw[..., 0] - pI[..., 0], pw[..., 1] - pI[..., 1], -pI[..., 2]], -1)
        pc = _mtv(R, dc)
        f_B = f_B + force
        tau_B = tau_B + _cross(pc, force)
        tau_jac = tau_jac - np.stack([_cross(fc_jac[..., :, k], pc) for k in range(3)], -1)
        y[..., 11 + 2 * i] = pw[..., 0]
        y[..., 12 + 2 * i] = pw[..., 1]
        y[..., 19 + i] = np.sqrt(np.sum(force * force, -1))
    xd = np.zeros(x.shape, f)
    xd[..., 0:3] = v
    xd[..., 7:10] = (f(1) / f(p["mass"])) * _mv(R, f_B)
    xd[..., 9] += f(p["gravity"])
    qw, qx, qy, qz = (x[..., 3 + i] for i in range(4))
    h = f(0.5)
    xd[..., 3] = h * (-qx * w[..., 0] - qy * w[..., 1] - qz * w[..., 2])
    xd[..., 4] = h * (qw * w[..., 0] + qy * w[..., 2] - qz * w[..., 1])
    xd[..., 5] = h * (qw * w[..., 1] + qz * w[..., 0] - qx * w[..., 2])
    xd[..., 6] = h * (qw * w[..., 2] + qx * w[..., 1] - qy * w[..., 0])
    J = np.array(p["J"], f)
    Jinv = np.array([1.0 / j for j in p["J"]], np.float64).astype(f)
    Jw = J * w
    xd[..., 10:13] = Jinv * (_cross(Jw, w) + tau_B)
    xd[..., STEER_ANGLE] = f(p["steering_constant"]) * (u[..., 1] / f(p["steer_command_angle_scale"]) - x[..., STEER_ANGLE])
    pbl = -np.array(p["cg"], f)
    y[..., 0:3] = vb + _cross(w, np.broadcast_to(pbl, w.shape))
    y[..., 3:6] = pI + _mv(R, np.broadcast_to(pbl, pI.shape))
    y[..., O_ROLL] = np.arctan2(f(2) * qz * qy + f(2) * qw * qx, qw * qw + qz * qz - qy * qy - qx * qx)
    y[..., O_PITCH] = -np.arcsin(np.clip(f(-2) * qw * qy + f(2) * qx * qz, f(-1), f(1)))
    y[..., O_YAW] = np.arctan2(f(2) * qy * qx + f(2) * qz * qw, qw * qw + qx * qx - qy * qy - qz * qz)
    y[..., O_STEER] = x[..., STEER_ANGLE]
    y[..., 10] = xd[..., STEER_ANGLE]
    # an exact zero (a car at rest, upright: v = 0 and R = I exactly) is +0 in every precision, so only a non-zero vel_x
    # near 0 can take copysign's other branch
    vx = vb[..., 0].astype(np.float64)
    margin["vel_x"] = np.where((brake > 0) & (vx != 0), np.abs(vx), np.inf)
    if not jac:
        return xd, y, margin
    Jwxw_jac = np.stack([_cross(J[k] * eye[k], w) - _cross(np.broadcast_to(eye[k], w.shape), Jw) for k in range(3)], -1)
    return xd, y, margin, Jinv[:, None] * (Jwxw_jac + tau_jac)


def _renormalise(xn):
    q = xn[..., 3:7]
    xn[..., 3:7] = q / np.sqrt(np.sum(q * q, -1, keepdims=True))
    return xn


def device_step(p, x, u, dt, dtype=np.float64):
    """(x_next, xdot, y of x, margins)"""
    xd, y, margin = deriv(p, x, u, dtype)
    xn = np.asarray(x).astype(dtype) + xd * dtype(dt)
    return _renormalise(xn), xd, y, margin


def host_step(p, x, u, dt, dtype=np.float64):
    xd, y, _, J = deriv(p, x, u, dtype, jac=True)
    f = dtype
    xn = np.asarray(x).astype(f) + xd * f(dt)
    M = np.eye(3, dtype=f) - f(dt) * J
    dw = np.einsum("...ij,...j->...i", np.linalg.inv(M.astype(np.float64)).astype(f) * f(dt), xd[..., 10:13])
    xn[..., 10:13] = np.asarray(x).astype(f)[..., 10:13] + dw
    return _renormalise(xn), xd, y


def step_cost(cp, y, f=np.float64):
    """RacerQuadraticCost at this model's indices (discount 1)."""
    dv = y[..., O_VEL_X] - f(cp.desired_speed)
    a = y[..., O_YAW] - f(cp.desired_yaw)
    dyaw = np.mod(a + np.pi, 2 * np.pi) - np.pi
    dy = y[..., O_POS_Y] - f(cp.desired_y)
    st = y[..., O_STEER]
    return (f(cp.speed_coeff) * dv * dv + f(cp.yaw_coeff) * dyaw * dyaw + f(cp.lateral_coeff) * dy * dy +
            f(cp.steer_coeff) * st * st)


def rollout(p, cp, x0, controls, dt, dtype=np.float64):
    """K1's rollout of controls [N, T, 2] (clamped to the control ranges) from x0 [S] or [N, S]: trajectory costs
    sum_t cost(y_t) / T, outputs [N, T, O], and per sample the smallest margin to each switch over the horizon:
    'spring' |f_k| / (m g / 4) of the spring clamp, 'slip' ||v_s| - v_slip| / v_slip of the Stribeck saturation, 'vel_x'
    |vel_x| where the brake is applied and vel_x is not exactly 0 (copysign's sign)."""
    N, T = controls.shape[:2]
    lo, hi = np.array(p["rng_lo"], np.float32), np.array(p["rng_hi"], np.float32)
    x = np.broadcast_to(np.asarray(x0, dtype), (N, S)).copy()
    total = np.zeros(N, np.float64)
    Y = np.zeros((N, T, O), dtype)
    worst = {k: np.full(N, np.inf) for k in ("spring", "slip", "vel_x")}
    for t in range(T):
        u = np.clip(controls[:, t], lo, hi)
        x, _, y, margin = device_step(p, x, u, dt, dtype)
        Y[:, t] = y
        total += step_cost(cp, y, dtype)
        for k in worst:
            worst[k] = np.minimum(worst[k], margin[k])
    return total / T, Y, worst
