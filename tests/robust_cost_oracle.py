"""Float32 restatement of the two robust costs and of the rollouts that use them — test infrastructure for
tests/test_robust_costs.py.

  di_robust_cost(p, y, device)   double_integrator_robust_cost.cu:9-39 (device: steep boundary 0.5, steep cost 0.5 * crash)
                                 and :41-69 (host: 0.75, 0.1 * crash)
  ar_robust_cost(p, tex, y)      ar_robust_cost.cu:13-132, device form: a point-sampled texel (floor of the texel
                                 coordinate, clamped), float32 sin / cos, the reference's double operations in float64
  di_rollout / di_rmppi_rollout  the double integrator's rollouts (di_dynamics.cu:14-22, x + xdot dt) with per-sample costs
                                 as the kernels form them: sum over t of the state cost, divided by T

Everything is vectorised over samples: y is [..., O].
"""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32


def _fma(a, b, c):
    """a * b + c rounded once (nvcc contracts these); float64 holds the float32 product exactly."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def _lin_interp(x, x_min, x_max, y_min, y_max):
    x_min, x_max, y_min, y_max = f32(x_min), f32(x_max), f32(y_min), f32(y_max)
    return _fma((x - x_min) / (x_max - x_min), (y_max - y_min), y_min)


def di_robust_cost(p, y, device: bool = True) -> np.ndarray:
    y = np.asarray(y, f32)
    s0, s1, s2, s3 = (y[..., i] for i in range(4))
    radial = _fma(s0, s0, s1 * s1)
    vel = np.sqrt(_fma(s2, s2, s3 * s3))
    mom = _fma(s0, s3, -(s1 * s2))
    r_in, r_out = np.sqrt(f32(p.inner_path_radius2)), np.sqrt(f32(p.outer_path_radius2))
    r_center = (r_in + r_out) / f32(2)
    norm = np.abs(np.sqrt(radial) - r_center) / ((r_out - r_in) * f32(0.5))
    crash = f32(p.crash_cost)
    if device:
        b, steep = f32(0.5), f32(0.5 * float(crash))
    else:
        b, steep = f32(0.75), f32(0.1 * float(crash))
    cost = np.where(norm <= b, _lin_interp(norm, 0, b, 0, steep),
                    np.where(norm <= 1.0, _lin_interp(norm, b, 1, steep, crash), crash)).astype(f32)
    vc = f32(p.velocity_cost)
    cost = _fma(vc, (vel - f32(p.velocity_desired)) ** 2, cost)
    cost = _fma(vc, (mom - f32(p.angular_momentum_desired)) ** 2, cost)
    return cost


def texel(p, tex, x, y):
    """Point-sampled float4 under world points (x, y): texture coordinate u * width, floored and clamped."""
    x, y = np.asarray(x, f32), np.asarray(y, f32)
    u = f32(p.r_c1[0]) * x + f32(p.r_c2[0]) * y + f32(p.trs[0])
    v = f32(p.r_c1[1]) * x + f32(p.r_c2[1]) * y + f32(p.trs[1])
    cx = np.clip(np.floor(u.astype(np.float64) * p.map_width), 0, p.map_width - 1).astype(np.int64)
    cy = np.clip(np.floor(v.astype(np.float64) * p.map_height), 0, p.map_height - 1).astype(np.int64)
    return tex[cy, cx]


def texel_coords(p, x, y):
    """Continuous texel coordinates (float64) of world points: their distance to the nearest integer is the distance to a
    texel edge."""
    u = p.r_c1[0] * np.asarray(x, np.float64) + p.r_c2[0] * np.asarray(y, np.float64) + p.trs[0]
    v = p.r_c1[1] * np.asarray(x, np.float64) + p.r_c2[1] * np.asarray(y, np.float64) + p.trs[1]
    return u * p.map_width, v * p.map_height


def ar_stabilizing_cost(p, y) -> np.ndarray:
    y = np.asarray(y, f32)
    vx, vy, roll = y[..., 4], y[..., 5], y[..., 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        slip = np.where(np.abs(vx.astype(np.float64)) < 0.001, f32(0),
                        np.abs(np.arctan((vy / np.abs(vx)).astype(np.float64)).astype(f32))).astype(f32)
    m = f32(p.max_slip_ang)
    slip_val = np.minimum(f32(1), slip / m)
    alpha = ((slip_val.astype(np.float64) - 0.75) / (1.0 - 0.75)).astype(f32)
    pen = np.where(slip.astype(np.float64) >= 0.75 * float(m), alpha * f32(p.crash_coeff), f32(0)).astype(f32)
    pen = np.where(np.abs(roll.astype(np.float64)) >= math.pi / 2, f32(p.crash_coeff), pen).astype(f32)
    return _fma(f32(p.slip_coeff), slip, pen)


def ar_costmap_cost(p, tex, y) -> np.ndarray:
    y = np.asarray(y, f32)
    yaw = y[..., 2]
    cs, sn = np.cos(yaw).astype(f32), np.sin(yaw).astype(f32)
    xf, yf = _fma(f32(p.front_d), cs, y[..., 0]), _fma(f32(p.front_d), sn, y[..., 1])
    xb, yb = _fma(f32(p.back_d), cs, y[..., 0]), _fma(f32(p.back_d), sn, y[..., 1])
    front, back = texel(p, tex, xf, yf), texel(p, tex, xb, yb)
    bt = f32(p.boundary_threshold)
    cv = np.minimum(f32(1), np.maximum(front[..., 0], back[..., 0]))
    alpha = ((cv - bt).astype(np.float64) / (1.0 - float(bt))).astype(f32)
    cost = np.where(cv >= bt, alpha * f32(p.crash_coeff), f32(0)).astype(f32)
    cost = np.where(front[..., 1] > f32(p.track_slop), _fma(f32(p.track_coeff), front[..., 1], cost), cost).astype(f32)
    target = front[..., 2] if p.desired_speed == -1 else f32(p.desired_speed)
    cost = _fma(f32(p.speed_coeff), np.abs(y[..., 4] - target), cost)
    cost = _fma(f32(p.heading_coeff), np.abs(np.sin(yaw).astype(f32) + front[..., 3]), cost)
    return cost


def ar_robust_cost(p, tex, y) -> np.ndarray:
    c = ar_stabilizing_cost(p, y) + ar_costmap_cost(p, tex, y)
    return np.where((c > f32(1e16)) | np.isnan(c), f32(1e16), c).astype(f32)


def ar_on_discontinuity(p, y, texel_tol=2e-3, thr_tol=1e-4) -> np.ndarray:
    """Where the robust cost jumps: a wheel within texel_tol of a texel edge, |roll| at pi/2, |vx| at 0.001, or the front
    texel's track value at track_slop (the last is judged on the texel the point falls in)."""
    y = np.asarray(y, np.float64)
    cs, sn = np.cos(y[..., 2]), np.sin(y[..., 2])
    edge = np.zeros(y.shape[:-1], bool)
    for d in (p.front_d, p.back_d):
        u, v = texel_coords(p, y[..., 0] + d * cs, y[..., 1] + d * sn)
        edge |= (np.abs(u - np.round(u)) < texel_tol) | (np.abs(v - np.round(v)) < texel_tol)
    roll = np.abs(np.abs(y[..., 3]) - math.pi / 2) < thr_tol
    vx = np.abs(np.abs(y[..., 4]) - 0.001) < thr_tol * 1e-2
    return edge | roll | vx


def ar_track_slop_crossing(p, tex, y) -> np.ndarray:
    y = np.asarray(y, f32)
    xf = y[..., 0] + f32(p.front_d) * np.cos(y[..., 2]).astype(f32)
    yf = y[..., 1] + f32(p.front_d) * np.sin(y[..., 2]).astype(f32)
    return np.abs(texel(p, tex, xf, yf)[..., 1] - f32(p.track_slop)) < 1e-6


def di_step(x, u, dt):
    """di_dynamics.cu:14-22 and dynamics.cu:118-129: x + xdot dt with xdot = (x2, x3, u0, u1)."""
    xdot = np.concatenate([x[..., 2:4], u], axis=-1)
    return _fma(xdot, f32(dt), x)


def di_rollout(p, x0, controls, dt, device=True) -> np.ndarray:
    """controls [N][T][2] (constrained). Per-sample cost sum_t c(y_t) / T, y_t the state after step t."""
    N, T, _ = controls.shape
    x = np.broadcast_to(np.asarray(x0, f32), (N, 4)).copy()
    run = np.zeros(N, f32)
    for t in range(T):
        x = di_step(x, controls[:, t], dt)
        run = (run + di_robust_cost(p, x, device)).astype(f32)
    return (run / f32(T)).astype(f32)


def di_rmppi_rollout(p, x0, samples, gains, dt, value_func_threshold, nominal_idx=0):
    """The RMPPI rollout (rmppi_kernels.cu:665-866) without likelihood-ratio or feedback costs (the sampler's
    control_cost_coeff is 0): x0 [2][S], samples [2][N][T][C] unconstrained (the double integrator has no limits),
    gains [T][S][C] or None. Returns costs [2][N]."""
    real_idx = 1 - nominal_idx
    _, N, T, _ = samples.shape
    xr = np.broadcast_to(np.asarray(x0[real_idx], f32), (N, 4)).copy()
    xn = np.broadcast_to(np.asarray(x0[nominal_idx], f32), (N, 4)).copy()
    run_r = np.zeros(N, f32)
    run_n = np.zeros(N, f32)
    for t in range(T):
        ur = samples[real_idx, :, t].astype(f32)
        if gains is not None:
            e = (xr - xn).astype(np.float64)
            ur = (ur + (e @ gains[t].astype(np.float64)).astype(f32)).astype(f32)
        xr = di_step(xr, ur, dt)
        xn = di_step(xn, samples[nominal_idx, :, t].astype(f32), dt)
        run_r = (run_r + di_robust_cost(p, xr)).astype(f32)
        run_n = (run_n + di_robust_cost(p, xn)).astype(f32)
    run_r = (run_r / f32(T)).astype(f32)
    run_n = (run_n / f32(T)).astype(f32)
    nom = (f32(0.5) * run_n + f32(0.5) * np.maximum(np.minimum(run_r, f32(value_func_threshold)), run_n)).astype(f32)
    out = np.zeros((2, N), f32)
    out[nominal_idx], out[real_idx] = nom, run_r
    return out
