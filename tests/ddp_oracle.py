"""CPU restatement of the reference's DDP feedback solve, the yardstick of the device kernel (csrc/ddp_kernel.cuh).

DDPFeedback::computeFeedback (feedback_controllers/DDP/ddp.cu:80-118) runs DDP::run (ddp/ddp.h:56-168) with the tracking
costs of ddp/ddp_tracking_costs.h. Restated here in float32 numpy, with the model's state derivative f and its analytic
Jacobian computeGrad for the four models that have one (cartpole_dynamics.cu:10-45, di_dynamics.cu:24-34, the exact
derivative of the quadrotor's f, ar_nn_model.cu:63-86 + fnn_helper.cu:312-347). Test infrastructure only.

Every function takes `dtype` so the float64 central differences of the tests can use the same f."""
import numpy as np

CARTPOLE, DOUBLE_INTEGRATOR, AUTORALLY_NN, QUADROTOR = 0, 1, 2, 4
GRAVITY = 9.81


class Model:
    """Parameters of one dynamics model, read from the host mirror's plugin object."""

    def __init__(self, dyn):
        self.id = dyn.DYN_ID
        self.S, self.C = dyn.STATE_DIM, dyn.CONTROL_DIM
        p = dyn.params
        self.u_lo = np.array([p.lim.rng_lo[i] for i in range(self.C)], np.float32)
        self.u_hi = np.array([p.lim.rng_hi[i] for i in range(self.C)], np.float32)
        if self.id == CARTPOLE:
            self.mc, self.mp, self.l, self.g = p.cart_mass, p.pole_mass, p.pole_length, p.gravity
        elif self.id == QUADROTOR:
            self.tau = np.array([p.tau_roll, p.tau_pitch, p.tau_yaw])
            self.mass = p.mass
        elif self.id == AUTORALLY_NN:
            th = np.asarray(dyn.nn_theta, np.float64)
            self.W1, self.b1 = th[:192].reshape(32, 6), th[192:224]
            self.W2, self.b2 = th[224:1248].reshape(32, 32), th[1248:1280]
            self.W3, self.b3 = th[1280:1408].reshape(4, 32), th[1408:1412]


def f(m: Model, x, u, dtype=np.float32):
    """state_der of one model step (ddp_model_wrapper.h:68-81)."""
    x, u = np.asarray(x, dtype), np.asarray(u, dtype)
    d = np.zeros(m.S, dtype)
    if m.id == CARTPOLE:
        mc, mp, l, g = (dtype(v) for v in (m.mc, m.mp, m.l, m.g))
        s, c, td, F = np.sin(x[2]), np.cos(x[2]), x[3], u[0]
        den = mc + mp * s * s
        d[0], d[2] = x[1], td
        d[1] = (F + mp * s * (l * td * td + g * c)) / den
        d[3] = (-F * c - mp * l * td * td * c * s - (mc + mp) * g * s) / (l * den)
    elif m.id == DOUBLE_INTEGRATOR:
        d[0], d[1], d[2], d[3] = x[2], x[3], u[0], u[1]
    elif m.id == QUADROTOR:
        v, q, w = x[3:6], x[6:10], x[10:13]
        a = u[3] / dtype(m.mass)
        d[0:3] = v
        d[3] = a * 2 * (q[1] * q[3] + q[0] * q[2])
        d[4] = a * 2 * (q[2] * q[3] - q[0] * q[1])
        d[5] = a * (q[0] ** 2 - q[1] ** 2 - q[2] ** 2 + q[3] ** 2) - dtype(GRAVITY)
        half = dtype(0.5)
        d[6] = half * (-w[0] * q[1] - w[1] * q[2] - w[2] * q[3])
        d[7] = half * (w[0] * q[0] - w[1] * q[3] + w[2] * q[2])
        d[8] = half * (w[0] * q[3] + w[1] * q[0] - w[2] * q[1])
        d[9] = half * (-w[0] * q[2] + w[1] * q[1] + w[2] * q[0])
        d[10:13] = (u[0:3] - w) / m.tau.astype(dtype)
    elif m.id == AUTORALLY_NN:
        s, c = np.sin(x[2]), np.cos(x[2])
        d[0] = c * x[4] - s * x[5]
        d[1] = s * x[4] + c * x[5]
        d[2] = -x[6]
        inp = np.concatenate([x[3:7], u[:2]]).astype(dtype)
        h1 = np.tanh(m.W1.astype(dtype) @ inp + m.b1.astype(dtype))
        h2 = np.tanh(m.W2.astype(dtype) @ h1 + m.b2.astype(dtype))
        d[3:7] = m.W3.astype(dtype) @ h2 + m.b3.astype(dtype)
    else:
        raise ValueError(m.id)
    return d


def grad(m: Model, x, u, dtype=np.float32):
    """Analytic A = df/dx [S][S], B = df/du [S][C] (the host twins of the plugins' computeGrad)."""
    x, u = np.asarray(x, dtype), np.asarray(u, dtype)
    S, C = m.S, m.C
    A, B = np.zeros((S, S), dtype), np.zeros((S, C), dtype)
    if m.id == CARTPOLE:
        mc, mp, l, g = (dtype(v) for v in (m.mc, m.mp, m.l, m.g))
        th, td, F = x[2], x[3], u[0]
        s, c = np.sin(th), np.cos(th)
        den = mc + mp * s * s
        A[0, 1] = 1
        A[1, 2] = (mp * c * (l * td * td + g * c) - g * mp * s * s) / den - \
            (2 * mp * c * s * (F + mp * s * (l * td * td + g * c))) / (den * den)
        A[1, 3] = (2 * l * mp * td * s) / den
        A[2, 3] = 1
        A[3, 2] = (F * s - g * c * (mp + mc) - l * mp * td * td * c * c + l * mp * td * td * s * s) / (l * den) + \
            (2 * mp * c * s * (l * mp * c * s * td * td + F * c + g * s * (mp + mc))) / ((l * den) * (l * den))
        A[3, 3] = -(2 * mp * td * c * s) / den
        B[1, 0] = 1 / den
        B[3, 0] = -c / (l * den)
    elif m.id == DOUBLE_INTEGRATOR:
        A[0, 2] = A[1, 3] = 1
        B[2, 0] = B[3, 1] = 1
    elif m.id == QUADROTOR:
        q, w = x[6:10], x[10:13]
        a = u[3] / dtype(m.mass)
        A[0:3, 3:6] = np.eye(3, dtype=dtype)
        dcm = np.array([[2 * q[2], 2 * q[3], 2 * q[0], 2 * q[1]],
                        [-2 * q[1], -2 * q[0], 2 * q[3], 2 * q[2]],
                        [2 * q[0], -2 * q[1], -2 * q[2], 2 * q[3]]], dtype)
        A[3:6, 6:10] = a * dcm
        B[3, 3] = 2 * (q[1] * q[3] + q[0] * q[2]) / dtype(m.mass)
        B[4, 3] = 2 * (q[2] * q[3] - q[0] * q[1]) / dtype(m.mass)
        B[5, 3] = (q[0] ** 2 - q[1] ** 2 - q[2] ** 2 + q[3] ** 2) / dtype(m.mass)
        A[6:10, 6:10] = dtype(0.5) * np.array([[0, -w[0], -w[1], -w[2]], [w[0], 0, w[2], -w[1]],
                                               [w[1], -w[2], 0, w[0]], [w[2], w[1], -w[0], 0]], dtype)
        A[6:10, 10:13] = dtype(0.5) * np.array([[-q[1], -q[2], -q[3]], [q[0], -q[3], q[2]], [q[3], q[0], -q[1]],
                                                [-q[2], q[1], q[0]]], dtype)
        tau = m.tau.astype(dtype)
        A[10:13, 10:13] = np.diag(-1 / tau)
        B[10:13, 0:3] = np.diag(1 / tau)
    elif m.id == AUTORALLY_NN:
        s, c = np.sin(x[2]), np.cos(x[2])
        A[0, 2], A[0, 4], A[0, 5] = -s * x[4] - c * x[5], c, -s
        A[1, 2], A[1, 4], A[1, 5] = c * x[4] - s * x[5], s, c
        A[2, 6] = -1
        W1, W2, W3 = (W.astype(dtype) for W in (m.W1, m.W2, m.W3))
        inp = np.concatenate([x[3:7], u[:2]]).astype(dtype)
        a1 = np.tanh(W1 @ inp + m.b1.astype(dtype))
        a2 = np.tanh(W2 @ a1 + m.b2.astype(dtype))
        J = ((W3 * (1 - a2 * a2)) @ W2 * (1 - a1 * a1)) @ W1  # [4][6]
        A[3:7, 3:7] = J[:, :4]
        B[3:7, :] = J[:, 4:]
    else:
        raise ValueError(m.id)
    return A, B


def _ldlt_solve(H, rhs):
    """Unpivoted LDLT of the symmetric C x C matrix H (lower triangle), then H^-1 rhs; None on a zero pivot."""
    C = H.shape[0]
    L, D = np.eye(C, dtype=H.dtype), np.zeros(C, H.dtype)
    for j in range(C):
        D[j] = H[j, j] - np.sum(L[j, :j] ** 2 * D[:j])
        if not np.isfinite(D[j]) or abs(D[j]) <= np.finfo(np.float32).tiny:
            return None
        for i in range(j + 1, C):
            L[i, j] = (H[i, j] - np.sum(L[i, :j] * L[j, :j] * D[:j])) / D[j]
    y = np.linalg.solve(L, rhs)
    return np.linalg.solve(L.T, y / D[:, None] if rhs.ndim == 2 else y / D)


def running_cost_derivatives(xx, uu, x_target, u_target, Q, R):
    """TrackingCostDDP::dc / d2c (ddp_tracking_costs.h): [Q (x - x*); R (u - u*)] and blkdiag(Q, R), no factor 2."""
    S, C = Q.shape[0], R.shape[0]
    H = np.zeros((S + C, S + C), Q.dtype)
    H[:S, :S], H[S:, S:] = Q, R
    return np.concatenate([Q @ (xx - x_target), R @ (uu - u_target)]), H


def terminal_cost_derivatives(xx, x_final, Q_f):
    """TrackingTerminalCost::dc / d2c: Q_f (x - x_f) and Q_f."""
    return Q_f @ (xx - x_final), Q_f


def ddp_run(m: Model, dt, x0, x_target, u_target, Q, Q_f, R, iters):
    """DDP::run (ddp.h:56-168) as DDPFeedback::computeFeedback calls it: initial controls = u_target, limits = the
    model's control ranges. Returns dict(gains [T][S][C], x [T][S], u [T][C], jac [T][S][S+C] of the last backward pass)."""
    f32 = np.float32
    S, C = m.S, m.C
    xt, ut = np.asarray(x_target, f32), np.asarray(u_target, f32)
    T = xt.shape[0]
    Q, Q_f, R, dt = np.asarray(Q, f32), np.asarray(Q_f, f32), np.asarray(R, f32), f32(dt)
    lo, hi = m.u_lo, m.u_hi
    x = np.zeros((T, S), f32)
    u = ut.copy()
    x[0] = x0
    for i in range(1, T):  # (2) columns 0 .. T-3 clamped, T-2 not
        if i < T - 1:
            u[i - 1] = np.maximum(np.minimum(u[i - 1], hi), lo)
        x[i] = x[i - 1] + f(m, x[i - 1], u[i - 1]) * dt
    K = np.zeros((T, C, S), f32)
    kff = np.zeros((T, C), f32)
    jac = np.zeros((T, S, S + C), f32)
    prev = f32(0)

    def cost(xx, uu, k):
        dx, du = xx - xt[k], uu - ut[k]
        return f32(dx @ (Q @ dx)) + f32(du @ (R @ du))

    for it in range(iters):
        for k in range(T):
            A, B = grad(m, x[k], u[k])
            jac[k, :, :S], jac[k, :, S:] = A, B
        dxT = x[T - 1] - xt[T - 1]
        Vx, _ = terminal_cost_derivatives(x[T - 1], xt[T - 1], Q_f)
        V_T = f32(dxT @ Vx)
        Vxx = f32(0.5) * (Q_f + Q_f.T)
        for k in range(T - 2, -1, -1):
            df = jac[k] * dt + np.eye(S, S + C, dtype=f32)
            Phi, Bk = df[:, :S], df[:, S:]
            dL, _ = running_cost_derivatives(x[k], u[k], xt[k], ut[k], Q, R)
            qx = dL[:S] * dt + Phi.T @ Vx
            qu = dL[S:] * dt + Bk.T @ Vx
            qux = Bk.T @ Vxx @ Phi
            qxx = Q * dt + Phi.T @ Vxx @ Phi
            quu = R * dt + Bk.T @ Vxx @ Bk
            sol = _ldlt_solve(quu, -np.concatenate([qux, qu[:, None]], axis=1))
            if sol is None:
                raise np.linalg.LinAlgError(f"LDLT failed at step {k}")
            K[k], kff[k] = sol[:, :S].astype(f32), sol[:, S].astype(f32)
            Wm = qxx + qux.T @ K[k]
            Vxx = f32(0.5) * (Wm + Wm.T)
            Vx = qx + qux.T @ kff[k]
        alpha = f32(1)
        while True:  # (6)
            xn, un = np.zeros((T, S), f32), np.zeros((T, C), f32)
            xn[0] = x[0]
            c = f32(0)
            for k in range(T - 1):
                un[k] = np.maximum(np.minimum(u[k] + alpha * kff[k] + K[k] @ (xn[k] - x[k]), hi), lo)
                c = f32(c + cost(xn[k], un[k], k) * dt)
                xn[k + 1] = xn[k] + f(m, xn[k], un[k]) * dt
            c = f32(c + V_T)
            if it == 0 or alpha < 1e-4 or c <= prev:
                x, u, prev = xn, un, c
                break
            alpha = f32(alpha * 0.5)
    return {"gains": np.ascontiguousarray(K.transpose(0, 2, 1)), "x": x, "u": u, "jac": jac}


def tracking_cost(xx, uu, x_target, u_target, Q, R):
    """TrackingCostDDP::c (ddp_tracking_costs.h)."""
    dx, du = np.asarray(xx) - x_target, np.asarray(uu) - u_target
    return float(dx @ Q @ dx + du @ R @ du)
