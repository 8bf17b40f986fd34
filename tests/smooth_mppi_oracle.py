"""The smooth-MPPI sampler (sampling_distributions/smooth-MPPI/smooth-MPPI.{cuh,cu}) as this engine defines it, restated
in float32 the way the kernels compute it, with a float64 twin written independently of it.

One solve of one distribution, with mu the nominal control [T][C], dmu the rate mean [T][C] the engine holds, s the
optimization stride and dt_s the sampler's own dt:
1. shift: every step samples around the previous rate mean's row min(s, T - 1) (the reference's in-place
   shiftControlTrajectory reads row min(t + s, s); past the horizon the engine takes the last row);
2. rates: v = dmu_b for sample 0 and t < s, sigma_d * eps for the pure-noise rows, fmaf(sigma_d, eps, dmu_b) otherwise;
3. controls: u = fmaf(v, dt_s, mu), pure-noise rows included;
4. the rollout is the Gaussian one on u (constraints, likelihood-ratio cost with mean mu);
5. update: dmu_new = sum_n w_n v_n / eta over the unconstrained rates, U_out = fmaf(dmu_new, dt_s, mu);
6. a burned draw broadcasts row min(1, T - 1) of the rate mean.
"""
import numpy as np

f32, f64 = np.float32, np.float64


def fmaf(a, b, c):
    """float32 fused multiply-add, exactly rounded. The float32 product is exact in float64; the float64 sum is rounded
    to odd (TwoSum gives its error, and an inexact sum with an even last bit moves one ulp towards the exact value), and a
    round-to-odd result with 53 >= 2 * 24 + 2 bits narrows to float32 as the exact value would."""
    p = np.asarray(a, f32).astype(f64) * np.asarray(b, f32).astype(f64)
    q = np.broadcast_to(np.asarray(c, f32).astype(f64), np.broadcast(p, np.asarray(c)).shape)
    p = np.broadcast_to(p, q.shape)
    s = p + q
    bb = s - p
    err = (p - (s - bb)) + (q - bb)
    even = (s.view(np.int64) & 1) == 0
    fix = (err != 0) & even & np.isfinite(s)
    s = np.where(fix, np.nextafter(s, s + err), s)
    return s.astype(f32)


def shift(dmu, stride):
    """shiftControlTrajectory (smooth-MPPI.cu:34-78) in place, in t order, with the read index clamped to the horizon."""
    out = np.array(dmu, f32)
    T = out.shape[0]
    for t in range(T):
        out[t] = out[max(0, min(min(t + stride, stride), T - 1))]
    return out


def shift64(dmu, stride):
    T = np.asarray(dmu).shape[0]
    return np.broadcast_to(np.asarray(dmu, f64)[max(0, min(stride, T - 1))], np.shape(dmu)).copy()


def _flags(N_total, n_local, n_offset, T, stride, pure_noise_pct):
    n = np.arange(n_local) + n_offset
    pure = n.astype(f32) >= f32(f32(1.0) - f32(pure_noise_pct)) * f32(N_total)  # gaussian.cu:108
    use_mean = (n == 0)[:, None] | (np.arange(T) < stride)[None, :]
    return pure, use_mean


def rates(eps, dmu_b, sd, stride, pure_noise_pct, N_total=None, n_offset=0):
    """eps [N][T][C], dmu_b [T][C] (the shifted rate mean), sd [C] (decayed). Returns v [N][T][C] in float32."""
    N, T, C = eps.shape
    pure, use_mean = _flags(N_total or N, N, n_offset, T, stride, pure_noise_pct)
    sd = np.asarray(sd, f32)[None, None, :]
    v = np.where(pure[:, None, None], fmaf(sd, eps, f32(-0.0)), fmaf(sd, eps, np.asarray(dmu_b, f32)[None]))
    return np.where(use_mean[:, :, None], np.asarray(dmu_b, f32)[None], v).astype(f32)


def rates64(eps, dmu_b, sd, stride, pure_noise_pct, N_total=None, n_offset=0):
    N, T, C = eps.shape
    pure, use_mean = _flags(N_total or N, N, n_offset, T, stride, pure_noise_pct)
    noise = np.asarray(sd, f64)[None, None, :] * np.asarray(eps, f64)
    v = noise + np.where(pure[:, None, None], 0.0, 1.0) * np.asarray(dmu_b, f64)[None]
    return np.where(use_mean[:, :, None], np.asarray(dmu_b, f64)[None], v)


def controls(v, mu, dt_s):
    """integrateNoise (smooth-MPPI.cu:16-32): u = mu + v dt_s for every row."""
    return fmaf(v, f32(dt_s), np.asarray(mu, f32)[None])


def controls64(v, mu, dt_s):
    return np.asarray(mu, f64)[None] + np.asarray(v, f64) * f64(f32(dt_s))


def weights64(costs, lam):
    c = np.asarray(costs, f64)
    w = np.exp(-(c - c.min()) / f64(lam))
    return w / w.sum()


def update64(costs, v, lam, mu, dt_s):
    """updateDistributionParamsFromDevice (smooth-MPPI.cu:204-240): the new rate mean from the unconstrained rates, and
    U_out = mu + dmu_new dt_s."""
    w = weights64(costs, lam)
    dmu_new = np.tensordot(w, np.asarray(v, f64), axes=(0, 0))
    return dmu_new, np.asarray(mu, f64) + dmu_new * f64(f32(dt_s))


def update(costs, v, lam, mu, dt_s):
    """The float32 restatement of the update: weights in float64 (the merge accumulates its normaliser in double), the
    weighted sum in float32, U_out by fmaf."""
    w = weights64(costs, lam).astype(f32)
    dmu_new = np.einsum("n,ntc->tc", w, np.asarray(v, f32), dtype=f32)
    return dmu_new, fmaf(dmu_new, f32(dt_s), mu)


def burn(dmu, n):
    """generateSamples(1, 0, ...) n times (mppi_controller.cu:95): the stride-1 shift, n times."""
    out = np.array(dmu, f32)
    for _ in range(n):
        out = shift(out, 1)
    return out
