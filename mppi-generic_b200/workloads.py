"""Synthetic workloads for the BASELINE.json configurations (SURVEY.md §8d "Synthetic inputs (fixed, seeded)").

Each builder returns a ``Workload`` holding the plugin objects (host mirrors of the reference classes), the solver
scalars and the initial conditions, so that tests, ``__graft_entry__.smoke()`` and ``bench.py`` all run the very same
configuration. Nothing here reads /root/reference or any dataset: weights and maps are generated from fixed seeds.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from . import host as H


@dataclass
class Workload:
    name: str
    controller: str  # "vanilla" | "tube"
    dyn: object
    cost: object
    sampler: object
    N: int
    T: int
    D: int
    dt: float
    lambda_: float
    alpha: float
    x0: np.ndarray  # [D][S]
    U0: np.ndarray  # [D][T][C]
    seed: int = 42
    optimization_stride: int = 1
    extra: dict = field(default_factory=dict)

    @property
    def noise_bytes(self) -> int:
        """Algorithmic HBM bytes of one rollout launch: one read of the unique noise buffer (SURVEY §8d)."""
        return self.N * self.T * self.dyn.CONTROL_DIM * 4

    def make_engine(self, **kw) -> "H.Engine":
        e = H.Engine(self.dyn, self.cost, self.sampler, self.N, self.T, self.D, **kw)
        e.set_solver(self.dt, self.lambda_, self.alpha)
        e.seed(self.seed, 0)
        return e


def cartpole(N: int = 8192, T: int = 100) -> Workload:
    """C1/C2: Cartpole + quadratic cost, VanillaMPPI (tests/controllers/vanilla_mppi_test.cu:18-28,81-93,
    examples/cartpole_example.cu:12-13)."""
    dyn = H.CartpoleDynamics(1.0, 1.0, 1.0)
    dyn.setControlRanges([(-5.0, 5.0)])
    cost = H.CartpoleQuadraticCost()
    p = cost.params
    p.cart_position_coeff, p.cart_velocity_coeff = 100.0, 10.0
    p.pole_angle_coeff, p.pole_angular_velocity_coeff = 200.0, 20.0
    p.control_cost_coeff[0] = 1.0
    p.terminal_cost_coeff = 0.0
    p.desired_terminal_state[:] = [-20.0, 0.0, math.pi, 0.0]
    sampler = H.GaussianDistribution(1, [5.0])
    sampler.setControlCostCoeff([1.0])
    x0 = np.zeros((1, 4), np.float32)
    U0 = np.zeros((1, T, 1), np.float32)
    return Workload(f"cartpole_vanilla_N{N}_T{T}", "vanilla", dyn, cost, sampler, N, T, 1, 0.01, 0.25, 0.01, x0, U0)


def double_integrator_tube(N: int = 16384, T: int = 150) -> Workload:
    """C3: DoubleIntegrator circular track (CORL2020), Tube-MPPI (examples/double_integrator_CORL2020.cu:29-39,316-352)."""
    dyn = H.DoubleIntegratorDynamics(1.0)
    cost = H.DoubleIntegratorCircleCost()
    sampler = H.GaussianDistribution(2, [1.0, 1.0])
    x0 = np.tile(np.array([2.0, 0.0, 0.0, 1.0], np.float32), (2, 1))
    U0 = np.zeros((2, T, 2), np.float32)
    return Workload(f"double_integrator_tube_N{N}_T{T}", "tube", dyn, cost, sampler, N, T, 2, 0.02, 2.0, 0.0, x0, U0,
                    extra={"nominal_threshold": 20.0})


def double_integrator_vanilla(N: int = 4096, T: int = 100) -> Workload:
    """DoubleIntegrator with a single distribution (examples/double_integrator_example.cu) — parity-test case."""
    w = double_integrator_tube(N, T)
    w.name, w.controller, w.D = f"double_integrator_vanilla_N{N}_T{T}", "vanilla", 1
    w.x0, w.U0 = w.x0[:1].copy(), w.U0[:1].copy()
    return w


def synthetic_nn_weights(seed: int = 1) -> np.ndarray:
    """theta_i ~ U(-1,1)/sqrt(fan_in), packed W (row-major out x in) then b per layer (fnn_helper.cu:176-183).
    The real Autorally network is a git-LFS stub in the reference tree (SURVEY §0), so weights are synthetic."""
    rng = np.random.RandomState(seed)
    layers = (6, 32, 32, 4)
    out = []
    for i in range(3):
        fan_in = layers[i]
        out.append((rng.uniform(-1, 1, layers[i + 1] * fan_in) / math.sqrt(fan_in)).astype(np.float32))
        out.append((rng.uniform(-1, 1, layers[i + 1]) / math.sqrt(fan_in)).astype(np.float32))
    th = np.concatenate(out)
    assert th.size == H.AR_NN_NUM_PARAMS
    return th


def track_map_standard() -> tuple:
    """In-memory replica of `track_map_standard.npz` (scripts/autorally/test/generateTestMaps.py:45-75):
    600 x 600 @ 20 ppm, channel0[i][j] = |15 - y| + x/30 with x = j/ppm, y = i/ppm; bounds x in [-13,17], y in [-10,20]."""
    ppm, width, height = 20, 30, 30
    i = np.arange(width * ppm, dtype=np.float64)[:, None]
    j = np.arange(height * ppm, dtype=np.float64)[None, :]
    x, y = j / ppm, i / ppm
    ch0 = (np.abs(height / 2.0 - y) + x / width).astype(np.float32)
    return ch0, (-13.0, 17.0), (-10.0, 20.0), float(ppm)


def autorally(N: int = 32768, T: int = 100) -> Workload:
    """C4: NeuralNetModel<7,2,3> + ARStandardCost on the generated test map (SURVEY §8d; ranges from
    tests/dynamics/ar_dynamics_nn_test.cu:52-58)."""
    dyn = H.NeuralNetModel([(-1.0, 1.0), (-2.0, 2.0)])
    dyn.updateModel([6, 32, 32, 4], synthetic_nn_weights(1))
    cost = H.ARStandardCost()
    ch0, xb, yb, ppm = track_map_standard()
    cost.loadTrackData(ch0, xb[0], xb[1], yb[0], yb[1], ppm)
    sampler = H.GaussianDistribution(2, [0.3, 0.3])
    x0 = np.array([[0.0, 0.0, 0.0, 0.0, 4.0, 0.0, 0.0]], np.float32)
    U0 = np.zeros((1, T, 2), np.float32)
    return Workload(f"autorally_nn_N{N}_T{T}", "vanilla", dyn, cost, sampler, N, T, 1, 0.02, 6.67, 0.0, x0, U0)


def track_map_robust() -> tuple:
    """In-memory replica of `track_map_robust.npz` (scripts/autorally/test/generateTestMaps.py:76-109): width 70, height 55
    at 20 ppm, bounds x in [-25, 45], y in [-50, 5]. The script fills [1400][1100] arrays (i: y = i/ppm, j: x = j/ppm)
    with channel0 = 1 where x > 50 or x < 15, else 0.6 where x > 40 or x < 25, else 0; channel1 = |55/2 - y| + x/70;
    channel2 = x; channel3 = atan2(y, x), and stores them flattened; ARStandardCostImpl::loadTrackData reads each flat
    channel as [height 1100][width 1400] rows. Returns (texels [1100][1400][4], x bounds, y bounds, ppm)."""
    ppm, width, height = 20, 70, 55
    i = np.arange(width * ppm, dtype=np.float64)[:, None]
    j = np.arange(height * ppm, dtype=np.float64)[None, :]
    x, y = j / ppm + 0.0 * i, i / ppm + 0.0 * j
    ch0 = np.where((x > 50) | (x < 15), 1.0, np.where((x > 40) | (x < 25), 0.6, 0.0))
    ch1 = np.abs(height / 2.0 - y) + x / width
    ch3 = np.arctan2(y, x)
    tex = np.stack([c.astype(np.float32).reshape(-1) for c in (ch0, ch1, x, ch3)], axis=-1)
    return tex.reshape(height * ppm, width * ppm, 4), (-25.0, 45.0), (-50.0, 5.0), float(ppm)


def autorally_robust(N: int = 32768, T: int = 100) -> Workload:
    """The C4 model with ARRobustCost on `track_map_robust()`: the robust cost's defaults (ar_robust_cost.cuh:11-28; speed
    from the map's .z channel) plus heading_coeff 20 (the reference's robust-cost test fixture), so every term is live.
    The start (22.5, 0) lies in the map's zero-boundary band."""
    w = autorally(N, T)
    cost = H.ARRobustCost()
    tex, xb, yb, _ = track_map_robust()
    cost.setTrackData(tex, xb[0], xb[1], yb[0], yb[1])
    cost.params.heading_coeff = 20.0
    w.cost = cost
    w.x0[0, :2] = [22.5137, 0.0071]
    w.name = f"autorally_robust_N{N}_T{T}"
    return w


def double_integrator_robust_tube(N: int = 16384, T: int = 150) -> Workload:
    """C3 with DoubleIntegratorRobustCost (examples/double_integrator_CORL2020.cu runTubeRC: crash_cost 100)."""
    w = double_integrator_tube(N, T)
    w.cost = H.DoubleIntegratorRobustCost()
    w.cost.params.crash_cost = 100.0
    w.name = f"double_integrator_robust_tube_N{N}_T{T}"
    return w


def synthetic_lstm_weights(hidden_dim: int = 4, head_hidden: int = 20, seed: int = 2) -> tuple:
    """(lstm, head) ~ U(-1,1)/sqrt(fan_in) in the reference's packed layouts (lstm_helper.cu:72-88, fnn_helper.cu:176-183),
    initial hidden / cell state zero (SURVEY §8d C5). The RACER networks are not in the reference tree."""
    rng = np.random.RandomState(seed)
    Hd, I = hidden_dim, H.RACER_LSTM_INPUT_DIM
    parts = [rng.uniform(-1, 1, 4 * Hd * Hd) / math.sqrt(Hd + I), rng.uniform(-1, 1, 4 * Hd * I) / math.sqrt(Hd + I),
             rng.uniform(-1, 1, 4 * Hd) / math.sqrt(Hd + I), np.zeros(2 * Hd)]
    lstm = np.concatenate(parts).astype(np.float32)
    IN = Hd + I
    head = np.concatenate([rng.uniform(-1, 1, head_hidden * IN) / math.sqrt(IN), rng.uniform(-1, 1, head_hidden) / math.sqrt(IN),
                           rng.uniform(-1, 1, head_hidden) / math.sqrt(head_hidden),
                           rng.uniform(-1, 1, 1) / math.sqrt(head_hidden)]).astype(np.float32)
    return lstm, head


def racer_lstm(N: int = 65536, T: int = 150, hidden_dim: int = 4, head_hidden: int = 20, colored: bool = True) -> Workload:
    """C5: RacerDubinsElevationLSTMSteering (the in-tree LSTM vehicle model, S19 C2 O28; constructor
    (3, 20, {23, 100, 2H}, 4, H, {H+4, 20, 1}, 11), tests/dynamics/racer_dubins_elevation_lstm_steering_model_test.cu:26-32)
    on flat terrain + ColoredNoise sampler (exponents (1, 1), offset_decay_rate 0.97, colored_noise.cuh:47-49) + our quadratic
    tracking cost (SURVEY §8d C5)."""
    dyn = H.RacerDubinsElevationLSTMSteering(3, 20, (23, 100, 2 * hidden_dim), 4, hidden_dim,
                                             (hidden_dim + 4, head_hidden, 1), 11)
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])  # throttle/brake, steering command
    dyn.setAllValues(*synthetic_lstm_weights(hidden_dim, head_hidden, 2))
    cost = H.RacerQuadraticCost()
    # with the reference's default coefficients (racer_dubins.cuh:78-82) full throttle saturates near 1.6 m/s
    cost.params.desired_speed = 1.2
    if colored:
        sampler = H.ColoredNoiseDistribution(2, [0.3, 0.3], [1.0, 1.0])
    else:
        sampler = H.GaussianDistribution(2, [0.3, 0.3])
    x0 = np.zeros((1, 19), np.float32)
    x0[0, 0] = 3.0  # VEL_X
    x0[0, 9:13] = 1e-6  # covariance diagonal floor (racer_dubins_elevation.cu stateFromMap)
    U0 = np.zeros((1, T, 2), np.float32)
    tag = "colored" if colored else "gaussian"
    return Workload(f"racer_lstm_H{hidden_dim}_{tag}_N{N}_T{T}", "vanilla", dyn, cost, sampler, N, T, 1, 0.02, 1.0, 0.0,
                    x0, U0)


def racer_lstm_gaussian(N: int = 4096, T: int = 100) -> Workload:
    return racer_lstm(N, T, colored=False)


def racer_lstm_h32(N: int = 65536, T: int = 150) -> Workload:
    """C5 at the tensor-core-relevant size of SURVEY §8d: hidden_dim 32 (gate matrix [36 x 128] per step), head {36, 20, 1}."""
    return racer_lstm(N, T, hidden_dim=32, head_hidden=20)


def racer_elevation_map(seed: int = 11, resolution: float = 0.5) -> "H.TwoDTextureHelper":
    """A rolling elevation map for the RACER workloads: x in [-10, 90], y in [-30, 30] m, heights from two gentle sine waves
    (amplitude 0.4 and 0.25 m, wavelengths 24 and 15 m) plus seeded noise in [0, 0.02) m."""
    xb, yb = (-10.0, 90.0), (-30.0, 30.0)
    w, h = int(round((xb[1] - xb[0]) / resolution)), int(round((yb[1] - yb[0]) / resolution))
    cx = xb[0] + (np.arange(w) + 0.5) * resolution
    cy = yb[0] + (np.arange(h) + 0.5) * resolution
    X, Y = np.meshgrid(cx, cy)  # [h][w]
    z = 0.4 * np.sin(2 * math.pi * X / 24.0) + 0.25 * np.cos(2 * math.pi * Y / 15.0)
    z = (z + 0.02 * np.random.RandomState(seed).uniform(0.0, 1.0, z.shape)).astype(np.float32)
    tex = H.TwoDTextureHelper()
    tex.setExtent(0, w, h)
    tex.updateTexture(0, z)
    tex.updateOrigin(0, (xb[0], yb[0], 0.0))
    tex.updateResolution(0, resolution)
    tex.enableTexture(0)
    return tex


def racer_elevation(N: int = 8192, T: int = 100, use_map: bool = True) -> Workload:
    """RacerDubinsElevation (reference default parameters) + our quadratic tracking cost, VanillaMPPI: hold 1.2 m/s along
    +x over racer_elevation_map() (flat ground when use_map is False)."""
    dyn = H.RacerDubinsElevation()
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])  # throttle/brake, steering command
    if use_map:
        dyn.tex_helper_ = racer_elevation_map()
    cost = H.RacerQuadraticCost()
    cost.params.desired_speed = 1.2
    sampler = H.GaussianDistribution(2, [0.3, 0.3])
    x0 = np.zeros((1, 19), np.float32)
    x0[0, 0] = 1.0  # VEL_X
    x0[0, 9:13] = 1e-6  # covariance diagonal floor
    U0 = np.zeros((1, T, 2), np.float32)
    return Workload(f"racer_elevation{'' if use_map else '_nomap'}_N{N}_T{T}", "vanilla", dyn, cost, sampler, N, T, 1, 0.02,
                    1.0, 0.0, x0, U0)


def racer_elevation_tube(N: int = 8192, T: int = 100, use_map: bool = True) -> Workload:
    """racer_elevation() with Tube-MPPI: two distributions, the nominal and the real system."""
    w = racer_elevation(N, T, use_map)
    w.name, w.controller, w.D = f"racer_elevation_tube{'' if use_map else '_nomap'}_N{N}_T{T}", "tube", 2
    w.x0, w.U0 = np.tile(w.x0, (2, 1)), np.tile(w.U0, (2, 1, 1))
    w.extra = {"nominal_threshold": 20.0}
    return w


def racer_hill_maps(seed: int = 13, resolution: float = 0.5) -> tuple:
    """(elevation, normals) helpers for the suspension model: x in [-10, 90], y in [-30, 30] m, twelve seeded Gaussian hills
    (heights 0.2 .. 0.8 m, widths 3 .. 8 m); the normals are (-dz/dx, -dz/dy, 1) normalised, from the heights' central
    differences."""
    xb, yb = (-10.0, 90.0), (-30.0, 30.0)
    w, h = int(round((xb[1] - xb[0]) / resolution)), int(round((yb[1] - yb[0]) / resolution))
    cx = xb[0] + (np.arange(w) + 0.5) * resolution
    cy = yb[0] + (np.arange(h) + 0.5) * resolution
    X, Y = np.meshgrid(cx, cy)  # [h][w]
    rng = np.random.RandomState(seed)
    z = np.zeros_like(X)
    for _ in range(12):
        x0, y0 = rng.uniform(*xb), rng.uniform(*yb)
        z += rng.uniform(0.2, 0.8) * np.exp(-((X - x0) ** 2 + (Y - y0) ** 2) / (2 * rng.uniform(3.0, 8.0) ** 2))
    dzdy, dzdx = np.gradient(z, resolution)
    n = np.stack([-dzdx, -dzdy, np.ones_like(z)], axis=-1)
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    elev = H.TwoDTextureHelper()
    elev.setExtent(0, w, h)
    elev.updateTexture(0, z.astype(np.float32))
    elev.updateOrigin(0, (xb[0], yb[0], 0.0))
    elev.updateResolution(0, resolution)
    elev.enableTexture(0)
    normals = H.TwoDTextureHelperFloat4()
    normals.setExtent(0, w, h)
    normals.updateTexture(0, np.concatenate([n, np.zeros(z.shape + (1,))], axis=-1).astype(np.float32))
    normals.updateOrigin(0, (xb[0], yb[0], 0.0))
    normals.updateResolution(0, resolution)
    normals.enableTexture(0)
    return elev, normals


def racer_suspension(N: int = 65536, T: int = 150, hidden_dim: int = 4, use_maps: bool = True, head_hidden: int = 20,
                     colored: bool = True) -> Workload:
    """RacerDubinsElevationSuspension at C5's settings (racer_lstm(): the same network, weights, sampler and cost) over
    racer_hill_maps(), or flat ground with upright normals when use_maps is False. The car starts at 3 m/s with its centre
    of gravity one wheel radius above the ground under it."""
    dyn = H.RacerDubinsElevationSuspension(3, 20, (23, 100, 2 * hidden_dim), 4, hidden_dim, (hidden_dim + 4, head_hidden, 1),
                                           11)
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    dyn.setAllValues(*synthetic_lstm_weights(hidden_dim, head_hidden, 2))
    x0 = np.zeros((1, 24), np.float32)
    x0[0, dyn.VEL_X] = 3.0
    x0[0, dyn.UNCERTAINTY_POS_X:dyn.UNCERTAINTY_POS_X + 4] = 1e-6
    ground = 0.0
    if use_maps:
        dyn.tex_helper_, dyn.normals_tex_helper_ = racer_hill_maps()
        ground = dyn.tex_helper_.queryTextureAtWorldPose(0, (dyn.params.c_g[0], 0.0, 0.0))
    x0[0, dyn.CG_POS_Z] = ground + dyn.params.wheel_radius
    cost = H.RacerQuadraticCost()
    cost.params.desired_speed = 1.2
    sampler = H.ColoredNoiseDistribution(2, [0.3, 0.3], [1.0, 1.0]) if colored else H.GaussianDistribution(2, [0.3, 0.3])
    U0 = np.zeros((1, T, 2), np.float32)
    tag = ("maps" if use_maps else "flat") + ("" if colored else "_gaussian")
    return Workload(f"racer_suspension_H{hidden_dim}_{tag}_N{N}_T{T}", "vanilla", dyn, cost, sampler, N, T, 1, 0.02, 1.0,
                    0.0, x0, U0)


def quadrotor(N: int = 8192, T: int = 100) -> Workload:
    """Quadrotor + quadratic cost, VanillaMPPI (instantiations/quadrotor_mppi/quadrotor_mppi.cuh): fly from the origin
    to a goal 4 m away and 2 m up, hovering there. The only CONTROL_DIM = 4 pair (one 16-byte noise group per step)."""
    dyn = H.QuadrotorDynamics()
    dyn.setControlRanges([(-3.0, 3.0), (-3.0, 3.0), (-3.0, 3.0), (0.0, 36.0)])
    cost = H.QuadrotorQuadraticCost()
    p = cost.params
    p.s_goal[0], p.s_goal[1], p.s_goal[2] = 4.0, 1.0, 2.0
    p.x_coeff, p.v_coeff, p.w_coeff = 10.0, 1.0, 0.5
    p.roll_coeff = p.pitch_coeff = p.yaw_coeff = 5.0
    sampler = H.GaussianDistribution(4, [0.5, 0.5, 0.5, 2.0])
    sampler.setControlCostCoeff([0.1, 0.1, 0.1, 0.01])
    x0 = dyn.getZeroState()[None, :].copy()
    U0 = np.zeros((1, T, 4), np.float32)
    U0[..., 3] = dyn.GRAVITY  # hover thrust (zero_control_[3])
    return Workload(f"quadrotor_vanilla_N{N}_T{T}", "vanilla", dyn, cost, sampler, N, T, 1, 0.02, 1.0, 0.0, x0, U0)


def quadrotor_gate_course() -> list:
    """Three gates as waypoints (x, y, z, heading). The gate's corners lie along `heading` (QuadrotorMapCostParams::
    updateWaypoint), so a gate crossed flying along +x has heading pi/2."""
    return [(6.0, 0.0, 2.0, math.pi / 2), (12.0, 2.0, 2.5, math.pi / 2 - 0.3), (18.0, 3.0, 2.0, math.pi / 2)]


def quadrotor_track_map(seed: int = 7, resolution: float = 0.25) -> tuple:
    """A track cost map for quadrotor_gate_course(): 0.5 per metre of horizontal distance from the polyline through the
    start and the gates, plus seeded noise in [0, 0.05). The map covers x in [-4, 24], y in [-8, 11]; outside it the cost's
    map term adds crash_coeff. Returns (TwoDTextureHelper, x bounds, y bounds)."""
    xb, yb = (-4.0, 24.0), (-8.0, 11.0)
    w, h = int(round((xb[1] - xb[0]) / resolution)), int(round((yb[1] - yb[0]) / resolution))
    pts = np.array([(0.0, 0.0)] + [g[:2] for g in quadrotor_gate_course()], np.float64)
    cx = xb[0] + (np.arange(w) + 0.5) * resolution
    cy = yb[0] + (np.arange(h) + 0.5) * resolution
    X, Y = np.meshgrid(cx, cy)  # [h][w]
    dist = np.full(X.shape, np.inf)
    for a, b in zip(pts[:-1], pts[1:]):
        ab = b - a
        t = np.clip(((X - a[0]) * ab[0] + (Y - a[1]) * ab[1]) / (ab @ ab), 0.0, 1.0)
        dist = np.minimum(dist, np.hypot(X - a[0] - t * ab[0], Y - a[1] - t * ab[1]))
    values = (0.5 * dist + 0.05 * np.random.RandomState(seed).uniform(0.0, 1.0, dist.shape)).astype(np.float32)
    tex = H.TwoDTextureHelper()
    tex.setExtent(0, w, h)
    tex.updateTexture(0, values)
    tex.updateOrigin(0, (xb[0], yb[0], 0.0))
    tex.updateResolution(0, resolution)
    tex.enableTexture(0)
    return tex, xb, yb


def quadrotor_gates(N: int = 8192, T: int = 100, use_map: bool = True) -> Workload:
    """Quadrotor + QuadrotorMapCost flying quadrotor_gate_course() over quadrotor_track_map() (without the map when
    use_map is False), VanillaMPPI. The cost starts with the start point as its previous waypoint and the first gate as
    its current one; advance_quadrotor_gate() moves to the next gate once the current one is passed. extra["gate"] is the
    index of the current gate."""
    w = quadrotor(N, T)
    cost = H.QuadrotorMapCost()
    cost.params.desired_speed = 3.0
    cost.params.dist_to_waypoint_coeff = 1.0
    start = (0.0, 0.0, 2.0, 0.0)
    cost.updateWaypoint(start)
    cost.updateWaypoint(quadrotor_gate_course()[0])
    if use_map:
        cost.tex_helper_ = quadrotor_track_map()[0]
    w.cost = cost
    w.x0[0, :3] = start[:3]
    w.name = f"quadrotor_gates{'' if use_map else '_nomap'}_N{N}_T{T}"
    w.extra = {"gate": 0, "start": start}
    return w


def advance_quadrotor_gate(w: Workload, state, radius: float = 1.0) -> bool:
    """Move the cost's waypoint to the next gate once `state` is within `radius` of the current gate or past its plane
    (the gate's plane contains the gate line and the vertical). Returns True if the waypoint moved."""
    gates = quadrotor_gate_course()
    g = w.extra["gate"]
    if g >= len(gates) - 1:
        return False
    gx, gy, gz, hd = gates[g]
    prev = w.extra["start"] if g == 0 else gates[g - 1]
    nx, ny = -math.sin(hd), math.cos(hd)  # normal of the gate line
    side = lambda x, y: (x - gx) * nx + (y - gy) * ny  # noqa: E731
    passed = side(state[0], state[1]) * side(prev[0], prev[1]) < 0
    if passed or math.dist(state[:3], (gx, gy, gz)) < radius:
        w.extra["gate"] = g + 1
        w.cost.updateWaypoint(gates[g + 1])
        return True
    return False


BUILDERS = {
    "racer_lstm": racer_lstm,
    "racer_lstm_gaussian": racer_lstm_gaussian,
    "racer_lstm_h32": racer_lstm_h32,
    "cartpole": cartpole,
    "double_integrator_tube": double_integrator_tube,
    "double_integrator_vanilla": double_integrator_vanilla,
    "autorally": autorally,
    "autorally_robust": autorally_robust,
    "double_integrator_robust_tube": double_integrator_robust_tube,
    "quadrotor": quadrotor,
    "quadrotor_gates": quadrotor_gates,
    "racer_elevation": racer_elevation,
    "racer_elevation_tube": racer_elevation_tube,
}


def by_name(name: str, N: Optional[int] = None, T: Optional[int] = None) -> Workload:
    kw = {}
    if N is not None:
        kw["N"] = N
    if T is not None:
        kw["T"] = T
    return BUILDERS[name](**kw)


def racer_rigid_suspension(N: int = 32768, T: int = 100, D: int = 1, colored: bool = False) -> Workload:
    """RacerSuspension (the rigid-body RACER vehicle, reference default parameters) + our quadratic tracking cost: from rest,
    upright at its equilibrium height (every spring at its rest length), drive at 5 m/s along +x. dt = 0.01: in the slip band
    the side friction's yaw eigenvalue is near -150 1/s, so the device's explicit step is stable only below about 0.013 s
    (DESIGN §8). D = 2: Tube-MPPI / RMPPI (nominal and real system). N and T as tools/racer_elevation_timing.py."""
    dyn = H.RacerSuspension()
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])  # throttle/brake, steering command
    cost = H.RacerQuadraticCost()
    cost.params.desired_speed = 5.0
    if colored:
        sampler = H.ColoredNoiseDistribution(2, [0.3, 0.3], [1.0, 1.0])
    else:
        sampler = H.GaussianDistribution(2, [0.3, 0.3])
    x0 = np.tile(dyn.getZeroState(), (D, 1))
    x0[:, dyn.P_I_Z] = dyn.restHeight()
    U0 = np.zeros((D, T, 2), np.float32)
    name = f"racer_rigid_suspension{'_tube' if D == 2 else ''}{'_colored' if colored else ''}_N{N}_T{T}"
    return Workload(name, "tube" if D == 2 else "vanilla", dyn, cost, sampler, N, T, D, 0.01, 1.0, 0.0, x0, U0,
                    extra={"nominal_threshold": 20.0} if D == 2 else {})
