"""RacerDubinsElevationSuspension (MPPIB_DYN_RACER_SUSPENSION_LSTM) with RacerQuadraticCost: the float4 map query, the host
twin and the device model against tests/racer_suspension_oracle.py, physics checks that do not go through the restatement,
and the K1 forms, sampled trajectories, the device-side roll-forward and a closed loop on the GPU."""
import ctypes as C
import math

import numpy as np
import pytest

from mppi_generic_b200 import workloads as W
import mppi_generic_b200 as m
from tests import racer_suspension_oracle as SO

H = m.host


def _net(dyn):
    return SO.Net(dyn.lstm_theta, dyn.hidden_dim, dyn.head_hidden)


def _blob(helper):
    return helper.blob() if helper.checkTextureUse(0) else None


# ---- the float4 map ------------------------------------------------------------------------------------------------
# two_d_texture_helper_test.cu:368-541: a 10 x 20 map of (i, i + 1, i + 2, i + 3), resolution 10; normalised query points
# and the value of channel x there
KNOWN = [((0.0, 0.0), 0.0), ((0.05, 0.0), 0.0), ((0.95, 0.0), 9.0), ((1.0, 0.0), 9.0), ((0.45, 0.0), 4.0),
         ((0.5, 0.0), 4.5), ((0.55, 0.0), 5.0), ((0.0, 0.0), 0.0), ((0.0, 0.025), 0.0), ((0.0, 0.05), 5.0),
         ((0.0, 0.075), 10.0), ((0.0, 0.975), 190.0), ((0.0, 1.0), 190.0), ((0.0, 0.475), 90.0), ((0.0, 0.5), 95.0),
         ((0.0, 0.525), 100.0)]


def _known_map(world):
    t = H.TwoDTextureHelperFloat4()
    t.setExtent(0, 10, 20)
    i = np.arange(200, dtype=np.float32)
    t.updateTexture(0, np.stack([i, i + 1, i + 2, i + 3], axis=-1))
    t.updateResolution(0, 10)
    if world:
        t.updateRotation(0, [[0, 1, 0], [1, 0, 0], [0, 0, 1]])
        t.updateOrigin(0, (1, 2, 3))
    t.enableTexture(0)
    return t


@pytest.mark.parametrize("world", [False, True], ids=["QueryTextureAtMapPose", "QueryTextureAtWorldPose"])
def test_float4_query_known_answers(world):
    t = _known_map(world)
    for (u, v), val in KNOWN:
        p = (v * 200 + 1, u * 100 + 2, 3.0) if world else (u * 100, v * 200, 0.0)
        want = np.array([val, val + 1, val + 2, val + 3], np.float32)
        np.testing.assert_allclose(t.queryTextureAtWorldPose(0, p), want, rtol=1e-6, atol=1e-5)
        np.testing.assert_allclose(SO.normals_at_world_pose(t.blob(), *p), want, rtol=1e-6, atol=1e-5)


def test_float4_query_against_scipy():
    """Each channel against an independent float64 bilinear interpolator (scipy map_coordinates, order 1, clamped)."""
    from scipy.ndimage import map_coordinates
    rng = np.random.RandomState(3)
    t = H.TwoDTextureHelperFloat4()
    t.setExtent(0, 13, 7)
    vals = rng.uniform(-1, 1, (7, 13, 4)).astype(np.float32)
    t.updateTexture(0, vals)
    t.updateResolution(0, 0.5)
    t.updateOrigin(0, (-1.0, 0.5, 0.0))
    t.enableTexture(0)
    for _ in range(200):
        wx, wy = rng.uniform(-2, 6), rng.uniform(-0.5, 5)
        qx = np.clip((wx + 1.0) / 0.5 - 0.5, 0, 12)
        qy = np.clip((wy - 0.5) / 0.5 - 0.5, 0, 6)
        want = [map_coordinates(vals[..., k].astype(np.float64), [[qy], [qx]], order=1, mode="nearest")[0] for k in range(4)]
        np.testing.assert_allclose(t.queryTextureAtWorldPose(0, (wx, wy, 0.0)), want, atol=2e-6)


# ---- ids, layout, host twin ----------------------------------------------------------------------------------------
def test_ids_dims_and_blob_layout():
    assert (H.DYN_RACER_SUSPENSION_LSTM, H.BLOB_NORMALS_MAP) == (6, 8)
    S, Cd, O = C.c_int(), C.c_int(), C.c_int()
    assert H.lib().mppib_host_dims(6, C.byref(S), C.byref(Cd), C.byref(O)) == 0
    assert (S.value, Cd.value, O.value) == (24, 2, 28)
    dyn = H.RacerDubinsElevationSuspension()
    assert (dyn.STATE_DIM, dyn.OUTPUT_DIM, dyn.model_dims()) == (24, 28, (4, 20))
    base = C.sizeof(H.RacerLSTMDynParams)
    assert C.sizeof(H.RacerSuspensionDynParams) == base + 9 * 4
    assert dyn.blob()[:base] == bytes(H.RacerDubinsElevationLSTMSteering().params)
    tail = np.frombuffer(dyn.blob()[base:], np.float32)
    f = np.float32
    np.testing.assert_array_equal(tail, np.array([14000, 1000, 1447, f(f(f(f(1) / f(12)) * f(1447)) * f(2)) * f(2.25),
                                                  f(f(f(1) / f(12)) * f(1447)) * f(11.25), 0.32, f(2.981) * f(0.5), 0, 0],
                                                 np.float32))


def _random_state(rng, maps=True):
    x = np.zeros(24, np.float32)
    x[SO.VEL_X] = rng.choice([rng.uniform(-0.2, 0.2), rng.uniform(0.2, 3.0), rng.uniform(3.0, 8.0), rng.uniform(-4, -0.2)])
    x[SO.YAW] = rng.uniform(-math.pi, math.pi)
    x[SO.POS_X], x[SO.POS_Y] = rng.uniform(0, 60), rng.uniform(-20, 20)
    x[SO.STEER_ANGLE] = rng.uniform(-0.5, 0.5)
    x[SO.BRAKE_STATE] = rng.uniform(0, 0.4)
    x[SO.ROLL], x[SO.PITCH] = rng.uniform(-0.2, 0.2, 2)
    x[SO.CG_POS_Z] = rng.uniform(0.2, 1.2)
    x[SO.CG_VEL_I_Z], x[SO.ROLL_RATE], x[SO.PITCH_RATE] = rng.uniform(-0.5, 0.5, 3)
    x[SO.STEER_ANGLE_RATE] = rng.uniform(-2, 2)
    x[SO.UNC0:SO.UNC0 + 4] = rng.uniform(1e-4, 0.1, 4)
    x[SO.UNC0 + 4:SO.UNC0 + 10] = rng.uniform(-1e-4, 1e-4, 6)
    return x


def _maps_workload(kind):
    """none / elev / both / partial (the reference test's partial maps: 10 x 20 at resolution 10, origin (1, 2, 3), the
    swapped rotation, the first 10 cells NaN, racer_dubins_elevation_suspension_test.cu)."""
    w = W.racer_suspension(1024, 40, 4, use_maps=kind in ("elev", "both"), colored=False)
    if kind == "elev":
        w.dyn.normals_tex_helper_ = H.TwoDTextureHelperFloat4()
    if kind == "partial":
        rng = np.random.RandomState(9)
        hgt = rng.uniform(0.0, 0.5, 200).astype(np.float32)
        hgt[:10] = np.nan
        nrm = np.concatenate([rng.uniform(-0.2, 0.2, (200, 2)), np.ones((200, 1)), np.zeros((200, 1))], 1).astype(np.float32)
        nrm[:10] = np.nan
        for t, v in ((w.dyn.tex_helper_, hgt), (w.dyn.normals_tex_helper_, nrm)):
            t.setExtent(0, 10, 20)
            t.updateTexture(0, v)
            t.updateResolution(0, 10)
            t.updateOrigin(0, (1, 2, 3))
            t.enableTexture(0)
        w.dyn.updateRotation([[0, 1, 0], [1, 0, 0], [0, 0, 1]])
    return w


@pytest.mark.parametrize("maps", ["none", "both", "partial"])
def test_host_twin_equals_host_restatement(maps):
    w = _maps_workload(maps)
    dyn = w.dyn
    p = SO.Params(dyn.params)
    net = _net(dyn)
    rng = np.random.RandomState(4)
    eb, nb = _blob(dyn.tex_helper_), _blob(dyn.normals_tex_helper_)
    for _ in range(150):
        x, u = _random_state(rng), rng.uniform(-1, 1, 2).astype(np.float32)
        h, c = rng.uniform(-0.5, 0.5, (2, dyn.hidden_dim)).astype(np.float32)
        a = dyn.step(x, u, 0.02, h, c)
        b = SO.step(p, net, x, u, 0.02, h, c, "host", np.float32, eb, nb)
        for v, r in zip(a, b):
            np.testing.assert_allclose(v, r, rtol=2e-5, atol=2e-5)


def test_restatement_float32_against_float64_and_host_minus_device():
    """float32 against float64, and host against device: with angles in range and the throttle's lower limit at -1 the two
    bodies differ only by the device's reciprocals and normalised angles, i.e. by rounding."""
    w = _maps_workload("both")
    p = SO.Params(w.dyn.params)
    net = _net(w.dyn)
    eb, nb = _blob(w.dyn.tex_helper_), _blob(w.dyn.normals_tex_helper_)
    rng = np.random.RandomState(1)
    for _ in range(100):
        x, u = _random_state(rng), rng.uniform(-1, 1, 2).astype(np.float32)
        h, c = net.initial()
        a = SO.step(p, net, x, u, 0.02, h, c, "device", np.float32, eb, nb)
        b = SO.step(p, net, x, u, 0.02, h, c, "device", np.float64, eb, nb)
        d = SO.step(p, net, x, u, 0.02, h, c, "host", np.float32, eb, nb)
        for i in range(3):
            r = b[i].astype(np.float64)
            assert np.all(np.abs(a[i] - r) <= 2e-4 * np.maximum(1.0, np.abs(r))), np.abs(a[i] - r).max()
            assert np.all(np.abs(a[i] - d[i]) <= 2e-4 * np.maximum(1.0, np.abs(d[i])))
    # the brake clamp: lower throttle limit -0.5 -> the host caps the brake state at 0.5, the device at 1
    w.dyn.setControlRanges([(-0.5, 1.0), (-1.0, 1.0)])
    p = SO.Params(w.dyn.params)
    x = _random_state(rng)
    x[SO.BRAKE_STATE] = 0.6
    h, c = net.initial()
    hn = SO.step(p, net, x, [-1.0, 0.0], 0.02, h, c, "host", np.float32, eb, nb)[0]
    dn = SO.step(p, net, x, [-1.0, 0.0], 0.02, h, c, "device", np.float32, eb, nb)[0]
    assert hn[SO.BRAKE_STATE] == np.float32(0.5) and dn[SO.BRAKE_STATE] > np.float32(0.5)
    assert w.dyn.step(x, [-1.0, 0.0], 0.02)[0][SO.BRAKE_STATE] == np.float32(0.5)


def test_flat_ground_at_rest_has_no_suspension_derivative():
    dyn = H.RacerDubinsElevationSuspension()
    x = np.zeros(24, np.float32)
    x[SO.CG_POS_Z] = dyn.params.wheel_radius
    _, xd, y, _, _ = dyn.step(x, np.zeros(2, np.float32), 0.01)
    for i in (SO.ROLL, SO.PITCH, SO.CG_POS_Z, SO.CG_VEL_I_Z, SO.ROLL_RATE, SO.PITCH_RATE):
        assert xd[i] == 0, i
    assert y[SO.O_WF_UP] == 0 and y[SO.O_WF_FWD] == 0 and y[SO.O_WF_SIDE] == 0
    assert y[SO.O_POS_I_Z] == np.float32(dyn.params.wheel_radius)


def _plane(dyn, a, b):
    """z = a x + b y over [-20, 20]^2 at 0.25 m, with its unit normal (-a, -b, 1) / |.| in the normals map."""
    res, n = 0.25, 160
    c = -20.0 + (np.arange(n) + 0.5) * res
    X, Y = np.meshgrid(c, c)
    dyn.setElevationMap((a * X + b * Y).astype(np.float32), res, (-20.0, -20.0, 0.0))
    nv = np.array([-a, -b, 1.0]) / math.sqrt(1 + a * a + b * b)
    dyn.setNormalsMap(np.tile(nv, (n, n, 1)).astype(np.float32), res, (-20.0, -20.0, 0.0))


@pytest.mark.parametrize("a,b", [(0.04, -0.03), (-0.05, 0.02)])
def test_settles_on_a_tilted_plane(a, b):
    """At VEL_X = 0 (no c_0 drive, no gravity term) and dt = 0.01, 2000 host steps from 5 cm above the plane settle the
    car: the wheel forces fall below 1 N and roll, pitch and heave match the plane's small-angle closed form roll = b,
    pitch = -a, CG_POS_Z = r + plane(x + c_g.x, y), to second order in the slope."""
    dyn = H.RacerDubinsElevationSuspension()
    dyn.params.c_0, dyn.params.gravity = 0.0, 0.0
    _plane(dyn, a, b)
    x = np.zeros(24, np.float32)
    x[SO.POS_X], x[SO.POS_Y] = 1.0, -2.0
    cgx, r = dyn.params.c_g[0], dyn.params.wheel_radius
    x[SO.CG_POS_Z] = r + a * (1.0 + cgx) + b * -2.0 + 0.05
    h, c = dyn.initial_hidden_cell()
    for _ in range(2000):
        x, xd, y, h, c = dyn.step(x, np.zeros(2, np.float32), 0.01, h, c)
    assert max(abs(y[SO.O_WF_UP]), y[SO.O_WF_FWD], y[SO.O_WF_SIDE]) < 1.0, y[10:13]
    assert np.abs(xd[[SO.CG_VEL_I_Z, SO.ROLL_RATE, SO.PITCH_RATE]]).max() < 1e-3
    s2 = 3 * (a * a + b * b)
    assert abs(x[SO.ROLL] - b) < s2 and abs(x[SO.PITCH] + a) < s2, (x[SO.ROLL], x[SO.PITCH])
    assert abs(x[SO.CG_POS_Z] - (r + a * (1.0 + cgx) + b * -2.0)) < s2 * (1 + cgx)


# The partial maps: map y = world x - 1, and their NaN cells are row 0, which the bilinear query reads wherever world x < 16.
PARTIAL_START = (12.5, 30.0)  # rear wheels at x = 12.5, front wheels at 15.5: every wheel starts on the NaN row


def _wheel_reads(dyn, x):
    """(finite, non-finite) counts of the four wheels' height and normal queries at state x (host queries, the wheel
    positions of racer_suspension_oracle.suspension with the host's sincos)."""
    roll, pitch, yaw = float(x[SO.ROLL]), float(x[SO.PITCH]), float(x[SO.YAW])
    sr, cr, sp, cp, sy, cy = math.sin(roll), math.cos(roll), math.sin(pitch), math.cos(pitch), math.sin(yaw), math.cos(yaw)
    good = bad = 0
    for bx, by in SO.WHEELS:
        p = (cp * cy * bx + (sr * sp * cy - cr * sy) * by + x[SO.POS_X], cp * sy * bx + (sr * sp * sy + cr * cy) * by +
             x[SO.POS_Y], -sp * bx + sr * cp * by)
        for v in (dyn.tex_helper_.queryTextureAtWorldPose(0, p), dyn.normals_tex_helper_.queryTextureAtWorldPose(0, p)):
            if np.isfinite(v).all():
                good += 1
            else:
                bad += 1
    return good, bad


@pytest.mark.parametrize("maps", ["none", "partial"])
def test_finite_500_step_trajectories(maps):
    """Over the partial maps the car starts on the NaN row and drives off it: both the NaN fallbacks (height
    CG_POS_Z - wheel_radius, normal (0, 0, 1)) and the finite reads are taken, and the state stays finite."""
    w = _maps_workload(maps)
    rng = np.random.RandomState(2)
    x = w.x0[0].copy()
    x[SO.POS_X], x[SO.POS_Y] = PARTIAL_START
    h, c = w.dyn.initial_hidden_cell()
    good = bad = 0
    for _ in range(500):
        if maps == "partial":
            g, b = _wheel_reads(w.dyn, x)
            good, bad = good + g, bad + b
        x, xd, y, h, c = w.dyn.step(x, rng.uniform(0.0, 1.0, 2).astype(np.float32), 0.02, h, c)
        assert np.isfinite(x).all() and np.isfinite(xd).all() and np.isfinite(y).all()
    if maps == "partial":
        assert bad > 100 and good > 100, (good, bad)


def test_state_from_map():
    dyn = H.RacerDubinsElevationSuspension()
    keys = dict(VEL_X=2.0, VEL_Z=0.1, POS_X=1.0, POS_Y=2.0, POS_Z=0.5, OMEGA_X=0.01, OMEGA_Y=0.02, ROLL=0.05, PITCH=-0.1,
                YAW=0.3, STEER_ANGLE=0.1, STEER_ANGLE_RATE=0.2, BRAKE_STATE=0.0)
    s = dyn.stateFromMap(keys)
    cgx = dyn.params.c_g[0]
    assert s[SO.CG_POS_Z] == pytest.approx(0.5 - math.sin(-0.1) * cgx, rel=1e-6)
    assert s[SO.CG_VEL_I_Z] == pytest.approx(0.1 * math.cos(-0.1) - 2.0 * math.sin(-0.1) - 0.02 * cgx, rel=1e-5)
    assert (s[SO.UNC0:SO.UNC0 + 4] == np.float32(1e-6)).all()
    assert np.isnan(dyn.stateFromMap({k: v for k, v in keys.items() if k != "YAW"})).all()


def test_workloads_and_engine_blob_rules():
    for use_maps in (False, True):
        w = W.racer_suspension(256, 20, 4, use_maps)
        assert w.dyn.DYN_ID == 6 and w.x0.shape == (1, 24)
        assert w.dyn.tex_helper_.checkTextureUse(0) == use_maps == w.dyn.normals_tex_helper_.checkTextureUse(0)
    try:
        e = w.make_engine()
    except H.MppibError as err:
        assert "no kernel registered" not in str(err)
        pytest.skip("no GPU")
    L = H.lib()
    nb = w.dyn.normals_tex_helper_.blob()
    assert L.mppib_set_blob(e._h, H.BLOB_NORMALS_MAP, nb.ctypes.data, nb.nbytes) == 0
    short = nb[:-16].copy()
    assert L.mppib_set_blob(e._h, H.BLOB_NORMALS_MAP, short.ctypes.data, short.nbytes) != 0
    eb = w.dyn.tex_helper_.blob()  # a float map is a quarter of the bytes a float4 map of the same extent needs
    assert L.mppib_set_blob(e._h, H.BLOB_NORMALS_MAP, eb.ctypes.data, eb.nbytes) != 0
    e.close()


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _restated_rollout(w, controls):
    p = SO.Params(w.dyn.params)
    net = _net(w.dyn)
    lo, hi = np.array(p.rng_lo, np.float32), np.array(p.rng_hi, np.float32)
    cp = w.cost.params
    eb, nb = _blob(w.dyn.tex_helper_), _blob(w.dyn.normals_tex_helper_)
    x = w.x0[0].astype(np.float32)
    h, c = net.initial()
    Y = np.zeros((w.T, 28), np.float32)
    run = np.float32(0)
    f = np.float32
    for t in range(w.T):
        u = np.minimum(np.maximum(controls[t], lo), hi).astype(np.float32)
        x, _, y, h, c = SO.step(p, net, x, u, w.dt, h, c, "device", np.float32, eb, nb)
        Y[t] = y
        dv = f(y[0] - f(cp.desired_speed))
        dyaw = SO.RO.normalize_angle(f(y[5] - f(cp.desired_yaw)), np.float32)
        dy = f(y[3] - f(cp.desired_y))
        run = f(run + (f(cp.speed_coeff) * dv * dv + f(cp.yaw_coeff) * dyaw * dyaw + f(cp.lateral_coeff) * dy * dy +
                       f(cp.steer_coeff) * y[8] * y[8]))
    return Y, run / f(w.T)


def _on_discontinuity(w, Y_a, Y_b, u, t):
    """A speed-bin edge (|vx| at 0.2 / 3, racer_dubins_elevation.cu:37-39), the brake switching on (throttle command at
    0) or, over the partial maps, a wheel crossing x = 16 m, where the NaN fallback hands over to the map, at step t or the
    step before it, on either trajectory. The maps are bilinear, hence continuous, and so is every other term of the
    step."""
    for k in (t - 1, t):
        if k < 0:
            continue
        if abs(float(u[k][0])) < 1e-5:
            return True
        for Y in (Y_a, Y_b):
            vx = abs(float(Y[k][0]))
            if min(abs(vx - 0.2), abs(vx - 3.0)) < 2e-3:
                return True
            x_rear, x_front = float(Y[k][2]), float(Y[k][2]) + 2.981 * math.cos(float(Y[k][5]))
            if w.extra.get("nan_edge_x") is not None and min(abs(x_rear - 16.0), abs(x_front - 16.0)) < 0.15:
                return True
    return False


def _parity(w, e, n_check=96, tol=1e-4):
    """Every checked sample's cost within `tol` of the restatement, or, for each one outside it, the device's own
    per-step dump sums to its cost and the first step at which the dump leaves the restatement sits on a discontinuity
    of the model (_on_discontinuity)."""
    U, _ = e.solve(w.x0, w.U0)
    c, samples = e.get_costs()[0], e.get_samples()[0]
    idx = np.random.RandomState(0).choice(w.N, n_check, replace=False)
    rel, outliers = [], []
    for n in idx:
        Y, ref = _restated_rollout(w, samples[n])
        rel.append(abs(float(c[n]) - float(ref)) / max(abs(float(ref)), 1.0))
        if rel[-1] > tol:
            outliers.append((n, Y))
    rel = np.array(rel)
    print(f"{w.name}: max rel {rel.max():.2e}, median {np.median(rel):.2e}, {len(outliers)} outside {tol}")
    assert np.median(rel) < 2e-5
    if outliers:
        ix = np.array([o[0] for o in outliers])
        outs_dev, costs_dev, _ = e.sample_trajectories(w.x0[0], w.U0[0], ix)
        np.testing.assert_allclose(costs_dev.sum(axis=1), c[ix], rtol=5e-6)
        lo, hi = np.array(w.dyn.params.lim.rng_lo[:2], np.float32), np.array(w.dyn.params.lim.rng_hi[:2], np.float32)
        for k, (n, Y) in enumerate(outliers):
            d = np.abs(outs_dev[k][:, :10] - Y[:, :10]).max(axis=1)
            bad = np.nonzero(d > 1e-4)[0]
            assert bad.size > 0, (n, "cost differs, outputs agree")
            u = np.clip(samples[n], lo, hi)
            assert _on_discontinuity(w, outs_dev[k], Y, u, int(bad[0])), (n, int(bad[0]), float(d[bad[0]]))
    cc = c.astype(np.float64)
    wts = np.exp(-(cc - cc.min()) / w.lambda_)
    np.testing.assert_allclose(U[0], np.tensordot(wts / wts.sum(), samples.astype(np.float64), axes=1), atol=2e-4)
    return c


FORMS = [("H4", 4, 0), ("H8", 8, 0), ("H32_simt", 32, H.FLAG_LSTM_SIMT), ("H32_tc", 32, 0)]


def _workload(maps, hidden, colored=False, N=1024, T=40):
    w = _maps_workload(maps)
    if hidden != 4 or colored:
        v = W.racer_suspension(N, T, hidden, use_maps=False, colored=colored)
        v.dyn.tex_helper_, v.dyn.normals_tex_helper_ = w.dyn.tex_helper_, w.dyn.normals_tex_helper_
        v.x0 = w.x0
        w = v
    w.sampler.setStdDev([0.6, 0.6])
    w.sampler.setControlCostCoeff([0.0, 0.0])
    if maps == "partial":
        w.x0[0, SO.POS_X], w.x0[0, SO.POS_Y] = PARTIAL_START
        assert _wheel_reads(w.dyn, w.x0[0]) == (0, 8)  # every wheel's height and normal start on the NaN row
        w.extra["nan_edge_x"] = 16.0
    return w


@pytest.mark.gpu
@pytest.mark.parametrize("maps", ["none", "elev", "both", "partial"])
@pytest.mark.parametrize("name,hidden,flags", FORMS, ids=[f[0] for f in FORMS])
def test_k1_matches_the_restatement(name, hidden, flags, maps):
    w = _workload(maps, hidden)
    e = w.make_engine(flags=flags | H.FLAG_WRITEBACK_CONTROLS)
    _parity(w, e)
    if maps == "partial":  # the rollouts leave the NaN row: both branches of the device's fallbacks run
        outs, _, _ = e.sample_trajectories(w.x0[0], w.U0[0], np.arange(0, w.N, 64))
        assert (outs[:, -1, 2] + 2.981 > 16.5).any()  # front wheels past the last x that reads the NaN row
    e.close()


STAGING = [("resident", 0, {}), ("no_tma", H.FLAG_NO_TMA, {}), ("stream", 0, {"MPPIB_STREAM": "1"})]


@pytest.mark.gpu
@pytest.mark.parametrize("colored", [False, True], ids=["gaussian", "colored"])
@pytest.mark.parametrize("name,flags,env", STAGING, ids=[s[0] for s in STAGING])
@pytest.mark.parametrize("hidden", [4, 32])
def test_k1_staging_and_samplers(hidden, name, flags, env, colored, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    w = _workload("both", hidden, colored)
    e = w.make_engine(flags=flags | H.FLAG_WRITEBACK_CONTROLS)
    if name == "no_tma":
        assert not e.launch_info()["uses_tma"]
    _parity(w, e)
    e.close()


@pytest.mark.gpu
def test_tensor_core_form_agrees_with_simt_form():
    w = _workload("both", 32)
    a = w.make_engine()
    b = w.make_engine(flags=H.FLAG_LSTM_SIMT)
    Ua, _ = a.solve(w.x0, w.U0)
    Ub, _ = b.solve(w.x0, w.U0)
    np.testing.assert_array_equal(a.get_noise(), b.get_noise())
    ca, cb = a.get_costs(), b.get_costs()
    assert (np.abs(ca - cb) / np.maximum(np.abs(cb), 1.0)).max() < 2e-5
    np.testing.assert_allclose(Ua, Ub, atol=2e-4)
    a.close()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("maps", ["none", "both"])
def test_sampled_trajectories_match_and_sum_to_k1(maps):
    w = _workload(maps, 4)
    e = w.make_engine(flags=H.FLAG_WRITEBACK_CONTROLS)
    e.solve(w.x0, w.U0)
    c, samples = e.get_costs()[0], e.get_samples()[0]
    idx = np.arange(0, w.N, 32)
    outs, costs, _ = e.sample_trajectories(w.x0[0], w.U0[0], idx)
    np.testing.assert_allclose(costs.sum(axis=1), c[idx], rtol=5e-6)
    for k, n in enumerate(idx[:16]):
        Y, _ = _restated_rollout(w, samples[n])
        scale = np.maximum(np.abs(Y).max(axis=0), 1.0)
        assert (np.abs(outs[k][:, :27] - Y[:, :27]) / scale[:27]).max() < 2e-3, k
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("maps", ["none", "both"])
def test_device_tail_matches_the_host_twin(maps):
    w = _workload(maps, 4, T=60)
    e = w.make_engine()
    U, _ = e.solve(w.x0, w.U0)
    _, st_d, out_d = e.nominal_trajectory(w.x0, U)
    e.close()
    st_h, out_h = np.zeros((w.T, 24), np.float32), np.zeros((w.T, 28), np.float32)
    w.dyn.output_trajectory(w.x0[0], U[0], w.T, w.dt, st_h, out_h)
    for a, b in ((st_d[0][1:], st_h[1:]), (out_d[0][1:], out_h[1:])):
        scale = np.maximum(np.abs(b).max(axis=0, keepdims=True), 1.0)
        assert (np.abs(a - b) / scale).max() < 1e-3, float((np.abs(a - b) / scale).max())


@pytest.mark.gpu
def test_unsupported_paths():
    """D = 2 (Tube-MPPI, and RMPPI, which needs two distributions) is MPPIB_ERR_UNSUPPORTED for this model; RMPPI at D = 1
    is MPPIB_ERR_INVALID_ARG as for every model; mppib_set_ddp stores the weights and mppib_ddp_feedback is
    MPPIB_ERR_UNSUPPORTED (no analytic Jacobian)."""
    w = W.racer_suspension(1024, 20, 4, True)
    for flags in (0, H.FLAG_RMPPI):
        with pytest.raises(H.MppibError) as err:
            H.Engine(w.dyn, w.cost, w.sampler, w.N, w.T, 2, flags=flags)
        assert err.value.status == -2 and "num_distributions == 1" in str(err.value)
    with pytest.raises(H.MppibError) as err:
        H.Engine(w.dyn, w.cost, w.sampler, w.N, w.T, 1, flags=H.FLAG_RMPPI)
    assert err.value.status == -1
    e = w.make_engine()
    Q = np.eye(24, dtype=np.float32)
    R = np.eye(2, dtype=np.float32)
    assert H.lib().mppib_set_ddp(e._h, Q.ctypes.data, Q.ctypes.data, R.ctypes.data, 1) == 0  # weights only, as for LSTM
    xt, ut = np.tile(w.x0[0], (w.T, 1)), np.zeros((w.T, 2), np.float32)
    gains = np.zeros((w.T, 24, 2), np.float32)
    rc = H.lib().mppib_ddp_feedback(e._h, w.T, w.x0[0].ctypes.data, xt.ctypes.data, ut.ctypes.data, 0, gains.ctypes.data,
                                    None, None, None)
    assert rc == -2, rc  # MPPIB_ERR_UNSUPPORTED: no analytic Jacobian
    e.close()


@pytest.mark.gpu
def test_closed_loop_over_the_hills_holds_speed():
    """VanillaMPPI over racer_hill_maps(): after 1 s the mean speed is within 0.3 m/s of the desired 1.2 m/s, roll and pitch
    stay within 0.3 rad and the state stays finite."""
    w = W.racer_suspension(4096, 50, 4, True, colored=False)
    w.x0[0, SO.VEL_X] = 1.0
    ctrl = m.VanillaMPPIController(w.dyn, w.cost, None, w.sampler, w.dt, 1, w.lambda_, w.alpha, w.T, w.N, seed=3)
    x = w.x0[0].copy()
    h, c = w.dyn.initial_hidden_cell()
    speeds, rp = [], []
    for t in range(150):
        ctrl.computeControl(x, 1)
        u = ctrl.getControlSeq()[0].astype(np.float32)
        w.dyn.enforceConstraints(x, u)
        x, _, _, h, c = w.dyn.step(x, u, w.dt, h, c)
        ctrl.slideControlSequence(1)
        assert np.isfinite(x).all()
        speeds.append(float(x[0]))
        rp.append(max(abs(float(x[SO.ROLL])), abs(float(x[SO.PITCH]))))
    print(f"closed loop: mean speed {np.mean(speeds[50:]):.3f}, max |roll|, |pitch| {max(rp):.3f}")
    assert abs(np.mean(speeds[50:]) - 1.2) < 0.3
    assert max(rp) < 0.3


# ---- the C++ layer ---------------------------------------------------------------------------------------------------
ROOT = __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__)))
LIB_DIR = ROOT + "/mppi-generic_b200"
CPP_EXE = ROOT + "/tests/cpp/racer_suspension_example.bin"


def _build_cpp():
    import subprocess
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unused-variable", "-I", ROOT + "/include", "-c",
                           ROOT + "/tests/cpp/racer_suspension_example.cpp", "-o", CPP_EXE + ".o"])
    subprocess.check_call(["g++", CPP_EXE + ".o", "-o", CPP_EXE, "-L", LIB_DIR, "-lmppi_b200", "-Wl,-rpath," + LIB_DIR])


def _cpp_model():
    """The example's configure() in Python: the same parameters, weights and maps."""
    dyn = H.RacerDubinsElevationSuspension()
    dyn.params.spring_k, dyn.params.c_g[1] = 15000.0, 0.01
    dyn.setControlRanges([(-1.0, 1.0), (-1.0, 1.0)])
    f = np.float32
    lstm = np.zeros(dyn._lstm_block(), np.float32)
    i = np.arange(dyn._lstm_block() - 8)
    lstm[:-8] = f(0.3) * np.sin(f(0.7) * i.astype(np.float32) + f(0.1)).astype(np.float32)
    j = np.arange(8 * 20 + 20 + 20 + 1).astype(np.float32)
    dyn.setAllValues(lstm, f(0.3) * np.sin(f(0.7) * j + f(0.1)).astype(np.float32))
    X, Y = np.meshgrid(-10.0 + (np.arange(120) + 0.5) * 0.5, -15.0 + (np.arange(60) + 0.5) * 0.5)
    z = 0.4 * np.exp(-((X - 8.0) ** 2 + (Y - 1.0) ** 2) / 50.0)
    gx, gy = -z * 2 * (X - 8.0) / 50.0, -z * 2 * (Y - 1.0) / 50.0
    inv = 1.0 / np.sqrt(gx * gx + gy * gy + 1.0)
    dyn.setElevationMap(z.astype(np.float32), 0.5, (-10.0, -15.0, 0.0))
    dyn.setNormalsMap(np.stack([-gx * inv, -gy * inv, inv], -1).astype(np.float32), 0.5, (-10.0, -15.0, 0.0))
    return dyn


def test_cpp_blob_step_and_normals_match_python():
    """RacerDubinsElevationSuspension in C++ (built with plain g++ against the reference's include path) and the Python
    class write the same parameter bytes, take the same host step over the same maps (up to the maps' own float rounding)
    and query the float4 map alike."""
    import subprocess
    _build_cpp()
    out = subprocess.check_output([CPP_EXE, "blob"])
    dyn = _cpp_model()
    n = C.sizeof(H.RacerSuspensionDynParams)
    assert out[:n] == dyn.blob()
    vals = np.frombuffer(out[n:], np.float32)
    xn_c, xd_c, y_c, q_c = vals[:24], vals[24:48], vals[48:76], vals[76:80]
    x = np.zeros(24, np.float32)
    x[SO.VEL_X], x[SO.CG_POS_Z], x[SO.UNC0:SO.UNC0 + 4] = 2.0, 0.32, 1e-6
    x[SO.POS_X], x[SO.POS_Y], x[SO.YAW], x[SO.ROLL], x[SO.PITCH], x[SO.CG_POS_Z], x[SO.STEER_ANGLE_RATE] = \
        7.0, 0.5, 0.2, 0.02, -0.03, 0.45, 0.3
    xn, xd, y, _, _ = dyn.step(x, np.array([0.4, -0.2], np.float32), 0.02)
    for a, b in ((xn_c, xn), (xd_c, xd), (y_c, y)):
        np.testing.assert_allclose(a, b, rtol=1e-4, atol=1e-3)
    assert y_c[SO.O_WF_UP] != 0 and np.isfinite(y_c).all()
    np.testing.assert_allclose(q_c, dyn.getTextureHelperNormals().queryTextureAtWorldPose(0, (7.3, 0.7, 0.0)), atol=1e-6)


def test_cpp_example_links_against_the_library():
    """nm: the example needs the model's host twins and the controller's C ABI, and libmppi_b200.so defines them; without
    a device the example stops at the C ABI's NO_DEVICE error (exit code 5)."""
    import subprocess
    _build_cpp()
    und = subprocess.run(["nm", "--undefined-only", CPP_EXE + ".o"], capture_output=True, text=True, check=True).stdout
    lib = subprocess.run(["nm", "-D", "--defined-only", LIB_DIR + "/libmppi_b200.so"], capture_output=True, text=True,
                         check=True).stdout
    for sym in ("mppib_host_step_racer_suspension", "mppib_host_normals_at_world_pose", "mppib_create"):
        assert sym in und and sym in lib, sym
    p = subprocess.run([CPP_EXE], capture_output=True, text=True, timeout=900)
    if p.returncode == 5:
        assert "no CUDA device" in p.stdout
    else:
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]


@pytest.mark.gpu
def test_cpp_example_runs_vanilla_mppi_on_the_gpu():
    import subprocess
    _build_cpp()
    p = subprocess.run([CPP_EXE], capture_output=True, text=True, timeout=900)
    print(p.stdout)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "racer suspension example rc 0" in p.stdout
