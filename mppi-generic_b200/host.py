"""ctypes mirror of the reference's host-side plugin / controller interface over libmppi_b200.so.

The reference is header-only C++ (Eigen); its C++ twin here is ``include/mppi_b200/*.hpp``. This module is the same
surface for Python callers (tests, bench.py): identical class names, constructor arguments, method names and argument
meaning as the reference classes cited in each docstring. It contains NO numerics of its own: every number comes from
the C-ABI (``include/mppi_b200.h``) — the CUDA engine for the rollout-and-reduce path, and the exported host twins
(``include/mppi_b200/host_twins.h``) for the controller's CPU tail. If the library is missing, import fails loudly;
there is no Python / CPU fallback for the hot path.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import sys
import weakref
from typing import Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# MPPIB_LIB points experiments (tools/) at an alternative build of the same ABI; the product always loads the in-tree one
LIB_PATH = os.environ.get("MPPIB_LIB") or os.path.join(_HERE, "libmppi_b200.so")

MAX_C = 4  # MPPIB_MAX_CONTROL_DIM
MAX_D = 2  # MPPIB_MAX_DISTRIBUTIONS
FLT_MAX = 3.4028234663852886e38

# plugin ids (include/mppi_b200/params.h)
DYN_CARTPOLE, DYN_DOUBLE_INTEGRATOR, DYN_AUTORALLY_NN, DYN_RACER_LSTM, DYN_QUADROTOR = 0, 1, 2, 3, 4
DYN_RACER_DUBINS_ELEVATION = 5
DYN_RACER_SUSPENSION_LSTM = 6
DYN_RACER_SUSPENSION = 7
COST_CARTPOLE_QUADRATIC, COST_DI_CIRCLE, COST_AR_STANDARD, COST_RACER_QUADRATIC, COST_QUADROTOR_QUADRATIC = 0, 1, 2, 3, 4
COST_DI_ROBUST, COST_AR_ROBUST = 5, 6
COST_QUADROTOR_MAP = 7
SAMPLER_GAUSSIAN, SAMPLER_COLORED_NOISE, SAMPLER_NLN, SAMPLER_SMOOTH_MPPI = 0, 1, 2, 3
BLOB_DYN, BLOB_COST, BLOB_SAMPLER, BLOB_NN_WEIGHTS, BLOB_COSTMAP, BLOB_LSTM_WEIGHTS, BLOB_ELEVATION_MAP = range(7)
BLOB_COST_TEXTURE = 7
BLOB_NORMALS_MAP = 8
# QuadrotorMapCost's terms (host_twins.h: mppib_quadrotor_map_term)
QMAP_GATE_SIDE, QMAP_HEADING, QMAP_HEIGHT, QMAP_SPEED, QMAP_STABILIZING, QMAP_WAYPOINT = range(6)
FLAG_WRITEBACK_CONTROLS, FLAG_NO_TMA, FLAG_CURAND_HOST_API, FLAG_NO_PREFETCH, FLAG_NN_TENSOR, FLAG_RMPPI = 1, 2, 4, 8, 16, 32
FLAG_NN_MMA, FLAG_NN_FFMA2 = 64, 128
FLAG_NO_WARP_SPEC = 256
FLAG_LSTM_SIMT = 512
OPT_L2_FLUSH_BYTES = 1
OPT_COLORED_OFFSET_T = 2
OPT_P2P_ENABLE = 3
RACER_LSTM_INPUT_DIM = 4


def racer_lstm_num_params(hidden_dim: int, head_hidden: int) -> int:
    """MPPIB_RACER_LSTM_NUM_PARAMS (params.h): LSTM block (lstm_helper.cu:72-88) + head {H+4, L1, 1} (fnn_helper.cu:176-183)."""
    H, L1 = hidden_dim, head_hidden
    return 4 * H * H + 4 * H * 4 + 6 * H + (H + 4) * L1 + L1 + L1 + 1
AR_NN_NUM_PARAMS = 1412


class MppibError(RuntimeError):
    """Raised for any negative mppib_status (the reference would print and exit(): utils/gpu_err_chk.cuh:32-40)."""

    def __init__(self, status: int, what: str):
        super().__init__(f"libmppi_b200: status {status}: {what}")
        self.status = status


# ---------------------------------------------------------------------------------------------------------------
# POD blobs (field-for-field with include/mppi_b200/params.h)
class ControlLimits(C.Structure):
    _fields_ = [("rng_lo", C.c_float * MAX_C), ("rng_hi", C.c_float * MAX_C), ("deadband", C.c_float * MAX_C),
                ("zero_control", C.c_float * MAX_C)]

    def __init__(self):
        super().__init__()
        self.set_defaults()

    def set_defaults(self) -> None:
        """dynamics.cuh:99-106: unbounded ranges, zero deadband / zero control. NOTE: ctypes does not run __init__ for
        a struct nested inside another struct, so every dynamics blob calls this explicitly."""
        for i in range(MAX_C):
            self.rng_lo[i] = -FLT_MAX
            self.rng_hi[i] = FLT_MAX
            self.deadband[i] = 0.0
            self.zero_control[i] = 0.0


class CartpoleDynParams(C.Structure):
    _fields_ = [("lim", ControlLimits), ("cart_mass", C.c_float), ("pole_mass", C.c_float),
                ("pole_length", C.c_float), ("gravity", C.c_float)]


class DIDynParams(C.Structure):
    _fields_ = [("lim", ControlLimits), ("system_noise", C.c_float)]


class ARNNDynParams(C.Structure):
    _fields_ = [("lim", ControlLimits)]


class QuadrotorDynParams(C.Structure):
    _fields_ = [("lim", ControlLimits), ("tau_roll", C.c_float), ("tau_pitch", C.c_float), ("tau_yaw", C.c_float),
                ("mass", C.c_float)]


class QuadrotorCostParams(C.Structure):
    _fields_ = [("control_cost_coeff", C.c_float * MAX_C), ("discount", C.c_float), ("s_goal", C.c_float * 13),
                ("x_coeff", C.c_float), ("v_coeff", C.c_float), ("use_euler", C.c_int), ("q_coeff", C.c_float),
                ("roll_coeff", C.c_float), ("pitch_coeff", C.c_float), ("yaw_coeff", C.c_float),
                ("w_coeff", C.c_float), ("terminal_cost_coeff", C.c_float)]


class QuadrotorMapCostParams(C.Structure):
    """mppib_quadrotor_map_cost_params (params.h): QuadrotorMapCostParams without r_c1 / r_c2 / trs. updateWaypoint /
    updateGateBoundaries run in the library (mppib_host_quadrotor_map_update_*), so the C++ and Python mirrors write the same
    bytes."""
    _fields_ = [("control_cost_coeff", C.c_float * MAX_C), ("discount", C.c_float), ("attitude_coeff", C.c_float),
                ("crash_coeff", C.c_float), ("dist_to_waypoint_coeff", C.c_float), ("heading_coeff", C.c_float),
                ("heading_power", C.c_float), ("height_coeff", C.c_float), ("track_coeff", C.c_float),
                ("speed_coeff", C.c_float), ("track_slop", C.c_float), ("gate_pass_cost", C.c_float),
                ("curr_waypoint", C.c_float * 4), ("prev_waypoint", C.c_float * 4), ("curr_gate_left", C.c_float * 3),
                ("curr_gate_right", C.c_float * 3), ("prev_gate_left", C.c_float * 3), ("prev_gate_right", C.c_float * 3),
                ("end_waypoint", C.c_float * 4), ("desired_speed", C.c_float), ("gate_margin", C.c_float),
                ("min_dist_to_gate_side", C.c_float), ("track_boundary_cost", C.c_float), ("gate_width", C.c_float)]

    def set_defaults(self) -> None:
        """quadrotor_map_cost.cuh:14-60."""
        for i in range(MAX_C):
            self.control_cost_coeff[i] = 1.0
        self.discount = 1.0
        self.attitude_coeff, self.crash_coeff, self.dist_to_waypoint_coeff = 10.0, 1000.0, 0.0
        self.heading_coeff, self.heading_power, self.height_coeff = 5.0, 1.0, 5.0
        self.track_coeff, self.speed_coeff, self.track_slop, self.gate_pass_cost = 10.0, 5.0, 0.0, -150.0
        for i in range(4):
            self.end_waypoint[i] = float("nan")
        self.desired_speed, self.gate_margin, self.min_dist_to_gate_side = 5.0, 0.5, 0.5
        self.track_boundary_cost, self.gate_width = 2.5, 2.15

    def updateWaypoint(self, x: float, y: float, z: float, heading: float = 0.0) -> bool:
        rc = lib().mppib_host_quadrotor_map_update_waypoint(C.byref(self), C.c_float(x), C.c_float(y), C.c_float(z),
                                                            C.c_float(heading))
        _check(min(rc, 0))
        return rc == 1

    def updateGateBoundaries(self, left_x: float, left_y: float, left_z: float, right_x: float, right_y: float,
                             right_z: float) -> bool:
        rc = lib().mppib_host_quadrotor_map_update_gate_boundaries(
            C.byref(self), *[C.c_float(v) for v in (left_x, left_y, left_z, right_x, right_y, right_z)])
        _check(min(rc, 0))
        return rc == 1


class RacerLSTMDynParams(C.Structure):
    _fields_ = [("lim", ControlLimits), ("c_t", C.c_float * 3), ("c_b", C.c_float * 3), ("c_v", C.c_float * 3),
                ("c_0", C.c_float), ("steering_constant", C.c_float), ("steer_command_angle_scale", C.c_float),
                ("steer_angle_scale", C.c_float), ("max_steer_angle", C.c_float), ("max_steer_rate", C.c_float),
                ("steer_accel_constant", C.c_float), ("steer_accel_drag_constant", C.c_float),
                ("brake_delay_constant", C.c_float), ("brake_delay_constant_neg", C.c_float),
                ("max_brake_rate_neg", C.c_float), ("max_brake_rate_pos", C.c_float), ("wheel_base", C.c_float),
                ("low_min_throttle", C.c_float), ("gravity", C.c_float), ("gear_sign", C.c_int),
                ("clamp_ax", C.c_float), ("K_x", C.c_float), ("K_y", C.c_float), ("K_yaw", C.c_float),
                ("K_vel_x", C.c_float), ("Q_x_acc", C.c_float), ("Q_x_v", C.c_float * 3), ("Q_y_f", C.c_float),
                ("Q_omega_v", C.c_float), ("Q_omega_steering", C.c_float)]


class RacerSuspensionDynParams(C.Structure):
    """mppib_racer_suspension_dyn_params (params.h): the LSTM model's fields, then RacerDubinsElevationSuspensionParams' own
    (racer_dubins_elevation_suspension_lstm.cuh:54-63); c_g is the centre of gravity in the body frame."""
    _fields_ = RacerLSTMDynParams._fields_ + [("spring_k", C.c_float), ("drag_c", C.c_float), ("mass", C.c_float),
                                              ("I_xx", C.c_float), ("I_yy", C.c_float), ("wheel_radius", C.c_float),
                                              ("c_g", C.c_float * 3)]


class RacerRigidSuspensionDynParams(C.Structure):
    """mppib_racer_rigid_suspension_dyn_params (params.h): RacerSuspensionParams (racer_suspension.cuh:8-128) field for
    field, float3 as three floats, the derived fields included."""
    _fields_ = [("lim", ControlLimits), ("wheel_radius", C.c_float), ("mass", C.c_float), ("wheel_base", C.c_float),
                ("width", C.c_float), ("height", C.c_float), ("gravity", C.c_float), ("k_s", C.c_float * 4),
                ("c_s", C.c_float * 4), ("l_0", C.c_float * 4), ("cg_pos_wrt_base_link", C.c_float * 3),
                ("wheel_pos_wrt_base_link", (C.c_float * 3) * 4), ("Jxx", C.c_float), ("Jyy", C.c_float),
                ("Jzz", C.c_float), ("mu", C.c_float), ("v_slip", C.c_float), ("c_t", C.c_float), ("c_b", C.c_float),
                ("c_v", C.c_float), ("c_0", C.c_float), ("steering_constant", C.c_float),
                ("steer_command_angle_scale", C.c_float), ("gear_sign", C.c_int)]

    def recalcParams(self) -> None:
        """RacerSuspensionParams::recalcParams (racer_suspension.cuh:113-127): the float expressions as the reference's
        types evaluate them, the inertias in double."""
        f32 = np.float32
        wb, w, h, m, g = f32(self.wheel_base), f32(self.width), f32(self.height), f32(self.mass), f32(self.gravity)
        self.cg_pos_wrt_base_link[:] = [wb / f32(2), 0.0, f32(0.2)]
        for i in range(4):
            self.l_0[i] = f32(self.wheel_radius) + m / f32(4) * -g / f32(self.k_s[i])
        for i, (x, y) in enumerate(((wb, w / f32(2)), (wb, -w / f32(2)), (0.0, w / f32(2)), (0.0, -w / f32(2)))):
            self.wheel_pos_wrt_base_link[i][:] = [x, y, 0.0]
        d = lambda a, b: 1.0 / 12 * float(m) * float(f32(a * a + b * b))  # noqa: E731
        self.Jxx, self.Jyy, self.Jzz = d(h, w), d(h, wb), d(wb, w)


class RacerQuadraticCostParams(C.Structure):
    _fields_ = [("control_cost_coeff", C.c_float * MAX_C), ("discount", C.c_float), ("desired_speed", C.c_float),
                ("speed_coeff", C.c_float), ("desired_yaw", C.c_float), ("yaw_coeff", C.c_float),
                ("desired_y", C.c_float), ("lateral_coeff", C.c_float), ("steer_coeff", C.c_float)]


class HostLSTM(C.Structure):
    _fields_ = [("theta", C.c_void_p), ("hidden_dim", C.c_int), ("head_hidden", C.c_int), ("hidden", C.c_void_p),
                ("cell", C.c_void_p), ("map", C.c_void_p)]


class HostInitLSTM(C.Structure):
    """mppib_host_init_lstm (host_twins.h)."""
    _fields_ = [("lstm_theta", C.c_void_p), ("input_dim", C.c_int), ("hidden_dim", C.c_int), ("head_theta", C.c_void_p),
                ("head_layers", C.c_void_p), ("head_num_layers", C.c_int), ("init_len", C.c_int)]


class ElevationMapHeader(C.Structure):
    """mppib_elevation_map_header (params.h): TextureParams of the RACER models' map 0."""
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("origin", C.c_float * 3), ("rotations", C.c_float * 9),
                ("resolution", C.c_float * 3), ("use", C.c_int)]


class TwoDTextureHelper:
    """Host handle of TwoDTextureHelper<float> (utils/texture_helpers/two_d_texture_helper.cuh) for ONE map, with the
    reference's method names: setExtent / updateTexture / updateOrigin / updateRotation / updateResolution / enableTexture /
    disableTexture / checkTextureUse / queryTextureAtWorldPose. The values are kept row-major ([height][width]); blob() is
    what travels as MPPIB_BLOB_ELEVATION_MAP (copyToDevice happens when the owning model's parameters are pushed)."""

    def __init__(self):
        self.hdr = ElevationMapHeader()
        self.hdr.width = self.hdr.height = 0
        for i, v in enumerate((1, 0, 0, 0, 1, 0, 0, 0, 1)):
            self.hdr.rotations[i] = v
        for i in range(3):
            self.hdr.origin[i], self.hdr.resolution[i] = 0.0, 1.0
        self.hdr.use = 0
        self.values: Optional[np.ndarray] = None
        self._blob: Optional[np.ndarray] = None

    def setExtent(self, index: int, width: int, height: int) -> None:
        self.hdr.width, self.hdr.height = int(width), int(height)
        self._blob = None

    def updateTexture(self, index: int, values, column_major: bool = False) -> None:
        v = _f32(values).reshape(-1)
        w, h = self.hdr.width, self.hdr.height
        if v.size != w * h:
            raise ValueError(f"invalid size to updateTexture {v.size} != {w * h}")  # two_d_texture_helper.cu:27-32
        self.values = (v.reshape(w, h).T if column_major else v.reshape(h, w)).copy()
        self._blob = None

    def updateOrigin(self, index: int, origin) -> None:
        for i in range(3):
            self.hdr.origin[i] = float(origin[i])
        self._blob = None

    def updateRotation(self, index: int, rows) -> None:
        r = _f32(rows).reshape(9)
        for i in range(9):
            self.hdr.rotations[i] = float(r[i])
        self._blob = None

    def updateResolution(self, index: int, resolution) -> None:
        res = np.broadcast_to(np.asarray(resolution, np.float32), (3,))
        for i in range(3):
            self.hdr.resolution[i] = float(res[i])
        self._blob = None

    def enableTexture(self, index: int = 0) -> None:
        self.hdr.use = 1
        self._blob = None

    def disableTexture(self, index: int = 0) -> None:
        self.hdr.use = 0
        self._blob = None

    def checkTextureUse(self, index: int = 0) -> bool:
        return bool(self.hdr.use) and self.values is not None

    def blob(self) -> Optional[np.ndarray]:
        """Header + values as one byte array (None until a texture has been given)."""
        if self.values is None:
            return None
        if self._blob is None:
            self._blob = np.concatenate([np.frombuffer(bytes(self.hdr), np.uint8), self.values.reshape(-1).view(np.uint8)])
        return self._blob

    def queryTextureAtWorldPose(self, index: int, point) -> float:
        b = self.blob()
        L = lib()
        L.mppib_host_elevation_at_world_pose.restype = C.c_float
        L.mppib_host_elevation_at_world_pose.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float]
        return float(L.mppib_host_elevation_at_world_pose(b.ctypes.data, float(point[0]), float(point[1]), float(point[2])))


class TwoDTextureHelperFloat4(TwoDTextureHelper):
    """TwoDTextureHelper<float4> for ONE map (RacerDubinsElevationSuspension's normals_tex_helper_): the same methods, values
    [height][width][4]; blob() travels as MPPIB_BLOB_NORMALS_MAP and queryTextureAtWorldPose returns the four channels."""

    def updateTexture(self, index: int, values, column_major: bool = False) -> None:
        v = _f32(values).reshape(-1, 4)
        w, h = self.hdr.width, self.hdr.height
        if v.shape[0] != w * h:
            raise ValueError(f"invalid size to updateTexture {v.shape[0]} != {w * h}")  # two_d_texture_helper.cu:27-32
        self.values = (v.reshape(w, h, 4).transpose(1, 0, 2) if column_major else v.reshape(h, w, 4)).copy()
        self._blob = None

    def queryTextureAtWorldPose(self, index: int, point) -> np.ndarray:
        b = self.blob()
        out = np.zeros(4, np.float32)
        L = lib()
        L.mppib_host_normals_at_world_pose.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_void_p]
        L.mppib_host_normals_at_world_pose(b.ctypes.data, float(point[0]), float(point[1]), float(point[2]),
                                           out.ctypes.data)
        return out


class CartpoleCostParams(C.Structure):
    _fields_ = [("control_cost_coeff", C.c_float * MAX_C), ("discount", C.c_float),
                ("cart_position_coeff", C.c_float), ("cart_velocity_coeff", C.c_float),
                ("pole_angle_coeff", C.c_float), ("pole_angular_velocity_coeff", C.c_float),
                ("terminal_cost_coeff", C.c_float), ("desired_terminal_state", C.c_float * 4)]


class DICircleCostParams(C.Structure):
    _fields_ = [("control_cost_coeff", C.c_float * MAX_C), ("discount", C.c_float), ("velocity_cost", C.c_float),
                ("crash_cost", C.c_float), ("velocity_desired", C.c_float), ("inner_path_radius2", C.c_float),
                ("outer_path_radius2", C.c_float), ("angular_momentum_desired", C.c_float)]


class ARStandardCostParams(C.Structure):
    _fields_ = [("control_cost_coeff", C.c_float * MAX_C), ("discount", C.c_float), ("desired_speed", C.c_float),
                ("speed_coeff", C.c_float), ("track_coeff", C.c_float), ("max_slip_ang", C.c_float),
                ("slip_coeff", C.c_float), ("track_slop", C.c_float), ("crash_coeff", C.c_float),
                ("boundary_threshold", C.c_float), ("grid_res", C.c_int), ("r_c1", C.c_float * 3),
                ("r_c2", C.c_float * 3), ("trs", C.c_float * 3), ("l1_cost", C.c_int), ("front_d", C.c_float),
                ("back_d", C.c_float), ("map_width", C.c_int), ("map_height", C.c_int)]


class ARRobustCostParams(C.Structure):
    """mppib_ar_robust_cost_params: the ARStandardCostParams fields in the same order, then heading_coeff."""
    _fields_ = ARStandardCostParams._fields_ + [("heading_coeff", C.c_float)]


class GaussianParams(C.Structure):
    _fields_ = [("std_dev", C.c_float * (MAX_C * MAX_D)), ("control_cost_coeff", C.c_float * MAX_C),
                ("pure_noise_trajectories_percentage", C.c_float), ("std_dev_decay", C.c_float),
                ("sum_strides", C.c_int), ("use_same_noise_for_all_distributions", C.c_int),
                ("exponents", C.c_float * (MAX_C * MAX_D)), ("offset_decay_rate", C.c_float), ("fmin", C.c_float)]


class SmoothMPPIParams(C.Structure):
    """mppib_smooth_mppi_params (SmoothMPPIParams, smooth-MPPI.cuh:15-24): the Gaussian blob, then the sampler's own dt."""
    _fields_ = [("gaussian", GaussianParams), ("dt", C.c_float)]


class Desc(C.Structure):
    _fields_ = [("dynamics_id", C.c_int), ("cost_id", C.c_int), ("sampler_id", C.c_int), ("num_rollouts", C.c_int),
                ("num_timesteps", C.c_int), ("num_distributions", C.c_int), ("device", C.c_int),
                ("flags", C.c_uint), ("stream", C.c_void_p), ("rank", C.c_int), ("world_size", C.c_int),
                ("model_dims", C.c_int * 8)]


class SolveStats(C.Structure):
    _fields_ = [("baseline", C.c_float), ("normalizer", C.c_float), ("sum_w2", C.c_float), ("pad", C.c_float)]


class Timing(C.Structure):
    _fields_ = [("noise_ms", C.c_float), ("rollout_ms", C.c_float), ("reduce_ms", C.c_float),
                ("total_ms", C.c_float), ("samples", C.c_int)]


# every symbol include/mppi_b200.h and include/mppi_b200/host_twins.h declare (tests check the .so exports them all)
ABI_SYMBOLS = [
    "mppib_create", "mppib_destroy", "mppib_load_plugin", "mppib_register_pair", "mppib_set_blob", "mppib_set_solver", "mppib_seed", "mppib_burn_draws",
    "mppib_get_rng_offset", "mppib_get_derivative_mean", "mppib_set_derivative_mean", "mppib_comm_unique_id", "mppib_comm_init", "mppib_solve", "mppib_solve_async",
    "mppib_solve_wait", "mppib_set_option", "mppib_set_noise",
    "mppib_draw_noise", "mppib_rollout_only", "mppib_reduce_only", "mppib_get_costs", "mppib_get_noise",
    "mppib_get_samples", "mppib_get_weights", "mppib_enable_timing", "mppib_get_timing", "mppib_get_launch_info",
    "mppib_get_rng_info",
    "mppib_local_rollouts", "mppib_strerror", "mppib_last_error", "mppib_version",
    "mppib_host_dims", "mppib_host_enforce_constraints", "mppib_host_step", "mppib_host_smooth_controls",
    "mppib_host_slide_controls", "mppib_host_output_trajectory", "mppib_host_free_energy",
    "mppib_host_merge_records", "mppib_host_step_lstm", "mppib_host_output_trajectory_lstm",
    "mppib_host_step_racer_dubins_elevation", "mppib_host_output_trajectory_racer_dubins_elevation",
    "mppib_host_grad_racer_dubins_elevation", "mppib_host_step_racer_suspension",
    "mppib_host_output_trajectory_racer_suspension", "mppib_host_normals_at_world_pose",
    "mppib_host_state_deriv_racer_rigid_suspension", "mppib_host_step_racer_rigid_suspension",
    "mppib_host_output_trajectory_racer_rigid_suspension",
    "mppib_host_elevation_at_world_pose", "mppib_host_static_settling", "mppib_host_lstm_initialize",
    "mppib_set_rmppi", "mppib_init_eval", "mppib_set_tsallis", "mppib_sample_trajectories", "mppib_nominal_trajectory", "mppib_compute_control", "mppib_host_npz_read", "mppib_comm_p2p_handle", "mppib_comm_p2p_open", "mppib_host_rmppi_line_search_weights", "mppib_host_rmppi_candidates",
    "mppib_host_rmppi_best_index", "mppib_set_ddp", "mppib_ddp_feedback",
    "mppib_host_state_cost", "mppib_host_ar_robust_stabilizing_cost", "mppib_host_ar_robust_costmap_cost",
    "mppib_host_quadrotor_map_term", "mppib_host_quadrotor_map_dist_to_waypoint",
    "mppib_host_quadrotor_map_update_waypoint", "mppib_host_quadrotor_map_update_gate_boundaries",
]

_lib = None


def lib() -> C.CDLL:
    """Load libmppi_b200.so (built by ``__graft_entry__.build()`` / ``mppi-generic_b200/build.sh``). No fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "— the MPPI engine has no Python/CPU fallback")
    L = C.CDLL(LIB_PATH)
    fp, vp, ip = C.POINTER(C.c_float), C.c_void_p, C.POINTER(C.c_int)
    L.mppib_create.argtypes = [C.POINTER(vp), C.POINTER(Desc)]
    L.mppib_destroy.argtypes = [vp]
    L.mppib_set_blob.argtypes = [vp, C.c_int, vp, C.c_size_t]
    L.mppib_set_solver.argtypes = [vp, C.c_float, C.c_float, C.c_float]
    L.mppib_seed.argtypes = [vp, C.c_ulonglong, C.c_ulonglong]
    L.mppib_burn_draws.argtypes = [vp, C.c_int]
    L.mppib_get_rng_offset.argtypes = [vp, C.POINTER(C.c_ulonglong)]
    L.mppib_get_derivative_mean.argtypes = [vp, vp]
    L.mppib_set_derivative_mean.argtypes = [vp, vp]
    L.mppib_comm_unique_id.argtypes = [vp]
    L.mppib_comm_init.argtypes = [vp, vp]
    L.mppib_comm_p2p_handle.argtypes = [vp, vp]
    L.mppib_comm_p2p_open.argtypes = [vp, vp]
    L.mppib_solve.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, C.POINTER(SolveStats)]
    L.mppib_solve_async.argtypes = [vp, vp, vp, C.c_int, C.c_int]
    L.mppib_solve_wait.argtypes = [vp, vp, C.POINTER(SolveStats)]
    L.mppib_set_option.argtypes = [vp, C.c_int, C.c_longlong]
    L.mppib_set_noise.argtypes = [vp, vp, C.c_size_t]
    L.mppib_draw_noise.argtypes = [vp]
    L.mppib_rollout_only.argtypes = [vp, vp, vp, C.c_int, C.c_int]
    L.mppib_reduce_only.argtypes = [vp, vp, C.POINTER(SolveStats)]
    for f in ("mppib_get_costs", "mppib_get_noise", "mppib_get_samples", "mppib_get_weights"):
        getattr(L, f).argtypes = [vp, vp]
    L.mppib_enable_timing.argtypes = [vp, C.c_int]
    L.mppib_get_timing.argtypes = [vp, C.POINTER(Timing)]
    L.mppib_get_launch_info.argtypes = [vp, ip, ip, ip, ip, ip]
    L.mppib_get_rng_info.argtypes = [vp, ip, ip, ip]
    L.mppib_local_rollouts.argtypes = [vp, ip, ip]
    L.mppib_strerror.argtypes = [C.c_int]
    L.mppib_strerror.restype = C.c_char_p
    L.mppib_last_error.restype = C.c_char_p
    L.mppib_host_dims.argtypes = [C.c_int, ip, ip, ip]
    L.mppib_host_enforce_constraints.argtypes = [C.c_int, vp, vp]
    L.mppib_host_state_cost.argtypes = [C.c_int, vp, vp, vp, C.c_int, vp, vp]
    L.mppib_host_ar_robust_stabilizing_cost.argtypes = [vp, vp, vp]
    L.mppib_host_ar_robust_costmap_cost.argtypes = [vp, vp, vp, vp]
    L.mppib_host_quadrotor_map_term.argtypes = [vp, C.c_int, vp, vp]
    L.mppib_host_quadrotor_map_dist_to_waypoint.argtypes = [vp, vp]
    L.mppib_host_quadrotor_map_dist_to_waypoint.restype = C.c_float
    L.mppib_host_quadrotor_map_update_waypoint.argtypes = [vp] + [C.c_float] * 4
    L.mppib_host_quadrotor_map_update_gate_boundaries.argtypes = [vp] + [C.c_float] * 6
    L.mppib_host_step.argtypes = [C.c_int, vp, vp, vp, vp, C.c_float, vp, vp, vp]
    L.mppib_host_smooth_controls.argtypes = [vp, vp, C.c_int, C.c_int]
    L.mppib_host_smooth_controls.restype = None
    L.mppib_host_slide_controls.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp]
    L.mppib_host_slide_controls.restype = None
    L.mppib_host_output_trajectory.argtypes = [C.c_int, vp, vp, vp, vp, C.c_int, C.c_float, vp, vp]
    L.mppib_host_step_lstm.argtypes = [vp, C.POINTER(HostLSTM), vp, vp, C.c_float, vp, vp, vp]
    L.mppib_host_output_trajectory_lstm.argtypes = [vp, C.POINTER(HostLSTM), vp, vp, C.c_int, C.c_float, vp, vp]
    L.mppib_host_step_racer_dubins_elevation.argtypes = [vp, vp, vp, vp, C.c_float, vp, vp, vp]
    L.mppib_host_output_trajectory_racer_dubins_elevation.argtypes = [vp, vp, vp, vp, C.c_int, C.c_float, vp, vp]
    L.mppib_host_grad_racer_dubins_elevation.argtypes = [vp, vp, vp, vp, vp]
    L.mppib_host_step_racer_suspension.argtypes = [vp, C.POINTER(HostLSTM), vp, vp, vp, C.c_float, vp, vp, vp]
    L.mppib_host_output_trajectory_racer_suspension.argtypes = [vp, C.POINTER(HostLSTM), vp, vp, vp, C.c_int, C.c_float,
                                                                 vp, vp]
    L.mppib_host_state_deriv_racer_rigid_suspension.argtypes = [vp, vp, vp, vp, vp, vp]
    L.mppib_host_step_racer_rigid_suspension.argtypes = [vp, vp, vp, C.c_float, vp, vp, vp]
    L.mppib_host_output_trajectory_racer_rigid_suspension.argtypes = [vp, vp, vp, C.c_int, C.c_float, vp, vp]
    L.mppib_set_rmppi.argtypes = [vp, C.c_float, vp]
    L.mppib_set_tsallis.argtypes = [vp, C.c_float, C.c_float]
    L.mppib_init_eval.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, C.c_int, vp]
    L.mppib_host_rmppi_line_search_weights.argtypes = [C.c_int, vp]
    L.mppib_host_rmppi_line_search_weights.restype = None
    L.mppib_host_rmppi_candidates.argtypes = [C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, vp]
    L.mppib_host_rmppi_candidates.restype = None
    L.mppib_host_rmppi_best_index.argtypes = [vp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, vp]
    L.mppib_host_free_energy.argtypes = [C.POINTER(SolveStats), C.c_int, C.c_float, vp]
    L.mppib_host_free_energy.restype = None
    L.mppib_host_merge_records.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, vp]
    L.mppib_host_npz_read.argtypes = [C.c_char_p, C.c_char_p, vp, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int * 4),
                                      ip]
    L.mppib_sample_trajectories.argtypes = [vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp]
    L.mppib_nominal_trajectory.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.mppib_compute_control.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, C.POINTER(SolveStats)]
    L.mppib_load_plugin.argtypes = [C.c_char_p]
    L.mppib_set_ddp.argtypes = [vp, vp, vp, vp, C.c_int]
    L.mppib_ddp_feedback.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, vp]
    _lib = L
    return L


def _check(rc: int) -> None:
    if rc != 0:
        L = lib()
        msg = (L.mppib_last_error() or b"").decode() or (L.mppib_strerror(rc) or b"").decode()
        raise MppibError(rc, msg)


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# ---------------------------------------------------------------------------------------------------------------
# Plugins — host objects that own the POD parameters, like the reference's host classes do
class _Dynamics:
    """Base of the dynamics plugins (include/mppi/dynamics/dynamics.cuh:67-68). Subclasses set DYN_ID / dims / params."""
    DYN_ID = -1
    STATE_DIM = CONTROL_DIM = OUTPUT_DIM = 0

    def __init__(self):
        self.params = None
        self.nn_theta: Optional[np.ndarray] = None

    def model_dims(self) -> Sequence[int]:
        """Constructor-time architecture arguments that size the kernel (mppib_desc.model_dims)."""
        return ()

    def output_trajectory(self, x0, u, T: int, dt: float, states: np.ndarray, outputs: np.ndarray) -> None:
        """Controller::computeOutputTrajectoryHelper (controller.cuh:643-663) with this model's host step."""
        _check(lib().mppib_host_output_trajectory(self.DYN_ID, C.byref(self.params), _ptr(self.nn_theta),
                                                  _ptr(_f32(x0)), _ptr(u), T, C.c_float(dt), _ptr(states),
                                                  _ptr(outputs)))

    def enforceLeash(self, state_true, state_nominal, leash_values) -> np.ndarray:
        """Dynamics::enforceLeash (dynamics.cuh:448-466): component-wise pull of the planner's initial state towards the
        true one. Models with non-Euclidean states override it (RacerDubins)."""
        t, n, l = _f32(state_true), _f32(state_nominal), _f32(leash_values)
        leashed = t + np.clip(n - t, -l, l)
        return np.where(l < np.abs(n - t), leashed, n).astype(np.float32)

    # dynamics.cuh:163-175
    def setControlRanges(self, control_rngs: Sequence[Sequence[float]]):
        for i, (lo, hi) in enumerate(control_rngs):
            self.params.lim.rng_lo[i] = lo
            self.params.lim.rng_hi[i] = hi

    def setControlDeadbands(self, deadband: Sequence[float]):
        for i, v in enumerate(deadband):
            self.params.lim.deadband[i] = v

    @property
    def zero_control_(self) -> np.ndarray:
        return np.array([self.params.lim.zero_control[i] for i in range(self.CONTROL_DIM)], dtype=np.float32)

    def getZeroState(self) -> np.ndarray:
        return np.zeros(self.STATE_DIM, dtype=np.float32)

    def blob(self) -> bytes:
        return bytes(self.params)

    # host twins (dynamics.cuh:250-300)
    def enforceConstraints(self, state: np.ndarray, control: np.ndarray) -> None:
        u = _f32(control)
        _check(lib().mppib_host_enforce_constraints(self.DYN_ID, C.byref(self.params), _ptr(u)))
        control[...] = u

    def step(self, state, control, dt: float):
        """Returns (next_state, state_der, output) — Dynamics::step host twin (dynamics.cuh:283-290)."""
        x, u = _f32(state), _f32(control)
        xn = np.zeros(self.STATE_DIM, np.float32)
        xd = np.zeros(self.STATE_DIM, np.float32)
        y = np.zeros(self.OUTPUT_DIM, np.float32)
        _check(lib().mppib_host_step(self.DYN_ID, C.byref(self.params), _ptr(self.nn_theta), _ptr(x), _ptr(u),
                                     C.c_float(dt), _ptr(xn), _ptr(xd), _ptr(y)))
        return xn, xd, y


class CartpoleDynamics(_Dynamics):
    """dynamics/cartpole/cartpole_dynamics.cuh:44-52 — CartpoleDynamics(cart_mass, pole_mass, pole_length)."""
    DYN_ID, STATE_DIM, CONTROL_DIM, OUTPUT_DIM = DYN_CARTPOLE, 4, 1, 4

    def __init__(self, cart_mass: float = 1.0, pole_mass: float = 1.0, pole_length: float = 1.0):
        super().__init__()
        self.params = CartpoleDynParams()
        self.params.lim.set_defaults()
        self.params.cart_mass, self.params.pole_mass, self.params.pole_length = cart_mass, pole_mass, pole_length
        self.params.gravity = 9.81  # cartpole_dynamics.cuh:101


class DoubleIntegratorDynamics(_Dynamics):
    """dynamics/double_integrator/di_dynamics.cuh — DoubleIntegratorDynamics(system_noise)."""
    DYN_ID, STATE_DIM, CONTROL_DIM, OUTPUT_DIM = DYN_DOUBLE_INTEGRATOR, 4, 2, 4

    def __init__(self, system_noise: float = 1.0):
        super().__init__()
        self.params = DIDynParams()
        self.params.lim.set_defaults()
        self.params.system_noise = system_noise


class QuadrotorDynamics(_Dynamics):
    """dynamics/quadrotor/quadrotor_dynamics.cuh:69-… — QuadrotorDynamics() / QuadrotorDynamics(control_rngs).
    State POS(3) VEL(3) QUAT_W..Z ANG_VEL(3); controls ANG_RATE_X/Y/Z, THRUST."""
    DYN_ID, STATE_DIM, CONTROL_DIM, OUTPUT_DIM = DYN_QUADROTOR, 13, 4, 13
    GRAVITY = 9.81  # utils/math_utils.h:45

    def __init__(self, control_rngs: Optional[Sequence[Sequence[float]]] = None, mass: float = 1.0):
        super().__init__()
        self.params = QuadrotorDynParams()
        self.params.lim.set_defaults()
        self.params.tau_roll = self.params.tau_pitch = self.params.tau_yaw = 0.25
        self.params.mass = mass
        if control_rngs is not None:  # quadrotor_dynamics.cu:4-9
            self.setControlRanges(control_rngs)
        else:  # quadrotor_dynamics.cu:11-19: thrust in [0, 36]
            self.params.lim.rng_lo[3], self.params.lim.rng_hi[3] = 0.0, 36.0
        self.params.lim.zero_control[3] = self.GRAVITY

    def getZeroState(self) -> np.ndarray:  # quadrotor_dynamics.cu:200-205
        z = np.zeros(self.STATE_DIM, dtype=np.float32)
        z[6] = 1.0
        return z


class NeuralNetModel(_Dynamics):
    """dynamics/autorally/ar_nn_model.cuh — NeuralNetModel<7,2,3>(control_rngs); 6-32-32-4 tanh network."""
    DYN_ID, STATE_DIM, CONTROL_DIM, OUTPUT_DIM = DYN_AUTORALLY_NN, 7, 2, 8
    LAYERS = (6, 32, 32, 4)

    def __init__(self, control_rngs: Optional[Sequence[Sequence[float]]] = None):
        super().__init__()
        self.params = ARNNDynParams()
        self.params.lim.set_defaults()
        if control_rngs is not None:
            self.setControlRanges(control_rngs)
        self.nn_theta = np.zeros(AR_NN_NUM_PARAMS, np.float32)

    def updateModel(self, description: Sequence[int], data) -> None:
        """ar_nn_model.cu:40-45 -> FNNHelper::updateModel (fnn_helper.cu:218-257): packed W (row-major out x in), b per layer."""
        if tuple(description) != self.LAYERS:
            raise ValueError("Invalid model trying to to be set for NN")  # fnn_helper.cu:224-227
        data = _f32(data).ravel()
        if data.size != AR_NN_NUM_PARAMS or not np.all(np.isfinite(data)):
            raise ValueError("NN parameter vector must hold 1412 finite floats")
        self.nn_theta = data.copy()

    def loadParams(self, model_path: str) -> None:
        """ar_nn_model.cu:58-61 -> FNNHelper::loadParams (fnn_helper.cu:44-127): npz arrays "dynamics_W<i>" (out x in) and
        "dynamics_b<i>", i = 1..; read through the library's own npz reader (mppib_host_npz_read) like the C++ mirror."""
        layers, chunks, i = [], [], 1
        while True:
            try:
                b = npz_read(model_path, f"dynamics_b{i}")
            except MppibError:
                if i == 1:
                    raise
                break
            W_ = npz_read(model_path, f"dynamics_W{i}")
            if i == 1:
                layers.append(W_.size // b.size)
            layers.append(b.size)
            chunks += [W_.ravel(), b.ravel()]
            i += 1
        self.updateModel(layers, np.concatenate(chunks))


def _npz_has(path: str, name: str) -> bool:
    try:
        npz_read(path, name)
        return True
    except MppibError:
        return False


def npz_read(path: str, name: str) -> np.ndarray:
    """One array of a .npz archive through mppib_host_npz_read (float32, original shape)."""
    count, ndim = C.c_size_t(), C.c_int()
    shape = (C.c_int * 4)()
    _check(lib().mppib_host_npz_read(path.encode(), name.encode(), None, 0, C.byref(count), C.byref(shape), C.byref(ndim)))
    out = np.empty(count.value, np.float32)
    _check(lib().mppib_host_npz_read(path.encode(), name.encode(), _ptr(out), out.size, None, None, None))
    return out.reshape([shape[i] for i in range(ndim.value)])


class RacerDubinsElevation(_Dynamics):
    """dynamics/racer_dubins/racer_dubins_elevation.cuh — RacerDubinsElevation() / RacerDubinsElevation(params): the
    parametric RACER vehicle (S19 C2 O28) with first-order steering and no per-sample memory, so Tube-MPPI and RMPPI roll it
    out. Its blob is RacerDubinsElevationParams (params.h: mppib_racer_dubins_elevation_dyn_params). Elevation map:
    ``getTextureHelper()`` / ``setElevationMap``."""
    DYN_ID, STATE_DIM, CONTROL_DIM, OUTPUT_DIM = DYN_RACER_DUBINS_ELEVATION, 19, 2, 28

    def enforceLeash(self, state_true, state_nominal, leash_values) -> np.ndarray:
        """RacerDubinsImpl::enforceLeash (racer_dubins.cu:177-230): x / y leashed in the body frame of the true state, yaw by
        its shortest angular distance (and re-normalised), the rest component-wise; starts from state_true."""
        YAW, PX, PY = 1, 2, 3  # racer_dubins.cuh state indices: VEL_X, YAW, POS_X, POS_Y, ...
        t, n, l = _f32(state_true), _f32(state_nominal), _f32(leash_values)
        f32, pi = np.float32, np.float32(math.pi)

        def normalize(a):  # angle_utils.cuh:20-26
            r = np.fmod(f32(a + pi), f32(2.0) * pi)
            return f32(r + pi) if r <= 0 else f32(r - pi)
        out = t.copy()
        dx, dy = n[PX] - t[PX], n[PY] - t[PY]
        cy, sy = f32(math.cos(t[YAW])), f32(math.sin(t[YAW]))
        dxb = np.clip(dx * cy + dy * sy, -l[PX], l[PX])
        dyb = np.clip(-dx * sy + dy * cy, -l[PY], l[PY])
        out[PX] += dxb * cy - dyb * sy
        out[PY] += dxb * sy + dyb * cy
        for i in range(self.STATE_DIM):
            if i in (PX, PY):
                continue
            diff = normalize(n[i] - t[i]) if i == YAW else n[i] - t[i]
            if l[i] < abs(diff):
                out[i] = t[i] + np.clip(diff, -l[i], l[i])
                if i == YAW:
                    out[i] = normalize(out[i])
            else:
                out[i] = n[i]
        return out.astype(np.float32)

    def __init__(self, params: Optional[RacerLSTMDynParams] = None):
        super().__init__()
        p = RacerLSTMDynParams()
        p.lim.set_defaults()
        # racer_dubins.cuh:78-104, racer_dubins_elevation.cuh:47-59
        for i, v in enumerate((1.3, 2.6, 3.9)):
            p.c_t[i] = v
        for i, v in enumerate((2.5, 3.5, 4.5)):
            p.c_b[i] = v
        for i, v in enumerate((3.7, 4.7, 5.7)):
            p.c_v[i] = v
        p.c_0 = 4.9
        p.steering_constant, p.steer_command_angle_scale, p.steer_angle_scale = 0.6, 5.0, -9.1
        p.max_steer_angle, p.max_steer_rate = 0.5, 5.0
        p.steer_accel_constant, p.steer_accel_drag_constant = 12.1, 1.0
        p.brake_delay_constant, p.brake_delay_constant_neg = 6.6, 8.2
        p.max_brake_rate_neg, p.max_brake_rate_pos = 0.9, 0.33
        p.wheel_base, p.low_min_throttle, p.gravity, p.gear_sign = 0.3, 0.13, -9.81, 1
        p.clamp_ax = 5.5
        p.K_x = p.K_y = p.K_yaw = p.K_vel_x = 1.0
        p.Q_x_acc = 1.0
        for i, v in enumerate((41.74219, -0.8187027, -2.2131343)):
            p.Q_x_v[i] = v
        p.Q_y_f, p.Q_omega_v, p.Q_omega_steering = 0.1, 0.001, 0.0
        self.params = p
        if params is not None:
            C.memmove(C.byref(self.params), C.byref(params), C.sizeof(RacerLSTMDynParams))
        self.tex_helper_ = TwoDTextureHelper()  # racer_dubins_elevation.cuh: tex_helper_ (map 0 = elevation)

    def getParams(self) -> RacerLSTMDynParams:
        out = RacerLSTMDynParams()
        C.memmove(C.byref(out), C.byref(self.params), C.sizeof(RacerLSTMDynParams))
        return out

    def setParams(self, params: RacerLSTMDynParams) -> None:
        C.memmove(C.byref(self.params), C.byref(params), C.sizeof(RacerLSTMDynParams))

    def getTextureHelper(self) -> "TwoDTextureHelper":
        return self.tex_helper_

    def setElevationMap(self, values, resolution, origin=(0.0, 0.0, 0.0), rotation=None, enable: bool = True) -> None:
        """Convenience over the texture helper: values [height][width] (row i = y cell, column j = x cell)."""
        v = _f32(values)
        t = self.tex_helper_
        t.setExtent(0, v.shape[1], v.shape[0])
        t.updateTexture(0, v)
        t.updateResolution(0, resolution)
        t.updateOrigin(0, origin)
        if rotation is not None:
            t.updateRotation(0, rotation)
        t.enableTexture(0) if enable else t.disableTexture(0)

    def staticSettling(self, yaw: float, x: float, y: float, roll: float = 0.0, pitch: float = 0.0):
        """RACER::computeStaticSettling on the host (racer_dubins.cu:359-434): returns (roll, pitch, height)."""
        L = lib()
        L.mppib_host_static_settling.restype = C.c_float
        L.mppib_host_static_settling.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float, C.POINTER(C.c_float),
                                                 C.POINTER(C.c_float)]
        b = self.tex_helper_.blob()
        r, p_ = C.c_float(roll), C.c_float(pitch)
        h = L.mppib_host_static_settling(None if b is None else b.ctypes.data, yaw, x, y, C.byref(r), C.byref(p_))
        return r.value, p_.value, float(h)

    def _map_ptr(self):
        b = self.tex_helper_.blob()
        return None if b is None else b.ctypes.data

    def step(self, state, control, dt: float):
        """Host step (racer_dubins_elevation.cu:229-255); returns (next_state, state_der, output)."""
        x, u = _f32(state), _f32(control)
        xn, xd, y = np.zeros(19, np.float32), np.zeros(19, np.float32), np.zeros(28, np.float32)
        _check(lib().mppib_host_step_racer_dubins_elevation(C.addressof(self.params), self._map_ptr(), _ptr(x), _ptr(u),
                                                             dt, _ptr(xn), _ptr(xd), _ptr(y)))
        return xn, xd, y

    def computeGrad(self, state, control):
        """RacerDubinsElevationImpl::computeGrad (racer_dubins_elevation.cu:257-334): returns (A [19][19], B [19][2])."""
        A, B = np.zeros((19, 19), np.float32), np.zeros((19, 2), np.float32)
        _check(lib().mppib_host_grad_racer_dubins_elevation(C.addressof(self.params), _ptr(_f32(state)), _ptr(_f32(control)),
                                                             _ptr(A), _ptr(B)))
        return A, B

    def output_trajectory(self, x0, u, T: int, dt: float, states: np.ndarray, outputs: np.ndarray) -> None:
        _check(lib().mppib_host_output_trajectory_racer_dubins_elevation(C.addressof(self.params), self._map_ptr(),
                                                                          _ptr(_f32(x0)), _ptr(_f32(u)), T, dt,
                                                                          _ptr(states), _ptr(outputs)))


class RacerDubinsElevationLSTMSteering(RacerDubinsElevation):
    """dynamics/racer_dubins/racer_dubins_elevation_lstm_steering.cuh:34-49 —
    RacerDubinsElevationLSTMSteering(init_input_dim, init_hidden_dim, init_output_layers, input_dim, hidden_dim,
    output_layers, init_len). The prediction LSTM (input_dim must be 4, output_layers = [hidden_dim + 4, L1, 1]) runs
    inside the rollout; the init network (LSTMLSTMHelper) only produces the initial hidden / cell state from a history
    buffer on the host (updateFromBuffer, :215-232) and is represented here by that state itself
    (``setInitialHiddenCell``), or computed by the init network itself (``setAllValuesInit`` / ``loadParamsInit`` +
    ``initializeLSTM`` / ``updateFromBuffer``). Elevation map: ``getTextureHelper()`` / ``setElevationMap``."""
    DYN_ID, STATE_DIM, CONTROL_DIM, OUTPUT_DIM = DYN_RACER_LSTM, 19, 2, 28

    def __init__(self, init_input_dim: int = 3, init_hidden_dim: int = 20, init_output_layers: Sequence[int] = (23, 100, 8),
                 input_dim: int = 4, hidden_dim: int = 4, output_layers: Sequence[int] = (8, 20, 1), init_len: int = 11):
        super().__init__()
        output_layers = tuple(output_layers)
        if input_dim != RACER_LSTM_INPUT_DIM:
            raise ValueError("the steering LSTM takes 4 inputs (lstm_steering.cu:148-151)")
        if len(output_layers) != 3 or output_layers[0] != hidden_dim + input_dim or output_layers[2] != 1:
            raise ValueError("output_layers must be [hidden_dim + 4, L1, 1] (lstm_helper.cu:41)")
        if tuple(init_output_layers)[-1] != 2 * hidden_dim:
            raise ValueError("init network must output 2 * hidden_dim values (lstm_lstm_helper.cu:11)")
        self.hidden_dim, self.head_hidden = hidden_dim, output_layers[1]
        # the init network (LSTMLSTMHelper::init_model_, lstm_lstm_helper.cu:4-12): host-only, zero-initialised like the
        # reference's constructor leaves it
        self.init_input_dim, self.init_hidden_dim, self.init_len = init_input_dim, init_hidden_dim, init_len
        self.init_output_layers = tuple(int(v) for v in init_output_layers)
        if self.init_output_layers[0] != init_hidden_dim + init_input_dim:
            raise ValueError("init_output_layers[0] must be init_hidden_dim + init_input_dim (lstm_helper.cu:41)")
        Hi, Ii = init_hidden_dim, init_input_dim
        self.init_lstm_theta = np.zeros(4 * Hi * Hi + 4 * Hi * Ii + 6 * Hi, np.float32)
        self.init_head_theta = np.zeros(sum(a * b + b for a, b in zip(self.init_output_layers[:-1],
                                                                     self.init_output_layers[1:])), np.float32)
        self.lstm_theta = np.zeros(racer_lstm_num_params(self.hidden_dim, self.head_hidden), np.float32)

    def model_dims(self) -> Sequence[int]:
        return (self.hidden_dim, self.head_hidden)

    def _lstm_block(self) -> int:
        H = self.hidden_dim
        return 4 * H * H + 4 * H * RACER_LSTM_INPUT_DIM + 6 * H

    def setAllValues(self, lstm, output) -> None:
        """LSTMHelper::setAllValues(lstm, output) (lstm_helper.cuh:65-72): packed LSTM weights incl. the initial hidden /
        cell vectors, then the packed head."""
        lstm, output = _f32(lstm).ravel(), _f32(output).ravel()
        if lstm.size != self._lstm_block() or lstm.size + output.size != self.lstm_theta.size:
            raise ValueError("wrong number of LSTM / head parameters")
        if not (np.all(np.isfinite(lstm)) and np.all(np.isfinite(output))):
            raise ValueError("LSTM parameters must be finite")
        self.lstm_theta = np.concatenate([lstm, output]).astype(np.float32)

    def loadParamsLSTM(self, model_path: str, prefix: str = "") -> None:
        """LSTMHelper::loadParams (utils/nn_helpers/lstm_helper.cu:496-585) for the prediction network: npz arrays
        "<prefix>lstm/weight_hh_l0" [4H][H], "lstm/weight_ih_l0" [4H][4], "lstm/bias_hh_l0" + "lstm/bias_ih_l0" [4H] in
        PyTorch's gate order (input, forget, cell, output) and the head as "<prefix>output/dynamics_W<i>" / "_b<i>"; a leading
        "model/" is tried like the reference does (:520-523). The packed order here is the reference's i, f, o, c
        (lstm_helper.cu:72-88). The initial hidden / cell state (the init network's output) is left untouched."""
        if prefix and not prefix.endswith("/"):
            prefix += "/"
        try:
            npz_read(model_path, "model/" + prefix + "lstm/weight_hh_l0")
            prefix = "model/" + prefix
        except MppibError:
            pass
        H, I = self.hidden_dim, 4
        whh = npz_read(model_path, prefix + "lstm/weight_hh_l0").astype(np.float64)
        wih = npz_read(model_path, prefix + "lstm/weight_ih_l0").astype(np.float64)
        bias = (npz_read(model_path, prefix + "lstm/bias_hh_l0").astype(np.float64) +
                npz_read(model_path, prefix + "lstm/bias_ih_l0").astype(np.float64))
        if whh.shape != (4 * H, H) or wih.shape != (4 * H, I) or bias.shape != (4 * H,):
            raise ValueError(f"LSTM arrays do not match hidden_dim = {H}, input_dim = {I}")
        order = (0, 1, 3, 2)  # file blocks i, f, c(g), o -> packed i, f, o, c
        lstm = np.concatenate([np.concatenate([whh[k * H:(k + 1) * H].ravel() for k in order]),
                               np.concatenate([wih[k * H:(k + 1) * H].ravel() for k in order]),
                               np.concatenate([bias[k * H:(k + 1) * H] for k in order]),
                               self.lstm_theta[self._lstm_block() - 2 * H:self._lstm_block()]])
        head, i = [], 1
        while True:
            try:
                b = npz_read(model_path, f"{prefix}output/dynamics_b{i}")
            except MppibError:
                if i == 1:
                    raise
                break
            head += [npz_read(model_path, f"{prefix}output/dynamics_W{i}").ravel(), b.ravel()]
            i += 1
        self.setAllValues(lstm, np.concatenate(head))

    # ---- the init network (LSTMLSTMHelper) ---------------------------------------------------------------------------------
    def setAllValuesInit(self, lstm, output) -> None:
        """getInitModel()->setAllValues(lstm, output): the init LSTM block (lstm_helper.cu:72-88 order, with its own initial
        hidden / cell) and its head (fnn_helper.cu:176-183)."""
        lstm, output = _f32(lstm).ravel(), _f32(output).ravel()
        if lstm.size != self.init_lstm_theta.size or output.size != self.init_head_theta.size:
            raise ValueError(f"init network: expected {self.init_lstm_theta.size} + {self.init_head_theta.size} values")
        self.init_lstm_theta, self.init_head_theta = lstm.copy(), output.copy()

    def loadParamsInit(self, model_path: str, prefix: str = "") -> None:
        """LSTMLSTMHelper::loadParams (lstm_lstm_helper.cu:101-118): the "<prefix>init_" arrays of the npz file — same
        names and PyTorch gate order as the prediction network (loadParamsLSTM), head of any depth — and "init_length"
        (+ 1, :33-38) when the file has it."""
        if prefix and not prefix.endswith("/"):
            prefix += "/"
        try:
            npz_read(model_path, "model/" + prefix + "init_lstm/weight_hh_l0")
            prefix = "model/" + prefix
        except MppibError:
            pass
        ip = prefix + "init_"
        H, I = self.init_hidden_dim, self.init_input_dim
        whh = npz_read(model_path, ip + "lstm/weight_hh_l0").astype(np.float64)
        wih = npz_read(model_path, ip + "lstm/weight_ih_l0").astype(np.float64)
        bias = (npz_read(model_path, ip + "lstm/bias_hh_l0").astype(np.float64) +
                npz_read(model_path, ip + "lstm/bias_ih_l0").astype(np.float64))
        if whh.shape != (4 * H, H) or wih.shape != (4 * H, I) or bias.shape != (4 * H,):
            raise ValueError(f"init LSTM arrays do not match init_hidden_dim = {H}, init_input_dim = {I}")
        order = (0, 1, 3, 2)  # file blocks i, f, c(g), o -> packed i, f, o, c
        lstm = np.concatenate([np.concatenate([whh[k * H:(k + 1) * H].ravel() for k in order]),
                               np.concatenate([wih[k * H:(k + 1) * H].ravel() for k in order]),
                               np.concatenate([bias[k * H:(k + 1) * H] for k in order]),
                               self.init_lstm_theta[-2 * H:]])
        head, i = [], 1
        while True:
            try:
                b = npz_read(model_path, f"{ip}output/dynamics_b{i}")
            except MppibError:
                if i == 1:
                    raise
                break
            head += [npz_read(model_path, f"{ip}output/dynamics_W{i}").ravel(), b.ravel()]
            i += 1
        self.setAllValuesInit(lstm, np.concatenate(head))
        try:
            self.init_len = int(npz_read(model_path, "init_length").ravel()[0]) + 1
        except MppibError:
            pass

    def initializeLSTM(self, buffer) -> None:
        """LSTMLSTMHelper::initializeLSTM (lstm_lstm_helper.cu:50-73). buffer [init_input_dim][cols] like the reference's
        matrix (one column per past time step, cols >= init_len): runs the init network over the last init_len columns and
        installs its output as the prediction LSTM's initial hidden / cell state."""
        b = _f32(buffer)
        if b.ndim != 2 or b.shape[0] != self.init_input_dim or b.shape[1] < self.init_len:
            raise ValueError(f"buffer must be [{self.init_input_dim}][>= {self.init_len}]")
        cols = np.ascontiguousarray(b.T)  # [cols][input_dim]
        layers = np.asarray(self.init_output_layers, np.int32)
        net = HostInitLSTM(self.init_lstm_theta.ctypes.data, self.init_input_dim, self.init_hidden_dim,
                           self.init_head_theta.ctypes.data, layers.ctypes.data, len(layers), self.init_len)
        out = np.zeros(2 * self.hidden_dim, np.float32)
        L = lib()
        L.mppib_host_lstm_initialize.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        _check(L.mppib_host_lstm_initialize(C.byref(net), cols.ctypes.data, cols.shape[0], out.ctypes.data))
        self.setInitialHiddenCell(out[:self.hidden_dim], out[self.hidden_dim:])

    def updateFromBuffer(self, buffer: dict) -> bool:
        """racer_dubins_elevation_lstm_steering.cu:215-233: rows STEER_ANGLE * 0.2, STEER_ANGLE_RATE * 0.2, CAN_STEER_CMD of
        the history buffer feed the init network. Returns False when a key is missing (like the reference). The new initial
        state reaches an existing engine with the next push of the model's parameters (Controller::setParams)."""
        keys = ("STEER_ANGLE", "STEER_ANGLE_RATE", "CAN_STEER_CMD")
        if any(k not in buffer for k in keys):
            return False
        init_buffer = np.stack([_f32(buffer["STEER_ANGLE"]) * np.float32(0.2), _f32(buffer["STEER_ANGLE_RATE"]) * np.float32(0.2),
                                _f32(buffer["CAN_STEER_CMD"])])
        self.initializeLSTM(init_buffer)
        return True

    def setInitialHiddenCell(self, hidden, cell) -> None:
        """LSTMHelper::updateLSTMInitialStates (lstm_helper.cu:98-110)."""
        H, base = self.hidden_dim, self._lstm_block() - 2 * self.hidden_dim
        self.lstm_theta[base:base + H] = _f32(hidden)
        self.lstm_theta[base + H:base + 2 * H] = _f32(cell)

    def _host_net(self, hidden: np.ndarray, cell: np.ndarray) -> HostLSTM:
        b = self.tex_helper_.blob()
        return HostLSTM(self.lstm_theta.ctypes.data, self.hidden_dim, self.head_hidden, hidden.ctypes.data,
                        cell.ctypes.data, None if b is None else b.ctypes.data)

    def initial_hidden_cell(self):
        H, base = self.hidden_dim, self._lstm_block() - 2 * self.hidden_dim
        return self.lstm_theta[base:base + H].copy(), self.lstm_theta[base + H:base + 2 * H].copy()

    def step(self, state, control, dt: float, hidden=None, cell=None):
        """Host step; returns (next_state, state_der, output, hidden, cell)."""
        h0, c0 = self.initial_hidden_cell()
        h = h0 if hidden is None else _f32(hidden).copy()
        c = c0 if cell is None else _f32(cell).copy()
        x, u = _f32(state), _f32(control)
        xn, xd, y = np.zeros(19, np.float32), np.zeros(19, np.float32), np.zeros(28, np.float32)
        net = self._host_net(h, c)
        _check(lib().mppib_host_step_lstm(C.byref(self.params), C.byref(net), _ptr(x), _ptr(u), C.c_float(dt),
                                          _ptr(xn), _ptr(xd), _ptr(y)))
        return xn, xd, y, h, c

    def output_trajectory(self, x0, u, T: int, dt: float, states: np.ndarray, outputs: np.ndarray) -> None:
        h, c = self.initial_hidden_cell()
        net = self._host_net(h, c)
        _check(lib().mppib_host_output_trajectory_lstm(C.byref(self.params), C.byref(net), _ptr(_f32(x0)), _ptr(u), T,
                                                       C.c_float(dt), _ptr(states), _ptr(outputs)))


class RacerDubinsElevationSuspension(RacerDubinsElevationLSTMSteering):
    """dynamics/racer_dubins/racer_dubins_elevation_suspension_lstm.cuh — RacerDubinsElevationSuspension(init_input_dim,
    init_hidden_dim, init_output_layers, input_dim, hidden_dim, output_layers, init_len) / RacerDubinsElevationSuspension(path):
    the LSTM-steering vehicle (S24 C2 O28) whose roll, pitch and heave are integrated from four spring-damper wheels over the
    elevation map (``getTextureHelper()``) and the normals map (``getTextureHelperNormals()``). The network, its weights
    and model_dims are the LSTM model's. One distribution only, like the LSTM model."""
    DYN_ID, STATE_DIM, CONTROL_DIM, OUTPUT_DIM = DYN_RACER_SUSPENSION_LSTM, 24, 2, 28
    # racer_dubins_elevation_suspension_lstm.cuh:25-52
    (VEL_X, YAW, POS_X, POS_Y, STEER_ANGLE, BRAKE_STATE, ROLL, PITCH, CG_POS_Z, CG_VEL_I_Z, ROLL_RATE, PITCH_RATE,
     STEER_ANGLE_RATE) = range(13)
    UNCERTAINTY_POS_X = 13  # ... the ten entries to 22, then FILLER_1

    def __init__(self, init_input_dim=3, init_hidden_dim: int = 20, init_output_layers: Sequence[int] = (23, 100, 8),
                 input_dim: int = 4, hidden_dim: int = 4, output_layers: Sequence[int] = (8, 20, 1), init_len: int = 11):
        path = init_input_dim if isinstance(init_input_dim, str) else None
        if path:  # the architecture as the file's arrays give it (LSTMLSTMHelper(path), lstm_lstm_helper.cu:14-31)
            pre = "model/" if _npz_has(path, "model/lstm/weight_hh_l0") else ""
            H = npz_read(path, pre + "lstm/weight_hh_l0").shape[1]
            L1 = npz_read(path, pre + "output/dynamics_W1").shape[0]
            init_input_dim, init_hidden_dim, init_output_layers = 3, 20, (23, 100, 2 * H)
            input_dim, hidden_dim, output_layers, init_len = 4, H, (H + 4, L1, 1), 11
        super().__init__(init_input_dim, init_hidden_dim, init_output_layers, input_dim, hidden_dim, output_layers,
                         init_len)
        base = self.params
        p = RacerSuspensionDynParams()
        C.memmove(C.byref(p), C.byref(base), C.sizeof(RacerLSTMDynParams))
        # racer_dubins_elevation_suspension_lstm.cuh:54-63
        p.spring_k, p.drag_c, p.mass = 14000.0, 1000.0, 1447.0
        m32 = np.float32(1447.0)
        p.I_xx = float(np.float32(np.float32(np.float32(np.float32(1.0) / np.float32(12)) * m32) * np.float32(2)) *
                       np.float32(2.25))
        p.I_yy = float(np.float32(np.float32(np.float32(1.0) / np.float32(12)) * m32) * np.float32(2.25 + 9.0))
        p.wheel_radius = 0.32
        p.c_g[0], p.c_g[1], p.c_g[2] = float(np.float32(2.981) * np.float32(0.5)), 0.0, 0.0
        self.params = p
        self.normals_tex_helper_ = TwoDTextureHelperFloat4()
        if path:
            self.loadParamsLSTM(path)

    def getParams(self) -> RacerSuspensionDynParams:
        out = RacerSuspensionDynParams()
        C.memmove(C.byref(out), C.byref(self.params), C.sizeof(RacerSuspensionDynParams))
        return out

    def setParams(self, params: RacerSuspensionDynParams) -> None:
        C.memmove(C.byref(self.params), C.byref(params), C.sizeof(RacerSuspensionDynParams))

    def getTextureHelperNormals(self) -> "TwoDTextureHelperFloat4":
        return self.normals_tex_helper_

    def updateRotation(self, rotation) -> None:
        """Both maps take the same rotation (racer_dubins_elevation_suspension_lstm.cuh:133-137)."""
        self.tex_helper_.updateRotation(0, rotation)
        self.normals_tex_helper_.updateRotation(0, rotation)

    def setNormalsMap(self, normals, resolution, origin=(0.0, 0.0, 0.0), rotation=None, enable: bool = True) -> None:
        """Convenience over the normals helper: normals [height][width][3 or 4] (w = 0 when three are given)."""
        v = _f32(normals)
        if v.shape[-1] == 3:
            v = np.concatenate([v, np.zeros(v.shape[:-1] + (1,), np.float32)], axis=-1)
        t = self.normals_tex_helper_
        t.setExtent(0, v.shape[1], v.shape[0])
        t.updateTexture(0, v)
        t.updateResolution(0, resolution)
        t.updateOrigin(0, origin)
        if rotation is not None:
            t.updateRotation(0, rotation)
        t.enableTexture(0) if enable else t.disableTexture(0)

    def stateFromMap(self, m: dict) -> np.ndarray:
        """racer_dubins_elevation_suspension_lstm.cu:527-611: CG_POS_Z is the z of the centre of gravity in the world frame,
        CG_VEL_I_Z the base link's inertial vertical speed less OMEGA_Y * c_g.x; the uncertainty diagonal gets a 1e-6
        floor. A missing key gives an all-NaN state."""
        keys = ("VEL_X", "VEL_Z", "POS_X", "POS_Y", "POS_Z", "OMEGA_X", "OMEGA_Y", "ROLL", "PITCH", "YAW", "STEER_ANGLE",
                "STEER_ANGLE_RATE", "BRAKE_STATE")
        if any(k not in m for k in keys):
            return np.full(24, np.nan, np.float32)
        f = np.float32
        s = np.zeros(24, np.float32)
        g = [f(self.params.c_g[i]) for i in range(3)]
        s[self.POS_X], s[self.POS_Y], s[self.VEL_X] = m["POS_X"], m["POS_Y"], m["VEL_X"]
        pitch = f(m["PITCH"])
        bl_v_I_z = f(f(f(m["VEL_Z"]) * f(math.cos(pitch))) - f(f(m["VEL_X"]) * f(math.sin(pitch))))
        s[self.CG_VEL_I_Z] = bl_v_I_z - f(m["OMEGA_Y"]) * g[0]
        s[self.STEER_ANGLE], s[self.STEER_ANGLE_RATE] = m["STEER_ANGLE"], m["STEER_ANGLE_RATE"]
        s[self.ROLL], s[self.PITCH], s[self.YAW] = m["ROLL"], m["PITCH"], m["YAW"]
        # bodyOffsetToWorldPoseEuler(c_g, (x, y, POS_Z), (roll, pitch, yaw)): the z row of Euler2DCM_NWU (host branch)
        sr, cr = f(math.sin(f(m["ROLL"]))), f(math.cos(f(m["ROLL"])))
        sp, cp = f(math.sin(pitch)), f(math.cos(pitch))
        s[self.CG_POS_Z] = f(f(f(-sp * g[0]) + f(sr * cp) * g[1]) + f(cr * cp) * g[2]) + f(m["POS_Z"])
        s[self.ROLL_RATE], s[self.PITCH_RATE], s[self.BRAKE_STATE] = m["OMEGA_X"], m["OMEGA_Y"], m["BRAKE_STATE"]
        for i in range(4):
            s[self.UNCERTAINTY_POS_X + i] = max(s[self.UNCERTAINTY_POS_X + i], f(1e-6))
        return s

    def _normals_ptr(self):
        b = self.normals_tex_helper_.blob()
        return None if b is None else b.ctypes.data

    def step(self, state, control, dt: float, hidden=None, cell=None):
        """Host step (racer_dubins_elevation_suspension_lstm.cu:168-197); returns (next_state, state_der, output, hidden,
        cell)."""
        h0, c0 = self.initial_hidden_cell()
        h = h0 if hidden is None else _f32(hidden).copy()
        c = c0 if cell is None else _f32(cell).copy()
        x, u = _f32(state), _f32(control)
        xn, xd, y = np.zeros(24, np.float32), np.zeros(24, np.float32), np.zeros(28, np.float32)
        net = self._host_net(h, c)
        _check(lib().mppib_host_step_racer_suspension(C.addressof(self.params), C.byref(net), self._normals_ptr(), _ptr(x),
                                                      _ptr(u), C.c_float(dt), _ptr(xn), _ptr(xd), _ptr(y)))
        return xn, xd, y, h, c

    def output_trajectory(self, x0, u, T: int, dt: float, states: np.ndarray, outputs: np.ndarray) -> None:
        h, c = self.initial_hidden_cell()
        net = self._host_net(h, c)
        _check(lib().mppib_host_output_trajectory_racer_suspension(C.addressof(self.params), C.byref(net),
                                                                   self._normals_ptr(), _ptr(_f32(x0)), _ptr(_f32(u)), T,
                                                                   C.c_float(dt), _ptr(states), _ptr(outputs)))


class RacerSuspension(_Dynamics):
    """dynamics/racer_suspension/racer_suspension.cuh — RacerSuspension() / RacerSuspension(params): the 6-DoF rigid-body
    RACER vehicle (S14 C2 O26) on four spring-damper wheels over the plane z = 0. Its blob is RacerSuspensionParams
    (params.h: mppib_racer_rigid_suspension_dyn_params); call ``params.recalcParams()`` after changing a base field. The
    texture helper exists for API compatibility: the model reads no map."""
    DYN_ID, STATE_DIM, CONTROL_DIM, OUTPUT_DIM = DYN_RACER_SUSPENSION, 14, 2, 26
    P_I_X, P_I_Y, P_I_Z, ATTITUDE_QW, V_I_X, OMEGA_B_X, STEER_ANGLE = 0, 1, 2, 3, 7, 10, 13
    BASELINK_VEL_B_X, BASELINK_POS_I_Y, YAW, ROLL, PITCH, OUT_STEER_ANGLE = 0, 4, 6, 7, 8, 9

    def __init__(self, params: Optional[RacerRigidSuspensionDynParams] = None):
        super().__init__()
        p = RacerRigidSuspensionDynParams()
        p.lim.set_defaults()
        # racer_suspension.cuh:70-111
        p.wheel_radius, p.mass, p.wheel_base, p.width, p.height, p.gravity = 0.32, 1447.0, 2.981, 1.5, 1.5, -9.81
        for i in range(4):
            p.k_s[i], p.c_s[i] = 14000.0, 2000.0
        p.mu, p.v_slip = 0.65, 0.1
        p.c_t, p.c_b, p.c_v, p.c_0 = 3.0, 10.0, 0.2, 0.0
        p.steering_constant, p.steer_command_angle_scale, p.gear_sign = 0.6, -2.45, 1
        p.recalcParams()
        self.params = p
        if params is not None:
            self.setParams(params)
        self.tex_helper_ = TwoDTextureHelper()

    def getParams(self) -> RacerRigidSuspensionDynParams:
        out = RacerRigidSuspensionDynParams()
        C.memmove(C.byref(out), C.byref(self.params), C.sizeof(RacerRigidSuspensionDynParams))
        return out

    def setParams(self, params: RacerRigidSuspensionDynParams) -> None:
        C.memmove(C.byref(self.params), C.byref(params), C.sizeof(RacerRigidSuspensionDynParams))

    def getTextureHelper(self) -> "TwoDTextureHelper":
        return self.tex_helper_

    def getZeroState(self) -> np.ndarray:
        z = np.zeros(self.STATE_DIM, dtype=np.float32)
        z[self.ATTITUDE_QW] = 1.0
        return z

    def restHeight(self) -> float:
        """P_I_Z of the car upright at rest in equilibrium: each spring is wheel_radius long, compressed from its rest length
        l_0 by mass / 4 * (-gravity) / k_s, so the four spring forces carry the weight."""
        return float(np.float32(self.params.wheel_radius) + np.float32(self.params.cg_pos_wrt_base_link[2]))

    def computeStateDeriv(self, state, control, omega_jacobian: bool = False):
        """Host computeStateDeriv (racer_suspension.cu:93-298): returns (state_der, output[, omegaJacobian 3x3])."""
        xd, y, J = np.zeros(14, np.float32), np.zeros(26, np.float32), np.zeros((3, 3), np.float32)
        _check(lib().mppib_host_state_deriv_racer_rigid_suspension(C.addressof(self.params), _ptr(_f32(state)),
                                                                    _ptr(_f32(control)), _ptr(xd), _ptr(y),
                                                                    _ptr(J) if omega_jacobian else None))
        return (xd, y, J) if omega_jacobian else (xd, y)

    def step(self, state, control, dt: float):
        """Host step (racer_suspension.cu:31-45): returns (next_state, state_der, output of `state`)."""
        xn, xd, y = np.zeros(14, np.float32), np.zeros(14, np.float32), np.zeros(26, np.float32)
        _check(lib().mppib_host_step_racer_rigid_suspension(C.addressof(self.params), _ptr(_f32(state)), _ptr(_f32(control)),
                                                             dt, _ptr(xn), _ptr(xd), _ptr(y)))
        return xn, xd, y

    def updateState(self, state, state_der, dt: float) -> np.ndarray:
        """racer_suspension.cu:47-53: explicit Euler, then q / |q|."""
        xn = (_f32(state) + _f32(state_der) * np.float32(dt)).astype(np.float32)
        q = xn[3:7]
        xn[3:7] = q / np.float32(np.sqrt(np.float32(np.dot(q, q))))
        return xn

    def output_trajectory(self, x0, u, T: int, dt: float, states: np.ndarray, outputs: np.ndarray) -> None:
        _check(lib().mppib_host_output_trajectory_racer_rigid_suspension(C.addressof(self.params), _ptr(_f32(x0)),
                                                                          _ptr(_f32(u)), T, dt, _ptr(states),
                                                                          _ptr(outputs)))

    def enforceLeash(self, state_true, state_nominal, leash_values) -> np.ndarray:
        """RacerSuspension::enforceLeash (racer_suspension.cu:389-447): x / y in the body frame of the true state's yaw, the
        quaternion left as state_true has it, the other states component-wise."""
        t, n, l = _f32(state_true), _f32(state_nominal), _f32(leash_values)
        f32 = np.float32
        qw, qx, qy, qz = (float(v) for v in t[3:7])
        yaw = f32(math.atan2(2 * qy * qx + 2 * qz * qw, qw * qw + qx * qx - qy * qy - qz * qz))
        cy, sy = f32(math.cos(yaw)), f32(math.sin(yaw))
        out = t.copy()
        dx, dy = n[0] - t[0], n[1] - t[1]
        dxb = np.clip(dx * cy + dy * sy, -l[0], l[0])
        dyb = np.clip(-dx * sy + dy * cy, -l[1], l[1])
        out[0] += dxb * cy + -dyb * sy
        out[1] += dxb * sy + dyb * cy
        for i in range(2, 14):
            if 3 <= i < 7:
                continue
            d = n[i] - t[i]
            out[i] = t[i] + np.clip(d, -l[i], l[i]) if l[i] < abs(d) else n[i]
        return out.astype(np.float32)

    @staticmethod
    def _rotate(q, v):
        w, x, y, z = (float(c) for c in q)
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
        return R @ np.asarray(v, np.float64)

    def attitudeFromState(self, state) -> np.ndarray:
        """(w, x, y, z)"""
        return _f32(state)[3:7].copy()

    def positionFromState(self, state) -> np.ndarray:
        s = _f32(state)
        return (s[0:3] - self._rotate(s[3:7], list(self.params.cg_pos_wrt_base_link))).astype(np.float32)

    def velocityFromState(self, state) -> np.ndarray:
        s = _f32(state)
        q = s[3:7] * np.array([1, -1, -1, -1], np.float32)
        v_B = self._rotate(q, s[7:10])
        return (v_B + np.cross(s[10:13], -np.array(list(self.params.cg_pos_wrt_base_link)))).astype(np.float32)

    def angularRateFromState(self, state) -> np.ndarray:
        return _f32(state)[10:13].copy()

    def stateFromOdometry(self, q_B_to_I, pos_base_link_I, vel_base_link_B, omega_B) -> np.ndarray:
        s = np.zeros(14, np.float32)
        s[3:7] = q_B_to_I
        s[10:13] = omega_B
        cg = np.array(list(self.params.cg_pos_wrt_base_link), np.float64)
        s[0:3] = np.asarray(pos_base_link_I) + self._rotate(q_B_to_I, cg)
        s[7:10] = self._rotate(q_B_to_I, np.asarray(vel_base_link_B) + np.cross(omega_B, cg))
        return s


class _Cost:
    COST_ID = -1

    def __init__(self):
        self.params = None
        self.costmap: Optional[np.ndarray] = None

    def blob(self) -> bytes:
        return bytes(self.params)


USER_ID_BASE = 1000  # MPPIB_USER_ID_BASE: dynamics / cost ids of out-of-tree pairs


def load_plugin(path: str) -> None:
    """mppib_load_plugin: dlopen an out-of-tree pair library (plugins_example/) and let it register its pairs."""
    _check(lib().mppib_load_plugin(os.fsencode(path)))


class UserDynamics(_Dynamics):
    """Host handle of a user-registered dynamics (the device twin lives in the plugin library): ids, dimensions and the
    POD parameter struct, which must start with a ControlLimits field named `lim` like every built-in dynamics blob."""

    def __init__(self, dyn_id: int, state_dim: int, control_dim: int, output_dim: int, params: C.Structure):
        super().__init__()
        self.DYN_ID, self.STATE_DIM, self.CONTROL_DIM, self.OUTPUT_DIM = dyn_id, state_dim, control_dim, output_dim
        self.params = params
        self.params.lim.set_defaults()


class UserCost(_Cost):
    def __init__(self, cost_id: int, params: C.Structure):
        super().__init__()
        self.COST_ID, self.params = cost_id, params


class CartpoleQuadraticCost(_Cost):
    """cost_functions/cartpole/cartpole_quadratic_cost.cuh:10-23 (defaults reproduced)."""
    COST_ID = COST_CARTPOLE_QUADRATIC

    def __init__(self):
        super().__init__()
        p = CartpoleCostParams()
        for i in range(MAX_C):
            p.control_cost_coeff[i] = 1.0
        p.control_cost_coeff[0] = 10.0
        p.discount = 1.0
        p.cart_position_coeff, p.cart_velocity_coeff = 1000.0, 100.0
        p.pole_angle_coeff, p.pole_angular_velocity_coeff = 2000.0, 100.0
        p.terminal_cost_coeff = 0.0
        p.desired_terminal_state[:] = [0.0, 0.0, math.pi, 0.0]
        self.params = p


class DoubleIntegratorCircleCost(_Cost):
    """cost_functions/double_integrator/double_integrator_circle_cost.cuh:8-23 (defaults reproduced)."""
    COST_ID = COST_DI_CIRCLE

    def __init__(self):
        super().__init__()
        p = DICircleCostParams()
        for i in range(MAX_C):
            p.control_cost_coeff[i] = 1.0
        p.control_cost_coeff[0] = p.control_cost_coeff[1] = 0.01
        p.discount = 1.0
        p.velocity_cost, p.crash_cost, p.velocity_desired = 1.0, 1000.0, 2.0
        p.inner_path_radius2, p.outer_path_radius2 = 1.875 * 1.875, 2.125 * 2.125
        p.angular_momentum_desired = 2.0 * 2.0
        self.params = p


class ARStandardCost(_Cost):
    """cost_functions/autorally/ar_standard_cost.cuh:14-41 (defaults reproduced); map set with the methods below."""
    COST_ID = COST_AR_STANDARD

    def __init__(self):
        super().__init__()
        p = ARStandardCostParams()
        for i in range(MAX_C):
            p.control_cost_coeff[i] = 1.0
        p.control_cost_coeff[0] = p.control_cost_coeff[1] = 0.0
        p.discount = 1.0
        p.desired_speed, p.speed_coeff, p.track_coeff = 6.0, 4.25, 200.0
        p.max_slip_ang, p.slip_coeff, p.track_slop = 1.25, 10.0, 0.0
        p.crash_coeff, p.boundary_threshold, p.grid_res = 10000.0, 0.65, 10
        p.l1_cost, p.front_d, p.back_d = 0, 0.5, -0.5
        self.params = p

    def setCostmap(self, texels_float4: np.ndarray, width: int, height: int) -> None:
        """track_costs_ as float4 per texel, row-major [height][width][4] (ar_standard_cost.cu:101-143)."""
        t = _f32(texels_float4).reshape(height, width, 4)
        self.costmap = t
        self.params.map_width, self.params.map_height = width, height

    def updateTransform(self, m: np.ndarray, trs: Sequence[float]) -> None:
        """ar_standard_cost.cu:188-204: columns 0/1 of the 3x3 rotation and the translation."""
        for i in range(3):
            self.params.r_c1[i] = float(m[i][0])
            self.params.r_c2[i] = float(m[i][1])
            self.params.trs[i] = float(trs[i])

    def loadTrackDataFromFile(self, map_path: str) -> np.ndarray:
        """ARStandardCostImpl::loadTrackData(map_path) (ar_standard_cost.cu:85-142): npz with xBounds, yBounds,
        pixelsPerMeter, channel0..3 (row-major [height][width]). Returns the [height][width][4] texture."""
        xb, yb = npz_read(map_path, "xBounds"), npz_read(map_path, "yBounds")
        ppm = float(npz_read(map_path, "pixelsPerMeter").ravel()[0])
        w, h = int((xb[1] - xb[0]) * ppm), int((yb[1] - yb[0]) * ppm)
        if w <= 0 or h <= 0:
            raise ValueError("load track has invalid sizes")
        tex = np.zeros((h, w, 4), np.float32)
        for c in range(4):
            ch = npz_read(map_path, f"channel{c}")
            if ch.size != w * h:
                raise ValueError(f"channel{c} does not hold {w} x {h} values")
            tex[..., c] = ch.reshape(h, w)
        self.loadTrackData(tex[..., 0], float(xb[0]), float(xb[1]), float(yb[0]), float(yb[1]), ppm)
        self.setCostmap(tex, w, h)
        return tex

    def setTrackTransform(self, x_min: float, x_max: float, y_min: float, y_max: float) -> None:
        """The world->texture transform of ARStandardCostImpl::loadTrackData (ar_standard_cost.cu:416-474):
        R = diag(1/(x_max-x_min), 1/(y_max-y_min), 1), trs = (-x_min/(x_max-x_min), -y_min/(y_max-y_min), 1)."""
        R = np.zeros((3, 3), np.float32)
        R[0, 0] = 1.0 / (x_max - x_min)
        R[1, 1] = 1.0 / (y_max - y_min)
        R[2, 2] = 1.0
        trs = [-x_min / (x_max - x_min), -y_min / (y_max - y_min), 1.0]
        self.updateTransform(R, trs)

    def loadTrackData(self, channel0: np.ndarray, x_min: float, x_max: float, y_min: float, y_max: float,
                      ppm: float) -> None:
        """In-memory equivalent of ARStandardCostImpl::loadTrackData (ar_standard_cost.cu:416-474) for a map given as
        its channel-0 array [height][width]; channels 1-3 are zero; the world->texture transform is the reference's:
        R = diag(1/(x_max-x_min), 1/(y_max-y_min), 1), trs = (-x_min/(x_max-x_min), -y_min/(y_max-y_min), 1)."""
        h, w = channel0.shape
        tex = np.zeros((h, w, 4), np.float32)
        tex[..., 0] = channel0
        self.setCostmap(tex, w, h)
        self.setTrackTransform(x_min, x_max, y_min, y_max)


def _host_state_cost(cost, y, t: int = 0, crash: int = 0) -> float:
    """mppib_host_state_cost (host_twins.h) for one output vector."""
    L = lib()
    out = C.c_float()
    cr = C.c_int(crash)
    y = _f32(y)
    m = None if cost.costmap is None else _f32(cost.costmap)
    _check(L.mppib_host_state_cost(cost.COST_ID, C.byref(cost.params), None if m is None else _ptr(m), _ptr(y), int(t),
                                   C.byref(cr), C.byref(out)))
    return out.value


class DoubleIntegratorRobustCost(DoubleIntegratorCircleCost):
    """cost_functions/double_integrator/double_integrator_robust_cost.cuh: DoubleIntegratorCircleCostParams (defaults of
    double_integrator_circle_cost.cuh:8-23). Rollouts use the reference's device body; computeStateCost is its host body,
    whose steep-band constants differ (0.75 / 0.1 * crash_cost against 0.5 / 0.5 * crash_cost, DESIGN.md §8)."""
    COST_ID = COST_DI_ROBUST

    def computeStateCost(self, y, t: int = 0, crash_status=None) -> float:
        return _host_state_cost(self, y, t)

    def terminalCost(self, y) -> float:
        return 0.0

    def getLipshitzConstantCost(self) -> float:
        return float(self.params.crash_cost)  # double_integrator_robust_cost.cuh:19-22


class ARRobustCost(ARStandardCost):
    """cost_functions/autorally/ar_robust_cost.cuh (defaults of :11-28 reproduced); map handling as ARStandardCost. The
    costmap's four channels are all read: .x boundary, .y track position, .z speed (desired_speed == -1), .w heading."""
    COST_ID = COST_AR_ROBUST

    def __init__(self):
        super().__init__()
        std = self.params
        p = ARRobustCostParams()
        for name, _ in ARStandardCostParams._fields_:
            setattr(p, name, getattr(std, name))
        p.control_cost_coeff[0] = p.control_cost_coeff[1] = 0.0
        p.desired_speed, p.max_slip_ang = -1.0, 1.5
        p.track_coeff, p.slip_coeff, p.speed_coeff = 33.0, 0.0, 20.0
        p.crash_coeff, p.boundary_threshold, p.track_slop = 125000.0, 0.75, 0.0
        p.heading_coeff = 0.0
        self.params = p

    def setTrackData(self, texels_float4: np.ndarray, x_min: float, x_max: float, y_min: float, y_max: float) -> None:
        """A four-channel map [height][width][4] and its world bounds."""
        t = _f32(texels_float4)
        self.setCostmap(t, t.shape[1], t.shape[0])
        self.setTrackTransform(x_min, x_max, y_min, y_max)

    def getStabilizingCost(self, s) -> float:
        """ar_robust_cost.cu:13-38."""
        out = C.c_float()
        _check(lib().mppib_host_ar_robust_stabilizing_cost(C.byref(self.params), _ptr(_f32(s)), C.byref(out)))
        return out.value

    def getCostmapCost(self, s) -> float:
        """ar_robust_cost.cu:40-117, host branch (nearest texel)."""
        if self.costmap is None:
            raise MppibError(-9, "ARRobustCost has no costmap (call loadTrackData / setTrackData)")
        out = C.c_float()
        m = _f32(self.costmap)
        _check(lib().mppib_host_ar_robust_costmap_cost(C.byref(self.params), _ptr(m), _ptr(_f32(s)), C.byref(out)))
        return out.value

    def computeStateCost(self, y, t: int = 0, crash_status=None) -> float:
        """ar_robust_cost.cu:119-139."""
        if self.costmap is None:
            raise MppibError(-9, "ARRobustCost has no costmap (call loadTrackData / setTrackData)")
        return _host_state_cost(self, y, t)

    def terminalCost(self, y) -> float:
        return 0.0


class QuadrotorQuadraticCost(_Cost):
    """cost_functions/quadrotor/quadrotor_quadratic_cost.cuh:9-66 (defaults reproduced)."""
    COST_ID = COST_QUADROTOR_QUADRATIC

    def __init__(self):
        super().__init__()
        p = QuadrotorCostParams()
        for i in range(MAX_C):
            p.control_cost_coeff[i] = 2.0
        p.discount = 1.0
        p.s_goal[:] = [0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0]
        p.x_coeff = p.v_coeff = p.q_coeff = p.roll_coeff = p.pitch_coeff = p.yaw_coeff = p.w_coeff = 1.0
        p.use_euler = 1
        p.terminal_cost_coeff = 0.0
        self.params = p

    def getDesiredState(self) -> np.ndarray:
        return np.array(list(self.params.s_goal), dtype=np.float32)


class QuadrotorMapCost(_Cost):
    """cost_functions/quadrotor/quadrotor_map_cost.cuh (defaults of :14-60 reproduced). The map is ``tex_helper_``'s map 0
    (a TwoDTextureHelper), pushed with the cost's parameters as MPPIB_BLOB_COST_TEXTURE. computeStateCost and the
    compute*Cost terms are the reference's HOST bodies; the rollouts run its device body, which adds the costmap term and
    the crash flag and leaves the waypoint term out (DESIGN.md §8). updateWaypoint / updateGateBoundaries push to the
    engines built on this cost only when something changed, as in the reference (quadrotor_map_cost.cu:161-196)."""
    COST_ID = COST_QUADROTOR_MAP

    def __init__(self):
        super().__init__()
        p = QuadrotorMapCostParams()
        p.set_defaults()
        self.params = p
        self.tex_helper_ = TwoDTextureHelper()
        self._engines = weakref.WeakSet()
        self.params_pushes = 0  # paramsToDevice calls that reached an engine

    def _bind_engine(self, engine) -> None:
        self._engines.add(engine)

    def paramsToDevice(self) -> None:
        """The parameter blob and tex_helper_'s map to every open engine built on this cost."""
        pushed = False
        for e in list(self._engines):
            if e._h:
                e.push_cost()
                pushed = True
        if pushed:
            self.params_pushes += 1

    def updateWaypoint(self, x, y=None, z=None, heading: float = 0.0) -> None:
        """updateWaypoint(float4) or updateWaypoint(x, y, z, heading = 0)."""
        if y is None:
            x, y, z, heading = (float(v) for v in x)
        if self.params.updateWaypoint(x, y, z, heading):
            self.paramsToDevice()

    def updateGateBoundaries(self, *args) -> None:
        """(left float3, right float3), (list of >= 6 floats) or (left_x, left_y, left_z, right_x, right_y, right_z)."""
        if len(args) == 2:
            vals = list(args[0])[:3] + list(args[1])[:3]
        elif len(args) == 1:
            vals = list(args[0])
            if len(vals) < 6:  # quadrotor_map_cost.cu:176-181
                print(f"You need {6 - len(vals)} more floats in the call to updateGateBoundaries", file=sys.stderr)
                return
        else:
            vals = list(args)
        if self.params.updateGateBoundaries(*[float(v) for v in vals[:6]]):
            self.paramsToDevice()

    def computeStateCost(self, y, t: int = 0, crash_status=None) -> float:
        """quadrotor_map_cost.cu:63-90 (host body)."""
        return _host_state_cost(self, y, t)

    def terminalCost(self, y) -> float:
        return 0.0

    def _term(self, term: int, s) -> float:
        out = C.c_float()
        _check(lib().mppib_host_quadrotor_map_term(C.byref(self.params), term, _ptr(_f32(s)), C.byref(out)))
        return out.value

    def computeGateSideCost(self, s) -> float:
        return self._term(QMAP_GATE_SIDE, s)

    def computeHeadingCost(self, s) -> float:
        return self._term(QMAP_HEADING, s)

    def computeHeightCost(self, s) -> float:
        return self._term(QMAP_HEIGHT, s)

    def computeSpeedCost(self, s) -> float:
        return self._term(QMAP_SPEED, s)

    def computeStabilizingCost(self, s) -> float:
        return self._term(QMAP_STABILIZING, s)

    def computeWaypointCost(self, s) -> float:
        return self._term(QMAP_WAYPOINT, s)

    def distToWaypoint(self, s, waypoint) -> float:
        L = lib()
        L.mppib_host_quadrotor_map_dist_to_waypoint.restype = C.c_float
        w = _f32(list(waypoint)[:3] + [0.0])
        return float(L.mppib_host_quadrotor_map_dist_to_waypoint(_ptr(_f32(s)), _ptr(w)))


class RacerQuadraticCost(_Cost):
    """Quadratic tracking cost on the RACER output vector (ours; params.h: mppib_racer_quadratic_cost_params)."""
    COST_ID = COST_RACER_QUADRATIC

    def __init__(self):
        super().__init__()
        p = RacerQuadraticCostParams()
        p.discount = 1.0
        p.desired_speed, p.speed_coeff = 5.0, 4.0
        p.desired_yaw, p.yaw_coeff = 0.0, 20.0
        p.desired_y, p.lateral_coeff = 0.0, 2.0
        p.steer_coeff = 1.0
        self.params = p


class GaussianDistribution:
    """sampling_distributions/gaussian/gaussian.cuh:63-… — owns the sampling parameters (GaussianParamsImpl :21-61)."""
    SAMPLER_ID = SAMPLER_GAUSSIAN

    def __init__(self, control_dim: int, std_dev: Optional[Sequence[float]] = None):
        self.control_dim = control_dim
        p = GaussianParams()
        for i in range(MAX_C * MAX_D):
            p.std_dev[i] = 1.0
        p.pure_noise_trajectories_percentage = 0.01
        p.std_dev_decay = 1.0
        p.sum_strides = 32
        p.use_same_noise_for_all_distributions = 1
        p.offset_decay_rate = 0.97
        self.params = p
        if std_dev is not None:
            self.setStdDev(std_dev)

    def setStdDev(self, std_dev: Sequence[float], distribution: Optional[int] = None) -> None:
        ds = range(MAX_D) if distribution is None else [distribution]
        for d in ds:
            for c, v in enumerate(std_dev):
                self.params.std_dev[d * self.control_dim + c] = v

    def setControlCostCoeff(self, coeff: Sequence[float]) -> None:
        for c, v in enumerate(coeff):
            self.params.control_cost_coeff[c] = v

    def blob(self) -> bytes:
        return bytes(self.params)


class ColoredNoiseDistribution(GaussianDistribution):
    """sampling_distributions/colored_noise/colored_noise.cuh:41-… — Gaussian parameters + exponents per control
    (0 white, 1 pink, 2 brown), offset_decay_rate (0.97) and fmin."""
    SAMPLER_ID = SAMPLER_COLORED_NOISE

    def __init__(self, control_dim: int, std_dev: Optional[Sequence[float]] = None,
                 exponents: Optional[Sequence[float]] = None):
        super().__init__(control_dim, std_dev)
        if exponents is not None:
            self.setExponents(exponents)

    def setExponents(self, exponents: Sequence[float]) -> None:
        for c, v in enumerate(exponents):
            self.params.exponents[c] = v

    def setOffsetDecayRate(self, v: float) -> None:  # colored_noise.cuh setOffsetDecayRate
        self.params.offset_decay_rate = v


class NLNDistribution(GaussianDistribution):
    """sampling_distributions/nln/nln.cuh:20-74 — normal x log-normal noise (log-MPPI) with the Gaussian parameters, the
    Gaussian control rewrite and likelihood-ratio cost. One rank, one distribution."""
    SAMPLER_ID = SAMPLER_NLN

    def log_noise_mean_and_std_dev(self):
        """calculateLogMeanAndVariance (nln.cu:93-105), per control."""
        sd = np.array([self.params.std_dev[c] for c in range(self.control_dim)], np.float32)
        var = sd * sd
        return np.exp(np.float32(0.5) * var), np.sqrt(np.exp(var) * np.exp(var - np.float32(1.0)))


class SmoothMPPIDistribution(GaussianDistribution):
    """sampling_distributions/smooth-MPPI/smooth-MPPI.cuh — samples control rates with the Gaussian parameters and
    integrates them onto the nominal control over the sampler's own ``dt`` (default 0.015, not the controller's dt). The
    rate mean it carries from solve to solve lives in the engine (``Engine.get_derivative_mean``). One rank, one
    distribution."""
    SAMPLER_ID = SAMPLER_SMOOTH_MPPI

    def __init__(self, control_dim: int, std_dev: Optional[Sequence[float]] = None, dt: float = 0.015):
        super().__init__(control_dim, std_dev)
        self.dt = dt

    def getSamplingDistributionName(self) -> str:
        return "Smooth-MPPI"

    def blob(self) -> bytes:
        return bytes(SmoothMPPIParams(self.params, self.dt))


# ---------------------------------------------------------------------------------------------------------------
class Engine:
    """Thin RAII wrapper of the opaque mppib_engine (one per controller)."""

    def __init__(self, dyn: _Dynamics, cost: _Cost, sampler: GaussianDistribution, num_rollouts: int,
                 num_timesteps: int, num_distributions: int = 1, device: int = 0, flags: int = 0,
                 stream: Optional[int] = None, rank: int = 0, world_size: int = 1):
        self._h = C.c_void_p()
        self.dyn, self.cost, self.sampler = dyn, cost, sampler
        self.N, self.T, self.D = num_rollouts, num_timesteps, num_distributions
        self.S, self.Cdim, self.O = dyn.STATE_DIM, dyn.CONTROL_DIM, dyn.OUTPUT_DIM
        self.flags = flags
        d = Desc(dyn.DYN_ID, cost.COST_ID, sampler.SAMPLER_ID, num_rollouts, num_timesteps, num_distributions, device,
                 flags, stream, rank, world_size)
        for i, v in enumerate(dyn.model_dims()):
            d.model_dims[i] = v
        _check(lib().mppib_create(C.byref(self._h), C.byref(d)))
        self.push_params()
        if hasattr(cost, "_bind_engine"):
            cost._bind_engine(self)
        nl, no = C.c_int(), C.c_int()
        _check(lib().mppib_local_rollouts(self._h, C.byref(nl), C.byref(no)))
        self.n_local, self.n_offset = nl.value, no.value

    def push_cost(self) -> None:
        """The cost's parameter blob, and QuadrotorMapCost's map (tex_helper_ map 0) when it has one."""
        L = lib()
        b = self.cost.blob()
        _check(L.mppib_set_blob(self._h, BLOB_COST, b, len(b)))
        if self.cost.COST_ID == COST_QUADROTOR_MAP:
            m = self.cost.tex_helper_.blob()
            if m is not None:
                _check(L.mppib_set_blob(self._h, BLOB_COST_TEXTURE, m.ctypes.data, m.nbytes))

    def push_params(self) -> None:
        L = lib()
        b = self.dyn.blob()
        _check(L.mppib_set_blob(self._h, BLOB_DYN, b, len(b)))
        self.push_cost()
        b = self.sampler.blob()
        _check(L.mppib_set_blob(self._h, BLOB_SAMPLER, b, len(b)))
        if self.dyn.DYN_ID == DYN_AUTORALLY_NN:
            w = _f32(self.dyn.nn_theta)
            _check(L.mppib_set_blob(self._h, BLOB_NN_WEIGHTS, _ptr(w), w.nbytes))
        if self.dyn.DYN_ID in (DYN_RACER_LSTM, DYN_RACER_SUSPENSION_LSTM):
            w = _f32(self.dyn.lstm_theta)
            _check(L.mppib_set_blob(self._h, BLOB_LSTM_WEIGHTS, _ptr(w), w.nbytes))
        if self.dyn.DYN_ID in (DYN_RACER_LSTM, DYN_RACER_DUBINS_ELEVATION, DYN_RACER_SUSPENSION_LSTM):
            m = self.dyn.tex_helper_.blob()
            if m is not None:  # TwoDTextureHelper::copyToDevice
                _check(L.mppib_set_blob(self._h, BLOB_ELEVATION_MAP, m.ctypes.data, m.nbytes))
        if self.dyn.DYN_ID == DYN_RACER_SUSPENSION_LSTM:
            m = self.dyn.normals_tex_helper_.blob()
            if m is not None:
                _check(L.mppib_set_blob(self._h, BLOB_NORMALS_MAP, m.ctypes.data, m.nbytes))
        if self.cost.COST_ID in (COST_AR_STANDARD, COST_AR_ROBUST):
            if self.cost.costmap is None:
                raise MppibError(-9, f"{type(self.cost).__name__} has no costmap (call loadTrackData / setCostmap)")
            m = _f32(self.cost.costmap)
            _check(L.mppib_set_blob(self._h, BLOB_COSTMAP, _ptr(m), m.nbytes))

    def close(self) -> None:
        if self._h:
            lib().mppib_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # configuration
    def set_solver(self, dt: float, lambda_: float, alpha: float) -> None:
        _check(lib().mppib_set_solver(self._h, dt, lambda_, alpha))

    def seed(self, seed: int, offset: int = 0) -> None:
        _check(lib().mppib_seed(self._h, seed, offset))

    def burn_draws(self, n: int) -> None:
        _check(lib().mppib_burn_draws(self._h, n))

    def rng_offset(self) -> int:
        v = C.c_ulonglong()
        _check(lib().mppib_get_rng_offset(self._h, C.byref(v)))
        return v.value

    def get_derivative_mean(self) -> np.ndarray:
        """The smooth-MPPI sampler's rate mean [T][C] (mppib_get_derivative_mean)."""
        out = np.empty((self.T, self.Cdim), np.float32)
        _check(lib().mppib_get_derivative_mean(self._h, _ptr(out)))
        return out

    def set_derivative_mean(self, dmu) -> None:
        a = _f32(np.asarray(dmu, np.float32).reshape(self.T, self.Cdim))
        _check(lib().mppib_set_derivative_mean(self._h, _ptr(a)))

    def comm_init(self, unique_id: bytes) -> None:
        buf = C.create_string_buffer(unique_id, 128)
        _check(lib().mppib_comm_init(self._h, buf))

    def p2p_handle(self) -> bytes:
        """64-byte handle of this rank's gather buffer (mppib_comm_p2p_handle); all-gather them, then p2p_open."""
        buf = C.create_string_buffer(64)
        _check(lib().mppib_comm_p2p_handle(self._h, buf))
        return buf.raw

    def p2p_open(self, handles: Sequence[bytes]) -> None:
        blob = b"".join(handles)
        _check(lib().mppib_comm_p2p_open(self._h, blob))

    def p2p_setup(self, dist) -> bool:
        """Collective: exchange the gather-buffer handles through ``torch.distributed`` and switch every rank to the
        peer-memory exchange — or leave every rank on NCCL if any rank could not open its peers' buffers."""
        import torch
        world = dist.get_world_size()
        ok = 1
        try:
            mine = self.p2p_handle()
        except MppibError:
            mine, ok = b"\0" * 64, 0
        handles = [None] * world
        dist.all_gather_object(handles, mine)
        if ok:
            try:
                self.p2p_open(handles)
            except MppibError:
                ok = 0
        dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
        flag = torch.tensor([ok], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        all_ok = int(flag.item()) == 1
        if ok and not all_ok:
            self.set_option(OPT_P2P_ENABLE, 0)
        return all_ok

    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        _check(lib().mppib_comm_unique_id(buf))
        return buf.raw

    # hot path
    def solve(self, x0, U_in, optimization_stride: int = 1, iteration_num: int = 0):
        x0, U_in = _f32(x0), _f32(U_in)
        assert x0.size == self.D * self.S and U_in.size == self.D * self.T * self.Cdim
        U_out = np.empty((self.D, self.T, self.Cdim), np.float32)
        stats = (SolveStats * self.D)()
        _check(lib().mppib_solve(self._h, _ptr(x0), _ptr(U_in), optimization_stride, iteration_num, _ptr(U_out), stats))
        return U_out, [(s.baseline, s.normalizer, s.sum_w2) for s in stats]

    def solve_into(self, x0: np.ndarray, U_in: np.ndarray, U_out: np.ndarray, stats, optimization_stride: int = 1,
                   iteration_num: int = 0) -> None:
        """Allocation-free variant for timing loops: all arrays are caller-owned float32 C-contiguous."""
        _check(lib().mppib_solve(self._h, x0.ctypes.data, U_in.ctypes.data, optimization_stride, iteration_num,
                                 U_out.ctypes.data, stats))

    def solve_async(self, x0: np.ndarray, U_in: np.ndarray, optimization_stride: int = 1, iteration_num: int = 0):
        _check(lib().mppib_solve_async(self._h, x0.ctypes.data, U_in.ctypes.data, optimization_stride, iteration_num))

    def solve_wait(self):
        U_out = np.empty((self.D, self.T, self.Cdim), np.float32)
        stats = (SolveStats * self.D)()
        _check(lib().mppib_solve_wait(self._h, _ptr(U_out), stats))
        return U_out, [(s.baseline, s.normalizer, s.sum_w2) for s in stats]

    def set_option(self, option: int, value: int) -> None:
        _check(lib().mppib_set_option(self._h, option, value))

    def set_tsallis(self, gamma: float, r: float) -> None:
        _check(lib().mppib_set_tsallis(self._h, C.c_float(gamma), C.c_float(r)))

    def set_rmppi(self, value_func_threshold: float, feedback_gains=None) -> None:
        """feedback_gains: [T][S][C] (C x S column-major per step) or None."""
        g = None if feedback_gains is None else _f32(feedback_gains)
        _check(lib().mppib_set_rmppi(self._h, C.c_float(value_func_threshold), _ptr(g)))

    def set_ddp(self, Q, Q_f, R, num_iterations: int = 1) -> None:
        """DDPFeedback::setParams (mppib_set_ddp): Q, Q_f [S][S], R [C][C], iteration count."""
        S, Cd = self.S, self.Cdim
        q, qf, r = _f32(Q), _f32(Q_f), _f32(R)
        assert q.shape == (S, S) and qf.shape == (S, S) and r.shape == (Cd, Cd)
        _check(lib().mppib_set_ddp(self._h, _ptr(q), _ptr(qf), _ptr(r), int(num_iterations)))

    def ddp_feedback(self, x0, x_target, u_target, to_rmppi: bool = False, want_jacobians: bool = False):
        """DDPFeedback::computeFeedback on the device (mppib_ddp_feedback). Returns (gains [T][S][C], states [T][S],
        controls [T][C]) and, with want_jacobians, [A | B] [T][S][S+C] as a fourth element."""
        S, Cd = self.S, self.Cdim
        xt, ut = _f32(x_target), _f32(u_target)
        T = xt.shape[0]
        assert xt.shape == (T, S) and ut.shape == (T, Cd)
        gains = np.empty((T, S, Cd), np.float32)
        xs = np.empty((T, S), np.float32)
        us = np.empty((T, Cd), np.float32)
        jac = np.empty((T, S, S + Cd), np.float32) if want_jacobians else None
        _check(lib().mppib_ddp_feedback(self._h, T, _ptr(_f32(x0)), _ptr(xt), _ptr(ut), int(bool(to_rmppi)), _ptr(gains),
                                        _ptr(xs), _ptr(us), _ptr(jac)))
        return (gains, xs, us, jac) if want_jacobians else (gains, xs, us)

    def init_eval(self, candidates, strides, samples_per_candidate: int, U_nominal, optimization_stride: int = 1):
        cand = _f32(candidates)
        st = np.ascontiguousarray(strides, dtype=np.int32)
        K = cand.shape[0]
        costs = np.empty(K * samples_per_candidate, np.float32)
        _check(lib().mppib_init_eval(self._h, _ptr(cand), st.ctypes.data_as(C.c_void_p), K, samples_per_candidate,
                                     _ptr(_f32(U_nominal)), optimization_stride, _ptr(costs)))
        return costs

    def sample_trajectories(self, x0, U_nominal, sample_idx, U_opt=None, distribution: int = 0):
        """mppib_sample_trajectories: re-roll picked rollouts of the last solve. sample_idx: rank-local indices, -1 = U_opt.
        Returns (outputs [n][T][O], costs [n][T + 1], crash [n][T])."""
        idx = np.ascontiguousarray(sample_idx, dtype=np.int32)
        n = idx.size
        outputs = np.empty((n, self.T, self.dyn.OUTPUT_DIM), np.float32)
        costs = np.empty((n, self.T + 1), np.float32)
        crash = np.empty((n, self.T), np.int32)
        _check(lib().mppib_sample_trajectories(self._h, _ptr(_f32(x0)), _ptr(_f32(U_nominal)), distribution,
                                               idx.ctypes.data_as(C.c_void_p), n,
                                               None if U_opt is None else _ptr(_f32(U_opt)), _ptr(outputs), _ptr(costs),
                                               crash.ctypes.data_as(C.c_void_p)))
        return outputs, costs, crash

    def compute_control(self, x0, U, control_history=None, optimization_stride: int = 1, iteration_num: int = 0,
                        roll_forward: bool = True):
        """mppib_compute_control: the solve plus the host tail (smoothing, nominal roll-forward) in one C call. Returns
        (U [D][T][C] optimised and smoothed, states [D][T][S] or None, outputs [D][T][O] or None, stats)."""
        U = _f32(U).copy()
        states = np.empty((self.D, self.T, self.dyn.STATE_DIM), np.float32) if roll_forward else None
        outputs = np.empty((self.D, self.T, self.dyn.OUTPUT_DIM), np.float32) if roll_forward else None
        stats = (SolveStats * self.D)()
        _check(lib().mppib_compute_control(self._h, _ptr(_f32(x0)), _ptr(U), optimization_stride, iteration_num,
                                           None if control_history is None else _ptr(_f32(control_history)),
                                           _ptr(states), _ptr(outputs), stats))
        return U, states, outputs, [(s.baseline, s.normalizer, s.sum_w2) for s in stats]

    def nominal_trajectory(self, x0, U=None, control_history=None):
        """mppib_nominal_trajectory: the host tail of computeControl on the device (controller.cuh:557-586, 643-663).
        U None = the last solve's result, read on the device (may follow solve_async directly). control_history [2][C] or
        None (no smoothing). Returns (U_smoothed [D][T][C], states [D][T][S], outputs [D][T][O])."""
        Us = np.empty((self.D, self.T, self.Cdim), np.float32)
        states = np.empty((self.D, self.T, self.dyn.STATE_DIM), np.float32)
        outputs = np.empty((self.D, self.T, self.dyn.OUTPUT_DIM), np.float32)
        _check(lib().mppib_nominal_trajectory(self._h, _ptr(_f32(x0)), None if U is None else _ptr(_f32(U)),
                                              None if control_history is None else _ptr(_f32(control_history)),
                                              _ptr(Us), _ptr(states), _ptr(outputs)))
        return Us, states, outputs

    def set_noise(self, eps) -> None:
        eps = _f32(eps)
        _check(lib().mppib_set_noise(self._h, _ptr(eps), eps.size))

    def draw_noise(self) -> None:
        _check(lib().mppib_draw_noise(self._h))

    def rollout_only(self, x0, U_in, optimization_stride: int = 1, iteration_num: int = 0) -> None:
        x0, U_in = _f32(x0), _f32(U_in)
        _check(lib().mppib_rollout_only(self._h, _ptr(x0), _ptr(U_in), optimization_stride, iteration_num))

    def reduce_only(self):
        U_out = np.empty((self.D, self.T, self.Cdim), np.float32)
        stats = (SolveStats * self.D)()
        _check(lib().mppib_reduce_only(self._h, _ptr(U_out), stats))
        return U_out, [(s.baseline, s.normalizer, s.sum_w2) for s in stats]

    # read-backs
    def get_costs(self) -> np.ndarray:
        a = np.empty((self.D, self.n_local), np.float32)
        _check(lib().mppib_get_costs(self._h, _ptr(a)))
        return a

    def get_noise(self) -> np.ndarray:
        a = np.empty((self.n_local, self.T, self.Cdim), np.float32)
        _check(lib().mppib_get_noise(self._h, _ptr(a)))
        return a

    def get_samples(self) -> np.ndarray:
        a = np.empty((self.D, self.n_local, self.T, self.Cdim), np.float32)
        _check(lib().mppib_get_samples(self._h, _ptr(a)))
        return a

    def get_weights(self) -> np.ndarray:
        a = np.empty((self.D, self.n_local), np.float32)
        _check(lib().mppib_get_weights(self._h, _ptr(a)))
        return a

    def enable_timing(self, on: bool = True) -> None:
        _check(lib().mppib_enable_timing(self._h, int(on)))

    def timing(self) -> dict:
        t = Timing()
        _check(lib().mppib_get_timing(self._h, C.byref(t)))
        return {"noise_ms": t.noise_ms, "rollout_ms": t.rollout_ms, "reduce_ms": t.reduce_ms, "total_ms": t.total_ms,
                "samples": t.samples}

    def rng_info(self) -> dict:
        a, b, c = C.c_int(), C.c_int(), C.c_int()
        _check(lib().mppib_get_rng_info(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return {"own_kernel": bool(a.value), "chunks": b.value, "rounds_per_chunk": c.value}

    def launch_info(self) -> dict:
        g, b, s, t, k = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _check(lib().mppib_get_launch_info(self._h, C.byref(g), C.byref(b), C.byref(s), C.byref(t), C.byref(k)))
        return {"grid": g.value, "block": b.value, "smem_bytes": s.value, "uses_tma": bool(t.value),
                "kernels_per_solve": k.value}


# ---------------------------------------------------------------------------------------------------------------
class DDPParams:
    """feedback_controllers/DDP/ddp.cuh:16-26: tracking weights Q, Q_f [S][S], R [C][C] (identity) and num_iterations (1)."""

    def __init__(self, state_dim: int, control_dim: int):
        self.Q = np.eye(state_dim, dtype=np.float32)
        self.Q_f = np.eye(state_dim, dtype=np.float32)
        self.R = np.eye(control_dim, dtype=np.float32)
        self.num_iterations = 1


class DDPResult:
    """OptimizerResult (ddp/result.h) fields DDPFeedback exposes: state_trajectory [T][S], control_trajectory [T][C],
    feedback_gain [T][C][S] (K_t as C x S matrices)."""

    def __init__(self, T: int, S: int, Cd: int):
        self.state_trajectory = np.zeros((T, S), np.float32)
        self.control_trajectory = np.zeros((T, Cd), np.float32)
        self.feedback_gain = np.zeros((T, Cd, S), np.float32)


def _standalone_cost(dyn_id: int) -> "_Cost":
    # the in-tree pair of each model with an analytic Jacobian; DDP reads nothing of the cost
    if dyn_id == DYN_CARTPOLE:
        return CartpoleQuadraticCost()
    if dyn_id == DYN_DOUBLE_INTEGRATOR:
        return DoubleIntegratorCircleCost()
    if dyn_id == DYN_QUADROTOR:
        return QuadrotorQuadraticCost()
    if dyn_id == DYN_AUTORALLY_NN:
        c = ARStandardCost()
        c.setCostmap(np.zeros((4, 4), np.float32), 2, 2)
        return c
    raise MppibError(-2, f"dynamics {dyn_id} has no DDP kernel (no analytic Jacobian)")


class DDPFeedback:
    """feedback_controllers/DDP/ddp.cuh:97-141 — DDPFeedback(model, dt, num_timesteps). computeFeedback runs the iLQR solve
    on the GPU (mppib_ddp_feedback) with the engine it is bound to: a controller binds its own engine; used standalone it
    creates a minimal engine for its dynamics on first use. The solve uses the engine's dt, so a controller's DDPFeedback
    must be built with the controller's dt."""

    def __init__(self, model: _Dynamics, dt: float, num_timesteps: int):
        self.model_, self.dt_, self.num_timesteps_ = model, dt, num_timesteps
        S, Cd = model.STATE_DIM, model.CONTROL_DIM
        self.params_ = DDPParams(S, Cd)
        self.result_ = DDPResult(num_timesteps, S, Cd)
        self.fb_gain_traj_ = np.zeros((num_timesteps, S, Cd), np.float32)  # the feedback state, [t][s][c]
        self._engine: Optional[Engine] = None
        self._own_engine = False

    def bind(self, engine: "Engine", dt: float) -> None:
        if abs(float(dt) - float(self.dt_)) > 0.0:
            raise ValueError(f"DDPFeedback dt {self.dt_} differs from the controller's dt {dt}")
        if self._own_engine and self._engine is not None:
            self._engine.close()
        self._engine, self._own_engine = engine, False

    def _engine_for_solve(self) -> "Engine":
        if self._engine is None:
            cost = _standalone_cost(self.model_.DYN_ID)
            self._engine = Engine(self.model_, cost, GaussianDistribution(self.model_.CONTROL_DIM), 32, 2)
            self._engine.set_solver(self.dt_, 1.0, 0.0)
            self._own_engine = True
        elif self._own_engine:
            self._engine.push_params()  # the model's parameters may have changed since
        return self._engine

    def setParams(self, params: DDPParams) -> None:
        self.params_ = params

    def getParams(self) -> DDPParams:
        return self.params_

    def initTrackingController(self) -> None:
        """ddp.cu:51-67: zero gain trajectory."""
        S, Cd = self.model_.STATE_DIM, self.model_.CONTROL_DIM
        self.result_ = DDPResult(self.num_timesteps_, S, Cd)
        self.fb_gain_traj_[:] = 0.0

    def computeFeedback(self, init_state, goal_traj, control_traj, to_rmppi: bool = False) -> None:
        """ddp.cu:80-118. goal_traj [T][S], control_traj [T][C]."""
        e = self._engine_for_solve()
        p = self.params_
        e.set_ddp(p.Q, p.Q_f, p.R, p.num_iterations)
        gains, xs, us = e.ddp_feedback(init_state, goal_traj, control_traj, to_rmppi=to_rmppi)
        self.fb_gain_traj_ = gains
        self.result_.state_trajectory, self.result_.control_trajectory = xs, us
        self.result_.feedback_gain = np.ascontiguousarray(gains.transpose(0, 2, 1))

    def k(self, x_act, x_goal, t: int, fb_state: Optional[np.ndarray] = None) -> np.ndarray:
        """ddp.cuh:175-181: K_t (x_act - x_goal)."""
        g = self.fb_gain_traj_ if fb_state is None else fb_state
        return (_f32(x_act) - _f32(x_goal)) @ g[t]

    def interpolateFeedback(self, state, goal_state, rel_time: float, fb_state: Optional[np.ndarray] = None) -> np.ndarray:
        """feedback.cuh:216-228."""
        lower = int(rel_time / self.dt_)
        alpha = (rel_time - lower * self.dt_) / self.dt_
        return ((1 - alpha) * self.k(state, goal_state, lower, fb_state).astype(np.float64) +
                alpha * self.k(state, goal_state, lower + 1, fb_state).astype(np.float64)).astype(np.float32)

    def getFeedbackState(self) -> np.ndarray:
        return self.fb_gain_traj_

    def getFeedbackGainsEigen(self) -> np.ndarray:
        return self.result_.feedback_gain

    def close(self) -> None:
        if self._own_engine and self._engine is not None:
            self._engine.close()
        self._engine, self._own_engine = None, False


class _Controller:
    """Shared part of the controllers (include/mppi/controllers/controller.cuh:71-…). Trajectories are numpy arrays
    shaped like the reference's Eigen matrices transposed: control [T][C] (Eigen C x T column-major is the same
    memory), state [T][S], output [T][O]."""
    NUM_DISTRIBUTIONS = 1

    def __init__(self, model: _Dynamics, cost: _Cost, fb_controller, sampler: GaussianDistribution, dt: float,
                 max_iter: int, lambda_: float, alpha: float, num_timesteps: int, num_rollouts: int,
                 init_control_traj: Optional[np.ndarray] = None, seed: Optional[int] = None, device: int = 0,
                 flags: int = 0, stream: Optional[int] = None, rank: int = 0, world_size: int = 1,
                 lockstep_with_reference_ctor: bool = True):
        self.model_, self.cost_, self.fb_controller_, self.sampler_ = model, cost, fb_controller, sampler
        self.dt_, self.num_iters_, self.lambda_, self.alpha_ = dt, max_iter, lambda_, alpha
        self.num_timesteps_, self.num_rollouts_ = num_timesteps, num_rollouts
        T, Cd, S, O = num_timesteps, model.CONTROL_DIM, model.STATE_DIM, model.OUTPUT_DIM
        self.control_ = np.zeros((T, Cd), np.float32) if init_control_traj is None else _f32(init_control_traj).copy()
        self.control_history_ = np.zeros((2, Cd), np.float32)  # controller.cuh:968
        self.state_ = np.zeros((T, S), np.float32)
        self.output_ = np.zeros((T, O), np.float32)
        self.slide_control_scale_ = np.zeros(Cd, np.float32)  # controller.cuh:67
        self.baseline_ = [0.0] * self.NUM_DISTRIBUTIONS
        self.normalizer_ = [0.0] * self.NUM_DISTRIBUTIONS
        self.free_energy_statistics_ = {}
        self.perc_sampled_control_trajectories_ = 0.0  # controller.cuh:948-950
        self.num_top_control_trajectories_ = 0
        self.top_n_costs_ = np.zeros(0, np.float32)
        self.sampled_indices_ = np.zeros(0, np.int32)
        self.sampled_trajectories_ = self.sampled_costs_ = self.sampled_crash_status_ = None
        self._vis_inputs = None
        self._vis_rng = np.random.RandomState(0 if seed is None else seed)
        self.engine = Engine(model, cost, sampler, num_rollouts, num_timesteps, self.NUM_DISTRIBUTIONS, device, flags,
                             stream, rank, world_size)
        self.engine.set_solver(dt, lambda_, alpha)
        # controller.cuh:59 seeds from the wall clock; tests pass an explicit seed (ControllerParams::seed_ is unsigned)
        self.seed_ = (int.from_bytes(os.urandom(4), "little") if seed is None else seed) & 0xFFFFFFFF
        self.engine.seed(self.seed_, 0)
        if lockstep_with_reference_ctor:
            # chooseAppropriateKernel draws one full noise buffer in the constructor (mppi_controller.cu:95)
            self.engine.burn_draws(1)
        # feedback (controller.cuh:263-268): off until initFeedback(). The reference's Tube / RMPPI constructors switch it
        # on; here existing callers keep the behaviour they had, feed-forward only.
        self.enable_feedback_ = False
        self.propagated_feedback_state_trajectory_ = np.zeros((T, S), np.float32)
        if isinstance(fb_controller, DDPFeedback):
            fb_controller.bind(self.engine, dt)

    # getters (controller.cuh:409-436,510-517)
    def getControlSeq(self) -> np.ndarray:
        return self.control_

    def getTargetStateSeq(self) -> np.ndarray:
        return self.state_

    def getTargetOutputSeq(self) -> np.ndarray:
        return self.output_

    def getBaselineCost(self, ind: int = 0) -> float:
        return self.baseline_[ind]

    def getNormalizerCost(self, ind: int = 0) -> float:
        return self.normalizer_[ind]

    def getFreeEnergyStatistics(self) -> dict:
        return self.free_energy_statistics_

    def getSampledCostSeq(self) -> np.ndarray:
        return self.engine.get_costs()

    # ---- sampled (visualisation) trajectories: controller.cuh:279-297,724-763, controller.cu:55-179 --------------------
    def setPercentageSampledControlTrajectories(self, new_perc: float) -> None:
        self._need_writeback()
        self.perc_sampled_control_trajectories_ = float(new_perc)

    def setTopNSampledControlTrajectories(self, new_top_num_samples: int) -> None:
        self._need_writeback()
        self.num_top_control_trajectories_ = int(new_top_num_samples)

    def getPercentageSampledControlTrajectories(self) -> float:
        return self.perc_sampled_control_trajectories_

    def getNumberSampledTrajectories(self) -> int:
        return int(self.perc_sampled_control_trajectories_ * self.num_rollouts_)

    def getNumberTopControlTrajectories(self) -> int:
        return self.num_top_control_trajectories_

    def getTotalSampledTrajectories(self) -> int:
        return self.getNumberSampledTrajectories() + self.getNumberTopControlTrajectories()

    def getSampledOutputTrajectories(self) -> np.ndarray:
        return self.sampled_trajectories_

    def getSampledCostTrajectories(self) -> np.ndarray:
        return self.sampled_costs_

    def getSampledCrashStatusTrajectories(self) -> np.ndarray:
        return self.sampled_crash_status_

    def getTopNCosts(self) -> np.ndarray:
        return self.top_n_costs_

    def getTopTransformedCosts(self) -> np.ndarray:  # controller.cuh:294-297
        return self.top_n_costs_

    def getSampledIndices(self) -> np.ndarray:
        """Rank-local rollout index behind every sampled trajectory (-1 = the optimised control sequence)."""
        return self.sampled_indices_

    def _need_writeback(self) -> None:
        if not (self.engine.flags & FLAG_WRITEBACK_CONTROLS):
            raise MppibError(-9, "sampled trajectories need the stored controls: construct the controller with "
                                        "flags=FLAG_WRITEBACK_CONTROLS")

    def _pick_sampled_controls(self, state: np.ndarray, U_nominal: np.ndarray, U_opt: np.ndarray, costs: np.ndarray,
                               normalizer: float) -> None:
        """copySampledControlFromDevice + copyTopControlFromDevice (controller.cu:55-179): slot 0 is the optimised
        sequence, then a random subset drawn without replacement from the first 98 % of the rollouts (the tail holds the
        pure-noise samples), then the top-n by weight (= the n lowest costs)."""
        self.sampled_indices_ = pick_sampled_indices(self.getNumberSampledTrajectories(),
                                                     self.num_top_control_trajectories_, costs,
                                                     self.perc_sampled_control_trajectories_, self._vis_rng)
        self._vis_inputs = (state.copy(), U_nominal.copy(), U_opt.copy())
        n_top = self.num_top_control_trajectories_
        if n_top > 0:
            c = costs[self.sampled_indices_[-n_top:]].astype(np.float64)
            self.top_n_costs_ = (np.exp(-(c - float(costs.min())) / self.lambda_) / normalizer).astype(np.float32)
        else:
            self.top_n_costs_ = np.zeros(0, np.float32)

    def calculateSampledStateTrajectories(self) -> None:
        """controllers/MPPI/mppi_controller.cu:262-298 (launchVisualizeKernel + copies)."""
        if self.getTotalSampledTrajectories() <= 0 or self._vis_inputs is None:
            return
        x0, U_nominal, U_opt = self._vis_inputs
        out, costs, crash = self.engine.sample_trajectories(x0, U_nominal, self.sampled_indices_, U_opt)
        self.sampled_trajectories_, self.sampled_costs_, self.sampled_crash_status_ = out, costs, crash

    def getNumTimesteps(self) -> int:
        return self.num_timesteps_

    # host-only helpers of the base class (controller.cuh:317-393,765-768; controller.cu:274-283)
    def updateImportanceSampler(self, nominal_control) -> None:
        self.control_ = _f32(nominal_control).copy()

    def interpolateControls(self, rel_time: float, c_traj: np.ndarray) -> np.ndarray:
        lower = int(rel_time / self.dt_)
        alpha = (rel_time - lower * self.dt_) / self.dt_
        return ((1 - alpha) * c_traj[lower].astype(np.float64) + alpha * c_traj[lower + 1].astype(np.float64)).astype(np.float32)

    def getCurrentControl(self, state, rel_time: float, target_nominal_state, c_traj: np.ndarray) -> np.ndarray:
        """Controller::getCurrentControl (controller.cuh:329-346): interpolated control plus, when feedback is enabled,
        the interpolated DDP feedback on (state - target_nominal_state); constrained."""
        u = self.interpolateControls(rel_time, c_traj)
        if self.enable_feedback_:
            u = (u + self.interpolateFeedback(state, target_nominal_state, rel_time)).astype(np.float32)
        self.model_.enforceConstraints(None, u)
        return u

    # feedback surface (controller.cuh:263-268, 479-560, 709-721)
    def _fb(self) -> DDPFeedback:
        if self.fb_controller_ is None:
            self.fb_controller_ = DDPFeedback(self.model_, self.dt_, self.num_timesteps_)
            self.fb_controller_.bind(self.engine, self.dt_)
        return self.fb_controller_

    def initFeedback(self) -> None:
        self.enable_feedback_ = True
        self._fb().initTrackingController()

    def getFeedbackEnabled(self) -> bool:
        return self.enable_feedback_

    def disableFeedbackController(self) -> None:
        """Stops the DDP recomputation. On RMPPI the last gains stay in the engine and keep being applied, as the
        reference's rollout always reads its feedback controller's device gains; setFeedbackGains replaces them."""
        self.enable_feedback_ = False

    def setFeedbackParams(self, fb_params: DDPParams) -> None:
        self._fb().setParams(fb_params)

    def getFeedbackParams(self) -> DDPParams:
        return self._fb().getParams()

    def getActualStateSeq(self) -> np.ndarray:
        return self.state_

    def computeFeedbackHelper(self, state, state_traj, control_traj) -> None:
        if not self.enable_feedback_:
            return
        self.fb_controller_.computeFeedback(state, state_traj, control_traj)

    def computeFeedback(self, state) -> None:
        self.computeFeedbackHelper(state, self.getTargetStateSeq(), self.getControlSeq())

    def getFeedbackControl(self, state, goal_state, t: int) -> np.ndarray:
        return self.fb_controller_.k(state, goal_state, t)

    def interpolateFeedback(self, state, target_nominal_state, rel_time: float) -> np.ndarray:
        return self.fb_controller_.interpolateFeedback(state, target_nominal_state, rel_time)

    def computeFeedbackPropagatedStateSeq(self) -> None:
        """controller.cuh:479-501: roll the actual start state forward with the control plus the feedback on the target
        state sequence, through the model's host step."""
        if not self.enable_feedback_:
            return
        traj = self.propagated_feedback_state_trajectory_
        traj[0] = self.getActualStateSeq()[0]
        u_seq, x_tgt = self.getControlSeq(), self.getTargetStateSeq()
        for i in range(self.num_timesteps_ - 1):
            u = (u_seq[i] + self.getFeedbackControl(traj[i], x_tgt[i], i)).astype(np.float32)
            traj[i + 1], _, _ = self.model_.step(traj[i], u, self.dt_)

    def getFeedbackPropagatedStateSeq(self) -> np.ndarray:
        return self.propagated_feedback_state_trajectory_

    def setSlideControlScale(self, slide_control_scale) -> None:
        self.slide_control_scale_[:] = _f32(slide_control_scale)

    def getSampledNoise(self) -> np.ndarray:
        """The sampler's control buffer [NUM_ROLLOUTS][T][C] of distribution 0 (needs FLAG_WRITEBACK_CONTROLS)."""
        return self.engine.get_samples()[0]

    def getDt(self) -> float:
        return self.dt_

    def setSeedCUDARandomNumberGen(self, seed: int) -> None:  # controller.cu:200-207
        self.seed_ = seed & 0xFFFFFFFF
        self.engine.seed(self.seed_, 0)

    def setParams(self) -> None:
        """Push (possibly edited) plugin / solver parameters to the engine (Controller::setParams, controller.cuh:821-850)."""
        self.engine.push_params()
        self.engine.set_solver(self.dt_, self.lambda_, self.alpha_)

    def setDeviceSideTail(self, on: bool = True) -> None:
        """Not in the reference: run computeControl's host tail (controller.cuh:557-586, 643-663) as one device kernel
        (mppib_nominal_trajectory) instead of the library's host twins. VanillaMPPI / ColoredMPPI. Off by default: the
        host twins are faster (DESIGN.md §9)."""
        self.device_side_tail_ = bool(on)

    # host tail helpers — CPU, in the C library (controller.cuh:557-663)
    def _smooth(self, u: np.ndarray) -> None:
        lib().mppib_host_smooth_controls(_ptr(u), _ptr(self.control_history_), self.num_timesteps_,
                                         self.model_.CONTROL_DIM)

    def _slide(self, u: np.ndarray, steps: int) -> None:
        z = self.model_.zero_control_
        lib().mppib_host_slide_controls(_ptr(u), steps, self.num_timesteps_, self.model_.CONTROL_DIM, _ptr(z),
                                        _ptr(self.slide_control_scale_))

    def _output_trajectory(self, x0: np.ndarray, u: np.ndarray, states: np.ndarray, outputs: np.ndarray) -> None:
        self.model_.output_trajectory(x0, u, self.num_timesteps_, self.dt_, states, outputs)

    def _save_control_history(self, steps: int, u: np.ndarray) -> None:  # controller.cuh:602-616
        if steps == 1:
            self.control_history_[0] = self.control_history_[1]
            self.control_history_[1] = u[0]
        elif steps >= 2:
            self.control_history_[0] = u[steps - 2]
            self.control_history_[1] = u[steps - 1]

    def _free_energy(self, stats) -> dict:
        out = np.zeros(3, np.float32)
        st = SolveStats(*stats, 0.0)
        lib().mppib_host_free_energy(C.byref(st), self.num_rollouts_, C.c_float(self.lambda_), _ptr(out))
        return {"freeEnergyMean": float(out[0]), "freeEnergyVariance": float(out[1]),
                "freeEnergyModifiedVariance": float(out[2])}


def pick_sampled_indices(num_sampled: int, num_top: int, costs: np.ndarray, perc: float,
                         rng: np.random.RandomState) -> np.ndarray:
    """Sample selection of controller.cu:55-179 on rank-local rollout indices. Entry 0 of the sampled block stands for
    the optimised sequence (-1); entries 1.. are distinct rollouts from the first 98 % (all of them in order if
    perc > 0.98); the last num_top entries are the rollouts with the largest weights, i.e. the lowest costs."""
    N = costs.shape[0]
    idx = []
    if num_sampled > 0:
        if perc > 0.98:
            pool = np.arange(num_sampled)
        else:
            pool = rng.choice(int(N * 0.98), size=num_sampled, replace=False)
        idx = [-1] + [int(v) for v in pool[1:]]
    if num_top > 0:
        top = np.argpartition(costs, min(num_top, N) - 1)[:num_top]
        idx += [int(v) for v in top[np.argsort(costs[top], kind="stable")]]
    return np.asarray(idx, dtype=np.int32)


def merge_records(records: np.ndarray, lambda_: float, normalize: bool = True) -> np.ndarray:
    """records [nrec][D][pstride] -> merged [D][pstride] with the engine's K2 arithmetic (CPU twin, host_twins.h)."""
    r = _f32(records)
    nrec, D, pstride = r.shape
    out = np.zeros((D, pstride), np.float32)
    _check(lib().mppib_host_merge_records(_ptr(r), nrec, D, pstride - 4, pstride, C.c_float(lambda_), int(normalize),
                                          _ptr(out)))
    return out


class VanillaMPPIController(_Controller):
    """controllers/MPPI/mppi_controller.cuh:14-17 — same constructor arguments; NUM_ROLLOUTS / MAX_TIMESTEPS are runtime."""
    NUM_DISTRIBUTIONS = 1

    def computeControl(self, state, optimization_stride: int = 1) -> None:
        """controllers/MPPI/mppi_controller.cu:151-241."""
        state = _f32(state)
        prev_baseline = self.baseline_[0]
        for opt_iter in range(self.num_iters_):
            U_nominal = self.control_
            U, stats = self.engine.solve(state, self.control_, optimization_stride, opt_iter)
            self.control_ = U[0].copy()
            self.baseline_[0], self.normalizer_[0] = stats[0][0], stats[0][1]
            fe = self._free_energy(stats[0])
        if self.getTotalSampledTrajectories() > 0:  # mppi_controller.cu:232-240
            self._pick_sampled_controls(state, U_nominal, self.control_, self.engine.get_costs()[0], self.normalizer_[0])
        fe["normalizerPercent"] = self.normalizer_[0] / self.num_rollouts_
        fe["increase"] = self.baseline_[0] - prev_baseline
        fe["previousBaseline"] = prev_baseline
        self.free_energy_statistics_ = {"real_sys": fe}
        if getattr(self, "device_side_tail_", False):  # smoothing + roll-forward as one device kernel (SURVEY f2)
            Us, st, out = self.engine.nominal_trajectory(state.reshape(1, -1), self.control_[None], self.control_history_)
            self.control_, self.state_[...], self.output_[...] = Us[0].copy(), st[0], out[0]
        else:
            self._smooth(self.control_)  # smoothControlTrajectory
            self._output_trajectory(state, self.control_, self.state_, self.output_)  # computeStateTrajectory
        for i in range(self.num_timesteps_):  # mppi_controller.cu:227-231
            self.model_.enforceConstraints(None, self.control_[i])

    def slideControlSequence(self, steps: int) -> None:
        """controllers/MPPI/mppi_controller.cu (slideControlSequence): save history, then slide."""
        self._save_control_history(steps, self.control_)
        self._slide(self.control_, steps)


class ColoredMPPIController(VanillaMPPIController):
    """controllers/ColoredMPPI/colored_mppi_controller.cuh — VanillaMPPI's flow with the ColoredNoise sampler, an optional
    state leash (colored_mppi_controller.cu:150-153), Tsallis weights when gamma and r are both non-zero (:199-209) and
    the clamp of control 1 (:232-238). ``tsallis=True`` creates the engine with the control write-back buffer the
    Tsallis reduction needs."""

    def __init__(self, *args, tsallis: bool = False, **kw):
        if tsallis:
            kw["flags"] = kw.get("flags", 0) | FLAG_WRITEBACK_CONTROLS
        super().__init__(*args, **kw)
        self.gamma_, self.r_ = 0.0, 0.0
        self.leash_active_, self.leash_jump_ = False, 1
        self.state_leash_dist_ = np.zeros(self.model_.STATE_DIM, np.float32)

    def setGamma(self, gamma: float) -> None:
        self.gamma_ = gamma
        self._push_weighting()

    def setRExp(self, r: float) -> None:
        self.r_ = r
        self._push_weighting()

    def _push_weighting(self) -> None:
        on = self.gamma_ != 0 and self.r_ != 0
        self.engine.set_tsallis(self.gamma_ if on else 0.0, self.r_ if on else 0.0)

    def setLeashActive(self, v: bool) -> None:
        self.leash_active_ = v

    def setStateLeashLength(self, v: float, index: int = 0) -> None:
        self.state_leash_dist_[index] = v

    def computeControl(self, state, optimization_stride: int = 1) -> None:
        state = _f32(state).copy()
        if self.leash_active_:  # the model's own enforceLeash (colored_mppi_controller.cu:150-153)
            state = self.model_.enforceLeash(state, self.state_[self.leash_jump_], self.state_leash_dist_)
        super().computeControl(state, optimization_stride)
        if self.model_.CONTROL_DIM > 1:  # colored_mppi_controller.cu:232-238
            lo, hi = self.model_.params.lim.rng_lo[1], self.model_.params.lim.rng_hi[1]
            self.control_[:, 1] = np.clip(self.control_[:, 1], lo, hi)

    def slideControlSequence(self, steps: int) -> None:
        self.leash_jump_ = steps
        super().slideControlSequence(steps)


class TubeMPPIController(_Controller):
    """controllers/Tube-MPPI/tube_mppi_controller.cuh — actual + nominal system sharing one noise draw."""
    NUM_DISTRIBUTIONS = 2

    def __init__(self, *args, nominal_threshold: float = 20.0, **kwargs):
        super().__init__(*args, **kwargs)
        T = self.num_timesteps_
        self.nominal_control_trajectory_ = self.control_.copy()
        self.nominal_state_trajectory_ = np.zeros((T, self.model_.STATE_DIM), np.float32)
        self.nominal_output_trajectory_ = np.zeros((T, self.model_.OUTPUT_DIM), np.float32)
        self.nominalStateInit_ = False
        self.nominal_threshold_ = nominal_threshold
        self.nominal_state_used_ = 0

    def setNominalThreshold(self, v: float) -> None:
        self.nominal_threshold_ = v

    def getNominalThreshold(self) -> float:
        return self.nominal_threshold_

    # tube_mppi_controller.cuh:49-63: the controller's "solution" is the NOMINAL system; the actual one has its own getters
    def getControlSeq(self) -> np.ndarray:
        return self.nominal_control_trajectory_

    def getTargetStateSeq(self) -> np.ndarray:
        return self.nominal_state_trajectory_

    def getActualControlSeq(self) -> np.ndarray:
        return self.control_

    def getActualStateSeq(self) -> np.ndarray:
        return self.state_

    def _compute_state_trajectories(self, state: np.ndarray) -> None:
        # tube_mppi_controller.cu:345-350: actual from `state`, nominal from nominal_state_trajectory_.col(0)
        self._output_trajectory(state, self.control_, self.state_, self.output_)
        x0n = self.nominal_state_trajectory_[0].copy()
        self._output_trajectory(x0n, self.nominal_control_trajectory_, self.nominal_state_trajectory_,
                                self.nominal_output_trajectory_)

    def computeControl(self, state, optimization_stride: int = 1) -> None:
        """controllers/Tube-MPPI/tube_mppi_controller.cu:157-299."""
        state = _f32(state)
        if not self.nominalStateInit_:
            self.nominal_state_trajectory_[0] = state
            self.nominalStateInit_ = True
        prev = list(self.baseline_)
        for opt_iter in range(self.num_iters_):
            x0 = np.stack([state, self.nominal_state_trajectory_[0]])
            U_in = np.stack([self.control_, self.nominal_control_trajectory_])
            U, stats = self.engine.solve(x0, U_in, optimization_stride, opt_iter)
            self.control_ = U[0].copy()
            self.nominal_control_trajectory_ = U[1].copy()
            for d in range(2):
                self.baseline_[d], self.normalizer_[d] = stats[d][0], stats[d][1]
            fe = [self._free_energy(stats[0]), self._free_energy(stats[1])]
            self._compute_state_trajectories(state)
            if self.baseline_[0] < self.baseline_[1] + self.nominal_threshold_:  # :268-280
                self.nominal_state_used_ = 0
                self.nominal_state_trajectory_ = self.state_.copy()
                self.nominal_control_trajectory_ = self.control_.copy()
            else:
                self.nominal_state_used_ = 1
        # smoothControlTrajectory (tube_mppi_controller.cu:327-331) smooths the NOMINAL sequence
        self._smooth(self.nominal_control_trajectory_)
        self._compute_state_trajectories(state)
        for d, key in enumerate(("real_sys", "nominal_sys")):
            fe[d]["normalizerPercent"] = self.normalizer_[d] / self.num_rollouts_
            fe[d]["increase"] = self.baseline_[d] - prev[d]
            fe[d]["previousBaseline"] = prev[d]
            self.free_energy_statistics_[key] = fe[d]
        self.free_energy_statistics_["nominal_state_used"] = self.nominal_state_used_

    def updateNominalState(self, u) -> None:
        """tube_mppi_controller.cu:333-343: propagate the nominal state one step with control u."""
        xn, _, _ = self.model_.step(self.nominal_state_trajectory_[0], _f32(u), self.dt_)
        self.nominal_state_trajectory_[0] = xn

    def slideControlSequence(self, steps: int) -> None:
        """tube_mppi_controller.cu:314-325."""
        self.updateNominalState(self.nominal_control_trajectory_[0])
        self._save_control_history(steps, self.nominal_control_trajectory_)
        self._slide(self.nominal_control_trajectory_, steps)
        self._slide(self.control_, steps)


class RobustMPPIController(_Controller):
    """controllers/R-MPPI/robust_mppi_controller.cuh — RobustMPPIController(model, cost, fb_controller, sampler, dt, max_iter,
    lambda, alpha, value_function_threshold, num_timesteps, init_control_traj, num_candidate_nominal_states,
    optimization_stride). Distribution 0 = nominal system, 1 = real system (robust_mppi_controller.cu:637-640). After
    ``initFeedback()`` every updateImportanceSamplingControl recomputes the DDP gains on the device (the engine's feedback
    buffer is written by the kernel); otherwise the gain trajectory is an input (``setFeedbackGains``; none = no feedback)."""
    NUM_DISTRIBUTIONS = 2

    def __init__(self, model, cost, fb_controller, sampler, dt: float, max_iter: int, lambda_: float, alpha: float,
                 value_function_threshold: float, num_timesteps: int, num_rollouts: int, init_control_traj=None,
                 num_candidate_nominal_states: int = 9, optimization_stride: int = 1,
                 eval_samples_per_candidate: int = 64, **kw):
        kw["flags"] = kw.get("flags", 0) | FLAG_RMPPI
        super().__init__(model, cost, fb_controller, sampler, dt, max_iter, lambda_, alpha, num_timesteps, num_rollouts,
                         init_control_traj, **kw)
        self.value_function_threshold_ = value_function_threshold
        self.optimization_stride_ = optimization_stride
        self.eval_samples_per_candidate_ = eval_samples_per_candidate
        self.nominal_control_trajectory_ = self.control_.copy()
        self.nominal_control_history_ = np.zeros_like(self.control_history_)
        self.nominal_state_trajectory_ = np.zeros_like(self.state_)
        self.nominal_state_ = np.zeros(model.STATE_DIM, np.float32)
        self.nominal_state_init_ = False
        self.nominal_stride_, self.real_stride_, self.best_index_ = 0, 0, 0
        self.feedback_gains_ = None  # [T][S][C]
        self.candidate_free_energy_ = None
        self.updateNumCandidates(num_candidate_nominal_states)
        self.engine.set_rmppi(value_function_threshold, None)

    # robust_mppi_controller.cu:430-467
    def updateNumCandidates(self, n: int) -> None:
        if n * self.eval_samples_per_candidate_ > self.num_rollouts_:
            raise ValueError("(number of candidates) * (SAMPLES_PER_CANDIDATE) cannot exceed NUM_ROLLOUTS")
        if n < 3:
            raise ValueError("number of candidates must be greater or equal to 3")
        if n % 2 == 0:
            raise ValueError("number of candidates must be odd")
        self.num_candidate_nominal_states_ = n
        self.line_search_weights_ = np.zeros((3, n), np.float32)
        lib().mppib_host_rmppi_line_search_weights(n, _ptr(self.line_search_weights_))

    def getNumCandidates(self) -> int:
        return self.num_candidate_nominal_states_

    def setValueFunctionThreshold(self, v: float) -> None:
        self.value_function_threshold_ = v
        self.engine.set_rmppi(v, self.feedback_gains_)

    def getValueFunctionThreshold(self) -> float:
        return self.value_function_threshold_

    def setFeedbackGains(self, gains_cxs_per_step) -> None:
        """gains [T][C][S] (K_t as a C x S matrix) -> device layout [T][S][C] (Eigen column-major, ddp.cu:16). Explicit
        gains switch the DDP computation off until initFeedback() is called again."""
        g = _f32(gains_cxs_per_step)
        T, Cd, S = self.num_timesteps_, self.model_.CONTROL_DIM, self.model_.STATE_DIM
        assert g.shape == (T, Cd, S)
        self.enable_feedback_ = False
        self.feedback_gains_ = np.ascontiguousarray(g.transpose(0, 2, 1))
        self.engine.set_rmppi(self.value_function_threshold_, self.feedback_gains_)

    def computeFeedback(self, state) -> None:
        """robust_mppi_controller.cuh: a no-op — the gains are computed in updateImportanceSamplingControl."""

    def computeFeedbackHelper(self, state, state_traj, control_traj) -> None:
        """The DDP solve starts from the real state and tracks the nominal trajectory; its kernel writes the gains straight
        into the engine's feedback buffer, which the next RMPPI rollout applies."""
        if not self.enable_feedback_:
            return
        self.fb_controller_.computeFeedback(state, state_traj, control_traj, to_rmppi=True)
        self.feedback_gains_ = self.fb_controller_.getFeedbackState()

    def computeNominalFeedbackGains(self, state) -> None:  # robust_mppi_controller.cu:629-632
        self.computeFeedbackHelper(_f32(state), self.nominal_state_trajectory_, self.nominal_control_trajectory_)

    def getNominalControlSeq(self) -> np.ndarray:
        return self.nominal_control_trajectory_

    def getNominalStateSeq(self) -> np.ndarray:
        return self.nominal_state_trajectory_

    # robust_mppi_controller.cu:571-617
    def computeNominalStateAndStride(self, state, stride: int) -> None:
        state = _f32(state)
        if not self.nominal_state_init_:
            self.nominal_state_ = state.copy()
            self.nominal_state_init_ = True
            self.nominal_stride_ = 0
            return
        K, S = self.num_candidate_nominal_states_, self.model_.STATE_DIM
        cand = np.zeros((K, S), np.float32)
        strides = np.zeros(K, np.int32)
        lib().mppib_host_rmppi_candidates(K, S, _ptr(_f32(self.nominal_state_trajectory_[0])),
                                          _ptr(_f32(self.nominal_state_trajectory_[1])), _ptr(state), stride, _ptr(cand),
                                          strides.ctypes.data_as(C.c_void_p))
        costs = self.engine.init_eval(cand, strides, self.eval_samples_per_candidate_,
                                      self.nominal_control_trajectory_, stride)
        fe = np.zeros(K, np.float32)
        self.best_index_ = lib().mppib_host_rmppi_best_index(_ptr(costs), K, self.eval_samples_per_candidate_,
                                                             C.c_float(self.lambda_),
                                                             C.c_float(self.value_function_threshold_), self.best_index_,
                                                             _ptr(fe))
        self.candidate_free_energy_, self.candidate_nominal_states_, self.importance_sampler_strides_ = fe, cand, strides
        self.nominal_stride_ = int(strides[self.best_index_])
        self.nominal_state_ = cand[self.best_index_].copy()

    # robust_mppi_controller.cu:539-563
    def updateImportanceSamplingControl(self, state, stride: int) -> None:
        self.real_stride_ = stride
        self.computeNominalStateAndStride(state, stride)
        self._save_history(self.nominal_stride_, self.nominal_control_trajectory_, self.nominal_control_history_)
        self._save_history(self.real_stride_, self.control_, self.control_history_)
        self._slide(self.nominal_control_trajectory_, self.nominal_stride_)
        self._output_trajectory(self.nominal_state_, self.nominal_control_trajectory_, self.nominal_state_trajectory_,
                                np.zeros_like(self.output_))
        self.computeNominalFeedbackGains(state)

    def _save_history(self, steps: int, u: np.ndarray, hist: np.ndarray) -> None:  # controller.cuh:602-616
        if steps == 1:
            hist[0] = hist[1]
            hist[1] = u[0]
        elif steps >= 2:
            hist[0] = u[steps - 2]
            hist[1] = u[steps - 1]

    # robust_mppi_controller.cu:625-755
    def computeControl(self, state, optimization_stride: int = 1) -> None:
        state = _f32(state)
        if not self.nominal_state_init_:
            self.nominal_state_ = state.copy()
            self.nominal_state_init_ = True
        x0 = np.stack([self.nominal_state_, state]).astype(np.float32)
        for it in range(self.num_iters_):
            U_in = np.stack([self.nominal_control_trajectory_, self.nominal_control_trajectory_]).astype(np.float32)
            U, stats = self.engine.solve(x0, U_in, optimization_stride, it)
            self.nominal_control_trajectory_ = U[0].copy()
            self.control_ = U[1].copy()
            for d in range(2):
                self.baseline_[d], self.normalizer_[d] = stats[d][0], stats[d][1]
        self.free_energy_statistics_ = {"nominal_sys": self._free_energy(stats[0]), "real_sys": self._free_energy(stats[1]),
                                        "nominal_state_used": self.best_index_}
        self._smooth_with(self.control_, self.control_history_)
        self._smooth_with(self.nominal_control_trajectory_, self.nominal_control_history_)
        self._output_trajectory(self.nominal_state_, self.nominal_control_trajectory_, self.nominal_state_trajectory_,
                                self.output_)
        self.state_ = self.nominal_state_trajectory_

    def _smooth_with(self, u: np.ndarray, hist: np.ndarray) -> None:
        lib().mppib_host_smooth_controls(_ptr(u), _ptr(hist), self.num_timesteps_, self.model_.CONTROL_DIM)

    def slideControlSequence(self, steps: int) -> None:
        """robust_mppi_controller.cuh:186-190: a no-op — the nominal control slides by its own stride inside
        updateImportanceSamplingControl, which the plant calls before each optimisation."""
