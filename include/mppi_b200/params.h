/*
 * mppi_b200/params.h — plain-C parameter blobs that cross the C-ABI (include/mppi_b200.h).
 *
 * The reference keeps every plugin's parameters in a POD struct that it memcpy's to the device
 * (include/mppi/utils/managed.cuh:121-131). Templates cannot cross a C ABI, so the same information
 * crosses it here as fixed-layout C structs selected by a plugin id. Each struct cites the reference
 * struct whose fields it carries. All floats are IEEE binary32, all ints 32 bit, no padding surprises
 * (only 4-byte members).
 */
#ifndef MPPI_B200_PARAMS_H_
#define MPPI_B200_PARAMS_H_

#ifdef __cplusplus
extern "C" {
#endif

#define MPPIB_MAX_CONTROL_DIM 4
#define MPPIB_MAX_DISTRIBUTIONS 2 /* sampling_distributions/gaussian/gaussian.cuh:20-25 (MAX_DISTRIBUTIONS_T = 2) */

/* ---- plugin ids -------------------------------------------------------------------------------- */
enum mppib_dynamics_id
{
  MPPIB_DYN_CARTPOLE = 0,          /* dynamics/cartpole/cartpole_dynamics.cuh            S4 C1 O4 */
  MPPIB_DYN_DOUBLE_INTEGRATOR = 1, /* dynamics/double_integrator/di_dynamics.cuh         S4 C2 O4 */
  MPPIB_DYN_AUTORALLY_NN = 2,      /* dynamics/autorally/ar_nn_model.cuh NeuralNetModel<7,2,3>  S7 C2 O8 */
  MPPIB_DYN_RACER_LSTM = 3,        /* dynamics/racer_dubins/racer_dubins_elevation_lstm_steering.cuh S19 C2 O28 */
  MPPIB_DYN_QUADROTOR = 4,         /* dynamics/quadrotor/quadrotor_dynamics.cuh          S13 C4 O13 */
  MPPIB_DYN_RACER_DUBINS_ELEVATION = 5, /* dynamics/racer_dubins/racer_dubins_elevation.cuh  S19 C2 O28 */
  MPPIB_DYN_RACER_SUSPENSION_LSTM = 6,  /* dynamics/racer_dubins/racer_dubins_elevation_suspension_lstm.cuh S24 C2 O28 */
  MPPIB_DYN_RACER_SUSPENSION = 7,       /* dynamics/racer_suspension/racer_suspension.cuh (rigid body)  S14 C2 O26 */
  MPPIB_DYN_COUNT
};

enum mppib_cost_id
{
  MPPIB_COST_CARTPOLE_QUADRATIC = 0, /* cost_functions/cartpole/cartpole_quadratic_cost.cuh */
  MPPIB_COST_DI_CIRCLE = 1,          /* cost_functions/double_integrator/double_integrator_circle_cost.cuh */
  MPPIB_COST_AR_STANDARD = 2,        /* cost_functions/autorally/ar_standard_cost.cuh */
  MPPIB_COST_RACER_QUADRATIC = 3,    /* ours (SURVEY §8d C5): quadratic on speed / yaw, documented in DESIGN.md */
  MPPIB_COST_QUADROTOR_QUADRATIC = 4, /* cost_functions/quadrotor/quadrotor_quadratic_cost.cuh */
  MPPIB_COST_DI_ROBUST = 5,          /* cost_functions/double_integrator/double_integrator_robust_cost.cuh (circle params) */
  MPPIB_COST_AR_ROBUST = 6,          /* cost_functions/autorally/ar_robust_cost.cuh */
  MPPIB_COST_QUADROTOR_MAP = 7,      /* cost_functions/quadrotor/quadrotor_map_cost.cuh (map: MPPIB_BLOB_COST_TEXTURE) */
  MPPIB_COST_COUNT
};

enum mppib_sampler_id
{
  MPPIB_SAMPLER_GAUSSIAN = 0,     /* sampling_distributions/gaussian/gaussian.cuh */
  MPPIB_SAMPLER_COLORED_NOISE = 1, /* sampling_distributions/colored_noise/colored_noise.cuh */
  MPPIB_SAMPLER_NLN = 2,           /* sampling_distributions/nln/nln.cuh: normal x log-normal noise, GaussianParams */
  MPPIB_SAMPLER_SMOOTH_MPPI = 3    /* sampling_distributions/smooth-MPPI/smooth-MPPI.cuh: sampled control rates,
                                      mppib_smooth_mppi_params */
};

/* ---- Dynamics base: control limits (dynamics/dynamics.cuh:133,511-512) ------------------------- */
typedef struct mppib_control_limits
{
  float rng_lo[MPPIB_MAX_CONTROL_DIM];   /* control_rngs_[i].x, default -FLT_MAX (dynamics.cuh:103) */
  float rng_hi[MPPIB_MAX_CONTROL_DIM];   /* control_rngs_[i].y, default +FLT_MAX (dynamics.cuh:104) */
  float deadband[MPPIB_MAX_CONTROL_DIM]; /* control_deadband_, default 0 */
  float zero_control[MPPIB_MAX_CONTROL_DIM]; /* zero_control_, default 0 */
} mppib_control_limits;

/* ---- Dynamics parameter blobs ------------------------------------------------------------------- */
typedef struct mppib_cartpole_dyn_params /* dynamics/cartpole/cartpole_dynamics.cuh:27-37 */
{
  mppib_control_limits lim;
  float cart_mass;   /* default 1 */
  float pole_mass;   /* default 1 */
  float pole_length; /* default 1 */
  float gravity;     /* gravity_ = 9.81 (cartpole_dynamics.cuh:101) */
} mppib_cartpole_dyn_params;

typedef struct mppib_di_dyn_params /* dynamics/double_integrator/di_dynamics.cuh:9-25 */
{
  mppib_control_limits lim;
  float system_noise; /* host-side disturbance only; unused on the rollout path */
} mppib_di_dyn_params;

/* NeuralNetModel<7,2,3>: limits here; the 6-32-32-4 weights travel as a separate blob
 * (MPPIB_BLOB_NN_WEIGHTS) in the reference's packed layout: per layer W (row-major out x in) then b
 * (utils/nn_helpers/fnn_helper.cu:176-183). */
#define MPPIB_AR_NN_NUM_PARAMS 1412 /* (6+1)*32 + (32+1)*32 + (32+1)*4 */
typedef struct mppib_ar_nn_dyn_params
{
  mppib_control_limits lim;
} mppib_ar_nn_dyn_params;

/* RacerDubinsElevationLSTMSteering (dynamics/racer_dubins/racer_dubins_elevation_lstm_steering.cuh): the parametric
 * fields of RacerDubinsParams (racer_dubins.cuh:78-104) + RacerDubinsElevationParams (racer_dubins_elevation.cuh:47-59).
 * The LSTM architecture is a constructor argument in the reference (lstm_steering.cu:11-22) and therefore travels in
 * mppib_desc.model_dims = { hidden_dim H, head hidden width L1 } (LSTM input dim is 4, head layers {H+4, L1, 1});
 * the weights travel as MPPIB_BLOB_LSTM_WEIGHTS in the reference's packed layouts:
 *   LSTM  W_im W_fm W_om W_cm (H x H row-major each) | W_ii W_fi W_oi W_ci (H x 4) | b_i b_f b_o b_c (H) |
 *         initial_hidden (H) | initial_cell (H)                               (utils/nn_helpers/lstm_helper.cu:72-88)
 *   head  per layer W (row-major out x in) then b                              (utils/nn_helpers/fnn_helper.cu:176-183)
 * Elevation map: not built yet (flat terrain == TwoDTextureHelper::checkTextureUse(0) false, racer_dubins.cu:427-432). */
#define MPPIB_RACER_LSTM_INPUT_DIM 4
#define MPPIB_RACER_LSTM_NUM_PARAMS(H, L1) \
  (4 * (H) * (H) + 4 * (H) * 4 + 6 * (H) + ((H) + 4) * (L1) + (L1) + (L1) + 1)
typedef struct mppib_racer_lstm_dyn_params
{
  mppib_control_limits lim;
  float c_t[3];                    /* 1.3, 2.6, 3.9 */
  float c_b[3];                    /* 2.5, 3.5, 4.5 */
  float c_v[3];                    /* 3.7, 4.7, 5.7 */
  float c_0;                       /* 4.9 */
  float steering_constant;         /* 0.6 */
  float steer_command_angle_scale; /* 5 */
  float steer_angle_scale;         /* -9.1 */
  float max_steer_angle;           /* 0.5 */
  float max_steer_rate;            /* 5 */
  float steer_accel_constant;      /* 12.1 */
  float steer_accel_drag_constant; /* 1.0 */
  float brake_delay_constant;      /* 6.6 */
  float brake_delay_constant_neg;  /* 8.2 */
  float max_brake_rate_neg;        /* 0.9 */
  float max_brake_rate_pos;        /* 0.33 */
  float wheel_base;                /* 0.3 */
  float low_min_throttle;          /* 0.13 */
  float gravity;                   /* -9.81 */
  int gear_sign;                   /* 1 */
  float clamp_ax;                  /* 5.5 */
  float K_x, K_y, K_yaw, K_vel_x;  /* 1 */
  float Q_x_acc;                   /* 1 */
  float Q_x_v[3];                  /* 41.74219, -0.8187027, -2.2131343 */
  float Q_y_f;                     /* 0.1 */
  float Q_omega_v;                 /* 0.001 */
  float Q_omega_steering;          /* 0 */
} mppib_racer_lstm_dyn_params;

/* RacerDubinsElevation (dynamics/racer_dubins/racer_dubins_elevation.cuh): RacerDubinsElevationParams, the same fields as
 * the LSTM model's blob, which carries exactly them. steer_accel_constant / steer_accel_drag_constant are unused by this
 * model (its steering is first order, racer_dubins.cu:296-304). Map: MPPIB_BLOB_ELEVATION_MAP; no weights. */
typedef mppib_racer_lstm_dyn_params mppib_racer_dubins_elevation_dyn_params;

/* RacerDubinsElevationSuspension (dynamics/racer_dubins/racer_dubins_elevation_suspension_lstm.cuh:14-64): the LSTM model's
 * blob followed by RacerDubinsElevationSuspensionParams' own fields. The steering network, model_dims and
 * MPPIB_BLOB_LSTM_WEIGHTS are exactly the LSTM model's. Maps: MPPIB_BLOB_ELEVATION_MAP (wheel heights, unset = 0) and
 * MPPIB_BLOB_NORMALS_MAP (terrain normals, unset = (0, 0, 1)), both optional. */
typedef struct mppib_racer_suspension_dyn_params
{
  mppib_racer_lstm_dyn_params base;
  float spring_k;     /* 14000 N / m */
  float drag_c;       /* 1000 N s / m */
  float mass;         /* 1447 kg */
  float I_xx;         /* mass * 2 * 1.5^2 / 12 */
  float I_yy;         /* mass * (1.5^2 + 3^2) / 12 */
  float wheel_radius; /* 0.32 m */
  float c_g[3];       /* centre of gravity in the body frame: (2.981 / 2, 0, 0) */
} mppib_racer_suspension_dyn_params;

/* RacerSuspension (dynamics/racer_suspension/racer_suspension.cuh:8-128, RacerSuspensionParams), the 6-DoF rigid body on
 * four spring-damper wheels, field for field: float3 as three floats, the fields recalcParams() derives included (the host
 * classes derive them; the engine reads them as given). Not to be confused with id 6's mppib_racer_suspension_dyn_params.
 * Wheels in the order front left, front right, rear left, rear right. No map: the model's ground is the plane z = 0. */
typedef struct mppib_racer_rigid_suspension_dyn_params
{
  mppib_control_limits lim;
  float wheel_radius;                  /* 0.32 m */
  float mass;                          /* 1447 kg */
  float wheel_base;                    /* 2.981 m */
  float width;                         /* 1.5 m */
  float height;                        /* 1.5 m */
  float gravity;                       /* -9.81 */
  float k_s[4];                        /* 14000 N / m */
  float c_s[4];                        /* 2000 N s / m */
  float l_0[4];                        /* derived: wheel_radius + mass / 4 * (-gravity) / k_s[i] */
  float cg_pos_wrt_base_link[3];       /* derived: (wheel_base / 2, 0, 0.2) */
  float wheel_pos_wrt_base_link[4][3]; /* derived: (wheel_base, +-width / 2, 0), (0, +-width / 2, 0) */
  float Jxx, Jyy, Jzz;                 /* derived, in double: mass / 12 * (sum of two squared extents) */
  float mu;                            /* 0.65 */
  float v_slip;                        /* 0.1 m / s */
  float c_t;                           /* 3.0 */
  float c_b;                           /* 10.0 */
  float c_v;                           /* 0.2 */
  float c_0;                           /* 0 */
  float steering_constant;             /* 0.6 */
  float steer_command_angle_scale;     /* -2.45 */
  int gear_sign;                       /* 1 (not read by the model) */
} mppib_racer_rigid_suspension_dyn_params;

/* Elevation map of the RACER models (utils/texture_helpers/texture_helper.cuh:11-56 TextureParams + two_d_texture_helper.cu):
 * MPPIB_BLOB_ELEVATION_MAP = this header followed by width * height floats, row-major (value at row i, column j =
 * data[i * width + j]: TwoDTextureHelper's cpu_values_ layout). Clamp addressing, bilinear filtering, normalised
 * coordinates (the TextureParams defaults). `use` is enableTexture / checkTextureUse (texture_helper.cu): with use == 0 the
 * model settles on flat ground (racer_dubins.cu:427-432). */
typedef struct mppib_elevation_map_header
{
  int width, height;   /* cudaExtent: width = x cells, height = y cells (both >= 2) */
  float origin[3];     /* TextureParams::origin */
  float rotations[9];  /* TextureParams::rotations[3], row-major: map = R (world - origin) */
  float resolution[3]; /* metres per cell */
  int use;
} mppib_elevation_map_header;
/* MPPIB_BLOB_NORMALS_MAP (TwoDTextureHelper<float4> map 0 of RacerDubinsElevationSuspension: normals_tex_helper_) is the
 * same header followed by width * height float4 (x, y, z, w), row-major, queried with the same clamp + bilinear formula per
 * channel. */

/* QuadrotorDynamics (dynamics/quadrotor/quadrotor_dynamics.cuh:9-63). State POS(3) VEL(3) QUAT_W..Z(4) ANG_VEL(3);
 * controls ANG_RATE_X/Y/Z, THRUST. The default constructor's thrust range [0, 36] and zero_control[3] = GRAVITY
 * (quadrotor_dynamics.cu:11-19) are set by the host-side mirror, they are not part of the params struct. */
#define MPPIB_GRAVITY 9.81f /* utils/math_utils.h:45 */
typedef struct mppib_quadrotor_dyn_params
{
  mppib_control_limits lim;
  float tau_roll;  /* 0.25 */
  float tau_pitch; /* 0.25 */
  float tau_yaw;   /* 0.25 */
  float mass;      /* 1 kg */
} mppib_quadrotor_dyn_params;

/* ---- Cost parameter blobs ----------------------------------------------------------------------- */
typedef struct mppib_cartpole_cost_params /* cost_functions/cartpole/cartpole_quadratic_cost.cuh:10-23 */
{
  float control_cost_coeff[MPPIB_MAX_CONTROL_DIM]; /* CostParams<1> (cost.cuh:17-31); unused on device (cost.cuh:205-208) */
  float discount;
  float cart_position_coeff;         /* 1000 */
  float cart_velocity_coeff;         /* 100 */
  float pole_angle_coeff;            /* 2000 */
  float pole_angular_velocity_coeff; /* 100 */
  float terminal_cost_coeff;         /* 0 */
  float desired_terminal_state[4];   /* {0,0,pi,0} */
} mppib_cartpole_cost_params;

typedef struct mppib_di_circle_cost_params /* cost_functions/double_integrator/double_integrator_circle_cost.cuh:8-23 */
{
  float control_cost_coeff[MPPIB_MAX_CONTROL_DIM];
  float discount;                 /* 1.0 */
  float velocity_cost;            /* 1 */
  float crash_cost;               /* 1000 */
  float velocity_desired;         /* 2 */
  float inner_path_radius2;       /* 1.875^2 */
  float outer_path_radius2;       /* 2.125^2 */
  float angular_momentum_desired; /* 2*velocity_desired */
} mppib_di_circle_cost_params;

typedef struct mppib_ar_standard_cost_params /* cost_functions/autorally/ar_standard_cost.cuh:14-41 */
{
  float control_cost_coeff[MPPIB_MAX_CONTROL_DIM];
  float discount;           /* CostParams default 1.0 */
  float desired_speed;      /* 6.0 */
  float speed_coeff;        /* 4.25 */
  float track_coeff;        /* 200 */
  float max_slip_ang;       /* 1.25 */
  float slip_coeff;         /* 10 */
  float track_slop;         /* 0 */
  float crash_coeff;        /* 10000 */
  float boundary_threshold; /* 0.65 */
  int grid_res;             /* 10 (unused on the path) */
  float r_c1[3];            /* R matrix col 1 */
  float r_c2[3];            /* R matrix col 2 */
  float trs[3];             /* translation */
  int l1_cost;              /* ARStandardCostImpl::l1_cost_ (ar_standard_cost.cuh), default 0 */
  float front_d;            /* FRONT_D = 0.5  (ar_standard_cost.cuh) */
  float back_d;             /* BACK_D = -0.5 */
  int map_width;            /* texture width  (costmap travels as MPPIB_BLOB_COSTMAP, float4 per texel) */
  int map_height;           /* texture height */
} mppib_ar_standard_cost_params;

/* ARRobustCostParams (cost_functions/autorally/ar_robust_cost.cuh:6-29): every field of the standard blob, in the same order,
 * then heading_coeff. The shared prefix is what the costmap upload (MPPIB_BLOB_COSTMAP reads map_width / map_height) and
 * the map helpers read, so they take either blob. */
typedef struct mppib_ar_robust_cost_params
{
  float control_cost_coeff[MPPIB_MAX_CONTROL_DIM]; /* 0, 0 */
  float discount;           /* 1.0 */
  float desired_speed;      /* -1: follow the map's speed channel (.z) */
  float speed_coeff;        /* 20 */
  float track_coeff;        /* 33 */
  float max_slip_ang;       /* 1.5 */
  float slip_coeff;         /* 0 */
  float track_slop;         /* 0 */
  float crash_coeff;        /* 125000 */
  float boundary_threshold; /* 0.75 */
  int grid_res;             /* 10 (unused on the path) */
  float r_c1[3];
  float r_c2[3];
  float trs[3];
  int l1_cost;              /* unused by this cost */
  float front_d;            /* 0.5 */
  float back_d;             /* -0.5 */
  int map_width;
  int map_height;
  float heading_coeff;      /* 0 */
} mppib_ar_robust_cost_params;

#ifdef __cplusplus
#include <stddef.h>
#define MPPIB_AR_PREFIX_SAME(f) \
  static_assert(offsetof(mppib_ar_robust_cost_params, f) == offsetof(mppib_ar_standard_cost_params, f), #f);
MPPIB_AR_PREFIX_SAME(control_cost_coeff)
MPPIB_AR_PREFIX_SAME(discount)
MPPIB_AR_PREFIX_SAME(desired_speed)
MPPIB_AR_PREFIX_SAME(speed_coeff)
MPPIB_AR_PREFIX_SAME(track_coeff)
MPPIB_AR_PREFIX_SAME(max_slip_ang)
MPPIB_AR_PREFIX_SAME(slip_coeff)
MPPIB_AR_PREFIX_SAME(track_slop)
MPPIB_AR_PREFIX_SAME(crash_coeff)
MPPIB_AR_PREFIX_SAME(boundary_threshold)
MPPIB_AR_PREFIX_SAME(grid_res)
MPPIB_AR_PREFIX_SAME(r_c1)
MPPIB_AR_PREFIX_SAME(r_c2)
MPPIB_AR_PREFIX_SAME(trs)
MPPIB_AR_PREFIX_SAME(l1_cost)
MPPIB_AR_PREFIX_SAME(front_d)
MPPIB_AR_PREFIX_SAME(back_d)
MPPIB_AR_PREFIX_SAME(map_width)
MPPIB_AR_PREFIX_SAME(map_height)
static_assert(offsetof(mppib_ar_robust_cost_params, heading_coeff) == sizeof(mppib_ar_standard_cost_params),
              "heading_coeff follows the standard prefix");
#undef MPPIB_AR_PREFIX_SAME
/* the rigid-body RACER blob: 16 limit floats, then 45 four-byte fields in RacerSuspensionParams' order */
static_assert(offsetof(mppib_racer_rigid_suspension_dyn_params, wheel_radius) == 64, "limits first");
static_assert(offsetof(mppib_racer_rigid_suspension_dyn_params, l_0) == 64 + 14 * 4, "l_0");
static_assert(offsetof(mppib_racer_rigid_suspension_dyn_params, Jxx) == 64 + 33 * 4, "Jxx");
static_assert(offsetof(mppib_racer_rigid_suspension_dyn_params, gear_sign) == 64 + 44 * 4, "gear_sign last");
static_assert(sizeof(mppib_racer_rigid_suspension_dyn_params) == 244, "no padding");
#endif

/* Quadratic tracking cost on the RACER output vector (ours: the RACER cost classes are not in the reference tree,
 * SURVEY §8d C5). cost = speed_coeff (y[VEL_B_X] - desired_speed)^2 + yaw_coeff angdist(y[YAW], desired_yaw)^2
 *                      + lateral_coeff (y[POS_I_Y] - desired_y)^2 + steer_coeff y[STEER_ANGLE]^2, times discount^t;
 * terminal cost 0. */
typedef struct mppib_racer_quadratic_cost_params
{
  float control_cost_coeff[MPPIB_MAX_CONTROL_DIM];
  float discount;      /* 1.0 */
  float desired_speed; /* 5.0 */
  float speed_coeff;   /* 4.0 */
  float desired_yaw;   /* 0.0 */
  float yaw_coeff;     /* 20.0 */
  float desired_y;     /* 0.0 */
  float lateral_coeff; /* 2.0 */
  float steer_coeff;   /* 1.0 */
} mppib_racer_quadratic_cost_params;

/* QuadrotorQuadraticCost (cost_functions/quadrotor/quadrotor_quadratic_cost.cuh:9-66) */
typedef struct mppib_quadrotor_cost_params
{
  float control_cost_coeff[MPPIB_MAX_CONTROL_DIM]; /* 2, 2, 2, 2; unused on device (cost.cuh:205-208) */
  float discount;                                  /* CostParams default 1.0 (unused by this cost) */
  float s_goal[13];                                /* x(3) v(3) q(4: 1,0,0,0) w(3) */
  float x_coeff;                                   /* 1 */
  float v_coeff;                                   /* 1 */
  int use_euler;                                   /* true */
  float q_coeff;                                   /* 1 */
  float roll_coeff;                                /* 1 */
  float pitch_coeff;                               /* 1 */
  float yaw_coeff;                                 /* 1 */
  float w_coeff;                                   /* 1 */
  float terminal_cost_coeff;                       /* 0 */
} mppib_quadrotor_cost_params;

/* QuadrotorMapCostParams (cost_functions/quadrotor/quadrotor_map_cost.cuh:14-91) without r_c1 / r_c2 / trs, which only
 * the reference's float4 track texture reads and no cost body does. float4 waypoints are (x, y, z, heading), float3
 * gate corners (x, y, z). The cost's map is TwoDTextureHelper<float> map 0 and travels as MPPIB_BLOB_COST_TEXTURE in
 * the mppib_elevation_map_header format; without it the costmap term is 0 (checkTextureUse(0) false). */
typedef struct mppib_quadrotor_map_cost_params
{
  float control_cost_coeff[MPPIB_MAX_CONTROL_DIM]; /* 1, 1, 1, 1 */
  float discount;                                  /* CostParams default 1.0 (unused by this cost) */
  float attitude_coeff;                            /* 10 */
  float crash_coeff;                               /* 1000 */
  float dist_to_waypoint_coeff;                    /* 0 */
  float heading_coeff;                             /* 5 */
  float heading_power;                             /* 1 */
  float height_coeff;                              /* 5 */
  float track_coeff;                               /* 10 */
  float speed_coeff;                               /* 5 */
  float track_slop;                                /* 0 */
  float gate_pass_cost;                            /* -150 */
  float curr_waypoint[4];                          /* 0, 0, 0, 0 */
  float prev_waypoint[4];                          /* 0, 0, 0, 0 */
  float curr_gate_left[3];                         /* 0, 0, 0 */
  float curr_gate_right[3];                        /* 0, 0, 0 */
  float prev_gate_left[3];                         /* 0, 0, 0 */
  float prev_gate_right[3];                        /* 0, 0, 0 */
  float end_waypoint[4];                           /* NaN x 4 (unused by the cost bodies) */
  float desired_speed;                             /* 5 m/s */
  float gate_margin;                               /* 0.5 m */
  float min_dist_to_gate_side;                     /* 0.5 m */
  float track_boundary_cost;                       /* 2.5 */
  float gate_width;                                /* 2.15 m */
} mppib_quadrotor_map_cost_params;
/* ---- Sampler parameter blob (sampling_distribution.cuh:14-29, gaussian.cuh:21-61) --------------- */
typedef struct mppib_gaussian_params
{
  float std_dev[MPPIB_MAX_CONTROL_DIM * MPPIB_MAX_DISTRIBUTIONS]; /* [d][c] with stride CONTROL_DIM of the plugin */
  float control_cost_coeff[MPPIB_MAX_CONTROL_DIM];                /* default 0 (gaussian.cuh:26) */
  float pure_noise_trajectories_percentage;                       /* 0.01 */
  float std_dev_decay;                                            /* 1.0 */
  int sum_strides;                          /* 32; kept for API parity, this engine's reduction does not use it */
  int use_same_noise_for_all_distributions; /* 1 (sampling_distribution.cuh:20) */
  /* ColoredNoise extras (colored_noise.cuh:41-60); ignored by the Gaussian sampler */
  float exponents[MPPIB_MAX_CONTROL_DIM * MPPIB_MAX_DISTRIBUTIONS]; /* default 0 == white */
  float offset_decay_rate;                                          /* 0.97 */
  float fmin;                                                       /* 0.0 */
} mppib_gaussian_params;

/* SmoothMPPIParams (smooth-MPPI.cuh:15-24): the Gaussian blob, then the sampler's own integration step. The rates are
 * sampled with the Gaussian fields; a control is mu + rate * dt. The blob of MPPIB_BLOB_SAMPLER_PARAMS on a
 * MPPIB_SAMPLER_SMOOTH_MPPI engine. */
typedef struct mppib_smooth_mppi_params
{
  mppib_gaussian_params gaussian;
  float dt; /* 0.015 (smooth-MPPI.cuh:21); not the controller's dt */
} mppib_smooth_mppi_params;

#ifdef __cplusplus
}
#endif
#endif /* MPPI_B200_PARAMS_H_ */
