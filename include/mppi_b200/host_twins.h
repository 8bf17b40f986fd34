/*
 * mppi_b200/host_twins.h — CPU twins of the plugins and the controller's host tail, exported by libmppi_b200.so
 * (mppi-generic_b200/csrc/host_twins.cpp). Each replaces a host method of the reference's templated classes:
 *   mppib_host_enforce_constraints  Dynamics::enforceConstraints          include/mppi/dynamics/dynamics.cuh:250-264
 *   mppib_host_step                 Dynamics::step (host)                 dynamics.cuh:283-290
 *   mppib_host_smooth_controls      Controller::smoothControlTrajectoryHelper   controllers/controller.cuh:557-586
 *   mppib_host_slide_controls       Controller::slideControlSequenceHelper      controller.cuh:588-600
 *   mppib_host_output_trajectory    Controller::computeOutputTrajectoryHelper   controller.cuh:643-663
 *   mppib_host_step_lstm / mppib_host_output_trajectory_lstm   the same two for RacerDubinsElevationLSTMSteering
 *   mppib_host_step_racer_suspension / mppib_host_output_trajectory_racer_suspension   ... for RacerDubinsElevationSuspension
 *   mppib_host_step_racer_rigid_suspension / _output_trajectory_racer_rigid_suspension ... for RacerSuspension (rigid body)
 *   mppib_host_free_energy          mppi::kernels::computeFreeEnergy      include/mppi/core/mppi_common.cu:1065-1081
 *   mppib_host_merge_records        (no reference counterpart: the log-sum-exp merge of rollout shards, SURVEY §8e)
 *   mppib_host_state_cost           the robust costs' and QuadrotorMapCost's host computeStateCost and terms (below)
 * Arrays: u / history are [T][C] / [2][C] (== Eigen C x T / C x 2 column-major), states [T][S], outputs [T][O].
 */
#ifndef MPPI_B200_HOST_TWINS_H_
#define MPPI_B200_HOST_TWINS_H_
#include <stddef.h>

#include "../mppi_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
int mppib_host_dims(int dyn_id, int* S, int* C, int* O);
int mppib_host_enforce_constraints(int dyn_id, const void* dyn_params, float* u);
int mppib_host_step(int dyn_id, const void* dyn_params, const float* nn_theta, const float* x, const float* u,
                    float dt, float* x_next, float* xdot, float* y);
void mppib_host_smooth_controls(float* u, const float* history, int T, int C);
void mppib_host_slide_controls(float* u, int steps, int T, int C, const float* zero_control, const float* scale);
int mppib_host_output_trajectory(int dyn_id, const void* dyn_params, const float* nn_theta, const float* x0,
                                 const float* u, int T, float dt, float* states, float* outputs);
/* RacerDubinsElevationLSTMSteering (racer_dubins_elevation_lstm_steering.cu:90-118): the model carries its LSTM's
 * hidden / cell vectors from step to step, so its host twin takes them explicitly (updated in place by _step_lstm;
 * _output_trajectory_lstm starts from the initial state stored in the weight blob and leaves `net` untouched). */
typedef struct mppib_host_lstm
{
  const float* theta; /* MPPIB_BLOB_LSTM_WEIGHTS layout (params.h) */
  int hidden_dim;     /* H */
  int head_hidden;    /* L1 */
  float* hidden;      /* [H] */
  float* cell;        /* [H] */
  const mppib_elevation_map_header* map; /* header + width * height floats (params.h), or NULL = flat ground */
} mppib_host_lstm;
/* TwoDTextureHelper<float>::queryTextureAtWorldPose on the host (texture_helper.cu:94-134,274-280 + two_d_texture_helper.cu:
 * 151-243: clamp addressing, bilinear filter) — what the RACER models' computeStaticSettling samples. */
float mppib_host_elevation_at_world_pose(const mppib_elevation_map_header* map, float x, float y, float z);
/* RACER::computeStaticSettling (racer_dubins.cu:359-434): roll / pitch in: current, out: settled; returns the height. */
float mppib_host_static_settling(const mppib_elevation_map_header* map, float yaw, float x, float y, float* roll,
                                 float* pitch);
int mppib_host_step_lstm(const void* dyn_params, const mppib_host_lstm* net, const float* x, const float* u, float dt,
                         float* x_next, float* xdot, float* y);
int mppib_host_output_trajectory_lstm(const void* dyn_params, const mppib_host_lstm* net, const float* x0,
                                      const float* u, int T, float dt, float* states, float* outputs);
/* RacerDubinsElevation (racer_dubins_elevation.cu:229-255, host step): the host body, which differs from the device one
 * (DESIGN §8) in sinf / tanf / sincosf without normalizeAngle and in its brake clamp [0, -control_rngs_[0].x]. map may be
 * NULL (flat ground). */
int mppib_host_step_racer_dubins_elevation(const void* dyn_params, const mppib_elevation_map_header* map, const float* x,
                                           const float* u, float dt, float* x_next, float* xdot, float* y);
/* RacerDubinsElevation::computeGrad (racer_dubins_elevation.cu:257-334): A [19][19] and B [19][2], row-major. */
int mppib_host_grad_racer_dubins_elevation(const void* dyn_params, const float* x, const float* u, float* A, float* B);
int mppib_host_output_trajectory_racer_dubins_elevation(const void* dyn_params, const mppib_elevation_map_header* map,
                                                        const float* x0, const float* u, int T, float dt, float* states,
                                                        float* outputs);
/* RacerDubinsElevationSuspension (racer_dubins_elevation_suspension_lstm.cu:59-197,420-525, host step): the LSTM model's
 * network and elevation map in `net` (net->map, NULL = height 0), the normals map (header + width * height float4, NULL =
 * (0, 0, 1)) apart. The host body differs from the device one (DESIGN §8) in sincosf / sinf / tanf of raw angles and in
 * its brake clamp [0, -control_rngs_[0].x]. S = 24, O = 28; the LSTM state in `net` is updated in place by the step, and
 * the trajectory starts from the initial state in the weight blob. */
int mppib_host_step_racer_suspension(const void* dyn_params, const mppib_host_lstm* net,
                                     const mppib_elevation_map_header* normals, const float* x, const float* u, float dt,
                                     float* x_next, float* xdot, float* y);
int mppib_host_output_trajectory_racer_suspension(const void* dyn_params, const mppib_host_lstm* net,
                                                  const mppib_elevation_map_header* normals, const float* x0,
                                                  const float* u, int T, float dt, float* states, float* outputs);
/* RacerSuspension, the rigid body (dynamics/racer_suspension/racer_suspension.cu; blob mppib_racer_rigid_suspension_dyn_params,
 * S = 14, O = 26). _state_deriv: the host computeStateDeriv (:93-298) on the plane z = 0, outputs of x, and when
 * omega_jacobian != NULL the 3x3 omegaJacobian row-major, as written (f_r_B_i_Jac = f_r_C_i_Jac, :215). _step: the host
 * step (:31-45), the body rates by approximate implicit Euler through that Jacobian, then q / |q|; y = the outputs of x.
 * The device step is explicit Euler on every state (DESIGN §8). */
int mppib_host_state_deriv_racer_rigid_suspension(const void* dyn_params, const float* x, const float* u, float* xdot,
                                                  float* y, float* omega_jacobian);
int mppib_host_step_racer_rigid_suspension(const void* dyn_params, const float* x, const float* u, float dt, float* x_next,
                                           float* xdot, float* y);
int mppib_host_output_trajectory_racer_rigid_suspension(const void* dyn_params, const float* x0, const float* u, int T,
                                                        float dt, float* states, float* outputs);
/* TwoDTextureHelper<float4>::queryTextureAtWorldPose on the host: out4 = the four channels, each by the float map's
 * formula (mppib_host_elevation_at_world_pose); map NULL: (0, 0, 1, 0). */
void mppib_host_normals_at_world_pose(const mppib_elevation_map_header* map, float x, float y, float z, float* out4);
/* LSTMLSTMHelper::initializeLSTM (utils/nn_helpers/lstm_lstm_helper.cu:50-73): the INIT network — an LSTM (input_dim, hidden_dim)
 * with an FNN head on [h; x] (layers {hidden_dim + input_dim, ..., 2 * H_prediction}) — runs over the last init_len columns
 * of a buffer of past inputs, starting from its own initial hidden / cell state; the head's output after the last column is
 * the prediction LSTM's initial hidden (first half) and cell (second half) state. Host-only in the reference too.
 *   lstm_theta  W_im W_fm W_om W_cm [H x H each] | W_ii W_fi W_oi W_ci [H x I each] | b_i b_f b_o b_c [H each] |
 *               initial hidden [H] | initial cell [H]                      (lstm_helper.cu:72-88)
 *   head_theta  packed W (out x in, row-major) then b, layer after layer   (fnn_helper.cu:176-183); tanh between layers
 *   buffer      [cols][input_dim]: element (t, r) = the reference's buffer(r, t); cols >= init_len
 *   out         [head_layers[head_num_layers - 1]] */
typedef struct mppib_host_init_lstm
{
  const float* lstm_theta;
  int input_dim, hidden_dim;
  const float* head_theta;
  const int* head_layers;
  int head_num_layers;
  int init_len;
} mppib_host_init_lstm;
int mppib_host_lstm_initialize(const mppib_host_init_lstm* net, const float* buffer, int cols, float* out);
/* RobustMPPI host logic (controllers/R-MPPI/robust_mppi_controller.cu:351-362,472-537): line-search weights [3][K],
 * nominal-state candidates [K][S] + importance-sampler strides [K], best candidate (returns previous_best if none
 * is under the value-function threshold). */
void mppib_host_rmppi_line_search_weights(int num_candidates, float* out);
void mppib_host_rmppi_candidates(int num_candidates, int S, const float* nominal_x_k, const float* nominal_x_kp1,
                                 const float* real_x_kp1, int stride, float* candidates, int* strides);
int mppib_host_rmppi_best_index(const float* costs, int num_candidates, int samples_per_candidate, float lambda,
                                float value_func_threshold, int previous_best, float* free_energy);
void mppib_host_free_energy(const mppib_solve_stats* st, int num_rollouts, float lambda, float* out3);
/* CPU twin of the K2 merge (csrc/combine_kernel.cuh): records [nrec][D][pstride] = (beta, eta, sum w^2, -, V[TC]). */
int mppib_host_merge_records(const float* records, int nrec, int D, int TC, int pstride, float lambda, int normalize,
                             float* out);
/* One array of a NumPy .npz archive, converted to float — the input format of the reference's FNNHelper::loadParams
 * (utils/nn_helpers/fnn_helper.cu:44-127: "dynamics_W<i>" / "dynamics_b<i>", float64) and ARStandardCostImpl::loadTrackData
 * (cost_functions/autorally/ar_standard_cost.cu:85-142: "xBounds", "yBounds", "pixelsPerMeter", "channel0..3", float32),
 * which go through cnpy::npz_load. `name` without ".npy". Stored and deflated members; little-endian f4 / f8 / i4 / i8; C
 * order; up to 4 dimensions. out == NULL: only *count / shape4 / *ndim are filled. */
int mppib_host_npz_read(const char* path, const char* name, float* out, size_t capacity, size_t* count, int* shape4,
                        int* ndim);
/* Host bodies of the robust costs, which the reference calls directly (cost.computeStateCost(y, t, &crash),
 * ARRobustCost::getStabilizingCost / getCostmapCost):
 *   MPPIB_COST_DI_ROBUST  double_integrator_robust_cost.cu:41-69: the HOST constants (steep boundary 0.75, steep cost
 *                         0.1 * crash_cost); the rollouts use the device body's 0.5 / 0.5 * crash_cost, as in the reference
 *   MPPIB_COST_AR_ROBUST  ar_robust_cost.cu:13-132, host branch: cosf / sinf and the nearest texel (std::round after the
 *                         clamps of :64-70); costmap = float4 per texel, row-major [map_height][map_width]
 *   MPPIB_COST_QUADROTOR_MAP  quadrotor_map_cost.cu:63-90, the host body: gate side + height + heading + speed +
 *                         stabilizing + waypoint terms and the gate-pass term; no costmap term and no crash flag (the
 *                         rollouts use the device body, :92-144). `costmap` is not read.
 * `params` is the cost's parameter blob (params.h). Other cost ids: MPPIB_ERR_UNSUPPORTED. No cost reads t or crash. */
int mppib_host_state_cost(int cost_id, const void* params, const float* costmap, const float* y, int t, int* crash,
                          float* cost);
int mppib_host_ar_robust_stabilizing_cost(const mppib_ar_robust_cost_params* params, const float* s, float* cost);
int mppib_host_ar_robust_costmap_cost(const mppib_ar_robust_cost_params* params, const float* costmap, const float* s,
                                      float* cost);
/* QuadrotorMapCost's __host__ __device__ terms (quadrotor_map_cost.cu:199-357), host side, one per `term`; an unknown
 * term is MPPIB_ERR_INVALID_ARG. distToWaypoint (:146-152) takes the waypoint as (x, y, z[, heading]). */
enum mppib_quadrotor_map_term
{
  MPPIB_QMAP_GATE_SIDE = 0,   /* computeGateSideCost    :264-323 */
  MPPIB_QMAP_HEADING = 1,     /* computeHeadingCost     :210-238 */
  MPPIB_QMAP_HEIGHT = 2,      /* computeHeightCost      :325-357 */
  MPPIB_QMAP_SPEED = 3,       /* computeSpeedCost       :240-252 */
  MPPIB_QMAP_STABILIZING = 4, /* computeStabilizingCost :199-208 */
  MPPIB_QMAP_WAYPOINT = 5     /* computeWaypointCost    :254-262 */
};
int mppib_host_quadrotor_map_term(const mppib_quadrotor_map_cost_params* params, int term, const float* s, float* cost);
float mppib_host_quadrotor_map_dist_to_waypoint(const float* s, const float* waypoint);
/* QuadrotorMapCostParams::updateWaypoint / updateGateBoundaries (quadrotor_map_cost.cuh:62-90): shift curr -> prev and set
 * the new values (updateWaypoint derives the gate corners x +- cosf(heading) gate_width, y +- sinf(heading) gate_width).
 * Return 1 if anything changed, 0 if not (the cost pushes its parameters only then), MPPIB_ERR_INVALID_ARG for NULL. Both
 * the C++ and the Python mirror call these, so they produce the same bytes. */
int mppib_host_quadrotor_map_update_waypoint(mppib_quadrotor_map_cost_params* p, float x, float y, float z, float heading);
int mppib_host_quadrotor_map_update_gate_boundaries(mppib_quadrotor_map_cost_params* p, float left_x, float left_y,
                                                    float left_z, float right_x, float right_y, float right_z);
#ifdef __cplusplus
}
#endif
#endif
