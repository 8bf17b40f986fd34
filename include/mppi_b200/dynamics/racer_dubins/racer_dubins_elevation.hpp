/*
 * RacerDubinsElevation — host class of include/mppi/dynamics/racer_dubins/racer_dubins_elevation.cuh (parameters:
 * racer_dubins.cuh:13-104, racer_dubins_elevation.cuh:16-59). S19 C2 O28, the parametric RACER vehicle: first-order
 * steering and nothing carried between steps but the state, so Tube-MPPI and RMPPI roll it out and DDPFeedback takes its
 * computeGrad. Same constructors as the reference: RacerDubinsElevation(stream), RacerDubinsElevation(params, stream).
 * Map 0 of getTextureHelper() is the elevation map computeStaticSettling samples.
 */
#pragma once
#include <cmath>
#include <memory>
#include <string>

#include "../dynamics.hpp"
#include "../../utils/texture_helpers/two_d_texture_helper.hpp"

struct RacerDubinsElevationParams
{
  enum class StateIndex : int
  {
    VEL_X = 0, YAW, POS_X, POS_Y, STEER_ANGLE, BRAKE_STATE, ROLL, PITCH, STEER_ANGLE_RATE, UNCERTAINTY_POS_X,
    UNCERTAINTY_POS_Y, UNCERTAINTY_YAW, UNCERTAINTY_VEL_X, UNCERTAINTY_POS_X_Y, UNCERTAINTY_POS_X_YAW,
    UNCERTAINTY_POS_X_VEL_X, UNCERTAINTY_POS_Y_YAW, UNCERTAINTY_POS_Y_VEL_X, UNCERTAINTY_YAW_VEL_X, NUM_STATES
  };
  enum class ControlIndex : int { THROTTLE_BRAKE = 0, STEER_CMD, NUM_CONTROLS };
  enum class OutputIndex : int
  {
    BASELINK_VEL_B_X = 0, BASELINK_VEL_B_Y, BASELINK_POS_I_X, BASELINK_POS_I_Y, BASELINK_POS_I_Z, YAW, ROLL, PITCH,
    STEER_ANGLE, STEER_ANGLE_RATE, WHEEL_FORCE_UP_MAX, WHEEL_FORCE_FWD_MAX, WHEEL_FORCE_SIDE_MAX, ACCEL_X, ACCEL_Y,
    OMEGA_Z, TOTAL_VELOCITY, UNCERTAINTY_POS_X, UNCERTAINTY_POS_Y, UNCERTAINTY_YAW, UNCERTAINTY_VEL_X,
    UNCERTAINTY_POS_X_Y, UNCERTAINTY_POS_X_YAW, UNCERTAINTY_POS_X_VEL_X, UNCERTAINTY_POS_Y_YAW, UNCERTAINTY_POS_Y_VEL_X,
    UNCERTAINTY_YAW_VEL_X, FILLER_1, NUM_OUTPUTS
  };
  // racer_dubins.cuh:78-104
  float c_t[3] = { 1.3f, 2.6f, 3.9f };
  float c_b[3] = { 2.5f, 3.5f, 4.5f };
  float c_v[3] = { 3.7f, 4.7f, 5.7f };
  float c_0 = 4.9f;
  float steering_constant = .6f;
  float steer_command_angle_scale = 5;
  float steer_angle_scale = -9.1f;
  float max_steer_angle = 0.5f;
  float max_steer_rate = 5;
  float steer_accel_constant = 12.1f;
  float steer_accel_drag_constant = 1.0f;
  float brake_delay_constant = 6.6f;
  float brake_delay_constant_neg = 8.2f;
  float max_brake_rate_neg = 0.9f;
  float max_brake_rate_pos = 0.33f;
  float wheel_base = 0.3f;
  float low_min_throttle = 0.13f;
  float gravity = -9.81f;
  int gear_sign = 1;
  // racer_dubins_elevation.cuh:47-59
  float clamp_ax = 5.5f;
  float K_x = 1.0f, K_y = 1.0f, K_yaw = 1.0f, K_vel_x = 1.0f;
  float Q_x_acc = 1.0f;
  float Q_x_v[3] = { 41.74219f, -0.8187027f, -2.2131343f };
  float Q_y_f = 0.1f;
  float Q_omega_v = 0.001f;
  float Q_omega_steering = 0.0f;
};

// the blob both RACER elevation models send: RacerDubinsElevationParams field by field (params.h)
inline mppib_racer_dubins_elevation_dyn_params racer_elevation_blob(const RacerDubinsElevationParams& p)
{
  mppib_racer_dubins_elevation_dyn_params b{};
  for (int i = 0; i < 3; i++)
  {
    b.c_t[i] = p.c_t[i];
    b.c_b[i] = p.c_b[i];
    b.c_v[i] = p.c_v[i];
    b.Q_x_v[i] = p.Q_x_v[i];
  }
  b.c_0 = p.c_0;
  b.steering_constant = p.steering_constant;
  b.steer_command_angle_scale = p.steer_command_angle_scale;
  b.steer_angle_scale = p.steer_angle_scale;
  b.max_steer_angle = p.max_steer_angle;
  b.max_steer_rate = p.max_steer_rate;
  b.steer_accel_constant = p.steer_accel_constant;
  b.steer_accel_drag_constant = p.steer_accel_drag_constant;
  b.brake_delay_constant = p.brake_delay_constant;
  b.brake_delay_constant_neg = p.brake_delay_constant_neg;
  b.max_brake_rate_neg = p.max_brake_rate_neg;
  b.max_brake_rate_pos = p.max_brake_rate_pos;
  b.wheel_base = p.wheel_base;
  b.low_min_throttle = p.low_min_throttle;
  b.gravity = p.gravity;
  b.gear_sign = p.gear_sign;
  b.clamp_ax = p.clamp_ax;
  b.K_x = p.K_x, b.K_y = p.K_y, b.K_yaw = p.K_yaw, b.K_vel_x = p.K_vel_x;
  b.Q_x_acc = p.Q_x_acc;
  b.Q_y_f = p.Q_y_f;
  b.Q_omega_v = p.Q_omega_v;
  b.Q_omega_steering = p.Q_omega_steering;
  return b;
}

// RacerDubinsImpl::enforceLeash (racer_dubins.cu:177-230): positions are leashed in the body frame of the true state, yaw by
// its shortest angular distance (and re-normalised), every other state component-wise; starts from state_true
template <int S>
inline void racer_enforce_leash(const Eigen::Ref<const Eigen::Matrix<float, S, 1>>& state_true,
                                const Eigen::Ref<const Eigen::Matrix<float, S, 1>>& state_nominal,
                                const Eigen::Ref<const Eigen::Matrix<float, S, 1>>& leash_values,
                                Eigen::Ref<Eigen::Matrix<float, S, 1>> state_output)
{
  typedef RacerDubinsElevationParams::StateIndex SI;
  const int PX = (int)SI::POS_X, PY = (int)SI::POS_Y, YW = (int)SI::YAW;
  auto normalize = [](float a) {  // angle_utils.cuh:20-26
    const float pi = 3.14159265358979323846f;
    const float r = fmodf(a + pi, 2.0f * pi);
    return r <= 0.0f ? r + pi : r - pi;
  };
  for (int i = 0; i < S; i++)
    state_output(i) = state_true(i);
  float dx = state_nominal(PX) - state_true(PX), dy = state_nominal(PY) - state_true(PY);
  const float cy = cosf(state_true(YW)), sy = sinf(state_true(YW));
  float dx_body = dx * cy + dy * sy, dy_body = -dx * sy + dy * cy;
  dx_body = fminf(fmaxf(dx_body, -leash_values(PX)), leash_values(PX));
  dy_body = fminf(fmaxf(dy_body, -leash_values(PY)), leash_values(PY));
  state_output(PX) += dx_body * cy + -dy_body * sy;
  state_output(PY) += dx_body * sy + dy_body * cy;
  for (int i = 0; i < S; i++)
  {
    if (i == PX || i == PY)
      continue;
    const float diff = (i == YW) ? normalize(state_nominal(i) - state_true(i)) : state_nominal(i) - state_true(i);
    if (leash_values(i) < fabsf(diff))
    {
      state_output(i) = state_true(i) + fminf(fmaxf(diff, -leash_values(i)), leash_values(i));
      if (i == YW)
        state_output(i) = normalize(state_output(i));
    }
    else
      state_output(i) = state_nominal(i);
  }
}

class RacerDubinsElevation
  : public MPPI_internal::Dynamics<RacerDubinsElevation, mppib_racer_dubins_elevation_dyn_params,
                                   MPPIB_DYN_RACER_DUBINS_ELEVATION, 19, 2, 28>
{
public:
  typedef RacerDubinsElevationParams DYN_PARAMS_T;
  using PARENT = MPPI_internal::Dynamics<RacerDubinsElevation, mppib_racer_dubins_elevation_dyn_params,
                                         MPPIB_DYN_RACER_DUBINS_ELEVATION, 19, 2, 28>;
  typedef Eigen::Matrix<float, 19, 19> dfdx;
  typedef Eigen::Matrix<float, 19, 2> dfdu;
  // the cost of the small engine a standalone DDPFeedback solves on (ddp.cuh): the in-tree pair of this model
  static const int DDP_COST_ID = MPPIB_COST_RACER_QUADRATIC;

  RacerDubinsElevation(cudaStream_t stream = 0) : PARENT(stream)
  {
  }
  RacerDubinsElevation(DYN_PARAMS_T& params, cudaStream_t stream = 0) : PARENT(stream), params_(params)
  {
  }
  void setParams(const DYN_PARAMS_T& p)
  {
    params_ = p;
  }
  DYN_PARAMS_T getParams() const
  {
    return params_;
  }
  std::string getDynamicsModelName() const override
  {
    return "RACER Dubins Elevation Model";
  }
  void enforceLeash(const Eigen::Ref<const state_array>& state_true, const Eigen::Ref<const state_array>& state_nominal,
                    const Eigen::Ref<const state_array>& leash_values, Eigen::Ref<state_array> state_output) override
  {
    racer_enforce_leash<STATE_DIM>(state_true, state_nominal, leash_values, state_output);
  }
  mppib_racer_dubins_elevation_dyn_params modelBlob() const
  {
    return racer_elevation_blob(params_);
  }
  TwoDTextureHelper<float>* getTextureHelper()
  {
    return tex_helper_.get();
  }
  // ---- engine hooks (controller.hpp) -------------------------------------------------------------------------------
  int pushModelBlobs(mppib_engine* e) const
  {
    if (!tex_helper_->hasData())
      return MPPIB_OK;
    const std::vector<unsigned char>& m = tex_helper_->blob();  // TwoDTextureHelper::copyToDevice
    return mppib_set_blob(e, MPPIB_BLOB_ELEVATION_MAP, m.data(), m.size());
  }
  int hostOutputTrajectory(const float* x0, const float* u, int T, float dt, float* states, float* outputs) const
  {
    auto b = this->blob();
    return mppib_host_output_trajectory_racer_dubins_elevation(&b, tex_helper_->header(), x0, u, T, dt, states, outputs);
  }
  // ---- host methods ------------------------------------------------------------------------------------------------
  // racer_dubins_elevation.cu:229-255 (host step)
  void step(Eigen::Ref<state_array> state, Eigen::Ref<state_array> next_state, Eigen::Ref<state_array> state_der,
            const Eigen::Ref<const control_array>& control, Eigen::Ref<output_array> output, const float /*t*/,
            const float dt)
  {
    float x[19], u[2], xn[19], xd[19], y[28];
    for (int i = 0; i < 19; i++)
      x[i] = state(i);
    u[0] = control(0), u[1] = control(1);
    auto b = this->blob();
    MPPIB_HANDLE(mppib_host_step_racer_dubins_elevation(&b, tex_helper_->header(), x, u, dt, xn, xd, y));
    for (int i = 0; i < 19; i++)
    {
      next_state(i) = xn[i];
      state_der(i) = xd[i];
    }
    for (int i = 0; i < 28; i++)
      output(i) = y[i];
  }
  void computeStateDeriv(const Eigen::Ref<const state_array>& state, const Eigen::Ref<const control_array>& control,
                         Eigen::Ref<state_array> state_der)
  {
    state_array s = state, nx;
    output_array y;
    step(s, nx, state_der, control, y, 0.0f, 0.01f);
  }
  // racer_dubins_elevation.cu:257-334
  bool computeGrad(const Eigen::Ref<const state_array>& state, const Eigen::Ref<const control_array>& control,
                   Eigen::Ref<dfdx> A, Eigen::Ref<dfdu> B)
  {
    float x[19], u[2], a[19 * 19], bb[19 * 2];
    for (int i = 0; i < 19; i++)
      x[i] = state(i);
    u[0] = control(0), u[1] = control(1);
    auto b = this->blob();
    MPPIB_HANDLE(mppib_host_grad_racer_dubins_elevation(&b, x, u, a, bb));
    for (int r = 0; r < 19; r++)
    {
      for (int c = 0; c < 19; c++)
        A(r, c) = a[r * 19 + c];
      for (int c = 0; c < 2; c++)
        B(r, c) = bb[r * 2 + c];
    }
    return true;
  }

private:
  DYN_PARAMS_T params_;
  std::shared_ptr<TwoDTextureHelper<float>> tex_helper_ = std::make_shared<TwoDTextureHelper<float>>(1);
};
