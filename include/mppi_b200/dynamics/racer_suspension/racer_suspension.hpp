/*
 * RacerSuspension — host class of include/mppi/dynamics/racer_suspension/racer_suspension.cuh (parameters :8-128, body
 * racer_suspension.cu). S14 C2 O26: the 6-DoF rigid-body RACER vehicle, quaternion attitude and body rates, on four
 * spring-damper wheels with Stribeck side friction. Same constructors as the reference: RacerSuspension(stream),
 * RacerSuspension(params, stream). The ground is the plane z = 0 (the reference's map query is commented out); the texture
 * helper exists for API compatibility and nothing reads its map.
 */
#pragma once
#include <cmath>
#include <memory>
#include <string>

#include "../dynamics.hpp"
#include "../../utils/texture_helpers/two_d_texture_helper.hpp"

struct RacerSuspensionParams
{
  enum class StateIndex : int
  {
    P_I_X = 0, P_I_Y, P_I_Z, ATTITUDE_QW, ATTITUDE_QX, ATTITUDE_QY, ATTITUDE_QZ, V_I_X, V_I_Y, V_I_Z, OMEGA_B_X, OMEGA_B_Y,
    OMEGA_B_Z, STEER_ANGLE, NUM_STATES
  };
  enum class ControlIndex : int { THROTTLE_BRAKE = 0, STEER_CMD, NUM_CONTROLS };
  enum class OutputIndex : int
  {
    BASELINK_VEL_B_X = 0, BASELINK_VEL_B_Y, BASELINK_VEL_B_Z, BASELINK_POS_I_X, BASELINK_POS_I_Y, BASELINK_POS_I_Z, YAW,
    ROLL, PITCH, STEER_ANGLE, STEER_ANGLE_RATE, WHEEL_POS_I_FL_X, WHEEL_POS_I_FL_Y, WHEEL_POS_I_FR_X, WHEEL_POS_I_FR_Y,
    WHEEL_POS_I_RL_X, WHEEL_POS_I_RL_Y, WHEEL_POS_I_RR_X, WHEEL_POS_I_RR_Y, WHEEL_FORCE_B_FL, WHEEL_FORCE_B_FR,
    WHEEL_FORCE_B_RL, WHEEL_FORCE_B_RR, ACCEL_X, ACCEL_Y, OMEGA_Z, NUM_OUTPUTS
  };
  static const int WHEEL_FRONT_LEFT = 0;
  static const int WHEEL_FRONT_RIGHT = 1;
  static const int WHEEL_REAR_LEFT = 2;
  static const int WHEEL_REAR_RIGHT = 3;
  // suspension model
  float wheel_radius = 0.32f;
  float mass = 1447;
  float wheel_base = 2.981f;
  float width = 1.5f;
  float height = 1.5f;
  float gravity = -9.81f;
  float k_s[4] = { 14000, 14000, 14000, 14000 };
  float c_s[4] = { 2000, 2000, 2000, 2000 };
  float l_0[4];
  float3 cg_pos_wrt_base_link;
  float3 wheel_pos_wrt_base_link[4];
  float Jxx, Jyy, Jzz;
  float mu = 0.65f;
  float v_slip = 0.1f;
  // throttle model
  float c_t = 3.0f;
  float c_b = 10.0f;
  float c_v = 0.2f;
  float c_0 = 0;
  // steering model
  float steering_constant = .6f;
  float steer_command_angle_scale = -2.45f;
  int gear_sign = 1;

  RacerSuspensionParams()
  {
    recalcParams();
  }
  // racer_suspension.cuh:113-127: the derived fields, the inertias in double
  void recalcParams()
  {
    cg_pos_wrt_base_link = make_float3(wheel_base / 2, 0, 0.2f);
    for (int i = 0; i < 4; i++)
      l_0[i] = wheel_radius + mass / 4 * (-gravity) / k_s[i];
    wheel_pos_wrt_base_link[0] = make_float3(wheel_base, width / 2, 0);
    wheel_pos_wrt_base_link[1] = make_float3(wheel_base, -width / 2, 0);
    wheel_pos_wrt_base_link[2] = make_float3(0, width / 2, 0);
    wheel_pos_wrt_base_link[3] = make_float3(0, -width / 2, 0);
    Jxx = (float)(1.0 / 12 * mass * (height * height + width * width));
    Jyy = (float)(1.0 / 12 * mass * (height * height + wheel_base * wheel_base));
    Jzz = (float)(1.0 / 12 * mass * (wheel_base * wheel_base + width * width));
  }
};

// the blob: RacerSuspensionParams field for field, float3 as three floats (params.h)
inline mppib_racer_rigid_suspension_dyn_params racer_rigid_suspension_blob(const RacerSuspensionParams& p)
{
  mppib_racer_rigid_suspension_dyn_params b{};
  b.wheel_radius = p.wheel_radius;
  b.mass = p.mass;
  b.wheel_base = p.wheel_base;
  b.width = p.width;
  b.height = p.height;
  b.gravity = p.gravity;
  for (int i = 0; i < 4; i++)
  {
    b.k_s[i] = p.k_s[i];
    b.c_s[i] = p.c_s[i];
    b.l_0[i] = p.l_0[i];
    b.wheel_pos_wrt_base_link[i][0] = p.wheel_pos_wrt_base_link[i].x;
    b.wheel_pos_wrt_base_link[i][1] = p.wheel_pos_wrt_base_link[i].y;
    b.wheel_pos_wrt_base_link[i][2] = p.wheel_pos_wrt_base_link[i].z;
  }
  b.cg_pos_wrt_base_link[0] = p.cg_pos_wrt_base_link.x;
  b.cg_pos_wrt_base_link[1] = p.cg_pos_wrt_base_link.y;
  b.cg_pos_wrt_base_link[2] = p.cg_pos_wrt_base_link.z;
  b.Jxx = p.Jxx, b.Jyy = p.Jyy, b.Jzz = p.Jzz;
  b.mu = p.mu;
  b.v_slip = p.v_slip;
  b.c_t = p.c_t, b.c_b = p.c_b, b.c_v = p.c_v, b.c_0 = p.c_0;
  b.steering_constant = p.steering_constant;
  b.steer_command_angle_scale = p.steer_command_angle_scale;
  b.gear_sign = p.gear_sign;
  return b;
}

class RacerSuspension : public MPPI_internal::Dynamics<RacerSuspension, mppib_racer_rigid_suspension_dyn_params,
                                                       MPPIB_DYN_RACER_SUSPENSION, 14, 2, 26>
{
public:
  typedef RacerSuspensionParams DYN_PARAMS_T;
  using PARENT = MPPI_internal::Dynamics<RacerSuspension, mppib_racer_rigid_suspension_dyn_params,
                                         MPPIB_DYN_RACER_SUSPENSION, 14, 2, 26>;
  typedef RacerSuspensionParams::StateIndex SI;
  static const int TEXTURE_ELEVATION_MAP = 0;

  RacerSuspension(cudaStream_t stream = 0) : PARENT(stream)
  {
  }
  RacerSuspension(DYN_PARAMS_T& params, cudaStream_t stream = 0) : PARENT(stream), params_(params)
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
    return "RACER Suspension Model";
  }
  mppib_racer_rigid_suspension_dyn_params modelBlob() const
  {
    return racer_rigid_suspension_blob(params_);
  }
  TwoDTextureHelper<float>* getTextureHelper()
  {
    return tex_helper_.get();
  }

  // ---- host methods ------------------------------------------------------------------------------------------------
  // racer_suspension.cu:31-45: the body rates by approximate implicit Euler; output = the outputs of `state`
  void step(Eigen::Ref<state_array> state, Eigen::Ref<state_array> next_state, Eigen::Ref<state_array> state_der,
            const Eigen::Ref<const control_array>& control, Eigen::Ref<output_array> output, const float /*t*/,
            const float dt)
  {
    float x[14], u[2], xn[14], xd[14], y[26];
    for (int i = 0; i < 14; i++)
      x[i] = state(i);
    u[0] = control(0), u[1] = control(1);
    auto b = this->blob();
    MPPIB_HANDLE(mppib_host_step_racer_rigid_suspension(&b, x, u, dt, xn, xd, y));
    for (int i = 0; i < 14; i++)
    {
      next_state(i) = xn[i];
      state_der(i) = xd[i];
    }
    for (int i = 0; i < 26; i++)
      output(i) = y[i];
  }
  // :47-53: explicit Euler, then q / |q|
  void updateState(const Eigen::Ref<const state_array>& state, Eigen::Ref<state_array> next_state,
                   Eigen::Ref<state_array> state_der, const float dt)
  {
    for (int i = 0; i < 14; i++)
      next_state(i) = state(i) + state_der(i) * dt;
    const int q0 = (int)SI::ATTITUDE_QW;
    const float n = sqrtf(next_state(q0) * next_state(q0) + next_state(q0 + 1) * next_state(q0 + 1) +
                          next_state(q0 + 2) * next_state(q0 + 2) + next_state(q0 + 3) * next_state(q0 + 3));
    for (int i = 0; i < 4; i++)
      next_state(q0 + i) = next_state(q0 + i) / n;
  }
  // :93-298 on flat ground; omegaJacobian as the reference computes it (:215 as written)
  void computeStateDeriv(const Eigen::Ref<const state_array>& state, const Eigen::Ref<const control_array>& control,
                         Eigen::Ref<state_array> state_der, Eigen::Ref<output_array> output,
                         Eigen::Matrix3f* omegaJacobian = nullptr)
  {
    float x[14], u[2], xd[14], y[26], jac[9];
    for (int i = 0; i < 14; i++)
      x[i] = state(i);
    u[0] = control(0), u[1] = control(1);
    auto b = this->blob();
    MPPIB_HANDLE(mppib_host_state_deriv_racer_rigid_suspension(&b, x, u, xd, y, omegaJacobian ? jac : nullptr));
    for (int i = 0; i < 14; i++)
      state_der(i) = xd[i];
    for (int i = 0; i < 26; i++)
      output(i) = y[i];
    if (omegaJacobian)
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++)
          (*omegaJacobian)(r, c) = jac[r * 3 + c];
  }
  void computeStateDeriv(const Eigen::Ref<const state_array>& state, const Eigen::Ref<const control_array>& control,
                         Eigen::Ref<state_array> state_der)
  {
    output_array y;
    computeStateDeriv(state, control, state_der, y);
  }
  // :389-447: x / y leashed in the body frame of the true state's yaw, the quaternion taken from the true state, every
  // other state component-wise
  void enforceLeash(const Eigen::Ref<const state_array>& state_true, const Eigen::Ref<const state_array>& state_nominal,
                    const Eigen::Ref<const state_array>& leash_values, Eigen::Ref<state_array> state_output) override
  {
    const int PX = (int)SI::P_I_X, PY = (int)SI::P_I_Y, Q0 = (int)SI::ATTITUDE_QW;
    float dx = state_nominal(PX) - state_true(PX), dy = state_nominal(PY) - state_true(PY);
    const float qw = state_true(Q0), qx = state_true(Q0 + 1), qy = state_true(Q0 + 2), qz = state_true(Q0 + 3);
    const float yaw = atan2f(2.0f * qy * qx + 2.0f * qz * qw, qw * qw + qx * qx - qy * qy - qz * qz);
    float dx_body = dx * cosf(yaw) + dy * sinf(yaw);
    float dy_body = -dx * sinf(yaw) + dy * cosf(yaw);
    dx_body = fminf(fmaxf(dx_body, -leash_values(PX)), leash_values(PX));
    dy_body = fminf(fmaxf(dy_body, -leash_values(PY)), leash_values(PY));
    dx = dx_body * cosf(yaw) + -dy_body * sinf(yaw);
    dy = dx_body * sinf(yaw) + dy_body * cosf(yaw);
    state_output(PX) += dx;
    state_output(PY) += dy;
    for (int i = 0; i < STATE_DIM; i++)
    {
      if (i == PX || i == PY || (i >= Q0 && i < Q0 + 4))
        continue;
      const float diff = fabsf(state_nominal(i) - state_true(i));
      if (leash_values(i) < diff)
        state_output(i) =
            state_true(i) + fminf(fmaxf(state_nominal(i) - state_true(i), -leash_values(i)), leash_values(i));
      else
        state_output(i) = state_nominal(i);
    }
  }
  // :339-387
  Eigen::Quaternionf attitudeFromState(const Eigen::Ref<const state_array>& state) const
  {
    const int Q0 = (int)SI::ATTITUDE_QW;
    return Eigen::Quaternionf(state(Q0), state(Q0 + 1), state(Q0 + 2), state(Q0 + 3));
  }
  Eigen::Vector3f positionFromState(const Eigen::Ref<const state_array>& state) const
  {
    const Eigen::Vector3f cg = attitudeFromState(state) * vec(params_.cg_pos_wrt_base_link);
    Eigen::Vector3f p;
    for (int i = 0; i < 3; i++)
      p(i) = state((int)SI::P_I_X + i) - cg(i);
    return p;
  }
  Eigen::Vector3f velocityFromState(const Eigen::Ref<const state_array>& state) const
  {
    Eigen::Vector3f v_I, w;
    for (int i = 0; i < 3; i++)
    {
      v_I(i) = state((int)SI::V_I_X + i);
      w(i) = state((int)SI::OMEGA_B_X + i);
    }
    const Eigen::Vector3f v_B = attitudeFromState(state).conjugate() * v_I;
    const float3 c = params_.cg_pos_wrt_base_link;
    const float pb[3] = { -c.x, -c.y, -c.z };
    Eigen::Vector3f out;
    out(0) = v_B(0) + (w(1) * pb[2] - w(2) * pb[1]);
    out(1) = v_B(1) + (w(2) * pb[0] - w(0) * pb[2]);
    out(2) = v_B(2) + (w(0) * pb[1] - w(1) * pb[0]);
    return out;
  }
  Eigen::Vector3f angularRateFromState(const Eigen::Ref<const state_array>& state) const
  {
    Eigen::Vector3f w;
    for (int i = 0; i < 3; i++)
      w(i) = state((int)SI::OMEGA_B_X + i);
    return w;
  }
  state_array stateFromOdometry(const Eigen::Quaternionf& q_B_to_I, const Eigen::Vector3f& pos_base_link_I,
                                const Eigen::Vector3f& vel_base_link_B, const Eigen::Vector3f& omega_B) const
  {
    state_array s = state_array::Zero();
    const int Q0 = (int)SI::ATTITUDE_QW;
    s(Q0) = q_B_to_I.w(), s(Q0 + 1) = q_B_to_I.x(), s(Q0 + 2) = q_B_to_I.y(), s(Q0 + 3) = q_B_to_I.z();
    const Eigen::Vector3f cg = vec(params_.cg_pos_wrt_base_link);
    const Eigen::Vector3f cg_I = q_B_to_I * cg;
    Eigen::Vector3f v_B;
    v_B(0) = vel_base_link_B(0) + (omega_B(1) * cg(2) - omega_B(2) * cg(1));
    v_B(1) = vel_base_link_B(1) + (omega_B(2) * cg(0) - omega_B(0) * cg(2));
    v_B(2) = vel_base_link_B(2) + (omega_B(0) * cg(1) - omega_B(1) * cg(0));
    const Eigen::Vector3f v_I = q_B_to_I * v_B;
    for (int i = 0; i < 3; i++)
    {
      s((int)SI::OMEGA_B_X + i) = omega_B(i);
      s((int)SI::P_I_X + i) = pos_base_link_I(i) + cg_I(i);
      s((int)SI::V_I_X + i) = v_I(i);
    }
    return s;
  }

private:
  static Eigen::Vector3f vec(const float3& f)
  {
    Eigen::Vector3f v;
    v(0) = f.x, v(1) = f.y, v(2) = f.z;
    return v;
  }
  DYN_PARAMS_T params_;
  std::shared_ptr<TwoDTextureHelper<float>> tex_helper_ = std::make_shared<TwoDTextureHelper<float>>(1);
};
