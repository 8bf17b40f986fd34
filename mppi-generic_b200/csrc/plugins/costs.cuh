/*
 * plugins/costs.cuh — device twins of the reference's Cost plugins (include/mppi/cost_functions/cost.cuh:34-35 contract:
 * initializeCosts, computeStateCost, computeControlCost (== 0, cost.cuh:205-208), computeRunningCost, terminalCost).
 * One thread owns one sample, so `crash_status` is a thread-private int that is sticky across the horizon exactly as
 * in the reference's single-kernel path (SURVEY.md Appendix B.2; mppi_common.cu:77-78).
 */
#pragma once
#include "../device_utils.cuh"
#include "../../../include/mppi_b200/params.h"
#include "texture_map.cuh"

namespace mppib
{
namespace plugins
{
template <class CLASS_T, class PARAMS_T>
struct Cost
{
  using Params = PARAMS_T;
  struct Aux
  {
  };
  // per-block shared scratch ("theta_c" in the reference, cost.cuh:186-189) as a function of the horizon
  __host__ __device__ static constexpr int sharedFloats(int /*T*/)
  {
    return 0;
  }
  // block-cooperative setup of theta_c (Cost::initializeCosts, cost.cuh:186-189)
  __device__ static __forceinline__ void initializeCosts(const Params&, const Aux&, float* /*theta_c*/, int /*T*/)
  {
  }
  __device__ static __forceinline__ float computeControlCost(const Params&, const float* /*u*/, int /*t*/)
  {
    return 0.0f;  // cost.cuh:205-208
  }
  // cost.cu:40-53
  template <class AUX>
  __device__ static __forceinline__ float computeRunningCost(const Params& p, const AUX& aux, const float* theta_c,
                                                             const float* y, const float* u, int t, int* crash)
  {
    return CLASS_T::computeStateCost(p, aux, theta_c, y, t, crash) + CLASS_T::computeControlCost(p, u, t);
  }
};

// powf(discount, t) is the same number for every sample of a block: it is evaluated once per time step into theta_c
// (identical function, identical arguments => identical bits to the reference's per-sample powf call).
template <class PARAMS_T>
__device__ __forceinline__ void fill_discount_table(const PARAMS_T& p, float* theta_c, int T)
{
  for (int t = threadIdx.x; t < T; t += blockDim.x)
    theta_c[t] = powf(p.discount, t);
}

// cost_functions/cartpole/cartpole_quadratic_cost.cu:20-43
struct CartpoleQuadraticCost : public Cost<CartpoleQuadraticCost, mppib_cartpole_cost_params>
{
  __device__ static __forceinline__ float computeStateCost(const Params& params_, const Aux&, const float*,
                                                           const float* state, int, int*)
  {
    return (state[0] - params_.desired_terminal_state[0]) * (state[0] - params_.desired_terminal_state[0]) *
               params_.cart_position_coeff +
           (state[1] - params_.desired_terminal_state[1]) * (state[1] - params_.desired_terminal_state[1]) *
               params_.cart_velocity_coeff +
           (state[2] - params_.desired_terminal_state[2]) * (state[2] - params_.desired_terminal_state[2]) *
               params_.pole_angle_coeff +
           (state[3] - params_.desired_terminal_state[3]) * (state[3] - params_.desired_terminal_state[3]) *
               params_.pole_angular_velocity_coeff;
  }
  __device__ static __forceinline__ float terminalCost(const Params& params_, const Aux& a, const float* state)
  {
    return computeStateCost(params_, a, nullptr, state, 0, nullptr) * params_.terminal_cost_coeff;
  }
};

// cost_functions/double_integrator/double_integrator_circle_cost.cu:8-32
struct DoubleIntegratorCircleCost : public Cost<DoubleIntegratorCircleCost, mppib_di_circle_cost_params>
{
  __host__ __device__ static constexpr int sharedFloats(int T)
  {
    return T;
  }
  __device__ static __forceinline__ void initializeCosts(const Params& p, const Aux&, float* theta_c, int T)
  {
    fill_discount_table(p, theta_c, T);
  }
  __device__ static __forceinline__ float computeStateCost(const Params& params_, const Aux&, const float* theta_c,
                                                           const float* s, int timestep, int*)
  {
    float radial_position = s[0] * s[0] + s[1] * s[1];
    float current_velocity = sqrtf(s[2] * s[2] + s[3] * s[3]);
    float current_angular_momentum = s[0] * s[3] - s[1] * s[2];
    float cost = 0;
    const float crash = theta_c[timestep] * params_.crash_cost;  // powf(discount, timestep); loaded unconditionally, then selected
    if ((radial_position < params_.inner_path_radius2) || (radial_position > params_.outer_path_radius2))
    {
      cost += crash;
    }
    cost += params_.velocity_cost * fabsf(current_velocity - params_.velocity_desired);
    cost += params_.velocity_cost * fabsf(current_angular_momentum - params_.angular_momentum_desired);
    return cost;
  }
  __device__ static __forceinline__ float terminalCost(const Params&, const Aux&, const float*)
  {
    return 0.0f;
  }
};

// utils/math_utils.h:90-94 (linInterp) and :149-155 (normDistFromCenter), float operands as there
__device__ __forceinline__ float linInterp(const float x, const float x_min, const float x_max, const float y_min,
                                           const float y_max)
{
  return (x - x_min) / (x_max - x_min) * (y_max - y_min) + y_min;
}
__device__ __forceinline__ float normDistFromCenter(const float r, const float r_in, const float r_out)
{
  float r_center = (r_in + r_out) / 2.0f;
  float r_width = (r_out - r_in);
  float dist_from_center = fabsf(r - r_center);
  float norm_dist = dist_from_center / (r_width * 0.5f);
  return norm_dist;
}

// cost_functions/double_integrator/double_integrator_robust_cost.cu:9-39 (device body; terminalCost :76-79 == 0). The
// reference's host body (:41-69) uses other constants (steep boundary 0.75, steep cost 0.1 * crash_cost); it is restated
// in host_twins.cpp, each side keeping its own as the reference does (DESIGN.md §8).
struct DoubleIntegratorRobustCost : public Cost<DoubleIntegratorRobustCost, mppib_di_circle_cost_params>
{
  __device__ static __forceinline__ float computeStateCost(const Params& params_, const Aux&, const float*, const float* s,
                                                           int, int*)
  {
    float radial_position = s[0] * s[0] + s[1] * s[1];
    float current_velocity = sqrtf(s[2] * s[2] + s[3] * s[3]);
    float current_angular_momentum = s[0] * s[3] - s[1] * s[2];
    float cost = 0;
    float normalized_dist_from_center = normDistFromCenter(sqrtf(radial_position), sqrtf(params_.inner_path_radius2),
                                                           sqrtf(params_.outer_path_radius2));
    const float steep_percent_boundary = 0.5f;
    const float steep_cost = 0.5f * params_.crash_cost;  // 0.5 * crash_cost in double: exact, so the same float
    if (normalized_dist_from_center <= steep_percent_boundary)
      cost += linInterp(normalized_dist_from_center, 0, steep_percent_boundary, 0, steep_cost);
    if (normalized_dist_from_center > steep_percent_boundary && normalized_dist_from_center <= 1.0f)
      cost += linInterp(normalized_dist_from_center, steep_percent_boundary, 1, steep_cost, params_.crash_cost);
    if (normalized_dist_from_center > 1.0f)
      cost += params_.crash_cost;
    cost += params_.velocity_cost * powf(current_velocity - params_.velocity_desired, 2);
    cost += params_.velocity_cost * powf(current_angular_momentum - params_.angular_momentum_desired, 2);
    return cost;
  }
  __device__ static __forceinline__ float terminalCost(const Params&, const Aux&, const float*)
  {
    return 0.0f;
  }
};

// cost_functions/autorally/ar_standard_cost.cu:284-413 (device branches)
struct ARStandardCost : public Cost<ARStandardCost, mppib_ar_standard_cost_params>
{
  static constexpr float MAX_COST_VALUE = 1e16f;
  struct Aux
  {
    cudaTextureObject_t costmap_tex;  // float4 texels, point filter, clamp, normalised coords (ar_standard_cost.cu:160-171)
  };
  __host__ __device__ static constexpr int sharedFloats(int T)
  {
    return T;
  }
  __device__ static __forceinline__ void initializeCosts(const Params& p, const Aux&, float* theta_c, int T)
  {
    fill_discount_table(p, theta_c, T);
  }
  // ar_standard_cost.cu:206-243 (device branch). Shared with ARRobustCost: P is either cost's blob, both start with the
  // mppib_ar_standard_cost_params fields (params.h)
  template <class P>
  __device__ static __forceinline__ float4 queryTextureTransformed(const P& p, const Aux& aux, float x, float y)
  {
    float u = p.r_c1[0] * x + p.r_c2[0] * y + p.trs[0];
    float v = p.r_c1[1] * x + p.r_c2[1] * y + p.trs[1];
    // An affine map transform (third row 0 0 1: every track map the reference ships) has w == 1 exactly and u / 1 == u, so
    // the four IEEE divisions of a step (66 SASS instructions) are skipped on a block-uniform test of the parameters;
    // projective transforms keep them.
    if (p.r_c1[2] == 0.0f && p.r_c2[2] == 0.0f && p.trs[2] == 1.0f)
      return tex2D<float4>(aux.costmap_tex, u, v);
    float w = p.r_c1[2] * x + p.r_c2[2] * y + p.trs[2];
    return tex2D<float4>(aux.costmap_tex, u / w, v / w);
  }
  __device__ static __forceinline__ float getSpeedCost(const Params& p, const float* s)
  {
    float cost = 0;
    float error = s[4] - p.desired_speed;
    if (p.l1_cost)
      cost = fabsf(error);
    else
      cost = error * error;
    return (p.speed_coeff * cost);
  }
  __device__ static __forceinline__ float getStabilizingCost(const Params& p, const float* s, int* crash_status)
  {
    float stabilizing_cost = 0;
    // reference compares against the double literal 0.001 (ar_standard_cost.cu:304); float(0.001) is the smallest float
    // above it, so `>=` on floats is the identical predicate
    if (fabsf(s[4]) >= 0.001f)
    {
      float slip = -atanf(s[5] / fabsf(s[4]));
      stabilizing_cost = p.slip_coeff * (slip * slip);  // powf(slip, 2) in the reference: <= 2 ulp apart
      if (fabsf(slip) > p.max_slip_ang)
      {
        stabilizing_cost += p.crash_coeff;
      }
    }
    // fabs(s[3]) > M_PI_2 in double (ar_standard_cost.cu:315); float(pi/2) is the smallest float above pi/2
    if (fabsf(s[3]) >= 1.57079632679489661923f)
    {
      crash_status[0] = 1;
    }
    return stabilizing_cost;
  }
  __device__ static __forceinline__ float getCrashCost(const Params& p, const int* crash)
  {
    return crash[0] > 0 ? p.crash_coeff : 0.0f;
  }
  __device__ static __forceinline__ float getTrackCost(const Params& p, const Aux& aux, const float* s, int* crash)
  {
    float track_cost = 0;
    float sn, cs;
    __sincosf(s[2], &sn, &cs);  // __cosf / __sinf in the reference (ar_standard_cost.cu:342-346)
    float x_front = s[0] + p.front_d * cs;
    float y_front = s[1] + p.front_d * sn;
    float x_back = s[0] + p.back_d * cs;
    float y_back = s[1] + p.back_d * sn;
    float track_cost_front = queryTextureTransformed(p, aux, x_front, y_front).x;
    float track_cost_back = queryTextureTransformed(p, aux, x_back, y_back).x;
    track_cost = (fabsf(track_cost_front) + fabsf(track_cost_back)) / 2.0f;
    if (fabsf(track_cost) < p.track_slop)
      track_cost = 0;
    else
      track_cost = p.track_coeff * track_cost;
    if (track_cost_front >= p.boundary_threshold || track_cost_back >= p.boundary_threshold)
      crash[0] = 1;
    return track_cost;
  }
  __device__ static __forceinline__ float computeStateCost(const Params& p, const Aux& aux, const float* theta_c,
                                                           const float* s, int timestep, int* crash_status)
  {
#ifdef MPPIB_EXP_NO_COST
    return s[4] * s[4];
#endif
#ifdef MPPIB_EXP_NO_TEX
    float track_cost = s[0] + s[1];
#else
    float track_cost = getTrackCost(p, aux, s, crash_status);
#endif
    float speed_cost = getSpeedCost(p, s);
    float stabilizing_cost = getStabilizingCost(p, s, crash_status);
    float crash_cost = theta_c[timestep] * getCrashCost(p, crash_status);  // powf(discount, timestep)
    float cost = speed_cost + crash_cost + track_cost + stabilizing_cost;
    if (cost > MAX_COST_VALUE || isnan(cost))
      cost = MAX_COST_VALUE;
    return cost;
  }
  __device__ static __forceinline__ float terminalCost(const Params&, const Aux&, const float*)
  {
    return 0.0f;
  }
};

// cost_functions/autorally/ar_robust_cost.cu:13-132 (device branches): the Autorally map cost written for RMPPI. Smooth
// penalties replace the sticky crash flag (so `crash_status` is never written and there is no discount table), and a
// heading term follows the map's .w channel. The texels are read through the same texture as ARStandardCost's.
// Mixed-precision operations of the reference are kept: its double literals make the slip threshold, the slip and boundary
// ramps double arithmetic; its float-literal comparisons are restated on floats where that is the identical predicate.
struct ARRobustCost : public Cost<ARRobustCost, mppib_ar_robust_cost_params>
{
  static constexpr float MAX_COST_VALUE = 1e16f;
  using Aux = ARStandardCost::Aux;
  __device__ static __forceinline__ void initializeCosts(const Params&, const Aux&, float*, int)
  {
  }
  // ar_robust_cost.cu:13-38
  __device__ static __forceinline__ float getStabilizingCost(const Params& p, const float* s)
  {
    float penalty_val = 0;
    float slip;
    // fabs(s[4]) < 0.001 in double; float(0.001) is the smallest float above 0.001, so `<` on floats is the same predicate
    if (fabsf(s[4]) < 0.001f)
      slip = 0;
    else
      slip = fabsf(-atanf(s[5] / fabsf(s[4])));
    if ((double)slip >= 0.75 * (double)p.max_slip_ang)
    {
      float slip_val = fminf(1.0f, slip / p.max_slip_ang);
      float alpha = (float)(((double)slip_val - 0.75) / (1.0 - 0.75));
      penalty_val = alpha * p.crash_coeff;
    }
    // fabs(s[3]) >= M_PI_2 in double; float(pi/2) is the smallest float above pi/2
    if (fabsf(s[3]) >= 1.57079632679489661923f)
      penalty_val = p.crash_coeff;
    return p.slip_coeff * slip + penalty_val;
  }
  // ar_robust_cost.cu:40-117 (device branch)
  __device__ static __forceinline__ float getCostmapCost(const Params& p, const Aux& aux, const float* s)
  {
    float cost = 0;
    float sn, cs;
    __sincosf(s[2], &sn, &cs);  // __cosf / __sinf in the reference (ar_robust_cost.cu:47-50)
    float x_front = s[0] + p.front_d * cs;
    float y_front = s[1] + p.front_d * sn;
    float x_back = s[0] + p.back_d * cs;
    float y_back = s[1] + p.back_d * sn;
    const float4 track_params_front = ARStandardCost::queryTextureTransformed(p, aux, x_front, y_front);
    const float4 track_params_back = ARStandardCost::queryTextureTransformed(p, aux, x_back, y_back);
    float constraint_val = fminf(1.0f, fmaxf(track_params_front.x, track_params_back.x));
    if (constraint_val >= p.boundary_threshold)
    {
      // float numerator, double division by (1.0 - boundary_threshold), narrowed on assignment
      float alpha = (float)((double)(constraint_val - p.boundary_threshold) / (1.0 - (double)p.boundary_threshold));
      cost += alpha * p.crash_coeff;
    }
    if (track_params_front.y > p.track_slop)
      cost += p.track_coeff * track_params_front.y;
    if (p.desired_speed == -1)
      cost += p.speed_coeff * fabsf(s[4] - track_params_front.z);
    else
      cost += p.speed_coeff * fabsf(s[4] - p.desired_speed);
    cost += p.heading_coeff * fabsf(sinf(s[2]) + track_params_front.w);  // the accurate sinf, as in the reference
    return cost;
  }
  // ar_robust_cost.cu:119-132
  __device__ static __forceinline__ float computeStateCost(const Params& p, const Aux& aux, const float*, const float* s,
                                                           int, int*)
  {
    float stabilizing_cost = getStabilizingCost(p, s);
    float costmap_cost = getCostmapCost(p, aux, s);
    float cost = stabilizing_cost + costmap_cost;
    if (cost > MAX_COST_VALUE || isnan(cost))
      cost = MAX_COST_VALUE;
    return cost;
  }
  __device__ static __forceinline__ float terminalCost(const Params&, const Aux&, const float*)
  {
    return 0.0f;  // ARStandardCostImpl::terminalCost
  }
};

// Quadratic tracking cost on the RACER output vector (ours, params.h: mppib_racer_quadratic_cost_params; the RACER cost
// classes are not in the reference tree), at the output indices of BASELINK_VEL_B_X, BASELINK_POS_I_Y, YAW and
// STEER_ANGLE of the model it is paired with. One cost id: the pair table picks the layout through the class.
template <int VEL_X, int POS_Y, int YAW, int STEER>
struct RacerQuadraticCostAt : public Cost<RacerQuadraticCostAt<VEL_X, POS_Y, YAW, STEER>, mppib_racer_quadratic_cost_params>
{
  using Params = mppib_racer_quadratic_cost_params;
  using Aux = typename Cost<RacerQuadraticCostAt, Params>::Aux;
  __host__ __device__ static constexpr int sharedFloats(int T)
  {
    return T;
  }
  __device__ static __forceinline__ void initializeCosts(const Params& p, const Aux&, float* theta_c, int T)
  {
    fill_discount_table(p, theta_c, T);
  }
  __device__ static __forceinline__ float computeStateCost(const Params& p, const Aux&, const float* theta_c,
                                                           const float* y, int t, int*)
  {
    const float dv = y[VEL_X] - p.desired_speed;
    const float dyaw = normalizeAngle(y[YAW] - p.desired_yaw);
    const float dy = y[POS_Y] - p.desired_y;
    const float st = y[STEER];
    const float cost =
        p.speed_coeff * dv * dv + p.yaw_coeff * dyaw * dyaw + p.lateral_coeff * dy * dy + p.steer_coeff * st * st;
    return cost * theta_c[t];
  }
  __device__ static __forceinline__ float terminalCost(const Params&, const Aux&, const float*)
  {
    return 0.0f;
  }
};
// the RACER-Dubins output layout, racer_dubins.cuh:35-76 (every RACER model but the rigid body)
struct RacerQuadraticCost : RacerQuadraticCostAt<0, 3, 5, 8>
{
};
// RacerSuspension's output layout, racer_suspension.cuh:36-65
struct RacerRigidQuadraticCost : RacerQuadraticCostAt<0, 4, 6, 9>
{
};

// cost_functions/quadrotor/quadrotor_quadratic_cost.cu:70-132 (device body) with the float-array quaternion helpers of
// utils/math_utils.h:166-211 (QuatInv / QuatMultiply normalised with rsqrtf) and :263-270 (Quat2EulerNWU).
// The reference's NaN guard `sum * (1 - isnan(sum)) + isnan(sum) * MAX_COST_VALUE` evaluates to NaN for a NaN sum
// (NaN * 0), exactly like the unguarded host body, so it is not restated: a NaN cost stays NaN on both sides.
struct QuadrotorQuadraticCost : public Cost<QuadrotorQuadraticCost, mppib_quadrotor_cost_params>
{
  __device__ static __forceinline__ float computeStateCost(const Params& p, const Aux&, const float*, const float* s, int,
                                                           int*)
  {
    float s_diff[13];
#pragma unroll
    for (int i = 0; i < 13; i++)
    {
      const float d = s[i] - p.s_goal[i];
      s_diff[i] = d * d;  // powf(x, 2)
    }
    // QuatSubtract(s + 6, s_goal + 6): q_goal * inverse(q), normalised
    const float* q = s + 6;
    const float* g = p.s_goal + 6;
    const float inv_norm = rsqrtf(MPPIB_SQ(q[0]) + MPPIB_SQ(q[1]) + MPPIB_SQ(q[2]) + MPPIB_SQ(q[3]));
    const float a0 = q[0] * inv_norm, a1 = -q[1] * inv_norm, a2 = -q[2] * inv_norm, a3 = -q[3] * inv_norm;
    float d[4];
    d[0] = g[0] * a0 - g[1] * a1 - g[2] * a2 - g[3] * a3;
    d[1] = g[1] * a0 + g[0] * a1 - g[3] * a2 + g[2] * a3;
    d[2] = g[2] * a0 + g[3] * a1 + g[0] * a2 - g[1] * a3;
    d[3] = g[3] * a0 - g[2] * a1 + g[1] * a2 + g[0] * a3;
    const float dn = rsqrtf(MPPIB_SQ(d[0]) + MPPIB_SQ(d[1]) + MPPIB_SQ(d[2]) + MPPIB_SQ(d[3]));
#pragma unroll
    for (int i = 0; i < 4; i++)
      d[i] *= dn;
    float sum = 0.0f;
#pragma unroll
    for (int i = 0; i < 3; i++)
      s_diff[i] *= p.x_coeff;
#pragma unroll
    for (int i = 3; i < 6; i++)
      s_diff[i] *= p.v_coeff;
    if (!p.use_euler)
    {
#pragma unroll
      for (int i = 6; i < 10; i++)
        s_diff[i] = p.q_coeff * d[i - 6];
    }
    else
    {
#pragma unroll
      for (int i = 6; i < 10; i++)
        s_diff[i] = 0.0f;
      const float r_diff = atan2f(2.0f * d[3] * d[2] + 2.0f * d[0] * d[1],
                                  d[0] * d[0] + d[3] * d[3] - d[2] * d[2] - d[1] * d[1]);
      const float temp = -2.0f * d[0] * d[2] + 2.0f * d[1] * d[3];
      const float p_diff = -asinf(fmaxf(fminf(1.0f, temp), -1.0f));
      const float y_diff = atan2f(2.0f * d[2] * d[1] + 2.0f * d[3] * d[0],
                                  d[0] * d[0] + d[1] * d[1] - d[2] * d[2] - d[3] * d[3]);
      sum += p.roll_coeff * MPPIB_SQ(r_diff);
      sum += p.pitch_coeff * MPPIB_SQ(p_diff);
      sum += p.yaw_coeff * MPPIB_SQ(y_diff);
    }
#pragma unroll
    for (int i = 10; i < 13; i++)
      s_diff[i] *= p.w_coeff;
#pragma unroll
    for (int i = 0; i < 13; i++)
      sum += s_diff[i];
    return sum;
  }
  __device__ static __forceinline__ float terminalCost(const Params& p, const Aux& a, const float* s)
  {
    return p.terminal_cost_coeff * computeStateCost(p, a, nullptr, s, 0, nullptr);
  }
};

// cost_functions/quadrotor/quadrotor_map_cost.cu:92-144 (device body; terminalCost :397-407 == 0) with the float-array
// helpers Quat2EulerNWU / Quat2DCM of utils/math_utils.h:263-283 and angle_utils::shortestAngularDistance. The reference's
// host body (:63-90) is another function: no costmap term, no crash flag, and computeWaypointCost added. It is restated in
// host_twins.cpp, each side keeping its own (DESIGN.md §8). The device printf calls of the gate and map terms are not
// restated. The map is tex_helper_'s map 0 (MPPIB_BLOB_COST_TEXTURE), read through texture_map.cuh.
struct QuadrotorMapCost : public Cost<QuadrotorMapCost, mppib_quadrotor_map_cost_params>
{
  struct Aux
  {
    ElevationMap map;  // hdr.use == 0: no map, the costmap term is 0 (checkTextureUse(0) false)
  };
  __device__ static __forceinline__ void initializeCosts(const Params&, const Aux&, float*, int)
  {
  }
  // :146-152: sqrt of a float sum
  __device__ static __forceinline__ float distToWaypoint(const float* s, const float* w)
  {
    return sqrtf(MPPIB_SQ(s[0] - w[0]) + MPPIB_SQ(s[1] - w[1]) + MPPIB_SQ(s[2] - w[2]));
  }
  // :359-395. Outside [0, 1] of the normalised map adds crash_coeff directly (not through the flag), and the clamped map
  // is still read.
  __device__ static __forceinline__ float computeCostmapCost(const Params& p, const Aux& aux, const float* s)
  {
    float cost = 0;
    if (!aux.map.hdr.use)
      return cost;
    const float2 tc = worldPoseToTexCoord(aux.map.hdr, s[0], s[1], s[2]);
    if (tc.x < 0.0f || tc.x > 1.0f || tc.y < 0.0f || tc.y > 1.0f)
      cost += p.crash_coeff;
    const float track_cost =
        queryTextureBilinear(aux.map, tc.x * (float)aux.map.hdr.width - 0.5f, tc.y * (float)aux.map.hdr.height - 0.5f);
    if (track_cost > p.track_slop)
      cost += p.track_coeff * track_cost;
    if (track_cost > p.track_boundary_cost)
      cost += p.crash_coeff;
    return cost;
  }
  // :264-323. Only the along-gate component from the right corner and the cross product are used; it fires within
  // min_dist_to_gate_side of the gate line, in the bands [-0.5, 0) and (1, 1.5] along it.
  __device__ static __forceinline__ float computeGateSideCost(const Params& p, const float* s)
  {
    float cost = 0;
    const float gx = p.curr_gate_left[0] - p.curr_gate_right[0], gy = p.curr_gate_left[1] - p.curr_gate_right[1];
    const float rx = s[0] - p.curr_gate_right[0], ry = s[1] - p.curr_gate_right[1];
    const float perp_dist = rx * gy - ry * gx;
    const float comp = (rx * gx + ry * gy) / (gx * gx + gy * gy);
    if (fabsf(perp_dist) < p.min_dist_to_gate_side &&
        ((comp < 0.0f && comp >= -0.5f) || (comp > 1.0f && comp <= 1.5f)))
      cost += p.crash_coeff * fabsf(comp);
    return cost;
  }
  // :325-357. The weights and the interpolated height are double operations (the literals 0.001 and 1.0) narrowed to
  // float; the `height_diff < 0` branch of the reference is dead (a square), and +400 is added when the SQUARED height
  // difference exceeds gate_width.
  __device__ static __forceinline__ float computeHeightCost(const Params& p, const float* s)
  {
    float cost = 0;
    const float d1 = sqrtf(MPPIB_SQ(s[0] - p.prev_waypoint[0]) + MPPIB_SQ(s[1] - p.prev_waypoint[1]));
    const float d2 = sqrtf(MPPIB_SQ(s[0] - p.curr_waypoint[0]) + MPPIB_SQ(s[1] - p.curr_waypoint[1]));
    const float w1 = (float)((double)d1 / ((double)(d1 + d2) + 0.001));
    const float w2 = (float)((double)d2 / ((double)(d1 + d2) + 0.001));
    const float interpolated_height =
        (float)((1.0 - (double)w1) * (double)p.prev_waypoint[2] + (1.0 - (double)w2) * (double)p.curr_waypoint[2]);
    const float height_diff = MPPIB_SQ(fabsf(s[2] - interpolated_height));
    cost += p.height_coeff * height_diff;
    if (height_diff > p.gate_width)
      cost += 400;
    return cost;
  }
  // :210-238: the yaw of the world-frame velocity Quat2DCM(q) v against the bearing to the waypoint, outside gate_margin
  __device__ static __forceinline__ float computeHeadingCost(const Params& p, const float* s)
  {
    float cost = 0;
    const float* q = s + 6;
    const float vx = s[3], vy = s[4], vz = s[5];
    const float R00 = MPPIB_SQ(q[0]) + MPPIB_SQ(q[1]) - MPPIB_SQ(q[2]) - MPPIB_SQ(q[3]);
    const float R01 = 2 * (q[1] * q[2] - q[0] * q[3]);
    const float R02 = 2 * (q[1] * q[3] + q[0] * q[2]);
    const float R10 = 2 * (q[1] * q[2] + q[0] * q[3]);
    const float R11 = MPPIB_SQ(q[0]) - MPPIB_SQ(q[1]) + MPPIB_SQ(q[2]) - MPPIB_SQ(q[3]);
    const float R12 = 2 * (q[2] * q[3] - q[0] * q[1]);
    const float yaw = atan2f(R10 * vx + R11 * vy + R12 * vz, R00 * vx + R01 * vy + R02 * vz);
    const float w_heading = atan2f(p.curr_waypoint[1] - s[1], p.curr_waypoint[0] - s[0]);
    if (distToWaypoint(s, p.curr_waypoint) > p.gate_margin)
      cost += p.heading_coeff * powf(fabsf(normalizeAngle(yaw - w_heading)), p.heading_power);
    return cost;
  }
  // :240-252
  __device__ static __forceinline__ float computeSpeedCost(const Params& p, const float* s)
  {
    const float speed = sqrtf(s[3] * s[3] + s[4] * s[4]);
    return p.speed_coeff * MPPIB_SQ(speed - p.desired_speed);
  }
  // :199-208: roll and pitch of Quat2EulerNWU
  __device__ static __forceinline__ float computeStabilizingCost(const Params& p, const float* s)
  {
    float roll, pitch, yaw;
    quat2EulerNWU(s + 6, roll, pitch, yaw);
    return p.attitude_coeff * (MPPIB_SQ(roll) + MPPIB_SQ(pitch));
  }
  // :92-144. computeWaypointCost is evaluated but not added on the device, so it is not computed here. A non-zero gate
  // cost raises the sticky crash flag, which then adds crash_coeff at every later step of the sample.
  __device__ static __forceinline__ float computeStateCost(const Params& p, const Aux& aux, const float*, const float* s,
                                                           int, int* crash_status)
  {
    const float costmap_cost = computeCostmapCost(p, aux, s);
    const float gate_cost = computeGateSideCost(p, s);
    const float height_cost = computeHeightCost(p, s);
    const float heading_cost = computeHeadingCost(p, s);
    const float speed_cost = computeSpeedCost(p, s);
    const float stable_cost = computeStabilizingCost(p, s);
    if (gate_cost != 0)
      *crash_status = 1;
    float cost = costmap_cost + gate_cost + height_cost + heading_cost + speed_cost + stable_cost;
    if (distToWaypoint(s, p.curr_waypoint) < p.gate_margin)
      cost += p.gate_pass_cost;
    cost += *crash_status * p.crash_coeff;
    return cost;
  }
  __device__ static __forceinline__ float terminalCost(const Params&, const Aux&, const float*)
  {
    return 0.0f;
  }
};

}  // namespace plugins
}  // namespace mppib
