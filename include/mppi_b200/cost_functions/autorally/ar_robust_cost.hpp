/* ARRobustCost — include/mppi/cost_functions/autorally/ar_robust_cost.cuh:6-67. The map handling is ARStandardCost's
 * (MPPI_internal::ARMapCost: setTrackData, loadTrackData, updateTransform, costmap()); the rollouts run the device body in
 * libmppi_b200.so (csrc/plugins/costs.cuh), the host methods below the reference's host branch (host_twins.h). */
#pragma once
#include <cmath>
#include <utility>

#include "ar_standard_cost.hpp"

struct ARRobustCostParams : public ARStandardCostParams
{
  float heading_coeff = 0.0;
  ARRobustCostParams()
  {  // ar_robust_cost.cuh:11-28
    control_cost_coeff[0] = 0.0;
    control_cost_coeff[1] = 0.0;
    desired_speed = -1;
    max_slip_ang = 1.5;
    track_coeff = 33.0;
    slip_coeff = 0.0;
    speed_coeff = 20.0;
    crash_coeff = 125000;
    boundary_threshold = 0.75;
    track_slop = 0;
  }
};

class ARRobustCost
  : public MPPI_internal::ARMapCost<ARRobustCost, ARRobustCostParams, mppib_ar_robust_cost_params, MPPIB_COST_AR_ROBUST>
{
public:
  using PARENT_CLASS =
      MPPI_internal::ARMapCost<ARRobustCost, ARRobustCostParams, mppib_ar_robust_cost_params, MPPIB_COST_AR_ROBUST>;
  ARRobustCost(cudaStream_t stream = 0)
  {
  }
  std::string getCostFunctionName() const override
  {
    return "AutoRally robust cost function";
  }
  mppib_ar_robust_cost_params blob() const
  {
    mppib_ar_robust_cost_params b = PARENT_CLASS::blob();
    b.heading_coeff = params_.heading_coeff;
    return b;
  }
  // ar_robust_cost.cu:13-38
  float getStabilizingCost(const float* s) const
  {
    const mppib_ar_robust_cost_params b = blob();
    float c = 0.0f;
    mppib_host_ar_robust_stabilizing_cost(&b, s, &c);
    return c;
  }
  // ar_robust_cost.cu:40-117, host branch (nearest texel of the CPU copy of the map); NaN without a map
  float getCostmapCost(const float* s) const
  {
    const mppib_ar_robust_cost_params b = blob();
    float c = NAN;
    mppib_host_ar_robust_costmap_cost(&b, costmap(), s, &c);
    return c;
  }
  // ar_robust_cost.cu:119-139: stabilizing + costmap cost, MAX_COST_VALUE on overflow or NaN. Takes the output vector as a
  // pointer or as anything with data() (the Eigen output_array of the reference's signature).
  float computeStateCost(const float* y, int timestep = 0, int* crash_status = nullptr) const
  {
    const mppib_ar_robust_cost_params b = blob();
    float c = NAN;
    mppib_host_state_cost(MPPIB_COST_AR_ROBUST, &b, costmap(), y, timestep, crash_status, &c);
    return c;
  }
  template <class V, class = decltype(std::declval<const V&>().data())>
  float computeStateCost(const V& y, int timestep = 0, int* crash_status = nullptr) const
  {
    return computeStateCost(static_cast<const float*>(y.data()), timestep, crash_status);
  }
  template <class V>
  float terminalCost(const V&) const
  {
    return 0.0f;
  }
};
