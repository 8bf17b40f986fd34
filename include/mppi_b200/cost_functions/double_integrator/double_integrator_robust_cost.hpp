/* DoubleIntegratorRobustCost — include/mppi/cost_functions/double_integrator/double_integrator_robust_cost.cuh:6-28: the
 * circle track's parameters (DoubleIntegratorCircleCostParams, the same blob) with ramps instead of the crash step. The
 * rollouts run the reference's device body (steep boundary 0.5, steep cost 0.5 * crash_cost: csrc/plugins/costs.cuh); the
 * host computeStateCost below is its host body (0.75, 0.1 * crash_cost: host_twins.h), as in the reference. */
#pragma once
#include <cmath>
#include <utility>

#include "double_integrator_circle_cost.hpp"

class DoubleIntegratorRobustCost
  : public MPPI_internal::Cost<DoubleIntegratorRobustCost, DoubleIntegratorCircleCostParams, mppib_di_circle_cost_params,
                               MPPIB_COST_DI_ROBUST>
{
public:
  DoubleIntegratorRobustCost(cudaStream_t stream = nullptr)
  {
  }
  std::string getCostFunctionName() const override
  {
    return "Double integrator robust cost";
  }
  mppib_di_circle_cost_params blob() const
  {
    mppib_di_circle_cost_params b{};
    fillBase(b);
    b.velocity_cost = params_.velocity_cost;
    b.crash_cost = params_.crash_cost;
    b.velocity_desired = params_.velocity_desired;
    b.inner_path_radius2 = params_.inner_path_radius2;
    b.outer_path_radius2 = params_.outer_path_radius2;
    b.angular_momentum_desired = params_.angular_momentum_desired;
    return b;
  }
  float getLipshitzConstantCost() const
  {
    return params_.crash_cost;
  }
  // double_integrator_robust_cost.cu:41-69 (host body)
  float computeStateCost(const float* s, int timestep = 0, int* crash_status = nullptr) const
  {
    const mppib_di_circle_cost_params b = blob();
    float c = NAN;
    mppib_host_state_cost(MPPIB_COST_DI_ROBUST, &b, nullptr, s, timestep, crash_status, &c);
    return c;
  }
  template <class V, class = decltype(std::declval<const V&>().data())>
  float computeStateCost(const V& s, int timestep = 0, int* crash_status = nullptr) const
  {
    return computeStateCost(static_cast<const float*>(s.data()), timestep, crash_status);
  }
  template <class V>
  float terminalCost(const V&) const
  {
    return 0.0f;  // double_integrator_robust_cost.cu:71-74
  }
};
