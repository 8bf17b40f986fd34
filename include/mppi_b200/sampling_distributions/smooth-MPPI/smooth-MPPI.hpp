/*
 * SmoothMPPIDistribution — host side of include/mppi/sampling_distributions/smooth-MPPI/smooth-MPPI.cuh (the Gaussian
 * parameters plus the sampler's own integration step dt). generateSamples (smooth-MPPI.cu:126-202: the rate-mean shift,
 * the Gaussian rate rewrite, integrateNoise) runs inside the engine's rollout kernel, and
 * updateDistributionParamsFromDevice (:204-240) inside its merge, which keeps the rate mean on the device from solve to
 * solve (mppib_get_derivative_mean / mppib_set_derivative_mean). One rank, one distribution.
 */
#pragma once
#include <string>

#include "../gaussian/gaussian.hpp"

namespace mppi
{
namespace sampling_distributions
{
template <int C_DIM, int MAX_DISTRIBUTIONS_T = 2>
struct SmoothMPPIParamsImpl : public GaussianParamsImpl<C_DIM, MAX_DISTRIBUTIONS_T>
{
  float dt = 0.015f;
  dim3 shift_trajectory_block;  // kept for API parity; the engine does not launch the shift kernel
  SmoothMPPIParamsImpl(int num_rollouts = 1, int num_timesteps = 1, int num_distributions = 1)
    : GaussianParamsImpl<C_DIM, MAX_DISTRIBUTIONS_T>(num_rollouts, num_timesteps, num_distributions)
  {
  }
};

template <int C_DIM>
using SmoothMPPIParams = SmoothMPPIParamsImpl<C_DIM, 2>;

template <class DYN_PARAMS_T, int C_DIM>
class SmoothMPPIDistributionImpl : public GaussianDistributionImpl<DYN_PARAMS_T, C_DIM>
{
public:
  typedef GaussianDistributionImpl<DYN_PARAMS_T, C_DIM> PARENT_CLASS;
  typedef SmoothMPPIParams<C_DIM> SAMPLING_PARAMS_T;
  static const int SAMPLER_ID = MPPIB_SAMPLER_SMOOTH_MPPI;
  SmoothMPPIDistributionImpl(cudaStream_t stream = 0) : PARENT_CLASS(stream)
  {
  }
  SmoothMPPIDistributionImpl(const SAMPLING_PARAMS_T& params, cudaStream_t stream = 0)
    : PARENT_CLASS(params, stream), dt_(params.dt)
  {
  }
  void setParams(const SAMPLING_PARAMS_T& params, bool synchronize = true)
  {
    PARENT_CLASS::setParams(params, synchronize);
    dt_ = params.dt;
  }
  SAMPLING_PARAMS_T getParams() const
  {
    SAMPLING_PARAMS_T p;
    static_cast<typename PARENT_CLASS::SAMPLING_PARAMS_T&>(p) = this->params_;
    p.dt = dt_;
    return p;
  }
  std::string getSamplingDistributionName() const
  {  // smooth-MPPI.cuh
    return "Smooth-MPPI";
  }
  mppib_smooth_mppi_params blob() const
  {
    mppib_smooth_mppi_params b{};
    b.gaussian = PARENT_CLASS::blob();
    b.dt = dt_;
    return b;
  }

protected:
  float dt_ = 0.015f;
};

template <class DYN_PARAMS_T>
using SmoothMPPIDistribution =
    SmoothMPPIDistributionImpl<DYN_PARAMS_T, (int)DYN_PARAMS_T::ControlIndex::NUM_CONTROLS>;
}  // namespace sampling_distributions
}  // namespace mppi
