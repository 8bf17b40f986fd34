// Host-layer check of the smooth-MPPI sampler: VanillaMPPIController on the cartpole with SmoothMPPIDistribution, included
// through the reference's path and linked to libmppi_b200.so with plain g++.
// Exit codes: 0 = ran and stayed finite, 5 = no CUDA device (expected on a CPU-only box), other = failure.
#include <mppi/sampling_distributions/smooth-MPPI/smooth-MPPI.cuh>
#include <mppi_b200/controllers/MPPI/mppi_controller.hpp>
#include <mppi_b200/cost_functions/cartpole/cartpole_quadratic_cost.hpp>
#include <mppi_b200/dynamics/cartpole/cartpole_dynamics.hpp>

#include <cmath>
#include <cstdio>

using SAMPLER_T = mppi::sampling_distributions::SmoothMPPIDistribution<CartpoleDynamics::DYN_PARAMS_T>;
struct NoFeedback
{
};

int main()
{
  {  // no device => status -5 from the C-ABI, no fallback
    mppib_engine* probe = nullptr;
    mppib_desc d{};
    d.dynamics_id = MPPIB_DYN_CARTPOLE;
    d.cost_id = MPPIB_COST_CARTPOLE_QUADRATIC;
    d.sampler_id = MPPIB_SAMPLER_SMOOTH_MPPI;
    d.num_rollouts = 64;
    d.num_timesteps = 10;
    d.num_distributions = 1;
    d.world_size = 1;
    const int rc = mppib_create(&probe, &d);
    if (rc == MPPIB_ERR_NO_DEVICE)
    {
      printf("no CUDA device: %s\n", mppib_last_error());
      return 5;
    }
    mppib_destroy(probe);
  }
  CartpoleDynamics model(1.0, 1.0, 1.0);
  CartpoleQuadraticCost cost;
  model.control_rngs_->x = -10.0f;
  model.control_rngs_->y = 10.0f;

  const float dt = 0.01f;
  const int num_timesteps = 100;
  auto sampler_params = SAMPLER_T::SAMPLING_PARAMS_T();
  sampler_params.std_dev[0] = 100.0f;  // a rate: a control sample spreads by dt * std_dev = 1.5
  sampler_params.dt = 0.015f;
  SAMPLER_T sampler(sampler_params);
  if (sampler.getSamplingDistributionName() != "Smooth-MPPI" || sampler.getParams().dt != 0.015f)
    return 6;

  VanillaMPPIController<CartpoleDynamics, CartpoleQuadraticCost, NoFeedback, num_timesteps, 2048, SAMPLER_T> controller(
      &model, &cost, nullptr, &sampler, dt, 1, 0.25f, 0.0f);
  auto params = controller.getParams();
  params.seed_ = 42;
  controller.setParams(params);
  if (controller.getFullName() != "Vanilla MPPI(Cartpole, Cartpole quadratic cost, Smooth-MPPI)")
  {
    printf("getFullName: %s\n", controller.getFullName().c_str());
    return 7;
  }

  CartpoleDynamics::state_array x = CartpoleDynamics::state_array::Zero(), xn, xdot;
  CartpoleDynamics::output_array y;
  for (int i = 0; i < 200; ++i)
  {
    controller.computeControl(x, 1);
    CartpoleDynamics::control_array u = controller.getControlSeq().col(0);
    model.enforceConstraints(x, u);
    model.step(x, xn, xdot, u, y, i, dt);
    x = xn;
    controller.slideControlSequence(1);
  }
  const float baseline = controller.getBaselineCost();
  printf("smooth-MPPI cartpole: baseline %f, state %f %f %f %f\n", baseline, x(0), x(1), x(2), x(3));
  for (int i = 0; i < 4; i++)
    if (!std::isfinite(x(i)))
      return 2;
  return std::isfinite(baseline) ? 0 : 3;
}
