// The reference's pre-built quadrotor map-cost controller (src/controllers/quadrotor/quadrotor_mppi.cu:7) used through its
// own include path and the instantiation library: compiled with -DMPPIB_USE_INSTANTIATION_LIBRARY and linked against
// libmppi_b200_controllers.so. The quadrotor flies from (0, 0, 2) through a gate at (6, 0, 2) to one at (12, 2, 2.5), over
// a track map whose cost grows with the distance from the course; the waypoint moves on once the first gate is passed.
// Exit codes: 0 = both gates passed with no gate-side hit on the flown states, 5 = no CUDA device, other = failure.
#include <mppi/instantiations/quadrotor_mppi/quadrotor_mppi.cuh>

#include <cmath>
#include <cstdio>

using DYN = QuadrotorDynamics;
using COST = QuadrotorMapCost;
using FB = DDPFeedback<DYN, 100>;
using CTRL = VanillaMPPIController<DYN, COST, FB, 100, 512>;  // a pre-built one
using SAMPLER_T = mppi::sampling_distributions::GaussianDistribution<DYN::DYN_PARAMS_T>;

int main()
{
  {  // no device => status -5 from the C ABI, no fallback
    mppib_engine* probe = nullptr;
    mppib_desc d{};
    d.dynamics_id = MPPIB_DYN_QUADROTOR;
    d.cost_id = MPPIB_COST_QUADROTOR_MAP;
    d.num_rollouts = 64;
    d.num_timesteps = 10;
    d.num_distributions = 1;
    d.world_size = 1;
    if (mppib_create(&probe, &d) == MPPIB_ERR_NO_DEVICE)
    {
      printf("no CUDA device: %s\n", mppib_last_error());
      return 5;
    }
    mppib_destroy(probe);
  }
  DYN model;
  std::array<float2, 4> rngs = { float2{ -3.0f, 3.0f }, float2{ -3.0f, 3.0f }, float2{ -3.0f, 3.0f }, float2{ 0.0f, 36.0f } };
  model.setControlRanges(rngs);
  COST cost;
  auto cp = cost.getParams();
  cp.desired_speed = 3.0f;
  cp.dist_to_waypoint_coeff = 1.0f;
  cost.setParams(cp);
  const float gates[2][4] = { { 6.0f, 0.0f, 2.0f, (float)M_PI_2 }, { 12.0f, 2.0f, 2.5f, (float)M_PI_2 - 0.3f } };
  cost.updateWaypoint(0.0f, 0.0f, 2.0f, 0.0f);
  cost.updateWaypoint(float4{ gates[0][0], gates[0][1], gates[0][2], gates[0][3] });
  // track map: 0.5 per metre of distance from the line y = x / 6 (x in [-4, 24], y in [-8, 11], 0.25 m cells)
  const int W = 112, Hh = 76;
  std::vector<float> values(W * Hh);
  for (int i = 0; i < Hh; i++)
    for (int j = 0; j < W; j++)
    {
      const float x = -4.0f + (j + 0.5f) * 0.25f, y = -8.0f + (i + 0.5f) * 0.25f;
      values[i * W + j] = 0.5f * fabsf(y - x / 6.0f) / sqrtf(1.0f + 1.0f / 36.0f);
    }
  cudaExtent ext = make_cudaExtent(W, Hh, 0);
  cost.tex_helper_->setExtent(0, ext);
  cost.tex_helper_->updateTexture(0, values);
  cost.tex_helper_->updateOrigin(0, make_float3(-4.0f, -8.0f, 0.0f));
  cost.tex_helper_->updateResolution(0, 0.25f);
  cost.tex_helper_->enableTexture(0);

  auto sp = SAMPLER_T::SAMPLING_PARAMS_T();
  const float sd[4] = { 0.5f, 0.5f, 0.5f, 2.0f };
  const float cc[4] = { 0.1f, 0.1f, 0.1f, 0.01f };
  for (int i = 0; i < 4; i++)
  {
    sp.std_dev[i] = sd[i];
    sp.control_cost_coeff[i] = cc[i];
  }
  SAMPLER_T sampler(sp);
  FB fb(&model, 0.02f);
  const float dt = 0.02f;
  CTRL::control_trajectory init = CTRL::control_trajectory::Zero();
  for (int t = 0; t < 100; t++)
    init(3, t) = model.zero_control_[3];
  try
  {
    CTRL ctrl(&model, &cost, &fb, &sampler, dt, 1, 1.0f, 0.0f, 100, init);
    DYN::state_array x = model.getZeroState(), xn, xd;
    x[2] = 2.0f;
    DYN::output_array y;
    const int pushes0 = cost.paramsPushes();
    cost.updateWaypoint(float4{ gates[0][0], gates[0][1], gates[0][2], gates[0][3] });  // unchanged: no push
    if (cost.paramsPushes() != pushes0)
    {
      printf("an unchanged waypoint was pushed\n");
      return 3;
    }
    int gate = 0, hits = 0;
    for (int it = 0; it < 700 && gate < 2; it++)
    {
      ctrl.computeControl(x, 1);
      DYN::control_array u = ctrl.getControlSeq().col(0);
      model.enforceConstraints(x, u);
      model.step(x, xn, xd, u, y, it, dt);
      x = xn;
      ctrl.slideControlSequence(1);
      hits += cost.computeGateSideCost(x.data()) != 0.0f;
      if (it % 100 == 0)
        printf("step %d: (%.2f, %.2f, %.2f)\n", it, x[0], x[1], x[2]);
      // passed when the flight crosses the gate's plane (gate line + vertical)
      const float nx = -sinf(gates[gate][3]), ny = cosf(gates[gate][3]);
      if ((x[0] - gates[gate][0]) * nx + (x[1] - gates[gate][1]) * ny < 0.0f)
      {
        printf("gate %d passed at step %d: (%.2f, %.2f, %.2f)\n", gate, it, x[0], x[1], x[2]);
        if (++gate < 2)
          cost.updateWaypoint(gates[gate][0], gates[gate][1], gates[gate][2], gates[gate][3]);
      }
    }
    printf("gates passed %d, gate-side hits %d, parameter pushes %d\n", gate, hits, cost.paramsPushes());
    return (gate == 2 && hits == 0 && cost.paramsPushes() == pushes0 + 1) ? 0 : 1;
  }
  catch (const std::exception& e)
  {
    printf("exception: %s\n", e.what());
    return 2;
  }
}
