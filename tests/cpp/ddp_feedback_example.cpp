// DDP feedback through the C++ host layer, written like the reference's examples/double_integrator_CORL2020.cu and
// tests/feedback_controllers/ddp_test.cu: DDPParams set with .diagonal() <<, Tube-MPPI with initFeedback /
// computeFeedback / getFeedbackControl on the circular track under a large disturbance, RMPPI recomputing its gains in
// updateImportanceSamplingControl, and a standalone DDPFeedback.
// Exit codes: 0 = every check held, 5 = no CUDA device (expected on a CPU-only machine), other = failure.
#include <mppi/controllers/R-MPPI/robust_mppi_controller.cuh>
#include <mppi/feedback_controllers/DDP/ddp.cuh>
#include <mppi_b200/controllers/Tube-MPPI/tube_mppi_controller.hpp>
#include <mppi_b200/cost_functions/double_integrator/double_integrator_circle_cost.hpp>
#include <mppi_b200/dynamics/double_integrator/di_dynamics.hpp>

#include <cmath>
#include <cstdio>
#include <random>

using DI = DoubleIntegratorDynamics;
using SAMPLER_T = mppi::sampling_distributions::GaussianDistribution<DI::DYN_PARAMS_T>;
const int T = 50;
using FB_T = DDPFeedback<DI, T>;

static bool off_track(const DI::state_array& x)
{  // tests/controllers/tube_mppi_test.cu:10-23
  const float r2 = x(0) * x(0) + x(1) * x(1);
  return r2 < 1.675f * 1.675f || r2 > 2.325f * 2.325f;
}

int main()
{
  {  // no device => status -5 from the C ABI, no fallback
    mppib_engine* probe = nullptr;
    mppib_desc d{};
    d.dynamics_id = MPPIB_DYN_DOUBLE_INTEGRATOR;
    d.cost_id = MPPIB_COST_DI_CIRCLE;
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
  const float dt = 0.02f;
  DDPParams<DI> fb_params;  // examples/double_integrator_CORL2020.cu weights
  fb_params.Q.diagonal() << 500, 500, 100, 100;
  fb_params.Q_f = fb_params.Q;
  fb_params.R = DDPParams<DI>::ControlCostWeight::Identity();
  int rc = 0;

  {  // Tube-MPPI: the applied control is the nominal first control plus the DDP feedback
    DI model(1.0f);
    DoubleIntegratorCircleCost cost;
    SAMPLER_T sampler;
    auto sp = sampler.getParams();
    sp.control_cost_coeff[0] = sp.control_cost_coeff[1] = 1.0f;
    sampler.setParams(sp);
    FB_T fb(&model, dt);
    TubeMPPIController<DI, DoubleIntegratorCircleCost, FB_T, T, 1024> tube(&model, &cost, &fb, &sampler, dt, 3, 4.0f, 0.0f);
    tube.setFeedbackParams(fb_params);
    tube.initFeedback();
    DI::state_array x;
    x << 2, 0, 0, 1;
    std::mt19937 gen(0);
    std::normal_distribution<float> n01(0.0f, 1.0f);
    float max_fb = 0.0f;
    for (int t = 0; t < 200; t++)
    {
      if (off_track(x))
      {
        printf("tube: left the track at step %d\n", t);
        rc = 2;
        break;
      }
      tube.computeControl(x, 1);
      tube.computeFeedback(x);
      DI::state_array x_nom = tube.getTargetStateSeq().col(0);
      DI::control_array u_fb = tube.getFeedbackControl(x, x_nom, 0);
      DI::control_array u = tube.getControlSeq().col(0);
      for (int i = 0; i < 2; i++)
      {
        u(i) += u_fb(i);
        max_fb = fmaxf(max_fb, fabsf(u_fb(i)));
      }
      DI::state_array xn, xd;
      DI::output_array y;
      model.step(x, xn, xd, u, y, t, dt);
      x = xn;
      x(2) += 10.0f * dt * n01(gen);  // system variance 100
      x(3) += 10.0f * dt * n01(gen);
      tube.slideControlSequence(1);
    }
    printf("tube: radius after 200 steps %f, largest feedback %f\n", sqrtf(x(0) * x(0) + x(1) * x(1)), max_fb);
    if (!(max_fb > 0.0f) || !tube.getFeedbackEnabled())
      rc = 3;
  }
  {  // RMPPI: initFeedback, then every updateImportanceSamplingControl recomputes the gains on the device
    DI model(1.0f);
    DoubleIntegratorCircleCost cost;
    SAMPLER_T sampler;
    FB_T fb(&model, dt);
    using RMPPI = RobustMPPIController<DI, DoubleIntegratorCircleCost, FB_T, T, 2048>;
    RMPPI rmppi(&model, &cost, &fb, &sampler, dt, 1, 2.0f, 0.0f, 20.0f);
    rmppi.setFeedbackParams(fb_params);
    rmppi.initFeedback();
    DI::state_array x;
    x << 2, 0, 0, 1;
    std::mt19937 gen(1);
    std::normal_distribution<float> n01(0.0f, 1.0f);
    float rmin = 10.0f, rmax = 0.0f;
    for (int t = 0; t < 80; t++)
    {
      rmppi.updateImportanceSamplingControl(x, 1);
      rmppi.computeControl(x, 1);
      DI::state_array x_nom = rmppi.getNominalStateSeq().col(0);
      DI::control_array u = rmppi.getNominalControlSeq().col(0), u_fb = rmppi.getFeedbackControl(x, x_nom, 0);
      for (int i = 0; i < 2; i++)
        u(i) += u_fb(i);
      DI::state_array xn, xd;
      DI::output_array y;
      model.step(x, xn, xd, u, y, t, dt);
      x = xn;
      x(2) += 0.2f * sqrtf(dt) * n01(gen);
      x(3) += 0.2f * sqrtf(dt) * n01(gen);
      const float r = sqrtf(x(0) * x(0) + x(1) * x(1));
      if (t >= 20)
      {
        rmin = fminf(rmin, r);
        rmax = fmaxf(rmax, r);
      }
    }
    const auto K0 = fb.getFeedbackGainsEigen()[0];
    printf("rmppi: radius in [%f, %f] after step 20, K_0(0,0) %f\n", rmin, rmax, K0(0, 0));
    if (!(rmin > 1.6f && rmax < 2.4f) || K0(0, 0) == 0.0f)
      rc = 4;
  }
  {  // standalone DDPFeedback (its own engine): the solve tracks a reachable straight-line trajectory
    DI model(1.0f);
    FB_T fb(&model, dt);
    DDPParams<DI> p;
    p.Q.diagonal() << 100, 100, 10, 10;
    p.Q_f = p.Q;
    p.num_iterations = 3;
    fb.setParams(p);
    fb.initTrackingController();
    FB_T::state_trajectory goal = FB_T::state_trajectory::Zero();
    FB_T::control_trajectory u = FB_T::control_trajectory::Zero();
    for (int t = 0; t < T; t++)
    {
      goal(0, t) = 1.0f * t * dt;
      goal(2, t) = 1.0f;
    }
    DI::state_array x0 = DI::state_array::Zero();
    x0(1) = 0.1f;
    fb.computeFeedback(x0, goal, u);
    const float err = fabsf(fb.result_.state_trajectory(1, T - 1) - goal(1, T - 1));
    printf("standalone: final y error %f (start 0.1)\n", err);
    if (!(err < 0.1f))
      rc = 6;
  }
  printf("ddp example rc %d\n", rc);
  return rc;
}
