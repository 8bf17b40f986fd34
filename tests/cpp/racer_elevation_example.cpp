// RacerDubinsElevation through the C++ host layer, written against the reference's include paths: Tube-MPPI and RMPPI,
// each with DDPFeedback<RacerDubinsElevation, T> gains, holding 1.4 m/s along +x over a rolling elevation map under a push
// on speed and heading every step, and a standalone DDPFeedback. Compiled with plain g++.
// `racer_elevation_example blob` prints the model's parameter blob (configured as in tests/test_racer_dubins_elevation.py)
// and its host computeGrad at one state, and needs no device.
// Exit codes: 0 = every check held, 5 = no CUDA device (expected on a CPU-only machine), other = failure.
#include <mppi/controllers/R-MPPI/robust_mppi_controller.cuh>
#include <mppi/dynamics/racer_dubins/racer_dubins_elevation.cuh>
#include <mppi/feedback_controllers/DDP/ddp.cuh>
#include <mppi_b200/controllers/Tube-MPPI/tube_mppi_controller.hpp>
#include <mppi_b200/cost_functions/racer/racer_quadratic_cost.hpp>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

using DYN = RacerDubinsElevation;
using SAMPLER_T = mppi::sampling_distributions::GaussianDistribution<DYN::DYN_PARAMS_T>;
const int T = 50;
using FB_T = DDPFeedback<DYN, T>;

static void configure(DYN& model)
{
  auto p = model.getParams();
  p.c_t[1] = 2.75f;
  p.wheel_base = 0.35f;
  model.setParams(p);
  std::array<float2, 2> rngs;
  for (auto& r : rngs)
    r.x = -1.0f, r.y = 1.0f;
  model.setControlRanges(rngs);
}

// workloads.racer_elevation_map(): two sine waves over x in [-10, 90], y in [-30, 30] m, 0.5 m cells (no noise here)
static void add_map(DYN& model)
{
  const int w = 200, h = 120;
  std::vector<float> z((size_t)w * h);
  for (int i = 0; i < h; i++)
    for (int j = 0; j < w; j++)
    {
      const float x = -10.0f + (j + 0.5f) * 0.5f, y = -30.0f + (i + 0.5f) * 0.5f;
      z[(size_t)i * w + j] = 0.4f * sinf(2.0f * 3.14159265f * x / 24.0f) + 0.25f * cosf(2.0f * 3.14159265f * y / 15.0f);
    }
  auto* tex = model.getTextureHelper();
  cudaExtent ext = make_cudaExtent(w, h, 0);
  tex->updateTexture(0, z, ext);
  tex->updateOrigin(0, make_float3(-10.0f, -30.0f, 0.0f));
  tex->updateResolution(0, 0.5f);
  tex->enableTexture(0);
}

static RacerQuadraticCost make_cost()
{
  RacerQuadraticCost cost;
  auto cp = cost.getParams();
  cp.desired_speed = 1.4f;  // above the 0.87 m/s a coasting vehicle holds over the map
  cp.speed_coeff = 20.0f;
  cost.setParams(cp);
  return cost;
}

static DDPParams<DYN> fb_params()
{
  DDPParams<DYN> p;
  p.Q = DDPParams<DYN>::StateCostWeight::Zero();
  const float q[6] = { 20, 30, 5, 5, 1, 0.1f };
  for (int i = 0; i < 6; i++)
    p.Q(i, i) = q[i];
  p.Q_f = p.Q;
  p.R = DDPParams<DYN>::ControlCostWeight::Identity();
  return p;
}

template <bool RMPPI, class CTRL>
static bool run(const char* name, CTRL& ctrl, DYN& model, unsigned seed)
{
  const float dt = 0.02f;
  DYN::state_array x = DYN::state_array::Zero();
  x(0) = 1.0f;
  for (int i = 9; i < 13; i++)
    x(i) = 1e-6f;
  std::mt19937 gen(seed);
  std::normal_distribution<float> n01(0.0f, 1.0f);
  double sum_v = 0.0;
  float max_yaw = 0.0f;
  int n = 0;
  for (int t = 0; t < 150; t++)
  {
    DYN::control_array u;
    if constexpr (RMPPI)
    {
      ctrl.updateImportanceSamplingControl(x, 1);
      ctrl.computeControl(x, 1);
      DYN::state_array x_nom = ctrl.getNominalStateSeq().col(0);
      u = ctrl.getNominalControlSeq().col(0);
      const DYN::control_array fb = ctrl.getFeedbackControl(x, x_nom, 0);
      u(0) += fb(0), u(1) += fb(1);
    }
    else
    {
      ctrl.computeControl(x, 1);
      ctrl.computeFeedback(x);
      DYN::state_array x_nom = ctrl.getTargetStateSeq().col(0);
      u = ctrl.getControlSeq().col(0);
      const DYN::control_array fb = ctrl.getFeedbackControl(x, x_nom, 0);
      u(0) += fb(0), u(1) += fb(1);
    }
    model.enforceConstraints(x, u);
    DYN::state_array xn, xd;
    DYN::output_array y;
    model.step(x, xn, xd, u, y, t, dt);
    x = xn;
    x(0) += 0.3f * sqrtf(dt) * n01(gen);
    x(1) += 0.05f * sqrtf(dt) * n01(gen);
    if (!RMPPI)
      ctrl.slideControlSequence(1);
    if (t >= 50)
    {
      sum_v += x(0);
      max_yaw = fmaxf(max_yaw, fabsf(x(1)));
      n++;
    }
  }
  const float mean_v = (float)(sum_v / n);
  printf("%s: mean speed %f after 1 s, largest |yaw| %f, pitch %f\n", name, mean_v, max_yaw, x(7));
  return fabsf(mean_v - 1.4f) < 0.3f && max_yaw < 0.2f;  // coasting would be 0.53 off
}

int main(int argc, char** argv)
{
  if (argc > 1 && strcmp(argv[1], "blob") == 0)
  {
    DYN model;
    configure(model);
    const auto b = model.blob();
    fwrite(&b, sizeof(b), 1, stdout);
    DYN::state_array x = DYN::state_array::Zero();
    x(0) = 1.5f, x(1) = 0.3f, x(4) = 0.1f, x(7) = 0.05f;
    DYN::control_array u;
    u << 0.4f, 0.1f;
    DYN::dfdx A;
    DYN::dfdu B;
    model.computeGrad(x, u, A, B);
    float buf[19 * 21];
    for (int r = 0; r < 19; r++)
    {
      for (int c = 0; c < 19; c++)
        buf[r * 21 + c] = A(r, c);
      buf[r * 21 + 19] = B(r, 0);
      buf[r * 21 + 20] = B(r, 1);
    }
    fwrite(buf, sizeof(buf), 1, stdout);
    return 0;
  }
  {  // no device => status -5 from the C ABI, no fallback
    mppib_engine* probe = nullptr;
    mppib_desc d{};
    d.dynamics_id = MPPIB_DYN_RACER_DUBINS_ELEVATION;
    d.cost_id = MPPIB_COST_RACER_QUADRATIC;
    d.num_rollouts = 64;
    d.num_timesteps = 10;
    d.num_distributions = 2;
    d.world_size = 1;
    if (mppib_create(&probe, &d) == MPPIB_ERR_NO_DEVICE)
    {
      printf("no CUDA device: %s\n", mppib_last_error());
      return 5;
    }
    mppib_destroy(probe);
  }
  const float dt = 0.02f;
  int rc = 0;
  {
    DYN model;
    configure(model);
    add_map(model);
    RacerQuadraticCost cost = make_cost();
    SAMPLER_T sampler;
    auto sp = sampler.getParams();
    sp.std_dev[0] = sp.std_dev[1] = sp.std_dev[2] = sp.std_dev[3] = 0.3f;
    sampler.setParams(sp);
    FB_T fb(&model, dt);
    TubeMPPIController<DYN, RacerQuadraticCost, FB_T, T, 2048> tube(&model, &cost, &fb, &sampler, dt, 3, 1.0f, 0.0f);
    tube.setFeedbackParams(fb_params());
    tube.initFeedback();
    if (!run<false>("tube", tube, model, 0) || !tube.getFeedbackEnabled())
      rc = 2;
  }
  {
    DYN model;
    configure(model);
    add_map(model);
    RacerQuadraticCost cost = make_cost();
    SAMPLER_T sampler;
    auto sp = sampler.getParams();
    sp.std_dev[0] = sp.std_dev[1] = sp.std_dev[2] = sp.std_dev[3] = 0.3f;
    sampler.setParams(sp);
    FB_T fb(&model, dt);
    RobustMPPIController<DYN, RacerQuadraticCost, FB_T, T, 2048> rmppi(&model, &cost, &fb, &sampler, dt, 1, 1.0f, 0.0f,
                                                                       20.0f);
    rmppi.setFeedbackParams(fb_params());
    rmppi.initFeedback();
    if (!run<true>("rmppi", rmppi, model, 1))
      rc = 3;
    const auto K0 = fb.getFeedbackGainsEigen()[0];
    float kmax = 0.0f;
    for (int c = 0; c < 2; c++)
      for (int i = 0; i < 19; i++)
        kmax = fmaxf(kmax, fabsf(K0(c, i)));
    if (kmax == 0.0f)
      rc = 4;
  }
  {  // standalone DDPFeedback (its own engine): track a straight line at 1.2 m/s from 0.3 m to the side
    DYN model;
    configure(model);
    FB_T fb(&model, dt);
    DDPParams<DYN> p = fb_params();
    p.num_iterations = 5;
    fb.setParams(p);
    fb.initTrackingController();
    FB_T::state_trajectory goal = FB_T::state_trajectory::Zero();
    FB_T::control_trajectory u = FB_T::control_trajectory::Zero();
    for (int t = 0; t < T; t++)
    {
      goal(0, t) = 1.2f;
      goal(2, t) = 1.2f * t * dt;
    }
    DYN::state_array x0 = DYN::state_array::Zero();
    x0(0) = 1.2f;
    x0(3) = 0.3f;
    fb.computeFeedback(x0, goal, u);
    const float err = fabsf(fb.result_.state_trajectory(3, T - 1));
    printf("standalone: final lateral error %f (start 0.3)\n", err);
    if (!(err < 0.3f))
      rc = 6;
  }
  printf("racer elevation example rc %d\n", rc);
  return rc;
}
