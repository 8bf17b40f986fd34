// The seven runs of the reference's RMPPI paper experiment (examples/double_integrator_CORL2020.cu) through the C++ host
// layer: Vanilla MPPI (system noise 1 and 100, circle cost), Vanilla with the robust cost, Tube-MPPI with both costs and
// RMPPI with both costs, all on the circular track under the same seed-7 std::mt19937 disturbance, with DDP feedback
// (Q = diag(500, 500, 100, 100)). The .npy dumps of the original are left out; each run prints its count of tube failures
// (radius outside [1.675, 2.325], the reference's tubeFailure) and of steps whose host robust cost (crash_cost 100) exceeds
// 1000, and RMPPI's computeDF at the last step.
// Exit codes: 0 = both RMPPI runs stayed in the tube, 2 = one did not, 5 = no CUDA device (expected on a CPU-only machine).
// With the argument --probe the binary stops after the device probe (exit code 0 with a device, 5 without).
#include <mppi/controllers/MPPI/mppi_controller.cuh>
#include <mppi/controllers/R-MPPI/robust_mppi_controller.cuh>
#include <mppi/controllers/Tube-MPPI/tube_mppi_controller.cuh>
#include <mppi/cost_functions/double_integrator/double_integrator_circle_cost.cuh>
#include <mppi/cost_functions/double_integrator/double_integrator_robust_cost.cuh>
#include <mppi/dynamics/double_integrator/di_dynamics.cuh>
#include <mppi/feedback_controllers/DDP/ddp.cuh>

#include <cmath>
#include <cstdio>
#include <random>
#include <string>
#include <type_traits>
#include <vector>

using Dyn = DoubleIntegratorDynamics;
using SCost = DoubleIntegratorCircleCost;
using RCost = DoubleIntegratorRobustCost;
const int num_timesteps = 50;
const int total_time_horizon = 5000;
using Feedback = DDPFeedback<Dyn, num_timesteps>;
using Sampler = mppi::sampling_distributions::GaussianDistribution<Dyn::DYN_PARAMS_T>;

const float dt = 0.02;
const int max_iter = 1;
const float lambda = 2;
const float alpha = 0.0;

static bool tubeFailure(const Dyn::state_array& s)
{  // double_integrator_CORL2020.cu:12-24
  const float inner_path_radius2 = 1.675 * 1.675;
  const float outer_path_radius2 = 2.325 * 2.325;
  const float radial_position = s(0) * s(0) + s(1) * s(1);
  return radial_position < inner_path_radius2 || radial_position > outer_path_radius2;
}

struct Counts
{
  int tube_failures = 0;
  int robust_cost_over_1000 = 0;
  float df = 0;
};

enum Kind
{
  VANILLA,
  TUBE,
  RMPPI
};

template <class CTRL, class COST>
static Counts run(CTRL& controller, Dyn& model, const std::vector<float>& noise)
{
  RCost judge;  // the host robust cost every run is scored with (crash_cost 100, as in the robust-cost runs)
  auto jp = judge.getParams();
  jp.crash_cost = 100;
  judge.setParams(jp);
  Counts c;
  Dyn::state_array x;
  x << 2, 0, 0, 1;
  const float noise_scale = sqrtf(model.getParams().system_noise) * dt;
  for (int t = 0; t < total_time_horizon; ++t)
  {
    if (tubeFailure(x))
      c.tube_failures++;
    if (judge.computeStateCost(x, t) > 1000)
      c.robust_cost_over_1000++;
    if constexpr (std::is_same<CTRL, RobustMPPIController<Dyn, COST, Feedback, num_timesteps, 1024, Sampler>>::value)
      controller.updateImportanceSamplingControl(x, 1);
    controller.computeControl(x, 1);
    controller.computeFeedback(x);
    controller.computeFeedbackPropagatedStateSeq();
    if constexpr (std::is_same<CTRL, RobustMPPIController<Dyn, COST, Feedback, num_timesteps, 1024, Sampler>>::value)
      c.df = controller.computeDF();
    auto nominal_trajectory = controller.getTargetStateSeq();
    Dyn::control_array current_control = controller.getControlSeq().col(0);
    Dyn::state_array x_nom = nominal_trajectory.col(0);
    Dyn::control_array fb_control = controller.getFeedbackControl(x, x_nom, 0);
    for (int i = 0; i < Dyn::CONTROL_DIM; i++)
      current_control(i) += fb_control(i);
    Dyn::state_array xn, xd;
    Dyn::output_array y;
    model.step(x, xn, xd, current_control, y, t, dt);
    x = xn;
    if constexpr (std::is_same<CTRL, TubeMPPIController<Dyn, COST, Feedback, num_timesteps, 1024, Sampler>>::value)
      controller.updateNominalState(current_control);
    for (int i = 2; i < 4; i++)  // x += noise.col(t) * sqrt(system_noise) * dt
      x(i) += noise[(size_t)t * 2 + (i - 2)] * noise_scale;
    controller.slideControlSequence(1);
  }
  return c;
}

template <class COST>
static Counts experiment(Kind kind, float system_noise, float crash_cost, const std::vector<float>& noise,
                         float nominal_threshold = 20)
{
  Sampler::SAMPLING_PARAMS_T sampler_params;
  for (int i = 0; i < Dyn::CONTROL_DIM; i++)
    sampler_params.std_dev[i] = 1;
  Dyn model(system_noise);
  COST cost;
  if (crash_cost > 0)
  {
    auto params = cost.getParams();
    params.crash_cost = crash_cost;
    cost.setParams(params);
  }
  Sampler sampler(sampler_params);
  Feedback fb_controller(&model, dt);
  auto fb_params = fb_controller.getParams();
  fb_params.Q.diagonal() << 500, 500, 100, 100;
  fb_controller.setParams(fb_params);
  if (kind == VANILLA)
  {
    VanillaMPPIController<Dyn, COST, Feedback, num_timesteps, 1024, Sampler> controller(
        &model, &cost, &fb_controller, &sampler, dt, max_iter, lambda, alpha);
    controller.initFeedback();
    return run<decltype(controller), COST>(controller, model, noise);
  }
  if (kind == TUBE)
  {
    TubeMPPIController<Dyn, COST, Feedback, num_timesteps, 1024, Sampler> controller(&model, &cost, &fb_controller,
                                                                                     &sampler, dt, max_iter, lambda, alpha);
    controller.setNominalThreshold(nominal_threshold);  // runTube: 20 (:352), runTubeRC: 2 (:444)
    controller.initFeedback();  // on in the reference's Tube constructor; explicit in this layer
    return run<decltype(controller), COST>(controller, model, noise);
  }
  const float value_function_threshold = 20.0;
  RobustMPPIController<Dyn, COST, Feedback, num_timesteps, 1024, Sampler> controller(
      &model, &cost, &fb_controller, &sampler, dt, max_iter, lambda, alpha, value_function_threshold);
  controller.initFeedback();  // on in the reference's RMPPI constructor; explicit in this layer
  return run<decltype(controller), COST>(controller, model, noise);
}

int main(int argc, char** argv)
{
  {  // no device => status -5 from the C ABI, no fallback
    mppib_engine* probe = nullptr;
    mppib_desc d{};
    d.dynamics_id = MPPIB_DYN_DOUBLE_INTEGRATOR;
    d.cost_id = MPPIB_COST_DI_ROBUST;
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
    if (argc > 1 && std::string(argv[1]) == "--probe")
    {
      printf("CUDA device present\n");
      return 0;
    }
  }
  // double_integrator_CORL2020.cu:721-740: the same noise for every run
  std::mt19937 gen;
  gen.seed(7);
  std::normal_distribution<float> normal_distribution(0, 1);
  std::vector<float> noise((size_t)total_time_horizon * 2);
  for (int t = 0; t < total_time_horizon; ++t)
    for (int i = 0; i < 2; ++i)
      noise[(size_t)t * 2 + i] = normal_distribution(gen);

  struct Row
  {
    const char* name;
    Counts c;
  };
  std::vector<Row> rows;
  rows.push_back({ "vanilla", experiment<SCost>(VANILLA, 1, 0, noise) });
  rows.push_back({ "vanilla_large", experiment<SCost>(VANILLA, 100, 0, noise) });
  rows.push_back({ "vanilla_large_rc", experiment<RCost>(VANILLA, 100, 100, noise) });
  rows.push_back({ "tube_sc", experiment<SCost>(TUBE, 100, 0, noise) });
  rows.push_back({ "tube_rc", experiment<RCost>(TUBE, 100, 100, noise, 2) });
  rows.push_back({ "rmppi_sc", experiment<SCost>(RMPPI, 100, 0, noise) });
  rows.push_back({ "rmppi_rc", experiment<RCost>(RMPPI, 100, 100, noise) });
  int rc = 0;
  for (const Row& r : rows)
  {
    printf("run %s: tube_failures %d robust_cost_over_1000 %d df %f\n", r.name, r.c.tube_failures,
           r.c.robust_cost_over_1000, r.c.df);
    if ((r.name[0] == 'r') && r.c.tube_failures > 0)
      rc = 2;
  }
  printf("corl2020 rc %d\n", rc);
  return rc;
}
