// RacerSuspension (the rigid-body RACER vehicle) through the C++ host layer, written against the reference's include paths
// and compiled with plain g++: VanillaMPPI and ColoredMPPI drive it from rest towards 5 m/s with the host step as the
// plant; Tube-MPPI and RMPPI (without feedback gains) run it for a few steps, keeping it finite and upright.
// `racer_rigid_suspension_example blob` writes the parameter blob (control ranges [-1, 1]), the reference OmegaJacobian
// case's state derivative, omegaJacobian and host step (dt 0.02), and the odometry round-trip errors to stdout as raw
// floats, and needs no device.
// Exit codes: 0 = every check held, 5 = no CUDA device (expected on a CPU-only machine), other = failure.
#include <mppi/controllers/ColoredMPPI/colored_mppi_controller.cuh>
#include <mppi/controllers/MPPI/mppi_controller.cuh>
#include <mppi/controllers/R-MPPI/robust_mppi_controller.cuh>
#include <mppi/controllers/Tube-MPPI/tube_mppi_controller.cuh>
#include <mppi/dynamics/racer_suspension/racer_suspension.cuh>
#include <mppi/sampling_distributions/colored_noise/colored_noise.cuh>
#include <mppi_b200/cost_functions/racer/racer_quadratic_cost.hpp>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>

using DYN = RacerSuspension;
using SI = RacerSuspensionParams::StateIndex;
using OI = RacerSuspensionParams::OutputIndex;
struct NoFeedback
{
};

static void configure(DYN& model)
{
  std::array<float2, 2> rngs = { float2{ -1.0f, 1.0f }, float2{ -1.0f, 1.0f } };
  model.setControlRanges(rngs);
}

static DYN::state_array rest_state(const DYN& model)
{
  DYN::state_array x = DYN::state_array::Zero();
  x((int)SI::ATTITUDE_QW) = 1.0f;
  x((int)SI::P_I_Z) = model.getParams().wheel_radius + model.getParams().cg_pos_wrt_base_link.z;
  return x;
}

// closed loop from rest: the host step is the plant; returns the speed after `steps` control periods (negative: failure)
template <class CTRL>
static float drive(const char* name, CTRL& ctrl, DYN& model, int steps, float dt)
{
  DYN::state_array x = rest_state(model), xn, xd;
  DYN::output_array y;
  float tilt = 0.0f;
  for (int it = 0; it < steps; it++)
  {
    ctrl.computeControl(x, 1);
    DYN::control_array u = ctrl.getControlSeq().col(0);
    model.enforceConstraints(x, u);
    model.step(x, xn, xd, u, y, it, dt);
    x = xn;
    ctrl.slideControlSequence(1);
    for (int i = 0; i < DYN::STATE_DIM; i++)
      if (!std::isfinite(x(i)))
        return -1.0f;
    tilt = fmaxf(tilt, fmaxf(fabsf(y((int)OI::ROLL)), fabsf(y((int)OI::PITCH))));
  }
  const float speed = model.velocityFromState(x)(0);
  printf("%s: speed %.3f m/s after %d steps, y %.3f m, max |roll|, |pitch| %.4f\n", name, speed, steps,
         x((int)SI::P_I_Y), tilt);
  return tilt < 0.05f ? speed : -2.0f;
}

int main(int argc, char** argv)
{
  DYN model;
  configure(model);
  if (argc > 1 && strcmp(argv[1], "blob") == 0)
  {
    auto b = model.blob();
    fwrite(&b, sizeof(b), 1, stdout);
    DYN plain;  // racer_suspension_model_test.cu:108-143
    DYN::state_array x = DYN::state_array::Zero(), xd, xn;
    x((int)SI::ATTITUDE_QW) = 1, x((int)SI::OMEGA_B_X) = 0.1f, x((int)SI::OMEGA_B_Y) = -0.03f;
    x((int)SI::OMEGA_B_Z) = 0.02f, x((int)SI::V_I_X) = 2;
    DYN::control_array u = DYN::control_array::Zero();
    DYN::output_array y;
    Eigen::Matrix3f J;
    plain.computeStateDeriv(x, u, xd, y, &J);
    fwrite(xd.data(), sizeof(float), 14, stdout);
    float j[9];
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++)
        j[r * 3 + c] = J(r, c);
    fwrite(j, sizeof(j), 1, stdout);
    plain.step(x, xn, xd, u, y, 0.0f, 0.02f);
    fwrite(xn.data(), sizeof(float), 14, stdout);
    // odometry round trip: state -> (q, base link position, body velocity, rates) -> state
    DYN::state_array s = rest_state(plain);
    const float yaw = 0.4f;
    s((int)SI::ATTITUDE_QW) = cosf(yaw / 2), s((int)SI::ATTITUDE_QZ) = sinf(yaw / 2);
    s((int)SI::P_I_X) = 3.0f, s((int)SI::V_I_X) = 1.5f, s((int)SI::V_I_Y) = -0.4f, s((int)SI::OMEGA_B_Z) = 0.2f;
    const DYN::state_array back = plain.stateFromOdometry(plain.attitudeFromState(s), plain.positionFromState(s),
                                                          plain.velocityFromState(s), plain.angularRateFromState(s));
    float err[14];
    for (int i = 0; i < 14; i++)
      err[i] = back(i) - s(i);
    fwrite(err, sizeof(err), 1, stdout);
    return 0;
  }
  {  // fail-loudly probe: no device => status -5 from the C-ABI, no fallback
    mppib_engine* probe = nullptr;
    mppib_desc d{};
    d.dynamics_id = MPPIB_DYN_RACER_SUSPENSION;
    d.cost_id = MPPIB_COST_RACER_QUADRATIC;
    d.sampler_id = MPPIB_SAMPLER_GAUSSIAN;
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
  RacerQuadraticCost cost;
  auto cp = cost.getParams();
  cp.desired_speed = 5.0f;
  cost.setParams(cp);
  const int T = 100;
  const float dt = 0.01f;
  int rc = 0;
  try
  {
    {
      using SAMPLER_T = mppi::sampling_distributions::GaussianDistribution<DYN::DYN_PARAMS_T>;
      auto sp = SAMPLER_T::SAMPLING_PARAMS_T();
      sp.std_dev[0] = sp.std_dev[1] = 0.3f;
      SAMPLER_T sampler(sp);
      VanillaMPPIController<DYN, RacerQuadraticCost, NoFeedback, T, 8192> ctrl(&model, &cost, nullptr, &sampler, dt, 1,
                                                                               1.0f, 0.0f);
      if (!(drive("vanilla", ctrl, model, 80, dt) > 1.2f))
        rc = 2;
    }
    {
      using SAMPLER_T = mppi::sampling_distributions::ColoredNoiseDistribution<DYN::DYN_PARAMS_T>;
      auto sp = SAMPLER_T::SAMPLING_PARAMS_T();
      sp.std_dev[0] = sp.std_dev[1] = 0.3f;
      sp.exponents[0] = sp.exponents[1] = 1.0f;
      SAMPLER_T sampler(sp);
      ColoredMPPIController<DYN, RacerQuadraticCost, NoFeedback, T, 8192> ctrl(&model, &cost, nullptr, &sampler, dt, 1,
                                                                               1.0f, 0.0f);
      if (!(drive("colored", ctrl, model, 80, dt) > 1.2f))
        rc = 3;
    }
    {  // Tube-MPPI and RMPPI: two systems per sample
      using SAMPLER_T = mppi::sampling_distributions::GaussianDistribution<DYN::DYN_PARAMS_T>;
      auto sp = SAMPLER_T::SAMPLING_PARAMS_T();
      sp.std_dev[0] = sp.std_dev[1] = sp.std_dev[2] = sp.std_dev[3] = 0.3f;
      SAMPLER_T sampler(sp);
      TubeMPPIController<DYN, RacerQuadraticCost, NoFeedback, T, 4096> tube(&model, &cost, nullptr, &sampler, dt, 1,
                                                                            1.0f, 0.0f);
      if (drive("tube", tube, model, 20, dt) < -0.5f)
        rc = 6;
      RobustMPPIController<DYN, RacerQuadraticCost, NoFeedback, T, 4096> rmppi(&model, &cost, nullptr, &sampler, dt, 1,
                                                                               1.0f, 0.0f, 20.0f);
      if (drive("rmppi", rmppi, model, 20, dt) < -0.5f)
        rc = 7;
    }
  }
  catch (const std::exception& e)
  {
    printf("exception: %s\n", e.what());
    return std::string(e.what()).find("no CUDA device") != std::string::npos ? 5 : 4;
  }
  printf("racer rigid suspension example rc %d\n", rc);
  return rc;
}
