// RacerDubinsElevationSuspension through the C++ host layer, written against the reference's include paths: VanillaMPPI
// holding 1.2 m/s over a hill with its elevation and normals maps, then the model's host step. Compiled with plain g++.
// `racer_suspension_example blob` writes the model's parameter blob, one host step (next state, state derivative,
// output) and one normals query to stdout as raw floats, and needs no device.
// Exit codes: 0 = every check held, 5 = no CUDA device (expected on a CPU-only machine), other = failure.
#include <mppi/controllers/MPPI/mppi_controller.cuh>
#include <mppi/dynamics/racer_dubins/racer_dubins_elevation_suspension_lstm.cuh>
#include <mppi_b200/cost_functions/racer/racer_quadratic_cost.hpp>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

using DYN = RacerDubinsElevationSuspension;
struct NoFeedback
{
};

// one hill, z = 0.4 exp(-((x - 8)^2 + (y - 1)^2) / 50), over x in [-10, 50], y in [-15, 15] m at 0.5 m; normals
// (-dz/dx, -dz/dy, 1) normalised, from the analytic gradient
static float hill(float x, float y)
{
  return 0.4f * expf(-((x - 8.0f) * (x - 8.0f) + (y - 1.0f) * (y - 1.0f)) / 50.0f);
}

static void configure(DYN& model)
{
  auto p = model.getParams();
  p.spring_k = 15000.0f;
  p.c_g.y = 0.01f;
  model.setParams(p);
  std::array<float2, 2> rngs = { float2{ -1.0f, 1.0f }, float2{ -1.0f, 1.0f } };
  model.setControlRanges(rngs);
  // weights 0.3 sin(0.7 i + 0.1), initial hidden / cell zero
  std::vector<float> lstm(model.lstmBlock(), 0.0f), head(8 * 20 + 20 + 20 + 1);
  for (int i = 0; i < model.lstmBlock() - 8; i++)
    lstm[i] = 0.3f * sinf(0.7f * i + 0.1f);
  for (size_t i = 0; i < head.size(); i++)
    head[i] = 0.3f * sinf(0.7f * i + 0.1f);
  model.setAllValues(lstm, head);
  const int w = 120, h = 60;
  std::vector<float> z((size_t)w * h);
  std::vector<float4> n((size_t)w * h);
  for (int i = 0; i < h; i++)
    for (int j = 0; j < w; j++)
    {
      const float x = -10.0f + (j + 0.5f) * 0.5f, y = -15.0f + (i + 0.5f) * 0.5f, v = hill(x, y);
      const float gx = -v * 2.0f * (x - 8.0f) / 50.0f, gy = -v * 2.0f * (y - 1.0f) / 50.0f;
      const float inv = 1.0f / sqrtf(gx * gx + gy * gy + 1.0f);
      z[(size_t)i * w + j] = v;
      n[(size_t)i * w + j] = float4{ -gx * inv, -gy * inv, inv, 0.0f };
    }
  cudaExtent ext = make_cudaExtent(w, h, 0);
  auto* tex = model.getTextureHelper();
  tex->updateTexture(0, z, ext);
  tex->updateOrigin(0, make_float3(-10.0f, -15.0f, 0.0f));
  tex->updateResolution(0, 0.5f);
  tex->enableTexture(0);
  auto* nrm = model.getTextureHelperNormals();
  nrm->updateTexture(0, n, ext);
  nrm->updateOrigin(0, make_float3(-10.0f, -15.0f, 0.0f));
  nrm->updateResolution(0, 0.5f);
  nrm->enableTexture(0);
}

static DYN::state_array start_state(DYN& model, float vx)
{
  std::map<std::string, float> m = { { "VEL_X", vx }, { "VEL_Z", 0.0f }, { "POS_X", 0.0f }, { "POS_Y", 0.0f },
                                     { "POS_Z", 0.32f }, { "OMEGA_X", 0.0f }, { "OMEGA_Y", 0.0f }, { "ROLL", 0.0f },
                                     { "PITCH", 0.0f }, { "YAW", 0.0f }, { "STEER_ANGLE", 0.0f },
                                     { "STEER_ANGLE_RATE", 0.0f }, { "BRAKE_STATE", 0.0f } };
  return model.stateFromMap(m);
}

int main(int argc, char** argv)
{
  std::vector<int> init_output_layers = { 23, 100, 8 };
  std::vector<int> output_layers = { 8, 20, 1 };
  DYN model(3, 20, init_output_layers, 4, 4, output_layers, 11);
  configure(model);
  if (argc > 1 && strcmp(argv[1], "blob") == 0)
  {
    auto b = model.blob();
    fwrite(&b, sizeof(b), 1, stdout);
    DYN::state_array x = start_state(model, 2.0f), xn, xd;
    x(2) = 7.0f, x(3) = 0.5f, x(1) = 0.2f, x(6) = 0.02f, x(7) = -0.03f, x(8) = 0.45f, x(12) = 0.3f;
    DYN::control_array u;
    u << 0.4f, -0.2f;
    DYN::output_array y;
    model.initializeDynamics(x, u, y, 0.0f, 0.02f);
    model.step(x, xn, xd, u, y, 0.0f, 0.02f);
    fwrite(xn.data(), sizeof(float), 24, stdout);
    fwrite(xd.data(), sizeof(float), 24, stdout);
    fwrite(y.data(), sizeof(float), 28, stdout);
    const float4 q = model.getTextureHelperNormals()->queryTextureAtWorldPose(0, make_float3(7.3f, 0.7f, 0.0f));
    fwrite(&q, sizeof(q), 1, stdout);
    return 0;
  }
  {  // fail-loudly probe: no device => status -5 from the C-ABI, no fallback
    mppib_engine* probe = nullptr;
    mppib_desc d{};
    d.dynamics_id = MPPIB_DYN_RACER_SUSPENSION_LSTM;
    d.cost_id = MPPIB_COST_RACER_QUADRATIC;
    d.sampler_id = MPPIB_SAMPLER_GAUSSIAN;
    d.num_rollouts = 64;
    d.num_timesteps = 10;
    d.num_distributions = 1;
    d.world_size = 1;
    d.model_dims[0] = 4;
    d.model_dims[1] = 20;
    int rc = mppib_create(&probe, &d);
    if (rc == MPPIB_ERR_NO_DEVICE)
    {
      printf("no CUDA device: %s\n", mppib_last_error());
      return 5;
    }
    mppib_destroy(probe);
  }
  RacerQuadraticCost cost;
  auto cp = cost.getParams();
  cp.desired_speed = 1.2f;
  cost.setParams(cp);
  using SAMPLER_T = mppi::sampling_distributions::GaussianDistribution<DYN::DYN_PARAMS_T>;
  auto sp = SAMPLER_T::SAMPLING_PARAMS_T();
  for (int i = 0; i < 2; i++)
    sp.std_dev[i] = 0.3f;
  SAMPLER_T sampler(sp);
  const int T = 50;
  const float dt = 0.02f;
  try
  {
    VanillaMPPIController<DYN, RacerQuadraticCost, NoFeedback, T, 4096> ctrl(&model, &cost, nullptr, &sampler, dt, 1, 1.0f,
                                                                            0.0f);
    DYN::state_array x = start_state(model, 1.0f), xn, xd;
    DYN::output_array y;
    DYN::control_array u0 = DYN::control_array::Zero();
    model.initializeDynamics(x, u0, y, 0.0f, dt);
    double speed = 0.0;
    float max_tilt = 0.0f, max_force = 0.0f;
    const int steps = 600;  // 12 s from x = 0 towards the hill at x = 8 m
    for (int it = 0; it < steps; it++)
    {
      ctrl.computeControl(x, 1);
      DYN::control_array u = ctrl.getControlSeq().col(0);
      model.step(x, xn, xd, u, y, it, dt);
      x = xn;
      ctrl.slideControlSequence(1);
      bool finite = true;
      for (int i = 0; i < DYN::STATE_DIM; i++)
        finite = finite && std::isfinite(x(i));
      if (!finite)
      {
        printf("non-finite state at step %d\n", it);
        return 2;
      }
      if (it >= 100)
        speed += x(0) / (steps - 100);
      max_tilt = fmaxf(max_tilt, fmaxf(fabsf(x(6)), fabsf(x(7))));
      max_force = fmaxf(max_force, y(10));
    }
    printf("racer suspension example: x %.2f m, mean speed %.3f (set-point %.2f), max |roll|, |pitch| %.3f, "
           "max wheel force %.1f N\n",
           x(2), speed, cp.desired_speed, max_tilt, max_force);
    // speed held, the hill felt (roll / pitch away from 0) but the car kept level, and the wheels carried load
    const int rc =
        (fabs(speed - cp.desired_speed) < 0.3 && max_tilt > 0.01f && max_tilt < 0.3f && max_force > 0.0f) ? 0 : 3;
    printf("racer suspension example rc %d\n", rc);
    return rc;
  }
  catch (const std::exception& e)
  {
    printf("exception: %s\n", e.what());
    return std::string(e.what()).find("no CUDA device") != std::string::npos ? 5 : 4;
  }
}
