/*
 * tests/plugins/softmin_probe_pair.cu — an out-of-tree (dynamics, cost) pair whose trajectory costs the test chooses, bit for
 * bit, through the noise it hands the engine (mppib_set_noise). It exists to test the softmin reduction (K1's block partials,
 * K2's merge, the Tsallis weights) on costs the in-tree models never produce: +inf, ties, spreads where expf underflows,
 * near-equal costs of 1e16, negative costs. Built by tests/plugins/build.sh; registered under ids 1001 / 1001.
 *
 * The recipe (tests/test_gpu_softmin.py): C = 2, mean 0, sigma 1, so the sampled control is fma(1, eps, +-0) = eps exactly;
 * control ranges +-FLT_MAX, no deadband; dt = 1, x0 = 0.
 *   - state x[0] integrates u[0] (xdot[0] = u[0]): with eps[n][t][0] = 0 for every t but one step t0 >= optimization_stride,
 *     x[0] after the horizon is exactly eps[n][t0][0] (0 + v * 1 = v, then + 0 * 1);
 *   - the running cost is 0 and the terminal cost reads that state once: horizon * x[0], so the engine's trajectory cost
 *     0 / T + (T * x[0]) / T is x[0] whenever T is a power of two (for other T it is what float arithmetic makes of it);
 *   - the control clamp turns +inf into FLT_MAX, so a state >= inf_at (FLT_MAX) costs +inf;
 *   - sample 0 is noise-free (gaussian.cu:101) and rolls the mean, so its state is exactly 0: a state of 0 costs zero_cost.
 * u[1] is never read by the model: it is a free payload channel whose weighted average U[t][1] the test checks.
 */
#include "../../mppi-generic_b200/csrc/engine_internal.cuh"

struct softmin_probe_dyn_params
{
  mppib_control_limits lim;  // every dynamics blob starts with the control limits (enforceConstraints)
};
struct softmin_probe_cost_params
{
  float control_cost_coeff[MPPIB_MAX_CONTROL_DIM];  // CostParams<C> prefix (cost.cuh:18-30)
  float discount;
  float horizon;    // T: the terminal cost is horizon * x[0], so that the engine's division by T gives x[0] back
  float inf_at;     // states >= inf_at cost +inf
  float zero_cost;  // cost of a state of exactly 0 (sample 0, or any sample whose chosen cost is 0)
};

struct SoftminProbeDynamics : public mppib::plugins::Dynamics<SoftminProbeDynamics, softmin_probe_dyn_params, 1, 2, 1>
{
  static constexpr int MAX_SPT = 2;  // build the two-samples-per-thread form of the generic kernel too
  __device__ static __forceinline__ void computeDynamics(const Params&, const float*, const float*, const float* u,
                                                         float* xdot)
  {
    xdot[0] = u[0];
  }
};
struct SoftminProbeCost : public mppib::plugins::Cost<SoftminProbeCost, softmin_probe_cost_params>
{
  __device__ static __forceinline__ float computeStateCost(const Params&, const Aux&, const float*, const float*, int, int*)
  {
    return 0.0f;
  }
  __device__ static __forceinline__ float terminalCost(const Params& p, const Aux&, const float* y)
  {
    if (y[0] >= p.inf_at)
      return INFINITY;
    return p.horizon * (y[0] == 0.0f ? p.zero_cost : y[0]);
  }
};

extern "C" int mppib_plugin_init(void)
{
  return register_pair<SoftminProbeDynamics, SoftminProbeCost>(MPPIB_USER_ID_BASE + 1, MPPIB_USER_ID_BASE + 1);
}
