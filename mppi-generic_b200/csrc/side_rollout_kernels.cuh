/*
 * side_rollout_kernels.cuh — the three one-thread-per-rollout kernels that run beside the solve (side_rollouts.cuh owns
 * their buffers): init-eval (RMPPI's nominal-state candidates), sampled trajectories and the device-side roll-forward of the
 * host tail. Each thread rolls out one system through the pieces below; each kernel keeps what is its own: where the
 * controls come from, what it stores per step, its horizon, and whether it enforces the control constraints.
 */
#pragma once
#include "rollout_kernel.cuh"

namespace mppib
{
// Shared memory of a side kernel, in floats: the dynamics' (theta_s) rounded up to whole float4s, then the cost's
// (theta_c). The cost's part starts at side_smem_floats(dyn_shared_floats, 0).
__host__ __device__ inline int side_smem_floats(int dyn_shared_floats, int cost_shared_floats)
{
  return ((dyn_shared_floats + 3) / 4) * 4 + cost_shared_floats;
}

// One system rolled out by one thread: its state, output and the model's carry. ARGS holds the model (dyn, dyn_aux) and dt.
template <class DYN>
struct SideSystem
{
  static constexpr int S = DYN::STATE_DIM, C = DYN::CONTROL_DIM, O = DYN::OUTPUT_DIM;
  float x[1][S], y[1][O];
  typename DYN::Carry carry[1];

  // x = x0, y = 0, then initializeDynamics, which may fill theta_s cooperatively: a __syncthreads must follow
  template <class ARGS>
  __device__ __forceinline__ void init(const ARGS& args, float* theta_s, const float* x0)
  {
#pragma unroll
    for (int i = 0; i < S; i++)
      x[0][i] = x0[i];
#pragma unroll
    for (int i = 0; i < O; i++)
      y[0][i] = 0.0f;
    DYN::initializeDynamics(args.dyn, args.dyn_aux, theta_s, carry[0], x[0], y[0]);
  }
  // step t under u (mppi_common.cu:120): x becomes the next state, y its output
  template <class ARGS>
  __device__ __forceinline__ void step(const ARGS& args, float* theta_s, const float (&u)[1][C], int t)
  {
    float x_next[1][S], xdot[1][S];
#pragma unroll
    for (int i = 0; i < S; i++)
      xdot[0][i] = 0.0f;
    DYN::template stepBatch<1>(args.dyn, args.dyn_aux, theta_s, carry, x, x_next, xdot, u, y, t, args.dt);
#pragma unroll
    for (int i = 0; i < S; i++)
      x[0][i] = x_next[0][i];
  }
};

// The likelihood-ratio cost's scale k_i / sigma_i^2 of distribution d, as K1 hoists it (likelihood_ratio_cost). Returns
// false when every control_cost_coeff is zero (the sampler's default): the term is then skipped.
template <int C>
__device__ __forceinline__ bool likelihood_ratio_scale(const SamplerArgs& samp, int d, float (&lr_scale)[C])
{
  bool lr_on = false;
#pragma unroll
  for (int c = 0; c < C; c++)
  {
    lr_scale[c] = samp.control_cost_coeff[c] / (samp.std_dev[d][c] * samp.std_dev[d][c]);
    lr_on = lr_on || (samp.control_cost_coeff[c] != 0.0f);
  }
  return lr_on;
}

// initEvalKernel, core/rmppi_kernels.cu:230-356: K candidate nominal states x `samples` noise rows; candidate k replays
// the sampled controls shifted by its stride (control at step t = sample at min(t + stride_k, T - 1); the engine refuses a
// negative stride) and only the trajectory cost is kept. One thread per (candidate, sample); the noise rows are the first
// `samples` rows of the block the sampler just drew (readControlSample(candidate_sample_idx, ...), :292-294), read straight
// from HBM/L2.
template <class DYN, class COST>
struct InitEvalArgs
{
  typename DYN::Params dyn;
  typename COST::Params cost;
  typename DYN::Aux dyn_aux;
  typename COST::Aux cost_aux;
  SamplerArgs samp;
  const float* eps;         // [n_local][T][C]
  const float* candidates;  // [K][S]
  const int* strides;       // [K]
  float* costs;             // [K * samples]
  int num_candidates, samples, T, opt_stride, dyn_shared_floats;
  float dt, lambda, alpha;
  float means[kMaxMeanFloats];  // [T][C] nominal control (distribution 0)
};

template <class DYN, class COST>
__global__ void __launch_bounds__(DYN::MAX_BLOCK_THREADS) init_eval_kernel(const __grid_constant__ InitEvalArgs<DYN, COST> args)
{
  constexpr int S = DYN::STATE_DIM, C = DYN::CONTROL_DIM;
  extern __shared__ unsigned char smem_raw[];
  float* theta_s = reinterpret_cast<float*>(smem_raw);
  float* theta_c = theta_s + side_smem_floats(args.dyn_shared_floats, 0);
  const int T = args.T;
  const int gid = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = args.num_candidates * args.samples;
  const bool valid = gid < total;
  const int k = valid ? gid / args.samples : 0, j = valid ? gid % args.samples : 0;
  SideSystem<DYN> sys;
  sys.init(args, theta_s, args.candidates + k * S);
  COST::initializeCosts(args.cost, args.cost_aux, theta_c, T);
  __syncthreads();
  const int stride = args.strides[k];
  const bool pure_noise_row = (float)j >= args.samp.pure_noise_threshold;    // the row's own flags: setGaussianControls
  const bool pure_noise_lr = (float)gid >= args.samp.pure_noise_threshold;   // LR cost is called with global_idx (:331-333)
  float lr_scale[C];
  const bool lr_on = likelihood_ratio_scale<C>(args.samp, 0, lr_scale);
  const float half_lambda_1ma = 0.5f * args.lambda * (1.0f - args.alpha);
  float running = 0.0f;
  int crash = 0;
  float u[1][C];
  for (int t = 0; t < T; t++)
  {
    const int ct = min(t + stride, T - 1);
    const bool use_mean = (j == 0) || (ct < args.opt_stride);
#pragma unroll
    for (int c = 0; c < C; c++)
      u[0][c] = sample_control(args.means[ct * C + c], args.samp.std_dev_decayed[0][c],
                               __ldg(args.eps + ((size_t)j * T + ct) * C + c), use_mean, pure_noise_row);
    DYN::enforceConstraints(args.dyn, sys.x[0], u[0]);
    sys.step(args, theta_s, u, t);
    running += COST::computeRunningCost(args.cost, args.cost_aux, theta_c, sys.y[0], u[0], t, &crash);
    if (lr_on)
      running += likelihood_ratio_cost<C>(lr_scale, args.means + t * C, u[0], pure_noise_lr, half_lambda_1ma);
  }
  running += COST::terminalCost(args.cost, args.cost_aux, sys.y[0]);
  running /= (float)T;
  if (valid)
    args.costs[gid] = running;
}

// ---- sampled (visualisation) trajectories (SURVEY §8 f2) -----------------------------------------------------------------
// The reference's visualizeKernel (core/mppi_common.cu:364-520) re-rolls the control samples the host picked after a
// solve (controller.cu:55-179: the optimised sequence, a random subset, the top-n by weight) and dumps every step's
// output, running cost and crash flag. Here: one thread per picked rollout, controls read back from the written-back
// control buffer of the last solve (already constrained, so enforceConstraints is not applied a second time: deadbands
// are not idempotent), index -1 = the optimised sequence `opt` (constraints applied). Row layout of `costs`: [t] = (state
// cost + likelihood-ratio cost of step t) / T exactly as K1 accumulates them, [T] = terminal cost / T, so that a row sums
// to the rollout's trajectory cost (the reference's kernel mixes strides T and T + 1 between its running and terminal
// writes, :482-520, which scrambles every row but the first; that is not reproduced).
template <class DYN, class COST>
struct SampledTrajArgs
{
  typename DYN::Params dyn;
  typename COST::Params cost;
  typename DYN::Aux dyn_aux;
  typename COST::Aux cost_aux;
  SamplerArgs samp;
  const float* controls;  // [n_local][T][C] of the chosen distribution
  const float* opt;       // [T][C] or nullptr
  const int* sample_idx;  // [n]
  float* outputs;         // [n][T][O]
  float* costs;           // [n][T + 1]
  int* crash;             // [n][T]
  int n, T, n_offset, distribution, dyn_shared_floats;
  float dt, lambda, alpha;
  float x0[32];
  float means[kMaxMeanFloats];  // [T][C] nominal control of the chosen distribution
};

template <class DYN, class COST>
__global__ void __launch_bounds__(DYN::MAX_BLOCK_THREADS)
    sampled_traj_kernel(const __grid_constant__ SampledTrajArgs<DYN, COST> args)
{
  constexpr int S = DYN::STATE_DIM, C = DYN::CONTROL_DIM, O = DYN::OUTPUT_DIM;
  static_assert(S <= 32, "x0 travels in the parameter block");
  extern __shared__ unsigned char smem_raw[];
  float* theta_s = reinterpret_cast<float*>(smem_raw);
  float* theta_c = theta_s + side_smem_floats(args.dyn_shared_floats, 0);
  const int T = args.T;
  const int gid = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = gid < args.n;
  const int idx = valid ? args.sample_idx[gid] : 0;
  const bool from_opt = idx < 0;
  const float* useq = from_opt ? args.opt : args.controls + (size_t)idx * T * C;
  SideSystem<DYN> sys;
  sys.init(args, theta_s, args.x0);
  COST::initializeCosts(args.cost, args.cost_aux, theta_c, T);
  __syncthreads();
  const bool pure_noise = !from_opt && (float)(args.n_offset + idx) >= args.samp.pure_noise_threshold;
  float lr_scale[C];
  const bool lr_on = likelihood_ratio_scale<C>(args.samp, args.distribution, lr_scale);
  const float half_lambda_1ma = 0.5f * args.lambda * (1.0f - args.alpha);
  const float inv_T = 1.0f / (float)T;
  int crash = 0;
  float u[1][C];
  for (int t = 0; t < T; t++)
  {
#pragma unroll
    for (int c = 0; c < C; c++)
      u[0][c] = __ldg(useq + (size_t)t * C + c);
    if (from_opt)
      DYN::enforceConstraints(args.dyn, sys.x[0], u[0]);
    sys.step(args, theta_s, u, t);
    float step_cost = COST::computeRunningCost(args.cost, args.cost_aux, theta_c, sys.y[0], u[0], t, &crash);
    if (lr_on)
      step_cost += likelihood_ratio_cost<C>(lr_scale, args.means + t * C, u[0], pure_noise, half_lambda_1ma);
    if (valid)
    {
#pragma unroll
      for (int i = 0; i < O; i++)
        args.outputs[((size_t)gid * T + t) * O + i] = sys.y[0][i];
      args.costs[(size_t)gid * (T + 1) + t] = step_cost * inv_T;
      args.crash[(size_t)gid * T + t] = crash;
    }
  }
  if (valid)
    args.costs[(size_t)gid * (T + 1) + T] = COST::terminalCost(args.cost, args.cost_aux, sys.y[0]) * inv_T;
}

// =================================================================================================================
// Device-side host tail (SURVEY §8 f2): what Controller::computeControl runs on the HOST after the weighted update —
// smoothControlTrajectoryHelper (controller.cuh:557-586: Savitzky-Golay (-3 12 17 12 -3)/35 over [history(2) | u(T) | u_last
// u_last]) and computeOutputTrajectoryHelper (controller.cuh:643-663: state(0) = x0, output(0) from initializeDynamics, then
// T - 1 step() calls with the constrained controls) — as ONE kernel chained behind K2 on the solve's stream: it reads the
// optimised sequence straight from the result record, so a whole computeControl needs one host wait. One thread per system
// (D <= 2); the other lanes of the warp run along (the mma.sync forms of the network need full warps) and store nothing.
// It is a T-step dependent chain on one thread: slower than the vectorised host twins (DESIGN.md §9), hence opt-in.
template <class DYN>
struct NominalTrajArgs
{
  typename DYN::Params dyn;
  typename DYN::Aux dyn_aux;
  const float* u_src;   // system d's [T][C] at u_src + d * u_stride (the result record, or an uploaded copy)
  float* u_out;         // [D][T][C]   smoothed (or copied) controls
  float* states;        // [D][T][S]
  float* outputs;       // [D][T][O]
  int T, D, u_stride, smooth, dyn_shared_floats;
  float dt;
  float x0[MPPIB_MAX_DISTRIBUTIONS][32];
  float history[2][MPPIB_MAX_CONTROL_DIM];
};

template <class DYN>
__global__ void __launch_bounds__(64) nominal_traj_kernel(const __grid_constant__ NominalTrajArgs<DYN> args)
{
  constexpr int S = DYN::STATE_DIM, C = DYN::CONTROL_DIM, O = DYN::OUTPUT_DIM;
  static_assert(S <= 32, "x0 travels in the parameter block");
  extern __shared__ unsigned char smem_raw[];
  float* theta_s = reinterpret_cast<float*>(smem_raw);
  const int T = args.T, D = args.D;
  // ---- smoothing: every element is independent, the block shares them out ----
  for (int i = threadIdx.x; i < D * T * C; i += blockDim.x)
  {
    const int d = i / (T * C), t = (i / C) % T, c = i % C;
    const float* u = args.u_src + (size_t)d * args.u_stride;
    float v = u[t * C + c];
    if (args.smooth)
    {
      const float coef[5] = { -3.0f / 35.0f, 12.0f / 35.0f, 17.0f / 35.0f, 12.0f / 35.0f, -3.0f / 35.0f };
      float acc = 0.0f;
#pragma unroll
      for (int k = 0; k < 5; k++)
      {
        const int tt = t + k - 2;  // index into u; -2, -1 = the history, >= T = the last control held
        const float b = tt < 0 ? args.history[tt + 2][c] : u[(tt < T ? tt : T - 1) * C + c];
        acc += coef[k] * b;
      }
      v = acc;
    }
    args.u_out[i] = v;
  }
  const bool valid = threadIdx.x < D;
  const int d = valid ? threadIdx.x : 0;
  SideSystem<DYN> sys;
  sys.init(args, theta_s, args.x0[d]);
  __syncthreads();  // theta_s filled, u_out written
  float* st = args.states + (size_t)d * T * S;
  float* ot = args.outputs + (size_t)d * T * O;
  const float* useq = args.u_out + (size_t)d * T * C;
  if (valid)
  {
#pragma unroll
    for (int i = 0; i < S; i++)
      st[i] = sys.x[0][i];
    // row 0 follows the HOST initializeDynamics, which is what computeOutputTrajectoryHelper calls (dynamics.cuh:416-423:
    // y <- x on the first min(S, O) entries); the reference's device initializeDynamics of the RACER model differs
    // (setOutputs(state, state, output), lstm_steering.cu:128)
#pragma unroll
    for (int i = 0; i < O; i++)
      ot[i] = i < S ? sys.x[0][i < S ? i : 0] : 0.0f;
  }
  float u[1][C];
  for (int t = 0; t < T - 1; t++)
  {
#pragma unroll
    for (int c = 0; c < C; c++)
      u[0][c] = useq[(size_t)t * C + c];
    DYN::enforceConstraints(args.dyn, sys.x[0], u[0]);
    sys.step(args, theta_s, u, t);
    if (valid)
    {
#pragma unroll
      for (int i = 0; i < S; i++)
        st[(size_t)(t + 1) * S + i] = sys.x[0][i];
#pragma unroll
      for (int i = 0; i < O; i++)
        ot[(size_t)(t + 1) * O + i] = sys.y[0][i];
    }
  }
}
}  // namespace mppib
