/*
 * engine_internal.cuh — the engine's internal types, shared by csrc/engine.cu and by OUT-OF-TREE PLUGIN LIBRARIES.
 *
 * The reference lets a user compile any Dynamics / Cost against its templates (dynamics.cuh:67-76, cost.cuh:34-35,
 * utils/managed.cuh:109-135). Templates cannot cross a C ABI, so here a (dynamics, cost) pair is a REGISTERED kernel
 * instantiation: the built-in pairs are registered by engine.cu; a user pair is compiled into a second shared library from
 * this header — `make_entry<MyDynamics, MyCost>(dyn_id, cost_id)` instantiates K1 (resident / streaming / RMPPI variants),
 * the side kernels (init-eval, sampled trajectories, the roll-forward: side_rollout_kernels.cuh) and the DDP kernel for it
 * — and handed to the engine with mppib_register_pair(); see plugins_example/ and INTEGRATION.md §E. The plugin library
 * and libmppi_b200.so must be built from the same source revision (kEngineAbi is checked at registration).
 * Six parts of the engine have an owner of their own, declared in their headers and defined in engine.cu: the noise
 * draw (NoiseSource, noise_source.cuh), K1 itself: its pair entry, its K1Plan (the form and geometry, chosen once), the
 * tensor maps, costs and written-back controls (Rollout, rollout.cuh), the merge from K1's block partials to the result
 * record (Reduction, reduction.cuh), the model's blobs: parameters, weights and maps (ModelParams, model_params.cuh), the
 * feedback controller: DDP's weights and workspace and RMPPI's gains (Feedback, feedback.cuh), and the side rollouts'
 * scratch (SideRollouts, side_rollouts.cuh). Pair<>::kernel maps the plan's form to the instantiation that launches. K1
 * reads the current noise buffer, its plan and buffers, writes the partials and takes the model's blobs and the gains
 * through their accessors; the DDP launch reads the weights, the side launches their inputs and outputs. The stage timing
 * of a solve is a seventh, StageTimer, declared below.
 */
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cufft.h>
#include <curand.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <typeinfo>
#include <vector>

#include "../../include/mppi_b200.h"
#include "combine_kernel.cuh"
#include "ddp_kernel.cuh"
#include "device_resources.cuh"
#include "feedback.cuh"
#include "model_params.cuh"
#include "noise_source.cuh"
#include "plugins/costs.cuh"
#include "plugins/dynamics.cuh"
#include "reduction.cuh"
#include "rollout.cuh"
#include "rollout_kernel.cuh"
#include "rollout_kernel_ar_ws.cuh"
#include "rollout_kernel_nn_tc.cuh"
#include "side_rollout_kernels.cuh"
#include "side_rollouts.cuh"

extern "C" int mppib_set_last_error(int status, const char* fmt, ...);
template <class... A>
static inline int fail(int status, const char* fmt, A... a)
{
  return mppib_set_last_error(status, fmt, a...);
}

#define CUDA_TRY(expr)                                                                                                 \
  do                                                                                                                   \
  {                                                                                                                    \
    cudaError_t _e = (expr);                                                                                           \
    if (_e != cudaSuccess)                                                                                             \
    {                                                                                                                  \
      cudaGetLastError();                                                                                              \
      return fail(MPPIB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__);         \
    }                                                                                                                  \
  } while (0)

#define CURAND_TRY(expr)                                                                                               \
  do                                                                                                                   \
  {                                                                                                                    \
    curandStatus_t _s = (expr);                                                                                        \
    if (_s != CURAND_STATUS_SUCCESS)                                                                                   \
      return fail(MPPIB_ERR_CURAND, "%s failed: curandStatus %d (%s:%d)", #expr, (int)_s, __FILE__, __LINE__);         \
  } while (0)

using namespace mppib;

// ---- stage timing (mppib_enable_timing / mppib_get_timing; definitions in engine.cu) -----------------------------------
// Events at the start of a solve, after the noise draw, after K1 and after K2. Whether a solve is timed is decided once, as
// it is enqueued; a drained solve adds a sample only if it was timed and timing is still on. With several solves in flight
// the events hold the last one's, which alone is counted.
class StageTimer : NoCopy
{
public:
  cudaError_t create();
  void enable(bool on);  // and reset the sums
  // a solve is being enqueued: it is timed iff timing is on; stage 0, then stages i = 1 .. 3
  cudaError_t start(cudaStream_t s) { timed_ = on_; return mark(0, s); }
  cudaError_t mark(int i, cudaStream_t s) { return timed_ ? cudaEventRecord(ev_[i], s) : cudaSuccess; }
  bool timed() const { return timed_; }  // the solve enqueued last
  void collect();                        // after the stream has drained: one sample, if that solve counts
  int read(mppib_timing* out) const;

private:
  Event ev_[4];
  bool on_ = false, timed_ = false;
  double sum_ms_[4] = { 0, 0, 0, 0 };
  long n_ = 0;
};

// ---- engine state -----------------------------------------------------------------------------------------------
// Every device resource is a member that releases itself (device_resources.cuh); a buffer that grows does so through
// reserve(). ~mppib_engine (engine.cu) drains the stream and releases what must go before it; the members follow.
struct mppib_engine
{
  ~mppib_engine();
  // the stream comes before every buffer and event, so that it is destroyed after them
  Stream stream;  // the solve's stream: the engine's own, or mppib_desc.stream borrowed

  mppib_desc desc{};
  int S = 0, C = 0, O = 0, D = 1;
  int N = 0, T = 0, TC = 0;
  int n_local = 0, n_offset = 0;
  int num_sms = 0;  // multiprocessors of the device (grid-stride kernels launch up to 16 CTAs per SM)
  bool rmppi = false;  // MPPIB_FLAG_RMPPI

  // solver scalars
  float dt = 0.01f, lambda = 1.0f, alpha = 0.0f;

  ModelParams model;  // the dynamics and cost blobs, weights and maps (model_params.cuh)
  NoiseSource noise;  // K0 / K0c / NLN draw, its sampler parameters, two buffers and prefetch (noise_source.cuh)
  Rollout rollout;    // K1: pair entry, plan, tensor maps, costs and written-back controls, weights, L2 flush (rollout.cuh)
  Feedback feedback;  // DDP's weights, workspace and status, RMPPI's gains and value-function threshold (feedback.cuh)
  SideRollouts side;  // init-eval, sampled trajectories and the device-side roll-forward (side_rollouts.cuh)
  int pending = 0;    // solves enqueued and not yet waited for
  // smooth-MPPI: the nominal control [T][C] of the last K1, which its merge integrates the new rate mean onto
  std::vector<float> smooth_mu;

  // K1's block partials, K2 and the cross-rank merge, the result record, Tsallis weights, NCCL and KX (reduction.cuh)
  Reduction reduction;
  StageTimer timer;

  bool solved_once = false;
};

// ---- registry of (dynamics, cost) pairs compiled into this library ---------------------------------------------
template <class AUX>
struct AuxFill
{
  static void fill(AUX&, const ModelParams&)
  {
  }
};
template <>
struct AuxFill<plugins::AutorallyNNDynamics::Aux>
{
  static void fill(plugins::AutorallyNNDynamics::Aux& a, const ModelParams& m)
  {
    a.theta_d = m.nn_weights();
  }
};
template <>
struct AuxFill<plugins::RacerLSTMDynamics::Aux>
{
  static void fill(plugins::RacerLSTMDynamics::Aux& a, const ModelParams& m)
  {
    a.theta_d = m.lstm_weights();
    a.H = m.dims()[0];
    a.L1 = m.dims()[1];
    a.elev = m.elevation_map();
  }
};
template <>
struct AuxFill<plugins::RacerSuspensionParts::Aux>
{
  static void fill(plugins::RacerSuspensionParts::Aux& a, const ModelParams& m)
  {
    AuxFill<plugins::RacerLSTMDynamics::Aux>::fill(a, m);
    a.normals = m.normals_map();
  }
};
template <>
struct AuxFill<plugins::RacerDubinsElevationDynamics::Aux>
{
  static void fill(plugins::RacerDubinsElevationDynamics::Aux& a, const ModelParams& m)
  {
    a.elev = m.elevation_map();
  }
};
template <>
struct AuxFill<plugins::ARStandardCost::Aux>
{
  static void fill(plugins::ARStandardCost::Aux& a, const ModelParams& m)
  {
    a.costmap_tex = m.costmap();
  }
};
template <>
struct AuxFill<plugins::QuadrotorMapCost::Aux>
{
  static void fill(plugins::QuadrotorMapCost::Aux& a, const ModelParams& m)
  {
    a.map = m.cost_texture();
  }
};

// the dynamics' parameter blob and device resources, as every per-pair kernel takes them
template <class P, class AUX>
static void fill_dyn_args(P& dyn, AUX& aux, const mppib_engine& e)
{
  memcpy(&dyn, e.model.dyn(), sizeof(dyn));
  AuxFill<AUX>::fill(aux, e.model);
}
// ... and the cost's, the solver scalars, and the sampler at optimisation iteration `iter` (std_dev_decay^iter,
// gaussian.cu:423)
template <class A>
static void fill_pair_args(A& a, const mppib_engine& e, int iter)
{
  fill_dyn_args(a.dyn, a.dyn_aux, e);
  a.dt = e.dt;
  a.lambda = e.lambda;
  a.alpha = e.alpha;
  memcpy(&a.cost, e.model.cost(), sizeof(a.cost));
  AuxFill<decltype(a.cost_aux)>::fill(a.cost_aux, e.model);
  const mppib_gaussian_params& sampler = e.noise.params();
  const float decay = powf(sampler.std_dev_decay, (float)iter);
  for (int d = 0; d < MPPIB_MAX_DISTRIBUTIONS; d++)
    for (int c = 0; c < MPPIB_MAX_CONTROL_DIM; c++)
    {
      const float sd = (c < e.C) ? sampler.std_dev[d * e.C + c] : 1.0f;
      a.samp.std_dev[d][c] = sd;
      a.samp.std_dev_decayed[d][c] = decay * sd;  // gaussian.cu:86-90
    }
  for (int c = 0; c < MPPIB_MAX_CONTROL_DIM; c++)
    a.samp.control_cost_coeff[c] = sampler.control_cost_coeff[c];
  a.samp.pure_noise_threshold = (1.0f - sampler.pure_noise_trajectories_percentage) * e.N;  // gaussian.cu:108
}

template <class DYN, class COST>
struct Pair
{
  using Args = RolloutArgs<DYN, COST>;
  using Kernel = void (*)(Args, CUtensorMap);
  using SmoothArgs = SmoothRolloutArgs<DYN, COST>;
  using SmoothKernel = void (*)(SmoothArgs, CUtensorMap);

  static constexpr bool kHasTensorCoreVariant = std::is_same<DYN, plugins::AutorallyNNDynamics>::value &&
                                                std::is_same<COST, plugins::ARStandardCost>::value;
  // the warp-specialised K1 runs either map cost (rollout_kernel_ar_ws.cuh is templated on it)
  static constexpr bool kHasWarpSpecVariant = std::is_same<DYN, plugins::AutorallyNNMmaDynamics<32>>::value &&
                                              (std::is_same<COST, plugins::ARStandardCost>::value ||
                                               std::is_same<COST, plugins::ARRobustCost>::value);
  // The K1 instantiation of the plan's form, with the streaming form and control write-back as given. Null, with the
  // reason recorded, when this pair is not built for it.
  static Kernel kernel(const K1Plan& k, bool stream, bool wb)
  {
    switch (k.form)
    {
      case K1Form::Wgmma:
        if constexpr (kHasTensorCoreVariant)
          return wb ? rollout_kernel_ar_tc<true> : rollout_kernel_ar_tc<false>;
        break;
      case K1Form::WarpSpec:
        if constexpr (kHasWarpSpecVariant)
          return k.ws_pspw == 16 ? ar_ws_kernel_for<COST, 16>(wb, stream)
                                 : (k.ws_pspw == 8 ? ar_ws_kernel_for<COST, 8>(wb, stream) : ar_ws_kernel_for<COST, 32>(wb, stream));
        break;
      case K1Form::Rmppi:
        if constexpr (DYN::MAX_DISTRIBUTIONS >= 2)
          return rollout_kernel<DYN, COST, 2, true, 1, true>;
        break;
      case K1Form::GenericSpt2:
        if constexpr (DYN::MAX_SPT >= 2)
          return wb ? rollout_kernel<DYN, COST, 1, true, 2> : rollout_kernel<DYN, COST, 1, false, 2>;
        fail(MPPIB_ERR_UNSUPPORTED, "this dynamics model is built for one sample per thread only");
        return nullptr;
      case K1Form::Generic:
        if (k.D == 1)
          return stream ? (wb ? rollout_kernel<DYN, COST, 1, true, 1, false, true> : rollout_kernel<DYN, COST, 1, false, 1, false, true>)
                        : (wb ? rollout_kernel<DYN, COST, 1, true, 1> : rollout_kernel<DYN, COST, 1, false, 1>);
        if constexpr (DYN::MAX_DISTRIBUTIONS >= 2)
          return stream ? (wb ? rollout_kernel<DYN, COST, 2, true, 1, false, true> : rollout_kernel<DYN, COST, 2, false, 1, false, true>)
                        : (wb ? rollout_kernel<DYN, COST, 2, true, 1> : rollout_kernel<DYN, COST, 2, false, 1>);
        break;
    }
    // choose_k1 takes the wgmma and warp-specialised forms only for an entry that has them: what is left is D = 2
    fail(MPPIB_ERR_UNSUPPORTED, "this dynamics model is built for num_distributions == 1 only");
    return nullptr;
  }
  // The smooth-MPPI sampler's instantiation (rollout_kernel_smooth) of a generic form; choose_k1 takes no other form for it
  static SmoothKernel smooth_kernel(const K1Plan& k, bool stream, bool wb)
  {
    if (k.form == K1Form::Generic)
      return stream ? (wb ? rollout_kernel_smooth<DYN, COST, true, 1, true> : rollout_kernel_smooth<DYN, COST, false, 1, true>)
                    : (wb ? rollout_kernel_smooth<DYN, COST, true, 1> : rollout_kernel_smooth<DYN, COST, false, 1>);
    if (k.form == K1Form::GenericSpt2)
    {
      if constexpr (DYN::MAX_SPT >= 2)
        return wb ? rollout_kernel_smooth<DYN, COST, true, 2> : rollout_kernel_smooth<DYN, COST, false, 2>;
    }
    fail(MPPIB_ERR_UNSUPPORTED, "the smooth-MPPI sampler runs on the generic rollout kernel only");
    return nullptr;
  }
  // Sets the dynamic shared memory limit of kernel(k, stream, wb) (smooth_kernel for a smooth plan) to `smem` and, with
  // blocks_per_sm, asks how many CTAs of `threads` threads are resident per SM. Runs in the module that holds the kernels: a
  // plugin library links a CUDA runtime of its own, and only that one knows its kernels.
  static int kernel_attributes(const K1Plan& k, bool stream, bool wb, size_t smem, int threads, int* blocks_per_sm)
  {
    const void* f = k.smooth ? (const void*)smooth_kernel(k, stream, wb) : (const void*)kernel(k, stream, wb);
    if (!f)
      return MPPIB_ERR_UNSUPPORTED;
    CUDA_TRY(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (blocks_per_sm)
      CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, f, threads, smem));
    return MPPIB_OK;
  }

  // the parameter block both samplers' kernels share
  static void fill_launch_args(Args& a, mppib_engine& e, const float* x0, const float* U_in, int opt_stride, int iter)
  {
    const Rollout& r = e.rollout;
    const K1Plan& k = r.plan();
    fill_pair_args(a, e, iter);
    a.eps = e.noise.eps();
    a.costs = r.costs();
    a.partials = e.reduction.partials();
    a.headers = e.reduction.headers();
    a.controls_out = r.controls();
    a.n_local = e.n_local;
    a.n_offset = e.n_offset;
    a.T = e.T;
    a.nchunks = r.nchunks();
    a.pstride = e.reduction.pstride();
    a.opt_stride = opt_stride;
    a.use_tma = k.use_tma ? 1 : 0;
    a.dyn_shared_floats = k.dyn_shared_floats;
    a.ring = k.stream ? k.ring : 0;
    a.stream_readback = k.stream_readback ? 1 : 0;
    a.fb_gains = e.feedback.gains();
    a.value_func_threshold = e.feedback.threshold();
    a.lambda_inv = (float)(1.0 / e.lambda);  // mppi_controller.cu:201-202: 1.0 / lambda in double, narrowed
    memcpy(a.x0, x0, sizeof(float) * e.D * e.S);
    memcpy(a.means, U_in, sizeof(float) * e.D * e.TC);
  }

  static int launch(mppib_engine& e, const float* x0, const float* U_in, int opt_stride, int iter)
  {
    static_assert(sizeof(Args) < 30000, "kernel parameter block too large");
    const Rollout& r = e.rollout;
    const K1Plan& k = r.plan();
    if (k.smooth)
      return launch_smooth(e, x0, U_in, opt_stride, iter);
    Args a;
    fill_launch_args(a, e, x0, U_in, opt_stride, iter);
    kernel(k, k.stream, r.controls() != nullptr)<<<k.grid, k.threads, k.smem_bytes, e.stream>>>(
        a, r.tensor_map(e.noise.current()));
    CUDA_TRY(cudaGetLastError());
    return MPPIB_OK;
  }

  static int launch_smooth(mppib_engine& e, const float* x0, const float* U_in, int opt_stride, int iter)
  {
    static_assert(sizeof(SmoothArgs) < 30000, "kernel parameter block too large");
    const Rollout& r = e.rollout;
    const K1Plan& k = r.plan();
    SmoothArgs a;
    fill_launch_args(a, e, x0, U_in, opt_stride, iter);
    a.rate_mean = e.noise.rate_mean();
    a.dt_s = e.noise.smooth_dt();
    smooth_kernel(k, k.stream, r.controls() != nullptr)<<<k.grid, k.threads, k.smem_bytes, e.stream>>>(
        a, r.tensor_map(e.noise.current()));
    CUDA_TRY(cudaGetLastError());
    return MPPIB_OK;
  }
};

// The launch the side kernels share (side_rollout_kernels.cuh): one thread per item, 64 per CTA; shared memory = the
// dynamics' floats for 64 threads, then `cost_floats` (side_smem_floats), plus 16 bytes
template <class DYN, class Kernel, class Args>
static int launch_helper_kernel(Kernel kernel, Args& a, const mppib_engine& e, int cost_floats, int items)
{
  static_assert(sizeof(Args) < 30000, "kernel parameter block too large");
  const int threads = 64;
  a.dyn_shared_floats = DYN::sharedFloats(e.desc.model_dims, threads);
  const size_t smem = (size_t)side_smem_floats(a.dyn_shared_floats, cost_floats) * sizeof(float) + 16;
  CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<(items + threads - 1) / threads, threads, smem, e.stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  return MPPIB_OK;
}

// launchInitEvalKernel (core/rmppi_kernels.cu:912-937) for this pair, on e.side's candidates and strides
template <class DYN, class COST>
static int init_eval_launch(mppib_engine& e, int num_candidates, int samples, const float* U_nominal, int opt_stride)
{
  InitEvalArgs<DYN, COST> a;
  fill_pair_args(a, e, 0);  // generateSamples(stride, 0, ...): iteration 0
  a.eps = e.noise.eps();
  a.candidates = e.side.eval_candidates();
  a.strides = e.side.eval_strides();
  a.costs = e.side.eval_costs();
  a.num_candidates = num_candidates;
  a.samples = samples;
  a.T = e.T;
  a.opt_stride = opt_stride;
  memcpy(a.means, U_nominal, sizeof(float) * e.TC);
  return launch_helper_kernel<DYN>(init_eval_kernel<DYN, COST>, a, e, COST::sharedFloats(e.T), num_candidates * samples);
}

// launchVisualizeKernel (core/mppi_common.cu:1376-1420) for this pair, on e.side's indices: see sampled_traj_kernel
template <class DYN, class COST>
static int sampled_traj_launch(mppib_engine& e, const float* x0, const float* U_nominal, int distribution, int n)
{
  SampledTrajArgs<DYN, COST> a;
  fill_pair_args(a, e, 0);
  a.controls = e.rollout.controls() + (size_t)distribution * e.n_local * e.TC;
  a.opt = e.side.sample_opt();
  a.sample_idx = e.side.sample_idx();
  a.outputs = e.side.sample_outputs();
  a.costs = e.side.sample_costs();
  a.crash = e.side.sample_crash();
  a.n = n;
  a.T = e.T;
  a.n_offset = e.n_offset;
  a.distribution = distribution;
  memcpy(a.x0, x0, sizeof(float) * e.S);
  memcpy(a.means, U_nominal, sizeof(float) * e.TC);
  return launch_helper_kernel<DYN>(sampled_traj_kernel<DYN, COST>, a, e, COST::sharedFloats(e.T), n);
}

// device-side host tail for this pair's dynamics, from and into e.side's buffers: see nominal_traj_kernel
template <class DYN>
static int nominal_traj_launch(mppib_engine& e, const float* x0, const float* history)
{
  NominalTrajArgs<DYN> a;
  fill_dyn_args(a.dyn, a.dyn_aux, e);
  a.u_src = e.side.nominal_src();
  a.u_stride = e.side.nominal_stride();
  a.u_out = e.side.nominal_controls();
  a.states = e.side.nominal_states();
  a.outputs = e.side.nominal_outputs();
  a.T = e.T;
  a.D = e.D;
  a.smooth = history != nullptr;
  a.dt = e.dt;
  memset(a.x0, 0, sizeof(a.x0));
  memset(a.history, 0, sizeof(a.history));
  for (int d = 0; d < e.D; d++)
    memcpy(a.x0[d], x0 + (size_t)d * e.S, sizeof(float) * e.S);
  if (history)
    for (int k = 0; k < 2; k++)
      memcpy(a.history[k], history + (size_t)k * e.C, sizeof(float) * e.C);
  return launch_helper_kernel<DYN>(nominal_traj_kernel<DYN>, a, e, 0, 1);
}

// DDPFeedback::computeFeedback for this pair's dynamics (ddp_kernel.cuh), with e.feedback's weights, workspace and status
// word (Feedback::compute has put the targets and the initial controls in the workspace); gains_d = the destination of
// the gain trajectory, or null
template <class DYN>
static int ddp_launch(mppib_engine& e, int T, const float* x0, float* gains_d)
{
  using Args = ddp::DdpArgs<DYN>;
  constexpr int C = DYN::CONTROL_DIM;
  static_assert(sizeof(Args) < 4000, "kernel parameter block too large");
  Args a;
  fill_dyn_args(a.dyn, a.aux, e);
  memcpy(a.Q, e.feedback.Q(), sizeof(a.Q));
  memcpy(a.Qf, e.feedback.Q_f(), sizeof(a.Qf));
  memcpy(a.R, e.feedback.R(), sizeof(a.R));
  memcpy(a.x0, x0, sizeof(a.x0));
  for (int c = 0; c < C; c++)
  {
    a.u_lo[c] = a.dyn.lim.rng_lo[c];
    a.u_hi[c] = a.dyn.lim.rng_hi[c];
  }
  a.dt = e.dt;
  a.T = T;
  a.iters = e.feedback.iters();
  a.ws = e.feedback.ws();
  a.gains = gains_d;
  a.status = e.feedback.status();
  ddp::ddp_kernel<DYN><<<1, ddp::kThreads, 0, e.stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  return MPPIB_OK;
}
template <class DYN>
constexpr int (*ddp_launcher())(mppib_engine&, int, const float*, float*)
{
  if constexpr (DYN::HAS_GRAD)
    return &ddp_launch<DYN>;
  else
    return nullptr;
}

struct PairEntry
{
  int dyn_id, cost_id;
  int S, C, O;
  size_t dyn_bytes, cost_bytes;
  int (*dyn_shared_floats)(const int*, int);
  int max_block_threads;
  int max_spt;
  int spw;  // DYN::SAMPLES_PER_WARP: 32 = one sample per lane; 16 / 8 = sub-warp sample groups (plugins/nn_mma.cuh)
  bool has_warp_spec;  // Pair<>::kHasWarpSpecVariant: K1Form::WarpSpec is built for this pair
  bool has_wgmma;      // Pair<>::kHasTensorCoreVariant: K1Form::Wgmma is built for this pair
  int (*cost_shared_floats)(int);
  int (*launch)(mppib_engine&, const float*, const float*, int, int);
  // Pair<>::kernel_attributes: K1's shared memory limit and occupancy, for a plan, streaming form and write-back
  int (*kernel_attributes)(const K1Plan&, bool stream, bool wb, size_t smem, int threads, int* blocks_per_sm);
  int (*init_eval)(mppib_engine&, int, int, const float*, int);
  int (*sampled_traj)(mppib_engine&, const float*, const float*, int, int);
  int (*nominal_traj)(mppib_engine&, const float*, const float*);
  int (*ddp)(mppib_engine&, int, const float*, float*);  // null: the dynamics have no analytic Jacobian (HAS_GRAD)
};
template <class DYN, class COST>
constexpr PairEntry make_entry(int dyn_id, int cost_id)
{
  return PairEntry{ dyn_id,
                    cost_id,
                    DYN::STATE_DIM,
                    DYN::CONTROL_DIM,
                    DYN::OUTPUT_DIM,
                    sizeof(typename DYN::Params),
                    sizeof(typename COST::Params),
                    &DYN::sharedFloats,
                    DYN::MAX_BLOCK_THREADS,
                    DYN::MAX_SPT,
                    DYN::SAMPLES_PER_WARP,
                    Pair<DYN, COST>::kHasWarpSpecVariant,
                    Pair<DYN, COST>::kHasTensorCoreVariant,
                    &COST::sharedFloats,
                    &Pair<DYN, COST>::launch,
                    &Pair<DYN, COST>::kernel_attributes,
                    &init_eval_launch<typename DYN::AuxDyn, COST>,
                    &sampled_traj_launch<typename DYN::AuxDyn, COST>,
                    &nominal_traj_launch<typename DYN::AuxDyn>,
                    ddp_launcher<typename DYN::AuxDyn>() };
}

// ---- registration of out-of-tree pairs -------------------------------------------------------------------------------------
// Layout fingerprint of the internal structs a plugin library shares with libmppi_b200.so: both must come from the same
// source revision. It takes the entry's function signatures too (as their type's name), because a launcher's arguments can
// change while every size stays the same.
inline unsigned engine_abi()
{
  using Slots = void (*)(decltype(PairEntry::dyn_shared_floats), decltype(PairEntry::cost_shared_floats),
                         decltype(PairEntry::launch), decltype(PairEntry::kernel_attributes),
                         decltype(PairEntry::init_eval), decltype(PairEntry::sampled_traj),
                         decltype(PairEntry::nominal_traj), decltype(PairEntry::ddp));
  unsigned h = (unsigned)(sizeof(mppib_engine) * 131u + sizeof(PairEntry) * 7u + sizeof(SamplerArgs));
  for (const char* c = typeid(Slots).name(); *c; c++)
    h = h * 31u + (unsigned char)*c;
  return h;
}
extern "C" int mppib_register_pair(const void* pair_entry, size_t entry_bytes, unsigned abi);
// what a plugin's mppib_plugin_init() calls, once per pair: ids >= MPPIB_USER_ID_BASE
template <class DYN, class COST>
inline int register_pair(int dyn_id, int cost_id)
{
  const PairEntry e = make_entry<DYN, COST>(dyn_id, cost_id);
  return mppib_register_pair(&e, sizeof(e), engine_abi());
}
