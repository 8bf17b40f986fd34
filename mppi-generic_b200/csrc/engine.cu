/*
 * engine.cu — the C-ABI (include/mppi_b200.h) and the host-side orchestration of one MPPI solve on one H100:
 *   K0 noise draw (cuRAND XORWOW, same generator / seed / offset / count as controllers/controller.cu:192-207 and
 *      sampling_distributions/gaussian/gaussian.cu:380-381, so sample indexing is bit-identical to the reference)
 *   K1 fused rollout                (rollout_kernel.cuh)
 *   K2 baseline / weights / average (combine_kernel.cuh)  [+ one NCCL all-gather and a second K2 when world_size > 1]
 * One stream, no host round trip between the kernels (the reference synchronises three times per iteration,
 * controllers/MPPI/mppi_controller.cu:187-218); x0 and the nominal controls travel in the kernel parameter bank and
 * the result record is written by K2 straight into mapped pinned host memory, so a solve issues no cudaMemcpy.
 *
 * The engine never computes on the CPU: without a CUDA device mppib_create fails with MPPIB_ERR_NO_DEVICE.
 */
#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <type_traits>
#include <mutex>
#include <vector>

#include "../../include/mppi_b200.h"
#include "combine_kernel.cuh"
#include "noise_colored.cuh"
#include "noise_xorwow.cuh"
#include "plugins/costs.cuh"
#include "plugins/dynamics.cuh"
#include "rollout_kernel.cuh"
#include "rollout_kernel_ar_ws.cuh"
#include "rollout_kernel_nn_tc.cuh"
#include "engine_internal.cuh"
#include "../../include/mppi_b200/host_twins.h"
#include "host_model.h"

namespace
{
// ---- minimal NCCL binding, resolved lazily with dlopen so single-GPU users need no NCCL at all --------------------
struct NcclUniqueId
{
  char internal[128];
};
struct NcclApi
{
  void* handle = nullptr;
  int (*GetUniqueId)(NcclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, NcclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int /*ncclDataType_t*/, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool load()
  {
    if (handle)
      return true;
    const char* names[] = { "libnccl.so.2", "libnccl.so" };
    for (const char* n : names)
    {
      handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (handle)
        break;
    }
    if (!handle)
      return false;
    GetUniqueId = (decltype(GetUniqueId))dlsym(handle, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(handle, "ncclCommInitRank");
    CommDestroy = (decltype(CommDestroy))dlsym(handle, "ncclCommDestroy");
    AllGather = (decltype(AllGather))dlsym(handle, "ncclAllGather");
    GetErrorString = (decltype(GetErrorString))dlsym(handle, "ncclGetErrorString");
    return GetUniqueId && CommInitRank && CommDestroy && AllGather;
  }
};
NcclApi g_nccl;
constexpr int kNcclFloat = 7;  // ncclFloat32

}  // namespace


// The library's error channel: a thread-local message behind mppib_last_error(). Exported (not part of the public header):
// the other translation units (npz_reader.cpp) and out-of-tree plugin libraries (engine_internal.cuh: fail()) report
// through it.
static thread_local std::string g_last_error;
extern "C" int mppib_set_last_error(int status, const char* fmt, ...)
{
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return status;
}

using namespace mppib;

static const PairEntry kPairs[] = {
  make_entry<plugins::CartpoleDynamics, plugins::CartpoleQuadraticCost>(MPPIB_DYN_CARTPOLE,
                                                                        MPPIB_COST_CARTPOLE_QUADRATIC),
  make_entry<plugins::DoubleIntegratorDynamics, plugins::DoubleIntegratorCircleCost>(MPPIB_DYN_DOUBLE_INTEGRATOR,
                                                                                     MPPIB_COST_DI_CIRCLE),
  make_entry<plugins::AutorallyNNDynamics, plugins::ARStandardCost>(MPPIB_DYN_AUTORALLY_NN, MPPIB_COST_AR_STANDARD),
  make_entry<plugins::DoubleIntegratorDynamics, plugins::DoubleIntegratorRobustCost>(MPPIB_DYN_DOUBLE_INTEGRATOR,
                                                                                     MPPIB_COST_DI_ROBUST),
  make_entry<plugins::AutorallyNNDynamics, plugins::ARRobustCost>(MPPIB_DYN_AUTORALLY_NN, MPPIB_COST_AR_ROBUST),
  make_entry<plugins::RacerLSTMDynamics, plugins::RacerQuadraticCost>(MPPIB_DYN_RACER_LSTM, MPPIB_COST_RACER_QUADRATIC),
  make_entry<plugins::QuadrotorDynamics, plugins::QuadrotorQuadraticCost>(MPPIB_DYN_QUADROTOR,
                                                                          MPPIB_COST_QUADROTOR_QUADRATIC),
  make_entry<plugins::QuadrotorDynamics, plugins::QuadrotorMapCost>(MPPIB_DYN_QUADROTOR, MPPIB_COST_QUADROTOR_MAP),
  make_entry<plugins::RacerDubinsElevationDynamics, plugins::RacerQuadraticCost>(MPPIB_DYN_RACER_DUBINS_ELEVATION,
                                                                                 MPPIB_COST_RACER_QUADRATIC),
  make_entry<plugins::RacerSuspensionLSTMDynamics, plugins::RacerQuadraticCost>(MPPIB_DYN_RACER_SUSPENSION_LSTM,
                                                                                MPPIB_COST_RACER_QUADRATIC),
  make_entry<plugins::RacerRigidSuspensionDynamics, plugins::RacerRigidQuadraticCost>(MPPIB_DYN_RACER_SUSPENSION,
                                                                                      MPPIB_COST_RACER_QUADRATIC),
};

// RacerDubinsElevationLSTMSteering and RacerDubinsElevationSuspension with the steering LSTM on tensor cores (hidden_dim
// 32, head width <= 24)
static const PairEntry kPairsLstmMma[] = {
  make_entry<plugins::RacerLSTMMmaDynamics, plugins::RacerQuadraticCost>(MPPIB_DYN_RACER_LSTM, MPPIB_COST_RACER_QUADRATIC),
  make_entry<plugins::RacerSuspensionLSTMMmaDynamics, plugins::RacerQuadraticCost>(MPPIB_DYN_RACER_SUSPENSION_LSTM,
                                                                                   MPPIB_COST_RACER_QUADRATIC),
};
// the models whose steering is RacerDubinsElevationLSTMSteering's network: model_dims = { H, L1 }, weights in
// MPPIB_BLOB_LSTM_WEIGHTS, one distribution
static bool has_steering_lstm(int dyn_id)
{
  return dyn_id == MPPIB_DYN_RACER_LSTM || dyn_id == MPPIB_DYN_RACER_SUSPENSION_LSTM;
}
constexpr int kWsPspw8MaxRollouts = 6144;   // see mppib_create (warp-specialised Autorally K1)
// the Autorally pair's default form, one entry per samples-per-warp width (chosen at create time from n_local)
static const PairEntry kPairsMma[] = {
  make_entry<plugins::AutorallyNNMmaDynamics<32>, plugins::ARStandardCost>(MPPIB_DYN_AUTORALLY_NN, MPPIB_COST_AR_STANDARD),
  make_entry<plugins::AutorallyNNMmaDynamics<16>, plugins::ARStandardCost>(MPPIB_DYN_AUTORALLY_NN, MPPIB_COST_AR_STANDARD),
  make_entry<plugins::AutorallyNNMmaDynamics<8>, plugins::ARStandardCost>(MPPIB_DYN_AUTORALLY_NN, MPPIB_COST_AR_STANDARD),
  make_entry<plugins::AutorallyNNMmaDynamics<32>, plugins::ARRobustCost>(MPPIB_DYN_AUTORALLY_NN, MPPIB_COST_AR_ROBUST),
  make_entry<plugins::AutorallyNNMmaDynamics<16>, plugins::ARRobustCost>(MPPIB_DYN_AUTORALLY_NN, MPPIB_COST_AR_ROBUST),
  make_entry<plugins::AutorallyNNMmaDynamics<8>, plugins::ARRobustCost>(MPPIB_DYN_AUTORALLY_NN, MPPIB_COST_AR_ROBUST),
};

// pairs registered by plugin libraries (mppib_register_pair); std::vector grows, so entries are kept by pointer
static std::vector<PairEntry*>& user_pairs()
{
  static std::vector<PairEntry*> v;
  return v;
}

// ---- the noise draw (noise_source.cuh) ----------------------------------------------------------------------------
// n zeroed floats after room for the offset-alignment lead-in of a library draw (see gen_draw); *out = their start
static cudaError_t alloc_with_lead(DeviceBuffer<float>& b, size_t n, cudaStream_t s, float** out)
{
  const size_t lead = 8192, total = lead + n + 8;  // cudaMalloc is 256-B aligned and 8192 * 4 keeps that
  const cudaError_t rc = b.alloc(total);
  *out = rc == cudaSuccess ? b + lead : nullptr;
  return rc != cudaSuccess ? rc : cudaMemsetAsync(b, 0, total * sizeof(float), s);
}

// the <1>, <2> or <4> instantiation of a noise kernel for control dimension C: the built-in pairs have C = 1, 2 or 4,
// and mppib_register_pair refuses any other C
template <class K>
static K for_c(int C, K k1, K k2, K k4)
{
  return C == 1 ? k1 : (C == 2 ? k2 : k4);
}

int NoiseSource::create(const mppib_desc& desc, int N, int n_offset, int n_local, int T, int C, int num_sms,
                        cudaStream_t stream, int side_priority)
{
  sampler_ = desc.sampler_id;
  world_ = desc.world_size;
  n_local_ = n_local;
  T_ = T;
  C_ = C;
  num_sms_ = num_sms;
  stream_ = stream;
  const bool colored = sampler_ == MPPIB_SAMPLER_COLORED_NOISE, nln = sampler_ == MPPIB_SAMPLER_NLN;
  {
    // normals per generateSamples call and this rank's slice of them
    // colored_noise.cu:341-343 / gaussian.cu:380 / nln.cu:114-122 (C log-normal planes of N*T, then N*T*C normals)
    const unsigned long long per_rollout =
        colored ? 2ULL * C * (T + 1) : (nln ? 2ULL * T * C : (unsigned long long)T * C);
    draw_global_ = per_rollout * (unsigned long long)N;
    draw_start_ = per_rollout * (unsigned long long)n_offset;
    draw_local_ = (size_t)(per_rollout * (unsigned long long)n_local);
  }
  const size_t noise_floats = (size_t)n_local * T * C;
  CUDA_TRY(alloc_with_lead(alloc_[0], noise_floats, stream_, &eps_[0]));
  eps_[1] = eps_[0];
  CUDA_TRY(last_gen_.create(cudaEventDisableTiming));
  if (!(desc.flags & MPPIB_FLAG_NO_PREFETCH) && !getenv("MPPIB_NO_PREFETCH"))
  {
    CUDA_TRY(alloc_with_lead(alloc_[1], noise_floats, stream_, &eps_[1]));
    CUDA_TRY(side_.create(cudaStreamNonBlocking, side_priority));
    for (int i = 0; i < 2; i++)
    {
      CUDA_TRY(k1_done_[i].create(cudaEventDisableTiming));
      CUDA_TRY(gen_done_[i].create(cudaEventDisableTiming));
    }
  }
  if (nln)
    CUDA_TRY(nln_.alloc(noise_floats));
  if (smooth())
  {  // the reference leaves deriv_action_mean_d_ uninitialised (smooth-MPPI.cu:112-123); here it starts at zero
    CUDA_TRY(rate_mean_.alloc((size_t)T * C));
    CUDA_TRY(cudaMemsetAsync(rate_mean_, 0, (size_t)T * C * sizeof(float), stream_));
  }
  if (colored)
  {
    // spectrum (the raw draw), time-domain buffer, tables and the reference's plan (colored_noise.cu:236-282)
    const size_t batch = (size_t)n_local * C;
    CUDA_TRY(alloc_with_lead(spec_alloc_, draw_local_, stream_, &spec_));
    CUDA_TRY(time_.alloc(batch * 2 * T));
    CUDA_TRY(coeffs_.alloc((size_t)C * (T + 1)));
    CUDA_TRY(sigma_.alloc((size_t)C));
    CUDA_TRY(decay_pow_.alloc((size_t)T));
    CUDA_TRY(rearr_.create(cudaEventDisableTiming));
    const cufftResult fr = plan_.make(cufftPlan1d, 2 * T, CUFFT_C2R, (int)batch);
    if (fr != CUFFT_SUCCESS)
      return fail(MPPIB_ERR_CUDA, "cufftPlan1d(%d, C2R, %zu) failed: %d", 2 * T, batch, (int)fr);
  }

  // own XORWOW draw: possible when a solve's block is a whole number of 8192-normal rounds (the states then sit at the
  // same place of every block and one fixed jump takes them from solve to solve). A rank slice that starts or ends
  // inside a round (e.g. 1024 x 100 normals per rank at 8 GPUs) is drawn in WINDOW mode: whole rounds around it, stores
  // predicated to the slice — the library fallback would re-seed 4096 subsequences on every solve.
  const bool xw_aligned = (draw_local_ % 8192) == 0 && (draw_start_ % 8192ULL) == 0;
  if (!nln && !(desc.flags & MPPIB_FLAG_CURAND_HOST_API) && !getenv("MPPIB_CURAND_HOST_API") &&
      (draw_global_ % 8192ULL) == 0 && draw_local_ > 0 && (xw_aligned || !colored))
  {
    const unsigned long long w0 = draw_start_ / 8192ULL, w1 = (draw_start_ + draw_local_ + 8191ULL) / 8192ULL;
    xw_window_ = !xw_aligned;
    xw_first_round_ = w0;
    xw_lead_ = (unsigned)(draw_start_ - w0 * 8192ULL);
    const int rounds_local = (int)(w1 - w0);
    const unsigned long long rounds_global = draw_global_ / 8192ULL;
    xw_chunks_ = 1;
    for (int cand = 1; cand <= 64 && cand <= rounds_local; cand++)
      if (rounds_local % cand == 0 && (rounds_local / cand >= 4 || cand == 1))
        xw_chunks_ = cand;
    xw_rounds_per_chunk_ = rounds_local / xw_chunks_;
    const unsigned long long jump_draws = 2ULL * (rounds_global - (unsigned long long)xw_rounds_per_chunk_);
    std::vector<uint32_t> tables;
    xorwow_nibble_tables(XorwowMatrix::power(jump_draws), tables);
    xw_jump_ = (uint32_t)(kXorwowWeyl * (uint32_t)(jump_draws & 0xffffffffULL));
    const size_t nstates = (size_t)xw_chunks_ * kXorwowStreams;
    CUDA_TRY(xw_states_.alloc(nstates * 6));
    CUDA_TRY(xw_tables_.alloc(tables.size()));
    CUDA_TRY(cudaMemcpyAsync(xw_tables_, tables.data(), tables.size() * sizeof(uint32_t), cudaMemcpyHostToDevice,
                             stream_));
    CUDA_TRY(cudaStreamSynchronize(stream_));
    xw_enabled_ = true;
    if (getenv("MPPIB_DEBUG"))
      fprintf(stderr, "[mppib] create: noise source %p states %p tables %p (%zu B)\n", (void*)this, (void*)xw_states_,
              (void*)xw_tables_, tables.size() * sizeof(uint32_t));
  }

  // Controller::createAndSeedCUDARandomNumberGen (controller.cu:192-207): XORWOW, seed, offset 0
  CURAND_TRY(gen_.make(curandCreateGenerator, CURAND_RNG_PSEUDO_DEFAULT));
  CURAND_TRY(curandSetStream(gen_, stream_));
  return seed(0ULL, 0ULL);
}

int NoiseSource::set_params(const mppib_gaussian_params& sp)
{
  if (sampler_ == MPPIB_SAMPLER_COLORED_NOISE)
  {
    // frequency weights and sigma, computed like ColoredNoiseDistribution::generateSamples does on the host every
    // call (colored_noise.cu:294-338): fftfreq(2T), low-frequency cutoff, f^(-beta_c/2), theoretical std dev
    const int n2 = 2 * T_, F = T_ + 1, Cn = C_;
    // sample frequency i / 2T (colored_noise.cuh:24-34); the s frequencies below the cutoff take the first one at or
    // above it, when there is one
    const float cutoff_freq = fmaxf(sp.fmin, 1.0f / n2);
    int s = 0;
    while (s < F && s / (1.0f * n2) < cutoff_freq)
      s++;
    std::vector<float> coeffs((size_t)Cn * F);  // Eigen MatrixXf(F, C) is column-major: [c][f]
    for (int i = 0; i < F; i++)
      for (int c = 0; c < Cn; c++)
        coeffs[(size_t)c * F + i] = powf(((i < s && s < F) ? s : i) / (1.0f * n2), -sp.exponents[c] / 2.0f);
    float sigma[MPPIB_MAX_CONTROL_DIM] = { 0 };
    for (int i = 0; i < Cn; i++)
    {
      for (int j = 1; j < F - 1; j++)
        sigma[i] += coeffs[(size_t)i * F + j] * coeffs[(size_t)i * F + j];
      const float last = coeffs[(size_t)i * F + F - 1] * ((1.0f + (n2 % 2)) / 2.0f);
      sigma[i] += last * last;
      sigma[i] = 2.0f * sqrtf(sigma[i]) / n2;
      if (!(sigma[i] > 0.0f) || !std::isfinite(sigma[i]))
        return fail(MPPIB_ERR_INVALID_ARG, "ColoredNoise: exponent %g gives a non-finite spectrum", sp.exponents[i]);
    }
    if (side_)
      CUDA_TRY(cudaStreamSynchronize(side_));
    CUDA_TRY(cudaStreamSynchronize(stream_));
    CUDA_TRY(cudaMemcpy(coeffs_, coeffs.data(), coeffs.size() * sizeof(float), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(sigma_, sigma, Cn * sizeof(float), cudaMemcpyHostToDevice));
    colored_decay_table_kernel<<<(T_ + 127) / 128, 128, 0, stream_>>>(decay_pow_, T_, sp.offset_decay_rate);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(stream_));
    prefetch_valid_ = false;  // a prefetched block was shaped with the old table
  }
  if (sampler_ == MPPIB_SAMPLER_NLN && have_params_ && memcmp(sp.std_dev, params_.std_dev, sizeof(sp.std_dev)) != 0)
    prefetch_valid_ = false;  // a prefetched block drew its log-normal planes with the old std dev
  params_ = sp;
  have_params_ = true;
  return MPPIB_OK;
}

int NoiseSource::seed(unsigned long long seed, unsigned long long offset)
{
  if (side_)
    CUDA_TRY(cudaStreamSynchronize(side_));  // a prefetch may still be using the generator
  CUDA_TRY(cudaStreamSynchronize(stream_));
  CURAND_TRY(curandSetPseudoRandomGeneratorSeed(gen_, seed));
  CURAND_TRY(curandSetGeneratorOffset(gen_, 0ULL));
  seed_ = seed;
  rng_offset_ = offset;
  xw_pos_ = kNoPos;
  curand_pos_ = 0;  // the library generator sits at element 0 of the new stream
  prefetch_valid_ = false;
  return MPPIB_OK;
}

// smooth-MPPI: shiftControlTrajectory at stride 1 (smooth-MPPI.cu:34-78): every row of the rate mean becomes row `row`
__global__ void broadcast_row_kernel(float* __restrict__ a, int T, int C, int row)
{
  __shared__ float r[MPPIB_MAX_CONTROL_DIM];
  if (threadIdx.x < C)
    r[threadIdx.x] = a[row * C + threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.x; i < T * C; i += blockDim.x)
    a[i] = r[i % C];
}

int NoiseSource::burn(int n)
{
  // skipping is free for a counter-positioned stream: just move the absolute offset
  rng_offset_ += (unsigned long long)n * draw_global_;  // generators are re-positioned lazily by gen_draw
  prefetch_valid_ = false;
  // the draw chooseAppropriateKernel makes (generateSamples(1, 0, ...), mppi_controller.cu:95) shifts the rate mean too;
  // once it is constant over t, another shift changes nothing
  if (smooth() && n > 0)
  {
    broadcast_row_kernel<<<1, 256, 0, stream_>>>(rate_mean_, T_, C_, std::min(1, T_ - 1));
    CUDA_TRY(cudaGetLastError());
  }
  return MPPIB_OK;
}

int NoiseSource::read_rate_mean(float* host) const
{
  CUDA_TRY(cudaMemcpyAsync(host, rate_mean_, (size_t)T_ * C_ * sizeof(float), cudaMemcpyDeviceToHost, stream_));
  CUDA_TRY(cudaStreamSynchronize(stream_));
  return MPPIB_OK;
}

int NoiseSource::write_rate_mean(const float* host)
{
  CUDA_TRY(cudaMemcpyAsync(rate_mean_, host, (size_t)T_ * C_ * sizeof(float), cudaMemcpyHostToDevice, stream_));
  CUDA_TRY(cudaStreamSynchronize(stream_));
  return MPPIB_OK;
}

int NoiseSource::set_offset_t(long long offset_t)
{
  if (offset_t < 0 || offset_t >= 2 * T_)
    return fail(MPPIB_ERR_INVALID_ARG, "offset_t out of range");
  colored_offset_t_ = (int)offset_t;
  return MPPIB_OK;
}

// ColoredNoise: rearrangeNoise (colored_noise.cu:39-56) from the retained time-domain buffer into eps_[buf] on `st`.
int NoiseSource::colored_rearrange(int buf, cudaStream_t st, int offset_t)
{
  if (offset_t < 0 || offset_t >= 2 * T_)
    return fail(MPPIB_ERR_INVALID_ARG, "optimization_stride %d outside the 2T = %d colored-noise samples", offset_t,
                2 * T_);
  const size_t total = (size_t)n_local_ * T_;
  const dim3 block(256), grid((unsigned)((total + 255) / 256));
  float* dst = eps_[buf];
  for_c(C_, colored_rearrange_kernel<1>, colored_rearrange_kernel<2>, colored_rearrange_kernel<4>)
      <<<grid, block, 0, st>>>(time_, dst, sigma_, decay_pow_, n_local_, T_, offset_t);
  CUDA_TRY(cudaGetLastError());
  buf_offset_t_[buf] = offset_t;
  return MPPIB_OK;
}

// One generateSamples-equivalent draw (gaussian.cu:378-394 / colored_noise.cu:343-372) of the block of the global
// XORWOW stream that starts at global position `pos` (draw_global_ normals per block; this rank keeps elements
// [draw_start_, draw_start_ + draw_local_) of it) into eps_[buf], on `st`. Draws are totally ordered through
// last_gen_ because they share the generator state (and, for ColoredNoise, the spectrum / time buffers).
int NoiseSource::gen_draw(int buf, cudaStream_t st, unsigned long long pos, int offset_t)
{
  const bool colored = sampler_ == MPPIB_SAMPLER_COLORED_NOISE;
  const unsigned long long start = pos + draw_start_;
  const int F = T_ + 1;
  float* dst = colored ? spec_ : eps_[buf];
  bool scaled_in_draw = false;  // the engine's own generator applies configureFrequencyNoise on the way out
  if (any_gen_)
    CUDA_TRY(cudaStreamWaitEvent(st, last_gen_, 0));
  if (colored && rearr_recorded_)
    CUDA_TRY(cudaStreamWaitEvent(st, rearr_, 0));  // a re-rearrange may still be reading time_
  if (sampler_ == MPPIB_SAMPLER_NLN)
  {
    // NLNDistribution::generateSamples (nln.cu:114-128): C curandGenerateLogNormal calls of N*T values (mean 0, std dev
    // sigma_c) into plane c, one curandGenerateNormal of N*T*C, then createNLNNoise. Library generator, call after call like
    // the reference; re-positioning (seed / burn) is exact only where cuRAND honours absolute offsets (multiples of 8192,
    // tools/curand_probe.cu) and every call then stays on such a boundary.
    const size_t plane = (size_t)n_local_ * T_;
    if (plane & 1)
      return fail(MPPIB_ERR_UNSUPPORTED, "cuRAND draws need an even count (N * T = %zu)", plane);
    CURAND_TRY(curandSetStream(gen_, st));
    if (curand_pos_ != pos)
    {
      if ((pos % 8192ULL) != 0 || (plane % 8192) != 0)
        return fail(MPPIB_ERR_UNSUPPORTED, "NLN draws continue the generator call after call; re-positioning it to "
                                           "offset %llu needs N * T (= %zu) to be a multiple of 8192", pos, plane);
      CURAND_TRY(curandSetGeneratorOffset(gen_, pos));
    }
    for (int c = 0; c < C_; c++)
      CURAND_TRY(curandGenerateLogNormal(gen_, nln_ + (size_t)c * plane, plane, 0.0f, params_.std_dev[c]));
    CURAND_TRY(curandGenerateNormal(gen_, dst, plane * C_, 0.0f, 1.0f));
    const int blocks = (int)std::min<size_t>((plane + 255) / 256, (size_t)num_sms_ * 16);
    for_c(C_, nln_combine_kernel<1>, nln_combine_kernel<2>, nln_combine_kernel<4>)
        <<<blocks, 256, 0, st>>>(dst, nln_, n_local_, T_);
    CUDA_TRY(cudaGetLastError());
    curand_pos_ = pos + draw_global_;
  }
  else if (xw_enabled_ && (pos % 8192ULL) == 0)
  {
    const int nstates = xw_chunks_ * kXorwowStreams;
    if (xw_pos_ != pos)
    {
      xorwow_init_kernel<<<(nstates + 127) / 128, 128, 0, st>>>(seed_, pos / 8192ULL + xw_first_round_,
                                                             xw_rounds_per_chunk_, xw_chunks_, xw_states_);
      CUDA_TRY(cudaGetLastError());
    }
    if (colored)
      xorwow_normal_kernel<true><<<(nstates + 255) / 256, 256, 0, st>>>(xw_states_, xw_tables_, xw_jump_,
                                                                       xw_rounds_per_chunk_, xw_chunks_,
                                                                       reinterpret_cast<float2*>(dst), coeffs_, C_, F);
    else
      xorwow_normal_kernel<false><<<(nstates + 255) / 256, 256, 0, st>>>(
          xw_states_, xw_tables_, xw_jump_, xw_rounds_per_chunk_, xw_chunks_, reinterpret_cast<float2*>(dst), nullptr,
          1, 1, xw_lead_, xw_window_ ? (unsigned long long)draw_local_ : 0ULL);
    CUDA_TRY(cudaGetLastError());
    xw_pos_ = pos + draw_global_;
    scaled_in_draw = colored;
  }
  else
  {
    CURAND_TRY(curandSetStream(gen_, st));
    if (world_ == 1 && curand_pos_ == pos)
    {
      // generator already sits at `start`: plain continuation, exactly what the reference does call after call
      CURAND_TRY(curandGenerateNormal(gen_, dst, draw_local_, 0.0f, 1.0f));
    }
    else
    {
      // XORWOW default ordering interleaves 4096 streams x 2 normals: absolute offsets are honoured at multiples of
      // 8192 (tools/curand_probe.cu), so start from the aligned position below and discard the lead-in.
      const unsigned long long aligned = (start / 8192ULL) * 8192ULL;
      const size_t lead = (size_t)(start - aligned);
      if (((lead + draw_local_) & 1) != 0)
        return fail(MPPIB_ERR_UNSUPPORTED, "cuRAND normal draws need an even count (lead %zu + count %zu)", lead,
                    draw_local_);
      CURAND_TRY(curandSetGeneratorOffset(gen_, aligned));
      CURAND_TRY(curandGenerateNormal(gen_, dst - lead, lead + draw_local_, 0.0f, 1.0f));
    }
    curand_pos_ = (world_ == 1) ? pos + draw_global_ : kNoPos;
  }
  if (colored)
  {
    if (!scaled_in_draw)
    {
      const size_t ncomplex = draw_local_ / 2;
      const int blocks = (int)std::min<size_t>((ncomplex + 255) / 256, (size_t)num_sms_ * 16);
      colored_scale_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<float2*>(spec_), coeffs_, ncomplex, C_, F);
      CUDA_TRY(cudaGetLastError());
    }
    if (cufftSetStream(plan_, st) != CUFFT_SUCCESS)
      return fail(MPPIB_ERR_CUDA, "cufftSetStream failed");
    const cufftResult fr = cufftExecC2R(plan_, reinterpret_cast<cufftComplex*>(spec_), time_);
    if (fr != CUFFT_SUCCESS)
      return fail(MPPIB_ERR_CUDA, "cufftExecC2R failed: %d", (int)fr);
    if (int rc = colored_rearrange(buf, st, offset_t))
      return rc;
  }
  CUDA_TRY(cudaEventRecord(last_gen_, st));
  any_gen_ = true;
  return MPPIB_OK;
}

int NoiseSource::draw(int offset_t)
{
  if (prefetch_valid_ && prefetch_pos_ == rng_offset_)
  {
    cur_ ^= 1;
    CUDA_TRY(cudaStreamWaitEvent(stream_, gen_done_[cur_], 0));
    if (sampler_ == MPPIB_SAMPLER_COLORED_NOISE && buf_offset_t_[cur_] != offset_t)
    {
      // the prefetch assumed another optimization_stride: redo the (cheap) rearrange from the time-domain buffer,
      // which still holds this block (no later draw has been issued)
      if (int rc = colored_rearrange(cur_, stream_, offset_t))
        return rc;
      CUDA_TRY(cudaEventRecord(rearr_, stream_));
      rearr_recorded_ = true;
    }
  }
  else if (int rc = gen_draw(cur_, stream_, rng_offset_, offset_t))  // after every kernel that read eps_[cur_]
    return rc;
  prefetch_valid_ = false;
  rng_offset_ += draw_global_;
  if (sampler_ == MPPIB_SAMPLER_COLORED_NOISE)
    colored_offset_t_ = offset_t;  // what the next prefetch assumes
  return MPPIB_OK;
}

cudaError_t NoiseSource::read_by_kernel()
{
  if (!side_)
    return cudaSuccess;
  k1_recorded_[cur_] = true;
  return cudaEventRecord(k1_done_[cur_], stream_);
}

// After K1 of the current solve has been enqueued. The draw only has to wait for the kernel that last read that buffer.
int NoiseSource::prefetch()
{
  if (!side_)
    return MPPIB_OK;
  const int nb = cur_ ^ 1;
  if (k1_recorded_[nb])
    CUDA_TRY(cudaStreamWaitEvent(side_, k1_done_[nb], 0));
  if (int rc = gen_draw(nb, side_, rng_offset_, colored_offset_t_))
    return rc;
  CUDA_TRY(cudaEventRecord(gen_done_[nb], side_));
  prefetch_valid_ = true;
  prefetch_pos_ = rng_offset_;
  return MPPIB_OK;
}

// ---- the merge (reduction.cuh) ------------------------------------------------------------------------------------
// A kernel launch on `s`. `pdl` = programmatic dependent launch: the grid may start while the preceding kernel on the
// stream is still running and blocks at griddepcontrol.wait until that kernel has completed, which hides its launch latency.
template <class... P, class... A>
static cudaError_t launch_on(cudaStream_t s, bool pdl, void (*kernel)(P...), dim3 grid, dim3 block, A... args)
{
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.stream = s;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

int Reduction::create(int D, int TC, int grid, int world, int rank, cudaStream_t stream)
{
  D_ = D;
  TC_ = TC;
  grid_ = grid;
  world_ = world;
  rank_ = rank;
  stream_ = stream;
  pstride_ = ((kPartialHeader + TC + 3) / 4) * 4;
  const size_t rec = (size_t)D * pstride_;
  CUDA_TRY(partials_.alloc((size_t)grid * rec));
  CUDA_TRY(headers_.alloc((size_t)grid * D));
  CUDA_TRY(result_.alloc(rec));
  CUDA_TRY(result_h_.alloc(rec, cudaHostAllocMapped, &result_h_dev_));
  memset(result_h_, 0, rec * sizeof(float));
  if (world > 1)
  {
    CUDA_TRY(rank_rec_.alloc(rec));
    CUDA_TRY(gather_.alloc((size_t)world * rec));
    CUDA_TRY(gather_hdr_.alloc((size_t)world * D));
  }
  return MPPIB_OK;
}

int Reduction::set_grid(int grid)
{
  const size_t rec = (size_t)D_ * pstride_;
  CUDA_TRY(partials_.reserve((size_t)grid * rec, stream_));
  CUDA_TRY(headers_.reserve((size_t)grid * D_, stream_));
  grid_ = grid;
  return MPPIB_OK;
}

// What runs after the engine has drained the stream; the buffers follow.
Reduction::~Reduction()
{
  if (comm_ && g_nccl.CommDestroy)
    g_nccl.CommDestroy(comm_);
  for (void* p : peer_opened_)
    if (p)
      cudaIpcCloseMemHandle(p);
}

int Reduction::enqueue(bool after_k1, const float* costs, const float* controls, int n_local, float lambda)
{
  const float lambda_inv = (float)(1.0 / lambda);
  // K2 over nrec records: out (device) and, when given, out2 (the mapped host copy)
  auto k2 = [&](const float* records, const float4* headers, int nrec, int normalize, float* out, float* out2, bool pdl) {
    return launch_on(stream_, pdl, combine_kernel, dim3((TC_ + kCombineCols - 1) / kCombineCols, D_),
                     dim3(kCombineCols * kCombineGroups), records, headers, nrec, D_, TC_, pstride_, lambda_inv, normalize,
                     out, out2);
  };
  if (tsallis_gamma_ != 0.0f && tsallis_r_ != 0.0f)
  {
    // K2 for the global baseline (device copy only), then the Tsallis-weighted reduction of the written-back controls
    CUDA_TRY(k2(partials_, headers_, grid_, 1, result_, nullptr, after_k1));
    tsallis_reduce_kernel<<<dim3((TC_ + 31) / 32, D_), 512, 0, stream_>>>(costs, controls, n_local, D_, TC_, pstride_,
                                                                          tsallis_gamma_, tsallis_r_, result_,
                                                                          result_h_dev_);
    CUDA_TRY(cudaGetLastError());
    return MPPIB_OK;
  }
  if (world_ == 1)
  {
    CUDA_TRY(k2(partials_, headers_, grid_, 1, result_, result_h_dev_, after_k1));
    return MPPIB_OK;
  }
  // rank record (un-normalised) -> exchange -> merge of the world_ records (normalised)
  CUDA_TRY(k2(partials_, headers_, grid_, 0, rank_rec_, nullptr, after_k1));
  if (p2p_)
  {  // KX: push to peers over NVLink, wait for theirs, merge — one launch
    CUDA_TRY(launch_on(stream_, true, exchange_merge_kernel, dim3(1), dim3(512), (const float*)rank_rec_, peers_, world_,
                       rank_, D_, TC_, pstride_, lambda_inv, ++p2p_seq_, (float*)result_, result_h_dev_));
    return MPPIB_OK;
  }
  const int rc = g_nccl.AllGather(rank_rec_, gather_, (size_t)D_ * pstride_, kNcclFloat, comm_, stream_);
  if (rc != 0)
    return fail(MPPIB_ERR_NCCL, "ncclAllGather failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?");
  const int nh = world_ * D_;
  record_headers_kernel<<<(nh + 63) / 64, 64, 0, stream_>>>(gather_, world_, D_, pstride_, gather_hdr_);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(k2(gather_, gather_hdr_, world_, 1, result_, result_h_dev_, false));
  return MPPIB_OK;
}

// mppib_create and mppib_set_tsallis keep a smooth engine to one rank and exponential weights
int Reduction::enqueue_smooth(bool after_k1, float lambda, float* rate_mean, float dt, const float* mu)
{
  SmoothMerge m;  // 8 KB, copied into the launch's parameter block
  m.rate_mean = rate_mean;
  m.dt = dt;
  memcpy(m.mu, mu, sizeof(float) * TC_);
  CUDA_TRY(launch_on(stream_, after_k1, combine_kernel_smooth, dim3((TC_ + kCombineCols - 1) / kCombineCols, D_),
                     dim3(kCombineCols * kCombineGroups), (const float*)partials_, (const float4*)headers_, grid_, D_, TC_,
                     pstride_, (float)(1.0 / lambda), 1, (float*)result_, result_h_dev_, m));
  return MPPIB_OK;
}

void Reduction::read(float* U_out, mppib_solve_stats* stats) const
{
  for (int d = 0; d < D_; d++)
  {
    const float* r = result_h_ + (size_t)d * pstride_;
    if (stats)
    {
      stats[d].baseline = r[0];
      stats[d].normalizer = r[1];
      stats[d].sum_w2 = r[2];
      stats[d].pad = 0.0f;
    }
    if (U_out)
      memcpy(U_out + (size_t)d * TC_, r + kPartialHeader, sizeof(float) * TC_);
  }
}

int Reduction::set_tsallis(float gamma, float r, bool have_controls)
{
  if (gamma != 0.0f && r != 0.0f)
  {
    if (!have_controls)
      return fail(MPPIB_ERR_STATE, "Tsallis weights reduce the written-back controls: create the engine with "
                                   "MPPIB_FLAG_WRITEBACK_CONTROLS");
    if (world_ != 1)
      return fail(MPPIB_ERR_UNSUPPORTED, "Tsallis weights are built for one rank");
    if (r == 1.0f || !(gamma > 0.0f))
      return fail(MPPIB_ERR_INVALID_ARG, "Tsallis weights need gamma > 0 and r != 1");
  }
  tsallis_gamma_ = gamma;
  tsallis_r_ = r;
  return MPPIB_OK;
}

int Reduction::comm_init(const void* unique_id_128)
{
  if (world_ <= 1)
    return MPPIB_OK;
  if (!g_nccl.load())
    return fail(MPPIB_ERR_NCCL, "libnccl.so.2 could not be loaded: %s", dlerror());
  NcclUniqueId id;
  memcpy(&id, unique_id_128, sizeof(id));
  int rc = g_nccl.CommInitRank(&comm_, world_, id, rank_);
  if (rc != 0)
    return fail(MPPIB_ERR_NCCL, "ncclCommInitRank failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?");
  return MPPIB_OK;
}

int Reduction::p2p_handle(void* handle_64)
{
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  if (world_ < 2 || world_ > 8)
    return fail(MPPIB_ERR_UNSUPPORTED, "peer-memory exchange is built for 2..8 ranks");
  if (!p2p_gather_)
  {
    const size_t floats = (size_t)2 * world_ * D_ * pstride_ + 2 * world_ + 16;
    CUDA_TRY(p2p_gather_.alloc(floats));
    CUDA_TRY(cudaMemset(p2p_gather_, 0, floats * sizeof(float)));
  }
  cudaIpcMemHandle_t h;
  CUDA_TRY(cudaIpcGetMemHandle(&h, p2p_gather_));
  memcpy(handle_64, &h, 64);
  return MPPIB_OK;
}

int Reduction::p2p_open(const void* handles)
{
  if (!p2p_gather_)
    return fail(MPPIB_ERR_STATE, "call mppib_comm_p2p_handle first");
  const size_t gather_floats = (size_t)2 * world_ * D_ * pstride_;
  for (int r = 0; r < world_; r++)
  {
    float* base = nullptr;
    if (r == rank_)
      base = p2p_gather_;
    else
    {
      cudaIpcMemHandle_t h;
      memcpy(&h, (const char*)handles + (size_t)r * 64, 64);
      void* p = nullptr;
      cudaError_t rc = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
      if (rc != cudaSuccess)
      {
        cudaGetLastError();
        return fail(MPPIB_ERR_CUDA, "cudaIpcOpenMemHandle(rank %d) failed: %s — keep the NCCL path", r,
                    cudaGetErrorString(rc));
      }
      peer_opened_[r] = p;
      base = (float*)p;
    }
    peers_.gather[r] = base;
    peers_.flags[r] = reinterpret_cast<unsigned*>(base + gather_floats);
  }
  p2p_ = true;
  p2p_opened_ = true;
  return MPPIB_OK;
}

int Reduction::set_p2p(bool on)
{
  if (on && !p2p_opened_)
    return fail(MPPIB_ERR_STATE, "mppib_comm_p2p_open has not succeeded on this rank");
  if (!on && !comm_)
    return fail(MPPIB_ERR_STATE, "no NCCL communicator to fall back to (mppib_comm_init)");
  p2p_ = on;
  return MPPIB_OK;
}

static int check_ready(mppib_engine* e)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  if (!e->model.is_set(MPPIB_BLOB_DYN_PARAMS) || !e->model.is_set(MPPIB_BLOB_COST_PARAMS) || !e->noise.have_params())
    return fail(MPPIB_ERR_STATE, "dynamics / cost / sampler parameter blobs must be set before solving");
  if (int rc = e->model.ready_for_solve())
    return rc;
  if (!e->reduction.ready())
    return fail(MPPIB_ERR_STATE, "world_size > 1 but mppib_comm_init was not called");
  return MPPIB_OK;
}

// ---- the rollout kernel K1 (rollout.cuh) -----------------------------------------------------------------------------
// The descriptor flags and environment variables that choose K1's form or geometry, for A/B runs and tests of each form.
// Read once per mppib_create; each rule below validates the values it uses.
struct mppib::K1Overrides
{
  bool no_tma;     // MPPIB_FLAG_NO_TMA / MPPIB_NO_TMA: stage the noise with plain loads, never TMA
  bool nn_tensor;  // MPPIB_FLAG_NN_TENSOR / MPPIB_NN_TENSOR: Autorally network on wgmma (rollout_kernel_nn_tc.cuh)
  bool nn_ffma2;   // MPPIB_FLAG_NN_FFMA2 / MPPIB_NN_FFMA2: Autorally network as FP32 FFMA2s (the round-1 form)
  bool nn_mma;     // MPPIB_FLAG_NN_MMA: Autorally network on mma.sync even with one of the two above
  bool lstm_simt;  // MPPIB_FLAG_LSTM_SIMT / MPPIB_LSTM_SIMT: one-thread-per-sample LSTM at hidden_dim 32
  bool no_ws;      // MPPIB_FLAG_NO_WARP_SPEC / MPPIB_NO_WS: generic kernel for the Autorally pair
  bool bx_set;     // MPPIB_BX: samples per CTA
  int bx;
  bool spw_set;    // MPPIB_SPW = 32 / 16 / 8: samples per warp of the generic Autorally kernel (set: no warp-spec)
  int spw;
  int spt;         // MPPIB_SPT: samples per thread (0: unset)
  int ws_pspw;     // MPPIB_WS_PSPW = 32 / 16 / 8: samples per producer warp of the warp-specialised kernel (0: unset)
  bool stream_set; // MPPIB_STREAM = 0 / 1: force the resident or the streaming form
  bool stream;
  bool stream_readback;  // MPPIB_STREAM_READBACK: generic streaming form writes its controls back and re-reads them
};
// The pair entry for the descriptor: the built-in or registered pair, or the Autorally pair's mma.sync form and the LSTM's
// tensor-core form unless an override keeps the other. Needs no device, so these refusals come before any device work.
// *wgmma_asked: NN_TENSOR asks for the wgmma kernel of a pair that has one, even if NN_MMA then keeps the mma.sync entry.
int Rollout::pick(const mppib_desc& desc, K1Overrides* ov, const PairEntry** out, bool* wgmma_asked, bool fp16_ok)
{
  const char* bx = getenv("MPPIB_BX");
  const char* spw = getenv("MPPIB_SPW");
  const char* spt = getenv("MPPIB_SPT");
  const char* ws_pspw = getenv("MPPIB_WS_PSPW");
  const char* stream = getenv("MPPIB_STREAM");
  K1Overrides& o = *ov;
  o.no_tma = (desc.flags & MPPIB_FLAG_NO_TMA) || getenv("MPPIB_NO_TMA");
  o.nn_tensor = (desc.flags & MPPIB_FLAG_NN_TENSOR) || getenv("MPPIB_NN_TENSOR");
  o.nn_ffma2 = (desc.flags & MPPIB_FLAG_NN_FFMA2) || getenv("MPPIB_NN_FFMA2");
  o.nn_mma = (desc.flags & MPPIB_FLAG_NN_MMA) != 0;
  o.lstm_simt = (desc.flags & MPPIB_FLAG_LSTM_SIMT) || getenv("MPPIB_LSTM_SIMT");
  o.no_ws = (desc.flags & MPPIB_FLAG_NO_WARP_SPEC) || getenv("MPPIB_NO_WS");
  o.bx_set = bx != nullptr;
  o.bx = bx ? atoi(bx) : 0;
  o.spw_set = spw != nullptr;
  o.spw = spw ? atoi(spw) : 0;
  o.spt = spt ? atoi(spt) : 0;
  o.ws_pspw = ws_pspw ? atoi(ws_pspw) : 0;
  o.stream_set = stream != nullptr;
  o.stream = stream && atoi(stream) != 0;
  o.stream_readback = getenv("MPPIB_STREAM_READBACK") != nullptr;

  const PairEntry* entry = nullptr;
  for (const auto& p : kPairs)
    if (p.dyn_id == desc.dynamics_id && p.cost_id == desc.cost_id)
      entry = &p;
  for (const PairEntry* p : user_pairs())  // out-of-tree pairs (mppib_load_plugin / mppib_register_pair)
    if (p->dyn_id == desc.dynamics_id && p->cost_id == desc.cost_id)
      entry = p;
  *wgmma_asked = entry && entry->has_wgmma && o.nn_tensor;
  // Autorally pair: the network runs on register-level mma.sync by default (plugins/nn_mma.cuh). NN_FFMA2 keeps the FFMA2
  // form, NN_TENSOR selects the wgmma kernel (which is built on the FFMA2 entry). A network whose FP16 operands would
  // overflow (network_fits_fp16) keeps the FFMA2 entry even under NN_MMA: mma.sync would turn them into inf and NaN.
  if (entry && desc.dynamics_id == MPPIB_DYN_AUTORALLY_NN && (!(o.nn_ffma2 || o.nn_tensor) || o.nn_mma) && fp16_ok)
  {
    // samples per warp of the generic kernel's network (plugins/nn_mma.cuh): 32. Narrower sample groups (MPPIB_SPW = 16 / 8)
    // halve / quarter a warp's tensor work per step, but the step time of a lone warp barely moves: the chain, not the
    // work, is the limit — which the warp-specialised kernel (rollout_kernel_ar_ws.cuh, the default for D == 1) removes instead.
    const int spw = (o.spw == 16 || o.spw == 8) ? o.spw : 32;
    for (const auto& p : kPairsMma)
      if (p.cost_id == desc.cost_id && p.spw == spw)
        entry = &p;
  }
  // steering LSTM at hidden_dim 32 (head width <= 24): gates and head as mma.sync products, hidden / cell state in fragment
  // layout in registers (plugins/lstm_mma.cuh). LSTM_SIMT keeps the one-thread-per-sample network, and so does a network
  // whose FP16 operands would overflow (network_fits_fp16), where the tensor-core form would turn them into inf and NaN.
  if (entry && has_steering_lstm(desc.dynamics_id) && desc.model_dims[0] == lstm_mma::H &&
      desc.model_dims[1] <= 8 * lstm_mma::kHeadTiles && !o.lstm_simt && fp16_ok)
    for (const auto& p : kPairsLstmMma)
      if (p.dyn_id == desc.dynamics_id && p.cost_id == desc.cost_id)
        entry = &p;
  if (!entry)
    return fail(MPPIB_ERR_UNSUPPORTED, "no kernel registered for dynamics %d + cost %d", desc.dynamics_id, desc.cost_id);
  // the wgmma kernel (rollout_kernel_nn_tc.cuh) is built for ARStandardCost only: refuse rather than run another kernel
  if (desc.dynamics_id == MPPIB_DYN_AUTORALLY_NN && desc.cost_id == MPPIB_COST_AR_ROBUST && o.nn_tensor)
    return fail(MPPIB_ERR_UNSUPPORTED, "MPPIB_FLAG_NN_TENSOR: the tensor-core Autorally kernel supports ARStandardCost only, "
                                       "not ARRobustCost");
  *out = entry;
  return MPPIB_OK;
}

// Whether the model's network fits its tensor-core form's FP16 operands. Both forms split every operand into FP16 hi / lo
// halves (plugins/nn_mma.cuh, plugins/lstm_mma.cuh: split2), and a value of magnitude 65520 or more rounds to an infinite
// hi half, which makes the products NaN; the FP32 forms (FFMA2, SIMT) take such values as they are. So the FP16 form is
// kept only when every pre-scaled weight, and every input bound the engine knows, is below 65504 (the largest FP16
// value). A blob not yet set counts as fitting; the form is chosen again whenever the dynamics parameters or the weights
// are set (reselect_network_form). Biases need no check: both forms keep them in FP32 (C fragments). Models without an
// FP16 form always fit.
//  * Steering LSTM: the gate weights (x -log2 e, or 2 log2 e for the cell gate), head layer 1 (x 2 log2 e) and layer 2
//    (x -2), the initial hidden state, and the input bounds: the steering command's control range (in[2] is the clamped
//    command), max_steer_angle * 0.2 (in[0]) and max_steer_rate * 0.2 (in[3], the clamped parametric rate derivative).
//    Out of scope: a steer rate state that grows past 65504 / 0.2 at run time (in[1]), or an initial steer state outside
//    the limits, since neither is bounded by anything the engine is given. The hidden state itself stays in (-1, 1).
//  * Autorally network (nn_mma::load_weights): W1 x 2 log2 e, W2 x -4 log2 e, W3 x -2, and both control ranges (in[4],
//    in[5] are the clamped commands). Out of scope: states (roll, speeds, yaw rate) that grow past 65504 at run time.
static bool network_fits_fp16(const mppib_desc& desc, const ModelParams& m)
{
  const float kMax = 65504.0f;
  auto fits = [&](float v) { return fabsf(v) < kMax; };  // false for inf and NaN too
  if (desc.dynamics_id == MPPIB_DYN_AUTORALLY_NN)
  {
    if (m.is_set(MPPIB_BLOB_DYN_PARAMS))
    {
      const auto& lim = reinterpret_cast<const mppib_ar_nn_dyn_params*>(m.dyn())->lim;
      for (int c = 0; c < 2; c++)
        if (!fits(lim.rng_lo[c]) || !fits(lim.rng_hi[c]))
          return false;
    }
    if (m.is_set(MPPIB_BLOB_NN_WEIGHTS))
    {
      const std::vector<float>& g = m.nn_weights_host();
      for (int k = 0; k < 192; k++)  // W1
        if (!fits(g[k] * nn_mma::kTanhScale))
          return false;
      for (int k = 224; k < 1248; k++)  // W2
        if (!fits(g[k] * (-2.0f * nn_mma::kTanhScale)))
          return false;
      for (int k = 1280; k < 1408; k++)  // W3
        if (!fits(g[k] * -2.0f))
          return false;
    }
    return true;
  }
  if (!has_steering_lstm(desc.dynamics_id))
    return true;
  if (m.is_set(MPPIB_BLOB_DYN_PARAMS))
  {
    const auto* p = reinterpret_cast<const mppib_racer_lstm_dyn_params*>(m.dyn());
    if (!fits(p->lim.rng_lo[1]) || !fits(p->lim.rng_hi[1]) || !fits(p->max_steer_angle * 0.2f) ||
        !fits(p->max_steer_rate * 0.2f))
      return false;
  }
  if (m.is_set(MPPIB_BLOB_LSTM_WEIGHTS))
  {
    const int H = m.dims()[0], L1 = m.dims()[1], I = MPPIB_RACER_LSTM_INPUT_DIM, HH = H * H, IH = H * I;
    const std::vector<float>& g = m.lstm_weights_host();
    const float sig = -lstm_mma::kLog2e, cell = 2.0f * lstm_mma::kLog2e;
    for (int k = 0; k < 4 * HH; k++)  // W_im W_fm W_om W_cm
      if (!fits(g[k] * (k < 3 * HH ? sig : cell)))
        return false;
    for (int k = 0; k < 4 * IH; k++)  // W_ii W_fi W_oi W_ci
      if (!fits(g[4 * HH + k] * (k < 3 * IH ? sig : cell)))
        return false;
    const float* init_h = g.data() + 4 * HH + 4 * IH + 4 * H;
    for (int k = 0; k < H; k++)
      if (!fits(init_h[k]))
        return false;
    const float* hd = init_h + 2 * H;
    const int IN = H + I;
    for (int k = 0; k < L1 * IN; k++)  // W1
      if (!fits(hd[k] * cell))
        return false;
    for (int k = 0; k < L1; k++)  // W2
      if (!fits(-2.0f * hd[L1 * IN + L1 + k]))
        return false;
  }
  return true;
}

// resident CTAs per SM of the generic kernel's streaming form (registers, threads and shared memory all count), for
// choose_k1 before it takes that form; the rule queries the write-back instantiation whatever the engine's write-back
static int stream_blocks_per_sm(const PairEntry* entry, const K1Plan& plan, int threads, size_t smem)
{
  int n = 0;
  return entry->kernel_attributes(plan, true, true, smem, threads, &n) == MPPIB_OK ? n : 0;
}

// K1's plan for an engine whose sizes, flags and SM count are set, from its pair entry, the overrides and the device's
// limits (max_smem: per block, opted in; smem_per_sm: per multiprocessor): the generic, SPT = 2, RMPPI, warp-specialised or
// wgmma kernel, resident or streaming, and bx, threads, grid, shared memory. `wgmma_asked`: see Rollout::pick.
static int choose_k1(const mppib_engine& e, const PairEntry* entry, const K1Overrides& ov, bool wgmma_asked, int nchunks,
                     int max_smem, int smem_per_sm, K1Plan* out)
{
  // One thread per sample; bx samples per CTA, whole-horizon noise tile resident in shared memory. The rollout is bound by
  // the T-step dependency chain, so a CTA takes the same time whatever its width: the block width is chosen to put every CTA
  // in ONE wave (no tail wave running at a fraction of the chip), preferring the narrowest such width (more SMs busy, fewer
  // warps contending per scheduler); 64 if several waves are unavoidable.
  const mppib_desc& desc = e.desc;
  const int num_sms = e.num_sms;
  K1Plan p;
  p.D = e.D;
  const bool tma_ok = !ov.no_tma && e.TC % 4 == 0;
  // samples per thread (rollout_kernel.cuh): 1. SPT = 2 halves the shared-memory wavefronts per sample of the NN model
  // but a lone warp per scheduler cannot overlap its own FFMA2 / MUFU / latency phases the
  // way two warps do, and it measured slower. Kept selectable for experiments through MPPIB_SPT.
  p.spt = (ov.spt >= 1 && ov.spt <= entry->max_spt && (ov.spt == 1 || e.D == 1)) ? ov.spt : 1;
  p.lps = 32 / entry->spw;
  const int spt = p.spt, lps = p.lps;
  // Autorally pair, one system: the warp-specialised K1 (rollout_kernel_ar_ws.cuh) — a producer and a consumer warp per 32
  // samples. MPPIB_NO_WS / MPPIB_SPW / MPPIB_SPT keep the generic kernel (A/B runs, tests of the generic form).
  // the smooth-MPPI sampler is built into the generic kernel only
  p.smooth = e.noise.smooth();
  const bool ws = entry->has_warp_spec && e.D == 1 && !e.rmppi && spt == 1 && !ov.no_ws && !ov.spw_set && !p.smooth;
  p.form = ws ? K1Form::WarpSpec
              : (e.rmppi ? K1Form::Rmppi : (e.D == 1 && spt == 2 ? K1Form::GenericSpt2 : K1Form::Generic));
  // samples per producer warp: 16 while the GPU is throughput-bound; 8 (four producers per 32 samples, one per scheduler)
  // once it holds so few rollouts that a group's step time sets K1 (kWsPspw8MaxRollouts)
  p.ws_pspw = (ov.ws_pspw == 32 || ov.ws_pspw == 16 || ov.ws_pspw == 8) ? ov.ws_pspw
                                                                       : (e.n_local <= kWsPspw8MaxRollouts ? 8 : 16);
  const int ws_wpg = ar_ws::warpsPerGroup(p.ws_pspw);
  // shared memory of a CTA of b samples whose noise tile holds `chunks` 32-column slabs (all: resident; a ring: streaming)
  auto layout = [&](int b, int chunks) {
    const int dyn_floats = ws ? ar_ws::sharedFloats(b) : entry->dyn_shared_floats(desc.model_dims, b);
    return (int)rollout_smem_layout(b, chunks, e.D, e.TC, dyn_floats, entry->cost_shared_floats(e.T)).total;
  };
  auto smem_for = [&](int b) { return layout(b, nchunks); };
  const int unit = ws ? 32 : entry->spw * spt;  // samples per warp of threads
  const int max_bx = ws ? 32 * ar_ws::maxGroups(p.ws_pspw) : entry->max_block_threads / 32 * unit;  // samples per CTA (__launch_bounds__)
  auto threads_for = [&](int b) { return ws ? ws_wpg * b : b / spt * lps; };
  // resident CTAs per SM: shared memory (+1 KB the hardware reserves per CTA), threads, and for the warp-specialised kernel
  // its 128-register budget
  auto ctas_per_sm = [&](int b, int sm) {
    int n = std::min(std::min(smem_per_sm / (sm + 1024), 2048 / threads_for(b)), 32);
    if (ws)  // registers: __launch_bounds__(maxThreads, 1) lets ptxas use 65536 / maxThreads per thread
      n = std::min(n, ar_ws::maxThreads(p.ws_pspw) / threads_for(b));
    return n;
  };
  auto waves = [&](int b, int per_sm) {  // waves of CTAs of b samples at per_sm CTAs per SM
    const long per_wave = (long)per_sm * num_sms;
    return ((e.n_local + b - 1) / b + per_wave - 1) / per_wave;
  };
  int bx = ov.bx;  // MPPIB_BX, up to 512 here and clamped to max_bx below
  if (bx < unit || bx > 512 || (bx % unit) != 0)
    bx = 0;
  int ws_one_wave = 0;  // warp-specialised kernel: the one-CTA-per-SM width, when __launch_bounds__ allows it
  if (bx == 0 && ws)
  {
    // warp-specialised kernel: up to one warp per scheduler, one pair per CTA (no two producers ever share a scheduler);
    // beyond that ONE CTA per SM, as narrow as covers n_local, so that every SM is busy and the kernel's alternating role
    // table (P C C P C P P C) balances producers over the four schedulers. Wider than the resident tile fits: the wave rule
    // below, and then the streaming form at this width.
    const long pairs_total = (e.n_local + 31) / 32;
    if (ws_wpg * pairs_total <= 4L * num_sms)
      bx = 32;
    else
    {
      const int need = (int)(((e.n_local + num_sms - 1) / num_sms + 31) / 32) * 32;
      if (need <= max_bx)
        ws_one_wave = need;
      if (need <= max_bx && smem_for(need) <= max_smem)
        bx = need;
    }
  }
  if (bx == 0)
  {
    int best = 0;
    long best_waves = 1L << 40;
    for (int cand = ws ? unit : std::max(unit, 64 / lps); cand <= max_bx; cand += unit)
    {
      const int sm = smem_for(cand);
      if (sm > max_smem)
        break;
      const int per_sm = ctas_per_sm(cand, sm);
      if (per_sm < 1)
        break;
      const long w = waves(cand, per_sm);
      if (w < best_waves)
      {
        best_waves = w;
        best = cand;
      }
    }
    bx = best ? best : unit;
  }
  if (bx > max_bx)
    bx = max_bx;
  bx = (bx / unit) * unit;  // whole warps of threads
  if (bx < unit)
    bx = unit;
  while (smem_for(bx) > max_smem && bx > unit)
    bx -= unit;
  p.smem_bytes = (uint32_t)smem_for(bx);
  if ((int)p.smem_bytes > max_smem)
    return fail(MPPIB_ERR_SMEM, "noise tile needs %u B of shared memory, device allows %d", p.smem_bytes, max_smem);
  // tensor-core variant of the Autorally pair: fixed 128-sample CTAs (one warpgroup, two m64 wgmma tiles), streaming
  // noise ring. Opt-in: three exposed MMA round trips per step with few warps per SM to cover them.
  // MPPIB_FLAG_NN_MMA with NN_TENSOR keeps the mma.sync entry (Rollout::pick), which has no wgmma kernel: the form chosen
  // above launches, at the wgmma kernel's width and shared memory (streaming only in the warp-specialised form). This is
  // deliberate: the flag combination keeps the launch it has always had.
  const bool wgmma_width = wgmma_asked && e.D == 1 && tma_ok;
  if (wgmma_width)
  {
    if (entry->has_wgmma)
      p.form = K1Form::Wgmma;
    bx = nn_tc::kRows;
    p.smem_bytes = nn_tc::layout(e.TC, e.T).total;
    if ((int)p.smem_bytes > max_smem)
      return fail(MPPIB_ERR_SMEM, "tensor-core rollout needs %u B of shared memory, device allows %d", p.smem_bytes,
                  max_smem);
  }
  // Streaming form (STREAM in rollout_kernel.cuh and rollout_kernel_ar_ws.cuh): the noise slabs cycle through a ring, so
  // shared memory per sample no longer grows with T. Taken when the resident tile needs several waves and the ring needs
  // fewer; MPPIB_STREAM=0/1 overrides. The generic kernel streams through 2 buffers at 64 samples per CTA (or MPPIB_BX, here
  // up to max_bx), only with TMA, one sample per thread, outside RMPPI and the wgmma kernel. The warp-specialised kernel
  // streams through 3 at its one-CTA-per-SM width (on 132 SMs that is C4, N = 32768: the 256-sample resident tile does not
  // fit, and the 96-thread CTAs the wave rule falls back to run in two waves); forced, it also runs without TMA (the issuing
  // warp fills the ring with plain loads).
  {
    const int ring = ws ? ar_ws::kNoiseRing : p.ring;
    const bool env_bx_ok = ov.bx >= unit && ov.bx <= max_bx && (ov.bx % unit) == 0;
    const int sbx = ws ? ((ws_one_wave && !ov.bx_set) ? ws_one_wave : bx) : (env_bx_ok ? ov.bx : 64);
    const int sm_str = layout(sbx, ring);
    const bool auto_ok = tma_ok && nchunks > ring;
    if ((ws || (auto_ok && !e.rmppi && !wgmma_width && spt == 1)) && sm_str <= max_smem)
    {
      // the generic kernel asks the occupancy API (registers count too); the warp-specialised one's budget is fixed
      const int per_sm_str = ws ? std::max(1, ctas_per_sm(sbx, sm_str))
                                : stream_blocks_per_sm(entry, p, threads_for(sbx), (size_t)sm_str);
      if (per_sm_str > 0)
      {
        const long waves_res = waves(bx, std::max(1, ctas_per_sm(bx, smem_for(bx))));
        bool want = auto_ok && waves_res > 1 && waves(sbx, per_sm_str) < waves_res;
        if (ov.stream_set)
          want = ov.stream;
        if (want)
        {
          p.stream = true;
          // A/B: the round-1 form, controls written back and re-read by the epilogue (Rollout::create turns write-back on)
          p.stream_readback = !ws && ov.stream_readback;
          bx = sbx;
          p.smem_bytes = (uint32_t)sm_str;
        }
      }
    }
  }
  p.bx = bx;
  p.threads = p.form == K1Form::Wgmma ? nn_tc::kRows : threads_for(bx);
  p.dyn_shared_floats = ws ? ar_ws::sharedFloats(bx) : entry->dyn_shared_floats(desc.model_dims, bx);
  p.grid = (e.n_local + bx - 1) / bx;
  if (p.grid > kCombineMaxRecords)
    return fail(MPPIB_ERR_UNSUPPORTED, "%d rollout blocks exceed the combine kernel's %d records; raise MPPIB_BX", p.grid,
                kCombineMaxRecords);
  p.use_tma = tma_ok;
  *out = p;
  return MPPIB_OK;
}

// 2-D view of a noise buffer: rows = local rollouts, cols = T*C floats (row pitch T*C*4 B, must be 16-B multiple); box =
// one 32-column slab of bx rows
static int make_tensor_map(float* base, int TC, int n_local, int bx, CUtensorMap* out)
{
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                               const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                               CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess)
    return fail(MPPIB_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t gdim[2] = { (cuuint64_t)TC, (cuuint64_t)n_local };
  cuuint64_t gstride[1] = { (cuuint64_t)TC * sizeof(float) };
  cuuint32_t box[2] = { (cuuint32_t)kChunkFloats, (cuuint32_t)bx };
  cuuint32_t estride[2] = { 1, 1 };
  CUresult r = ((EncodeFn)fn)(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, gdim, gstride, box, estride,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(MPPIB_ERR_CUDA, "cuTensorMapEncodeTiled failed: CUresult %d", (int)r);
  return MPPIB_OK;
}

int Rollout::create(const mppib_engine& e, const PairEntry* entry, const K1Overrides& ov, bool wgmma_asked)
{
  pair_ = entry;
  stream_ = e.stream;
  D_ = e.D;
  n_local_ = e.n_local;
  TC_ = e.TC;
  nchunks_ = (e.TC + kChunkFloats - 1) / kChunkFloats;
  if (nchunks_ > kMaxChunks)
    return fail(MPPIB_ERR_UNSUPPORTED, "T*C = %d exceeds %d", e.TC, kMaxChunks * kChunkFloats);
  int max_smem = 0, smem_per_sm = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, e.desc.device));
  CUDA_TRY(cudaDeviceGetAttribute(&smem_per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, e.desc.device));
  if (int rc = choose_k1(e, entry, ov, wgmma_asked, nchunks_, max_smem, smem_per_sm, &plan_))
    return rc;
  const bool writeback = e.rmppi || (e.desc.flags & MPPIB_FLAG_WRITEBACK_CONTROLS) || plan_.stream_readback;
  CUDA_TRY(costs_.alloc((size_t)D_ * n_local_));
  if (writeback)
    CUDA_TRY(controls_.alloc((size_t)D_ * n_local_ * TC_));
  if (plan_.use_tma)
    for (int i = 0; i < 2; i++)
      if (int rc = make_tensor_map(e.noise.buffer(i), TC_, n_local_, plan_.bx, &tmap_[i]))
        return rc;
  return entry->kernel_attributes(plan_, plan_.stream, writeback, plan_.smem_bytes, plan_.threads, nullptr);
}

int Rollout::launch(mppib_engine& e, const float* x0, const float* U, int opt_stride, int iter) const
{
  return pair_->launch(e, x0, U, opt_stride, iter);
}

int Rollout::read_costs(float* host) const
{
  CUDA_TRY(cudaMemcpyAsync(host, costs_, (size_t)D_ * n_local_ * sizeof(float), cudaMemcpyDeviceToHost, stream_));
  CUDA_TRY(cudaStreamSynchronize(stream_));
  return MPPIB_OK;
}

int Rollout::read_controls(float* host) const
{
  if (!controls_)
    return fail(MPPIB_ERR_STATE, "engine was created without MPPIB_FLAG_WRITEBACK_CONTROLS");
  CUDA_TRY(cudaMemcpyAsync(host, controls_, (size_t)D_ * n_local_ * TC_ * sizeof(float), cudaMemcpyDeviceToHost, stream_));
  CUDA_TRY(cudaStreamSynchronize(stream_));
  return MPPIB_OK;
}

int Rollout::weights(float* host, const float* result, int pstride, float lambda)
{
  const size_t n = (size_t)D_ * n_local_;
  if (!weights_)
    CUDA_TRY(weights_.alloc(n));
  const dim3 grid((n_local_ + 255) / 256 > 1024 ? 1024 : (n_local_ + 255) / 256, D_);
  weights_kernel<<<grid, 256, 0, stream_>>>(costs_, result, n_local_, pstride, (float)(1.0 / lambda), weights_);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(host, weights_, n * sizeof(float), cudaMemcpyDeviceToHost, stream_));
  CUDA_TRY(cudaStreamSynchronize(stream_));
  return MPPIB_OK;
}

int Rollout::set_l2_flush(long long bytes)
{
  CUDA_TRY(cudaStreamSynchronize(stream_));
  l2_flush_.reset();
  if (bytes > 0)  // exactly that many bytes: a larger buffer would change what is flushed
    CUDA_TRY(l2_flush_.alloc((size_t)bytes));
  return MPPIB_OK;
}

cudaError_t Rollout::flush_l2() const
{
  return l2_flush_ ? cudaMemsetAsync(l2_flush_, 0, l2_flush_.capacity(), stream_) : cudaSuccess;
}

// =================================================================================================================
extern "C" {

int mppib_version(void)
{
  return 100;
}

// A (dynamics, cost) pair compiled out of tree from csrc/engine_internal.cuh (plugins_example/): the reference lets users
// instantiate its templates with their own classes (dynamics.cuh:67-76, cost.cuh:34-35); here they instantiate OUR kernels
// with their device twins in a second shared library and register the result. ids >= MPPIB_USER_ID_BASE.
int mppib_register_pair(const void* pair_entry, size_t entry_bytes, unsigned abi)
{
  if (!pair_entry)
    return fail(MPPIB_ERR_INVALID_ARG, "null pair entry");
  if (entry_bytes != sizeof(PairEntry) || abi != engine_abi())
    return fail(MPPIB_ERR_INVALID_ARG, "plugin built against another revision of libmppi_b200 (entry %zu / %zu bytes, abi %u / %u)",
                entry_bytes, sizeof(PairEntry), abi, engine_abi());
  const PairEntry* in = static_cast<const PairEntry*>(pair_entry);
  if (in->dyn_id < MPPIB_USER_ID_BASE || in->cost_id < MPPIB_USER_ID_BASE)
    return fail(MPPIB_ERR_INVALID_ARG, "user pairs take dynamics / cost ids >= %d (got %d, %d)", MPPIB_USER_ID_BASE, in->dyn_id,
                in->cost_id);
  if (in->C != 1 && in->C != 2 && in->C != 4)
    return fail(MPPIB_ERR_UNSUPPORTED, "CONTROL_DIM %d: must divide a 16-byte noise group (1, 2 or 4)", in->C);
  for (PairEntry*& p : user_pairs())
    if (p->dyn_id == in->dyn_id && p->cost_id == in->cost_id)
    {
      p = new PairEntry(*in);  // re-registration (plugin reloaded): engines made from the old entry keep it
      return MPPIB_OK;
    }
  user_pairs().push_back(new PairEntry(*in));
  return MPPIB_OK;
}

// dlopen a plugin library and run its `int mppib_plugin_init(void)` (which calls register_pair<...>() for each of its pairs)
int mppib_load_plugin(const char* path)
{
  if (!path)
    return fail(MPPIB_ERR_INVALID_ARG, "null path");
  void* h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
  if (!h)
    return fail(MPPIB_ERR_INVALID_ARG, "dlopen(%s) failed: %s", path, dlerror());
  // loading the same library again is a no-op (dlopen hands back the same handle; its pairs are registered already)
  static std::mutex mu;
  static std::vector<void*> loaded;
  std::lock_guard<std::mutex> lock(mu);
  for (void* l : loaded)
    if (l == h)
    {
      dlclose(h);  // drop the extra reference
      return MPPIB_OK;
    }
  typedef int (*init_fn)(void);
  init_fn init = (init_fn)dlsym(h, "mppib_plugin_init");
  if (!init)
  {
    dlclose(h);
    return fail(MPPIB_ERR_INVALID_ARG, "%s exports no mppib_plugin_init", path);
  }
  const int rc = init();
  if (rc == MPPIB_OK)
    loaded.push_back(h);
  else
    dlclose(h);  // e.g. built against another revision: a rebuilt file at the same path must be mapped afresh
  return rc;
}

const char* mppib_last_error(void)
{
  return g_last_error.c_str();
}

const char* mppib_strerror(int status)
{
  switch (status)
  {
    case MPPIB_OK:
      return "ok";
    case MPPIB_ERR_INVALID_ARG:
      return "invalid argument";
    case MPPIB_ERR_UNSUPPORTED:
      return "unsupported plugin combination or size";
    case MPPIB_ERR_CUDA:
      return "CUDA runtime error";
    case MPPIB_ERR_CURAND:
      return "cuRAND error";
    case MPPIB_ERR_NO_DEVICE:
      return "no CUDA device (the engine has no CPU fallback)";
    case MPPIB_ERR_NCCL:
      return "NCCL error";
    case MPPIB_ERR_SMEM:
      return "rollout tile does not fit in shared memory";
    case MPPIB_ERR_CUFFT:
      return "cuFFT error";
    case MPPIB_ERR_STATE:
      return "call order violated";
  }
  return "unknown status";
}

int mppib_create(mppib_engine** out, const mppib_desc* desc)
{
  if (!out || !desc)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  if (desc->num_rollouts <= 0 || desc->num_timesteps <= 0)
    return fail(MPPIB_ERR_INVALID_ARG, "num_rollouts and num_timesteps must be positive");
  if (desc->num_distributions < 1 || desc->num_distributions > MPPIB_MAX_DISTRIBUTIONS)
    return fail(MPPIB_ERR_INVALID_ARG, "num_distributions must be 1 or 2");
  const int world = desc->world_size <= 0 ? 1 : desc->world_size;
  if (desc->rank < 0 || desc->rank >= world)
    return fail(MPPIB_ERR_INVALID_ARG, "rank out of range");
  if (desc->sampler_id == MPPIB_SAMPLER_NLN && (desc->world_size != 1 || desc->num_distributions != 1))
    return fail(MPPIB_ERR_UNSUPPORTED, "the NLN sampler is built for one rank and one distribution");
  if (desc->sampler_id == MPPIB_SAMPLER_SMOOTH_MPPI && (desc->world_size > 1 || desc->num_distributions != 1))
    return fail(MPPIB_ERR_UNSUPPORTED, "the smooth-MPPI sampler is built for one rank and one distribution (the reference "
                                       "never writes the second distribution's controls, smooth-MPPI.cu:183-194)");
  if (desc->sampler_id != MPPIB_SAMPLER_GAUSSIAN && desc->sampler_id != MPPIB_SAMPLER_COLORED_NOISE &&
      desc->sampler_id != MPPIB_SAMPLER_NLN && desc->sampler_id != MPPIB_SAMPLER_SMOOTH_MPPI)
    return fail(MPPIB_ERR_UNSUPPORTED, "sampler %d is not built into this library", desc->sampler_id);
  if (desc->sampler_id == MPPIB_SAMPLER_COLORED_NOISE && desc->num_distributions != 1)
    return fail(MPPIB_ERR_UNSUPPORTED,
                "ColoredNoise draws independent noise per distribution (colored_noise.cu:291); only "
                "num_distributions == 1 is built");

  if (has_steering_lstm(desc->dynamics_id))
  {
    const char* model = desc->dynamics_id == MPPIB_DYN_RACER_LSTM ? "RacerDubinsElevationLSTMSteering" :
                                                                     "RacerDubinsElevationSuspension";
    const int H = desc->model_dims[0], L1 = desc->model_dims[1];
    if (H < 1 || H > plugins::RacerLSTMDynamics::MAX_HIDDEN || L1 < 1 || L1 > plugins::RacerLSTMDynamics::MAX_HEAD)
      return fail(MPPIB_ERR_INVALID_ARG, "%s: model_dims = {hidden_dim %d, head width %d} outside [1, %d] x [1, %d]", model,
                  H, L1, plugins::RacerLSTMDynamics::MAX_HIDDEN, plugins::RacerLSTMDynamics::MAX_HEAD);
    if (desc->num_distributions != 1)
      return fail(MPPIB_ERR_UNSUPPORTED, "%s is built for num_distributions == 1 only", model);
  }
  K1Overrides ov;
  const PairEntry* entry = nullptr;
  bool wgmma_asked = false;
  if (int rc = Rollout::pick(*desc, &ov, &entry, &wgmma_asked))
    return rc;
  if (desc->sampler_id == MPPIB_SAMPLER_SMOOTH_MPPI && wgmma_asked)
    return fail(MPPIB_ERR_UNSUPPORTED, "the smooth-MPPI sampler runs on the generic rollout kernel, not the tensor-core "
                                       "Autorally kernel (MPPIB_FLAG_NN_TENSOR)");

  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0)
  {
    cudaGetLastError();
    return fail(MPPIB_ERR_NO_DEVICE, "no CUDA device visible; libmppi_b200 has no CPU path");
  }
  if (desc->device < 0 || desc->device >= ndev)
    return fail(MPPIB_ERR_INVALID_ARG, "device %d out of range (%d devices)", desc->device, ndev);
  CUDA_TRY(cudaSetDevice(desc->device));

  std::unique_ptr<mppib_engine> owner(new mppib_engine());  // every early return below releases what was made so far
  mppib_engine* e = owner.get();
  e->desc = *desc;
  e->desc.world_size = world;
  e->S = entry->S;
  e->C = entry->C;
  e->O = entry->O;
  e->D = desc->num_distributions;
  e->N = desc->num_rollouts;
  e->T = desc->num_timesteps;
  e->TC = e->T * e->C;
  e->rmppi = (desc->flags & MPPIB_FLAG_RMPPI) != 0;
  if (e->rmppi && desc->num_distributions != 2)
    return fail(MPPIB_ERR_INVALID_ARG, "MPPIB_FLAG_RMPPI needs num_distributions == 2 (nominal, real)");

  if (e->D * e->TC > kMaxMeanFloats)
    return fail(MPPIB_ERR_UNSUPPORTED, "D*T*C = %d exceeds %d", e->D * e->TC, kMaxMeanFloats);

  // rollout sharding (SURVEY §8e): contiguous slices, remainder to the last rank
  const int per = e->N / world;
  e->n_offset = per * desc->rank;
  e->n_local = (desc->rank == world - 1) ? (e->N - e->n_offset) : per;
  if (e->n_local <= 0)
    return fail(MPPIB_ERR_INVALID_ARG, "rank %d of %d has no rollouts (N=%d)", desc->rank, world, e->N);

  CUDA_TRY(cudaDeviceGetAttribute(&e->num_sms, cudaDevAttrMultiProcessorCount, desc->device));

  int prio_lo = 0, prio_hi = 0;
  CUDA_TRY(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  if (desc->stream)
    e->stream.borrow((cudaStream_t)desc->stream);
  else
    CUDA_TRY(e->stream.create(cudaStreamNonBlocking, prio_hi));

  e->model.create(e->desc, entry->dyn_bytes, entry->cost_bytes, e->stream);
  e->feedback.create(e->S, e->C, e->T, e->stream);
  if (int rc = e->noise.create(e->desc, e->N, e->n_offset, e->n_local, e->T, e->C, e->num_sms, e->stream, prio_lo))
    return rc;
  if (int rc = e->rollout.create(*e, entry, ov, wgmma_asked))
    return rc;
  if (int rc = e->reduction.create(e->D, e->TC, e->rollout.plan().grid, world, desc->rank, e->stream))
    return rc;
  CUDA_TRY(e->timer.create());
  CUDA_TRY(cudaStreamSynchronize(e->stream));
  *out = owner.release();
  return MPPIB_OK;
}

// What must go before the members release themselves: the stream drained. The members follow in reverse order of
// declaration, the stream last (engine_internal.cuh); the noise source drains its own side stream, and the reduction
// releases the communicator and the peer mappings.
mppib_engine::~mppib_engine()
{
  cudaSetDevice(desc.device);
  if (stream)
    cudaStreamSynchronize(stream);
}

int mppib_destroy(mppib_engine* e)
{
  if (!e)
    return MPPIB_OK;
  if (getenv("MPPIB_DEBUG"))
    fprintf(stderr, "[mppib] destroy: engine %p\n", (void*)e);
  delete e;
  cudaGetLastError();
  return MPPIB_OK;
}

// ---- the model's blobs (model_params.cuh) ---------------------------------------------------------------------------
void ModelParams::create(const mppib_desc& desc, size_t dyn_bytes, size_t cost_bytes, cudaStream_t stream)
{
  stream_ = stream;
  dyn_id_ = desc.dynamics_id;
  cost_id_ = desc.cost_id;
  memcpy(dims_, desc.model_dims, sizeof(dims_));
  dyn_bytes_ = dyn_bytes;
  cost_bytes_ = cost_bytes;
}

// the blobs beyond its two parameter blobs that this pair takes
bool ModelParams::uses(int which) const
{
  switch (which)
  {
    case MPPIB_BLOB_NN_WEIGHTS:
      return dyn_id_ == MPPIB_DYN_AUTORALLY_NN;
    case MPPIB_BLOB_LSTM_WEIGHTS:
      return has_steering_lstm(dyn_id_);
    case MPPIB_BLOB_ELEVATION_MAP:
      return dyn_id_ == MPPIB_DYN_RACER_LSTM || dyn_id_ == MPPIB_DYN_RACER_DUBINS_ELEVATION ||
             dyn_id_ == MPPIB_DYN_RACER_SUSPENSION_LSTM;
    case MPPIB_BLOB_NORMALS_MAP:
      return dyn_id_ == MPPIB_DYN_RACER_SUSPENSION_LSTM;
    case MPPIB_BLOB_COSTMAP:  // the costs whose blobs share the mppib_ar_standard_cost_params prefix
      return cost_id_ == MPPIB_COST_AR_STANDARD || cost_id_ == MPPIB_COST_AR_ROBUST;
    case MPPIB_BLOB_COST_TEXTURE:
      return cost_id_ == MPPIB_COST_QUADROTOR_MAP;
  }
  return false;
}

// kernels of a solve still in flight (mppib_solve_async) read these from device memory: replacing one under them would be
// a use-after-free. The parameter blobs are copied into the kernel arguments at launch.
bool ModelParams::read_by_kernels(int which)
{
  return which == MPPIB_BLOB_NN_WEIGHTS || which == MPPIB_BLOB_LSTM_WEIGHTS || which == MPPIB_BLOB_COSTMAP ||
         which == MPPIB_BLOB_ELEVATION_MAP || which == MPPIB_BLOB_COST_TEXTURE || which == MPPIB_BLOB_NORMALS_MAP;
}

// the maps are optional: without one the ground is flat, every normal points up, and the costmap term is 0
int ModelParams::ready_for_solve() const
{
  if (uses(MPPIB_BLOB_NN_WEIGHTS) && !is_set(MPPIB_BLOB_NN_WEIGHTS))
    return fail(MPPIB_ERR_STATE, "MPPIB_BLOB_NN_WEIGHTS not set");
  if (uses(MPPIB_BLOB_COSTMAP) && !is_set(MPPIB_BLOB_COSTMAP))
    return fail(MPPIB_ERR_STATE, "MPPIB_BLOB_COSTMAP not set");
  if (uses(MPPIB_BLOB_LSTM_WEIGHTS) && !is_set(MPPIB_BLOB_LSTM_WEIGHTS))
    return fail(MPPIB_ERR_STATE, "MPPIB_BLOB_LSTM_WEIGHTS not set");
  return MPPIB_OK;
}

int ModelParams::ready_for_ddp() const
{
  if (!is_set(MPPIB_BLOB_DYN_PARAMS))
    return fail(MPPIB_ERR_STATE, "dynamics parameters were not set");
  if (uses(MPPIB_BLOB_NN_WEIGHTS) && !is_set(MPPIB_BLOB_NN_WEIGHTS))
    return fail(MPPIB_ERR_STATE, "network weights were not set");
  return MPPIB_OK;
}

// nbytes / 4 finite floats (fnn_helper.cu:244-247 asserts finiteness) to the device, allocated by the first upload (the
// size is fixed at create time), and the host copy
int ModelParams::upload_weights(Weights& w, int which, const char* what, const void* host, size_t nbytes)
{
  const float* f = (const float*)host;
  const size_t n = nbytes / sizeof(float);
  for (size_t i = 0; i < n; i++)
    if (!std::isfinite(f[i]))
      return fail(MPPIB_ERR_INVALID_ARG, "%s weight %zu is not finite", what, i);
  set_ &= ~(1u << which);  // the device copy changes from here on
  if (!w.d)
    CUDA_TRY(w.d.alloc(n));
  CUDA_TRY(cudaMemcpyAsync(w.d, host, nbytes, cudaMemcpyHostToDevice, stream_));
  CUDA_TRY(cudaStreamSynchronize(stream_));
  w.h.assign(f, f + n);
  return MPPIB_OK;
}

// A TwoDTextureHelper<float> (channels 1) or <float4> (channels 4) map in the mppib_elevation_map_header + row-major
// values format (params.h): validates the header, grows the device buffer when needed and copies the values. `what` names
// the blob in the error text.
int ModelParams::upload_map(Map& m, int which, const char* what, const void* host, size_t nbytes, int channels)
{
  if (nbytes < sizeof(mppib_elevation_map_header))
    return fail(MPPIB_ERR_INVALID_ARG, "%s: %zu bytes is smaller than its header", what, nbytes);
  mppib_elevation_map_header h;
  memcpy(&h, host, sizeof(h));
  if (h.width < 2 || h.height < 2 || h.width > 16384 || h.height > 16384)
    return fail(MPPIB_ERR_INVALID_ARG, "%s: extent %d x %d (need 2 .. 16384 cells per side)", what, h.width, h.height);
  const size_t cells = (size_t)h.width * h.height, floats = cells * channels;
  if (nbytes != sizeof(h) + floats * sizeof(float))
    return fail(MPPIB_ERR_INVALID_ARG, "%s: got %zu bytes, expected %zu (header + %d x %d x %d floats)", what, nbytes,
                sizeof(h) + floats * sizeof(float), h.width, h.height, channels);
  for (int i = 0; i < 3; i++)
    if (!std::isfinite(h.origin[i]) || !std::isfinite(h.resolution[i]) || h.resolution[i] == 0.0f)
      return fail(MPPIB_ERR_INVALID_ARG, "%s: origin / resolution component %d is not usable", what, i);
  for (int i = 0; i < 9; i++)
    if (!std::isfinite(h.rotations[i]))
      return fail(MPPIB_ERR_INVALID_ARG, "%s: rotation entry %d is not finite", what, i);
  set_ &= ~(1u << which);  // the device copy changes from here on
  CUDA_TRY(m.d.reserve(floats, stream_));
  CUDA_TRY(cudaMemcpyAsync(m.d, (const char*)host + sizeof(h), floats * sizeof(float), cudaMemcpyHostToDevice, stream_));
  CUDA_TRY(cudaStreamSynchronize(stream_));
  m.hdr = h;
  return MPPIB_OK;
}

int ModelParams::set(int which, const void* host, size_t nbytes)
{
  const unsigned char* b = (const unsigned char*)host;
  switch (which)
  {
    case MPPIB_BLOB_DYN_PARAMS:
      if (nbytes != dyn_bytes_)
        return fail(MPPIB_ERR_INVALID_ARG, "dynamics params: got %zu bytes, expected %zu", nbytes, dyn_bytes_);
      dyn_.assign(b, b + nbytes);
      break;
    case MPPIB_BLOB_COST_PARAMS:
      if (nbytes != cost_bytes_)
        return fail(MPPIB_ERR_INVALID_ARG, "cost params: got %zu bytes, expected %zu", nbytes, cost_bytes_);
      cost_.assign(b, b + nbytes);
      break;
    case MPPIB_BLOB_NN_WEIGHTS:
      if (!uses(which))
        return fail(MPPIB_ERR_INVALID_ARG, "NN weights given to a non-NN dynamics");
      if (nbytes != MPPIB_AR_NN_NUM_PARAMS * sizeof(float))
        return fail(MPPIB_ERR_INVALID_ARG, "NN weights: got %zu bytes, expected %zu", nbytes,
                    MPPIB_AR_NN_NUM_PARAMS * sizeof(float));
      if (int rc = upload_weights(nn_, which, "NN", host, nbytes))
        return rc;
      break;
    case MPPIB_BLOB_LSTM_WEIGHTS:
    {
      if (!uses(which))
        return fail(MPPIB_ERR_INVALID_ARG, "LSTM weights given to a dynamics without an LSTM");
      const size_t expect = (size_t)MPPIB_RACER_LSTM_NUM_PARAMS(dims_[0], dims_[1]) * sizeof(float);
      if (nbytes != expect)
        return fail(MPPIB_ERR_INVALID_ARG, "LSTM weights: got %zu bytes, expected %zu (H = %d, head width %d)", nbytes,
                    expect, dims_[0], dims_[1]);
      if (int rc = upload_weights(lstm_, which, "LSTM", host, nbytes))
        return rc;
      break;
    }
    case MPPIB_BLOB_ELEVATION_MAP:
      // TwoDTextureHelper<float>::updateTexture / updateOrigin / updateRotation / updateResolution / enableTexture +
      // copyToDevice of the RACER models' map 0 (racer_dubins_elevation.cuh: tex_helper_), in one blob
      if (!uses(which))
        return fail(MPPIB_ERR_INVALID_ARG, "elevation map given to a dynamics without one");
      // the values themselves may be NaN (unobserved cells): the model's own isfinite guards handle that (racer_dubins.cu:414-425)
      if (int rc = upload_map(elev_, which, "elevation map", host, nbytes))
        return rc;
      elev_h_.assign(b, b + nbytes);
      break;
    case MPPIB_BLOB_NORMALS_MAP:
      // TwoDTextureHelper<float4> normals_tex_helper_ of RacerDubinsElevationSuspension (suspension_lstm.cu:18-57); NaN
      // normals are the model's to handle (:291-294)
      if (!uses(which))
        return fail(MPPIB_ERR_INVALID_ARG, "normals map given to a dynamics without one");
      if (int rc = upload_map(normals_, which, "normals map", host, nbytes, 4))
        return rc;
      normals_h_.assign(b, b + nbytes);
      break;
    case MPPIB_BLOB_COST_TEXTURE:
      // QuadrotorMapCost's tex_helper_ map 0 (quadrotor_map_cost.cu:37-61), the same format
      if (!uses(which))
        return fail(MPPIB_ERR_INVALID_ARG, "cost texture given to a cost without one");
      if (int rc = upload_map(cost_tex_, which, "cost texture", host, nbytes))
        return rc;
      break;
    case MPPIB_BLOB_COSTMAP:
    {
      if (!uses(which))
        return fail(MPPIB_ERR_INVALID_ARG, "costmap given to a cost without a map");
      if (!is_set(MPPIB_BLOB_COST_PARAMS))
        return fail(MPPIB_ERR_STATE, "set MPPIB_BLOB_COST_PARAMS (map_width/map_height) before the costmap");
      mppib_ar_standard_cost_params cp;
      memcpy(&cp, cost_.data(), sizeof(cp));
      const size_t expect = (size_t)cp.map_width * cp.map_height * 4 * sizeof(float);
      if (cp.map_width <= 0 || cp.map_height <= 0 || nbytes != expect)
        return fail(MPPIB_ERR_INVALID_ARG, "costmap: got %zu bytes, expected %zu (%d x %d float4)", nbytes, expect,
                    cp.map_width, cp.map_height);
      // ar_standard_cost.cu:101-176: float4 array, clamp, point filter, element read, normalised coordinates
      cudaChannelFormatDesc ch = cudaCreateChannelDesc(32, 32, 32, 32, cudaChannelFormatKindFloat);
      cudaTextureDesc tex;
      memset(&tex, 0, sizeof(tex));
      tex.addressMode[0] = cudaAddressModeClamp;
      tex.addressMode[1] = cudaAddressModeClamp;
      tex.filterMode = cudaFilterModePoint;
      tex.readMode = cudaReadModeElementType;
      tex.normalizedCoords = 1;
      // a failed replace keeps the texture it held
      CUDA_TRY(costmap_.replace(ch, cp.map_width, cp.map_height, host, (size_t)cp.map_width * 16, tex, stream_));
      break;
    }
    default:
      return fail(MPPIB_ERR_INVALID_ARG, "unknown blob kind %d", which);
  }
  set_ |= 1u << which;
  return MPPIB_OK;
}

int ModelParams::host_roll(const float* x0, const float* u, int T, float dt, float* states, float* outputs) const
{
  // a blob is set only for a model that uses it (set())
  const auto map = [&](int which, const std::vector<unsigned char>& h) {
    return is_set(which) ? (const mppib_elevation_map_header*)h.data() : nullptr;
  };
  FnnT fnn;
  if (is_set(MPPIB_BLOB_NN_WEIGHTS))
    fnn_transpose(nn_.h.data(), fnn);
  const mppib_host_lstm lstm{ lstm_.h.data(), dims_[0], dims_[1], nullptr, nullptr, nullptr };
  const HostModel m{ dyn_id_,
                     dyn_.data(),
                     is_set(MPPIB_BLOB_NN_WEIGHTS) ? &fnn : nullptr,
                     is_set(MPPIB_BLOB_LSTM_WEIGHTS) ? &lstm : nullptr,
                     map(MPPIB_BLOB_ELEVATION_MAP, elev_h_),
                     map(MPPIB_BLOB_NORMALS_MAP, normals_h_) };
  return roll_forward(m, x0, u, T, dt, states, outputs);
}

// The network's form for the blobs as set now (Rollout::pick with network_fits_fp16): when it differs from the one K1 was
// planned for, K1 is planned again for the other entry, after the stream has drained. The side rollouts and DDP follow
// the entry.
static int reselect_network_form(mppib_engine* e)
{
  K1Overrides ov;
  const PairEntry* entry = nullptr;
  bool wgmma_asked = false;
  if (int rc = Rollout::pick(e->desc, &ov, &entry, &wgmma_asked, network_fits_fp16(e->desc, e->model)))
    return rc;
  if (entry == &e->rollout.pair())
    return MPPIB_OK;
  CUDA_TRY(cudaStreamSynchronize(e->stream));
  if (int rc = e->rollout.create(*e, entry, ov, wgmma_asked))
    return rc;
  return e->reduction.set_grid(e->rollout.plan().grid);
}

int mppib_set_blob(mppib_engine* e, int which, const void* host, size_t nbytes)
{
  if (!e || !host)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  if (e->pending != 0 && ModelParams::read_by_kernels(which))
    return fail(MPPIB_ERR_STATE, "mppib_set_blob(%d) while a solve is pending: call mppib_solve_wait first", which);
  if (which != MPPIB_BLOB_SAMPLER_PARAMS)
  {
    if (int rc = e->model.set(which, host, nbytes))
      return rc;
    const bool net_input = which == MPPIB_BLOB_DYN_PARAMS || which == MPPIB_BLOB_LSTM_WEIGHTS ||
                           which == MPPIB_BLOB_NN_WEIGHTS;
    const bool has_fp16_form = has_steering_lstm(e->desc.dynamics_id) || e->desc.dynamics_id == MPPIB_DYN_AUTORALLY_NN;
    return net_input && has_fp16_form ? reselect_network_form(e) : MPPIB_OK;
  }
  const size_t expect = e->noise.smooth() ? sizeof(mppib_smooth_mppi_params) : sizeof(mppib_gaussian_params);
  if (nbytes != expect)
    return fail(MPPIB_ERR_INVALID_ARG, "sampler params: got %zu bytes, expected %zu", nbytes, expect);
  mppib_gaussian_params sp;
  memcpy(&sp, host, sizeof(sp));  // the smooth blob begins with the Gaussian one
  const float smooth_dt = e->noise.smooth() ? static_cast<const mppib_smooth_mppi_params*>(host)->dt : 0.0f;
  if (!std::isfinite(smooth_dt))
    return fail(MPPIB_ERR_INVALID_ARG, "smooth-MPPI dt must be finite");
  if (e->D > 1 && !sp.use_same_noise_for_all_distributions)
    return fail(MPPIB_ERR_UNSUPPORTED,
                "use_same_noise_for_all_distributions = false is not supported (Tube-MPPI default is true, "
                "sampling_distribution.cuh:20)");
  for (int i = 0; i < e->D * e->C; i++)
    if (!(sp.std_dev[i] > 0.0f))
      return fail(MPPIB_ERR_INVALID_ARG, "std_dev[%d] must be positive", i);
  const int rc = e->noise.set_params(sp);
  if (rc == MPPIB_OK && e->noise.smooth())
    e->noise.set_smooth_dt(smooth_dt);
  return rc;
}

int mppib_set_solver(mppib_engine* e, float dt, float lambda, float alpha)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  if (!(dt > 0.0f) || !(lambda > 0.0f))
    return fail(MPPIB_ERR_INVALID_ARG, "dt and lambda must be positive");
  e->dt = dt;
  e->lambda = lambda;
  e->alpha = alpha;
  return MPPIB_OK;
}

int mppib_seed(mppib_engine* e, unsigned long long seed, unsigned long long offset)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->noise.seed(seed, offset);
}

int mppib_get_rng_offset(mppib_engine* e, unsigned long long* offset)
{
  if (!e || !offset)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  *offset = e->noise.offset();
  return MPPIB_OK;
}

int mppib_burn_draws(mppib_engine* e, int n)
{
  if (!e || n < 0)
    return fail(MPPIB_ERR_INVALID_ARG, "bad argument");
  if (e->noise.smooth())  // the burn shifts the rate mean on the device
    CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->noise.burn(n);
}

int mppib_get_derivative_mean(mppib_engine* e, float* host)
{
  if (!e || !host)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  if (!e->noise.smooth())
    return fail(MPPIB_ERR_INVALID_ARG, "only the smooth-MPPI sampler keeps a derivative (rate) mean");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->noise.read_rate_mean(host);
}

int mppib_set_derivative_mean(mppib_engine* e, const float* host)
{
  if (!e || !host)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  if (!e->noise.smooth())
    return fail(MPPIB_ERR_INVALID_ARG, "only the smooth-MPPI sampler keeps a derivative (rate) mean");
  if (e->pending != 0)
    return fail(MPPIB_ERR_STATE, "mppib_set_derivative_mean while a solve is pending: call mppib_solve_wait first");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->noise.write_rate_mean(host);
}

int mppib_comm_unique_id(void* unique_id_128)
{
  if (!unique_id_128)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  if (!g_nccl.load())
    return fail(MPPIB_ERR_NCCL, "libnccl.so.2 could not be loaded: %s", dlerror());
  NcclUniqueId id;
  int rc = g_nccl.GetUniqueId(&id);
  if (rc != 0)
    return fail(MPPIB_ERR_NCCL, "ncclGetUniqueId failed (%d)", rc);
  memcpy(unique_id_128, &id, sizeof(id));
  return MPPIB_OK;
}

int mppib_comm_init(mppib_engine* e, const void* unique_id_128)
{
  if (!e || !unique_id_128)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->reduction.comm_init(unique_id_128);
}

int mppib_comm_p2p_handle(mppib_engine* e, void* handle_64)
{
  if (!e || !handle_64)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->reduction.p2p_handle(handle_64);
}

int mppib_comm_p2p_open(mppib_engine* e, const void* handles)
{
  if (!e || !handles)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->reduction.p2p_open(handles);
}

int mppib_set_noise(mppib_engine* e, const float* host_eps, size_t count)
{
  if (!e || !host_eps)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  if (count != (size_t)e->n_local * e->TC)
    return fail(MPPIB_ERR_INVALID_ARG, "noise count %zu != n_local*T*C = %zu", count, (size_t)e->n_local * e->TC);
  CUDA_TRY(cudaSetDevice(e->desc.device));
  CUDA_TRY(cudaMemcpyAsync(e->noise.eps(), host_eps, count * sizeof(float), cudaMemcpyHostToDevice, e->stream));
  CUDA_TRY(cudaStreamSynchronize(e->stream));
  return MPPIB_OK;
}

int mppib_draw_noise(mppib_engine* e)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  int rc = e->noise.draw(e->noise.offset_t());
  if (rc != MPPIB_OK)
    return rc;
  CUDA_TRY(cudaStreamSynchronize(e->stream));
  return MPPIB_OK;
}

// K1, and for the smooth-MPPI sampler the nominal control its merge integrates onto
static int launch_k1(mppib_engine* e, const float* x0, const float* U_in, int optimization_stride, int iteration_num)
{
  if (e->noise.smooth())
    e->smooth_mu.assign(U_in, U_in + e->TC);
  return e->rollout.launch(*e, x0, U_in, optimization_stride, iteration_num);
}

// K2 (and its cross-rank or Tsallis stages) over the last K1's partials
static int enqueue_merge(mppib_engine* e, bool after_k1)
{
  static_assert(kSmoothMaxFloats == kMaxMeanFloats, "a smooth engine's T*C is bounded by the rollout's mean");
  if (e->noise.smooth())
    return e->reduction.enqueue_smooth(after_k1, e->lambda, e->noise.rate_mean(), e->noise.smooth_dt(),
                                       e->smooth_mu.data());
  return e->reduction.enqueue(after_k1, e->rollout.costs(), e->rollout.controls(), e->n_local, e->lambda);
}

int mppib_rollout_only(mppib_engine* e, const float* x0, const float* U_in, int optimization_stride, int iteration_num)
{
  int rc = check_ready(e);
  if (rc != MPPIB_OK)
    return rc;
  if (!x0 || !U_in)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  rc = launch_k1(e, x0, U_in, optimization_stride, iteration_num);
  if (rc != MPPIB_OK)
    return rc;
  CUDA_TRY(cudaStreamSynchronize(e->stream));
  e->solved_once = true;
  return MPPIB_OK;
}

int mppib_reduce_only(mppib_engine* e, float* U_out, mppib_solve_stats* stats)
{
  int rc = check_ready(e);
  if (rc != MPPIB_OK)
    return rc;
  if (!e->solved_once)
    return fail(MPPIB_ERR_STATE, "no rollout has been run yet");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  rc = enqueue_merge(e, false);
  if (rc != MPPIB_OK)
    return rc;
  CUDA_TRY(cudaStreamSynchronize(e->stream));
  e->reduction.read(U_out, stats);
  return MPPIB_OK;
}

// ---- stage timing (engine_internal.cuh) -------------------------------------------------------------------------------
cudaError_t StageTimer::create()
{
  for (Event& ev : ev_)
    if (cudaError_t rc = ev.create())
      return rc;
  return cudaSuccess;
}

void StageTimer::enable(bool on)
{
  on_ = on;
  for (double& s : sum_ms_)
    s = 0.0;
  n_ = 0;
}

void StageTimer::collect()
{
  if (!timed_ || !on_)
    return;
  timed_ = false;  // counted once
  float ms[4];
  if (cudaEventElapsedTime(&ms[0], ev_[0], ev_[1]) != cudaSuccess ||
      cudaEventElapsedTime(&ms[1], ev_[1], ev_[2]) != cudaSuccess ||
      cudaEventElapsedTime(&ms[2], ev_[2], ev_[3]) != cudaSuccess ||
      cudaEventElapsedTime(&ms[3], ev_[0], ev_[3]) != cudaSuccess)
  {
    cudaGetLastError();  // leave no error behind for the next launch's check
    return;
  }
  for (int i = 0; i < 4; i++)
    sum_ms_[i] += ms[i];
  n_++;
}

int StageTimer::read(mppib_timing* out) const
{
  if (n_ == 0)
    return fail(MPPIB_ERR_STATE, "timing not enabled or no synchronous solve since it was enabled");
  out->noise_ms = (float)(sum_ms_[0] / n_);
  out->rollout_ms = (float)(sum_ms_[1] / n_);
  out->reduce_ms = (float)(sum_ms_[2] / n_);
  out->total_ms = (float)(sum_ms_[3] / n_);
  out->samples = (int)n_;
  return MPPIB_OK;
}

static int enqueue_solve(mppib_engine* e, const float* x0, const float* U_in, int optimization_stride,
                         int iteration_num)
{
  CUDA_TRY(e->timer.start(e->stream));
  int rc = e->noise.draw(optimization_stride);
  if (rc != MPPIB_OK)
    return rc;
  CUDA_TRY(e->rollout.flush_l2());
  CUDA_TRY(e->timer.mark(1, e->stream));
  rc = launch_k1(e, x0, U_in, optimization_stride, iteration_num);
  if (rc != MPPIB_OK)
    return rc;
  rc = e->noise.prefetch();
  if (rc != MPPIB_OK)
    return rc;
  CUDA_TRY(e->timer.mark(2, e->stream));
  // a timed solve records an event between K1 and K2: no PDL then
  rc = enqueue_merge(e, /*after_k1=*/!e->timer.timed());
  if (rc != MPPIB_OK)
    return rc;
  CUDA_TRY(e->noise.read_by_kernel());  // K1 read it; recorded after K2, so nothing sits between K1 and PDL's K2
  CUDA_TRY(e->timer.mark(3, e->stream));
  e->pending++;
  return MPPIB_OK;
}

static int wait_solve(mppib_engine* e, float* U_out, mppib_solve_stats* stats)
{
  CUDA_TRY(cudaStreamSynchronize(e->stream));
  e->pending = 0;
  e->timer.collect();
  e->solved_once = true;
  e->reduction.read(U_out, stats);
  return MPPIB_OK;
}

int mppib_solve(mppib_engine* e, const float* x0, const float* U_in, int optimization_stride, int iteration_num,
                float* U_out, mppib_solve_stats* stats)
{
  int rc = check_ready(e);
  if (rc != MPPIB_OK)
    return rc;
  if (!x0 || !U_in || !U_out)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  rc = enqueue_solve(e, x0, U_in, optimization_stride, iteration_num);
  if (rc != MPPIB_OK)
    return rc;
  return wait_solve(e, U_out, stats);
}

// One iteration of Controller::computeControl (controllers/MPPI/mppi_controller.cu:151-241) as ONE call: the solve, then the
// host tail on its result with the parameter blobs the engine was given — smoothControlTrajectory (controller.cuh:557-586) and
// computeStateTrajectory (:643-663) through the library's host twins.
int mppib_compute_control(mppib_engine* e, const float* x0, float* U_inout, int optimization_stride, int iteration_num,
                          const float* control_history, float* states, float* outputs, mppib_solve_stats* stats)
{
  int rc = check_ready(e);
  if (rc != MPPIB_OK)
    return rc;
  if (!x0 || !U_inout || (states == nullptr) != (outputs == nullptr))
    return fail(MPPIB_ERR_INVALID_ARG, "null argument (states and outputs go together)");
  const int dyn = e->desc.dynamics_id;
  if (states && dyn >= MPPIB_USER_ID_BASE)
    return fail(MPPIB_ERR_UNSUPPORTED, "user dynamics have no host twin in the library: roll the state forward in the caller");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  rc = enqueue_solve(e, x0, U_inout, optimization_stride, iteration_num);
  if (rc != MPPIB_OK)
    return rc;
  rc = wait_solve(e, U_inout, stats);
  if (rc != MPPIB_OK)
    return rc;
  for (int d = 0; d < e->D; d++)
  {
    float* u = U_inout + (size_t)d * e->TC;
    if (control_history)
      mppib_host_smooth_controls(u, control_history, e->T, e->C);
    if (!states)
      continue;
    rc = e->model.host_roll(x0 + (size_t)d * e->S, u, e->T, e->dt, states + (size_t)d * e->T * e->S,
                            outputs + (size_t)d * e->T * e->O);
    if (rc != MPPIB_OK)
      return fail(rc, "host roll-forward failed for dynamics %d", dyn);
  }
  return MPPIB_OK;
}

int mppib_solve_async(mppib_engine* e, const float* x0, const float* U_in, int optimization_stride, int iteration_num)
{
  int rc = check_ready(e);
  if (rc != MPPIB_OK)
    return rc;
  if (!x0 || !U_in)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return enqueue_solve(e, x0, U_in, optimization_stride, iteration_num);
}

int mppib_solve_wait(mppib_engine* e, float* U_out, mppib_solve_stats* stats)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  if (e->pending == 0)
    return fail(MPPIB_ERR_STATE, "no solve in flight");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return wait_solve(e, U_out, stats);
}

int mppib_set_tsallis(mppib_engine* e, float gamma, float r)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  if (e->noise.smooth())
    return fail(MPPIB_ERR_UNSUPPORTED, "Tsallis weights are not built for the smooth-MPPI sampler");
  return e->reduction.set_tsallis(gamma, r, e->rollout.controls() != nullptr);
}

// ---- the feedback controller (feedback.cuh) ---------------------------------------------------------------------------
void Feedback::create(int S, int C, int T, cudaStream_t stream)
{
  S_ = S;
  C_ = C;
  T_ = T;
  stream_ = stream;
  Q_.assign((size_t)S * S, 0.0f);
  R_.assign((size_t)C * C, 0.0f);
  for (int i = 0; i < S; i++)
    Q_[(size_t)i * (S + 1)] = 1.0f;
  for (int i = 0; i < C; i++)
    R_[(size_t)i * (C + 1)] = 1.0f;
  Qf_ = Q_;
}

int Feedback::set_weights(const float* Q, const float* Q_f, const float* R, int iters)
{
  if (iters < 1)
    return fail(MPPIB_ERR_INVALID_ARG, "num_iterations must be >= 1 (got %d)", iters);
  for (int i = 0; i < S_ * S_; i++)
    if (!std::isfinite(Q[i]) || !std::isfinite(Q_f[i]))
      return fail(MPPIB_ERR_INVALID_ARG, "DDP weight Q / Q_f entry %d is not finite", i);
  for (int i = 0; i < C_ * C_; i++)
    if (!std::isfinite(R[i]))
      return fail(MPPIB_ERR_INVALID_ARG, "DDP weight R entry %d is not finite", i);
  Q_.assign(Q, Q + S_ * S_);
  Qf_.assign(Q_f, Q_f + S_ * S_);
  R_.assign(R, R + C_ * C_);
  iters_ = iters;
  return MPPIB_OK;
}

// The gains are read by the K1 of a solve still in flight, so they are freed only once the stream has drained; a new
// trajectory is copied in stream order, after that K1.
int Feedback::set_rmppi(float threshold, const float* host_gains)
{
  threshold_ = threshold;
  const size_t n = (size_t)T_ * S_ * C_;
  if (host_gains)
  {
    for (size_t i = 0; i < n; i++)
      if (!std::isfinite(host_gains[i]))
        return fail(MPPIB_ERR_INVALID_ARG, "feedback gain %zu is not finite", i);
    gains_set_ = false;  // the device copy changes from here on
    if (!gains_)
      CUDA_TRY(gains_.alloc(n));
    CUDA_TRY(cudaMemcpyAsync(gains_, host_gains, n * sizeof(float), cudaMemcpyHostToDevice, stream_));
    CUDA_TRY(cudaStreamSynchronize(stream_));
    gains_set_ = true;
  }
  else if (gains_)
  {
    gains_set_ = false;
    CUDA_TRY(cudaStreamSynchronize(stream_));
    gains_.reset();
  }
  return MPPIB_OK;
}

int Feedback::compute(mppib_engine& e, int T, const float* x0, const float* x_target, const float* u_target, bool to_rmppi,
                      float* gains, float* x_out, float* u_out, float* jac_out)
{
  const ddp::WsLayout L = ddp::ws_layout(T, S_, C_);
  CUDA_TRY(ws_.reserve(L.total, stream_));
  if (!status_)
    CUDA_TRY(status_.alloc(1));
  if (to_rmppi && !gains_)
    CUDA_TRY(gains_.alloc((size_t)T * S_ * C_));
  float* ws = ws_;
  CUDA_TRY(cudaMemcpyAsync(ws + L.xt, x_target, (size_t)T * S_ * sizeof(float), cudaMemcpyHostToDevice, stream_));
  CUDA_TRY(cudaMemcpyAsync(ws + L.ut, u_target, (size_t)T * C_ * sizeof(float), cudaMemcpyHostToDevice, stream_));
  // computeFeedback(x0, goal_traj, control_traj) starts DDP::run from control_traj, the control targets (ddp.cu:103-104)
  CUDA_TRY(cudaMemcpyAsync(ws + L.u, u_target, (size_t)T * C_ * sizeof(float), cudaMemcpyHostToDevice, stream_));
  if (int rc = e.rollout.pair().ddp(e, T, x0, to_rmppi ? gains_.get() : nullptr))
    return rc;
  int status = 0;
  CUDA_TRY(cudaMemcpyAsync(&status, status_, sizeof(int), cudaMemcpyDeviceToHost, stream_));
  CUDA_TRY(cudaStreamSynchronize(stream_));
  if (status != 0)
    return fail(MPPIB_ERR_INVALID_ARG, "DDP: the LDLT of Q_uu failed at step %d (the reference exits, ddp.h:112-116); "
                                       "gains left unchanged", status - 1);
  if (to_rmppi)
    gains_set_ = true;  // the kernel has written the whole trajectory
  if (gains)
    CUDA_TRY(cudaMemcpyAsync(gains, ws + L.K, (size_t)T * S_ * C_ * sizeof(float), cudaMemcpyDeviceToHost, stream_));
  if (x_out)
    CUDA_TRY(cudaMemcpyAsync(x_out, ws + L.x, (size_t)T * S_ * sizeof(float), cudaMemcpyDeviceToHost, stream_));
  if (u_out)
    CUDA_TRY(cudaMemcpyAsync(u_out, ws + L.u, (size_t)T * C_ * sizeof(float), cudaMemcpyDeviceToHost, stream_));
  if (jac_out)
    CUDA_TRY(cudaMemcpyAsync(jac_out, ws + L.jac, (size_t)T * S_ * (S_ + C_) * sizeof(float), cudaMemcpyDeviceToHost,
                             stream_));
  if (gains || x_out || u_out || jac_out)
    CUDA_TRY(cudaStreamSynchronize(stream_));
  return MPPIB_OK;
}

int mppib_set_rmppi(mppib_engine* e, float value_func_threshold, const float* feedback_gains)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  if (!e->rmppi)
    return fail(MPPIB_ERR_STATE, "engine was not created with MPPIB_FLAG_RMPPI");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->feedback.set_rmppi(value_func_threshold, feedback_gains);
}

int mppib_set_ddp(mppib_engine* e, const float* Q, const float* Q_f, const float* R, int num_iterations)
{
  if (!e || !Q || !Q_f || !R)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  return e->feedback.set_weights(Q, Q_f, R, num_iterations);
}

int mppib_ddp_feedback(mppib_engine* e, int T, const float* x0, const float* x_target, const float* u_target, int to_rmppi,
                       float* gains, float* x_out, float* u_out, float* jac_out)
{
  if (!e || !x0 || !x_target || !u_target)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  if (!e->rollout.pair().ddp)
    return fail(MPPIB_ERR_UNSUPPORTED, "dynamics %d has no analytic Jacobian (computeGrad): no DDP kernel is built for it",
                e->desc.dynamics_id);
  if (T < 2)
    return fail(MPPIB_ERR_INVALID_ARG, "DDP needs num_timesteps >= 2 (got %d)", T);
  if (to_rmppi && !e->rmppi)
    return fail(MPPIB_ERR_INVALID_ARG, "to_rmppi needs an engine created with MPPIB_FLAG_RMPPI");
  if (to_rmppi && T != e->T)
    return fail(MPPIB_ERR_INVALID_ARG, "to_rmppi needs T == the engine's horizon %d (got %d)", e->T, T);
  if (int rc = e->model.ready_for_ddp())
    return rc;
  if (e->pending != 0)
    return fail(MPPIB_ERR_STATE, "mppib_ddp_feedback while a solve is pending: call mppib_solve_wait first");
  const int S = e->S, C = e->C;
  for (int i = 0; i < S; i++)
    if (!std::isfinite(x0[i]))
      return fail(MPPIB_ERR_INVALID_ARG, "x0[%d] is not finite", i);
  for (size_t i = 0; i < (size_t)T * S; i++)
    if (!std::isfinite(x_target[i]))
      return fail(MPPIB_ERR_INVALID_ARG, "x_target entry %zu is not finite", i);
  for (size_t i = 0; i < (size_t)T * C; i++)
    if (!std::isfinite(u_target[i]))
      return fail(MPPIB_ERR_INVALID_ARG, "u_target entry %zu is not finite", i);
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->feedback.compute(*e, T, x0, x_target, u_target, to_rmppi != 0, gains, x_out, u_out, jac_out);
}

// ---- the side rollouts (side_rollouts.cuh) ----------------------------------------------------------------------------
int SideRollouts::init_eval(mppib_engine& e, const float* candidates, const int* strides, int K, int samples,
                            const float* U_nominal, int opt_stride, float* costs_out)
{
  const size_t total = (size_t)K * samples;
  CUDA_TRY(eval_states_.reserve((size_t)K * e.S, e.stream));
  CUDA_TRY(eval_strides_.reserve((size_t)K, e.stream));
  CUDA_TRY(eval_costs_.reserve(total, e.stream));
  CUDA_TRY(cudaMemcpyAsync(eval_states_, candidates, (size_t)K * e.S * sizeof(float), cudaMemcpyHostToDevice, e.stream));
  CUDA_TRY(cudaMemcpyAsync(eval_strides_, strides, (size_t)K * sizeof(int), cudaMemcpyHostToDevice, e.stream));
  if (int rc = e.noise.draw(opt_stride))  // sampler_->generateSamples(stride, 0, gen_) (:595)
    return rc;
  if (int rc = e.rollout.pair().init_eval(e, K, samples, U_nominal, opt_stride))
    return rc;
  CUDA_TRY(e.noise.read_by_kernel());  // the kernel above read the noise: later draws into its buffer wait for it
  CUDA_TRY(cudaMemcpyAsync(costs_out, eval_costs_, total * sizeof(float), cudaMemcpyDeviceToHost, e.stream));
  CUDA_TRY(cudaStreamSynchronize(e.stream));
  return MPPIB_OK;
}

int SideRollouts::sample(mppib_engine& e, const float* x0, const float* U_nominal, int distribution, const int* sample_idx,
                         int n, const float* U_opt, float* outputs, float* costs, int* crash)
{
  const size_t n_out = (size_t)n * e.T * e.O, n_cost = (size_t)n * (e.T + 1), n_crash = (size_t)n * e.T;
  CUDA_TRY(vis_idx_.reserve((size_t)n, e.stream));
  CUDA_TRY(vis_outputs_.reserve(n_out, e.stream));
  CUDA_TRY(vis_costs_.reserve(n_cost, e.stream));
  CUDA_TRY(vis_crash_.reserve(n_crash, e.stream));
  CUDA_TRY(cudaMemcpyAsync(vis_idx_, sample_idx, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, e.stream));
  have_opt_ = U_opt != nullptr;
  if (have_opt_)
  {
    CUDA_TRY(vis_opt_.reserve((size_t)e.TC, e.stream));
    CUDA_TRY(cudaMemcpyAsync(vis_opt_, U_opt, (size_t)e.TC * sizeof(float), cudaMemcpyHostToDevice, e.stream));
  }
  if (int rc = e.rollout.pair().sampled_traj(e, x0, U_nominal, distribution, n))
    return rc;
  CUDA_TRY(cudaMemcpyAsync(outputs, vis_outputs_, n_out * sizeof(float), cudaMemcpyDeviceToHost, e.stream));
  CUDA_TRY(cudaMemcpyAsync(costs, vis_costs_, n_cost * sizeof(float), cudaMemcpyDeviceToHost, e.stream));
  CUDA_TRY(cudaMemcpyAsync(crash, vis_crash_, n_crash * sizeof(int), cudaMemcpyDeviceToHost, e.stream));
  CUDA_TRY(cudaStreamSynchronize(e.stream));
  return MPPIB_OK;
}

int SideRollouts::nominal(mppib_engine& e, const float* x0, const float* U, const float* history, float* U_smoothed,
                          float* states, float* outputs)
{
  n_u_ = (size_t)e.D * e.TC;
  n_s_ = (size_t)e.D * e.T * e.S;
  const size_t n = n_u_ + n_s_ + (size_t)e.D * e.T * e.O;
  CUDA_TRY(nom_.reserve(n, e.stream));
  CUDA_TRY(nom_h_.reserve(n, cudaHostAllocDefault));
  nom_src_ = e.reduction.result() + kPartialHeader;  // the optimised sequence where K2 / KX left it
  nom_stride_ = e.reduction.pstride();
  if (U)
  {
    CUDA_TRY(nom_u_.reserve(n_u_, e.stream));
    CUDA_TRY(cudaMemcpyAsync(nom_u_, U, n_u_ * sizeof(float), cudaMemcpyHostToDevice, e.stream));
    nom_src_ = nom_u_;
    nom_stride_ = e.TC;
  }
  if (int rc = e.rollout.pair().nominal_traj(e, x0, history))
    return rc;
  CUDA_TRY(cudaMemcpyAsync(nom_h_, nom_, n * sizeof(float), cudaMemcpyDeviceToHost, e.stream));
  CUDA_TRY(cudaStreamSynchronize(e.stream));
  if (U_smoothed)
    memcpy(U_smoothed, nom_h_, n_u_ * sizeof(float));
  memcpy(states, nom_h_ + n_u_, n_s_ * sizeof(float));
  memcpy(outputs, nom_h_ + n_u_ + n_s_, (n - n_u_ - n_s_) * sizeof(float));
  return MPPIB_OK;
}

int mppib_init_eval(mppib_engine* e, const float* candidates, const int* strides, int num_candidates,
                    int samples_per_candidate, const float* U_nominal, int optimization_stride, float* costs_out)
{
  int rc = check_ready(e);
  if (rc != MPPIB_OK)
    return rc;
  if (!candidates || !strides || !U_nominal || !costs_out || num_candidates <= 0 || samples_per_candidate <= 0)
    return fail(MPPIB_ERR_INVALID_ARG, "bad argument");
  if (e->desc.world_size != 1)
    return fail(MPPIB_ERR_UNSUPPORTED, "init-eval runs on one rank (a few hundred rollouts)");
  if (e->noise.smooth())  // RMPPI's nominal-state search; the smooth sampler is built for one distribution
    return fail(MPPIB_ERR_UNSUPPORTED, "init-eval samples Gaussian controls; it is not built for the smooth-MPPI sampler");
  if (samples_per_candidate > e->n_local || (long)num_candidates * samples_per_candidate > e->N)
    return fail(MPPIB_ERR_INVALID_ARG, "(number of candidates) * (samples per candidate) cannot exceed NUM_ROLLOUTS");
  for (int k = 0; k < num_candidates; k++)
    if (strides[k] < 0)  // control min(t + stride, T - 1) of a row: a negative stride reads before the noise and the mean
      return fail(MPPIB_ERR_INVALID_ARG, "stride %d (candidate %d) is negative", strides[k], k);
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->side.init_eval(*e, candidates, strides, num_candidates, samples_per_candidate, U_nominal, optimization_stride,
                           costs_out);
}

int mppib_sample_trajectories(mppib_engine* e, const float* x0, const float* U_nominal, int distribution,
                              const int* sample_idx, int n, const float* U_opt, float* outputs, float* costs, int* crash)
{
  int rc = check_ready(e);
  if (rc != MPPIB_OK)
    return rc;
  if (!x0 || !U_nominal || !sample_idx || n <= 0 || !outputs || !costs || !crash)
    return fail(MPPIB_ERR_INVALID_ARG, "bad argument");
  if (distribution < 0 || distribution >= e->D)
    return fail(MPPIB_ERR_INVALID_ARG, "distribution %d out of range [0, %d)", distribution, e->D);
  if (!e->rollout.controls())
    return fail(MPPIB_ERR_STATE, "sampled trajectories re-roll the written-back controls: create the engine with "
                                 "MPPIB_FLAG_WRITEBACK_CONTROLS");
  if (e->rmppi)
    return fail(MPPIB_ERR_UNSUPPORTED, "sampled trajectories are built for the Vanilla / Tube / Colored rollouts");
  if (!e->solved_once)
    return fail(MPPIB_ERR_STATE, "no solve has been run yet");
  if (e->pending)
    return fail(MPPIB_ERR_STATE, "a solve is in flight (mppib_solve_wait first)");
  bool have_opt = false;
  for (int i = 0; i < n; i++)
  {
    if (sample_idx[i] < -1 || sample_idx[i] >= e->n_local)
      return fail(MPPIB_ERR_INVALID_ARG, "sample index %d (entry %d) outside [-1, %d)", sample_idx[i], i, e->n_local);
    have_opt = have_opt || sample_idx[i] < 0;
  }
  if (have_opt && !U_opt)
    return fail(MPPIB_ERR_INVALID_ARG, "index -1 needs U_opt");
  for (int i = 0; i < e->S; i++)
    if (!std::isfinite(x0[i]))
      return fail(MPPIB_ERR_INVALID_ARG, "x0[%d] is not finite", i);
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->side.sample(*e, x0, U_nominal, distribution, sample_idx, n, have_opt ? U_opt : nullptr, outputs, costs, crash);
}

// Device-side host tail (SURVEY §8 f2; controller.cuh:557-586, 643-663): see nominal_traj_kernel.
int mppib_nominal_trajectory(mppib_engine* e, const float* x0, const float* U, const float* control_history,
                             float* U_smoothed, float* states, float* outputs)
{
  int rc = check_ready(e);
  if (rc != MPPIB_OK)
    return rc;
  if (!x0 || !states || !outputs)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  if (!U && !e->solved_once && !e->pending)
    return fail(MPPIB_ERR_STATE, "U == NULL rolls out the last solve's result, and no solve has been run yet");
  if (e->T < 2)
    return fail(MPPIB_ERR_INVALID_ARG, "needs at least two time steps");
  for (int i = 0; i < e->D * e->S; i++)
    if (!std::isfinite(x0[i]))
      return fail(MPPIB_ERR_INVALID_ARG, "x0[%d] is not finite", i);
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->side.nominal(*e, x0, U, control_history, U_smoothed, states, outputs);
}

int mppib_set_option(mppib_engine* e, int option, long long value)
{
  if (e && option == MPPIB_OPT_P2P_ENABLE)
    return e->reduction.set_p2p(value != 0);
  if (e && option == MPPIB_OPT_COLORED_OFFSET_T)
    return e->noise.set_offset_t(value);
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  switch (option)
  {
    case MPPIB_OPT_L2_FLUSH_BYTES:
      return e->rollout.set_l2_flush(value);
  }
  return fail(MPPIB_ERR_INVALID_ARG, "unknown option %d", option);
}

int mppib_get_costs(mppib_engine* e, float* host_costs)
{
  if (!e || !host_costs)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->rollout.read_costs(host_costs);
}

int mppib_get_noise(mppib_engine* e, float* host_eps)
{
  if (!e || !host_eps)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  CUDA_TRY(cudaMemcpyAsync(host_eps, e->noise.eps(), (size_t)e->n_local * e->TC * sizeof(float), cudaMemcpyDeviceToHost,
                           e->stream));
  CUDA_TRY(cudaStreamSynchronize(e->stream));
  return MPPIB_OK;
}

int mppib_get_samples(mppib_engine* e, float* host_samples)
{
  if (!e || !host_samples)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->rollout.read_controls(host_samples);
}

int mppib_get_weights(mppib_engine* e, float* host_weights)
{
  if (!e || !host_weights)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  if (!e->solved_once)
    return fail(MPPIB_ERR_STATE, "no solve has been run yet");
  CUDA_TRY(cudaSetDevice(e->desc.device));
  return e->rollout.weights(host_weights, e->reduction.result(), e->reduction.pstride(), e->lambda);
}

int mppib_enable_timing(mppib_engine* e, int enable)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  e->timer.enable(enable != 0);
  return MPPIB_OK;
}

int mppib_get_timing(mppib_engine* e, mppib_timing* out)
{
  if (!e || !out)
    return fail(MPPIB_ERR_INVALID_ARG, "null argument");
  return e->timer.read(out);
}

int mppib_get_launch_info(mppib_engine* e, int* grid, int* block, int* smem_bytes, int* uses_tma,
                          int* kernels_per_solve)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  const K1Plan& k1 = e->rollout.plan();
  if (grid)
    *grid = k1.grid;
  if (block)
    *block = k1.threads;
  if (smem_bytes)
    *smem_bytes = (int)k1.smem_bytes;
  if (uses_tma)
    *uses_tma = k1.use_tma ? 1 : 0;
  if (kernels_per_solve)  // [K0] + K1 + K2 (+ K2'); cuRAND's own launches are not counted
    *kernels_per_solve = ((e->desc.world_size > 1) ? 3 : 2) + (e->noise.own_kernel() ? 1 : 0);
  return MPPIB_OK;
}

int mppib_get_rng_info(mppib_engine* e, int* own_kernel, int* chunks, int* rounds_per_chunk)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  if (own_kernel)
    *own_kernel = e->noise.own_kernel() ? 1 : 0;
  if (chunks)
    *chunks = e->noise.chunks();
  if (rounds_per_chunk)
    *rounds_per_chunk = e->noise.rounds_per_chunk();
  return MPPIB_OK;
}

int mppib_local_rollouts(mppib_engine* e, int* n_local, int* n_offset)
{
  if (!e)
    return fail(MPPIB_ERR_INVALID_ARG, "null engine");
  if (n_local)
    *n_local = e->n_local;
  if (n_offset)
    *n_offset = e->n_offset;
  return MPPIB_OK;
}

}  // extern "C"
