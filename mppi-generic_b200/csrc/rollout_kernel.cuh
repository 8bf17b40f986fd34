/*
 * rollout_kernel.cuh — K1, the fused per-sample rollout of the MPPI hot path, written for sm_90a.
 *
 * Replaces, in ONE kernel and one pass over the noise buffer:
 *   setGaussianControls           sampling_distributions/gaussian/gaussian.cu:17-277   (mean / sigma / special cases)
 *   rolloutKernel                 core/mppi_common.cu:28-146                           (read sample, constrain, step,
 *                                                                                       running cost + LR cost)
 *   rolloutDynamicsKernel + rolloutCostKernel   core/mppi_common.cu:148-362            (split variant; no y_d round trip)
 *   costArrayReduction / computeAndSaveCost     core/mppi_common.cu:843-853,1191-1254
 * and the per-block half of
 *   computeBaselineCost / normExpKernel / computeNormalizer / weightedReductionKernel
 *                                 core/mppi_common.cu:686-737,858-900,1055-1063,1115-1160
 * (each block emits its own min-cost baseline, exp-weights sum and exp-weighted control sum; K2 — combine_kernel.cuh —
 *  merges the block partials with the usual log-sum-exp rescale, exactly like the cross-GPU merge).
 *
 * Design:
 *   - one thread owns one sample (and all D systems of it: Tube-MPPI's actual + nominal share the noise draw,
 *     gaussian.cu:378-389, which gives every thread D independent dependency chains); state, output, control and the
 *     running cost live in registers. No blockDim.y lane cooperation => no barriers inside the T-step loop (the
 *     reference pays 4 barrier waits + 2 __syncthreads per step, mppi_common.cu:98-137).
 *   - the block's noise rows [BX samples][T*C floats] — one contiguous HBM range — are staged to shared memory by
 *     TMA (cp.async.bulk.tensor.2d, 128-byte swizzle, one mbarrier per 32-column slab so the first time steps can
 *     start while later slabs are still in flight). Threads read their row with conflict-free LDS.128.
 *   - the raw N(0,1) buffer is read exactly once from HBM and never rewritten: mean/sigma/special cases and the
 *     control constraints are applied on the fly, and the exp-weighted control sum is taken from the SAME shared
 *     tile in the epilogue. Algorithmic HBM traffic = N*T*C*4 bytes (SURVEY.md §8d).
 */
#pragma once
#include <type_traits>

#include "device_utils.cuh"
#include "../../include/mppi_b200/params.h"

namespace mppib
{
constexpr int kMaxStateDim = 32;
constexpr int kMaxMeanFloats = 2048;  // D*T*C carried in the kernel parameter bank
constexpr int kMaxChunks = 32;        // T*C <= 1024

// sampler quantities the kernel needs (gaussian.cuh:21-61), prepared on the host once per solve
struct SamplerArgs
{
  float std_dev[MPPIB_MAX_DISTRIBUTIONS][MPPIB_MAX_CONTROL_DIM];  // un-decayed (LR cost, gaussian.cu:489)
  float std_dev_decayed[MPPIB_MAX_DISTRIBUTIONS][MPPIB_MAX_CONTROL_DIM];  // * std_dev_decay^iter (gaussian.cu:423)
  float control_cost_coeff[MPPIB_MAX_CONTROL_DIM];
  float pure_noise_threshold;  // (1.0f - pure_noise_trajectories_percentage) * num_rollouts   (gaussian.cu:108)
};

template <class DYN, class COST>
struct RolloutArgs
{
  typename DYN::Params dyn;
  typename COST::Params cost;
  typename DYN::Aux dyn_aux;
  typename COST::Aux cost_aux;
  SamplerArgs samp;
  const float* eps;     // raw N(0,1) [n_local][T][C]
  float* costs;         // [D][n_local]
  float* partials;      // [gridDim.x][D][pstride]   V_b at [kPartialHeader..)
  float4* headers;      // [gridDim.x][D]  (beta_b, eta_b, sum w^2_b, 0): compact copy for K2's first pass
  float* controls_out;  // optional [D][n_local][T][C] (MPPIB_FLAG_WRITEBACK_CONTROLS), else nullptr
  int n_local;          // rollouts on this rank
  int n_offset;         // global index of local rollout 0 (rank * N / world)
  int T;
  int nchunks;  // ceil(T*C / 32)
  int pstride;  // floats per (block, distribution) partial record
  int opt_stride;
  int use_tma;
  int dyn_shared_floats;  // DYN::sharedFloats(model_dims, blockDim.x): theta_s size (run-time for the LSTM model)
  int ring;               // > 0: streaming variant, noise slabs cycle through `ring` shared-memory buffers
  int stream_readback;    // streaming variant, A/B switch: 1 = weighted sum from the written-back controls (round-1 form)
  // RMPPI (rollout_kernel<..., RMPPI = true>): distribution 0 = nominal system, 1 = real system
  const float* fb_gains;       // DDP feedback gains [T][S][C] (column-major C x S per step) or nullptr (no feedback)
  float value_func_threshold;  // robust_mppi_controller.cuh: value_function_threshold_
  float dt, lambda, alpha, lambda_inv;
  float x0[MPPIB_MAX_DISTRIBUTIONS * kMaxStateDim];  // [D][S]
  float means[kMaxMeanFloats];                       // [D][T][C] importance-sampler mean == nominal control
};

// The smooth-MPPI sampler's K1 (SmoothMPPIDistribution, smooth-MPPI.cu): the Gaussian arguments, then the engine-held rate
// mean and the sampler's own dt. A kernel of its own type, so that the Gaussian kernels' parameter block stays as it is.
template <class DYN, class COST>
struct SmoothRolloutArgs : RolloutArgs<DYN, COST>
{
  const float* rate_mean;  // [T][C] dmu, written by the previous solve's merge (stream order)
  float dt_s;              // SmoothMPPIParams::dt (smooth-MPPI.cuh:21), not the controller's dt
};

// gaussian.cu:101-121: the three cases of setGaussianControls for one element
// Branch-free: x + (-0.0f) == x for every float (including both zeros), so the pure-noise case sd * eps is the same FFMA with
// the addend -0.0f, and the three cases become two selects instead of two divergent-branch regions per control and step.
__device__ __forceinline__ float sample_control(float mean, float sd, float eps, bool use_mean, bool pure_noise)
{
  const float v = fmaf(sd, eps, pure_noise ? -0.0f : mean);  // nvcc contracts the reference's `mean + std_dev * eps` to this FFMA
  return use_mean ? mean : v;
}

// element i (0..3) of a 16-byte group without forcing it into local memory when i is not a compile-time constant
__device__ __forceinline__ float group_elem(const float4& v, int i)
{
  return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w));
}

// gaussian.cu:481-569 (device formula): 0.5*lambda*(1-alpha) * sum_i k_i * mean_i * (mean_i - 2 u_i) / sigma_i^2, mean = 0
// for the pure-noise tail. k_i / sigma_i^2 is loop-invariant and hoisted (lr_scale), which moves one rounding.
template <int C>
__device__ __forceinline__ float likelihood_ratio_cost(const float* lr_scale, const float* mean_t, const float* u,
                                                       bool pure_noise, float half_lambda_1ma)
{
  float cost = 0.0f;
#pragma unroll
  for (int i = 0; i < C; i++)
  {
    const float mean_i = pure_noise ? 0.0f : mean_t[i];
    cost += lr_scale[i] * mean_i * (mean_i - 2.0f * u[i]);
  }
  return half_lambda_1ma * cost;
}

// The block epilogue's exp-weighted sum of the constrained controls of step t (weightedReductionKernel, mppi_common.cu:710-737)
// over the block's rows [r_lo, r_hi), added to acc in row order. The value of a row comes from the shared tile (`slab` = the
// step's column in its slab, `grp` its 16-byte group) or, from_global, from gsrc ([n_local][T][C]); `recompute`: that value is
// noise and the constrained control is formed from it as the rollout did. Rows in blocks of 8 (r_lo a multiple of 8): the
// swizzle term (grp ^ (r & 7)) << 4 is then a per-lane constant of the unrolled body. The loads of a block are issued first and
// unconditionally (rows past r_hi are clamped and get weight 0), so eight loads are in flight per thread instead of one
// load-use round trip per row — when they read L2 / HBM a serialised loop would expose one memory latency per row.
// RATES (smooth-MPPI): the recomputed value is the sampled rate with mean_t = the rate mean, and it is not constrained — the
// rate mean is the weighted average of the unconstrained rates (smooth-MPPI.cu:215-219).
template <class DYN, class ARGS, bool RATES = false>
__device__ __forceinline__ void weighted_control_rows(const ARGS& args, int d, int t, int row0, int r_lo, int r_hi,
                                                      const unsigned char* slab, int grp, const float* mean_t,
                                                      bool t_uses_mean, const float* wrow, bool from_global,
                                                      const float* gsrc, bool recompute, float* acc)
{
  constexpr int C = DYN::CONTROL_DIM;
  const int T = args.T;
  for (int r8 = r_lo; r8 < r_hi; r8 += 8)
  {
    float v[8][C];
#pragma unroll
    for (int i = 0; i < 8; i++)
    {
      const int r = min(r8 + i, r_hi - 1);
      if (from_global)
      {
        const float* q = gsrc + ((size_t)(row0 + r) * T + t) * C;
#pragma unroll
        for (int c = 0; c < C; c++)
          v[i][c] = __ldg(q + c);
      }
      else
      {
        const float* p = reinterpret_cast<const float*>(slab + r * kChunkBytes + ((grp ^ (r & 7)) << 4));
#pragma unroll
        for (int c = 0; c < C; c++)
          v[i][c] = p[c];
      }
    }
#pragma unroll
    for (int i = 0; i < 8; i++)
    {
      const int r = r8 + i;
      float u[C];
#pragma unroll
      for (int c = 0; c < C; c++)
        u[c] = v[i][c];
      if (recompute)
      {
        const int ng = args.n_offset + row0 + min(r, r_hi - 1);
        const bool pn = (float)ng >= args.samp.pure_noise_threshold;
        const bool um = t_uses_mean || (ng == 0);
#pragma unroll
        for (int c = 0; c < C; c++)
          u[c] = sample_control(mean_t[c], args.samp.std_dev_decayed[d][c], v[i][c], um, pn);
        if (!RATES)
          DYN::enforceConstraints(args.dyn, nullptr, u);
      }
      const float w = (r < r_hi) ? wrow[r] : 0.0f;
#pragma unroll
      for (int c = 0; c < C; c++)
        acc[c] = fmaf(w, u[c], acc[c]);
    }
  }
}

// shared-memory carve-up (bytes); the tile base is rounded up to 1024 B inside the kernel (SWIZZLE_128B atom)
struct RolloutSmem
{
  uint32_t tile, means, theta, theta_c, weights, scratch, bars, total;
};
// tile_chunks = nchunks for the resident whole-horizon tile, = the ring depth for the streaming variant
__host__ __device__ inline RolloutSmem rollout_smem_layout(int bx, int tile_chunks, int D, int TC, int dyn_shared_floats,
                                                           int cost_shared_floats)
{
  RolloutSmem s;
  uint32_t off = 0;
  s.tile = off;
  off += (uint32_t)tile_chunks * bx * kChunkBytes;
  s.means = off;
  off += ((uint32_t)(D * TC + 3) / 4) * 16;
  s.theta = off;
  off += ((uint32_t)(dyn_shared_floats + 3) / 4) * 16;
  s.theta_c = off;
  off += ((uint32_t)(cost_shared_floats + 3) / 4) * 16;
  s.weights = off;
  off += ((uint32_t)(D * bx + 3) / 4) * 16;
  s.scratch = off;
  off += 3 * 32 * 4;  // per-warp partials for (min | sum w | sum w^2)
  s.bars = off;
  off += (uint32_t)kMaxChunks * 8;
  s.total = off + 1024;  // slack for the 1024-B round-up of the base
  return s;
}

// SPT = samples per thread. 1 everywhere except for models whose step re-reads block-shared weights (the NN): there a
// second sample in the same thread reuses every weight row it loads, which halves the shared-memory wavefronts per
// sample — the busiest unit of that kernel (DESIGN.md §3) — and gives the in-order
// issue two independent dependency chains to interleave. Thread `thr` owns tile rows thr + sp * blockDim.x.
//
// RMPPI = true (D == 2, WRITEBACK): the fused form of rolloutRMPPIKernel, core/rmppi_kernels.cu:665-866 — the real system
// (d = 1) adds the feedback K_t (x_real - x_nominal) to its sampled control before the constraints; the real cost takes
// running + likelihood-ratio cost, its tracking cost running + feedback cost (gaussian.cu:572-629); the nominal cost is
// 0.5 c_nom + 0.5 max(min(tracking_real, value_func_threshold), c_nom) + its likelihood-ratio cost. The real system's
// applied control depends on the state, so the block's weighted average reads it back from the write-back buffer.
//
// STREAM = true (TMA): the noise does not stay resident. Its 32-column slabs cycle through a small ring of shared-memory
// buffers (TMA refills a buffer as soon as every thread is done with it) and the block's weighted average, which needs every
// control of the horizon once the weights are known, recomputes them from a SECOND read of the block's noise rows instead of writing the controls to HBM and reading them
// back. The re-read follows the block's first read by one horizon and may partly hit L2, but it pays without that: at
// worst it is one more read of the block's noise (C5's whole buffer, 78.6 MB, is larger than H100's 50 MB L2), against a
// write plus a read of the same number of control bytes. Shared memory per sample drops from T*C*4 bytes to ring*128, so long horizons no longer cap the
// block count per SM — the resident tile of C5 (T*C = 300) allows 4 warps per SM and several waves, the ring 12+ warps and one.
//
// ARGS = SmoothRolloutArgs (rollout_kernel_smooth): the smooth-MPPI sampler. Each element's rate v is sampled around the rate
// mean as the Gaussian sampler samples a control (the three cases of sample_control), the control is u = mu + v dt_s, and the
// epilogue's weighted sum takes the unconstrained rates, recomputed from the noise, which the tile therefore keeps.
template <class DYN, class COST, int D, bool WRITEBACK, int SPT, bool RMPPI, bool STREAM, class ARGS>
__device__ __forceinline__ void rollout_body(const ARGS& args, const CUtensorMap& tmap)
{
  constexpr bool SMOOTH = !std::is_same<ARGS, RolloutArgs<DYN, COST>>::value;
  static_assert(!SMOOTH || (D == 1 && !RMPPI), "smooth-MPPI is built for one distribution");
  constexpr int S = DYN::STATE_DIM, C = DYN::CONTROL_DIM, O = DYN::OUTPUT_DIM;
  static_assert(C == 1 || C == 2 || C == 4, "CONTROL_DIM must divide a 16-byte group");
  static_assert(D <= MPPIB_MAX_DISTRIBUTIONS, "too many distributions");
  static_assert(SPT == 1 || D == 1, "several samples per thread are built for one distribution");
  static_assert(!RMPPI || (D == 2 && WRITEBACK && SPT == 1), "RMPPI: two systems, controls kept in HBM");
  static_assert(!STREAM || (SPT == 1 && !RMPPI), "streaming variant: one sample per thread, no feedback");
  constexpr int STEPS_PER_GROUP = 4 / C;
  constexpr int M = SPT * D;  // systems rolled out by one thread: member m = sp * D + d

  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);

  // SPW = samples per warp (DYN::SAMPLES_PER_WARP). 32: lane l owns tile row (warp * 32 + l). Fewer (models whose step is
  // warp-collective, plugins/nn_mma.cuh): lanes l, l + SPW, ... carry the same row and compute the same values; the first
  // of them (`owner`) alone stores the cost and contributes to the block's sums.
  constexpr int SPW = DYN::SAMPLES_PER_WARP;
  static_assert(SPW == 32 || SPT == 1, "sub-warp sample groups are built for one sample per thread");
  const int nthr = blockDim.x;
  const int bx = (SPW == 32) ? nthr * SPT : (nthr >> 5) * SPW;  // samples (tile rows) per block
  const int thr = threadIdx.x;
  const bool owner = (SPW == 32) || ((thr & 31) < SPW);
  const int T = args.T;
  const int TC = T * C;
  const int nchunks = args.nchunks;
  const int ring = STREAM ? args.ring : nchunks;
  const RolloutSmem L = rollout_smem_layout(bx, ring, D, TC, args.dyn_shared_floats, COST::sharedFloats(T));
  unsigned char* tile = smem + L.tile;
  float* means_s = reinterpret_cast<float*>(smem + L.means);
  float* theta_s = reinterpret_cast<float*>(smem + L.theta);
  float* theta_c = reinterpret_cast<float*>(smem + L.theta_c);
  float* w_s = reinterpret_cast<float*>(smem + L.weights);
  float* red_s = reinterpret_cast<float*>(smem + L.scratch);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bars);

  pdl_launch_dependents();           // K2 may be scheduled now; it waits for this grid to finish before reading
  const int row0 = blockIdx.x * bx;  // first local rollout of this block
  int row[SPT], n_loc[SPT];
  bool valid[SPT], pure_noise[SPT], zero_noise_sample[SPT];
#pragma unroll
  for (int sp = 0; sp < SPT; sp++)
  {
    row[sp] = (SPW == 32) ? thr + sp * nthr : (thr >> 5) * SPW + (thr & (SPW - 1));
    n_loc[sp] = row0 + row[sp];
    valid[sp] = owner && n_loc[sp] < args.n_local;
    const int n_glob = args.n_offset + n_loc[sp];
    int pn = (float)n_glob >= args.samp.pure_noise_threshold;  // gaussian.cu:108, :505
    int zn = (n_glob == 0);                                    // gaussian.cu:101
    pure_noise[sp] = pn != 0;
    zero_noise_sample[sp] = zn != 0;
  }

  // ---- stage the block's noise rows -------------------------------------------------------------------------------
  if (args.use_tma)
  {
    if (thr == 0)
    {
      tma_prefetch_desc(&tmap);
      for (int k = 0; k < nchunks && k < ring; k++)
        mbar_init(&bars[k], 1);
      fence_barrier_init();
    }
    __syncthreads();
    if (thr == 0)
    {
      for (int k = 0; k < nchunks && k < ring; k++)
      {
        mbar_arrive_expect_tx(&bars[k], (uint32_t)bx * kChunkBytes);
        tma_load_2d(tile + (size_t)k * bx * kChunkBytes, &tmap, k * kChunkFloats, row0, &bars[k]);
      }
    }
  }
  else
  {
    // plain-load fallback (T*C not a multiple of 4, or MPPIB_FLAG_NO_TMA): coalesced LDG of the contiguous block
    // range, scattered into the same swizzled layout; out-of-range elements are zero like TMA's OOB fill.
    const float* src = args.eps + (size_t)row0 * TC;
    const int rows_here = min(bx, args.n_local - row0);
    const int total = bx * nchunks * kChunkFloats;
    for (int i = thr; i < total; i += nthr)
    {
      const int r = i / (nchunks * kChunkFloats);
      const int col = i - r * (nchunks * kChunkFloats);
      float v = 0.0f;
      if (r < rows_here && col < TC)
        v = __ldg(src + (size_t)r * TC + col);
      const int chunk = col >> 5, within = col & 31;
      *reinterpret_cast<float*>(tile + tile_offset_bytes(bx, chunk, r, within >> 2) + ((within & 3) << 2)) = v;
    }
  }

  // ---- block-shared read-only data --------------------------------------------------------------------------------
  for (int i = thr; i < D * TC; i += nthr)
    means_s[i] = args.means[i];

  // ---- per-sample state in registers ------------------------------------------------------------------------------
  float x[M][S], y[M][O], running_cost[M], extra_cost[M];
  int crash_status[M];
#pragma unroll
  for (int m = 0; m < M; m++)
  {
#pragma unroll
    for (int i = 0; i < S; i++)
      x[m][i] = args.x0[(m % D) * S + i];
#pragma unroll
    for (int i = 0; i < O; i++)
      y[m][i] = 0.0f;
    running_cost[m] = 0.0f;
    extra_cost[m] = 0.0f;
    crash_status[m] = 0;
  }
  // initializeDynamics fills theta_s cooperatively (FNNHelper::initialize) and seeds y; initializeCosts fills theta_c
  // (mppi_common.cu:94-96)
  typename DYN::Carry carry[M];
#pragma unroll
  for (int m = 0; m < M; m++)
  {
    DYN::initializeDynamics(args.dyn, args.dyn_aux, theta_s, carry[m], x[m], y[m]);
  }
  COST::initializeCosts(args.cost, args.cost_aux, theta_c, T);
  __syncthreads();

  // likelihood-ratio term: skipped altogether when every control_cost_coeff is zero (the sampler's default)
  float lr_scale[D][C];
  bool lr_on = false;
#pragma unroll
  for (int d = 0; d < D; d++)
#pragma unroll
    for (int c = 0; c < C; c++)
    {
      lr_scale[d][c] = args.samp.control_cost_coeff[c] / (args.samp.std_dev[d][c] * args.samp.std_dev[d][c]);
      lr_on = lr_on || (args.samp.control_cost_coeff[c] != 0.0f);
    }
  float half_lambda_1ma = 0.5f * args.lambda * (1.0f - args.alpha);

  // ---- the horizon ----------------------------------------------------------------------------------------------
  // One loop over the horizon's 16-byte noise groups (4 / C steps each); slab k = groups 8k .. 8k+7. Everything a step
  // needs that does not change along the horizon — the row's byte offset and swizzle key, the decayed sigmas, the special
  // sample flags — is computed here once and pinned in registers (the optimiser otherwise re-derives the shared-memory
  // carve-up and re-reads the parameter bank every step: ~70 of the NN kernel's ~690 instructions per step).
  uint32_t row_off[SPT], swz[SPT];
#pragma unroll
  for (int sp = 0; sp < SPT; sp++)
  {
    row_off[sp] = (uint32_t)row[sp] * kChunkBytes;
    swz[sp] = (uint32_t)row[sp] & 7u;
  }
  float sd_dec[D][C];
#pragma unroll
  for (int d = 0; d < D; d++)
#pragma unroll
    for (int c = 0; c < C; c++)
    {
      sd_dec[d][c] = args.samp.std_dev_decayed[d][c];
    }
  const int opt_stride = args.opt_stride;
  // smooth-MPPI: the shift (shiftControlTrajectory, smooth-MPPI.cu:34-78) reads row min(t + s, s) in place, in t order, so
  // every step samples around the previous rate mean's row s; a stride past the horizon takes the last row
  float dmu[C], dt_s = 0.0f;
  if constexpr (SMOOTH)
  {
    const int r = max(0, min(opt_stride, T - 1));
#pragma unroll
    for (int c = 0; c < C; c++)
      dmu[c] = args.rate_mean[r * C + c];
    dt_s = args.dt_s;
  }
  const int ngroups = (TC + 3) >> 2;
  const uint32_t slab_bytes = (uint32_t)bx * kChunkBytes;
  unsigned char* slab = tile;
  int slot = 0;
#pragma unroll 1
  for (int gi = 0; gi < ngroups; gi++)
  {
    const int k = gi >> 3, g = gi & 7;
    if (g == 0)
    {
      slot = STREAM ? (k % ring) : k;  // buffer that holds slab k
      if (args.use_tma)
        mbar_wait(&bars[slot], STREAM ? ((k / ring) & 1) : 0);
      slab = tile + (size_t)slot * slab_bytes;
    }
    unsigned char* gp[SPT];
    float4 e4[SPT];
#pragma unroll
    for (int sp = 0; sp < SPT; sp++)
    {
      gp[sp] = slab + row_off[sp] + (((uint32_t)g ^ swz[sp]) << 4);
      e4[sp] = *reinterpret_cast<const float4*>(gp[sp]);
    }
    // light models: the 4/C steps of a 16-byte group are unrolled; heavy ones (NN) keep one copy of the step body
#pragma unroll(DYN::UNROLL_STEPS ? STEPS_PER_GROUP : 1)
    for (int s = 0; s < STEPS_PER_GROUP; s++)
    {
      const int t = gi * STEPS_PER_GROUP + s;
      if (t >= T)
        break;
      float u[M][C], x_next[M][S], xdot[M][S], ufb[C];
#pragma unroll
      for (int m = 0; m < M; m++)
      {
        const int sp = m / D, d = m % D;
        const bool use_mean = zero_noise_sample[sp] || (t < opt_stride);
        const float* mean_t = means_s + (d * T + t) * C;
#pragma unroll
        for (int c = 0; c < C; c++)
        {
          if constexpr (SMOOTH)  // integrateNoise (smooth-MPPI.cu:16-32): a pure-noise row keeps mu too
            u[m][c] = fmaf(sample_control(dmu[c], sd_dec[d][c], group_elem(e4[sp], s * C + c), use_mean, pure_noise[sp]),
                           dt_s, mean_t[c]);
          else
            u[m][c] = sample_control(mean_t[c], sd_dec[d][c], group_elem(e4[sp], s * C + c), use_mean, pure_noise[sp]);
        }
        if (RMPPI && m == 1)
        {  // fb_controller->k(x, x_nom, t) (rmppi_kernels.cu:770-784; DDP: K_t e, ddp.cu:11-45 in its host form)
#pragma unroll
          for (int c = 0; c < C; c++)
            ufb[c] = 0.0f;
          if (args.fb_gains != nullptr)
          {
            const float* Kt = args.fb_gains + (size_t)t * S * C;
#pragma unroll
            for (int i = 0; i < S; i++)
            {
              const float e = x[1][i] - x[0][i];
#pragma unroll
              for (int c = 0; c < C; c++)
                ufb[c] = fmaf(__ldg(Kt + i * C + c), e, ufb[c]);
            }
          }
#pragma unroll
          for (int c = 0; c < C; c++)
            u[m][c] += ufb[c];
        }
        DYN::enforceConstraints(args.dyn, x[m], u[m]);  // mppi_common.cu:108-111
        if (D == 1 && !STREAM && !SMOOTH)
        {
          // single system: the constrained control replaces the noise in the shared tile (what writeControlSample does
          // in HBM, mppi_common.cu:117), so the epilogue's weighted sum reads it back instead of recomputing it
#pragma unroll
          for (int c = 0; c < C; c++)
            reinterpret_cast<float*>(gp[sp])[s * C + c] = u[m][c];
        }
        if (WRITEBACK)
        {  // compat / debug path: keep the constrained samples in HBM like the reference
          if (valid[sp])
          {
            float* dst = args.controls_out + (((size_t)d * args.n_local + n_loc[sp]) * T + t) * C;
#pragma unroll
            for (int c = 0; c < C; c++)
              dst[c] = u[m][c];
          }
        }
#pragma unroll
        for (int i = 0; i < S; i++)
          xdot[m][i] = 0.0f;
      }
      DYN::template stepBatch<M>(args.dyn, args.dyn_aux, theta_s, carry, x, x_next, xdot, u, y, t, args.dt);  // mppi_common.cu:120
#pragma unroll
      for (int m = 0; m < M; m++)
      {
        const int sp = m / D, d = m % D;
        float step_cost = COST::computeRunningCost(args.cost, args.cost_aux, theta_c, y[m], u[m], t, &crash_status[m]);
        float lr_cost = 0.0f;
        if (lr_on)
          lr_cost = likelihood_ratio_cost<C>(lr_scale[d], means_s + (d * T + t) * C, u[m], pure_noise[sp],
                                             half_lambda_1ma);  // :126-128
        if (!RMPPI)
          running_cost[m] += step_cost + lr_cost;
        else if (m == 0)
        {  // nominal system: rmppi_kernels.cu:806-811
          running_cost[m] += step_cost;
          extra_cost[m] += lr_cost;
        }
        else
        {  // real system: :813-819; computeFeedbackCost = 0.5 lambda (1 - alpha) sum_i k_i u_fb,i^2 / sigma_i^2
          running_cost[m] += step_cost + lr_cost;
          float fb_cost = 0.0f;
#pragma unroll
          for (int c = 0; c < C; c++)
            fb_cost += lr_scale[d][c] * (ufb[c] * ufb[c]);
          extra_cost[m] += step_cost + half_lambda_1ma * fb_cost;
        }
#pragma unroll
        for (int i = 0; i < S; i++)
          x[m][i] = x_next[m][i];
      }
    }
    if (STREAM && (g == 7 || gi == ngroups - 1))
    {
      __syncthreads();  // every thread is done with this slab's buffer
      if (thr == 0 && k + ring < nchunks)
      {
        mbar_arrive_expect_tx(&bars[slot], (uint32_t)bx * kChunkBytes);
        tma_load_2d(tile + (size_t)slot * bx * kChunkBytes, &tmap, (k + ring) * kChunkFloats, row0, &bars[slot]);
      }
    }
  }

  // ---- per-sample cost (computeAndSaveCost, mppi_common.cu:843-853) ------------------------------------------------
  float cost[M];
#pragma unroll
  for (int m = 0; m < M; m++)
    cost[m] = running_cost[m] / (float)T + COST::terminalCost(args.cost, args.cost_aux, y[m]) / (float)T;
  if (RMPPI)
  {  // rmppi_kernels.cu:836-858
    const float term_nom = COST::terminalCost(args.cost, args.cost_aux, y[0]);
    const float term_real = COST::terminalCost(args.cost, args.cost_aux, y[M - 1]);
    const float c_real = (running_cost[M - 1] + term_real) / (float)T;
    const float tracking_real = (extra_cost[M - 1] + term_real) / (float)T;
    float c_nom = (running_cost[0] + term_nom) / (float)T;
    const float tracking_nom = extra_cost[0] / (float)T;
    c_nom = 0.5f * c_nom + 0.5f * fmaxf(fminf(tracking_real, args.value_func_threshold), c_nom);
    c_nom += tracking_nom;
    cost[0] = c_nom;
    cost[M - 1] = c_real;
  }
#pragma unroll
  for (int m = 0; m < M; m++)
  {
    const int sp = m / D, d = m % D;
    if (valid[sp])
      args.costs[(size_t)d * args.n_local + n_loc[sp]] = cost[m];
  }
  if (RMPPI || (STREAM && WRITEBACK))
    __threadfence_block();  // the epilogue reads other threads' written-back controls

  // ---- block partial of the softmin-weighted control average ------------------------------------------------------
  const int lane = thr & 31, warp = thr >> 5, nwarps = (nthr + 31) >> 5;
#pragma unroll
  for (int d = 0; d < D; d++)
  {
    // block baseline
    float mn = INFINITY;
#pragma unroll
    for (int sp = 0; sp < SPT; sp++)
      mn = fminf(mn, valid[sp] ? cost[sp * D + d] : INFINITY);
    float m = warp_min(mn);
    if (lane == 0)
      red_s[warp] = m;
    __syncthreads();
    float beta_b = red_s[0];
    for (int i = 1; i < nwarps; i++)
      beta_b = fminf(beta_b, red_s[i]);
    // normExpTransform (mppi_common.cu:958-966) against the block baseline
    float wsum = 0.0f, w2sum = 0.0f;
#pragma unroll
    for (int sp = 0; sp < SPT; sp++)
    {
      const float w = valid[sp] ? softmin_weight(cost[sp * D + d], beta_b, args.lambda_inv) : 0.0f;
      if (owner)
        w_s[d * bx + row[sp]] = w;
      wsum += w;
      w2sum += w * w;
    }
    const float sw = warp_sum(wsum), sw2 = warp_sum(w2sum);
    if (lane == 0)
    {
      red_s[32 + warp] = sw;
      red_s[64 + warp] = sw2;
    }
    __syncthreads();
    if (thr == 0)
    {
      float eta_b = 0.0f, w2_b = 0.0f;
      for (int i = 0; i < nwarps; i++)
      {
        eta_b += red_s[32 + i];
        w2_b += red_s[64 + i];
      }
      args.headers[(size_t)blockIdx.x * D + d] = make_float4(beta_b, eta_b, w2_b, 0.0f);
    }
    __syncthreads();  // red_s reused by the next distribution
  }

  // exp-weighted sum of the CONSTRAINED sampled controls (weightedReductionKernel, mppi_common.cu:710-737), taken
  // from the shared tile: thread j owns time step j (all C components so enforceConstraints sees the full u).
  // D == 1: the tile already holds the constrained controls. D == 2: the tile still holds the shared noise and each
  // system's control is recomputed from it (RMPPI's real system: read back, see above).
  const int rows_here = min(bx, args.n_local - row0);
#pragma unroll
  for (int d = 0; d < D; d++)
  {
    float* out = args.partials + ((size_t)blockIdx.x * D + d) * args.pstride + kPartialHeader;
    for (int t = thr; t < T; t += nthr)
    {
      float acc[C];
#pragma unroll
      for (int c = 0; c < C; c++)
        acc[c] = 0.0f;
      const float* mean_t = means_s + (d * T + t) * C;
      const int col = t * C;
      const int chunk = col >> 5, within = col & 31, grp = within >> 2;
      const bool t_uses_mean = t < args.opt_stride;
      const unsigned char* slab = tile + (size_t)chunk * bx * kChunkBytes + ((within & 3) << 2);
      const float* wrow = w_s + d * bx;
      // rows in blocks of 8: the swizzle term (grp ^ (r & 7)) << 4 is then a per-lane constant of the unrolled body. The
      // loads of a block are issued first and unconditionally (rows past the end are clamped and get weight 0), so eight
      // loads are in flight per thread instead of one load-use round trip per row — this loop reads L2 / HBM in the streaming
      // and RMPPI forms, where a serialised loop would expose one memory latency per row.
      const bool from_global = (RMPPI && d == 1) || STREAM;
      const bool readback = !SMOOTH && ((RMPPI && d == 1) || (STREAM && WRITEBACK && args.stream_readback));
      const float* gsrc = readback ? args.controls_out + (size_t)d * args.n_local * T * C : args.eps;
      // the value is noise unless it comes from the constrained tile or the written-back controls: recompute the constrained
      // control (resident tile with D == 2, or the streaming variant, whose ring no longer holds it: a second read of eps
      // instead of a write + read of u)
      if constexpr (SMOOTH)  // the rates, around the rate mean, from the noise
        weighted_control_rows<DYN, ARGS, true>(args, d, t, row0, 0, rows_here, slab, grp, dmu, t_uses_mean, wrow,
                                               from_global, gsrc, true, acc);
      else
        weighted_control_rows<DYN>(args, d, t, row0, 0, rows_here, slab, grp, mean_t, t_uses_mean, wrow, from_global, gsrc,
                                   !(D == 1 && !STREAM) && !readback, acc);
#pragma unroll
      for (int c = 0; c < C; c++)
        out[col + c] = acc[c];
    }
  }
}

template <class DYN, class COST, int D, bool WRITEBACK, int SPT, bool RMPPI = false, bool STREAM = false>
__global__ void __launch_bounds__(DYN::MAX_BLOCK_THREADS) rollout_kernel(const __grid_constant__ RolloutArgs<DYN, COST> args,
                                                      const __grid_constant__ CUtensorMap tmap)
{
  rollout_body<DYN, COST, D, WRITEBACK, SPT, RMPPI, STREAM>(args, tmap);
}

// the smooth-MPPI sampler's K1: one distribution, resident or streaming, one or two samples per thread
template <class DYN, class COST, bool WRITEBACK, int SPT, bool STREAM = false>
__global__ void __launch_bounds__(DYN::MAX_BLOCK_THREADS)
    rollout_kernel_smooth(const __grid_constant__ SmoothRolloutArgs<DYN, COST> args, const __grid_constant__ CUtensorMap tmap)
{
  rollout_body<DYN, COST, 1, WRITEBACK, SPT, false, STREAM>(args, tmap);
}

}  // namespace mppib
