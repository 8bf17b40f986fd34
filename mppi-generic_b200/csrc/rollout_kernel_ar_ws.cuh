/*
 * rollout_kernel_ar_ws.cuh — K1 for the Autorally pair (NeuralNetModel<7,2,3> + ARStandardCost), warp-specialised.
 * Templated on the map cost: ARRobustCost (ar_robust_cost.cu:13-132) runs in the consumers the same way.
 *
 * Same contract as rollout_kernel<AutorallyNNMmaDynamics<32>, ARStandardCost, 1, WB, 1> (rollout_kernel.cuh): one pass over
 * the noise, per-sample cost, block partials of the softmin-weighted control average; the reference functions it replaces are
 * listed there (setGaussianControls gaussian.cu:17-277, rolloutKernel mppi_common.cu:28-146, computeAndSaveCost :843-853,
 * the block half of normExp / weighted reduction :958-966,1115-1160; model: ar_nn_model.cu:123-160 + fnn_helper.cu:419-484,
 * cost: ar_standard_cost.cu:284-413).
 *
 * Why a second kernel. A warp issues in order, so in the generic kernel one step of one warp is a single serial chain:
 * sample -> network -> state update -> sin/cos -> position update -> two map lookups -> slip angle -> cost, of the same length
 * however few samples a GPU holds. But only the NETWORK is recurrent: the network maps
 * (roll, vx, vy, yaw rate, steering, throttle) to the derivatives of (roll, vx, vy, yaw rate) — states 3..6 feed back into
 * it, while position and yaw (states 0..2), the map lookups and the whole cost only CONSUME states 3..6 and never feed the
 * network. The controls do not depend on the state at all (the constraints are a state-independent deadband + clamp).
 * So the step is cut along that line and given to two kinds of warps:
 *
 *   phase 0 (all warps)   noise tile -> constrained controls, in place in shared memory (what setGaussianControls +
 *                         enforceConstraints + writeControlSample do in HBM): no recurrence, fully parallel. Resident form
 *                         only; in the streaming form (below, STREAM) the consumers form them two groups ahead.
 *   producer warp         32 / 16 / 8 samples' network recurrence and nothing else, ENTIRELY in mma fragment layout: lane (g, t)
 *                         keeps states (3 + 2t, 4 + 2t) of its rows g, g+8, ... (t < 2), reads those rows' controls
 *                         from the tile (t == 2), and the C fragment it gets back from layer 3 is exactly the derivative
 *                         of its own slice (nn_mma.cuh: forward_frag) — no transposition through shared memory, no
 *                         __syncwarp inside the recurrence. Per 16-byte noise group (2 steps) it publishes states 3..6
 *                         of both steps into a small ring (mbarrier full / empty handshake).
 *   consumer warp         the same 32 samples, one per lane: waits for a ring slot, integrates position / yaw with the
 *                         full-precision sin / cos, runs the cost (two texture lookups, slip angle, crash flags) and the
 *                         likelihood-ratio term. Its chain per step is short and hides under the producer's.
 *
 * The two roles overlap inside one scheduler the way two independent warps do, which a single in-order instruction
 * stream cannot; the epilogue (block baseline, exp weights, weighted control sum from the tile) is the generic kernel's.
 * Arithmetic per sample is operation-for-operation that of the generic kernel (same sample_control, enforceConstraints,
 * forward_frag, fma state update, computeKinematics, computeRunningCost): the constrained controls agree bit for bit with the
 * generic kernel's and the costs to an ulp (tests/test_gpu_parity.py::test_autorally_warp_specialised_equals_generic).
 */
#pragma once
#include "rollout_kernel.cuh"
#include "plugins/costs.cuh"
#include "plugins/dynamics.cuh"

namespace mppib
{
namespace ar_ws
{
constexpr int kRing = 2;                 // slots per producer / consumer pair; one slot = one noise group = 2 time steps
constexpr int kSlotFloats = 2 * 32 * 4;  // [step in group][sample][states 3..6]
// PSPW = samples per PRODUCER warp. 32: one producer + one consumer warp per 32-sample group. 16: two producers (rows 0-15
// and 16-31 of the group, one m16 tile each) + one consumer — a producer's step is layer after layer of [MMAs -> ex2 / rcp ->
// conversions] with no overlap between layers inside one in-order warp, so two half-size producers that the scheduler
// interleaves finish a group's step in less time than one full-size producer.
// 8: four producers of 8 rows (rows 8..15 of their m16 tile are padding, activations skipped) + one consumer: the same tensor
// work per producer as with 16 rows but half the ex2 / rcp, each producer on its own scheduler — for a GPU that holds so few
// rollouts that a group's step time, not the chip's throughput, sets K1 (multi-GPU strong scaling).
__host__ __device__ constexpr int warpsPerGroup(int pspw)
{
  return 32 / pspw + 1;
}
__host__ __device__ constexpr int maxGroups(int pspw)
{
  return pspw == 8 ? 4 : 8;  // 32-sample groups per block: 256 samples, 128 for the 5-warp groups (register budget)
}
__host__ __device__ constexpr int maxThreads(int pspw)
{
  return warpsPerGroup(pspw) * 32 * maxGroups(pspw);
}
// floats of the block's `theta_s` region for bx samples: fragment-ordered weights, then the rings, then the barriers
// (kRing full + kRing empty per pair, 8 bytes each)
__host__ __device__ constexpr int sharedFloats(int bx)
{
  return nn_mma::kFixedFloats + (bx / 32) * (kRing * kSlotFloats + kRing * 4);
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// streaming form: noise slabs in the block's shared-memory ring. Three, so that the refill of a buffer can wait for the
// slowest warp of the block to leave its slab a whole slab (16 steps) after the issuing warp did, and still land a slab
// ahead of the first reader.
constexpr int kNoiseRing = 3;
}  // namespace ar_ws

using ArWsDyn = plugins::AutorallyNNMmaDynamics<32>;
// the kernel's parameter block for map cost COST (ARStandardCost or ARRobustCost)
template <class COST>
using ArWsArgs = RolloutArgs<ArWsDyn, COST>;

namespace ar_ws
{
// the constrained controls of one 16-byte noise group (steps t0 and t0 + 1) of one sample, as the generic kernel forms them
// (sample_control + enforceConstraints: gaussian.cu:101-121, dynamics.cu:97-116); the second step's pair is unused when
// t0 + 1 == T
template <class ARGS>
__device__ __forceinline__ float2 step_controls(const ARGS& args, const float* means_s, float2 e, int t, bool zn, bool pn)
{
  const float2 m = *reinterpret_cast<const float2*>(means_s + 2 * t);
  const bool um = zn || t < args.opt_stride;
  float u[2] = { sample_control(m.x, args.samp.std_dev_decayed[0][0], e.x, um, pn),
                 sample_control(m.y, args.samp.std_dev_decayed[0][1], e.y, um, pn) };
  ArWsDyn::enforceConstraints(args.dyn, nullptr, u);
  return make_float2(u[0], u[1]);
}
template <class ARGS>
__device__ __forceinline__ float4 group_controls(const ARGS& args, const float* means_s, float4 e, int t0, bool zn,
                                                 bool pn)
{
  const float2 u = step_controls(args, means_s, make_float2(e.x, e.y), t0, zn, pn);
  const float2 v = step_controls(args, means_s, make_float2(e.z, e.w), t0 + 1, zn, pn);
  return make_float4(u.x, u.y, v.x, v.y);
}
}  // namespace ar_ws

// STREAM = false: the block's whole-horizon noise tile stays resident and phase 0 turns it into constrained controls in place.
// STREAM = true: its 32-column slabs cycle through a ring of kNoiseRing buffers, so that shared memory per sample no longer
// grows with T and one CTA of 256 samples fits an SM (C4 in one wave on 132 SMs, where the resident tile would need two).
// Every buffer has a "full" barrier (TMA completion, or the issuing warp's plain loads) and an "empty" one that each warp of
// the block arrives on once it has read its last group of the slab. One warp issues the refills: the consumer of group 0,
// the lightest chain in the block. On entering slab k it waits until every warp has left slab k - 2 and refills that buffer
// with slab k + 1. The consumers turn their rows' groups into constrained controls in place, kRing groups ahead, with the
// same operations as phase 0 (controls_in_place below), and the epilogue recomputes them from a second read of eps
// (rollout_kernel.cuh, STREAM).
template <class COST, bool WRITEBACK, int PSPW, bool STREAM>
__global__ void __launch_bounds__(ar_ws::maxThreads(PSPW), 1)
    rollout_kernel_ar_ws(const __grid_constant__ ArWsArgs<COST> args, const __grid_constant__ CUtensorMap tmap)
{
  static_assert(PSPW == 32 || PSPW == 16 || PSPW == 8, "samples per producer warp");
  static_assert(ar_ws::kNoiseRing >= 3, "the refill of slab k + 1 waits for slab k - 2");
  constexpr int NP = 32 / PSPW;                 // producer warps per 32-sample group
  constexpr int WPG = NP + 1;                   // warps per group
  constexpr int MT = PSPW == 32 ? 2 : 1;        // m16 tiles per producer
  constexpr bool BOT = PSPW >= 16;              // rows g + 8 of the tile carry samples
  constexpr int NR = PSPW / 8;                  // rows a producer lane carries (g + 8 j)
  using DYN = ArWsDyn;
  constexpr int S = 7, C = 2, O = 8;
  using namespace ar_ws;

  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);

  const int nthr = blockDim.x;
  const int npairs = nthr / (32 * WPG);  // 32-sample groups of this block
  const int bx = npairs * 32;            // samples (tile rows) per block
  const int thr = threadIdx.x, lane = thr & 31, warp = thr >> 5;
  const int T = args.T;
  const int TC = T * C;
  const int nchunks = args.nchunks;
  const RolloutSmem L =
      rollout_smem_layout(bx, STREAM ? kNoiseRing : nchunks, 1, TC, args.dyn_shared_floats, COST::sharedFloats(T));
  unsigned char* tile = smem + L.tile;
  float* means_s = reinterpret_cast<float*>(smem + L.means);
  float* theta_s = reinterpret_cast<float*>(smem + L.theta);
  float* theta_c = reinterpret_cast<float*>(smem + L.theta_c);
  float* w_s = reinterpret_cast<float*>(smem + L.weights);
  float* red_s = reinterpret_cast<float*>(smem + L.scratch);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bars);
  float* rings = theta_s + nn_mma::kFixedFloats;
  uint64_t* ring_bars = reinterpret_cast<uint64_t*>(rings + npairs * kRing * kSlotFloats);  // [pair][full 0..R-1 | empty 0..R-1]

  pdl_launch_dependents();
  const int row0 = blockIdx.x * bx;
  const uint32_t slab_bytes = (uint32_t)bx * kChunkBytes;
  uint64_t* slab_empty = bars + kNoiseRing;  // streaming: [full 0..R-1 | empty 0..R-1]
  const int issuer = NP == 1 ? 1 : 0;        // streaming: the warp that refills the ring, the consumer of group 0
  // streaming: slab k of the block's rows -> its ring buffer, by the issuing warp
  auto fill_slab = [&](int k) {
    const int b = k % kNoiseRing;
    unsigned char* dst = tile + (size_t)b * slab_bytes;
    if (args.use_tma)
    {
      if (lane == 0)
      {
        mbar_arrive_expect_tx(&bars[b], slab_bytes);
        tma_load_2d(dst, &tmap, k * kChunkFloats, row0, &bars[b]);
      }
    }
    else
    {  // plain loads (T*C not a multiple of 4: rows are 8-byte aligned); out-of-range elements are zero like TMA's OOB fill
      const float* src = args.eps + (size_t)row0 * TC;
      const int rows_avail = min(bx, args.n_local - row0);
      for (int i = lane; i < bx * 16; i += 32)
      {
        const int r = i >> 4, col = k * kChunkFloats + (i & 15) * 2;
        float2 v = make_float2(0.0f, 0.0f);
        if (r < rows_avail && col < TC)
          v = __ldg(reinterpret_cast<const float2*>(src + (size_t)r * TC + col));
        *reinterpret_cast<float2*>(dst + tile_offset_bytes(bx, 0, r, (i & 15) >> 1) + ((i & 1) << 3)) = v;
      }
      __syncwarp();
      if (lane == 0)
        mbar_arrive(&bars[b]);
    }
  };

  // ---- stage the block's noise rows (identical to the generic kernel) ------------------------------------------------
  if (thr == 0)
  {
    if (args.use_tma)
      tma_prefetch_desc(&tmap);
    if (STREAM)
      for (int b = 0; b < kNoiseRing; b++)
      {
        mbar_init(&bars[b], 1);
        mbar_init(&slab_empty[b], nthr >> 5);  // every warp of the block
      }
    else if (args.use_tma)
      for (int k = 0; k < nchunks; k++)
        mbar_init(&bars[k], 1);
    for (int i = 0; i < npairs * kRing * 2; i++)
      mbar_init(&ring_bars[i], (i % (2 * kRing)) < kRing ? NP : 1);  // full: every producer of the group; empty: its consumer
    fence_barrier_init();
  }
  __syncthreads();
  if (STREAM)
  {
    if (warp == issuer)
      for (int k = 0; k < nchunks && k < kNoiseRing; k++)
        fill_slab(k);
  }
  else if (args.use_tma)
  {
    if (thr == 0)
      for (int k = 0; k < nchunks; k++)
      {
        mbar_arrive_expect_tx(&bars[k], (uint32_t)bx * kChunkBytes);
        tma_load_2d(tile + (size_t)k * bx * kChunkBytes, &tmap, k * kChunkFloats, row0, &bars[k]);
      }
  }
  else
  {
    const float* src = args.eps + (size_t)row0 * TC;
    const int rows_avail = min(bx, args.n_local - row0);
    const int total = bx * nchunks * kChunkFloats;
    for (int i = thr; i < total; i += nthr)
    {
      const int r = i / (nchunks * kChunkFloats);
      const int col = i - r * (nchunks * kChunkFloats);
      float v = 0.0f;
      if (r < rows_avail && col < TC)
        v = __ldg(src + (size_t)r * TC + col);
      const int chunk = col >> 5, within = col & 31;
      *reinterpret_cast<float*>(tile + tile_offset_bytes(bx, chunk, r, within >> 2) + ((within & 3) << 2)) = v;
    }
  }
  for (int i = thr; i < TC; i += nthr)
    means_s[i] = args.means[i];
  nn_mma::load_weights(args.dyn_aux.theta_d, theta_s);
  COST::initializeCosts(args.cost, args.cost_aux, theta_c, T);
  __syncthreads();
  // streaming: noise group gi of block row r -> its constrained controls, in place in the ring (what phase 0 does for the
  // resident tile). The consumer of a row does it for group gi + kRing before it frees ring slot gi, which is what lets the
  // producers of that row start group gi + kRing, so the producers read finished controls; groups 0 .. kRing - 1 are done here.
  auto controls_in_place = [&](int r, int gi) {
    float4* p = reinterpret_cast<float4*>(tile + (size_t)((gi >> 3) % kNoiseRing) * slab_bytes + (uint32_t)r * kChunkBytes +
                                          ((uint32_t)((gi & 7) ^ (r & 7)) << 4));
    const int n_glob = args.n_offset + row0 + r;
    *p = group_controls(args, means_s, *p, 2 * gi, n_glob == 0, (float)n_glob >= args.samp.pure_noise_threshold);
  };
  if (STREAM)
  {
    mbar_wait(&bars[0], 0);
    for (int i = thr; i < bx * kRing; i += nthr)
      if (4 * (i % kRing) < TC)
        controls_in_place(i / kRing, i % kRing);
    __syncthreads();
  }

  // ---- phase 0 (resident tile): noise -> constrained controls, in place (mppi_common.cu:117) --------------------------
  if (!STREAM)
  {
    for (int k = 0; k < nchunks; k++)
    {
      if (args.use_tma)
        mbar_wait(&bars[k], 0);
      unsigned char* slab = tile + (size_t)k * bx * kChunkBytes;
      for (int idx = thr; idx < bx * 8; idx += nthr)
      {
        const int r = idx >> 3;
        const int grp = (idx & 7) ^ (r & 7);  // logical 16-byte group stored at physical position idx & 7
        const int col0 = k * kChunkFloats + grp * 4;
        if (col0 >= TC)
          continue;
        float4* p = reinterpret_cast<float4*>(slab + (size_t)idx * 16);
        const int n_glob = args.n_offset + row0 + r;
        const int t0 = col0 >> 1;
        const bool second = t0 + 1 < T;
        float4 e = *p;
        const float4 u = group_controls(args, means_s, e, t0, n_glob == 0, (float)n_glob >= args.samp.pure_noise_threshold);
        e = make_float4(u.x, u.y, second ? u.z : e.z, second ? u.w : e.w);
        *p = e;
        if (WRITEBACK && row0 + r < args.n_local)
        {
          float2* dst = reinterpret_cast<float2*>(args.controls_out + ((size_t)(row0 + r) * T + t0) * C);
          dst[0] = make_float2(e.x, e.y);
          if (second)
            dst[1] = make_float2(e.z, e.w);
        }
      }
    }
    __syncthreads();
  }

  const int ngroups = (TC + 3) >> 2;
  float cost = 0.0f;
  bool valid = false;
  int row = 0;

  // Which warps of a group produce and which consumes alternates so that every scheduler gets its share of producers (an SM
  // hands consecutive warps to its four schedulers in turn, and the producers carry nearly all MUFU and tensor work):
  //   PSPW 32: warps 2p, 2p+1 serve group p; roles with period 8:  P C C P  C P P C
  //   PSPW 16: warps 3p .. 3p+2 serve group p; the consumer is the first warp of even groups and the last of odd ones
  //            (period 12: C P P  P P C  C P P  P P C — one consumer and two producers per scheduler)
  //   PSPW  8: warps 5p .. 5p+4 serve group p; the consumer is the first: warps 5p and 5p+4 land on the same scheduler, so
  //            the light consumer shares with one producer and the other three producers have a scheduler each
  const int pair = warp / WPG;
  const int wi = warp - pair * WPG;
  const int c_off = (NP == 2) ? ((pair & 1) ? 2 : 0) : 0;  // the consumer's position inside its group (NP >= 2)
  const bool is_producer = (NP == 1) ? (((0x69u >> (warp & 7)) & 1u) != 0) : (wi != c_off);
  const int half = (NP == 1) ? 0 : (wi > c_off ? wi - 1 : wi);  // which PSPW rows of the group this producer owns
  if (is_producer)
  {
    // ---- producer: the network recurrence of PSPW samples in fragment layout ----------------------------------------
    const int g = lane >> 2, t = lane & 3;
    float* ring = rings + pair * kRing * kSlotFloats;
    uint64_t* full = ring_bars + pair * kRing * 2;
    uint64_t* empty = full + kRing;
    const int rbase = half * PSPW;  // first row of this producer inside the group
    float2 st[NR];  // states (3 + 2t, 4 + 2t) of rows rbase + g + 8 j; lanes t >= 2 carry zeros (and stay zero: padded outputs)
#pragma unroll
    for (int j = 0; j < NR; j++)
      st[j] = t == 0 ? make_float2(args.x0[3], args.x0[4]) : (t == 1 ? make_float2(args.x0[5], args.x0[6]) : make_float2(0.0f, 0.0f));
    uint32_t roff[NR];
#pragma unroll
    for (int j = 0; j < NR; j++)
    {
      roff[j] = (uint32_t)(pair * 32 + rbase + g + 8 * j) * kChunkBytes;
      asm volatile("" : "+r"(roff[j]));
    }
    const uint32_t swz = (uint32_t)g;  // (row & 7) of every one of the lane's rows
    const bool ctl_lane = (t == 2);
    const float dt = args.dt;
#pragma unroll 1
    for (int gi = 0; gi < ngroups; gi++)
    {
      const int k = gi >> 3, gg = gi & 7;
      if (STREAM && gg == 0)
        mbar_wait(&bars[k % kNoiseRing], (k / kNoiseRing) & 1);
      const unsigned char* slab = tile + (size_t)(STREAM ? k % kNoiseRing : k) * slab_bytes;
      const int slot = gi % kRing;
      mbar_wait(&empty[slot], (((unsigned)gi / kRing) & 1u) ^ 1u);  // streaming: also, the consumer has formed group gi
      float4 uu[NR];
#pragma unroll
      for (int j = 0; j < NR; j++)
        uu[j] = *reinterpret_cast<const float4*>(slab + roff[j] + (((uint32_t)gg ^ swz) << 4));
      if (STREAM && (gg == 7 || gi == ngroups - 1))
      {  // the warp's last read of this slab
        __syncwarp();
        if (lane == 0)
          mbar_arrive(&slab_empty[k % kNoiseRing]);
      }
      float* out = ring + slot * kSlotFloats;
#pragma unroll 1
      for (int s = 0; s < 2; s++)
      {
        if (gi * 2 + s >= T)
          break;
        uint32_t a_hi[MT][2], a_lo[MT][2];
        if (!BOT)
          a_hi[0][1] = a_lo[0][1] = 0u;
#pragma unroll
        for (int j = 0; j < NR; j++)
        {
          const float2 uv = s == 0 ? make_float2(uu[j].x, uu[j].y) : make_float2(uu[j].z, uu[j].w);
          const float2 v = ctl_lane ? uv : st[j];
          nn_mma::split2(v.x, v.y, a_hi[j >> 1][j & 1], a_lo[j >> 1][j & 1]);
        }
        float o[MT][4];
        nn_mma::forward_frag<MT, BOT>(theta_s, a_hi, a_lo, o);
#pragma unroll
        for (int j = 0; j < NR; j++)
        {  // x_next = x + xdot * dt (dynamics.cu:118-129), on the lane's own slice: row g + 8 j is C-fragment pair (j & 1) of m-tile j >> 1
          st[j].x = fmaf(o[j >> 1][2 * (j & 1)], dt, st[j].x);
          st[j].y = fmaf(o[j >> 1][2 * (j & 1) + 1], dt, st[j].y);
        }
        if (t < 2)
        {
#pragma unroll
          for (int j = 0; j < NR; j++)
            *reinterpret_cast<float2*>(out + s * 128 + (rbase + g + 8 * j) * 4 + 2 * t) = st[j];
        }
      }
      __syncwarp();
      if (lane == 0)
        mbar_arrive(&full[slot]);
    }
  }
  else
  {
    // ---- consumer: position / yaw integration, cost, likelihood-ratio term; one sample per lane -----------------------
    row = pair * 32 + lane;
    const int n_loc = row0 + row;
    valid = n_loc < args.n_local;
    const int n_glob = args.n_offset + n_loc;
    const bool pure_noise = (float)n_glob >= args.samp.pure_noise_threshold;
    const float* ring = rings + pair * kRing * kSlotFloats;
    uint64_t* full = ring_bars + pair * kRing * 2;
    uint64_t* empty = full + kRing;
    float x[S], y[O];
#pragma unroll
    for (int i = 0; i < S; i++)
      x[i] = args.x0[i];
#pragma unroll
    for (int i = 0; i < O; i++)
      y[i] = i < S ? x[i] : 0.0f;  // initializeDynamics: y <- x
    float lr_scale[C];
    bool lr_on = false;
#pragma unroll
    for (int c = 0; c < C; c++)
    {
      lr_scale[c] = args.samp.control_cost_coeff[c] / (args.samp.std_dev[0][c] * args.samp.std_dev[0][c]);
      lr_on = lr_on || (args.samp.control_cost_coeff[c] != 0.0f);
    }
    float half_lambda_1ma = 0.5f * args.lambda * (1.0f - args.alpha);
    asm volatile("" : "+f"(half_lambda_1ma));
    uint32_t roff = (uint32_t)row * kChunkBytes, swz = (uint32_t)row & 7u;
    asm volatile("" : "+r"(roff), "+r"(swz));
    const float dt = args.dt;
    float running_cost = 0.0f;
    int crash_status = 0;
#pragma unroll 1
    for (int gi = 0; gi < ngroups; gi++)
    {
      const int k = gi >> 3, gg = gi & 7;
      if (STREAM && gg == 0)
      {
        if (warp == issuer && k >= 2 && k + kNoiseRing - 2 < nchunks)
        {  // every warp has left slab k - 2: its buffer takes slab k + R - 2
          mbar_wait(&slab_empty[(k - 2) % kNoiseRing], ((k - 2) / kNoiseRing) & 1);
          fill_slab(k + kNoiseRing - 2);
        }
        mbar_wait(&bars[k % kNoiseRing], (k / kNoiseRing) & 1);
      }
      const unsigned char* slab = tile + (size_t)(STREAM ? k % kNoiseRing : k) * slab_bytes;
      float4 uu = *reinterpret_cast<const float4*>(slab + roff + (((uint32_t)gg ^ swz) << 4));
      if (STREAM)
      {
        if (gg == 7 || gi == ngroups - 1)
        {
          __syncwarp();
          if (lane == 0)
            mbar_arrive(&slab_empty[k % kNoiseRing]);
        }
        if (WRITEBACK && valid)
        {
          float2* dst = reinterpret_cast<float2*>(args.controls_out + ((size_t)n_loc * T + 2 * gi) * C);
          dst[0] = make_float2(uu.x, uu.y);
          if (2 * gi + 1 < T)
            dst[1] = make_float2(uu.z, uu.w);
        }
      }
      const int slot = gi % kRing;
      mbar_wait(&full[slot], ((unsigned)gi / kRing) & 1u);
      const float4* in = reinterpret_cast<const float4*>(ring + slot * kSlotFloats);
      const float4 xs0 = in[lane], xs1 = in[32 + lane];
      if (STREAM && gi + kRing < ngroups)
      {  // the producers of this row may start group gi + kRing once slot gi is free: form its controls first
        const int k2 = (gi + kRing) >> 3;
        if (k2 != k)
          mbar_wait(&bars[k2 % kNoiseRing], (k2 / kNoiseRing) & 1);
        controls_in_place(row, gi + kRing);
      }
      __syncwarp();
      if (lane == 0)
        mbar_arrive(&empty[slot]);
#pragma unroll
      for (int s = 0; s < 2; s++)
      {
        const int tt = gi * 2 + s;
        if (tt >= T)
          break;
        const float u[C] = { s == 0 ? uu.x : uu.z, s == 0 ? uu.y : uu.w };
        const float4 xs = s == 0 ? xs0 : xs1;
        float xdot[3];
        DYN::computeKinematics(args.dyn, x, xdot);  // ar_nn_model.cu:123-128
#pragma unroll
        for (int i = 0; i < 3; i++)
          x[i] = x[i] + xdot[i] * dt;  // dynamics.cu:118-129
        x[3] = xs.x, x[4] = xs.y, x[5] = xs.z, x[6] = xs.w;
#pragma unroll
        for (int i = 0; i < S; i++)
          y[i] = x[i];  // stateToOutput
        float step_cost = COST::computeRunningCost(args.cost, args.cost_aux, theta_c, y, u, tt, &crash_status);
        if (lr_on)
          step_cost += likelihood_ratio_cost<C>(lr_scale, means_s + tt * C, u, pure_noise, half_lambda_1ma);
        running_cost += step_cost;
      }
    }
    // computeAndSaveCost, mppi_common.cu:843-853
    cost = running_cost / (float)T + COST::terminalCost(args.cost, args.cost_aux, y) / (float)T;
    if (valid)
      args.costs[n_loc] = cost;
  }

  // ---- block partial of the softmin-weighted control average (the generic kernel's epilogue for D == 1) -------------
  const int nwarps = nthr >> 5;
  {
    const float m = warp_min(valid ? cost : INFINITY);
    if (lane == 0)
      red_s[warp] = m;
    __syncthreads();
    float beta_b = red_s[0];
    for (int i = 1; i < nwarps; i++)
      beta_b = fminf(beta_b, red_s[i]);
    const float w = valid ? softmin_weight(cost, beta_b, args.lambda_inv) : 0.0f;  // normExpTransform, mppi_common.cu:958-966
    if (!is_producer)
      w_s[row] = w;
    const float sw = warp_sum(w), sw2 = warp_sum(w * w);
    if (lane == 0 && !is_producer)
    {
      red_s[32 + pair] = sw;
      red_s[64 + pair] = sw2;
    }
    __syncthreads();
    if (thr == 0)
    {
      float eta_b = 0.0f, w2_b = 0.0f;
      for (int i = 0; i < npairs; i++)  // per 32-sample group, in the generic kernel's warp order
      {
        eta_b += red_s[32 + i];
        w2_b += red_s[64 + i];
      }
      args.headers[blockIdx.x] = make_float4(beta_b, eta_b, w2_b, 0.0f);
    }
  }
  // exp-weighted sum of the constrained controls (weightedReductionKernel, mppi_common.cu:710-737). Resident tile: thread j
  // owns time step j and reads the controls phase 0 left in the tile. Streaming: they are recomputed from a second read of
  // eps, which comes from L2 / HBM, so the block's rows are split into `nslices` slices of whole 8-row blocks that
  // nslices * T threads sum at once (T = 100 would otherwise leave 668 of C4's 768 threads idle, each active one with a
  // 256-row chain of loads); the slice sums are added in slice order through the free ring.
  const int rows_here = min(bx, args.n_local - row0);
  float* out = args.partials + (size_t)blockIdx.x * args.pstride + kPartialHeader;
  const int nslices = STREAM && T <= nthr ? nthr / T : 1;
  const int slice_rows = ((rows_here + nslices - 1) / nslices + 7) & ~7;
  float* slice_s = reinterpret_cast<float*>(tile);  // [slice][T][C]; every warp has left the ring (barriers above)
  for (int i = thr; i < nslices * T; i += nthr)
  {
    const int s = i / T, t = i - s * T;
    float acc[C] = { 0.0f, 0.0f };
    const int col = t * C;
    const int chunk = col >> 5, within = col & 31, grp = within >> 2;
    const unsigned char* slab = tile + (size_t)chunk * bx * kChunkBytes + ((within & 3) << 2);
    weighted_control_rows<DYN>(args, 0, t, row0, s * slice_rows, min((s + 1) * slice_rows, rows_here), slab, grp,
                               means_s + col, t < args.opt_stride, w_s, STREAM, args.eps, STREAM, acc);
#pragma unroll
    for (int c = 0; c < C; c++)
      (nslices == 1 ? out : slice_s)[i * C + c] = acc[c];
  }
  if (nslices > 1)
  {
    __syncthreads();
    for (int t = thr; t < T; t += nthr)
    {
#pragma unroll
      for (int c = 0; c < C; c++)
      {
        float acc = slice_s[t * C + c];
        for (int s = 1; s < nslices; s++)
          acc += slice_s[(s * T + t) * C + c];
        out[t * C + c] = acc;
      }
    }
  }
}

// the instantiation for map cost COST, PSPW samples per producer warp, control write-back and the streaming form
template <class COST>
using ArWsKernel = void (*)(ArWsArgs<COST>, CUtensorMap);
template <class COST, int PSPW>
inline ArWsKernel<COST> ar_ws_kernel_for(bool writeback, bool stream)
{
  if (stream)
    return writeback ? rollout_kernel_ar_ws<COST, true, PSPW, true> : rollout_kernel_ar_ws<COST, false, PSPW, true>;
  return writeback ? rollout_kernel_ar_ws<COST, true, PSPW, false> : rollout_kernel_ar_ws<COST, false, PSPW, false>;
}

}  // namespace mppib
