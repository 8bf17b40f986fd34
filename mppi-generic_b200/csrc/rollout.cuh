/*
 * rollout.cuh — K1, the fused rollout (rollout_kernel.cuh, rollout_kernel_ar_ws.cuh, rollout_kernel_nn_tc.cuh): the pair
 * entry that launches it, its plan (form and geometry), its TMA views of the two noise buffers, and what it writes beside
 * the block partials: the per-sample costs and, optionally, the written-back controls. Also the two buffers that serve it:
 * the importance weights of mppib_get_weights and the L2 flush. One member of mppib_engine; the definitions are in engine.cu.
 * - The plan is chosen once. pick() reads the overrides (descriptor flags and environment variables) and picks the pair
 *   entry with no device work, so its refusals come before any device is touched; create() chooses the plan against the
 *   device's limits, once the SM count and the noise buffers exist. The plan is the only record of what the overrides chose.
 * - The engine keeps written-back controls exactly when controls() is non-null: RMPPI, MPPIB_FLAG_WRITEBACK_CONTROLS or a
 *   plan with stream_readback. create() decides it once.
 * - read_costs, read_controls and weights copy on the solve's stream and drain it: they return the last K1's results.
 * - The L2 flush is exactly the bytes set (0: none). set_l2_flush drains the stream before it replaces the buffer;
 *   flush_l2() zeroes all of it on the stream, between the noise draw and K1, to evict the noise from L2.
 */
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/mppi_b200.h"
#include "device_resources.cuh"

struct PairEntry;

namespace mppib
{
// ---- K1's form and geometry, chosen once per engine (engine.cu: choose_k1) --------------------------------------------
enum class K1Form
{
  Generic,      // rollout_kernel.cuh, one sample per thread
  GenericSpt2,  // rollout_kernel.cuh, two samples per thread (MPPIB_SPT = 2)
  Rmppi,        // rollout_kernel.cuh, RMPPI: nominal and real system (MPPIB_FLAG_RMPPI)
  WarpSpec,     // rollout_kernel_ar_ws.cuh: Autorally pair, producer and consumer warps
  Wgmma,        // rollout_kernel_nn_tc.cuh: Autorally pair, the network on wgmma tensor cores
};
struct K1Plan
{
  K1Form form = K1Form::Generic;
  int D = 1;                     // distributions per sample, as the generic kernel is instantiated
  bool stream = false;           // noise slabs through a ring, controls kept in HBM (STREAM; generic or warp-specialised)
  bool stream_readback = false;  // generic streaming form, A/B (MPPIB_STREAM_READBACK): weighted sum from written-back controls
  int ws_pspw = 16;  // warp-specialised kernel: samples per producer warp; threads per CTA = bx * (32 / ws_pspw + 1)
  int spt = 1;       // samples per thread; generic kernel: threads per CTA = bx / spt * lps
  int lps = 1;       // lanes per sample = 32 / DYN::SAMPLES_PER_WARP (rollout_kernel.cuh: SPW)
  int ring = 2;      // noise slabs in the generic streaming form's ring
  int bx = 64;       // samples (noise-tile rows) per CTA
  int threads = 0;   // threads per CTA
  int grid = 0;
  uint32_t smem_bytes = 0;
  bool use_tma = false;
  int dyn_shared_floats = 0;  // the dynamics' shared floats for a CTA of bx samples
  bool smooth = false;        // the smooth-MPPI sampler's instantiation (rollout_kernel_smooth) of a generic form
};

struct K1Overrides;  // engine.cu: the descriptor flags and environment variables that choose K1's form or geometry

class Rollout : NoCopy
{
public:
  // The pair entry for the descriptor and the overrides; *wgmma_asked: NN_TENSOR asks for the wgmma kernel of a pair that
  // has one. fp16_ok: the model's network (steering LSTM or Autorally) and its known input bounds fit the FP16 operands of
  // its mma.sync form (engine.cu: network_fits_fp16). Needs no device.
  static int pick(const mppib_desc& desc, K1Overrides* ov, const PairEntry** entry, bool* wgmma_asked,
                  bool fp16_ok = true);
  // After the engine's sizes, flags and SM count are set and its noise source is created: the plan, write-back, the
  // buffers, the tensor maps and the kernel's attributes
  int create(const mppib_engine& e, const PairEntry* entry, const K1Overrides& ov, bool wgmma_asked);

  int launch(mppib_engine& e, const float* x0, const float* U, int opt_stride, int iter) const;
  int read_costs(float* host) const;     // [D][n_local]
  int read_controls(float* host) const;  // [D][n_local][T][C]; refused without write-back
  // the importance weights [D][n_local] of the last costs against the result record's baseline and normaliser
  int weights(float* host, const float* result, int pstride, float lambda);
  int set_l2_flush(long long bytes);
  cudaError_t flush_l2() const;

  const PairEntry& pair() const { return *pair_; }
  const K1Plan& plan() const { return plan_; }
  // for the launchers
  int nchunks() const { return nchunks_; }
  const CUtensorMap& tensor_map(int i) const { return tmap_[i]; }  // the view of noise.buffer(i)
  float* costs() const { return costs_; }
  float* controls() const { return controls_; }  // null: the engine keeps no controls

private:
  // the (dynamics, cost) pair's kernels and sizes: a built-in entry is static, and a registered one is never freed
  // (mppib_register_pair), so the pointer outlives the engine
  const PairEntry* pair_ = nullptr;
  K1Plan plan_;
  cudaStream_t stream_ = nullptr;
  int D_ = 1, n_local_ = 0, TC_ = 0, nchunks_ = 0;
  CUtensorMap tmap_[2]{};  // box: kChunkFloats columns by the plan's bx rows
  DeviceBuffer<float> costs_;     // [D][n_local]
  DeviceBuffer<float> controls_;  // optional [D][n_local][T][C]
  DeviceBuffer<float> weights_;   // allocated by the first weights()
  DeviceBuffer<unsigned char> l2_flush_;
};
}  // namespace mppib
