/*
 * side_rollouts.cuh — the rollouts that run beside the solve, one thread per rollout (side_rollout_kernels.cuh, launched
 * through the pair's PairEntry): init-eval (mppib_init_eval, RMPPI's nominal-state candidates), sampled trajectories
 * (mppib_sample_trajectories) and the device-side roll-forward of the host tail (mppib_nominal_trajectory). One member of
 * mppib_engine; the definitions are in engine.cu.
 * - Each operation sizes its scratch to what the call holds (reserve: a buffer only grows), copies in, launches, copies
 *   out and drains the stream before it returns.
 * - A pending solve: sampled trajectories refuse one (they read its written-back controls); the roll-forward with U = NULL
 *   chains behind one and reads its result record on the device; init-eval does not wait for one, it runs after the
 *   solve on the same stream.
 */
#pragma once
#include <cuda_runtime.h>

#include "../../include/mppi_b200.h"
#include "device_resources.cuh"

namespace mppib
{
class SideRollouts : NoCopy
{
public:
  // After the entry point's checks. init_eval: candidates [K][S], strides [K] (>= 0), costs_out [K * samples].
  int init_eval(mppib_engine& e, const float* candidates, const int* strides, int K, int samples, const float* U_nominal,
                int opt_stride, float* costs_out);
  // sample_idx [n] in [-1, n_local); U_opt: the sequence index -1 rolls out, null when no index is -1
  int sample(mppib_engine& e, const float* x0, const float* U_nominal, int distribution, const int* sample_idx, int n,
             const float* U_opt, float* outputs, float* costs, int* crash);
  // U [D][T][C], or null: the last solve's result; history [2][C], or null: no smoothing; U_smoothed may be null
  int nominal(mppib_engine& e, const float* x0, const float* U, const float* history, float* U_smoothed, float* states,
              float* outputs);

  // for the launchers: init-eval
  const float* eval_candidates() const { return eval_states_; }  // [K][S]
  const int* eval_strides() const { return eval_strides_; }      // [K]
  float* eval_costs() const { return eval_costs_; }              // [K * samples]
  // sampled trajectories
  const int* sample_idx() const { return vis_idx_; }                                // [n]
  const float* sample_opt() const { return have_opt_ ? vis_opt_.get() : nullptr; }  // [T][C] if an index is -1, or null
  float* sample_outputs() const { return vis_outputs_; }                            // [n][T][O]
  float* sample_costs() const { return vis_costs_; }                                // [n][T + 1]
  int* sample_crash() const { return vis_crash_; }                                  // [n][T]
  // roll-forward: system d's controls at nominal_src() + d * nominal_stride(); what the kernel writes, [D][T][*] each
  const float* nominal_src() const { return nom_src_; }
  int nominal_stride() const { return nom_stride_; }
  float* nominal_controls() const { return nom_; }
  float* nominal_states() const { return nom_ + n_u_; }
  float* nominal_outputs() const { return nom_ + n_u_ + n_s_; }

private:
  DeviceBuffer<float> eval_states_;
  DeviceBuffer<int> eval_strides_;
  DeviceBuffer<float> eval_costs_;
  DeviceBuffer<int> vis_idx_;
  DeviceBuffer<float> vis_opt_;
  DeviceBuffer<float> vis_outputs_;
  DeviceBuffer<float> vis_costs_;
  DeviceBuffer<int> vis_crash_;
  bool have_opt_ = false;
  DeviceBuffer<float> nom_;    // [D][T][C] smoothed controls | [D][T][S] states | [D][T][O] outputs
  PinnedBuffer<float> nom_h_;  // pinned host copy of the same
  DeviceBuffer<float> nom_u_;  // the caller's [D][T][C], when it passes its own U
  const float* nom_src_ = nullptr;
  int nom_stride_ = 0;
  size_t n_u_ = 0, n_s_ = 0;
};
}  // namespace mppib
