/*
 * feedback.cuh — the ancillary feedback controller of Tube-MPPI and RMPPI: DDPFeedback's weights and its solve on the device
 * (ddp_kernel.cuh, launched through the pair's PairEntry::ddp), and the [T][S][C] gain trajectory and value-function
 * threshold RMPPI's K1 reads. One member of mppib_engine; the definitions are in engine.cu.
 * - The weights start as DDPParams' defaults, Q = Q_f = I, R = I and one iteration, held as data like any other weights.
 * - The gain buffer counts as set only while it holds a whole trajectory: after set_rmppi's copy has succeeded, or after
 *   a to_rmppi solve has succeeded (the kernel writes the gains only then). Until then K1 gets no gains (gains() is null).
 */
#pragma once
#include <cuda_runtime.h>

#include <vector>

#include "../../include/mppi_b200.h"
#include "device_resources.cuh"

namespace mppib
{
class Feedback : NoCopy
{
public:
  // S states, C controls and the engine's horizon T (the length of RMPPI's gain trajectory); copies run on `stream`
  void create(int S, int C, int T, cudaStream_t stream);
  int set_weights(const float* Q, const float* Q_f, const float* R, int iters);  // mppib_set_ddp
  int set_rmppi(float threshold, const float* host_gains);                         // gains [T][S][C], or null: none
  // DDPFeedback::computeFeedback over horizon T from x0 around the targets; to_rmppi: the gains also become K1's. The
  // outputs the caller passes (each may be null) are copied back once the solve has succeeded.
  int compute(mppib_engine& e, int T, const float* x0, const float* x_target, const float* u_target, bool to_rmppi,
              float* gains, float* x_out, float* u_out, float* jac_out);

  // for the DDP launch: row-major weights, iterations, the workspace (ddp::ws_layout) and the status word
  const float* Q() const { return Q_.data(); }
  const float* Q_f() const { return Qf_.data(); }
  const float* R() const { return R_.data(); }
  int iters() const { return iters_; }
  float* ws() const { return ws_; }
  int* status() const { return status_; }
  // for K1: the gain trajectory, null unless it is set
  const float* gains() const { return gains_set_ ? gains_.get() : nullptr; }
  float threshold() const { return threshold_; }

private:
  cudaStream_t stream_ = nullptr;
  int S_ = 0, C_ = 0, T_ = 0;
  std::vector<float> Q_, Qf_, R_;
  int iters_ = 1;
  DeviceBuffer<float> ws_;  // for the longest horizon so far
  DeviceBuffer<int> status_;
  DeviceBuffer<float> gains_;  // [T][S][C]
  bool gains_set_ = false;
  float threshold_ = 1000.0f;  // robust_mppi_controller.cuh default
};
}  // namespace mppib
