/*
 * mppi_b200/dynamics/dynamics.hpp — host side of the Dynamics plugin contract
 * (reference: include/mppi/dynamics/dynamics.cuh:67-76 CRTP base, :99-175 control ranges, :250-300 host methods).
 * Same names, same Eigen signatures. The device twin of every model lives in libmppi_b200.so
 * (mppi-generic_b200/csrc/plugins/dynamics.cuh) and is selected by DYN_ID; the parameters cross the C-ABI as the POD
 * blob blob(). Host methods call the exported CPU twins (host_twins.h) so the arithmetic exists once.
 */
#pragma once
#include <cmath>
#include <array>
#include <cfloat>
#include <string>

#include "../utils/common.hpp"

namespace MPPI_internal
{
template <class CLASS_T, class BLOB_T, int DYN_ID_V, int S_DIM, int C_DIM, int O_DIM>
class Dynamics
{
public:
  static const int STATE_DIM = S_DIM;
  static const int CONTROL_DIM = C_DIM;
  static const int OUTPUT_DIM = O_DIM;
  static const int DYN_ID = DYN_ID_V;
  // the cost of the small engine a standalone DDPFeedback solves on (ddp.cuh): the id of the model's in-tree pair, equal to
  // the dynamics id for every model with a Jacobian but RacerDubinsElevation, which shadows it
  static const int DDP_COST_ID = DYN_ID_V;
  typedef BLOB_T BLOB;
  typedef Eigen::Matrix<float, C_DIM, 1> control_array;
  typedef Eigen::Matrix<float, S_DIM, 1> state_array;
  typedef Eigen::Matrix<float, O_DIM, 1> output_array;

  // public like in the reference (examples write model->control_rngs_->x = -5)
  float2 control_rngs_[C_DIM];
  float control_deadband_[C_DIM];
  control_array zero_control_ = control_array::Zero();

  Dynamics(cudaStream_t = 0)
  {
    for (int i = 0; i < C_DIM; i++)
    {  // dynamics.cuh:99-106
      control_rngs_[i].x = -FLT_MAX;
      control_rngs_[i].y = FLT_MAX;
      control_deadband_[i] = 0.0f;
    }
  }
  Dynamics(std::array<float2, C_DIM>& control_rngs, cudaStream_t = 0) : Dynamics()
  {
    setControlRanges(control_rngs);
  }
  virtual ~Dynamics() = default;

  void setControlRanges(std::array<float2, C_DIM>& control_rngs)
  {  // dynamics.cuh:163-170
    for (int i = 0; i < C_DIM; i++)
      control_rngs_[i] = control_rngs[i];
  }
  std::array<float2, C_DIM> getControlRanges() const
  {
    std::array<float2, C_DIM> r;
    for (int i = 0; i < C_DIM; i++)
      r[i] = control_rngs_[i];
    return r;
  }
  void setControlDeadbands(std::array<float, C_DIM>& db)
  {
    for (int i = 0; i < C_DIM; i++)
      control_deadband_[i] = db[i];
  }
  state_array getZeroState() const
  {
    return state_array::Zero();
  }
  // GPUSetup / freeCudaMem / bindToStream exist for source compatibility: device residency is owned by the engine
  void GPUSetup()
  {
  }
  void freeCudaMem()
  {
  }
  void bindToStream(cudaStream_t)
  {
  }

  // POD blob for mppib_set_blob(MPPIB_BLOB_DYN_PARAMS): model parameters + the limits above
  BLOB_T blob() const
  {
    BLOB_T b = static_cast<const CLASS_T*>(this)->modelBlob();
    for (int i = 0; i < MPPIB_MAX_CONTROL_DIM; i++)
    {
      b.lim.rng_lo[i] = i < C_DIM ? control_rngs_[i].x : -FLT_MAX;
      b.lim.rng_hi[i] = i < C_DIM ? control_rngs_[i].y : FLT_MAX;
      b.lim.deadband[i] = i < C_DIM ? control_deadband_[i] : 0.0f;
      b.lim.zero_control[i] = i < C_DIM ? zero_control_(i) : 0.0f;
    }
    return b;
  }
  const float* nnWeights() const
  {
    return nullptr;
  }
  // ---- engine hooks used by Controller (controller.hpp); models with constructor-time architecture or extra weight
  // blobs (the LSTM vehicle model) shadow them ---------------------------------------------------------------------
  void fillModelDims(int* /*dims[8]*/) const
  {
  }
  int pushModelBlobs(mppib_engine* e) const
  {
    const float* w = static_cast<const CLASS_T*>(this)->nnWeights();
    return w ? mppib_set_blob(e, MPPIB_BLOB_NN_WEIGHTS, w, MPPIB_AR_NN_NUM_PARAMS * sizeof(float)) : MPPIB_OK;
  }
  int hostOutputTrajectory(const float* x0, const float* u, int T, float dt, float* states, float* outputs) const
  {
    BLOB_T b = blob();
    return mppib_host_output_trajectory(DYN_ID_V, &b, static_cast<const CLASS_T*>(this)->nnWeights(), x0, u, T, dt,
                                        states, outputs);
  }

  // ---- host methods (dynamics.cuh:250-300) -----------------------------------------------------------------------
  void enforceConstraints(Eigen::Ref<state_array> /*state*/, Eigen::Ref<control_array> control)
  {
    float u[C_DIM];
    for (int i = 0; i < C_DIM; i++)
      u[i] = control(i);
    BLOB_T b = blob();
    MPPIB_HANDLE(mppib_host_enforce_constraints(DYN_ID_V, &b, u));
    for (int i = 0; i < C_DIM; i++)
      control(i) = u[i];
  }
  void step(Eigen::Ref<state_array> state, Eigen::Ref<state_array> next_state, Eigen::Ref<state_array> state_der,
            const Eigen::Ref<const control_array>& control, Eigen::Ref<output_array> output, const float /*t*/,
            const float dt)
  {
    float x[S_DIM], u[C_DIM], xn[S_DIM], xd[S_DIM], y[O_DIM];
    for (int i = 0; i < S_DIM; i++)
      x[i] = state(i);
    for (int i = 0; i < C_DIM; i++)
      u[i] = control(i);
    BLOB_T b = blob();
    MPPIB_HANDLE(mppib_host_step(DYN_ID_V, &b, static_cast<CLASS_T*>(this)->nnWeights(), x, u, dt, xn, xd, y));
    for (int i = 0; i < S_DIM; i++)
    {
      next_state(i) = xn[i];
      state_der(i) = xd[i];
    }
    for (int i = 0; i < O_DIM; i++)
      output(i) = y[i];
  }
  void computeStateDeriv(const Eigen::Ref<const state_array>& state, const Eigen::Ref<const control_array>& control,
                         Eigen::Ref<state_array> state_der)
  {
    state_array s = state, nx;
    output_array y;
    step(s, nx, state_der, control, y, 0.0f, 1.0f);
  }
  void updateState(Eigen::Ref<state_array> state, Eigen::Ref<state_array> state_der, const float dt)
  {  // dynamics.cuh:271-275 (deprecated in-place form)
    for (int i = 0; i < S_DIM; i++)
      state(i) = state(i) + state_der(i) * dt;
  }
  virtual std::string getDynamicsModelName() const
  {
    return "Dynamics model name not set";
  }
  // dynamics.cuh:448-466: pull the planner's initial state towards the true one, component by component; models whose
  // states are not all Euclidean override it (RacerDubins: racer_dubins.cu:177-230)
  virtual void enforceLeash(const Eigen::Ref<const state_array>& state_true, const Eigen::Ref<const state_array>& state_nominal,
                            const Eigen::Ref<const state_array>& leash_values, Eigen::Ref<state_array> state_output)
  {
    for (int i = 0; i < S_DIM; i++)
    {
      const float diff = fabsf(state_nominal(i) - state_true(i));
      if (leash_values(i) < diff)
        state_output(i) = state_true(i) + fminf(fmaxf(state_nominal(i) - state_true(i), -leash_values(i)), leash_values(i));
      else
        state_output(i) = state_nominal(i);
    }
  }
};
}  // namespace MPPI_internal
