/*
 * RobustMPPIController — host class of include/mppi/controllers/R-MPPI/robust_mppi_controller.cuh. Two systems run as ONE
 * engine solve created with MPPIB_FLAG_RMPPI: distribution 0 = nominal, 1 = real (robust_mppi_controller.cu:637-640);
 * the candidate line search runs through mppib_init_eval (computeNominalStateAndStride, :571-617) and the host logic
 * (line-search weights, candidates, strides, best index) through the library's host twins.
 *
 * Feedback: after initFeedback() (FB_T = DDPFeedback) every updateImportanceSamplingControl runs the DDP solve from the
 * real state around the nominal trajectory (robust_mppi_controller.cu:546-568, 629-632); the kernel writes the gains
 * straight into the engine's feedback buffer, which the next solve applies. Without it the gain trajectory is an input
 * (setFeedbackGains; explicit gains switch the computation off until initFeedback() is called again). With no gains at
 * all the real system runs without feedback. Like the reference's rollout, which always reads its feedback controller's
 * device gains, disableFeedbackController() stops the recomputation and leaves the last gains applied.
 */
#pragma once
#include <cstring>
#include <iostream>

#include "../controller.hpp"
#include "../../sampling_distributions/gaussian/gaussian.hpp"

template <int S_DIM, int C_DIM, int MAX_TIMESTEPS>
struct RobustMPPIParams : public ControllerParams<S_DIM, C_DIM, MAX_TIMESTEPS>
{  // robust_mppi_controller.cuh:44-53
  float value_function_threshold_ = 1000.0;
  int optimization_stride_ = 1;
  int num_candidate_nominal_states_ = 9;
  dim3 eval_cost_kernel_dim_;
  dim3 eval_dyn_kernel_dim_ = dim3(64, 1, 1);  // .x = samples per candidate (getNumEvalSamplesPerCandidate, :85-88)
};

template <class DYN_T, class COST_T, class FB_T, int MAX_TIMESTEPS, int NUM_ROLLOUTS,
          class SAMPLING_T = ::mppi::sampling_distributions::GaussianDistribution<typename DYN_T::DYN_PARAMS_T>,
          class PARAMS_T = RobustMPPIParams<DYN_T::STATE_DIM, DYN_T::CONTROL_DIM, MAX_TIMESTEPS>>
class RobustMPPIController
  : public Controller<DYN_T, COST_T, FB_T, SAMPLING_T, MAX_TIMESTEPS, NUM_ROLLOUTS, PARAMS_T, 2, MPPIB_FLAG_RMPPI>
{
public:
  typedef Controller<DYN_T, COST_T, FB_T, SAMPLING_T, MAX_TIMESTEPS, NUM_ROLLOUTS, PARAMS_T, 2, MPPIB_FLAG_RMPPI> PARENT_CLASS;
  using control_array = typename PARENT_CLASS::control_array;
  using control_trajectory = typename PARENT_CLASS::control_trajectory;
  using state_trajectory = typename PARENT_CLASS::state_trajectory;
  using output_trajectory = typename PARENT_CLASS::output_trajectory;
  using state_array = typename PARENT_CLASS::state_array;
  using output_array = typename PARENT_CLASS::output_array;
  typedef Eigen::Matrix<float, DYN_T::CONTROL_DIM, DYN_T::STATE_DIM> feedback_gain_matrix;

  RobustMPPIController(DYN_T* model, COST_T* cost, FB_T* fb_controller, SAMPLING_T* sampler, float dt, int max_iter,
                       float lambda, float alpha, float value_function_threshold, int num_timesteps = MAX_TIMESTEPS,
                       const Eigen::Ref<const control_trajectory>& init_control_traj = control_trajectory::Zero(),
                       int num_candidate_nominal_states = 9, int optimization_stride = 1, cudaStream_t stream = nullptr)
    : PARENT_CLASS(model, cost, fb_controller, sampler, dt, max_iter, lambda, alpha, num_timesteps, init_control_traj,
                   stream)
  {
    this->params_.value_function_threshold_ = value_function_threshold;
    this->params_.optimization_stride_ = optimization_stride;
    nominal_control_trajectory_ = init_control_traj;
    updateNumCandidates(num_candidate_nominal_states);
    pushRMPPI();
    this->chooseAppropriateKernel();
  }
  std::string getControllerName() override
  {
    return "Robust MPPI";
  }
  // ---- parameters (robust_mppi_controller.cuh:160-240) ------------------------------------------------------------
  float getValueFunctionThreshold() const
  {
    return this->params_.value_function_threshold_;
  }
  void setValueFunctionThreshold(float v)
  {
    this->params_.value_function_threshold_ = v;
    pushRMPPI();
  }
  int getNumCandidates() const
  {
    return this->params_.num_candidate_nominal_states_;
  }
  int getNumEvalSamplesPerCandidate() const
  {
    return this->params_.eval_dyn_kernel_dim_.x;
  }
  int getNumEvalRollouts() const
  {
    return getNumCandidates() * getNumEvalSamplesPerCandidate();
  }
  // robust_mppi_controller.cu:430-467
  void updateNumCandidates(int new_num_candidates)
  {
    if ((new_num_candidates * getNumEvalSamplesPerCandidate()) > NUM_ROLLOUTS)
    {
      std::cerr << "ERROR: (number of candidates) * (SAMPLES_PER_CANDIDATE) cannot exceed NUM_ROLLOUTS\n";
      std::terminate();
    }
    if (new_num_candidates < 3)
    {
      std::cerr << "ERROR: number of candidates must be greater or equal to 3\n";
      std::terminate();
    }
    if (new_num_candidates % 2 == 0)
    {
      std::cerr << "ERROR: number of candidates must be odd\n";
      std::terminate();
    }
    this->params_.num_candidate_nominal_states_ = new_num_candidates;
    candidate_nominal_states_.assign((size_t)new_num_candidates * DYN_T::STATE_DIM, 0.0f);
    importance_sampler_strides_.assign(new_num_candidates, 0);
    candidate_trajectory_costs_.assign(getNumEvalRollouts(), 0.0f);
    candidate_free_energy_.assign(new_num_candidates, 0.0f);
    line_search_weights_.assign((size_t)3 * new_num_candidates, 0.0f);
    mppib_host_rmppi_line_search_weights(new_num_candidates, line_search_weights_.data());
  }
  // the DDP gain trajectory: gains[t] = K_t (C x S); no gains => no feedback
  void setFeedbackGains(const std::vector<feedback_gain_matrix>& gains)
  {
    this->enable_feedback_ = false;
    const int T = this->getNumTimesteps();
    fb_gains_.assign((size_t)T * DYN_T::STATE_DIM * DYN_T::CONTROL_DIM, 0.0f);
    for (int t = 0; t < T && t < (int)gains.size(); t++)
      memcpy(&fb_gains_[(size_t)t * DYN_T::STATE_DIM * DYN_T::CONTROL_DIM], gains[t].data(),
             sizeof(float) * DYN_T::STATE_DIM * DYN_T::CONTROL_DIM);  // Eigen column-major C x S == [s][c]
    pushRMPPI();
  }
  control_trajectory getNominalControlSeq() const
  {
    return nominal_control_trajectory_;
  }
  state_trajectory getNominalStateSeq() const
  {
    return nominal_state_trajectory_;
  }
  state_trajectory getTargetStateSeq() const override
  {
    return nominal_state_trajectory_;
  }
  const std::vector<float>& getCandidateFreeEnergy() const
  {
    return candidate_free_energy_;
  }
  // robust_mppi_controller.cu:758-762: |x_fb(0) - x_fb(1)| + |x_nom(0) - x_fb(0)| on the feedback-propagated and the
  // nominal state trajectories (call computeFeedbackPropagatedStateSeq first)
  float computeDF()
  {
    const state_trajectory fb = this->getFeedbackPropagatedStateSeq();
    const state_trajectory nom = getTargetStateSeq();
    float a = 0.0f, b = 0.0f;
    for (int i = 0; i < DYN_T::STATE_DIM; i++)
    {
      a += (fb(i, 0) - fb(i, 1)) * (fb(i, 0) - fb(i, 1));
      b += (nom(i, 0) - fb(i, 0)) * (nom(i, 0) - fb(i, 0));
    }
    return sqrtf(a) + sqrtf(b);
  }
  int getBestIndex() const
  {
    return best_index_;
  }

  // robust_mppi_controller.cu:539-568
  void updateImportanceSamplingControl(const Eigen::Ref<const state_array>& state, int stride)
  {
    real_stride_ = stride;
    computeNominalStateAndStride(state, stride);
    this->saveControlHistoryHelper(nominal_stride_, nominal_control_trajectory_, nominal_control_history_);
    this->saveControlHistoryHelper(real_stride_, this->control_, this->control_history_);
    this->slideControlSequenceHelper(nominal_stride_, nominal_control_trajectory_);
    output_trajectory out = output_trajectory::Zero();
    this->computeOutputTrajectoryHelper(out, nominal_state_trajectory_, nominal_state_, nominal_control_trajectory_);
    computeNominalFeedbackGains(state);
  }
  // robust_mppi_controller.cu:629-632
  void computeNominalFeedbackGains(const Eigen::Ref<const state_array>& state)
  {
    computeFeedbackHelper(state, nominal_state_trajectory_, nominal_control_trajectory_);
  }
  // the gains go straight into the engine's feedback buffer (mppib_ddp_feedback with to_rmppi); the host copy is kept so a
  // re-created engine gets them back
  void computeFeedbackHelper(const Eigen::Ref<const state_array>& state, const Eigen::Ref<const state_trajectory>& state_traj,
                             const Eigen::Ref<const control_trajectory>& control_traj) override
  {
    if (!this->enable_feedback_)
      return;
    this->runFeedback(state, state_traj, control_traj, true);
    if constexpr (PARENT_CLASS::kHasDDPFeedback)
      fb_gains_ = this->fb_controller_->getFeedbackState().fb_gain_traj_;
    fb_gains_.resize((size_t)this->getNumTimesteps() * DYN_T::STATE_DIM * DYN_T::CONTROL_DIM);
  }
  // robust_mppi_controller.cuh: a no-op; the gains are computed in updateImportanceSamplingControl
  void computeFeedback(const Eigen::Ref<const state_array>& /*state*/) override
  {
  }
  // robust_mppi_controller.cu:571-617
  void computeNominalStateAndStride(const Eigen::Ref<const state_array>& state, int stride)
  {
    if (!nominal_state_init_)
    {
      nominal_state_ = state;
      nominal_state_init_ = true;
      nominal_stride_ = 0;
      return;
    }
    const int K = getNumCandidates(), spc = getNumEvalSamplesPerCandidate();
    state_array xk = nominal_state_trajectory_.col(0), xk1 = nominal_state_trajectory_.col(1), xr = state;
    mppib_host_rmppi_candidates(K, DYN_T::STATE_DIM, xk.data(), xk1.data(), xr.data(), stride,
                                candidate_nominal_states_.data(), importance_sampler_strides_.data());
    MPPIB_HANDLE(mppib_init_eval(this->engine_, candidate_nominal_states_.data(), importance_sampler_strides_.data(), K, spc,
                                 nominal_control_trajectory_.data(), stride, candidate_trajectory_costs_.data()));
    best_index_ = mppib_host_rmppi_best_index(candidate_trajectory_costs_.data(), K, spc, this->getLambda(),
                                              getValueFunctionThreshold(), best_index_, candidate_free_energy_.data());
    this->free_energy_statistics_.nominal_state_used = best_index_;
    nominal_stride_ = importance_sampler_strides_[best_index_];
    for (int i = 0; i < DYN_T::STATE_DIM; i++)
      nominal_state_(i) = candidate_nominal_states_[(size_t)best_index_ * DYN_T::STATE_DIM + i];
  }
  // robust_mppi_controller.cu:625-755
  void computeControl(const Eigen::Ref<const state_array>& state, int optimization_stride = 1) override
  {
    constexpr int S = DYN_T::STATE_DIM, C = DYN_T::CONTROL_DIM;
    const int T = this->getNumTimesteps();
    if (!nominal_state_init_)
    {
      nominal_state_ = state;
      nominal_state_init_ = true;
    }
    this->free_energy_statistics_.nominal_sys.previousBaseline = this->getBaselineCost(0);
    this->free_energy_statistics_.real_sys.previousBaseline = this->getBaselineCost(1);
    std::vector<float> x0s(2 * S), uin((size_t)2 * T * C), uout((size_t)2 * T * C);
    for (int i = 0; i < S; i++)
    {
      x0s[i] = nominal_state_(i);
      x0s[S + i] = state(i);
    }
    for (int opt_iter = 0; opt_iter < this->getNumIters(); opt_iter++)
    {  // both importance samplers are the nominal control (:643-645)
      memcpy(uin.data(), nominal_control_trajectory_.data(), sizeof(float) * T * C);
      memcpy(uin.data() + (size_t)T * C, nominal_control_trajectory_.data(), sizeof(float) * T * C);
      this->solve(x0s.data(), uin.data(), optimization_stride, opt_iter, uout.data());
      memcpy(nominal_control_trajectory_.data(), uout.data(), sizeof(float) * T * C);
      memcpy(this->control_.data(), uout.data() + (size_t)T * C, sizeof(float) * T * C);
    }
    this->smoothControlTrajectoryHelper(this->control_, this->control_history_);
    this->smoothControlTrajectoryHelper(nominal_control_trajectory_, nominal_control_history_);
    this->computeOutputTrajectoryHelper(this->output_, nominal_state_trajectory_, nominal_state_,
                                        nominal_control_trajectory_);
    this->state_ = nominal_state_trajectory_;
    auto& fe = this->free_energy_statistics_;
    fe.real_sys.normalizerPercent = this->getNormalizerCost(1) / NUM_ROLLOUTS;
    fe.real_sys.increase = this->getBaselineCost(1) - fe.real_sys.previousBaseline;
    fe.nominal_sys.normalizerPercent = this->getNormalizerCost(0) / NUM_ROLLOUTS;
    fe.nominal_sys.increase = this->getBaselineCost(0) - fe.nominal_sys.previousBaseline;
  }
  void slideControlSequence(int /*steps*/) override
  {  // robust_mppi_controller.cuh:186-190: done inside updateImportanceSamplingControl
  }

protected:
  void onEngineCreated() override
  {  // a re-created engine has lost the value-function threshold and the feedback gains
    pushRMPPI();
  }

private:
  void pushRMPPI()
  {
    MPPIB_HANDLE(mppib_set_rmppi(this->engine_, this->params_.value_function_threshold_,
                                 fb_gains_.empty() ? nullptr : fb_gains_.data()));
  }
  control_trajectory nominal_control_trajectory_ = control_trajectory::Zero();
  state_trajectory nominal_state_trajectory_ = state_trajectory::Zero();
  Eigen::Matrix<float, DYN_T::CONTROL_DIM, 2> nominal_control_history_ = Eigen::Matrix<float, DYN_T::CONTROL_DIM, 2>::Zero();
  state_array nominal_state_ = state_array::Zero();
  bool nominal_state_init_ = false;
  int nominal_stride_ = 0, real_stride_ = 0, best_index_ = 0;
  std::vector<float> candidate_nominal_states_, candidate_trajectory_costs_, candidate_free_energy_, line_search_weights_,
      fb_gains_;
  std::vector<int> importance_sampler_strides_;
};
