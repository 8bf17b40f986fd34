/*
 * mppi_b200/controllers/controller.hpp — host-side Controller base, mirroring include/mppi/controllers/controller.cuh:
 * same template parameters and order, same constructor arguments, same public methods for the hot path
 * (computeControl, getControlSeq, getTargetStateSeq, getTargetOutputSeq, getBaselineCost, getNormalizerCost,
 *  getFreeEnergyStatistics, slideControlSequence, setParams/getParams, setSeedCUDARandomNumberGen, getSampledCostSeq).
 * Everything device-side goes through the C-ABI engine (include/mppi_b200.h); the host tail — Savitzky-Golay smoothing,
 * nominal roll-forward, clamping (controller.cuh:557-663) — stays on the host like in the reference.
 *
 * Feedback (controller.cuh:263-268, 329-346, 395-399, 479-560, 709-721): when FB_T is a DDPFeedback (it has bindEngine) the
 * controller binds its engine into it on every engine creation, and initFeedback / computeFeedback / getFeedbackControl /
 * interpolateFeedback / computeFeedbackPropagatedStateSeq run the DDP solve on the GPU (feedback_controllers/DDP/ddp.cuh).
 * Deliberate deviation: feedback is off until initFeedback() is called (the reference's Tube / RMPPI constructors switch it
 * on), so existing users get what they had. With any other FB_T the surface compiles and does nothing.
 *
 * Not carried over: kernel-choice timing (chooseAppropriateKernel keeps its RNG side effect only: one burnt noise draw,
 * mppi_controller.cu:95).
 */
#pragma once
#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <random>
#include <memory>
#include <type_traits>
#include <utility>
#include <vector>

#include "../utils/common.hpp"

namespace mppi_b200
{
// FB_T is a DDPFeedback (feedback_controllers/DDP/ddp.cuh): the controllers' feedback surface is live only then
template <class FB, class = void>
struct has_ddp_feedback : std::false_type
{
};
template <class FB>
struct has_ddp_feedback<FB, decltype(std::declval<FB&>().bindEngine(nullptr), void())> : std::true_type
{
};
}  // namespace mppi_b200

// controller.cuh:22-38
struct freeEnergyEstimate
{
  float increase = -1;
  float previousBaseline = -1;
  float freeEnergyMean = -1;
  float freeEnergyVariance = -1;
  float freeEnergyModifiedVariance = -1;
  float normalizerPercent = -1;
};
struct MPPIFreeEnergyStatistics
{
  int nominal_state_used = 0;
  freeEnergyEstimate nominal_sys;
  freeEnergyEstimate real_sys;
};

enum class kernelType : int
{
  USE_SINGLE_KERNEL = 0,
  USE_SPLIT_KERNELS,
};

// controller.cuh:46-68
template <int S_DIM, int C_DIM, int MAX_TIMESTEPS>
struct ControllerParams
{
  static const int TEMPLATED_STATE_DIM = S_DIM;
  static const int TEMPLATED_CONTROL_DIM = C_DIM;
  static const int TEMPLATED_MAX_TIMESTEPS = MAX_TIMESTEPS;
  float dt_ = 0.01f;
  float lambda_ = 1.0;
  float alpha_ = 0.0;
  int num_timesteps_ = MAX_TIMESTEPS;
  int num_iters_ = 1;
  unsigned seed_ = (unsigned)std::chrono::system_clock::now().time_since_epoch().count();
  dim3 dynamics_rollout_dim_;  // accepted for source compatibility; the engine picks its own geometry
  dim3 cost_rollout_dim_;
  dim3 visualize_dim_ = dim3(32, 1, 1);
  int norm_exp_kernel_parallelization_ = 64;
  Eigen::Matrix<float, C_DIM, MAX_TIMESTEPS> init_control_traj_ = Eigen::Matrix<float, C_DIM, MAX_TIMESTEPS>::Zero();
  Eigen::Matrix<float, C_DIM, 1> slide_control_scale_ = Eigen::Matrix<float, C_DIM, 1>::Zero();
};

template <class DYN_T, class COST_T, class FB_T, class SAMPLING_T, int MAX_TIMESTEPS, int NUM_ROLLOUTS,
          class PARAMS_T = ControllerParams<DYN_T::STATE_DIM, DYN_T::CONTROL_DIM, MAX_TIMESTEPS>, int NUM_DISTRIBUTIONS = 1,
          unsigned ENGINE_FLAGS = 0u>
class Controller
{
public:
  typedef DYN_T TEMPLATED_DYNAMICS;
  typedef COST_T TEMPLATED_COSTS;
  typedef FB_T TEMPLATED_FEEDBACK;
  typedef PARAMS_T TEMPLATED_PARAMS;
  typedef SAMPLING_T TEMPLATED_SAMPLING;
  static const int TEMPLATED_DYNAMICS_STATE_DIM = DYN_T::STATE_DIM;
  using control_array = typename DYN_T::control_array;
  using state_array = typename DYN_T::state_array;
  using output_array = typename DYN_T::output_array;
  typedef Eigen::Matrix<float, DYN_T::CONTROL_DIM, MAX_TIMESTEPS> control_trajectory;
  typedef Eigen::Matrix<float, DYN_T::STATE_DIM, MAX_TIMESTEPS> state_trajectory;
  typedef Eigen::Matrix<float, DYN_T::OUTPUT_DIM, MAX_TIMESTEPS> output_trajectory;
  typedef Eigen::Matrix<float, NUM_ROLLOUTS, 1> sampled_cost_traj;
  typedef Eigen::Matrix<float, MAX_TIMESTEPS + 1, 1> cost_trajectory;  // +1 for terminal cost (controller.cuh:107)
#ifdef MPPIB_USING_EIGEN_SHIM
  typedef std::array<int, MAX_TIMESTEPS> crash_status_trajectory;  // the shim only carries float matrices
#else
  typedef Eigen::Matrix<int, MAX_TIMESTEPS, 1> crash_status_trajectory;  // controller.cuh:109
#endif

  Controller(DYN_T* model, COST_T* cost, FB_T* fb_controller, SAMPLING_T* sampler, float dt, int max_iter, float lambda,
             float alpha, int num_timesteps = MAX_TIMESTEPS,
             const Eigen::Ref<const control_trajectory>& init_control_traj = control_trajectory::Zero(),
             cudaStream_t stream = nullptr)
    : model_(model), cost_(cost), fb_controller_(fb_controller), sampler_(sampler)
  {
    params_.dt_ = dt;
    params_.num_iters_ = max_iter;
    params_.lambda_ = lambda;
    params_.alpha_ = alpha;
    params_.num_timesteps_ = (num_timesteps > 0 && num_timesteps <= MAX_TIMESTEPS) ? num_timesteps : MAX_TIMESTEPS;
    params_.init_control_traj_ = init_control_traj;
    control_ = init_control_traj;
    construct(stream);
  }
  Controller(DYN_T* model, COST_T* cost, FB_T* fb_controller, SAMPLING_T* sampler, PARAMS_T& params,
             cudaStream_t stream = nullptr)
    : model_(model), cost_(cost), fb_controller_(fb_controller), sampler_(sampler), params_(params)
  {
    control_ = params_.init_control_traj_;
    construct(stream);
  }
  virtual ~Controller()
  {  // controller.cuh:194-216: the controller frees the device side, not the plugin objects
    bindCostEngine(cost_, nullptr);
    if (engine_)
      mppib_destroy(engine_);
  }
  Controller(const Controller&) = delete;
  Controller& operator=(const Controller&) = delete;

  virtual void computeControl(const Eigen::Ref<const state_array>& state, int optimization_stride) = 0;
  virtual void slideControlSequence(int steps) = 0;
  virtual std::string getControllerName()
  {
    return "name not set";
  }

  // ---- sampled (visualisation) trajectories: controller.cuh:232,279-297,724-763, controller.cu:55-179 ----------------
  // The engine re-rolls the written-back controls of the last solve (mppib_sample_trajectories), so asking for sampled
  // trajectories turns MPPIB_FLAG_WRITEBACK_CONTROLS on (the engine is re-created once, like resizeSampledControlTrajectories
  // re-allocates the reference's buffers).
  void setPercentageSampledControlTrajectories(float new_perc)
  {
    perc_sampled_control_trajectories_ = new_perc;
    needWriteback();
  }
  void setTopNSampledControlTrajectories(int new_top_num_samples)
  {
    num_top_control_trajectories_ = new_top_num_samples;
    needWriteback();
  }
  float getPercentageSampledControlTrajectories() const
  {
    return perc_sampled_control_trajectories_;
  }
  int getNumberSampledTrajectories() const
  {
    return perc_sampled_control_trajectories_ * NUM_ROLLOUTS;
  }
  int getNumberTopControlTrajectories() const
  {
    return num_top_control_trajectories_;
  }
  int getTotalSampledTrajectories() const
  {
    return getNumberSampledTrajectories() + getNumberTopControlTrajectories();
  }
  virtual std::vector<output_trajectory> getSampledOutputTrajectories() const
  {
    return sampled_trajectories_;
  }
  virtual std::vector<cost_trajectory> getSampledCostTrajectories() const
  {
    return sampled_costs_;
  }
  virtual std::vector<crash_status_trajectory> getSampledCrashStatusTrajectories() const
  {
    return sampled_crash_status_;
  }
  std::vector<float> getTopNCosts() const
  {
    return top_n_costs_;
  }
  virtual std::vector<float> getTopTransformedCosts() const
  {  // controller.cuh:294-297
    return top_n_costs_;
  }
  // rollout index behind every sampled trajectory (-1 = the optimised control sequence)
  std::vector<int> getSampledIndices() const
  {
    return sampled_indices_;
  }
  // controllers/MPPI/mppi_controller.cu:262-298: launchVisualizeKernel + copies, here one C-ABI call
  virtual void calculateSampledStateTrajectories()
  {
    const int n = (int)sampled_indices_.size();
    if (n == 0 || !vis_inputs_valid_)
      return;
    const int T = getNumTimesteps();
    std::vector<float> out((size_t)n * T * DYN_T::OUTPUT_DIM), costs((size_t)n * (T + 1));
    std::vector<int> crash((size_t)n * T);
    MPPIB_HANDLE(mppib_sample_trajectories(engine_, vis_x0_.data(), vis_nominal_.data(), 0, sampled_indices_.data(), n,
                                           vis_opt_.data(), out.data(), costs.data(), crash.data()));
    sampled_trajectories_.assign(n, output_trajectory::Zero());
    sampled_costs_.assign(n, cost_trajectory::Zero());
    sampled_crash_status_.assign(n, crash_status_trajectory());
    for (int i = 0; i < n; i++)
    {
      for (int k = 0; k < T * DYN_T::OUTPUT_DIM; k++)
        sampled_trajectories_[i].data()[k] = out[(size_t)i * T * DYN_T::OUTPUT_DIM + k];
      for (int t = 0; t < T; t++)
      {
        sampled_costs_[i](t) = costs[(size_t)i * (T + 1) + t];
        sampled_crash_status_[i][t] = crash[(size_t)i * T + t];
      }
      for (int t = T; t < MAX_TIMESTEPS; t++)
        sampled_crash_status_[i][t] = 0;
      sampled_costs_[i](MAX_TIMESTEPS) = costs[(size_t)i * (T + 1) + T];  // terminal cost in the last slot
    }
  }

  // ---- names (controller.cuh:236-261) --------------------------------------------------------------------------------
  virtual std::string getDynamicsModelName() const
  {
    return model_->getDynamicsModelName();
  }
  virtual std::string getCostFunctionName() const
  {
    return cost_->getCostFunctionName();
  }
  virtual std::string getSamplingDistributionName() const
  {
    return sampler_->getSamplingDistributionName();
  }
  virtual std::string getFullName()
  {
    return getControllerName() + "(" + getDynamicsModelName() + ", " + getCostFunctionName() + ", " +
           getSamplingDistributionName() + ")";
  }
  // ---- host-only helpers of the base class (controller.cuh:317-393,530-533,620-622,765-768) --------------------------
  virtual void updateImportanceSampler(const Eigen::Ref<const control_trajectory>& nominal_control)
  {
    control_ = nominal_control;
  }
  // linear interpolation of a control trajectory at rel_time seconds after it was computed (controller.cuh:363-378)
  virtual control_array interpolateControls(double rel_time, control_trajectory& c_traj)
  {
    const int lower_idx = (int)(rel_time / getDt());
    const int upper_idx = lower_idx + 1;
    const double alpha = (rel_time - lower_idx * getDt()) / getDt();
    control_array out;
    for (int i = 0; i < DYN_T::CONTROL_DIM; i++)
      out(i) = (float)((1 - alpha) * c_traj(i, lower_idx) + alpha * c_traj(i, upper_idx));
    return out;
  }
  // controller.cuh:329-346: interpolated control plus, when feedback is enabled, the interpolated DDP feedback
  virtual control_array getCurrentControl(state_array& state, double rel_time, state_array& target_nominal_state,
                                          control_trajectory& c_traj)
  {
    control_array result = interpolateControls(rel_time, c_traj);
    if (enable_feedback_)
    {
      const control_array u_fb = interpolateFeedback(state, target_nominal_state, rel_time);
      for (int i = 0; i < DYN_T::CONTROL_DIM; i++)
        result(i) += u_fb(i);
    }
    state_array empty_state = model_->getZeroState();
    model_->enforceConstraints(empty_state, result);
    return result;
  }

  // ---- feedback (controller.cuh:263-268, 479-560, 709-721) ------------------------------------------------------------
  static constexpr bool kHasDDPFeedback = mppi_b200::has_ddp_feedback<FB_T>::value;
  virtual void initFeedback()
  {
    if constexpr (kHasDDPFeedback)
    {
      requireFeedbackController();
      enable_feedback_ = true;
      fb_controller_->initTrackingController();
    }
  }
  bool getFeedbackEnabled() const
  {
    return enable_feedback_;
  }
  void disableFeedbackController()
  {
    enable_feedback_ = false;
  }
  template <class FB_PARAMS>
  void setFeedbackParams(const FB_PARAMS& fb_params)
  {
    requireFeedbackController();
    fb_controller_->setParams(fb_params);
  }
  auto getFeedbackParams() const
  {
    return fb_controller_->getParams();
  }
  // DDP from `state` tracking state_traj / control_traj (ddp.cu:80-118)
  virtual void computeFeedbackHelper(const Eigen::Ref<const state_array>& state, const Eigen::Ref<const state_trajectory>& state_traj,
                                     const Eigen::Ref<const control_trajectory>& control_traj)
  {
    runFeedback(state, state_traj, control_traj, false);
  }
  virtual void computeFeedback(const Eigen::Ref<const state_array>& state)
  {
    computeFeedbackHelper(state, getTargetStateSeq(), getControlSeq());
  }
  virtual control_array getFeedbackControl(const Eigen::Ref<const state_array>& state,
                                           const Eigen::Ref<const state_array>& goal_state, int t)
  {
    if constexpr (kHasDDPFeedback)
      return fb_controller_->k(state, goal_state, t);
    return control_array::Zero();
  }
  virtual control_array interpolateFeedback(const Eigen::Ref<const state_array>& state,
                                            const Eigen::Ref<const state_array>& target_nominal_state, double rel_time)
  {
    if constexpr (kHasDDPFeedback)
      return fb_controller_->interpolateFeedback(state, target_nominal_state, rel_time);
    return control_array::Zero();
  }
  // controller.cuh:479-501: roll the actual start state forward with the control plus the feedback on the target states
  virtual void computeFeedbackPropagatedStateSeq()
  {
    if (!enable_feedback_)
      return;
    const state_trajectory target = getTargetStateSeq();
    const control_trajectory u_seq = getControlSeq();
    propagated_feedback_state_trajectory_.col(0) = state_.col(0);
    for (int i = 0; i < getNumTimesteps() - 1; i++)
    {
      state_array x = propagated_feedback_state_trajectory_.col(i), goal = target.col(i), xn, xdot;
      const control_array fb = getFeedbackControl(x, goal, i);
      control_array u;
      for (int c = 0; c < DYN_T::CONTROL_DIM; c++)
        u(c) = u_seq(c, i) + fb(c);
      output_array y;
      model_->step(x, xn, xdot, u, y, i, getDt());
      propagated_feedback_state_trajectory_.col(i + 1) = xn;
    }
  }
  state_trajectory getFeedbackPropagatedStateSeq() const
  {
    return propagated_feedback_state_trajectory_;
  }
  output_trajectory getActualOutputSeq() const
  {
    return output_;
  }
  virtual void resetControls()
  {  // controller.cuh:620-622 ("TODO" in the reference: a no-op there as well)
  }
  void setSlideControlScale(const Eigen::Ref<const control_array>& slide_control_scale)
  {
    params_.slide_control_scale_ = slide_control_scale;
  }
  // Controller::getSampledNoise (controller.cu:274-283): the sampler's control buffer, [NUM_ROLLOUTS][T][C]
  std::vector<float> getSampledNoise()
  {
    std::vector<float> v((size_t)NUM_DISTRIBUTIONS * NUM_ROLLOUTS * getNumTimesteps() * DYN_T::CONTROL_DIM);
    MPPIB_HANDLE(mppib_get_samples(engine_, v.data()));  // needs MPPIB_FLAG_WRITEBACK_CONTROLS (fails loudly otherwise)
    v.resize((size_t)NUM_ROLLOUTS * getNumTimesteps() * DYN_T::CONTROL_DIM);
    return v;
  }
  void setDebug(bool debug)
  {
    debug_ = debug;
  }
  bool getDebug() const
  {
    return debug_;
  }
  int getKernelChoiceAsInt() const
  {
    return (int)getKernelChoiceAsEnum();
  }

  // ---- getters (controller.cuh:409-436,510-517,773-776) ----------------------------------------------------------
  virtual control_trajectory getControlSeq() const
  {
    return control_;
  }
  virtual state_trajectory getTargetStateSeq() const
  {
    return state_;
  }
  virtual output_trajectory getTargetOutputSeq() const
  {
    return output_;
  }
  float getBaselineCost(int ind = 0) const
  {
    return baseline_[ind];
  }
  float getNormalizerCost(int ind = 0) const
  {
    return normalizer_[ind];
  }
  float getNormalizerPercent() const
  {
    return normalizer_[0] / NUM_ROLLOUTS;
  }
  MPPIFreeEnergyStatistics getFreeEnergyStatistics() const
  {
    return free_energy_statistics_;
  }
  sampled_cost_traj getSampledCostSeq()
  {  // trajectory costs of distribution 0 (raw costs; weights via mppib_get_weights)
    std::vector<float> c((size_t)NUM_DISTRIBUTIONS * NUM_ROLLOUTS);
    MPPIB_HANDLE(mppib_get_costs(engine_, c.data()));
    sampled_cost_traj r;
    for (int i = 0; i < NUM_ROLLOUTS; i++)
      r(i) = c[i];
    return r;
  }
  int getNumTimesteps() const
  {
    return params_.num_timesteps_;
  }
  float getDt() const
  {
    return params_.dt_;
  }
  float getLambda() const
  {
    return params_.lambda_;
  }
  float getAlpha() const
  {
    return params_.alpha_;
  }
  int getNumIters() const
  {
    return params_.num_iters_;
  }
  PARAMS_T getParams() const
  {
    return params_;
  }
  // controller.cuh:821-850
  virtual void setParams(const PARAMS_T& p)
  {
    const bool reseed = p.seed_ != params_.seed_;
    const bool retime = p.num_timesteps_ != params_.num_timesteps_;
    params_ = p;
    if (retime)
    {  // the horizon is baked into the engine's buffers
      createEngine();
    }
    else
    {
      pushParams();
      if (reseed)
        setSeedCUDARandomNumberGen(params_.seed_);
    }
  }
  void setDt(float dt)
  {
    params_.dt_ = dt;
    pushParams();
  }
  void setLambda(float lambda)
  {
    params_.lambda_ = lambda;
    pushParams();
  }
  void setAlpha(float alpha)
  {
    params_.alpha_ = alpha;
    pushParams();
  }
  void setNumIters(int n)
  {
    params_.num_iters_ = n;
  }
  void setNumTimesteps(int num_timesteps)
  {  // controller.cuh:665-676
    if (num_timesteps <= MAX_TIMESTEPS && num_timesteps > 0 && num_timesteps != params_.num_timesteps_)
    {
      params_.num_timesteps_ = num_timesteps;
      createEngine();
    }
  }
  // controller.cu:200-207: new seed, offset back to 0
  void setSeedCUDARandomNumberGen(unsigned seed)
  {
    params_.seed_ = seed;
    MPPIB_HANDLE(mppib_seed(engine_, seed, 0ULL));
  }
  void setCUDAStream(cudaStream_t stream)
  {  // controller.cuh:901: re-create the engine on the new stream
    stream_ = stream;
    createEngine();
  }
  // plugin parameters were edited through model_/cost_/sampler_: send them to the device (setParams -> paramsToDevice)
  void pushParams()
  {
    auto db = model_->blob();
    MPPIB_HANDLE(mppib_set_blob(engine_, MPPIB_BLOB_DYN_PARAMS, &db, sizeof(db)));
    auto cb = cost_->blob();
    MPPIB_HANDLE(mppib_set_blob(engine_, MPPIB_BLOB_COST_PARAMS, &cb, sizeof(cb)));
    auto sb = sampler_->blob();
    MPPIB_HANDLE(mppib_set_blob(engine_, MPPIB_BLOB_SAMPLER_PARAMS, &sb, sizeof(sb)));
    MPPIB_HANDLE(model_->pushModelBlobs(engine_));  // NN / LSTM weights
    pushCostmap(cost_);
    pushCostBlobs(cost_);
    MPPIB_HANDLE(mppib_set_solver(engine_, params_.dt_, params_.lambda_, params_.alpha_));
  }
  // kept for source compatibility (controller.cuh:299-302,886-894); the engine has a single fused kernel
  void setKernelChoice(kernelType)
  {
  }
  kernelType getKernelChoiceAsEnum() const
  {
    return kernelType::USE_SINGLE_KERNEL;
  }
  virtual void chooseAppropriateKernel()
  {  // mppi_controller.cu:44-143 draws one full noise buffer: keep the RNG in lock-step
    MPPIB_HANDLE(mppib_burn_draws(engine_, 1));
  }
  mppib_engine* engine()
  {
    return engine_;
  }

  // ---- host tail helpers (controller.cuh:557-663) -----------------------------------------------------------------
  void smoothControlTrajectoryHelper(Eigen::Ref<control_trajectory> u,
                                     const Eigen::Ref<const Eigen::Matrix<float, DYN_T::CONTROL_DIM, 2>>& control_history)
  {
    control_trajectory tmp = u;
    Eigen::Matrix<float, DYN_T::CONTROL_DIM, 2> h = control_history;
    mppib_host_smooth_controls(tmp.data(), h.data(), getNumTimesteps(), DYN_T::CONTROL_DIM);
    u = tmp;
  }
  virtual void slideControlSequenceHelper(int steps, Eigen::Ref<control_trajectory> u)
  {
    control_trajectory tmp = u;
    mppib_host_slide_controls(tmp.data(), steps, getNumTimesteps(), DYN_T::CONTROL_DIM, model_->zero_control_.data(),
                              params_.slide_control_scale_.data());
    u = tmp;
  }
  virtual void saveControlHistoryHelper(int steps, const Eigen::Ref<const control_trajectory>& u_trajectory,
                                        Eigen::Ref<Eigen::Matrix<float, DYN_T::CONTROL_DIM, 2>> u_history)
  {  // controller.cuh:602-616
    if (steps == 1)
    {
      u_history.col(0) = u_history.col(1);
      u_history.col(1) = u_trajectory.col(0);
    }
    else if (steps >= 2)
    {
      u_history.col(0) = u_trajectory.col(steps - 2);
      u_history.col(1) = u_trajectory.col(steps - 1);
    }
  }
  virtual void computeOutputTrajectoryHelper(Eigen::Ref<output_trajectory> output_result,
                                             Eigen::Ref<state_trajectory> state_result,
                                             const Eigen::Ref<const state_array>& x0,
                                             const Eigen::Ref<const control_trajectory>& u)
  {
    state_array x = x0;
    control_trajectory uu = u;
    state_trajectory st = state_trajectory::Zero();
    output_trajectory out = output_trajectory::Zero();
    MPPIB_HANDLE(model_->hostOutputTrajectory(x.data(), uu.data(), getNumTimesteps(), getDt(), st.data(), out.data()));
    state_result = st;
    output_result = out;
  }

  // Not in the reference: computeControl's host tail (smoothing + nominal roll-forward, controller.cuh:557-586, 643-663) as one
  // device kernel behind the solve (mppib_nominal_trajectory) instead of the host twins. Off by default (the host twins are
  // faster, DESIGN.md §9); VanillaMPPI / ColoredMPPI honour it.
  void setDeviceSideTail(bool on)
  {
    device_side_tail_ = on;
  }
  bool getDeviceSideTail() const
  {
    return device_side_tail_;
  }
  void deviceSideTail(const Eigen::Ref<const state_array>& x0, Eigen::Ref<control_trajectory> u,
                      const Eigen::Ref<const Eigen::Matrix<float, DYN_T::CONTROL_DIM, 2>>& control_history,
                      Eigen::Ref<state_trajectory> state_result, Eigen::Ref<output_trajectory> output_result)
  {
    state_array x = x0;
    control_trajectory uu = u, us = control_trajectory::Zero();
    Eigen::Matrix<float, DYN_T::CONTROL_DIM, 2> h = control_history;
    state_trajectory st = state_trajectory::Zero();
    output_trajectory out = output_trajectory::Zero();
    MPPIB_HANDLE(mppib_nominal_trajectory(engine_, x.data(), uu.data(), h.data(), us.data(), st.data(), out.data()));
    u = us;
    state_result = st;
    output_result = out;
  }

protected:
  bool enable_feedback_ = false;
  state_trajectory propagated_feedback_state_trajectory_ = state_trajectory::Zero();
  void requireFeedbackController()
  {
    if (!fb_controller_)
      throw std::runtime_error("this controller was built without a feedback controller (fb_controller == nullptr)");
  }
  // the DDP solve with the controller's trajectories, copied into the feedback controller's horizon
  void runFeedback(const Eigen::Ref<const state_array>& state, const Eigen::Ref<const state_trajectory>& state_traj,
                   const Eigen::Ref<const control_trajectory>& control_traj, bool to_rmppi)
  {
    if constexpr (kHasDDPFeedback)
    {
      if (!enable_feedback_)
        return;
      typename FB_T::state_trajectory st = FB_T::state_trajectory::Zero();
      typename FB_T::control_trajectory ct = FB_T::control_trajectory::Zero();
      const int n = std::min(getNumTimesteps(), (int)FB_T::FB_TIMESTEPS);
      for (int t = 0; t < n; t++)
      {
        for (int i = 0; i < DYN_T::STATE_DIM; i++)
          st(i, t) = state_traj(i, t);
        for (int i = 0; i < DYN_T::CONTROL_DIM; i++)
          ct(i, t) = control_traj(i, t);
      }
      state_array x = state;
      fb_controller_->computeFeedback(x, st, ct, to_rmppi);
    }
  }
  // every new engine is bound into the DDP feedback controller, so its solves run on the controller's engine and stream
  void bindFeedback()
  {
    if constexpr (kHasDDPFeedback)
      if (fb_controller_)
        fb_controller_->bindEngine(engine_);
  }
  bool device_side_tail_ = false;
  bool debug_ = false;
  unsigned extra_flags_ = 0u;  // engine flags a derived controller turns on at run time (re-creates the engine)
  float perc_sampled_control_trajectories_ = 0;  // controller.cuh:948-950
  int num_top_control_trajectories_ = 0;
  std::vector<float> top_n_costs_;
  std::vector<int> sampled_indices_;
  std::vector<output_trajectory> sampled_trajectories_;
  std::vector<cost_trajectory> sampled_costs_;
  std::vector<crash_status_trajectory> sampled_crash_status_;
  state_array vis_x0_ = state_array::Zero();
  control_trajectory vis_nominal_ = control_trajectory::Zero(), vis_opt_ = control_trajectory::Zero();
  bool vis_inputs_valid_ = false;
  std::mt19937 vis_gen_{ 0 };
  void needWriteback()
  {
    if (getTotalSampledTrajectories() > 0 && !(extra_flags_ & MPPIB_FLAG_WRITEBACK_CONTROLS))
    {
      extra_flags_ |= MPPIB_FLAG_WRITEBACK_CONTROLS;
      createEngine();
      vis_inputs_valid_ = false;
    }
  }
  // copySampledControlFromDevice + copyTopControlFromDevice (controller.cu:55-179), on rollout indices: slot 0 is the
  // optimised sequence, then distinct random rollouts from the first 98 % (the tail holds the pure-noise samples; all of
  // them in order above 98 %), then the top-n by weight = the n lowest trajectory costs
  void pickSampledControls(const Eigen::Ref<const state_array>& x0, const control_trajectory& u_nominal,
                           const control_trajectory& u_opt)
  {
    sampled_indices_.clear();
    top_n_costs_.clear();
    const int num_sampled = getNumberSampledTrajectories();
    if (num_sampled + num_top_control_trajectories_ <= 0)
      return;
    std::vector<float> c((size_t)NUM_DISTRIBUTIONS * NUM_ROLLOUTS);
    MPPIB_HANDLE(mppib_get_costs(engine_, c.data()));
    if (num_sampled > 0)
    {
      sampled_indices_.push_back(-1);
      if (perc_sampled_control_trajectories_ > 0.98f)
      {
        for (int i = 1; i < num_sampled; i++)
          sampled_indices_.push_back(i);
      }
      else
      {  // partial Fisher-Yates over [0, 0.98 N)
        std::vector<int> pool((size_t)(NUM_ROLLOUTS * 0.98));
        for (size_t i = 0; i < pool.size(); i++)
          pool[i] = (int)i;
        for (int i = 1; i < num_sampled && i <= (int)pool.size(); i++)
        {
          std::uniform_int_distribution<size_t> pick(i - 1, pool.size() - 1);
          std::swap(pool[i - 1], pool[pick(vis_gen_)]);
          sampled_indices_.push_back(pool[i - 1]);
        }
      }
    }
    if (num_top_control_trajectories_ > 0)
    {
      std::vector<int> order(NUM_ROLLOUTS);
      for (int i = 0; i < NUM_ROLLOUTS; i++)
        order[i] = i;
      const int k = std::min(num_top_control_trajectories_, NUM_ROLLOUTS);
      std::partial_sort(order.begin(), order.begin() + k, order.end(),
                        [&](int a, int b) { return c[a] < c[b] || (c[a] == c[b] && a < b); });
      for (int i = 0; i < k; i++)
      {
        sampled_indices_.push_back(order[i]);
        // trajectory_costs_[i] / normalizer (controller.cu:160): the normalised weight
        top_n_costs_.push_back(expf(-(c[order[i]] - baseline_[0]) / params_.lambda_) / normalizer_[0]);
      }
    }
    vis_x0_ = x0;
    vis_nominal_ = u_nominal;
    vis_opt_ = u_opt;
    vis_inputs_valid_ = true;
  }
  void construct(cudaStream_t stream)
  {
    stream_ = stream;
    for (int d = 0; d < NUM_DISTRIBUTIONS; d++)
      baseline_[d] = normalizer_[d] = 0.0f;
    createEngine();
  }
  // engine state that lives outside the parameter blobs (Tsallis weights, RMPPI gains / threshold): derived controllers
  // re-apply it here. Not reached from the base constructor (virtual dispatch), where they apply it themselves.
  virtual void onEngineCreated()
  {
  }
  void createEngine()
  {
    // a re-created engine must continue the noise stream where the old one stood (the reference keeps its generator across
    // setNumTimesteps / setCUDAStream), not restart it at offset 0
    unsigned long long rng_offset = 0ULL;
    const bool recreated = engine_ != nullptr;
    if (engine_)
    {
      MPPIB_HANDLE(mppib_get_rng_offset(engine_, &rng_offset));
      mppib_destroy(engine_);
      engine_ = nullptr;
    }
    mppib_desc d{};
    d.dynamics_id = DYN_T::DYN_ID;
    d.cost_id = COST_T::COST_ID;
    d.sampler_id = SAMPLING_T::SAMPLER_ID;
    d.num_rollouts = NUM_ROLLOUTS;
    d.num_timesteps = params_.num_timesteps_;
    d.num_distributions = NUM_DISTRIBUTIONS;
    d.device = 0;  // mppi_controller.cu:48
    d.flags = ENGINE_FLAGS | extra_flags_;  // e.g. MPPIB_FLAG_RMPPI for RobustMPPIController
    d.stream = (void*)stream_;
    d.rank = 0;
    d.world_size = 1;
    model_->fillModelDims(d.model_dims);
    MPPIB_HANDLE(mppib_create(&engine_, &d));
    pushParams();
    bindCostEngine(cost_, engine_);
    bindFeedback();
    // createAndSeedCUDARandomNumberGen (controller.cu:192-198) for a new controller; the old position for a re-creation
    MPPIB_HANDLE(mppib_seed(engine_, params_.seed_, recreated ? rng_offset : 0ULL));
    if (recreated)
      onEngineCreated();
  }
  template <class C>
  auto pushCostmap(C* c) -> decltype(c->costmapBytes(), void())
  {
    if (c->costmap())
      MPPIB_HANDLE(mppib_set_blob(engine_, MPPIB_BLOB_COSTMAP, c->costmap(), c->costmapBytes()));
  }
  void pushCostmap(...)
  {
  }
  // costs that push more than their parameter blob (QuadrotorMapCost: tex_helper_'s map), and that push it themselves when
  // their parameters change (updateWaypoint): they learn the engine of the controller built on them
  template <class C>
  auto pushCostBlobs(C* c) -> decltype(c->pushCostBlobs((mppib_engine*)nullptr), void())
  {
    c->pushCostBlobs(engine_);
  }
  void pushCostBlobs(...)
  {
  }
  template <class C>
  static auto bindCostEngine(C* c, mppib_engine* e) -> decltype(c->bindEngine(e), void())
  {
    if (c)
      c->bindEngine(e);
  }
  static void bindCostEngine(...)
  {
  }
  // one engine solve for all distributions; x0s [D][S], Us [D][T][C] in the engine's layout
  void solve(const float* x0s, const float* Us_in, int optimization_stride, int iter, float* Us_out)
  {
    mppib_solve_stats st[NUM_DISTRIBUTIONS];
    MPPIB_HANDLE(mppib_solve(engine_, x0s, Us_in, optimization_stride, iter, Us_out, st));
    for (int d = 0; d < NUM_DISTRIBUTIONS; d++)
    {
      baseline_[d] = st[d].baseline;
      normalizer_[d] = st[d].normalizer;
      float fe[3];
      mppib_host_free_energy(&st[d], NUM_ROLLOUTS, params_.lambda_, fe);
      freeEnergyEstimate& e = (d == 0) ? free_energy_statistics_.real_sys : free_energy_statistics_.nominal_sys;
      e.freeEnergyMean = fe[0];
      e.freeEnergyVariance = fe[1];
      e.freeEnergyModifiedVariance = fe[2];
    }
  }

  DYN_T* model_;
  COST_T* cost_;
  FB_T* fb_controller_;
  SAMPLING_T* sampler_;
  PARAMS_T params_;
  cudaStream_t stream_ = nullptr;
  mppib_engine* engine_ = nullptr;

  control_trajectory control_ = control_trajectory::Zero();
  Eigen::Matrix<float, DYN_T::CONTROL_DIM, 2> control_history_ = Eigen::Matrix<float, DYN_T::CONTROL_DIM, 2>::Zero();
  state_trajectory state_ = state_trajectory::Zero();
  output_trajectory output_ = output_trajectory::Zero();
  float baseline_[NUM_DISTRIBUTIONS];
  float normalizer_[NUM_DISTRIBUTIONS];
  MPPIFreeEnergyStatistics free_energy_statistics_;
};
