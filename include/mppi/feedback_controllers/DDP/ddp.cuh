// <mppi/feedback_controllers/DDP/ddp.cuh>: DDPParams and DDPFeedback with the reference's API
// (feedback_controllers/DDP/ddp.cuh:16-26, 97-141; ddp.cu:51-118). computeFeedback runs the iLQR solve of DDP::run on the GPU
// through the C ABI (mppib_set_ddp + mppib_ddp_feedback, kernel csrc/ddp_kernel.cuh); no Eigen decomposition is needed on
// the host. A controller binds its engine into its DDPFeedback (Controller::bindFeedback, re-bound in onEngineCreated); a
// DDPFeedback used standalone creates a minimal engine for its dynamics on first use. The solve uses the bound engine's dt,
// so a controller's DDPFeedback must be built with the controller's dt.
#pragma once
#include <mppi_b200/utils/common.hpp>

#include <cmath>
#include <vector>

template <class DYN_T>
struct DDPParams
{
  using StateCostWeight = Eigen::Matrix<float, DYN_T::STATE_DIM, DYN_T::STATE_DIM>;
  using Hessian = StateCostWeight;
  using ControlCostWeight = Eigen::Matrix<float, DYN_T::CONTROL_DIM, DYN_T::CONTROL_DIM>;

  StateCostWeight Q = StateCostWeight::Identity();
  Hessian Q_f = Hessian::Identity();
  ControlCostWeight R = ControlCostWeight::Identity();
  int num_iterations = 1;
};

// the gain trajectory K_t (C x S column-major per step = [t][s][c]), the layout mppib_set_rmppi takes
template <class DYN_T, int N_TIMESTEPS>
struct DDPFeedbackState
{
  static const int FEEDBACK_SIZE = DYN_T::CONTROL_DIM * DYN_T::STATE_DIM * N_TIMESTEPS;
  static const int NUM_TIMESTEPS = N_TIMESTEPS;
  std::vector<float> fb_gain_traj_ = std::vector<float>(FEEDBACK_SIZE, 0.0f);
};

template <class DYN_T, int NUM_TIMESTEPS>
class DDPFeedback
{
public:
  static const int S = DYN_T::STATE_DIM, C = DYN_T::CONTROL_DIM;
  static const int FB_TIMESTEPS = NUM_TIMESTEPS;
  typedef Eigen::Matrix<float, C, S> feedback_gain_matrix;
  typedef std::vector<feedback_gain_matrix> feedback_gain_trajectory;
  typedef typename DYN_T::state_array state_array;
  typedef typename DYN_T::control_array control_array;
  typedef Eigen::Matrix<float, S, NUM_TIMESTEPS> state_trajectory;
  typedef Eigen::Matrix<float, C, NUM_TIMESTEPS> control_trajectory;
  typedef DDPFeedbackState<DYN_T, NUM_TIMESTEPS> INTERNAL_STATE_T;
  typedef DDPParams<DYN_T> TEMPLATED_PARAMS;

  // OptimizerResult (ddp/result.h): the fields DDPFeedback fills
  struct Result
  {
    typename DDPFeedback::state_trajectory state_trajectory = DDPFeedback::state_trajectory::Zero();
    typename DDPFeedback::control_trajectory control_trajectory = DDPFeedback::control_trajectory::Zero();
    feedback_gain_trajectory feedback_gain = feedback_gain_trajectory(NUM_TIMESTEPS, feedback_gain_matrix::Zero());
  };

  DDPFeedback(DYN_T* model = nullptr, float dt = 0.01f, int num_timesteps = NUM_TIMESTEPS, cudaStream_t = 0)
    : model_(model), dt_(dt), num_timesteps_((num_timesteps > 0 && num_timesteps <= NUM_TIMESTEPS) ? num_timesteps
                                                                                                     : NUM_TIMESTEPS)
  {
  }
  ~DDPFeedback()
  {
    if (own_engine_)
      mppib_destroy(engine_);
  }
  DDPFeedback(const DDPFeedback&) = delete;
  DDPFeedback& operator=(const DDPFeedback&) = delete;

  // the engine computeFeedback runs on (a controller's); nullptr = create one on first use
  void bindEngine(mppib_engine* engine)
  {
    if (own_engine_)
      mppib_destroy(engine_);
    own_engine_ = false;
    engine_ = engine;
  }

  void setParams(const DDPParams<DYN_T>& params)
  {
    params_ = params;
  }
  DDPParams<DYN_T> getParams() const
  {
    return params_;
  }
  // ddp.cu:51-67: zero gain trajectory
  void initTrackingController()
  {
    result_ = Result();
    fb_state_ = INTERNAL_STATE_T();
  }

  // ddp.cu:80-118: DDP from init_state around goal_traj / control_traj (control_traj is also the initial control
  // sequence). to_rmppi = true (RobustMPPIController): the kernel also writes the gains into the bound engine's RMPPI
  // feedback buffer.
  void computeFeedback(const Eigen::Ref<const state_array>& init_state, const Eigen::Ref<const state_trajectory>& goal_traj,
                       const Eigen::Ref<const control_trajectory>& control_traj, bool to_rmppi = false)
  {
    mppib_engine* e = engineForSolve();
    const int T = num_timesteps_;
    std::vector<float> Q(S * S), Qf(S * S), R(C * C), x0(S), xt((size_t)T * S), ut((size_t)T * C);
    for (int i = 0; i < S; i++)
      for (int j = 0; j < S; j++)
      {
        Q[i * S + j] = params_.Q(i, j);
        Qf[i * S + j] = params_.Q_f(i, j);
      }
    for (int i = 0; i < C; i++)
      for (int j = 0; j < C; j++)
        R[i * C + j] = params_.R(i, j);
    for (int i = 0; i < S; i++)
      x0[i] = init_state(i);
    for (int t = 0; t < T; t++)
    {
      for (int i = 0; i < S; i++)
        xt[(size_t)t * S + i] = goal_traj(i, t);
      for (int i = 0; i < C; i++)
        ut[(size_t)t * C + i] = control_traj(i, t);
    }
    MPPIB_HANDLE(mppib_set_ddp(e, Q.data(), Qf.data(), R.data(), params_.num_iterations));
    std::vector<float> xs((size_t)T * S), us((size_t)T * C);
    MPPIB_HANDLE(mppib_ddp_feedback(e, T, x0.data(), xt.data(), ut.data(), to_rmppi ? 1 : 0, fb_state_.fb_gain_traj_.data(),
                                    xs.data(), us.data(), nullptr));
    for (int t = 0; t < T; t++)
    {
      for (int i = 0; i < S; i++)
        result_.state_trajectory(i, t) = xs[(size_t)t * S + i];
      for (int i = 0; i < C; i++)
        result_.control_trajectory(i, t) = us[(size_t)t * C + i];
      for (int s = 0; s < S; s++)
        for (int c = 0; c < C; c++)
          result_.feedback_gain[t](c, s) = fb_state_.fb_gain_traj_[((size_t)t * S + s) * C + c];
    }
  }

  // ddp.cuh:175-181: K_t (x_act - x_goal)
  control_array k(const Eigen::Ref<const state_array>& x_act, const Eigen::Ref<const state_array>& x_goal, int t) const
  {
    return k_(x_act, x_goal, t, fb_state_);
  }
  control_array k_(const Eigen::Ref<const state_array>& x_act, const Eigen::Ref<const state_array>& x_goal, int t,
                   const INTERNAL_STATE_T& fb_state) const
  {
    control_array u = control_array::Zero();
    const float* K = fb_state.fb_gain_traj_.data() + (size_t)t * S * C;
    for (int s = 0; s < S; s++)
    {
      const float e = x_act(s) - x_goal(s);
      for (int c = 0; c < C; c++)
        u(c) += K[s * C + c] * e;
    }
    return u;
  }
  // feedback.cuh:216-228
  control_array interpolateFeedback(const Eigen::Ref<const state_array>& state, const Eigen::Ref<const state_array>& goal_state,
                                    double rel_time) const
  {
    const int lower_idx = (int)(rel_time / dt_);
    const double alpha = (rel_time - lower_idx * dt_) / dt_;
    const control_array lo = k(state, goal_state, lower_idx), hi = k(state, goal_state, lower_idx + 1);
    control_array u;
    for (int c = 0; c < C; c++)
      u(c) = (float)((1 - alpha) * lo(c) + alpha * hi(c));
    return u;
  }
  const INTERNAL_STATE_T& getFeedbackState() const
  {
    return fb_state_;
  }
  feedback_gain_trajectory getFeedbackGainsEigen() const
  {
    return result_.feedback_gain;
  }
  std::vector<feedback_gain_matrix>& getFeedbackGainTrajectory()
  {
    return result_.feedback_gain;
  }
  float getDt() const
  {
    return dt_;
  }
  int getNumTimesteps() const
  {
    return num_timesteps_;
  }

  DYN_T* model_;
  Result result_;

private:
  mppib_engine* engineForSolve()
  {
    if (!engine_)
    {  // standalone: one small engine of the model's in-tree pair (Dynamics::DDP_COST_ID)
      mppib_desc d{};
      d.dynamics_id = DYN_T::DYN_ID;
      d.cost_id = DYN_T::DDP_COST_ID;
      d.num_rollouts = 32;
      d.num_timesteps = 2;
      d.num_distributions = 1;
      d.world_size = 1;
      MPPIB_HANDLE(mppib_create(&engine_, &d));
      own_engine_ = true;
      MPPIB_HANDLE(mppib_set_solver(engine_, dt_, 1.0f, 0.0f));
    }
    if (own_engine_)
    {  // the model's parameters may have changed since the last solve
      auto b = model_->blob();
      MPPIB_HANDLE(mppib_set_blob(engine_, MPPIB_BLOB_DYN_PARAMS, &b, sizeof(b)));
      MPPIB_HANDLE(model_->pushModelBlobs(engine_));
    }
    return engine_;
  }
  float dt_;
  int num_timesteps_;
  DDPParams<DYN_T> params_;
  INTERNAL_STATE_T fb_state_;
  mppib_engine* engine_ = nullptr;
  bool own_engine_ = false;
};
