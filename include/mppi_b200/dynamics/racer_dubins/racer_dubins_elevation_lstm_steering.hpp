/*
 * RacerDubinsElevationLSTMSteering — host class of
 * include/mppi/dynamics/racer_dubins/racer_dubins_elevation_lstm_steering.cuh:20-119 (parameters: racer_dubins.cuh:13-104,
 * racer_dubins_elevation.cuh:16-59). S19 C2 O28. Same constructor as the reference:
 *   RacerDubinsElevationLSTMSteering(init_input_dim, init_hidden_dim, init_output_layers,
 *                                    input_dim, hidden_dim, output_layers, init_len, stream)
 * The prediction LSTM (input_dim 4, head {hidden_dim + 4, L1, 1}) runs inside the rollout kernel; the init network
 * (LSTMLSTMHelper) only turns a history buffer into the initial hidden / cell state on the host (updateFromBuffer,
 * lstm_steering.cu:215-232) and is represented by that state (setInitialHiddenCell). Parameters: RacerDubinsElevationParams
 * (racer_dubins_elevation.hpp).
 */
#pragma once
#include <cmath>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "racer_dubins_elevation.hpp"

class RacerDubinsElevationLSTMSteering
  : public MPPI_internal::Dynamics<RacerDubinsElevationLSTMSteering, mppib_racer_lstm_dyn_params, MPPIB_DYN_RACER_LSTM, 19,
                                   2, 28>
{
public:
  typedef RacerDubinsElevationParams DYN_PARAMS_T;
  using PARENT = MPPI_internal::Dynamics<RacerDubinsElevationLSTMSteering, mppib_racer_lstm_dyn_params,
                                         MPPIB_DYN_RACER_LSTM, 19, 2, 28>;

  RacerDubinsElevationLSTMSteering(int init_input_dim, int init_hidden_dim, std::vector<int>& init_output_layers,
                                   int input_dim, int hidden_dim, std::vector<int>& output_layers, int init_len,
                                   cudaStream_t stream = 0)
    : hidden_dim_(hidden_dim)
  {
    if (input_dim != MPPIB_RACER_LSTM_INPUT_DIM)
      throw std::invalid_argument("the steering LSTM takes 4 inputs (lstm_steering.cu:148-151)");
    if (output_layers.size() != 3 || output_layers[0] != hidden_dim + input_dim || output_layers[2] != 1)
      throw std::invalid_argument("output_layers must be {hidden_dim + 4, L1, 1}");
    if (init_output_layers.empty() || init_output_layers.back() != 2 * hidden_dim)
      throw std::invalid_argument("init network must output 2 * hidden_dim values (lstm_lstm_helper.cu:11)");
    head_hidden_ = output_layers[1];
    theta_.assign((size_t)MPPIB_RACER_LSTM_NUM_PARAMS(hidden_dim_, head_hidden_), 0.0f);
    // the init network (LSTMLSTMHelper::init_model_, lstm_lstm_helper.cu:4-12): host-only, zero-initialised
    if (init_output_layers[0] != init_hidden_dim + init_input_dim)
      throw std::invalid_argument("init_output_layers[0] must be init_hidden_dim + init_input_dim (lstm_helper.cu:41)");
    init_input_dim_ = init_input_dim;
    init_hidden_dim_ = init_hidden_dim;
    init_len_ = init_len;
    init_layers_ = init_output_layers;
    init_lstm_.assign((size_t)4 * init_hidden_dim * init_hidden_dim + 4 * init_hidden_dim * init_input_dim + 6 * init_hidden_dim,
                      0.0f);
    size_t head = 0;
    for (size_t l = 0; l + 1 < init_layers_.size(); l++)
      head += (size_t)init_layers_[l] * init_layers_[l + 1] + init_layers_[l + 1];
    init_head_.assign(head, 0.0f);
  }
  // ---- the init network (LSTMLSTMHelper) ---------------------------------------------------------------------------
  // getInitModel()->setAllValues(lstm, output): LSTM block in lstm_helper.cu:72-88 order (with its own initial hidden / cell),
  // head in fnn_helper.cu:176-183 order
  void setAllValuesInit(const std::vector<float>& lstm, const std::vector<float>& output)
  {
    if (lstm.size() != init_lstm_.size() || output.size() != init_head_.size())
      throw std::invalid_argument("init network: expected " + std::to_string(init_lstm_.size()) + " + " +
                                  std::to_string(init_head_.size()) + " values");
    init_lstm_ = lstm;
    init_head_ = output;
  }
  int getInitLen() const
  {
    return init_len_;
  }
  // LSTMLSTMHelper::initializeLSTM (lstm_lstm_helper.cu:50-73). `buffer` is the reference's init_input_dim x cols matrix in
  // Eigen's column-major order (one column per past time step), cols >= init_len. The new initial hidden / cell state reaches
  // an existing engine with the next push of the model's blobs (Controller::setParams).
  void initializeLSTM(const float* buffer, int rows, int cols)
  {
    if (rows != init_input_dim_ || cols < init_len_)
      throw std::invalid_argument("initializeLSTM: buffer must be init_input_dim x (>= init_len)");
    mppib_host_init_lstm net{ init_lstm_.data(), init_input_dim_, init_hidden_dim_, init_head_.data(), init_layers_.data(),
                              (int)init_layers_.size(), init_len_ };
    std::vector<float> out((size_t)2 * hidden_dim_);
    MPPIB_HANDLE(mppib_host_lstm_initialize(&net, buffer, cols, out.data()));
    setInitialHiddenCell(std::vector<float>(out.begin(), out.begin() + hidden_dim_),
                         std::vector<float>(out.begin() + hidden_dim_, out.end()));
  }
  // racer_dubins_elevation_lstm_steering.cu:215-233 (buffer_trajectory = one vector of past values per key)
  bool updateFromBuffer(const std::map<std::string, std::vector<float>>& buffer)
  {
    const char* keys[3] = { "STEER_ANGLE", "STEER_ANGLE_RATE", "CAN_STEER_CMD" };
    for (const char* k : keys)
      if (buffer.find(k) == buffer.end())
        return false;
    const size_t cols = buffer.at("STEER_ANGLE").size();
    if (buffer.at("STEER_ANGLE_RATE").size() != cols || buffer.at("CAN_STEER_CMD").size() != cols || init_input_dim_ != 3)
      return false;
    std::vector<float> init_buffer(3 * cols);
    for (size_t t = 0; t < cols; t++)
    {
      init_buffer[3 * t] = buffer.at("STEER_ANGLE")[t] * 0.2f;
      init_buffer[3 * t + 1] = buffer.at("STEER_ANGLE_RATE")[t] * 0.2f;
      init_buffer[3 * t + 2] = buffer.at("CAN_STEER_CMD")[t];
    }
    initializeLSTM(init_buffer.data(), 3, (int)cols);
    return true;
  }
  void setParams(const DYN_PARAMS_T& p)
  {
    params_ = p;
  }
  DYN_PARAMS_T getParams() const
  {
    return params_;
  }
  bool checkRequiresBuffer() const
  {
    return true;  // lstm_steering.cu:15
  }
  void enforceLeash(const Eigen::Ref<const state_array>& state_true, const Eigen::Ref<const state_array>& state_nominal,
                    const Eigen::Ref<const state_array>& leash_values, Eigen::Ref<state_array> state_output) override
  {
    racer_enforce_leash<STATE_DIM>(state_true, state_nominal, leash_values, state_output);
  }
  int lstmBlock() const
  {
    return 4 * hidden_dim_ * hidden_dim_ + 4 * hidden_dim_ * MPPIB_RACER_LSTM_INPUT_DIM + 6 * hidden_dim_;
  }
  // LSTMHelper::loadParams (utils/nn_helpers/lstm_helper.cu:496-585) for the prediction network: npz arrays
  // "<prefix>lstm/weight_hh_l0" [4H][H], "lstm/weight_ih_l0" [4H][4], "lstm/bias_hh_l0" + "lstm/bias_ih_l0" [4H] in PyTorch's
  // gate order (input, forget, cell, output), head as "<prefix>output/dynamics_W<i>" / "_b<i>"; "model/" is tried first like
  // the reference does (:520-523). Packed order: i, f, o, c (lstm_helper.cu:72-88). The initial hidden / cell state (the init
  // network's output) is left untouched.
  void loadParamsLSTM(const std::string& model_path, std::string prefix = "")
  {
    if (!prefix.empty() && prefix.back() != '/')
      prefix += "/";
    if (mppib_host_npz_read(model_path.c_str(), ("model/" + prefix + "lstm/weight_hh_l0").c_str(), nullptr, 0, nullptr,
                            nullptr, nullptr) == MPPIB_OK)
      prefix = "model/" + prefix;
    const int H = hidden_dim_, I = MPPIB_RACER_LSTM_INPUT_DIM;
    auto read = [&](const std::string& name, size_t expect) {
      std::vector<float> v(expect);
      size_t n = 0;
      if (mppib_host_npz_read(model_path.c_str(), (prefix + name).c_str(), v.data(), v.size(), &n, nullptr, nullptr) !=
              MPPIB_OK ||
          n != expect)
        throw std::runtime_error("Could not load LSTM model (" + prefix + name + "): " + mppib_last_error());
      return v;
    };
    const std::vector<float> whh = read("lstm/weight_hh_l0", (size_t)4 * H * H), wih = read("lstm/weight_ih_l0", (size_t)4 * H * I),
                             bhh = read("lstm/bias_hh_l0", (size_t)4 * H), bih = read("lstm/bias_ih_l0", (size_t)4 * H);
    const int order[4] = { 0, 1, 3, 2 };  // file blocks i, f, c, o -> packed i, f, o, c
    std::vector<float> lstm(theta_.begin(), theta_.begin() + lstmBlock());
    size_t at = 0;
    for (int k : order)
      for (int i = 0; i < H * H; i++)
        lstm[at++] = whh[(size_t)k * H * H + i];
    for (int k : order)
      for (int i = 0; i < H * I; i++)
        lstm[at++] = wih[(size_t)k * H * I + i];
    for (int k : order)
      for (int i = 0; i < H; i++)
        lstm[at++] = (float)((double)bhh[k * H + i] + (double)bih[k * H + i]);
    const int IN = H + I, L1 = head_hidden_;
    std::vector<float> head;
    const std::vector<float> w1 = read("output/dynamics_W1", (size_t)L1 * IN), b1 = read("output/dynamics_b1", (size_t)L1),
                             w2 = read("output/dynamics_W2", (size_t)L1), b2 = read("output/dynamics_b2", 1);
    head.insert(head.end(), w1.begin(), w1.end());
    head.insert(head.end(), b1.begin(), b1.end());
    head.insert(head.end(), w2.begin(), w2.end());
    head.insert(head.end(), b2.begin(), b2.end());
    setAllValues(lstm, head);
  }
  const std::vector<float>& getTheta() const
  {  // packed LSTM block (incl. initial hidden / cell) followed by the packed head
    return theta_;
  }
  // LSTMHelper::setAllValues(lstm, output) (lstm_helper.cuh:65-72)
  void setAllValues(const std::vector<float>& lstm, const std::vector<float>& output)
  {
    if ((int)lstm.size() != lstmBlock() || lstm.size() + output.size() != theta_.size())
      throw std::invalid_argument("wrong number of LSTM / head parameters");
    for (float v : lstm)
      if (!std::isfinite(v))
        throw std::invalid_argument("LSTM parameters must be finite");
    for (float v : output)
      if (!std::isfinite(v))
        throw std::invalid_argument("LSTM parameters must be finite");
    std::copy(lstm.begin(), lstm.end(), theta_.begin());
    std::copy(output.begin(), output.end(), theta_.begin() + lstm.size());
  }
  // LSTMHelper::updateLSTMInitialStates (lstm_helper.cu:98-110)
  void setInitialHiddenCell(const std::vector<float>& hidden, const std::vector<float>& cell)
  {
    const int base = lstmBlock() - 2 * hidden_dim_;
    for (int i = 0; i < hidden_dim_; i++)
    {
      theta_[base + i] = hidden[i];
      theta_[base + hidden_dim_ + i] = cell[i];
    }
  }
  std::string getDynamicsModelName() const override
  {
    return "RACER Dubins LSTM Steering Model";
  }
  mppib_racer_lstm_dyn_params modelBlob() const
  {
    return racer_elevation_blob(params_);
  }
  // ---- engine hooks (controller.hpp) -------------------------------------------------------------------------------
  void fillModelDims(int* dims) const
  {
    dims[0] = hidden_dim_;
    dims[1] = head_hidden_;
  }
  int pushModelBlobs(mppib_engine* e) const
  {
    const int rc = mppib_set_blob(e, MPPIB_BLOB_LSTM_WEIGHTS, theta_.data(), theta_.size() * sizeof(float));
    if (rc != MPPIB_OK || !tex_helper_->hasData())
      return rc;
    const std::vector<unsigned char>& m = tex_helper_->blob();  // TwoDTextureHelper::copyToDevice
    return mppib_set_blob(e, MPPIB_BLOB_ELEVATION_MAP, m.data(), m.size());
  }
  // racer_dubins_elevation.cuh: getTextureHelper() — map 0 is the elevation map computeStaticSettling samples
  TwoDTextureHelper<float>* getTextureHelper()
  {
    return tex_helper_.get();
  }
  int hostOutputTrajectory(const float* x0, const float* u, int T, float dt, float* states, float* outputs) const
  {
    auto b = this->blob();
    std::vector<float> h(hidden_dim_), c(hidden_dim_);
    mppib_host_lstm net{ theta_.data(), hidden_dim_, head_hidden_, h.data(), c.data(), tex_helper_->header() };
    return mppib_host_output_trajectory_lstm(&b, &net, x0, u, T, dt, states, outputs);
  }
  // host step with the LSTM state kept inside the object, like the reference's host twin
  // (lstm_steering.cu:90-118; reset by initializeDynamics :230-237)
  void initializeDynamics(const Eigen::Ref<const state_array>&, const Eigen::Ref<const control_array>&,
                          Eigen::Ref<output_array>, float, float)
  {
    const int base = lstmBlock() - 2 * hidden_dim_;
    hidden_.assign(theta_.begin() + base, theta_.begin() + base + hidden_dim_);
    cell_.assign(theta_.begin() + base + hidden_dim_, theta_.begin() + base + 2 * hidden_dim_);
  }
  void step(Eigen::Ref<state_array> state, Eigen::Ref<state_array> next_state, Eigen::Ref<state_array> state_der,
            const Eigen::Ref<const control_array>& control, Eigen::Ref<output_array> output, const float /*t*/,
            const float dt)
  {
    if ((int)hidden_.size() != hidden_dim_)
    {
      output_array tmp;
      initializeDynamics(state, control, tmp, 0.0f, dt);
    }
    float x[19], u[2], xn[19], xd[19], y[28];
    for (int i = 0; i < 19; i++)
      x[i] = state(i);
    u[0] = control(0), u[1] = control(1);
    auto b = this->blob();
    mppib_host_lstm net{ theta_.data(), hidden_dim_, head_hidden_, hidden_.data(), cell_.data(), tex_helper_->header() };
    MPPIB_HANDLE(mppib_host_step_lstm(&b, &net, x, u, dt, xn, xd, y));
    for (int i = 0; i < 19; i++)
    {
      next_state(i) = xn[i];
      state_der(i) = xd[i];
    }
    for (int i = 0; i < 28; i++)
      output(i) = y[i];
  }

private:
  DYN_PARAMS_T params_;
  int hidden_dim_ = 4, head_hidden_ = 20;
  std::vector<float> theta_, hidden_, cell_;
  std::vector<float> init_lstm_, init_head_;  // the init network's weights (host only)
  std::vector<int> init_layers_;
  int init_input_dim_ = 0, init_hidden_dim_ = 0, init_len_ = 0;
  std::shared_ptr<TwoDTextureHelper<float>> tex_helper_ = std::make_shared<TwoDTextureHelper<float>>(1);
};
