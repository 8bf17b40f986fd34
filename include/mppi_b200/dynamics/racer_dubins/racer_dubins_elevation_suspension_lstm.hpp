/*
 * RacerDubinsElevationSuspension — host class of
 * include/mppi/dynamics/racer_dubins/racer_dubins_elevation_suspension_lstm.cuh:14-170. S24 C2 O28. The
 * RacerDubinsElevationLSTMSteering vehicle whose roll, pitch and heave are integrated from four spring-damper wheels over
 * the elevation map (getTextureHelper()) and the normals map (getTextureHelperNormals()). Same constructors as the
 * reference:
 *   RacerDubinsElevationSuspension(init_input_dim, init_hidden_dim, init_output_layers, input_dim, hidden_dim,
 *                                  output_layers, init_len, stream)
 *   RacerDubinsElevationSuspension(path, stream)   the prediction network's architecture and weights from an npz file
 *                                                  (loadParamsLSTM); the init network stays zero
 * The steering network, its weights, model_dims and the init network are the LSTM model's, held by an inner
 * RacerDubinsElevationLSTMSteering whose methods this class forwards. One distribution only (VanillaMPPI, ColoredMPPI).
 */
#pragma once
#include <cmath>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "racer_dubins_elevation_lstm_steering.hpp"

// racer_dubins_elevation_suspension_lstm.cuh:14-64
struct RacerDubinsElevationSuspensionParams : public RacerDubinsElevationParams
{
  enum class WheelIndex : int { FL = 0, FR, BL, BR, NUM_WHEELS };
  enum class StateIndex : int
  {
    VEL_X = 0, YAW, POS_X, POS_Y, STEER_ANGLE, BRAKE_STATE, ROLL, PITCH, CG_POS_Z, CG_VEL_I_Z, ROLL_RATE, PITCH_RATE,
    STEER_ANGLE_RATE, UNCERTAINTY_POS_X, UNCERTAINTY_POS_Y, UNCERTAINTY_YAW, UNCERTAINTY_VEL_X, UNCERTAINTY_POS_X_Y,
    UNCERTAINTY_POS_X_YAW, UNCERTAINTY_POS_X_VEL_X, UNCERTAINTY_POS_Y_YAW, UNCERTAINTY_POS_Y_VEL_X, UNCERTAINTY_YAW_VEL_X,
    FILLER_1, NUM_STATES
  };
  float spring_k = 14000.0f;                                // [N / m]
  float drag_c = 1000.0f;                                   // [N * s / m]
  float mass = 1447.0f;                                     // [kg]
  float I_xx = 1.0f / 12 * mass * 2 * (1.5f * 1.5f);        // [kg * m^2]
  float I_yy = 1.0f / 12 * mass * (1.5f * 1.5f + 3.0f * 3.0f);  // [kg * m^2]
  float wheel_radius = 0.32f;                               // [m]
  float3 c_g = make_float3(2.981f * 0.5f, 0.0f, 0.0f);
};

// mppib_racer_suspension_dyn_params with the LSTM blob as base, so that Dynamics::blob() reaches the control limits as `lim`
struct RacerSuspensionBlob : mppib_racer_lstm_dyn_params
{
  float spring_k, drag_c, mass, I_xx, I_yy, wheel_radius, c_g[3];
};
static_assert(sizeof(RacerSuspensionBlob) == sizeof(mppib_racer_suspension_dyn_params), "blob layout");

class RacerDubinsElevationSuspension
  : public MPPI_internal::Dynamics<RacerDubinsElevationSuspension, RacerSuspensionBlob, MPPIB_DYN_RACER_SUSPENSION_LSTM,
                                   24, 2, 28>
{
public:
  typedef RacerDubinsElevationSuspensionParams DYN_PARAMS_T;
  using PARENT = MPPI_internal::Dynamics<RacerDubinsElevationSuspension, RacerSuspensionBlob,
                                         MPPIB_DYN_RACER_SUSPENSION_LSTM, 24, 2, 28>;

  RacerDubinsElevationSuspension(int init_input_dim, int init_hidden_dim, std::vector<int>& init_output_layers,
                                 int input_dim, int hidden_dim, std::vector<int>& output_layers, int init_len,
                                 cudaStream_t stream = 0)
    : net_(init_input_dim, init_hidden_dim, init_output_layers, input_dim, hidden_dim, output_layers, init_len, stream)
    , hidden_dim_(hidden_dim)
    , head_hidden_(output_layers[1])
  {
  }
  explicit RacerDubinsElevationSuspension(const std::string& path, cudaStream_t stream = 0)
    : RacerDubinsElevationSuspension(fromFile(path), stream)
  {
    net_.loadParamsLSTM(path);
  }

  std::string getDynamicsModelName() const override
  {
    return "RACER Dubins LSTM Steering and Suspension Model";
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
    return true;
  }
  void enforceLeash(const Eigen::Ref<const state_array>& state_true, const Eigen::Ref<const state_array>& state_nominal,
                    const Eigen::Ref<const state_array>& leash_values, Eigen::Ref<state_array> state_output) override
  {
    racer_enforce_leash<STATE_DIM>(state_true, state_nominal, leash_values, state_output);
  }

  // ---- the steering network and the init network (RacerDubinsElevationLSTMSteering's) ----------------------------------
  int lstmBlock() const
  {
    return net_.lstmBlock();
  }
  void setAllValues(const std::vector<float>& lstm, const std::vector<float>& output)
  {
    net_.setAllValues(lstm, output);
  }
  void loadParamsLSTM(const std::string& model_path, std::string prefix = "")
  {
    net_.loadParamsLSTM(model_path, prefix);
  }
  void setInitialHiddenCell(const std::vector<float>& hidden, const std::vector<float>& cell)
  {
    net_.setInitialHiddenCell(hidden, cell);
  }
  const std::vector<float>& getTheta() const
  {
    return net_.getTheta();
  }
  void setAllValuesInit(const std::vector<float>& lstm, const std::vector<float>& output)
  {
    net_.setAllValuesInit(lstm, output);
  }
  int getInitLen() const
  {
    return net_.getInitLen();
  }
  void initializeLSTM(const float* buffer, int rows, int cols)
  {
    net_.initializeLSTM(buffer, rows, cols);
  }
  bool updateFromBuffer(const std::map<std::string, std::vector<float>>& buffer)
  {
    return net_.updateFromBuffer(buffer);
  }

  // ---- the maps ----------------------------------------------------------------------------------------------------
  TwoDTextureHelper<float>* getTextureHelper()
  {
    return net_.getTextureHelper();
  }
  TwoDTextureHelper<float4>* getTextureHelperNormals()
  {
    return &normals_tex_helper_;
  }
  // racer_dubins_elevation_suspension_lstm.cuh:133-137: both maps take the same rotation
  void updateRotation(std::array<float3, 3>& rotation)
  {
    net_.getTextureHelper()->updateRotation(0, rotation);
    normals_tex_helper_.updateRotation(0, rotation);
  }

  // racer_dubins_elevation_suspension_lstm.cu:527-611: CG_POS_Z is the centre of gravity's z in the world frame, CG_VEL_I_Z
  // the base link's inertial vertical speed less OMEGA_Y * c_g.x, the uncertainty diagonal gets a 1e-6 floor; a missing
  // key gives an all-NaN state
  state_array stateFromMap(const std::map<std::string, float>& map)
  {
    const char* keys[] = { "VEL_X", "VEL_Z", "POS_X", "POS_Y", "POS_Z", "OMEGA_X", "OMEGA_Y", "ROLL", "PITCH", "YAW",
                           "STEER_ANGLE", "STEER_ANGLE_RATE", "BRAKE_STATE" };
    for (const char* k : keys)
      if (map.find(k) == map.end())
        return state_array::Constant(NAN);
    state_array s = state_array::Zero();
    const float3 g = params_.c_g;
    s(2) = map.at("POS_X");
    s(3) = map.at("POS_Y");
    s(0) = map.at("VEL_X");
    const float pitch = map.at("PITCH");
    const float bl_v_I_z = map.at("VEL_Z") * cosf(pitch) - map.at("VEL_X") * sinf(pitch);
    s(9) = bl_v_I_z - map.at("OMEGA_Y") * g.x;
    s(4) = map.at("STEER_ANGLE");
    s(12) = map.at("STEER_ANGLE_RATE");
    s(6) = map.at("ROLL");
    s(7) = pitch;
    s(1) = map.at("YAW");
    // bodyOffsetToWorldPoseEuler(c_g, (x, y, POS_Z), (roll, pitch, yaw)): the z row of Euler2DCM_NWU (host branch)
    float sr, cr, sp, cp;
    sincosf(s(6), &sr, &cr);
    sincosf(pitch, &sp, &cp);
    s(8) = -sp * g.x + sr * cp * g.y + cr * cp * g.z + map.at("POS_Z");
    s(10) = map.at("OMEGA_X");
    s(11) = map.at("OMEGA_Y");
    s(5) = map.at("BRAKE_STATE");
    for (int i = 13; i < 17; i++)
      if (s(i) < 1e-6f)
        s(i) = 1e-6f;
    return s;
  }

  RacerSuspensionBlob modelBlob() const
  {
    RacerSuspensionBlob b{};
    static_cast<mppib_racer_lstm_dyn_params&>(b) = racer_elevation_blob(params_);
    b.spring_k = params_.spring_k;
    b.drag_c = params_.drag_c;
    b.mass = params_.mass;
    b.I_xx = params_.I_xx;
    b.I_yy = params_.I_yy;
    b.wheel_radius = params_.wheel_radius;
    b.c_g[0] = params_.c_g.x, b.c_g[1] = params_.c_g.y, b.c_g[2] = params_.c_g.z;
    return b;
  }

  // ---- engine hooks (controller.hpp) -------------------------------------------------------------------------------
  void fillModelDims(int* dims) const
  {
    net_.fillModelDims(dims);
  }
  int pushModelBlobs(mppib_engine* e)
  {
    int rc = net_.pushModelBlobs(e);  // LSTM weights and the elevation map
    if (rc != MPPIB_OK || !normals_tex_helper_.hasData())
      return rc;
    const std::vector<unsigned char>& m = normals_tex_helper_.blob();
    return mppib_set_blob(e, MPPIB_BLOB_NORMALS_MAP, m.data(), m.size());
  }
  int hostOutputTrajectory(const float* x0, const float* u, int T, float dt, float* states, float* outputs)
  {
    auto b = this->blob();
    std::vector<float> h(hidden_dim_), c(hidden_dim_);
    mppib_host_lstm net{ net_.getTheta().data(), hidden_dim_, head_hidden_, h.data(), c.data(),
                         net_.getTextureHelper()->header() };
    return mppib_host_output_trajectory_racer_suspension(&b, &net, normals_tex_helper_.header(), x0, u, T, dt, states,
                                                         outputs);
  }
  // host step with the LSTM state kept inside the object (reset by initializeDynamics)
  void initializeDynamics(const Eigen::Ref<const state_array>&, const Eigen::Ref<const control_array>&,
                          Eigen::Ref<output_array>, float, float)
  {
    const int base = net_.lstmBlock() - 2 * hidden_dim_;
    const std::vector<float>& th = net_.getTheta();
    hidden_.assign(th.begin() + base, th.begin() + base + hidden_dim_);
    cell_.assign(th.begin() + base + hidden_dim_, th.begin() + base + 2 * hidden_dim_);
  }
  // racer_dubins_elevation_suspension_lstm.cu:168-197 (host step)
  void step(Eigen::Ref<state_array> state, Eigen::Ref<state_array> next_state, Eigen::Ref<state_array> state_der,
            const Eigen::Ref<const control_array>& control, Eigen::Ref<output_array> output, const float /*t*/,
            const float dt)
  {
    if ((int)hidden_.size() != hidden_dim_)
    {
      output_array tmp;
      initializeDynamics(state, control, tmp, 0.0f, dt);
    }
    float x[24], u[2], xn[24], xd[24], y[28];
    for (int i = 0; i < 24; i++)
      x[i] = state(i);
    u[0] = control(0), u[1] = control(1);
    auto b = this->blob();
    mppib_host_lstm net{ net_.getTheta().data(), hidden_dim_, head_hidden_, hidden_.data(), cell_.data(),
                         net_.getTextureHelper()->header() };
    MPPIB_HANDLE(mppib_host_step_racer_suspension(&b, &net, normals_tex_helper_.header(), x, u, dt, xn, xd, y));
    for (int i = 0; i < 24; i++)
    {
      next_state(i) = xn[i];
      state_der(i) = xd[i];
    }
    for (int i = 0; i < 28; i++)
      output(i) = y[i];
  }

private:
  // the architecture an npz file holds: H from "lstm/weight_hh_l0" [4H][H], L1 from "output/dynamics_W1" [L1][H + 4]
  struct Arch
  {
    int H, L1;
  };
  static Arch fromFile(const std::string& path)
  {
    std::string prefix;
    if (mppib_host_npz_read(path.c_str(), "model/lstm/weight_hh_l0", nullptr, 0, nullptr, nullptr, nullptr) == MPPIB_OK)
      prefix = "model/";
    int shape[4] = {}, nd = 0;
    size_t n = 0;
    Arch a{};
    if (mppib_host_npz_read(path.c_str(), (prefix + "lstm/weight_hh_l0").c_str(), nullptr, 0, &n, shape, &nd) != MPPIB_OK ||
        nd != 2)
      throw std::runtime_error("Could not load LSTM model (" + path + "): " + mppib_last_error());
    a.H = shape[1];
    if (mppib_host_npz_read(path.c_str(), (prefix + "output/dynamics_W1").c_str(), nullptr, 0, &n, shape, &nd) != MPPIB_OK ||
        nd != 2)
      throw std::runtime_error("Could not load LSTM head (" + path + "): " + mppib_last_error());
    a.L1 = shape[0];
    return a;
  }
  // the reference test's init network (3, 20, {23, 100, 2H}, init_len 11) around the file's prediction network
  RacerDubinsElevationSuspension(Arch a, cudaStream_t stream)
    : RacerDubinsElevationSuspension(a, { 23, 100, 2 * a.H }, { a.H + 4, a.L1, 1 }, stream)
  {
  }
  RacerDubinsElevationSuspension(Arch a, std::vector<int> init_layers, std::vector<int> layers, cudaStream_t stream)
    : RacerDubinsElevationSuspension(3, 20, init_layers, 4, a.H, layers, 11, stream)
  {
  }

  DYN_PARAMS_T params_;
  RacerDubinsElevationLSTMSteering net_;
  int hidden_dim_ = 4, head_hidden_ = 20;
  std::vector<float> hidden_, cell_;
  TwoDTextureHelper<float4> normals_tex_helper_{ 1 };
};
