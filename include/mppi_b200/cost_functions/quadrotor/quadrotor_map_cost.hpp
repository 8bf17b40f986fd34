/* QuadrotorMapCost — include/mppi/cost_functions/quadrotor/quadrotor_map_cost.cuh:14-200. Device twin:
 * mppi-generic_b200/csrc/plugins/costs.cuh (QuadrotorMapCost). computeStateCost and the compute*Cost terms are the
 * reference's HOST bodies (host_twins.h: mppib_host_state_cost, mppib_host_quadrotor_map_term); the rollouts run its device
 * body, which adds the costmap term and the crash flag and leaves the waypoint term out (DESIGN.md §8). The reference's
 * float4 track texture (loadTrackData, changeCostmapSize, costmapToTexture, updateTransform, coorTransform, queryTexture*,
 * r_c1 / r_c2 / trs) is not built: no cost body reads it. The map the cost reads is tex_helper_'s map 0. */
#pragma once
#include <cmath>
#include <cstring>
#include <iostream>
#include <vector>

#include "../cost.hpp"
#include "../../utils/texture_helpers/two_d_texture_helper.hpp"

struct QuadrotorMapCostParams : public CostParams<4>
{
  float attitude_coeff = 10;
  float crash_coeff = 1000;
  float dist_to_waypoint_coeff = 0.0;
  float heading_coeff = 5;
  float heading_power = 1.0;  // power to take the difference in headings to
  float height_coeff = 5;
  float track_coeff = 10;
  float speed_coeff = 5;
  float track_slop = 0.0;
  float gate_pass_cost = -150;

  float4 curr_waypoint{ 0, 0, 0, 0 };
  float4 prev_waypoint{ 0, 0, 0, 0 };
  float3 curr_gate_left{ 0, 0, 0 };
  float3 curr_gate_right{ 0, 0, 0 };
  float3 prev_gate_left{ 0, 0, 0 };
  float3 prev_gate_right{ 0, 0, 0 };
  float4 end_waypoint{ NAN, NAN, NAN, NAN };

  float desired_speed = 5;            // [m/s]
  float gate_margin = 0.5;            // [m]
  float min_dist_to_gate_side = 0.5;  // [m]
  float track_boundary_cost = 2.5;
  float gate_width = 2.15;  // [m]

  QuadrotorMapCostParams()
  {
    for (int i = 0; i < 4; i++)
      control_cost_coeff[i] = 1;
  }
  // :62-76 / :78-90, run by the library so that every mirror writes the same bytes (cosf / sinf gate corners included)
  bool updateWaypoint(float x, float y, float z, float heading = 0)
  {
    mppib_quadrotor_map_cost_params b = toBlob();
    const int rc = mppib_host_quadrotor_map_update_waypoint(&b, x, y, z, heading);
    fromBlob(b);
    return rc == 1;
  }
  bool updateGateBoundaries(float left_x, float left_y, float left_z, float right_x, float right_y, float right_z)
  {
    mppib_quadrotor_map_cost_params b = toBlob();
    const int rc = mppib_host_quadrotor_map_update_gate_boundaries(&b, left_x, left_y, left_z, right_x, right_y, right_z);
    fromBlob(b);
    return rc == 1;
  }
  mppib_quadrotor_map_cost_params toBlob() const
  {
    mppib_quadrotor_map_cost_params b{};
    for (int i = 0; i < 4; i++)
      b.control_cost_coeff[i] = control_cost_coeff[i];
    b.discount = discount;
    b.attitude_coeff = attitude_coeff;
    b.crash_coeff = crash_coeff;
    b.dist_to_waypoint_coeff = dist_to_waypoint_coeff;
    b.heading_coeff = heading_coeff;
    b.heading_power = heading_power;
    b.height_coeff = height_coeff;
    b.track_coeff = track_coeff;
    b.speed_coeff = speed_coeff;
    b.track_slop = track_slop;
    b.gate_pass_cost = gate_pass_cost;
    put(b.curr_waypoint, curr_waypoint);
    put(b.prev_waypoint, prev_waypoint);
    put(b.curr_gate_left, curr_gate_left);
    put(b.curr_gate_right, curr_gate_right);
    put(b.prev_gate_left, prev_gate_left);
    put(b.prev_gate_right, prev_gate_right);
    put(b.end_waypoint, end_waypoint);
    b.desired_speed = desired_speed;
    b.gate_margin = gate_margin;
    b.min_dist_to_gate_side = min_dist_to_gate_side;
    b.track_boundary_cost = track_boundary_cost;
    b.gate_width = gate_width;
    return b;
  }

private:
  static void put(float* d, const float4& v)
  {
    d[0] = v.x, d[1] = v.y, d[2] = v.z, d[3] = v.w;
  }
  static void put(float* d, const float3& v)
  {
    d[0] = v.x, d[1] = v.y, d[2] = v.z;
  }
  void fromBlob(const mppib_quadrotor_map_cost_params& b)
  {  // only the waypoint / gate fields change
    curr_waypoint = float4{ b.curr_waypoint[0], b.curr_waypoint[1], b.curr_waypoint[2], b.curr_waypoint[3] };
    prev_waypoint = float4{ b.prev_waypoint[0], b.prev_waypoint[1], b.prev_waypoint[2], b.prev_waypoint[3] };
    curr_gate_left = float3{ b.curr_gate_left[0], b.curr_gate_left[1], b.curr_gate_left[2] };
    curr_gate_right = float3{ b.curr_gate_right[0], b.curr_gate_right[1], b.curr_gate_right[2] };
    prev_gate_left = float3{ b.prev_gate_left[0], b.prev_gate_left[1], b.prev_gate_left[2] };
    prev_gate_right = float3{ b.prev_gate_right[0], b.prev_gate_right[1], b.prev_gate_right[2] };
  }
};

class QuadrotorMapCost : public MPPI_internal::Cost<QuadrotorMapCost, QuadrotorMapCostParams,
                                                    mppib_quadrotor_map_cost_params, MPPIB_COST_QUADROTOR_MAP>
{
public:
  typedef Eigen::Matrix<float, 13, 1> output_array;
  QuadrotorMapCost(cudaStream_t stream = nullptr) : tex_helper_(new TwoDTextureHelper<float>(1, stream))
  {
  }
  ~QuadrotorMapCost()
  {
    delete tex_helper_;
  }
  QuadrotorMapCost(const QuadrotorMapCost&) = delete;
  QuadrotorMapCost& operator=(const QuadrotorMapCost&) = delete;
  std::string getCostFunctionName() const override
  {
    return std::string("Quadrotor Map Cost");
  }
  mppib_quadrotor_map_cost_params blob() const
  {
    return params_.toBlob();
  }

  // :63-90 (host body)
  float computeStateCost(const Eigen::Ref<const output_array> s, int timestep = 0, int* crash_status = nullptr)
  {
    const mppib_quadrotor_map_cost_params b = blob();
    float c = 0;
    mppi_b200::handle_status(mppib_host_state_cost(MPPIB_COST_QUADROTOR_MAP, &b, nullptr, s.data(), timestep,
                                                   crash_status, &c),
                             __FILE__, __LINE__);
    return c;
  }
  float terminalCost(const Eigen::Ref<const output_array>)
  {
    return 0;
  }
  float computeGateSideCost(const float* s)
  {
    return term(MPPIB_QMAP_GATE_SIDE, s);
  }
  float computeHeadingCost(const float* s)
  {
    return term(MPPIB_QMAP_HEADING, s);
  }
  float computeHeightCost(const float* s)
  {
    return term(MPPIB_QMAP_HEIGHT, s);
  }
  float computeSpeedCost(const float* s)
  {
    return term(MPPIB_QMAP_SPEED, s);
  }
  float computeStabilizingCost(const float* s)
  {
    return term(MPPIB_QMAP_STABILIZING, s);
  }
  float computeWaypointCost(const float* s)
  {
    return term(MPPIB_QMAP_WAYPOINT, s);
  }
  float distToWaypoint(const float* s, float4 waypoint)
  {
    const float w[4] = { waypoint.x, waypoint.y, waypoint.z, waypoint.w };
    return mppib_host_quadrotor_map_dist_to_waypoint(s, w);
  }

  // :154-196: the parameters (and tex_helper_'s map) go to the device only when something changed
  void updateWaypoint(float4 new_waypoint)
  {
    updateWaypoint(new_waypoint.x, new_waypoint.y, new_waypoint.z, new_waypoint.w);
  }
  void updateWaypoint(float x, float y, float z, float heading = 0)
  {
    if (params_.updateWaypoint(x, y, z, heading))
      paramsToDevice();
  }
  void updateGateBoundaries(float3 left_side, float3 right_side)
  {
    updateGateBoundaries(left_side.x, left_side.y, left_side.z, right_side.x, right_side.y, right_side.z);
  }
  void updateGateBoundaries(std::vector<float> boundaries)
  {
    if (boundaries.size() < 6)
    {
      std::cerr << "You need " << 6 - boundaries.size() << " more floats in the"
                << " call to updateGateBoundaries" << std::endl;
      return;
    }
    updateGateBoundaries(boundaries[0], boundaries[1], boundaries[2], boundaries[3], boundaries[4], boundaries[5]);
  }
  void updateGateBoundaries(float left_x, float left_y, float left_z, float right_x, float right_y, float right_z)
  {
    if (params_.updateGateBoundaries(left_x, left_y, left_z, right_x, right_y, right_z))
      paramsToDevice();
  }
  // Cost::paramsToDevice + tex_helper_->copyToDevice (:45-61), to the engine of the controller built on this cost
  void paramsToDevice()
  {
    if (!engine_)
      return;
    pushCostBlobs(engine_);
    params_pushes_++;
  }
  int paramsPushes() const
  {
    return params_pushes_;
  }

  // ---- engine hooks (controller.hpp) -------------------------------------------------------------------------------
  void bindEngine(mppib_engine* e)
  {
    engine_ = e;
  }
  void pushCostBlobs(mppib_engine* e)
  {
    const mppib_quadrotor_map_cost_params b = blob();
    MPPIB_HANDLE(mppib_set_blob(e, MPPIB_BLOB_COST_PARAMS, &b, sizeof(b)));
    if (tex_helper_->hasData())
    {
      const std::vector<unsigned char>& m = tex_helper_->blob();
      MPPIB_HANDLE(mppib_set_blob(e, MPPIB_BLOB_COST_TEXTURE, m.data(), m.size()));
    }
  }

  TwoDTextureHelper<float>* tex_helper_ = nullptr;

private:
  float term(int which, const float* s)
  {
    const mppib_quadrotor_map_cost_params b = blob();
    float c = 0;
    mppi_b200::handle_status(mppib_host_quadrotor_map_term(&b, which, s, &c), __FILE__, __LINE__);
    return c;
  }
  mppib_engine* engine_ = nullptr;
  int params_pushes_ = 0;
};
