/* ARStandardCost — include/mppi/cost_functions/autorally/ar_standard_cost.cuh:14-230. The cost map is supplied in memory
 * (changeCostmapSize + setTrackData / updateTransform); npz loading (cnpy) is out of scope (SURVEY §2 row 26). */
#pragma once
#include <vector>

#include <cstdio>
#include <string>
#include <vector>

#include "../cost.hpp"

// float3 / float4 stand-ins: utils/common.hpp (included through cost.hpp)

struct ARStandardCostParams : public CostParams<2>
{
  float desired_speed = 6.0;
  float speed_coeff = 4.25;
  float track_coeff = 200.0;
  float max_slip_ang = 1.25;
  float slip_coeff = 10.0;
  float track_slop = 0;
  float crash_coeff = 10000;
  float boundary_threshold = 0.65;
  int grid_res = 10;
  float3 r_c1{};
  float3 r_c2{};
  float3 trs{};
  ARStandardCostParams()
  {
    control_cost_coeff[0] = 0.0;
    control_cost_coeff[1] = 0.0;
  }
};

namespace MPPI_internal
{
// The map-owning part of the Autorally map costs (ARStandardCostImpl, ar_standard_cost.cu:35-204): the costmap, its
// world->texture transform and the blob fields every map cost shares (mppib_ar_standard_cost_params, the prefix of each map
// cost's blob). ARStandardCost and ARRobustCost differ only in their params, blob and cost id.
template <class CLASS_T, class PARAMS_T, class BLOB_T, int COST_ID_V>
class ARMapCost : public Cost<CLASS_T, PARAMS_T, BLOB_T, COST_ID_V>
{
public:
  const float FRONT_D = 0.5;
  const float BACK_D = -0.5;
  bool l1_cost_ = false;
  int getWidth() const
  {
    return width_;
  }
  int getHeight() const
  {
    return height_;
  }
  bool changeCostmapSize(int width, int height)
  {  // ar_standard_cost.cu:35-60
    if (width <= 0 || height <= 0)
      return false;
    width_ = width;
    height_ = height;
    track_costs_.assign((size_t)width * height, float4{ 0, 0, 0, 0 });
    return true;
  }
  std::vector<float4>& getTrackCostCPU()
  {
    return track_costs_;
  }
  // in-memory equivalent of loadTrackData (ar_standard_cost.cu:85-142): channel arrays are row-major [height][width]
  void setTrackData(const float* ch0, const float* ch1, const float* ch2, const float* ch3, float x_min, float x_max,
                    float y_min, float y_max, float ppm)
  {
    changeCostmapSize(int((x_max - x_min) * ppm), int((y_max - y_min) * ppm));
    for (int i = 0; i < width_ * height_; i++)
      track_costs_[i] = float4{ ch0[i], ch1 ? ch1[i] : 0.0f, ch2 ? ch2[i] : 0.0f, ch3 ? ch3[i] : 0.0f };
    this->params_.r_c1 = float3{ 1.0f / (x_max - x_min), 0, 0 };
    this->params_.r_c2 = float3{ 0, 1.0f / (y_max - y_min), 0 };
    this->params_.trs = float3{ -x_min / (x_max - x_min), -y_min / (y_max - y_min), 1 };
  }
  // ARStandardCostImpl::loadTrackData (ar_standard_cost.cu:85-142): npz with "xBounds", "yBounds", "pixelsPerMeter" and
  // "channel0".."channel3" (float32, row-major [height][width]); returns the CPU copy like the reference (empty on error)
  std::vector<float4> loadTrackData(std::string map_path)
  {
    float xb[2], yb[2], ppm[1];
    if (mppib_host_npz_read(map_path.c_str(), "xBounds", xb, 2, nullptr, nullptr, nullptr) != MPPIB_OK ||
        mppib_host_npz_read(map_path.c_str(), "yBounds", yb, 2, nullptr, nullptr, nullptr) != MPPIB_OK ||
        mppib_host_npz_read(map_path.c_str(), "pixelsPerMeter", ppm, 1, nullptr, nullptr, nullptr) != MPPIB_OK)
    {
      fprintf(stderr, "ERROR: map path invalid, %s (%s)\n", map_path.c_str(), mppib_last_error());
      return std::vector<float4>();
    }
    const int width = int((xb[1] - xb[0]) * ppm[0]), height = int((yb[1] - yb[0]) * ppm[0]);
    if (width <= 0 || height <= 0)
    {
      fprintf(stderr, "ERROR: load track has invalid sizes\n");
      return std::vector<float4>();
    }
    std::vector<float> ch[4];
    for (int c = 0; c < 4; c++)
    {
      ch[c].resize((size_t)width * height);
      size_t n = 0;
      const std::string key = "channel" + std::to_string(c);
      if (mppib_host_npz_read(map_path.c_str(), key.c_str(), ch[c].data(), ch[c].size(), &n, nullptr, nullptr) != MPPIB_OK ||
          n != ch[c].size())
      {
        fprintf(stderr, "ERROR: %s of %s does not hold %d x %d values (%s)\n", key.c_str(), map_path.c_str(), width, height,
                mppib_last_error());
        return std::vector<float4>();
      }
    }
    setTrackData(ch[0].data(), ch[1].data(), ch[2].data(), ch[3].data(), xb[0], xb[1], yb[0], yb[1], ppm[0]);
    return track_costs_;
  }
  void updateTransform(const Eigen::Matrix3f& m, const Eigen::Vector3f& trs)
  {  // ar_standard_cost.cu:188-204
    this->params_.r_c1 = float3{ m(0, 0), m(1, 0), m(2, 0) };
    this->params_.r_c2 = float3{ m(0, 1), m(1, 1), m(2, 1) };
    this->params_.trs = float3{ trs(0), trs(1), trs(2) };
  }
  const float* costmap() const
  {
    return track_costs_.empty() ? nullptr : &track_costs_[0].x;
  }
  size_t costmapBytes() const
  {
    return track_costs_.size() * sizeof(float4);
  }
  BLOB_T blob() const
  {
    BLOB_T b{};
    const PARAMS_T& p = this->params_;
    this->fillBase(b);
    b.desired_speed = p.desired_speed;
    b.speed_coeff = p.speed_coeff;
    b.track_coeff = p.track_coeff;
    b.max_slip_ang = p.max_slip_ang;
    b.slip_coeff = p.slip_coeff;
    b.track_slop = p.track_slop;
    b.crash_coeff = p.crash_coeff;
    b.boundary_threshold = p.boundary_threshold;
    b.grid_res = p.grid_res;
    b.r_c1[0] = p.r_c1.x, b.r_c1[1] = p.r_c1.y, b.r_c1[2] = p.r_c1.z;
    b.r_c2[0] = p.r_c2.x, b.r_c2[1] = p.r_c2.y, b.r_c2[2] = p.r_c2.z;
    b.trs[0] = p.trs.x, b.trs[1] = p.trs.y, b.trs[2] = p.trs.z;
    b.l1_cost = l1_cost_ ? 1 : 0;
    b.front_d = FRONT_D;
    b.back_d = BACK_D;
    b.map_width = width_;
    b.map_height = height_;
    return b;
  }

protected:
  int width_ = -1, height_ = -1;
  std::vector<float4> track_costs_;
};
}  // namespace MPPI_internal

class ARStandardCost : public MPPI_internal::ARMapCost<ARStandardCost, ARStandardCostParams, mppib_ar_standard_cost_params,
                                                       MPPIB_COST_AR_STANDARD>
{
public:
  ARStandardCost(cudaStream_t stream = 0)
  {
  }
  std::string getCostFunctionName() const override
  {
    return "AutoRally standard cost function";
  }
};
