/*
 * TwoDTextureHelper<float> / <float4> — host class of include/mppi/utils/texture_helpers/two_d_texture_helper.cuh (+ the
 * TextureHelper base, texture_helper.cuh:60-175) for the uses the in-scope models have, one map (index 0) each: the float
 * elevation map of the RACER models (sampled by RACER::computeStaticSettling, racer_dubins.cu:359-434, and by the
 * suspension model's wheels) and the float4 normals map of RacerDubinsElevationSuspension (MPPIB_BLOB_NORMALS_MAP). Same method names and argument meaning
 * (setExtent / updateTexture / updateOrigin / updateRotation / updateResolution / enableTexture / disableTexture /
 * checkTextureUse / copyToDevice / queryTextureAtWorldPose); the data is kept row-major as in cpu_values_ and travels to the
 * engine as MPPIB_BLOB_ELEVATION_MAP when the owning model's blobs are pushed (copyToDevice marks it dirty). The device side
 * evaluates the reference's HOST interpolation formula in FP32 (csrc/plugins/dynamics.cuh: elevation_at_world_pose).
 */
#pragma once
#include <array>
#include <cstring>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "../common.hpp"

template <class DATA_T>
class TwoDTextureHelper
{
  static_assert(std::is_same<DATA_T, float>::value || std::is_same<DATA_T, float4>::value,
                "the float elevation map and the float4 normals map are built");

public:
  explicit TwoDTextureHelper(int number = 1, cudaStream_t = nullptr)
  {
    if (number != 1)
      throw std::runtime_error("TwoDTextureHelper: one map (index 0) is built");
    memset(&hdr_, 0, sizeof(hdr_));
    hdr_.rotations[0] = hdr_.rotations[4] = hdr_.rotations[8] = 1.0f;
    hdr_.resolution[0] = hdr_.resolution[1] = hdr_.resolution[2] = 1.0f;
  }
  bool setExtent(int index, cudaExtent& extent)
  {
    check(index);
    if (extent.depth != 0)
      throw std::runtime_error("Error: extent in setExtent invalid, cannot use depth != 0 in 2D texture: using " +
                               std::to_string(extent.depth));
    const bool changed = (int)extent.width != hdr_.width || (int)extent.height != hdr_.height;
    hdr_.width = (int)extent.width;
    hdr_.height = (int)extent.height;
    dirty_ = true;
    return changed;
  }
  void updateTexture(const int index, std::vector<DATA_T>& values, bool column_major = false)
  {
    check(index);
    const int w = hdr_.width, h = hdr_.height;
    if ((int)values.size() != w * h)  // two_d_texture_helper.cu:27-32
      throw std::runtime_error(std::string("Error: invalid size to updateTexture ") + std::to_string(values.size()) +
                               " != " + std::to_string(w * h));
    values_.resize((size_t)w * h);
    if (column_major)
    {
      for (int j = 0; j < w; j++)
        for (int i = 0; i < h; i++)
          values_[(size_t)i * w + j] = values[(size_t)j * h + i];
    }
    else
      std::copy(values.begin(), values.end(), values_.begin());
    dirty_ = true;
  }
  void updateTexture(const int index, std::vector<DATA_T>& data, cudaExtent& extent, bool column_major = false)
  {
    setExtent(index, extent);
    updateTexture(index, data, column_major);
  }
  void updateOrigin(int index, float3 new_origin)
  {
    check(index);
    hdr_.origin[0] = new_origin.x, hdr_.origin[1] = new_origin.y, hdr_.origin[2] = new_origin.z;
    dirty_ = true;
  }
  void updateRotation(int index, std::array<float3, 3>& new_rotation)
  {
    check(index);
    for (int r = 0; r < 3; r++)
    {
      hdr_.rotations[3 * r] = new_rotation[r].x;
      hdr_.rotations[3 * r + 1] = new_rotation[r].y;
      hdr_.rotations[3 * r + 2] = new_rotation[r].z;
    }
    dirty_ = true;
  }
  void updateResolution(int index, float resolution)
  {
    check(index);
    hdr_.resolution[0] = hdr_.resolution[1] = hdr_.resolution[2] = resolution;
    dirty_ = true;
  }
  void updateResolution(int index, float3 resolution)
  {
    check(index);
    hdr_.resolution[0] = resolution.x, hdr_.resolution[1] = resolution.y, hdr_.resolution[2] = resolution.z;
    dirty_ = true;
  }
  void enableTexture(int index)
  {
    check(index);
    hdr_.use = 1;
    dirty_ = true;
  }
  void disableTexture(int index)
  {
    check(index);
    hdr_.use = 0;
    dirty_ = true;
  }
  bool checkTextureUse(int index) const
  {
    return index == 0 && hdr_.use != 0 && !values_.empty();
  }
  // The engine copy happens when the owning model pushes its blobs (Controller::setParams / engine creation); here the call
  // only finalises the host-side blob, so host queries (queryTextureAtWorldPose, the model's host step) see the new data.
  void copyToDevice(bool = false)
  {
    blob();
  }
  void GPUSetup()
  {
  }
  // TwoDTextureHelper::queryTextureCPU at a world pose (two_d_texture_helper.cu:151-243): clamp, bilinear, per channel;
  // without data: 0 / (0, 0, 1, 0)
  DATA_T queryTextureAtWorldPose(const int index, const float3& input)
  {
    check(index);
    if constexpr (std::is_same<DATA_T, float>::value)
      return mppib_host_elevation_at_world_pose(header(), input.x, input.y, input.z);
    else
    {
      float v[4];
      mppib_host_normals_at_world_pose(header(), input.x, input.y, input.z, v);
      return float4{ v[0], v[1], v[2], v[3] };
    }
  }
  // ---- engine hooks -------------------------------------------------------------------------------------------------
  bool hasData() const
  {
    return !values_.empty() && hdr_.width >= 2 && hdr_.height >= 2 && values_.size() == (size_t)hdr_.width * hdr_.height;
  }
  const std::vector<unsigned char>& blob()
  {  // mppib_elevation_map_header + values (params.h)
    if (dirty_ || blob_.empty())
    {
      blob_.resize(sizeof(hdr_) + values_.size() * sizeof(DATA_T));
      memcpy(blob_.data(), &hdr_, sizeof(hdr_));
      if (!values_.empty())
        memcpy(blob_.data() + sizeof(hdr_), values_.data(), values_.size() * sizeof(DATA_T));
      dirty_ = false;
    }
    return blob_;
  }
  const mppib_elevation_map_header* header()
  {
    return hasData() ? reinterpret_cast<const mppib_elevation_map_header*>(blob().data()) : nullptr;
  }

private:
  static void check(int index)
  {
    if (index != 0)
      throw std::runtime_error("TwoDTextureHelper: one map (index 0) is built");
  }
  mppib_elevation_map_header hdr_;
  std::vector<DATA_T> values_;
  std::vector<unsigned char> blob_;
  bool dirty_ = true;
};
