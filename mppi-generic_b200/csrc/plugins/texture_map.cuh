/*
 * plugins/texture_map.cuh — TwoDTextureHelper<float> map 0 on the device, shared by the RACER models' elevation map
 * (dynamics.cuh) and QuadrotorMapCost's costmap (costs.cuh), and TwoDTextureHelper<float4> map 0, the suspension model's
 * normals map. All travel in the mppib_elevation_map_header format (params.h).
 *
 * The reference samples a CUDA texture (clamp, bilinear, normalised coordinates) on the device and interpolates in software
 * on the host (two_d_texture_helper.cu:151-243 queryTextureCPU); the hardware filter carries 8-bit weights, so the two
 * disagree by up to 2^-9 of a cell's value step. Here the device evaluates the HOST formula in FP32 from four plain loads
 * (read-only cache): device, host twin and oracle then agree to rounding.
 */
#pragma once
#include "../device_utils.cuh"
#include "../../../include/mppi_b200/params.h"

namespace mppib
{
namespace plugins
{
struct ElevationMap
{
  const float* data;  // [height][width]
  mppib_elevation_map_header hdr;
};

// TextureHelper::worldPoseToMapPose (texture_helper.cu:94-105): world -> map frame (x, y)
__device__ __forceinline__ float2 worldPoseToMapPose(const mppib_elevation_map_header& h, float wx, float wy, float wz)
{
  const float dx = wx - h.origin[0], dy = wy - h.origin[1], dz = wz - h.origin[2];
  return make_float2(h.rotations[0] * dx + h.rotations[1] * dy + h.rotations[2] * dz,
                     h.rotations[3] * dx + h.rotations[4] * dy + h.rotations[5] * dz);
}
// TextureHelper::worldPoseToTexCoord (texture_helper.cu:107-134): [m] -> [cells] -> normalised coordinate
__device__ __forceinline__ float2 worldPoseToTexCoord(const mppib_elevation_map_header& h, float wx, float wy, float wz)
{
  const float2 mp = worldPoseToMapPose(h, wx, wy, wz);
  return make_float2((mp.x / h.resolution[0]) / (float)h.width, (mp.y / h.resolution[1]) / (float)h.height);
}
// TwoDTextureHelper::queryTextureCPU (two_d_texture_helper.cu:151-243) at array coordinates qx = u * width - 0.5,
// qy = v * height - 0.5 (the value sits at the cell centre): clamp, bilinear
__device__ __forceinline__ float queryTextureBilinear(const ElevationMap& m, float qx, float qy)
{
  const mppib_elevation_map_header& h = m.hdr;
  const float xmax = (float)(h.width - 1), ymax = (float)(h.height - 1);
  qx = qx > xmax ? xmax : (qx <= 0.0f ? 0.0f : qx);  // cudaAddressModeClamp (a NaN coordinate stays NaN -> NaN value)
  qy = qy > ymax ? ymax : (qy <= 0.0f ? 0.0f : qy);
  if (!(qx == qx) || !(qy == qy))
    return __int_as_float(0x7fc00000);
  const int x0 = min((int)floorf(qx), h.width - 2), y0 = min((int)floorf(qy), h.height - 2);
  const float* r0 = m.data + (size_t)y0 * h.width + x0;
  const float q11 = __ldg(r0), q12 = __ldg(r0 + 1), q21 = __ldg(r0 + h.width), q22 = __ldg(r0 + h.width + 1);
  const float fx1 = (float)(x0 + 1) - qx, fx0 = qx - (float)x0;  // (x_max - x) / 1, (x - x_min) / 1
  const float fy1 = (float)(y0 + 1) - qy, fy0 = qy - (float)y0;
  const float lo = q11 * fx1 + q12 * fx0, hi = q21 * fx1 + q22 * fx0;
  return lo * fy1 + hi * fy0;
}
// TwoDTextureHelper::queryTextureAtWorldPose (texture_helper.cu:274-280). The normalised coordinate is formed and scaled
// back to cells in one expression per axis: the same arithmetic as worldPoseToTexCoord, kept in this order because the
// RACER kernels' instruction schedule depends on it.
__device__ __forceinline__ float elevation_at_world_pose(const ElevationMap& m, float wx, float wy, float wz)
{
  const mppib_elevation_map_header& h = m.hdr;
  const float2 mp = worldPoseToMapPose(h, wx, wy, wz);
  const float qx = ((mp.x / h.resolution[0]) / (float)h.width) * (float)h.width - 0.5f;
  const float qy = ((mp.y / h.resolution[1]) / (float)h.height) * (float)h.height - 0.5f;
  return queryTextureBilinear(m, qx, qy);
}

// TwoDTextureHelper<float4> map 0 (RacerDubinsElevationSuspension's normals map): the same header, float4 per cell
struct NormalsMap
{
  const float4* data;  // [height][width]
  mppib_elevation_map_header hdr;
};
// queryTextureBilinear above, channel by channel, from four 16-byte read-only loads
__device__ __forceinline__ float4 queryTextureBilinear4(const NormalsMap& m, float qx, float qy)
{
  const mppib_elevation_map_header& h = m.hdr;
  const float xmax = (float)(h.width - 1), ymax = (float)(h.height - 1);
  qx = qx > xmax ? xmax : (qx <= 0.0f ? 0.0f : qx);
  qy = qy > ymax ? ymax : (qy <= 0.0f ? 0.0f : qy);
  if (!(qx == qx) || !(qy == qy))
  {
    const float nan = __int_as_float(0x7fc00000);
    return make_float4(nan, nan, nan, nan);
  }
  const int x0 = min((int)floorf(qx), h.width - 2), y0 = min((int)floorf(qy), h.height - 2);
  const float4* r0 = m.data + (size_t)y0 * h.width + x0;
  const float4 q11 = __ldg(r0), q12 = __ldg(r0 + 1), q21 = __ldg(r0 + h.width), q22 = __ldg(r0 + h.width + 1);
  const float fx1 = (float)(x0 + 1) - qx, fx0 = qx - (float)x0;
  const float fy1 = (float)(y0 + 1) - qy, fy0 = qy - (float)y0;
  auto lerp2 = [&](float a11, float a12, float a21, float a22) {
    const float lo = a11 * fx1 + a12 * fx0, hi = a21 * fx1 + a22 * fx0;
    return lo * fy1 + hi * fy0;
  };
  return make_float4(lerp2(q11.x, q12.x, q21.x, q22.x), lerp2(q11.y, q12.y, q21.y, q22.y),
                     lerp2(q11.z, q12.z, q21.z, q22.z), lerp2(q11.w, q12.w, q21.w, q22.w));
}
__device__ __forceinline__ float4 normal_at_world_pose(const NormalsMap& m, float wx, float wy, float wz)
{
  const mppib_elevation_map_header& h = m.hdr;
  const float2 mp = worldPoseToMapPose(h, wx, wy, wz);
  const float qx = ((mp.x / h.resolution[0]) / (float)h.width) * (float)h.width - 0.5f;
  const float qy = ((mp.y / h.resolution[1]) / (float)h.height) * (float)h.height - 0.5f;
  return queryTextureBilinear4(m, qx, qy);
}

}  // namespace plugins
}  // namespace mppib
