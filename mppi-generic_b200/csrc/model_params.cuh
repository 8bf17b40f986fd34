/*
 * model_params.cuh — the model a solve runs: every blob mppib_set_blob takes except the sampler's parameters (those are
 * NoiseSource's). The dynamics and cost parameter blobs are host copies that every launch copies into its kernel arguments;
 * the NN and LSTM weights, the costmap texture and the three maps (the RACER elevation map, the suspension model's
 * normals map and QuadrotorMapCost's cost texture, all in the mppib_elevation_map_header format) live in device memory. One member of mppib_engine; the
 * definitions are in engine.cu.
 * - Which blobs a pair takes follows from its dynamics and cost ids, here only (uses()).
 * - A blob counts as set once its upload has succeeded; an upload that fails after its validation leaves it unset.
 * - Kernels read the device blobs (read_by_kernels()), so those may not change while a solve is in flight.
 * - A map that is not set reads as off (hdr.use == 0): flat ground, upright normals, no costmap term.
 */
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <vector>

#include "../../include/mppi_b200.h"
#include "device_resources.cuh"
#include "plugins/texture_map.cuh"

namespace mppib
{
class ModelParams : NoCopy
{
public:
  // the pair's ids, model_dims and parameter blob sizes; weights and maps are copied on `stream`, which is then drained
  void create(const mppib_desc& desc, size_t dyn_bytes, size_t cost_bytes, cudaStream_t stream);
  int set(int which, const void* host, size_t nbytes);  // every kind but MPPIB_BLOB_SAMPLER_PARAMS
  bool is_set(int which) const { return (set_ >> which) & 1u; }
  static bool read_by_kernels(int which);
  int ready_for_solve() const;  // the weights and the costmap the pair needs are set
  int ready_for_ddp() const;    // the dynamics parameters and the weights the pair needs are set

  const unsigned char* dyn() const { return dyn_.data(); }
  const unsigned char* cost() const { return cost_.data(); }
  const int* dims() const { return dims_; }  // mppib_desc.model_dims
  const float* nn_weights() const { return nn_.d; }
  const std::vector<float>& nn_weights_host() const { return nn_.h; }
  const float* lstm_weights() const { return lstm_.d; }
  const std::vector<float>& lstm_weights_host() const { return lstm_.h; }
  cudaTextureObject_t costmap() const { return costmap_; }
  plugins::ElevationMap elevation_map() const { return view(elev_, MPPIB_BLOB_ELEVATION_MAP); }
  plugins::ElevationMap cost_texture() const { return view(cost_tex_, MPPIB_BLOB_COST_TEXTURE); }
  plugins::NormalsMap normals_map() const
  {
    const plugins::ElevationMap v = view(normals_, MPPIB_BLOB_NORMALS_MAP);
    return plugins::NormalsMap{ reinterpret_cast<const float4*>(v.data), v.hdr };
  }

  // mppib_compute_control's roll-forward of one distribution through the library's host twins, with the host copies of
  // the blobs; the dynamics is a built-in one
  int host_roll(const float* x0, const float* u, int T, float dt, float* states, float* outputs) const;

private:
  struct Weights
  {
    DeviceBuffer<float> d;
    std::vector<float> h;  // for host_roll
  };
  struct Map
  {
    DeviceBuffer<float> d;  // width * height values of `channels` floats each, row-major
    mppib_elevation_map_header hdr{};
  };
  bool uses(int which) const;
  int upload_weights(Weights& w, int which, const char* what, const void* host, size_t nbytes);
  int upload_map(Map& m, int which, const char* what, const void* host, size_t nbytes, int channels = 1);
  plugins::ElevationMap view(const Map& m, int which) const
  {
    plugins::ElevationMap v{ m.d, m.hdr };
    if (!is_set(which))
      v.hdr.use = 0;
    return v;
  }

  cudaStream_t stream_ = nullptr;
  int dyn_id_ = 0, cost_id_ = 0;
  int dims_[sizeof(mppib_desc::model_dims) / sizeof(int)] = {};
  size_t dyn_bytes_ = 0, cost_bytes_ = 0;
  unsigned set_ = 0;  // bit `which`: blob `which` is set
  std::vector<unsigned char> dyn_, cost_;
  Weights nn_, lstm_;
  Map elev_, cost_tex_, normals_;
  // the elevation and normals map blobs as set (header + values), the host twins' format
  std::vector<unsigned char> elev_h_, normals_h_;
  ArrayTexture costmap_;               // float4 array + its texture object
};
}  // namespace mppib
