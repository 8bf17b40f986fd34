/*
 * reduction.cuh — the back half of a solve: from K1's block partials to the result record the caller reads. K2
 * (combine_kernel.cuh), with the Tsallis reduction on one rank, and with the peer-memory exchange (KX) or the NCCL
 * all-gather across ranks. One member of mppib_engine; the definitions are in engine.cu.
 * K2 writes the record to device memory and straight into mapped pinned host memory, so read() needs no copy once the
 * stream has drained.
 */
#pragma once
#include <cuda_runtime.h>

#include "../../include/mppi_b200.h"
#include "combine_kernel.cuh"
#include "device_resources.cuh"

typedef struct ncclComm* ncclComm_t;

namespace mppib
{
class Reduction : NoCopy
{
public:
  ~Reduction();  // destroys the communicator and closes the peer mappings; the engine has drained the stream
  // K1's per-block outputs for `grid` blocks of D distributions over T*C controls, the result record and, for world > 1,
  // the rank record and the gather buffers; the merge runs on `stream`
  int create(int D, int TC, int grid, int world, int rank, cudaStream_t stream);
  // K1 re-planned at another grid (the steering LSTM's form chosen again): room for its partials, drained first
  int set_grid(int grid);
  float* partials() const { return partials_; }  // [grid][D][pstride]
  float4* headers() const { return headers_; }   // [grid][D] compact (beta, eta, sum w^2)
  int pstride() const { return pstride_; }       // floats per record: the header, then T*C, rounded up to 4
  const float* result() const { return result_; }  // [D][pstride] the last merge's record (device copy)
  // The merge of the partials K1 left. after_k1: K1 is the kernel just before on the stream, and K2 may start under it
  // (programmatic dependent launch). costs / controls: K1's [D][n_local] costs and written-back controls (Tsallis only).
  int enqueue(bool after_k1, const float* costs, const float* controls, int n_local, float lambda);
  // A smooth-MPPI engine's merge (one rank, exponential weights): also writes the new rate mean rate_mean [T][C], and the
  // result is mu + rate mean * dt
  int enqueue_smooth(bool after_k1, float lambda, float* rate_mean, float dt, const float* mu);
  void read(float* U_out, mppib_solve_stats* stats) const;  // after the stream has drained
  int set_tsallis(float gamma, float r, bool have_controls);  // both non-zero: Tsallis weights
  int comm_init(const void* unique_id_128);
  int p2p_handle(void* handle_64);
  int p2p_open(const void* handles);
  int set_p2p(bool on);
  bool ready() const { return world_ <= 1 || comm_ != nullptr; }  // a rank of several merges through NCCL or KX

private:
  cudaStream_t stream_ = nullptr;
  int D_ = 1, TC_ = 0, grid_ = 0, world_ = 1, rank_ = 0, pstride_ = 0;
  DeviceBuffer<float> partials_;
  DeviceBuffer<float4> headers_;
  DeviceBuffer<float> result_;
  PinnedBuffer<float> result_h_;    // mapped pinned host copy of result_, which K2 writes directly
  float* result_h_dev_ = nullptr;   // device alias of result_h_
  float tsallis_gamma_ = 0.0f, tsallis_r_ = 0.0f;
  // world > 1: this rank's record [D][pstride], the all-gathered records [world][D][pstride] and their headers [world][D]
  DeviceBuffer<float> rank_rec_;
  DeviceBuffer<float> gather_;
  DeviceBuffer<float4> gather_hdr_;
  ncclComm_t comm_ = nullptr;
  // peer-memory exchange (combine_kernel.cuh: exchange_merge_kernel)
  bool p2p_ = false;
  bool p2p_opened_ = false;
  DeviceBuffer<float> p2p_gather_;  // [2][world][D][pstride] followed by the flag words [2][world]
  PeerTable peers_{};
  void* peer_opened_[8] = { nullptr };
  unsigned p2p_seq_ = 0;
};
}  // namespace mppib
