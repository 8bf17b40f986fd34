/*
 * noise_source.cuh — the engine's control-noise draw (K0 noise_xorwow.cuh, K0c noise_colored.cuh, the NLN draw) and the
 * sampler parameters it draws with. One member of mppib_engine; the definitions are in engine.cu.
 * A prefetched block is used only when it was drawn at the current offset, with the current sampler parameters, into a
 * buffer no kernel still reads: seed(), burn() and set_params() drop it, draw() takes it, and read_by_kernel() records
 * the kernel that the next draw into the current buffer waits for.
 * The smooth-MPPI sampler draws as the Gaussian one does and keeps, besides, the rate mean it carries from solve to solve
 * (device memory, zero at create): K1 reads it, the solve's merge replaces it, and burn() broadcasts its row 1, each on the
 * solve's stream, so back-to-back solves stay in order without the host.
 */
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/mppi_b200.h"
#include "device_resources.cuh"

namespace mppib
{
class NoiseSource : NoCopy
{
public:
  ~NoiseSource()  // drains the side stream before the members release themselves
  {
    if (side_)
      cudaStreamSynchronize(side_);
  }
  // Sampler desc.sampler_id's draw for rollouts [n_offset, n_offset + n_local) of N on `stream` (prefetch: on a stream
  // of `side_priority`): both buffers, the own-XORWOW tables, the ColoredNoise plan, the generator at seed 0, offset 0
  int create(const mppib_desc& desc, int N, int n_offset, int n_local, int T, int C, int num_sms, cudaStream_t stream,
             int side_priority);
  int set_params(const mppib_gaussian_params& sp);  // validated by mppib_set_blob
  const mppib_gaussian_params& params() const { return params_; }
  bool have_params() const { return have_params_; }
  int seed(unsigned long long seed, unsigned long long offset);
  int burn(int n);  // skip n blocks (smooth-MPPI: and shift the rate mean as each draw would)
  unsigned long long offset() const { return rng_offset_; }
  int set_offset_t(long long offset_t);  // optimization_stride a ColoredNoise draw assumes until a solve names its own
  int offset_t() const { return colored_offset_t_; }
  // The block at offset() into the current buffer, ordered on the solve's stream (the prefetched block when it is that
  // one), and offset() moves past it.
  int draw(int offset_t);
  cudaError_t read_by_kernel();  // a kernel enqueued on the solve's stream since draw() reads the current buffer
  int prefetch();                // the next block into the other buffer on the side stream (no-op without prefetch)
  float* buffer(int i) const { return eps_[i]; }
  int current() const { return cur_; }
  float* eps() const { return eps_[cur_]; }  // [n_local][T][C]
  bool own_kernel() const { return xw_enabled_; }
  int chunks() const { return xw_chunks_; }
  int rounds_per_chunk() const { return xw_rounds_per_chunk_; }
  // smooth-MPPI sampler (mppib_smooth_mppi_params): the rate mean [T][C] and the sampler's dt
  bool smooth() const { return sampler_ == MPPIB_SAMPLER_SMOOTH_MPPI; }
  float* rate_mean() const { return rate_mean_; }
  float smooth_dt() const { return smooth_dt_; }
  void set_smooth_dt(float dt) { smooth_dt_ = dt; }
  int read_rate_mean(float* host) const;   // drains the stream
  int write_rate_mean(const float* host);  // ordered on the stream

private:
  int gen_draw(int buf, cudaStream_t st, unsigned long long pos, int offset_t);
  int colored_rearrange(int buf, cudaStream_t st, int offset_t);

  Stream side_;                    // prefetch stream (null when prefetch is off); first, so that it is destroyed last
  cudaStream_t stream_ = nullptr;  // the solve's stream
  int sampler_ = MPPIB_SAMPLER_GAUSSIAN;
  int n_local_ = 0, T_ = 0, C_ = 0, num_sms_ = 0, world_ = 1;
  mppib_gaussian_params params_{};
  bool have_params_ = false;
  // normals per generateSamples call: Gaussian N*T*C (gaussian.cu:380-381), ColoredNoise 2*N*C*(T+1) (:343 of
  // colored_noise.cu)
  unsigned long long draw_global_ = 0;  // whole job
  unsigned long long draw_start_ = 0;   // this rank's first normal inside the call's block
  size_t draw_local_ = 0;               // this rank's normals
  // generator
  CurandGenerator gen_;
  unsigned long long seed_ = 0;
  unsigned long long rng_offset_ = 0;  // absolute position (in normals) of the next GLOBAL draw to be CONSUMED
  static constexpr unsigned long long kNoPos = ~0ULL;
  unsigned long long curand_pos_ = kNoPos;  // global draw position the library generator sits at (world_size == 1 only)
  // own XORWOW draw (noise_xorwow.cuh): 4096 * xw_chunks_ persistent states
  bool xw_enabled_ = false;             // sizes allow it and MPPIB_FLAG_CURAND_HOST_API not set
  unsigned long long xw_pos_ = kNoPos;  // global draw position the states sit at (kNoPos = must be initialised)
  int xw_chunks_ = 0, xw_rounds_per_chunk_ = 0;
  unsigned xw_lead_ = 0;                   // window mode: floats of the first round before this rank's slice
  unsigned long long xw_first_round_ = 0;  // first round of the window, relative to the block's position
  bool xw_window_ = false;                 // the slice starts / ends inside an 8192-normal round
  uint32_t xw_jump_ = 0;
  DeviceBuffer<uint32_t> xw_states_, xw_tables_;
  // double buffer: the draw for solve s+1 runs on the side stream while K1/K2 of solve s run (it depends on nothing but
  // the RNG position); without prefetch both entries are the one buffer. A valid prefetch is in eps_[cur_ ^ 1].
  DeviceBuffer<float> alloc_[2];  // allocations incl. the offset-alignment lead-in
  float* eps_[2] = { nullptr, nullptr };
  int cur_ = 0;
  Event k1_done_[2];   // the kernel that read eps_[i] has finished
  Event gen_done_[2];  // the draw into eps_[i] has finished
  Event last_gen_;     // last draw on either stream (generator state ordering)
  bool k1_recorded_[2] = { false, false };
  bool any_gen_ = false;
  bool prefetch_valid_ = false;
  unsigned long long prefetch_pos_ = 0;
  // ColoredNoise sampler (noise_colored.cuh)
  DeviceBuffer<float> spec_alloc_;  // allocation incl. the offset-alignment lead-in
  float* spec_ = nullptr;           // [n_local*C][T+1] complex (float2) spectrum == the raw draw
  DeviceBuffer<float> time_;        // [n_local*C][2T] cuFFT output, kept until the next draw
  DeviceBuffer<float> coeffs_, sigma_, decay_pow_;  // [C][T+1] f^(-beta_c/2), [C] sigma_c, [T] offset_decay_rate^t
  CufftPlan plan_;
  int colored_offset_t_ = 1;        // optimization_stride assumed by draws issued before a solve names its own
  int buf_offset_t_[2] = { 1, 1 };  // stride the colored block in eps_[i] was rearranged with
  Event rearr_;                     // last re-rearrange on the solve's stream (time_ must outlive it)
  bool rearr_recorded_ = false;
  // NLN sampler: C log-normal planes + one normal block per draw (nln.cu:114-128)
  DeviceBuffer<float> nln_;  // [C][N][T]
  // smooth-MPPI sampler
  DeviceBuffer<float> rate_mean_;  // [T][C]
  float smooth_dt_ = 0.015f;
};
}  // namespace mppib
