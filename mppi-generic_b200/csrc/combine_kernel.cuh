/*
 * combine_kernel.cuh — K2, the baseline / normaliser / weighted-average merge, for sm_90a.
 *
 * Completes what the reference does with three host round trips (controllers/MPPI/mppi_controller.cu:187-218):
 *   computeBaselineCost  (host min over N,        core/mppi_common.cu:858-900)
 *   normExpKernel        (w = expf(-(c-beta)/lambda), :686-701,958-966)
 *   computeNormalizer    (host double sum,         :1055-1063)   and the sums computeFreeEnergy needs (:1065-1081)
 *   weightedReductionKernel (U_t = sum_n (w_n/eta) u_n,t   :710-737,1115-1160)
 * K1 already produced, per block b, (beta_b, eta_b, sum w^2_b, V_b[t][c] = sum_n w_n u_n) against its LOCAL baseline.
 * With beta = min_b beta_b and s_b = expf(-(beta_b - beta)/lambda):
 *     eta = sum_b s_b eta_b,   sum w^2 = sum_b s_b^2 w2_b,   U = (sum_b s_b V_b) / eta
 * which is algebraically the reference's two-pass formula (w_n = expf(-(c_n-beta_b)/lambda) * s_b). A record whose
 * baseline is +inf (every cost +inf) is empty, s_b = 0 (softmin.h). The same kernel
 * merges the per-GPU records after the NCCL all-gather (records = ranks, normalize = 1).
 *
 * Launch: grid (ceil(TC/32), D), block 512 = 16 warps x 32 columns; block-wide warp-shuffle reductions, the rescale
 * factors s_b staged once in shared memory, four record loads in flight per thread.
 * Output record layout == input record layout: [beta, eta, sum_w2, pad, V or U (TC floats)].
 */
#pragma once
#include "device_utils.cuh"

namespace mppib
{
constexpr int kCombineCols = 32;     // one warp-width of columns per block: 128-byte coalesced record reads
constexpr int kCombineGroups = 16;   // 16 warps split the records
constexpr int kCombineMaxRecords = 4096;

constexpr int kSmoothMaxFloats = 2048;  // T*C of a smooth-MPPI engine (one distribution: rollout_kernel.cuh's kMaxMeanFloats)

// The smooth-MPPI merge (updateDistributionParamsFromDevice, smooth-MPPI.cu:204-240): the merged average of the rates is
// the new rate mean, kept on the device for the next solve's K1, and the result is U = mu + dmu_new dt. mu is the nominal
// control of the rollout being merged, carried in the parameter block.
struct SmoothMerge
{
  float* rate_mean;  // [T][C]
  float dt;
  float mu[kSmoothMaxFloats];
};

template <bool SMOOTH>
__device__ __forceinline__ void combine_body(const float* __restrict__ records, const float4* __restrict__ headers,
                                             int nrec, int D, int TC, int pstride, float lambda_inv, int normalize,
                                             float* __restrict__ out, float* __restrict__ out2, const SmoothMerge* sm)
{
  __shared__ float scale_sh[kCombineMaxRecords];  // s_b = expf(-(beta_b - beta)/lambda)
  __shared__ float red_f[kCombineGroups];
  __shared__ double red_d[2][kCombineGroups];
  __shared__ float acc_sh[kCombineGroups][kCombineCols];
  __shared__ float beta_sh, eta_sh;
  __shared__ double w2_sh;

  const int d = blockIdx.y;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int col = blockIdx.x * kCombineCols + lane;
  const float* rec = records + (size_t)d * pstride;
  const size_t rstride = (size_t)D * pstride;

  pdl_wait_prerequisites();  // launched with programmatic stream serialisation: K1's results are complete from here on

  // 1. global baseline: first-minimum VALUE == plain min (mppi_common.cu:858-900). Headers are a compact float4 array.
  float m = INFINITY;
  float4 h[(kCombineMaxRecords + kCombineCols * kCombineGroups - 1) / (kCombineCols * kCombineGroups)];
#pragma unroll
  for (int i = 0; i < (int)(sizeof(h) / sizeof(h[0])); i++)
  {
    const int b = tid + i * (int)blockDim.x;
    h[i] = (b < nrec) ? headers[(size_t)b * D + d] : make_float4(INFINITY, 0.0f, 0.0f, 0.0f);
    m = fminf(m, h[i].x);
  }
  m = warp_min(m);
  if (lane == 0)
    red_f[warp] = m;
  __syncthreads();
  if (tid == 0)
  {
    float v = red_f[0];
    for (int i = 1; i < kCombineGroups; i++)
      v = fminf(v, red_f[i]);
    beta_sh = v;
  }
  __syncthreads();
  const float beta = beta_sh;

  // 2. per-record rescale factors, normaliser (double accumulate, mppi_common.cu:1055-1063) and sum of squares
  double eta = 0.0, w2 = 0.0;
#pragma unroll
  for (int i = 0; i < (int)(sizeof(h) / sizeof(h[0])); i++)
  {
    const int b = tid + i * (int)blockDim.x;
    if (b < nrec)
    {
      const float s = softmin_weight(h[i].x, beta, lambda_inv);  // 0 for an empty record (baseline +inf)
      scale_sh[b] = s;
      eta += (double)s * (double)h[i].y;
      w2 += (double)s * (double)s * (double)h[i].z;
    }
  }
  eta = warp_sum(eta);
  w2 = warp_sum(w2);
  if (lane == 0)
  {
    red_d[0][warp] = eta;
    red_d[1][warp] = w2;
  }
  __syncthreads();
  if (tid == 0)
  {
    double e = 0.0, q = 0.0;
    for (int i = 0; i < kCombineGroups; i++)
    {
      e += red_d[0][i];
      q += red_d[1][i];
    }
    eta_sh = (float)e;  // narrowed to float like the reference's return value
    w2_sh = q;
  }
  __syncthreads();

  // 3. column sums: warp g takes records g, g+16, ... ; 4 independent loads in flight per thread
  float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
  if (col < TC)
  {
    const float* colp = rec + kPartialHeader + col;
    int b = warp;
    for (; b + 3 * kCombineGroups < nrec; b += 4 * kCombineGroups)
    {
      const float v0 = colp[(size_t)b * rstride];
      const float v1 = colp[(size_t)(b + kCombineGroups) * rstride];
      const float v2 = colp[(size_t)(b + 2 * kCombineGroups) * rstride];
      const float v3 = colp[(size_t)(b + 3 * kCombineGroups) * rstride];
      a0 = fmaf(scale_sh[b], v0, a0);
      a1 = fmaf(scale_sh[b + kCombineGroups], v1, a1);
      a2 = fmaf(scale_sh[b + 2 * kCombineGroups], v2, a2);
      a3 = fmaf(scale_sh[b + 3 * kCombineGroups], v3, a3);
    }
    for (; b < nrec; b += kCombineGroups)
      a0 = fmaf(scale_sh[b], colp[(size_t)b * rstride], a0);
  }
  acc_sh[warp][lane] = (a0 + a1) + (a2 + a3);
  __syncthreads();
  if (warp == 0)
  {
    float a = 0.0f;
#pragma unroll
    for (int gq = 0; gq < kCombineGroups; gq++)
      a += acc_sh[gq][lane];
    const float eta_f = eta_sh;
    float* o = out + (size_t)d * pstride;
    float* o2 = out2 ? out2 + (size_t)d * pstride : nullptr;
    if (col < TC)
    {
      float v = normalize ? a / eta_f : a;
      if constexpr (SMOOTH)
      {
        sm->rate_mean[col] = v;
        v = fmaf(v, sm->dt, sm->mu[col]);
      }
      o[kPartialHeader + col] = v;
      if (o2)
        o2[kPartialHeader + col] = v;
    }
    if (blockIdx.x == 0 && lane == 0)
    {
      o[0] = beta;
      o[1] = eta_f;
      o[2] = (float)w2_sh;
      o[3] = 0.0f;
      if (o2)
      {
        o2[0] = beta;
        o2[1] = eta_f;
        o2[2] = (float)w2_sh;
        o2[3] = 0.0f;
      }
    }
  }
}

__global__ void __launch_bounds__(kCombineCols* kCombineGroups)
    combine_kernel(const float* __restrict__ records,   // [nrec][D][pstride]  (V at [kPartialHeader..))
                   const float4* __restrict__ headers,  // [nrec][D] (beta_b, eta_b, sum w^2_b, -)
                   int nrec, int D, int TC, int pstride, float lambda_inv, int normalize,
                   float* __restrict__ out,    // [D][pstride] (device)
                   float* __restrict__ out2)   // optional second copy (mapped host result), may be nullptr
{
  combine_body<false>(records, headers, nrec, D, TC, pstride, lambda_inv, normalize, out, out2, nullptr);
}

// K2 of a smooth-MPPI engine (one rank, one distribution, normalised)
__global__ void __launch_bounds__(kCombineCols* kCombineGroups)
    combine_kernel_smooth(const float* __restrict__ records, const float4* __restrict__ headers, int nrec, int D, int TC,
                          int pstride, float lambda_inv, int normalize, float* __restrict__ out, float* __restrict__ out2,
                          const __grid_constant__ SmoothMerge sm)
{
  combine_body<true>(records, headers, nrec, D, TC, pstride, lambda_inv, normalize, out, out2, &sm);
}

// KX — cross-GPU exchange + merge in ONE kernel over NVLink peer memory (world_size > 1, after K2 has produced this
// rank's un-normalised record). Replaces ncclAllGather + record_headers_kernel + a second K2 (three launches and the
// collective's launch latency): every rank stores its record straight into slot [rank] of every peer's gather buffer
// (P2P stores through NVSwitch), publishes a per-slot sequence flag with release semantics at system scope, spins
// (acquire) until all world_size flags of its own buffer carry this solve's sequence number, and merges the records
// in rank order — the same log-sum-exp arithmetic as K2's merge, so every rank computes the identical result.
// Slots are double-buffered by the parity of the sequence number: a peer can only push solve s+2 after it has seen this
// rank's push of s+1, which this rank issues after it finished merging s.
struct PeerTable
{
  float* gather[8];     // peer r's gather buffer  [2][world][D][pstride]
  unsigned* flags[8];   // peer r's flag words     [2][world]
};

__global__ void __launch_bounds__(512)
    exchange_merge_kernel(const float* __restrict__ rank_rec, const __grid_constant__ PeerTable peers, int world, int rank,
                          int D, int TC, int pstride, float lambda_inv, unsigned seq, float* __restrict__ out,
                          float* __restrict__ out2)
{
  __shared__ float scale_sh[2][8];
  __shared__ float eta_sh[2];
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int par = (int)(seq & 1u);
  const int rec = D * pstride;
  pdl_wait_prerequisites();  // K2 (this rank's record) is complete from here on
  // ---- push --------------------------------------------------------------------------------------------------------
  for (int p = 0; p < world; p++)
  {
    float* dst = peers.gather[p] + ((size_t)par * world + rank) * rec;
    for (int i = tid; i < rec; i += nthr)
      dst[i] = rank_rec[i];
  }
  __threadfence_system();
  __syncthreads();
  if (tid < world)
  {
    unsigned* f = peers.flags[tid] + par * world + rank;
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(seq) : "memory");
  }
  // ---- wait for every rank's record of this solve --------------------------------------------------------------------
  if (tid < world)
  {
    const unsigned* f = peers.flags[rank] + par * world + tid;
    unsigned v;
    do
    {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
    } while (v != seq);
  }
  __syncthreads();
  // ---- merge (rank order) --------------------------------------------------------------------------------------------
  const float* g = peers.gather[rank] + (size_t)par * world * rec;
  if (tid < D)
  {
    const int d = tid;
    float beta = INFINITY;
    for (int r = 0; r < world; r++)
      beta = fminf(beta, g[(size_t)r * rec + d * pstride]);
    double eta = 0.0, w2 = 0.0;
    for (int r = 0; r < world; r++)
    {
      const float* h = g + (size_t)r * rec + d * pstride;
      const float s = softmin_weight(h[0], beta, lambda_inv);  // 0 for an empty record (baseline +inf)
      scale_sh[d][r] = s;
      eta += (double)s * (double)h[1];
      w2 += (double)s * (double)s * (double)h[2];
    }
    const float eta_f = (float)eta;
    eta_sh[d] = eta_f;
    float* o = out + (size_t)d * pstride;
    o[0] = beta, o[1] = eta_f, o[2] = (float)w2, o[3] = 0.0f;
    if (out2)
    {
      float* o2 = out2 + (size_t)d * pstride;
      o2[0] = beta, o2[1] = eta_f, o2[2] = (float)w2, o2[3] = 0.0f;
    }
  }
  __syncthreads();
  for (int i = tid; i < D * TC; i += nthr)
  {
    const int d = i / TC, col = i - d * TC;
    float a = 0.0f;
    for (int r = 0; r < world; r++)
      a = fmaf(scale_sh[d][r], g[(size_t)r * rec + d * pstride + kPartialHeader + col], a);
    const float v = a / eta_sh[d];
    out[(size_t)d * pstride + kPartialHeader + col] = v;
    if (out2)
      out2[(size_t)d * pstride + kPartialHeader + col] = v;
  }
}

// Tsallis weighting (TsallisTransform core/mppi_common.cu:968-985 + computeNormalizer + weightedReductionKernel), used by
// ColoredMPPIController when gamma and r are non-zero (ColoredMPPI/colored_mppi_controller.cu:199-217). These weights
// are not a function of (c - beta) that factors over block baselines, so the block partials of K1 cannot be rescaled:
// K2 supplies the global baseline (record[0]) and this kernel reduces the written-back controls with the Tsallis
// weights. grid (ceil(T*C / 32), D), block 16 warps x 32 columns; every block recomputes the normaliser (N floats).
__global__ void __launch_bounds__(512)
    tsallis_reduce_kernel(const float* __restrict__ costs,     // [D][n]
                          const float* __restrict__ controls,  // [D][n][TC] constrained sampled controls
                          int n, int D, int TC, int pstride, float gamma, float r,
                          float* __restrict__ out,   // [D][pstride]: in = K2's record (beta at [0]); out = Tsallis result
                          float* __restrict__ out2)  // optional mapped host copy
{
  __shared__ float acc_sh[16][32];
  __shared__ double eta_sh[16], w2_sh[16];
  const int d = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + lane;
  const float beta = out[(size_t)d * pstride];
  const float* c = costs + (size_t)d * n;
  const float* u = controls + (size_t)d * n * TC;
  const float inv_rm1 = 1.0f / (r - 1.0f);
  float a = 0.0f;
  double eta = 0.0, w2 = 0.0;
  for (int i = warp; i < n; i += 16)
  {
    const float cost_dif = c[i] - beta;
    float w = 0.0f;
    if (cost_dif < gamma)
      w = expf(logf(1.0f - cost_dif / gamma) * inv_rm1);
    eta += (double)w;
    w2 += (double)w * (double)w;
    if (col < TC)
      a = fmaf(w, u[(size_t)i * TC + col], a);
  }
  acc_sh[warp][lane] = a;
  if (lane == 0)
  {
    eta_sh[warp] = eta;
    w2_sh[warp] = w2;
  }
  __syncthreads();
  if (warp == 0)
  {
    double e = 0.0, e2 = 0.0;
    float s = 0.0f;
#pragma unroll
    for (int g = 0; g < 16; g++)
    {
      e += eta_sh[g];
      e2 += w2_sh[g];
      s += acc_sh[g][lane];
    }
    const float eta_f = (float)e;
    float* o = out + (size_t)d * pstride;
    float* o2 = out2 ? out2 + (size_t)d * pstride : nullptr;
    __syncwarp();
    if (col < TC)
    {
      const float v = s / eta_f;
      o[kPartialHeader + col] = v;
      if (o2)
        o2[kPartialHeader + col] = v;
    }
    if (blockIdx.x == 0 && lane == 0)
    {  // baseline stays; normaliser and sum of squares describe the Tsallis weights
      o[1] = eta_f;
      o[2] = (float)e2;  // the free-energy statistics are taken over the Tsallis weights (mppi_common.cu:1065-1081)
      o[3] = 0.0f;
      if (o2)
      {
        o2[0] = beta;
        o2[1] = eta_f;
        o2[2] = (float)e2;
        o2[3] = 0.0f;
      }
    }
  }
}

// rank record (output of a non-normalising combine) -> compact header, for the cross-rank merge after the all-gather
__global__ void record_headers_kernel(const float* __restrict__ records, int nrec, int D, int pstride,
                                      float4* __restrict__ headers)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nrec * D)
  {
    const float* r = records + (size_t)i * pstride;
    headers[i] = make_float4(r[0], r[1], r[2], 0.0f);
  }
}

// w_n = expf(-(c_n - beta)/lambda) for read-back (trajectory_costs_d_ after launchNormExpKernel); not on the hot path.
__global__ void weights_kernel(const float* __restrict__ costs, const float* __restrict__ final_rec, int n, int pstride,
                               float lambda_inv, float* __restrict__ w)
{
  const int d = blockIdx.y;
  const float beta = final_rec[(size_t)d * pstride];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    w[(size_t)d * n + i] = expf(-lambda_inv * (costs[(size_t)d * n + i] - beta));
}

}  // namespace mppib
