/*
 * rollout_kernel_nn_tc.cuh — K1 for the Autorally pair (NeuralNetModel<7,2,3> + ARStandardCost) with the 6-32-32-4
 * forward pass on the Hopper warpgroup tensor cores (wgmma.mma_async, operands in shared memory, FP32 accumulators in
 * registers). Same contract and outputs as the generic rollout_kernel (rollout_kernel.cuh); only the place where the 1344
 * multiply-adds per step happen changes.
 *
 * Mapping. One CTA = 128 threads = one warpgroup = 128 samples: thread i owns sample i, so the per-sample code (control
 * sampling, constraints, kinematics, Euler update, map cost) stays thread-private exactly as in the SIMT kernel. A layer
 * is two m64 wgmma tiles (rows 0-63, 64-127) issued by the whole warpgroup. The operands live in shared memory in the
 * K-major / no-swizzle canonical layout ([k/4][row] slabs of 16 B). The accumulator fragment of a thread covers rows
 * 16w + g (+8) of each tile (w = warp, g = lane / 4), not its own sample: tanh and the hi/lo split are element-wise, so
 * each thread finishes the values it holds and writes them straight back as the next layer's A operand; the 4 outputs
 * of the last layer go back to their sample through a 2 KB table.
 *
 * Precision. TF32 alone (10-bit mantissa) is ~4e-4 off per layer and fails the FP32 parity bar of a 100-step
 * recurrence, so every product is the 3xTF32 split  a_hi*w_hi + a_lo*w_hi + a_hi*w_lo  (a_hi = rna_tf32(a), a_lo = a - a_hi).
 * Biases ride an extra K block against a constant-one activation column; weights and biases of the two tanh layers are
 * pre-scaled by 2*log2(e) so tanh(z) = 1 - 2/(exp2(z') + 1) needs no multiply.
 *
 * Shared memory per CTA ~85 KB (2-slab noise ring 32 KB, activations hi/lo 36 KB, weights hi/lo 14 KB, output table 2 KB,
 * small tables), so two CTAs are resident per SM and one covers the other's MMA round trips; the noise rows stream
 * through a two-slab TMA ring (the whole-horizon tile of the SIMT kernel would not leave room), and the epilogue
 * re-streams them (L2-resident) to form the block's exp-weighted control sum.
 */
#pragma once
#include "rollout_kernel.cuh"
#include "plugins/costs.cuh"
#include "plugins/dynamics.cuh"

namespace mppib
{
namespace nn_tc
{
constexpr int kRows = 128;          // samples per CTA == one warpgroup == two m64 tiles
constexpr int kSlabBytes = kRows * kChunkBytes;
constexpr int kAChunks = 10;        // 8 activation chunks (K = 32) + 2 chunks holding the constant-one column
constexpr float kTanhScale = 2.8853900817779268f;  // 2 * log2(e)

struct Smem
{
  uint32_t slabs, a_hi, a_lo, w1_hi, w1_lo, w2_hi, w2_lo, w3_hi, w3_lo, out, means, theta_c, weights, red, bars, total;
};
__host__ __device__ inline Smem layout(int TC, int T)
{
  Smem s;
  uint32_t off = 0;
  s.slabs = off;
  off += 2 * kSlabBytes;
  s.a_hi = off;
  off += kAChunks * kRows * 16;
  s.a_lo = off;
  off += 8 * kRows * 16;
  s.w1_hi = off;
  off += 2 * 32 * 16;
  s.w1_lo = off;
  off += 2 * 32 * 16;
  s.w2_hi = off;
  off += kAChunks * 32 * 16;
  s.w2_lo = off;
  off += kAChunks * 32 * 16;
  s.w3_hi = off;
  off += kAChunks * 8 * 16;
  s.w3_lo = off;
  off += kAChunks * 8 * 16;
  s.out = off;
  off += kRows * 16;
  s.means = off;
  off += ((uint32_t)(TC + 3) / 4) * 16;
  s.theta_c = off;
  off += ((uint32_t)(T + 3) / 4) * 16;
  s.weights = off;
  off += kRows * 4;
  s.red = off;
  off += 4 * 32 * 4 + 3 * 32 * 4;
  s.bars = off;
  off += 2 * 8;
  s.total = off + 1024;
  return s;
}

__device__ __forceinline__ float rna_tf32(float x)
{
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// wgmma shared-memory matrix descriptor, K-major, no swizzle (layout type 0): element (row, k) lives at
// base + (k/4)*LBO + (row/8)*SBO + (row%8)*16 + (k%4)*4
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}
__device__ __forceinline__ void wgmma_fence()
{
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit_and_wait()
{
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// D[64 x 32] (+)= A[64 x 8] * B[8 x 32], TF32 inputs, FP32 accumulate; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d)
{
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d)
      : "memory");
}
// D[64 x 8] (+)= A[64 x 8] * B[8 x 8]
__device__ __forceinline__ void wgmma_n8(float (&d)[4], uint64_t da, uint64_t db, uint32_t scale_d)
{
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %6, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k8.f32.tf32.tf32 {%0, %1, %2, %3}, %4, %5, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(da), "l"(db), "r"(scale_d)
      : "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d)
{
  if constexpr (N == 32)
    wgmma_n32(d, da, db, scale_d);
  else
    wgmma_n8(d, da, db, scale_d);
}
// One layer for the CTA's 128 rows: nkb K blocks of 8 (hi/lo split, three products each) plus, when `bias`, the
// constant-one block (chunks 8, 9 of A) against the bias rows of W (hi and lo). Issued by all four warps; returns with
// the accumulators complete.
template <int N>
__device__ __forceinline__ void mma_layer(float (&d)[2][N / 2], uint32_t a_hi_s, uint32_t a_lo_s, uint32_t w_hi_s,
                                          uint32_t w_lo_s, int nkb, bool bias)
{
  constexpr uint32_t kALbo = kRows * 16, kTile = 64 * 16, kWLbo = N * 16;
  wgmma_fence();
#pragma unroll 1
  for (int kb = 0; kb < nkb; kb++)
  {
    const uint64_t dwh = gmma_desc(w_hi_s + kb * 2 * kWLbo, kWLbo, 128);
    const uint64_t dwl = gmma_desc(w_lo_s + kb * 2 * kWLbo, kWLbo, 128);
#pragma unroll
    for (int m = 0; m < 2; m++)
    {
      const uint64_t dah = gmma_desc(a_hi_s + kb * 2 * kALbo + m * kTile, kALbo, 128);
      const uint64_t dal = gmma_desc(a_lo_s + kb * 2 * kALbo + m * kTile, kALbo, 128);
      wgmma_tf32<N>(d[m], dah, dwh, kb > 0 ? 1u : 0u);
      wgmma_tf32<N>(d[m], dal, dwh, 1u);
      wgmma_tf32<N>(d[m], dah, dwl, 1u);
    }
  }
  if (bias)
  {
    const uint64_t dwh = gmma_desc(w_hi_s + 8 * kWLbo, kWLbo, 128);
    const uint64_t dwl = gmma_desc(w_lo_s + 8 * kWLbo, kWLbo, 128);
#pragma unroll
    for (int m = 0; m < 2; m++)
    {
      const uint64_t dah = gmma_desc(a_hi_s + 8 * kALbo + m * kTile, kALbo, 128);
      wgmma_tf32<N>(d[m], dah, dwh, 1u);
      wgmma_tf32<N>(d[m], dah, dwl, 1u);
    }
  }
  wgmma_commit_and_wait();
}
// tanh of a pre-activation that was already scaled by 2*log2(e)
__device__ __forceinline__ float tanh_prescaled(float zs)
{
  float t, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(zs));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(t + 1.0f));
  return fmaf(-2.0f, r, 1.0f);
}
// The thread's accumulator fragment of a 32-wide layer -> tanh -> hi/lo TF32 parts -> chunks 0..7 of the A operand.
// Fragment element (m, 4j + e): row 64m + 16 warp + g + 8 (e >> 1), column 8j + 2q + (e & 1)  (g = lane / 4, q = lane % 4).
__device__ __forceinline__ void store_activations(unsigned char* a_hi, unsigned char* a_lo, int warp, int lane,
                                                  const float (&d)[2][16])
{
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int m = 0; m < 2; m++)
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int h = 0; h < 2; h++)
      {
        const int row = 64 * m + 16 * warp + g + 8 * h, col = 8 * j + 2 * q;
        const uint32_t off = (uint32_t)(col >> 2) * (kRows * 16) + row * 16 + (col & 3) * 4;
        const float v0 = tanh_prescaled(d[m][4 * j + 2 * h]), v1 = tanh_prescaled(d[m][4 * j + 2 * h + 1]);
        const float h0 = rna_tf32(v0), h1 = rna_tf32(v1);
        *reinterpret_cast<float2*>(a_hi + off) = make_float2(h0, h1);
        *reinterpret_cast<float2*>(a_lo + off) = make_float2(v0 - h0, v1 - h1);  // exact in FP32
      }
}
}  // namespace nn_tc

template <bool WRITEBACK>
__global__ void __launch_bounds__(nn_tc::kRows, 2)
    rollout_kernel_ar_tc(const __grid_constant__ RolloutArgs<plugins::AutorallyNNDynamics, plugins::ARStandardCost> args,
                         const __grid_constant__ CUtensorMap tmap)
{
  using namespace nn_tc;
  using DYN = plugins::AutorallyNNDynamics;
  using COST = plugins::ARStandardCost;
  constexpr int S = 7, C = 2, O = 8;

  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int T = args.T, TC = T * C, nchunks = args.nchunks;
  const Smem L = layout(TC, T);
  unsigned char* slabs = smem + L.slabs;
  float4* a_hi = reinterpret_cast<float4*>(smem + L.a_hi);
  float4* a_lo = reinterpret_cast<float4*>(smem + L.a_lo);
  float4* w1_hi = reinterpret_cast<float4*>(smem + L.w1_hi);
  float4* w1_lo = reinterpret_cast<float4*>(smem + L.w1_lo);
  float4* w2_hi = reinterpret_cast<float4*>(smem + L.w2_hi);
  float4* w2_lo = reinterpret_cast<float4*>(smem + L.w2_lo);
  float4* w3_hi = reinterpret_cast<float4*>(smem + L.w3_hi);
  float4* w3_lo = reinterpret_cast<float4*>(smem + L.w3_lo);
  float* means_s = reinterpret_cast<float*>(smem + L.means);
  float* theta_c = reinterpret_cast<float*>(smem + L.theta_c);
  float* w_s = reinterpret_cast<float*>(smem + L.weights);
  float* red_s = reinterpret_cast<float*>(smem + L.red);
  float4* out_s = reinterpret_cast<float4*>(smem + L.out);       // layer-3 outputs, [row] x 4
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bars);  // [0],[1]: slab full

  pdl_launch_dependents();
  const int row0 = blockIdx.x * kRows;
  const int n_loc = row0 + tid;
  const bool valid = n_loc < args.n_local;
  const int n_glob = args.n_offset + n_loc;

  // ---- one-time setup: barriers, first two noise slabs, weights ---------------------------------------------------
  if (tid == 0)
  {
    tma_prefetch_desc(&tmap);
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0)
  {
    for (int k = 0; k < 2 && k < nchunks; k++)
    {
      mbar_arrive_expect_tx(&bars[k], kSlabBytes);
      tma_load_2d(slabs + k * kSlabBytes, &tmap, k * kChunkFloats, row0, &bars[k]);
    }
  }
  {
    // weights: reference packed layout (fnn_helper.cu:176-183) -> K-major [k/4][n] float4 slabs, hi/lo TF32 parts;
    // k == fan_in is the bias column; the tanh layers are pre-scaled by 2*log2(e)
    const float* g = args.dyn_aux.theta_d;
    auto put = [](float4* hi, float4* lo, int idx, int comp, float v) {
      const float h = rna_tf32(v);
      reinterpret_cast<float*>(&hi[idx])[comp] = h;
      reinterpret_cast<float*>(&lo[idx])[comp] = v - h;
    };
    for (int i = tid; i < 2 * 32 * 4; i += kRows)
    {  // layer 1: K = 8 (6 inputs, bias at k = 6, zero at k = 7), N = 32
      const int kc = i / (32 * 4), n = (i / 4) % 32, c = i % 4, k = kc * 4 + c;
      const float v = (k < 6) ? g[n * 6 + k] : (k == 6 ? g[192 + n] : 0.0f);
      put(w1_hi, w1_lo, kc * 32 + n, c, v * kTanhScale);
    }
    for (int i = tid; i < kAChunks * 32 * 4; i += kRows)
    {  // layer 2: K = 32 (+ bias at k = 32), N = 32
      const int kc = i / (32 * 4), n = (i / 4) % 32, c = i % 4, k = kc * 4 + c;
      const float v = (k < 32) ? g[224 + n * 32 + k] : (k == 32 ? g[1248 + n] : 0.0f);
      put(w2_hi, w2_lo, kc * 32 + n, c, v * kTanhScale);
    }
    for (int i = tid; i < kAChunks * 8 * 4; i += kRows)
    {  // layer 3: K = 32 (+ bias), N = 8 (4 outputs, rows 4..7 zero), linear
      const int kc = i / (8 * 4), n = (i / 4) % 8, c = i % 4, k = kc * 4 + c;
      float v = 0.0f;
      if (n < 4)
        v = (k < 32) ? g[1280 + n * 32 + k] : (k == 32 ? g[1408 + n] : 0.0f);
      put(w3_hi, w3_lo, kc * 8 + n, c, v);
    }
    // constant-one activation column (chunk 8 = (1,0,0,0), chunk 9 = 0) — written once
    a_hi[8 * kRows + tid] = make_float4(1.0f, 0.0f, 0.0f, 0.0f);
    a_hi[9 * kRows + tid] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  }
  for (int i = tid; i < TC; i += kRows)
    means_s[i] = args.means[i];
  COST::initializeCosts(args.cost, args.cost_aux, theta_c, T);

  float x[S], y[O];
#pragma unroll
  for (int i = 0; i < S; i++)
    x[i] = args.x0[i];
#pragma unroll
  for (int i = 0; i < O; i++)
    y[i] = 0.0f;
#pragma unroll
  for (int i = 0; i < 7; i++)
    y[i] = x[i];  // initializeDynamics (dynamics.cuh:429-435)
  float running_cost = 0.0f;
  int crash_status = 0;

  fence_proxy_async();
  __syncthreads();
  const uint32_t a_hi_s = smem_u32(a_hi), a_lo_s = smem_u32(a_lo);
  unsigned char* a_hi_b = reinterpret_cast<unsigned char*>(a_hi);
  unsigned char* a_lo_b = reinterpret_cast<unsigned char*>(a_lo);

  const bool pure_noise = (float)n_glob >= args.samp.pure_noise_threshold;
  const bool zero_noise_sample = (n_glob == 0);
  float lr_scale[C];
  bool lr_on = false;
#pragma unroll
  for (int c = 0; c < C; c++)
  {
    lr_scale[c] = args.samp.control_cost_coeff[c] / (args.samp.std_dev[0][c] * args.samp.std_dev[0][c]);
    lr_on = lr_on || (args.samp.control_cost_coeff[c] != 0.0f);
  }
  const float half_lambda_1ma = 0.5f * args.lambda * (1.0f - args.alpha);

  const uint32_t w1h = smem_u32(w1_hi), w1l = smem_u32(w1_lo), w2h = smem_u32(w2_hi), w2l = smem_u32(w2_lo),
                 w3h = smem_u32(w3_hi), w3l = smem_u32(w3_lo);

  // ---- the horizon -------------------------------------------------------------------------------------------------
  uint32_t slab_use[2] = { 0, 0 };
  for (int k = 0; k < nchunks; k++)
  {
    const int buf = k & 1;
    mbar_wait(&bars[buf], slab_use[buf] & 1);
    slab_use[buf]++;
    const unsigned char* slab = slabs + buf * kSlabBytes;
#pragma unroll 1
    for (int g = 0; g < 8; g++)
    {
      const int col0 = k * kChunkFloats + g * 4;
      if (col0 >= TC)
        break;
      const float4 e4 = *reinterpret_cast<const float4*>(slab + tid * kChunkBytes + ((g ^ (tid & 7)) << 4));
#pragma unroll 1
      for (int s = 0; s < 2; s++)
      {
        const int t = col0 / C + s;
        if (t >= T)
          break;
        const bool use_mean = zero_noise_sample || (t < args.opt_stride);
        const float* mean_t = means_s + t * C;
        float u[C];
        u[0] = sample_control(mean_t[0], args.samp.std_dev_decayed[0][0], s == 0 ? e4.x : e4.z, use_mean, pure_noise);
        u[1] = sample_control(mean_t[1], args.samp.std_dev_decayed[0][1], s == 0 ? e4.y : e4.w, use_mean, pure_noise);
        DYN::enforceConstraints(args.dyn, x, u);
        if (WRITEBACK)
        {
          if (valid)
          {
            float* dst = args.controls_out + ((size_t)n_loc * T + t) * C;
            dst[0] = u[0];
            dst[1] = u[1];
          }
        }
        float xdot[S];
        DYN::computeKinematics(args.dyn, x, xdot);  // ar_nn_model.cu:123-128

        // ---- layer 1: inputs (roll, vx, vy, yaw rate, steering, throttle, 1, 0) ------------------------------------
        {
          const float in[8] = { x[3], x[4], x[5], x[6], u[0], u[1], 1.0f, 0.0f };
          float h[8], l[8];
#pragma unroll
          for (int i = 0; i < 8; i++)
          {
            h[i] = rna_tf32(in[i]);
            l[i] = in[i] - h[i];
          }
          a_hi[tid] = make_float4(h[0], h[1], h[2], h[3]);
          a_hi[kRows + tid] = make_float4(h[4], h[5], h[6], h[7]);
          a_lo[tid] = make_float4(l[0], l[1], l[2], l[3]);
          a_lo[kRows + tid] = make_float4(l[4], l[5], l[6], l[7]);
        }
        fence_proxy_async();
        __syncthreads();
        // every thread has consumed this slab's last group once it passed the barrier above: refill the buffer
        if (tid == 0 && g == 7 && s == 0 && k + 2 < nchunks)
        {
          mbar_arrive_expect_tx(&bars[buf], kSlabBytes);
          tma_load_2d(slabs + buf * kSlabBytes, &tmap, (k + 2) * kChunkFloats, row0, &bars[buf]);
        }
        float d32[2][16];
        mma_layer<32>(d32, a_hi_s, a_lo_s, w1h, w1l, 1, false);
        __syncthreads();  // the whole warpgroup's MMAs have read A before it is overwritten
        store_activations(a_hi_b, a_lo_b, warp, lane, d32);

        // ---- layer 2 ------------------------------------------------------------------------------------------------
        fence_proxy_async();
        __syncthreads();
        mma_layer<32>(d32, a_hi_s, a_lo_s, w2h, w2l, 4, true);
        __syncthreads();
        store_activations(a_hi_b, a_lo_b, warp, lane, d32);

        // ---- layer 3 (linear, 4 outputs): fragment -> the output table -> each thread's own sample ----------------
        fence_proxy_async();
        __syncthreads();
        {
          float d8[2][4];
          mma_layer<8>(d8, a_hi_s, a_lo_s, w3h, w3l, 4, true);
          const int gq = lane >> 2, q = lane & 3;
          if (q < 2)
          {
#pragma unroll
            for (int m = 0; m < 2; m++)
#pragma unroll
              for (int h = 0; h < 2; h++)
                reinterpret_cast<float2*>(&out_s[64 * m + 16 * warp + gq + 8 * h])[q] =
                    make_float2(d8[m][2 * h], d8[m][2 * h + 1]);
          }
        }
        __syncthreads();
        const float4 out4 = out_s[tid];
        xdot[3] = out4.x;
        xdot[4] = out4.y;
        xdot[5] = out4.z;
        xdot[6] = out4.w;

        // ---- Euler update, output, costs (dynamics.cu:118-155, mppi_common.cu:120-128) --------------------------------
#pragma unroll
        for (int i = 0; i < S; i++)
          x[i] = x[i] + xdot[i] * args.dt;
#pragma unroll
        for (int i = 0; i < S; i++)
          y[i] = x[i];
        float step_cost = COST::computeRunningCost(args.cost, args.cost_aux, theta_c, y, u, t, &crash_status);
        if (lr_on)
          step_cost += likelihood_ratio_cost<C>(lr_scale, mean_t, u, pure_noise, half_lambda_1ma);
        running_cost += step_cost;
      }
    }
  }

  // ---- per-sample cost and block partial (same as rollout_kernel) ------------------------------------------------------
  const float cost = running_cost / (float)T + COST::terminalCost(args.cost, args.cost_aux, y) / (float)T;
  if (valid)
    args.costs[n_loc] = cost;
  float* scratch = red_s + 4 * 32;
  {
    float m = warp_min(valid ? cost : INFINITY);
    if (lane == 0)
      scratch[warp] = m;
    __syncthreads();
    float beta_b = scratch[0];
    for (int i = 1; i < 4; i++)
      beta_b = fminf(beta_b, scratch[i]);
    const float w = valid ? softmin_weight(cost, beta_b, args.lambda_inv) : 0.0f;
    w_s[tid] = w;
    const float sw = warp_sum(w), sw2 = warp_sum(w * w);
    if (lane == 0)
    {
      scratch[32 + warp] = sw;
      scratch[64 + warp] = sw2;
    }
    __syncthreads();
    if (tid == 0)
    {
      float eta_b = 0.0f, w2_b = 0.0f;
      for (int i = 0; i < 4; i++)
      {
        eta_b += scratch[32 + i];
        w2_b += scratch[64 + i];
      }
      args.headers[blockIdx.x] = make_float4(beta_b, eta_b, w2_b, 0.0f);
    }
  }

  // exp-weighted sum of the constrained controls: re-stream the noise slabs (L2-resident) through the same ring;
  // thread (q, j) = (tid / 32, tid % 32) sums column j over rows [32q, 32q + 32), then the 4 quarters are added.
  __syncthreads();
  const int rows_here = min(kRows, args.n_local - row0);
  if (tid == 0)
  {
    for (int k = 0; k < 2 && k < nchunks; k++)
    {
      mbar_arrive_expect_tx(&bars[k], kSlabBytes);
      tma_load_2d(slabs + k * kSlabBytes, &tmap, k * kChunkFloats, row0, &bars[k]);
    }
  }
  float* out = args.partials + (size_t)blockIdx.x * args.pstride + kPartialHeader;
  for (int k = 0; k < nchunks; k++)
  {
    const int buf = k & 1;
    mbar_wait(&bars[buf], slab_use[buf] & 1);
    slab_use[buf]++;
    const unsigned char* slab = slabs + buf * kSlabBytes;
    const int col = k * kChunkFloats + lane;
    float acc = 0.0f;
    if (col < TC)
    {
      const int t = col >> 1, c = col & 1;
      const float* mean_t = means_s + t * C;
      const bool t_uses_mean = t < args.opt_stride;
      const int pair = (lane >> 1) << 1;  // first column of this time step inside the slab
      const int r_begin = warp * 32, r_end = min(r_begin + 32, rows_here);
      for (int r = r_begin; r < r_end; r++)
      {
        const float2 e2 = *reinterpret_cast<const float2*>(slab + r * kChunkBytes + (((pair >> 2) ^ (r & 7)) << 4) +
                                                           ((pair & 3) << 2));
        const int ng = args.n_offset + row0 + r;
        const bool pn = (float)ng >= args.samp.pure_noise_threshold;
        const bool um = t_uses_mean || (ng == 0);
        float u[C];
        u[0] = sample_control(mean_t[0], args.samp.std_dev_decayed[0][0], e2.x, um, pn);
        u[1] = sample_control(mean_t[1], args.samp.std_dev_decayed[0][1], e2.y, um, pn);
        DYN::enforceConstraints(args.dyn, nullptr, u);
        acc = fmaf(w_s[r], c == 0 ? u[0] : u[1], acc);
      }
    }
    red_s[warp * 32 + lane] = acc;
    __syncthreads();
    if (tid < 32 && col < TC)
      out[col] = (red_s[lane] + red_s[32 + lane]) + (red_s[64 + lane] + red_s[96 + lane]);
    if (tid == 0 && k + 2 < nchunks)
    {  // every thread passed the barrier above, i.e. is done with this buffer
      mbar_arrive_expect_tx(&bars[buf], kSlabBytes);
      tma_load_2d(slabs + buf * kSlabBytes, &tmap, (k + 2) * kChunkFloats, row0, &bars[buf]);
    }
    __syncthreads();  // red_s reuse
  }
}

}  // namespace mppib
