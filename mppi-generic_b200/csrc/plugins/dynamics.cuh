/*
 * plugins/dynamics.cuh — device twins of the reference's Dynamics plugins, re-bodied for one-thread-per-sample,
 * register-resident rollouts on sm_90a.
 *
 * The reference's plugin contract (include/mppi/dynamics/dynamics.cuh:67-76,250-300; device bodies
 * include/mppi/dynamics/dynamics.cu:83-155) is kept by NAME and MEANING — STATE_DIM / CONTROL_DIM / OUTPUT_DIM,
 * initializeDynamics, enforceConstraints, computeKinematics, computeDynamics, computeStateDeriv, updateState,
 * stateToOutput, step — but the bodies are static functions over a POD Params blob (include/mppi_b200/params.h)
 * instead of methods of a device-resident object, and x / xdot / y / u are thread-private register arrays instead of
 * per-sample shared-memory slices: there is no blockDim.y lane cooperation and therefore none of the
 * __syncthreads() the reference needs inside step() (dynamics.cu:137-141).
 *
 * `theta_s` keeps its reference meaning: per-block shared scratch the plugin requests (SHARED_FLOATS ==
 * SHARED_MEM_REQUEST_GRD_BYTES/4, managed.cuh:109-116), filled cooperatively in initializeDynamics.
 */
#pragma once
#include "../device_utils.cuh"
#include "../../../include/mppi_b200/params.h"
#include "nn_mma.cuh"
#include "lstm_mma.cuh"
#include "texture_map.cuh"

namespace mppib
{
namespace plugins
{
// dynamics.cu:97-116 — deadband then clamp. State-independent for every in-tree model.
template <int C>
__device__ __forceinline__ void enforceConstraintsDefault(const mppib_control_limits& lim, float* control)
{
#pragma unroll
  for (int i = 0; i < C; i++)
  {
    // both arms evaluated, one selected: no divergent-branch region in the step loop (same values as the if / else)
    const float u = control[i];
    const float shifted = u + lim.deadband[i] * -signf_ref(u);
    const float v = (fabsf(u) < lim.deadband[i]) ? lim.zero_control[i] : shifted;
    control[i] = fminf(fmaxf(lim.rng_lo[i], v), lim.rng_hi[i]);
  }
}

// CRTP base: the parts of Dynamics<CLASS_T, PARAMS_T> (dynamics.cu) every model shares.
template <class CLASS_T, class PARAMS_T, int S, int C, int O>
struct Dynamics
{
  using Params = PARAMS_T;
  static constexpr int STATE_DIM = S;
  static constexpr int CONTROL_DIM = C;
  static constexpr int OUTPUT_DIM = O;
  static constexpr int SHARED_FLOATS = 0;  // SHARED_MEM_REQUEST_GRD_BYTES / 4
  // theta_s size for models whose request depends on constructor arguments (mppib_desc.model_dims) and, for the
  // per-sample part (SHARED_MEM_REQUEST_BLK_BYTES), on the block width
  static int sharedFloats(const int* /*model_dims*/, int /*bx*/)
  {
    return CLASS_T::SHARED_FLOATS;
  }
  static constexpr int MAX_DISTRIBUTIONS = 2;  // systems one thread may roll out side by side (Tube / RMPPI)
  static constexpr int MAX_SPT = 1;  // samples one thread may roll out side by side (rollout_kernel.cuh: SPT)
  static constexpr int MAX_BLOCK_THREADS = 256;  // __launch_bounds__ of the rollout kernel for this model
  static constexpr bool UNROLL_STEPS = true;     // unroll the 4/C steps that share one 16-byte noise group
  // rollout_kernel.cuh: samples a warp carries. 32 = one per lane; fewer = lanes l, l + SPW, ... share a sample (models whose
  // step is warp-collective, plugins/nn_mma.cuh, shorten the per-warp chain this way when a GPU holds few rollouts)
  static constexpr int SAMPLES_PER_WARP = 32;
  using AuxDyn = CLASS_T;  // the form the one-thread-per-rollout auxiliary kernels (init-eval, sampled trajectories) instantiate
  // the model has an analytic Jacobian, computeGrad(p, aux, x, u, A, B): A = df/dx [S][S], B = df/du [S][C], both row-major
  // (Dynamics::computeGrad, dynamics.cuh:236-240). Only such models get the DDP feedback solver (ddp_kernel.cuh).
  static constexpr bool HAS_GRAD = false;
  // ddp_kernel.cuh evaluates f with the warp-cooperative network of AutorallyNNDynamics instead of computeStateDeriv
  static constexpr bool DDP_WARP_NN = false;
  struct Aux
  {
  };
  // per-sample state a model carries from step to step besides x (recurrent networks); lives in registers
  struct Carry
  {
  };

  // dynamics.cuh:429-435 — y <- x on the first min(S,O) entries. theta_s untouched by default.
  __device__ static __forceinline__ void initializeDynamics(const Params&, const Aux&, float* /*theta_s*/, const float* x,
                                                            float* y)
  {
#pragma unroll
    for (int i = 0; i < O && i < S; i++)
      y[i] = x[i];
  }
  // what the rollout kernel calls; models with a Carry override this one
  template <class AUX, class CARRY>
  __device__ static __forceinline__ void initializeDynamics(const Params& p, const AUX& aux, float* theta_s, CARRY&,
                                                            const float* x, float* y)
  {
    CLASS_T::initializeDynamics(p, aux, theta_s, x, y);
  }
  __device__ static __forceinline__ void enforceConstraints(const Params& p, const float* /*x*/, float* u)
  {
    enforceConstraintsDefault<C>(p.lim, u);
  }
  __device__ static __forceinline__ void computeKinematics(const Params&, const float*, float*)
  {
  }
  // dynamics.cu:83-95
  __device__ static __forceinline__ void computeStateDeriv(const Params& p, const float* theta_s, const float* x,
                                                           const float* u, float* xdot)
  {
    CLASS_T::computeKinematics(p, x, xdot);
    CLASS_T::computeDynamics(p, theta_s, x, u, xdot);
  }
  // dynamics.cu:118-129 — explicit Euler
  __device__ static __forceinline__ void updateState(const float* x, float* x_next, const float* xdot, float dt)
  {
#pragma unroll
    for (int i = 0; i < S; i++)
      x_next[i] = x[i] + xdot[i] * dt;
  }
  // dynamics.cu:144-155
  __device__ static __forceinline__ void stateToOutput(const float* x, float* y)
  {
#pragma unroll
    for (int i = 0; i < O && i < S; i++)
      y[i] = x[i];
  }
  // dynamics.cu:131-142
  // M systems of one thread advanced together (Tube's actual + nominal, or SPT samples); models that can share work
  // between them (weight loads) override this
  template <int M, class AUX, class CARRY>
  __device__ static __forceinline__ void stepBatch(const Params& p, const AUX& aux, float* theta_s, CARRY (&carry)[M],
                                                   const float (&x)[M][S], float (&x_next)[M][S], float (&xdot)[M][S],
                                                   const float (&u)[M][C], float (&y)[M][O], int t, float dt)
  {
#pragma unroll
    for (int m = 0; m < M; m++)
      CLASS_T::step(p, aux, theta_s, carry[m], x[m], x_next[m], xdot[m], u[m], y[m], t, dt);
  }
  template <class AUX, class CARRY>
  __device__ static __forceinline__ void step(const Params& p, const AUX&, float* theta_s, CARRY&, const float* x,
                                              float* x_next, float* xdot, const float* u, float* y, int /*t*/, float dt)
  {
    CLASS_T::computeStateDeriv(p, theta_s, x, u, xdot);
    CLASS_T::updateState(x, x_next, xdot, dt);
    CLASS_T::stateToOutput(x_next, y);
  }
};

// ---- Cartpole: dynamics/cartpole/cartpole_dynamics.cu:89-107 (device body) ----------------------------------------
struct CartpoleDynamics : public Dynamics<CartpoleDynamics, mppib_cartpole_dyn_params, 4, 1, 4>
{
  __device__ static __forceinline__ void computeDynamics(const Params& p, const float*, const float* state,
                                                         const float* control, float* state_der)
  {
    float theta = normalizeAngle(state[2]);
    const float sin_theta = __sinf(theta);
    const float cos_theta = __cosf(theta);
    float theta_dot = state[3];
    float force = control[0];
    float m_c = p.cart_mass;
    float m_p = p.pole_mass;
    float l_p = p.pole_length;
    const float gravity_ = p.gravity;

    // cartpole_dynamics.cu:100-106 with the two reciprocals taken by rcp_nr (denominators >= m_c > 0)
    const float denom = m_c + m_p * MPPIB_SQ(sin_theta);
    state_der[0] = state[1];
    state_der[1] = rcp_nr(denom) * (force + m_p * sin_theta * (l_p * MPPIB_SQ(theta_dot) + gravity_ * cos_theta));
    state_der[2] = theta_dot;
    state_der[3] = rcp_nr(l_p * denom) * (-force * cos_theta - m_p * l_p * MPPIB_SQ(theta_dot) * cos_theta * sin_theta -
                                          (m_c + m_p) * gravity_ * sin_theta);
  }

  static constexpr bool HAS_GRAD = true;
  // cartpole_dynamics.cu:10-45, term for term. In the exact derivative the second quotient of A(3, 2) has one more factor
  // pole_length in its numerator; the two agree at pole_length == 1, the reference's default.
  __device__ static bool computeGrad(const Params& p, const Aux&, const float* x, const float* u, float* A, float* B)
  {
    const float th = x[2], td = x[3], F = u[0];
    const float s = sinf(th), c = cosf(th), mc = p.cart_mass, mp = p.pole_mass, l = p.pole_length, g = p.gravity;
    const float den = mc + mp * s * s;
    for (int i = 0; i < 16; i++)
      A[i] = 0.0f;
    for (int i = 0; i < 4; i++)
      B[i] = 0.0f;
    A[0 * 4 + 1] = 1.0f;
    A[1 * 4 + 2] = (mp * c * (l * td * td + g * c) - g * mp * s * s) / den -
                   (2 * mp * c * s * (F + mp * s * (l * td * td + g * c))) / (den * den);
    A[1 * 4 + 3] = (2 * l * mp * td * s) / den;
    A[2 * 4 + 3] = 1.0f;
    A[3 * 4 + 2] = (F * s - g * c * (mp + mc) - l * mp * td * td * c * c + l * mp * td * td * s * s) / (l * den) +
                   (2 * mp * c * s * (l * mp * c * s * td * td + F * c + g * s * (mp + mc))) / ((l * den) * (l * den));
    A[3 * 4 + 3] = -(2 * mp * td * c * s) / den;
    B[1] = 1.0f / den;
    B[3] = -c / (l * den);
    return true;
  }
};

// ---- Double integrator: dynamics/double_integrator/di_dynamics.cu:46-53 -------------------------------------------
struct DoubleIntegratorDynamics : public Dynamics<DoubleIntegratorDynamics, mppib_di_dyn_params, 4, 2, 4>
{
  __device__ static __forceinline__ void computeDynamics(const Params&, const float*, const float* state,
                                                         const float* control, float* state_der)
  {
    state_der[0] = state[2];
    state_der[1] = state[3];
    state_der[2] = control[0];
    state_der[3] = control[1];
  }

  static constexpr bool HAS_GRAD = true;
  // di_dynamics.cu:24-34
  __device__ static bool computeGrad(const Params&, const Aux&, const float*, const float*, float* A, float* B)
  {
    for (int i = 0; i < 16; i++)
      A[i] = 0.0f;
    for (int i = 0; i < 8; i++)
      B[i] = 0.0f;
    A[0 * 4 + 2] = 1.0f;
    A[1 * 4 + 3] = 1.0f;
    B[2 * 2 + 0] = 1.0f;
    B[3 * 2 + 1] = 1.0f;
    return true;
  }
};

// ---- Autorally NeuralNetModel<7,2,3>: dynamics/autorally/ar_nn_model.cu:123-160 + FNNHelper::forward
//      (utils/nn_helpers/fnn_helper.cu:419-484) -------------------------------------------------------------------
// One thread = one sample; the 6-32-32-4 forward pass is 1344 FMAs per step, written as FP32 pairs (fma2_rn, "FFMA2": two
// FFMAs on sm_90): the two halves of every pair are two adjacent OUTPUT neurons, so the accumulation over
// the inputs k runs in the reference's order (k ascending, bias added last, fnn_helper.cu:463-472) and each neuron's sum
// is bit-identical to a scalar FFMA chain. Weights sit in shared memory TRANSPOSED ([in][out]) so one broadcast LDS.128
// (all lanes read the same address: one wavefront) feeds two FFMA2.
// Tried and rejected: weights as kernel parameters (constant-bank operands, `FFMA R, R, UR, R` fed by LDCU.128).
// One issue slot per MAC and no shared-memory traffic, but the constant cache that backs LDCU holds ~4 KB: the 5.6 KB
// network misses on every pass and K1 got slower.
//   theta_s: WT1[6][32] | b1[32] | WT2[32][32] | b2[32] | WT3[32][4] | b3[4]      (1412 floats, like the reference)
__device__ __forceinline__ float tanh_fast(float x)
{
  // tanh(x) = 1 - 2 / (exp(2x) + 1) with ex2.approx / rcp.approx: |abs error| < 2e-7 over the whole range (the
  // reference's tanhf, activation_functions.cuh:15-26, is ~1 ulp; its own FNN test bound is 1e-4, fnn_helper_test.cu:546)
  float t, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(x * 2.8853900817779268f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(t + 1.0f));
  return fmaf(-2.0f, r, 1.0f);
}

struct AutorallyNNDynamics : public Dynamics<AutorallyNNDynamics, mppib_ar_nn_dyn_params, 7, 2, 8>
{
  static constexpr int DYNAMICS_DIM = 4;  // S_DIM - K_DIM
  static constexpr int L1_W = 0, L1_B = L1_W + 6 * 32, L2_W = L1_B + 32, L2_B = L2_W + 32 * 32, L3_W = L2_B + 32,
                       L3_B = L3_W + 32 * 4;
  static constexpr int SHARED_FLOATS = L3_B + 4;  // 1412
  // Tried and rejected: splitting every layer's neurons over two adjacent lanes of a warp (SHFL.BFLY exchange, 2048
  // warps instead of 1024 at N = 32768) — parity-green but slower: the weight rows are then no longer warp-uniform
  // addresses, every LDS.128 costs twice the shared-memory wavefronts per sample, and that data pipe is already the
  // busiest unit of this form.
  // The opposite move — TWO SAMPLES PER THREAD (stepBatch below), every weight row feeding twice the FFMA2s — halves the
  // wavefronts and is slower as well: one warp per scheduler cannot overlap its own phases. It stays
  // selectable (MPPIB_SPT=2) and serves Tube-MPPI's two systems, which share the weight rows through the same code.
  static constexpr int MAX_SPT = 2;
  static constexpr int MAX_BLOCK_THREADS = 256;   // 99 registers/thread: up to 7 warps of samples share one SM's tile
  static constexpr bool UNROLL_STEPS = false;     // one copy of the 1344-FMA step body
  struct Aux
  {
    const float* theta_d;  // reference packed layout, MPPIB_AR_NN_NUM_PARAMS floats (fnn_helper.cu:176-183)
  };

  using Dynamics<AutorallyNNDynamics, mppib_ar_nn_dyn_params, 7, 2, 8>::initializeDynamics;  // the Carry overload
  // FNNHelper::initialize (fnn_helper.cu:385-416): block-cooperative global -> shared copy, transposing W on the way.
  __device__ static __forceinline__ void initializeDynamics(const Params&, const Aux& aux, float* theta_s,
                                                            const float* x, float* y)
  {
    const float* g = aux.theta_d;
    for (int i = threadIdx.x; i < SHARED_FLOATS; i += blockDim.x)
    {
      float v;
      if (i < L1_B)
      {  // WT1[k][j] = W1[j][k]
        const int k = i >> 5, j = i & 31;
        v = g[j * 6 + k];
      }
      else if (i < L2_W)
        v = g[192 + (i - L1_B)];
      else if (i < L2_B)
      {
        const int q = i - L2_W, k = q >> 5, j = q & 31;
        v = g[224 + j * 32 + k];
      }
      else if (i < L3_W)
        v = g[1248 + (i - L2_B)];
      else if (i < L3_B)
      {
        const int q = i - L3_W, k = q >> 2, j = q & 3;
        v = g[1280 + j * 32 + k];
      }
      else
        v = g[1408 + (i - L3_B)];
      theta_s[i] = v;
    }
#pragma unroll
    for (int i = 0; i < 7; i++)
      y[i] = x[i];
  }

  // ar_nn_model.cu:123-128 (cosf / sinf, not the fast intrinsics, in the reference's device code): full-precision sine and
  // cosine from one shared range reduction (device_utils.cuh: sincos_cw, 1.5 ulp)
  __device__ static __forceinline__ void computeKinematics(const Params&, const float* state, float* state_der)
  {
    float sn, cs;
    sincos_cw(state[2], &sn, &cs);
    state_der[0] = cs * state[4] - sn * state[5];
    state_der[1] = sn * state[4] + cs * state[5];
    state_der[2] = -state[6];
  }

  // One weight row (all OUT outputs of input k) as OUT/4 broadcast LDS.128. `volatile` keeps the loads in program
  // order, which is how the software pipeline below is expressed: row k+1 is requested BEFORE the FFMA2s of row k, so the
  // ~30-cycle shared-memory latency is covered by arithmetic even when a scheduler holds a single warp (ptxas otherwise
  // funnels every load through one register quad and stalls on each).
  template <int OUT>
  __device__ static __forceinline__ void load_row(float4 (&w)[OUT / 4], const float* row)
  {
    const uint32_t a = smem_u32(row);
#pragma unroll
    for (int j4 = 0; j4 < OUT / 4; j4++)
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(w[j4].x), "=f"(w[j4].y), "=f"(w[j4].z), "=f"(w[j4].w)
                   : "r"(a + 16u * j4));
  }

  // One dense layer. TANH_IN: the inputs are the previous layer's PRE-activations and tanh is applied to input k+1 while
  // the FFMA2s of input k issue — the MUFU work (ex2 + rcp per tanh) then overlaps the FMA pipe inside a single warp
  // instead of forming a separate phase between the layers (with < 2 warps per scheduler nothing else would hide it).
  // TANH_OUT is applied in the epilogue (unused by the lazy pipeline, kept for the tensor-core variant's reference use).
  template <int IN, int OUT, bool TANH_IN, bool TANH_OUT>
  __device__ static __forceinline__ void layer(const float* __restrict__ WT, const float* __restrict__ b,
                                               const float* in, float* out)
  {
    float2 acc[OUT / 2];
#pragma unroll
    for (int j = 0; j < OUT / 2; j++)
      acc[j] = make_float2(0.0f, 0.0f);
    float4 w[OUT / 4], wn[OUT / 4];
    load_row<OUT>(w, WT);
    float x_cur = TANH_IN ? tanh_fast(in[0]) : in[0];
#pragma unroll
    for (int k = 0; k < IN; k++)
    {
      if (k + 1 < IN)
        load_row<OUT>(wn, WT + (k + 1) * OUT);
      else
        load_row<OUT>(wn, b);  // the bias row rides the same pipeline
      float x_next = 0.0f;
      if (k + 1 < IN)
        x_next = TANH_IN ? tanh_fast(in[k + 1]) : in[k + 1];
      const float2 xk = make_float2(x_cur, x_cur);
#pragma unroll
      for (int j4 = 0; j4 < OUT / 4; j4++)
      {
        acc[2 * j4] = fma2_rn(make_float2(w[j4].x, w[j4].y), xk, acc[2 * j4]);
        acc[2 * j4 + 1] = fma2_rn(make_float2(w[j4].z, w[j4].w), xk, acc[2 * j4 + 1]);
      }
#pragma unroll
      for (int j4 = 0; j4 < OUT / 4; j4++)
        w[j4] = wn[j4];
      x_cur = x_next;
    }
    // w now holds the bias row
#pragma unroll
    for (int j4 = 0; j4 < OUT / 4; j4++)
    {
      const float t0 = acc[2 * j4].x + w[j4].x, t1 = acc[2 * j4].y + w[j4].y, t2 = acc[2 * j4 + 1].x + w[j4].z,
                  t3 = acc[2 * j4 + 1].y + w[j4].w;
      out[4 * j4 + 0] = TANH_OUT ? tanh_fast(t0) : t0;
      out[4 * j4 + 1] = TANH_OUT ? tanh_fast(t1) : t1;
      out[4 * j4 + 2] = TANH_OUT ? tanh_fast(t2) : t2;
      out[4 * j4 + 3] = TANH_OUT ? tanh_fast(t3) : t3;
    }
  }

  __device__ static __forceinline__ void computeDynamics(const Params&, const float* theta_s, const float* state,
                                                         const float* control, float* state_der)
  {
    float a0[6], a1[32], a2[32], a3[4];
#pragma unroll
    for (int i = 0; i < DYNAMICS_DIM; i++)
      a0[i] = state[i + (7 - DYNAMICS_DIM)];
    a0[4] = control[0];
    a0[5] = control[1];
    // a1, a2 hold PRE-activations; the consuming layer applies tanh as it walks its inputs
    layer<6, 32, false, false>(theta_s + L1_W, theta_s + L1_B, a0, a1);
    layer<32, 32, true, false>(theta_s + L2_W, theta_s + L2_B, a1, a2);
    layer<32, 4, true, false>(theta_s + L3_W, theta_s + L3_B, a2, a3);
#pragma unroll
    for (int i = 0; i < DYNAMICS_DIM; i++)
      state_der[i + (7 - DYNAMICS_DIM)] = a3[i];
  }

  static constexpr bool HAS_GRAD = true;
  static constexpr bool DDP_WARP_NN = true;
  // NeuralNetModel::computeGrad (ar_nn_model.cu:63-86): the kinematic rows, then the network's input Jacobian by
  // back-propagation through the two tanh layers (FNNHelper::computeGrad, fnn_helper.cu:312-347). One thread, weights read
  // from the packed blob in global memory (W row-major out x in, then b, per layer).
  __device__ static bool computeGrad(const Params&, const Aux& aux, const float* x, const float* u, float* A, float* B)
  {
    const float* g = aux.theta_d;
    const float *W1 = g, *b1 = g + 192, *W2 = g + 224, *b2 = g + 1248, *W3 = g + 1280;
    for (int i = 0; i < 49; i++)
      A[i] = 0.0f;
    for (int i = 0; i < 14; i++)
      B[i] = 0.0f;
    float sn, cs;
    sincosf(x[2], &sn, &cs);
    A[0 * 7 + 2] = -sn * x[4] - cs * x[5];
    A[0 * 7 + 4] = cs;
    A[0 * 7 + 5] = -sn;
    A[1 * 7 + 2] = cs * x[4] - sn * x[5];
    A[1 * 7 + 4] = sn;
    A[1 * 7 + 5] = cs;
    A[2 * 7 + 6] = -1.0f;
    const float in[6] = { x[3], x[4], x[5], x[6], u[0], u[1] };
    float a1[32], d1[32], d2[32];
    for (int j = 0; j < 32; j++)
    {
      float z = 0.0f;
      for (int k = 0; k < 6; k++)
        z = fmaf(__ldg(W1 + j * 6 + k), in[k], z);
      a1[j] = tanhf(z + __ldg(b1 + j));
      d1[j] = 1.0f - a1[j] * a1[j];  // tanh_deriv
    }
    for (int j = 0; j < 32; j++)
    {
      float z = 0.0f;
      for (int k = 0; k < 32; k++)
        z = fmaf(__ldg(W2 + j * 32 + k), a1[k], z);
      const float a2 = tanhf(z + __ldg(b2 + j));
      d2[j] = 1.0f - a2 * a2;
    }
    for (int i = 0; i < 4; i++)
    {
      // row i of d out / d in = W3[i] diag(d2) W2 diag(d1) W1
      float r[6] = { 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f };
      for (int j = 0; j < 32; j++)
      {
        float gj = 0.0f;
        for (int k = 0; k < 32; k++)
          gj = fmaf(__ldg(W3 + i * 32 + k) * d2[k], __ldg(W2 + k * 32 + j), gj);
        gj *= d1[j];
        for (int m = 0; m < 6; m++)
          r[m] = fmaf(gj, __ldg(W1 + j * 6 + m), r[m]);
      }
      for (int m = 0; m < 4; m++)
        A[(3 + i) * 7 + 3 + m] = r[m];
      B[(3 + i) * 2 + 0] = r[4];
      B[(3 + i) * 2 + 1] = r[5];
    }
    return true;
  }
  // The same dense layer for M samples of one thread: one weight row (LDS.128 quads, broadcast) feeds M * OUT/2 FFMA2s.
  // Per-neuron accumulation order unchanged (k ascending, bias last), so every sample's values are those of layer<>.
  template <int IN, int OUT, bool TANH_IN, int M>
  __device__ static __forceinline__ void layerBatch(const float* __restrict__ WT, const float* __restrict__ b,
                                                    const float (&in)[M][IN], float (&out)[M][OUT])
  {
    float2 acc[M][OUT / 2];
#pragma unroll
    for (int m = 0; m < M; m++)
#pragma unroll
      for (int j = 0; j < OUT / 2; j++)
        acc[m][j] = make_float2(0.0f, 0.0f);
    // software pipeline as in layer<>: row k+1 (or the bias row) and the tanh of input k+1 are requested before the
    // FFMA2s of row k, so their latencies sit under arithmetic even when the thread's warp is alone on its scheduler
    float4 w[OUT / 4], wn[OUT / 4];
    load_row<OUT>(w, WT);
    float x_cur[M], x_next[M];
#pragma unroll
    for (int m = 0; m < M; m++)
      x_cur[m] = TANH_IN ? tanh_fast(in[m][0]) : in[m][0];
#pragma unroll
    for (int k = 0; k < IN; k++)
    {
      if (k + 1 < IN)
        load_row<OUT>(wn, WT + (k + 1) * OUT);
      else
        load_row<OUT>(wn, b);
#pragma unroll
      for (int m = 0; m < M; m++)
        x_next[m] = (k + 1 < IN) ? (TANH_IN ? tanh_fast(in[m][k + 1]) : in[m][k + 1]) : 0.0f;
#pragma unroll
      for (int m = 0; m < M; m++)
      {
        const float2 xk = make_float2(x_cur[m], x_cur[m]);
#pragma unroll
        for (int j4 = 0; j4 < OUT / 4; j4++)
        {
          acc[m][2 * j4] = fma2_rn(make_float2(w[j4].x, w[j4].y), xk, acc[m][2 * j4]);
          acc[m][2 * j4 + 1] = fma2_rn(make_float2(w[j4].z, w[j4].w), xk, acc[m][2 * j4 + 1]);
        }
      }
#pragma unroll
      for (int j4 = 0; j4 < OUT / 4; j4++)
        w[j4] = wn[j4];
#pragma unroll
      for (int m = 0; m < M; m++)
        x_cur[m] = x_next[m];
    }
    // w now holds the bias row
#pragma unroll
    for (int m = 0; m < M; m++)
#pragma unroll
      for (int j4 = 0; j4 < OUT / 4; j4++)
      {
        out[m][4 * j4 + 0] = acc[m][2 * j4].x + w[j4].x;
        out[m][4 * j4 + 1] = acc[m][2 * j4].y + w[j4].y;
        out[m][4 * j4 + 2] = acc[m][2 * j4 + 1].x + w[j4].z;
        out[m][4 * j4 + 3] = acc[m][2 * j4 + 1].y + w[j4].w;
      }
  }

  template <int M, class AUX, class CARRY>
  __device__ static __forceinline__ void stepBatch(const Params& p, const AUX& aux, float* theta_s, CARRY (&carry)[M],
                                                   const float (&x)[M][7], float (&x_next)[M][7], float (&xdot)[M][7],
                                                   const float (&u)[M][2], float (&y)[M][8], int t, float dt)
  {
    if constexpr (M == 1)
    {
      step(p, aux, theta_s, carry[0], x[0], x_next[0], xdot[0], u[0], y[0], t, dt);
    }
    else
    {
      float a0[M][6], a1[M][32], a2[M][32], a3[M][4];
#pragma unroll
      for (int m = 0; m < M; m++)
      {
        computeKinematics(p, x[m], xdot[m]);
#pragma unroll
        for (int i = 0; i < DYNAMICS_DIM; i++)
          a0[m][i] = x[m][i + (7 - DYNAMICS_DIM)];
        a0[m][4] = u[m][0];
        a0[m][5] = u[m][1];
      }
      layerBatch<6, 32, false, M>(theta_s + L1_W, theta_s + L1_B, a0, a1);
      layerBatch<32, 32, true, M>(theta_s + L2_W, theta_s + L2_B, a1, a2);
      layerBatch<32, 4, true, M>(theta_s + L3_W, theta_s + L3_B, a2, a3);
#pragma unroll
      for (int m = 0; m < M; m++)
      {
#pragma unroll
        for (int i = 0; i < DYNAMICS_DIM; i++)
          xdot[m][i + (7 - DYNAMICS_DIM)] = a3[m][i];
        updateState(x[m], x_next[m], xdot[m], dt);
        stateToOutput(x_next[m], y[m]);
      }
    }
  }
};

// ---- Autorally NeuralNetModel<7,2,3> with the network on the legacy tensor path (plugins/nn_mma.cuh): a warp evaluates
//      SPW = 32 / 16 / 8 samples with mma.sync (FP16 hi / lo split, three products, FP32 accumulate). With SPW < 32 the
//      lanes l, l + SPW, ... of a warp carry the same sample (rollout_kernel.cuh: SAMPLES_PER_WARP) and only the first
//      owns its results: a shorter per-step chain per warp and more warps per scheduler when a GPU holds few rollouts.
//      Everything around the network is AutorallyNNDynamics'. The default form of the pair (engine.cu). -------------------
template <int SPW>
struct AutorallyNNMmaDynamics : public Dynamics<AutorallyNNMmaDynamics<SPW>, mppib_ar_nn_dyn_params, 7, 2, 8>
{
  using Base = Dynamics<AutorallyNNMmaDynamics<SPW>, mppib_ar_nn_dyn_params, 7, 2, 8>;
  using Params = typename Base::Params;
  static constexpr int DYNAMICS_DIM = 4;
  static constexpr int SAMPLES_PER_WARP = SPW;
  using AuxDyn = AutorallyNNMmaDynamics<32>;  // the auxiliary kernels map one lane to one rollout
  static constexpr int MAX_SPT = 1;
  static constexpr int MAX_BLOCK_THREADS = SPW == 32 ? 256 : 512;  // <= 256 samples per block either way
  static constexpr bool UNROLL_STEPS = false;
  using Aux = AutorallyNNDynamics::Aux;
  // fragment-ordered weights + transposition scratch per warp; bx = samples per block
  static int sharedFloats(const int* /*model_dims*/, int bx)
  {
    return nn_mma::sharedFloats(bx * (32 / SPW), SPW);
  }
  using Base::initializeDynamics;  // the Carry overload
  __device__ static __forceinline__ void initializeDynamics(const Params&, const Aux& aux, float* theta_s,
                                                            const float* x, float* y)
  {
    nn_mma::load_weights(aux.theta_d, theta_s);
#pragma unroll
    for (int i = 0; i < 7; i++)
      y[i] = x[i];
  }
  __device__ static __forceinline__ void computeKinematics(const Params& p, const float* state, float* state_der)
  {
    AutorallyNNDynamics::computeKinematics(p, state, state_der);
  }
  static constexpr bool HAS_GRAD = true;
  static constexpr bool DDP_WARP_NN = true;
  __device__ static bool computeGrad(const Params& p, const Aux& aux, const float* x, const float* u, float* A, float* B)
  {
    return AutorallyNNDynamics::computeGrad(p, aux, x, u, A, B);
  }
  // warp-collective: every lane of the warp calls it (the rollout kernels keep out-of-range rows running)
  __device__ static __forceinline__ void computeDynamics(const Params&, const float* theta_s, const float* state,
                                                         const float* control, float* state_der)
  {
    float in[6], out[4];
#pragma unroll
    for (int i = 0; i < DYNAMICS_DIM; i++)
      in[i] = state[i + (7 - DYNAMICS_DIM)];
    in[4] = control[0];
    in[5] = control[1];
    float* scratch = const_cast<float*>(theta_s) + nn_mma::kFixedFloats + (threadIdx.x >> 5) * nn_mma::scratchPerWarp(SPW);
    nn_mma::forward<SPW>(theta_s, scratch, in, out);
#pragma unroll
    for (int i = 0; i < DYNAMICS_DIM; i++)
      state_der[i + (7 - DYNAMICS_DIM)] = out[i];
  }
};

// ---- RacerDubinsElevationLSTMSteering: dynamics/racer_dubins/racer_dubins_elevation_lstm_steering.cu:131-213,240-262
//      (device step / computeLSTMSteering / updateState), racer_dubins.cu:281-293 (brake delay),
//      racer_dubins_elevation.cu:767-806 (parametric acceleration, device), :336-515,662-741 (uncertainty propagation),
//      LSTMHelper::forward utils/nn_helpers/lstm_helper.cu:341-463 + FNN head (fnn_helper.cu:419-484) -----------------
// One thread = one sample. The parametric model and the 4x4 covariance propagation live in registers (fully unrolled);
// the LSTM has constructor-time dimensions (Aux::H, Aux::L1 from mppib_desc.model_dims), so its weights and the
// per-sample hidden / cell vectors live in shared memory:
//   theta_s: gate rows  [i < H][ j < 4 : (W_ii,W_fi,W_oi,W_ci)[i][j] | j < H : (W_im,W_fm,W_om,W_cm)[i][j] | bias ] float4
//            head       W1T[j < H+4][k < L1p] | b1[L1p] | w2[L1p] | b2 (4)                (L1p = L1 rounded up to 4)
//            per sample hA[H][bx] | hB[H][bx] | c[H][bx]   (element [j][tid]: conflict-free, h double-buffered by step parity)
// so one broadcast LDS.128 brings the four gate weights of a (row, input) pair and every accumulation runs in the
// reference's order (inputs, then hidden, then bias; lstm_helper.cu:411-431). The elevation map is not built: flat
// terrain (TwoDTextureHelper::checkTextureUse false => roll = pitch = height = 0, racer_dubins.cu:427-432).
// The RACER models' elevation map: TwoDTextureHelper<float> map 0 (utils/texture_helpers/), read through texture_map.cuh,
// which evaluates the reference's HOST interpolation formula on the device.
// RACER::computeStaticSettling (racer_dubins.cu:359-434): wheel contact heights from the map -> roll, pitch, height
__device__ __forceinline__ void racer_static_settling(const ElevationMap& m, float yaw, float x, float y, float& roll,
                                                      float& pitch, float& height)
{
  height = 0.0f;
  if (!m.hdr.use)
  {
    roll = 0.0f;
    pitch = 0.0f;
    return;
  }
  // math::Euler2DCM_NWU (math_utils.h:457-482, device branch) with the CURRENT roll / pitch and the NEXT yaw; offsets have z = 0
  float sr, cr, sp, cp, sy, cy;
  __sincosf(normalizeAngle(roll), &sr, &cr);
  __sincosf(normalizeAngle(pitch), &sp, &cp);
  __sincosf(normalizeAngle(yaw), &sy, &cy);
  const float M00 = cp * cy, M01 = sr * sp * cy - cr * sy, M10 = cp * sy, M11 = sr * sp * sy + cr * cy, M20 = -sp,
              M21 = sr * cp;
  const float L = 2.981f, W = 0.737f;  // wheel base / half track of the vehicle (racer_dubins.cu:364-367)
  float hgt[4];
#pragma unroll
  for (int k = 0; k < 4; k++)
  {  // front left, front right, rear left, rear right
    const float ox = (k < 2) ? L : 0.0f, oy = (k & 1) ? -W : W;
    hgt[k] = elevation_at_world_pose(m, M00 * ox + M01 * oy + x, M10 * ox + M11 * oy + y, M20 * ox + M21 * oy + 0.0f);
  }
  const float fl = hgt[0], fr = hgt[1], rl = hgt[2], rr = hgt[3];
  const float front_diff = fmaxf(fminf(fl - fr, 0.736f * 2.0f), -0.736f * 2.0f);
  const float rear_diff = fmaxf(fminf(rl - rr, 0.736f * 2.0f), -0.736f * 2.0f);
  roll = (asinf(front_diff / (0.737f * 2.0f)) + asinf(rear_diff / (0.737f * 2.0f))) / 2.0f;
  const float left_diff = fmaxf(fminf(rl - fl, 2.98f), -2.98f);
  const float right_diff = fmaxf(fminf(rr - fr, 2.98f), -2.98f);
  pitch = (asinf(left_diff / 2.981f) + asinf(right_diff / 2.981f)) / 2.0f;
  height = (rl + rr) / 2.0f;
  const float pi = 3.14159265358979323846f;
  if (!isfinite(roll) || fabsf(roll) > pi)
    roll = 2.0f * pi;
  if (!isfinite(pitch) || fabsf(pitch) > pi)
    pitch = 2.0f * pi;
  if (!isfinite(height))
    height = 0.0f;
}

// The pieces of the device step the RACER elevation models share (RacerDubinsElevation, its LSTM-steering child and the
// suspension model): state / output indices, setOutputs, the parametric derivatives, the uncertainty propagation and the
// static settling. Each model adds its own steering and updateState between them. The first eight states are the same in
// every layout; STEER_RATE_INDEX and UNC_INDEX place the steering rate and the ten uncertainty entries (8 and 9 in the
// 19-state models, 12 and 13 in the 24-state suspension model).
template <int STEER_RATE_INDEX, int UNC_INDEX>
struct RacerElevationPartsT
{
  enum
  {
    VEL_X = 0, YAW, POS_X, POS_Y, STEER_ANGLE, BRAKE_STATE, ROLL, PITCH
  };
  enum
  {
    STEER_ANGLE_RATE = STEER_RATE_INDEX
  };
  enum
  {
    UNC_POS_X = UNC_INDEX, UNC_POS_Y, UNC_YAW, UNC_VEL_X, UNC_POS_X_Y, UNC_POS_X_YAW, UNC_POS_X_VEL_X, UNC_POS_Y_YAW,
    UNC_POS_Y_VEL_X, UNC_YAW_VEL_X
  };
  enum
  {
    O_VEL_B_X = 0, O_VEL_B_Y, O_POS_I_X, O_POS_I_Y, O_POS_I_Z, O_YAW, O_ROLL, O_PITCH, O_STEER_ANGLE, O_STEER_ANGLE_RATE,
    O_WF_UP, O_WF_FWD, O_WF_SIDE, O_ACCEL_X, O_ACCEL_Y, O_OMEGA_Z, O_TOTAL_VELOCITY, O_UNC_POS_X, O_UNC_POS_Y, O_UNC_YAW,
    O_UNC_VEL_X, O_UNC_POS_X_Y, O_UNC_POS_X_YAW, O_UNC_POS_X_VEL_X, O_UNC_POS_Y_YAW, O_UNC_POS_Y_VEL_X, O_UNC_YAW_VEL_X
  };
  enum
  {
    U_VEL_X = 0, U_YAW, U_POS_X, U_POS_Y
  };
  __host__ __device__ static constexpr int cm(int row, int col)
  {
    return col * 4 + row;  // mm::columnMajorIndex(row, col, 4)
  }

  // setOutputs, racer_dubins_elevation.cu:69-227
  __device__ static __forceinline__ void setOutputs(const float* state_der, const float* next_state, float* output)
  {
    output[O_VEL_B_X] = next_state[VEL_X];
    output[O_VEL_B_Y] = 0.0f;
    output[O_POS_I_X] = next_state[POS_X];
    output[O_POS_I_Y] = next_state[POS_Y];
    output[O_PITCH] = next_state[PITCH];
    output[O_ROLL] = next_state[ROLL];
    output[O_YAW] = next_state[YAW];
    output[O_STEER_ANGLE] = next_state[STEER_ANGLE];
    output[O_STEER_ANGLE_RATE] = next_state[STEER_ANGLE_RATE];
    output[O_WF_UP] = NAN;
    output[O_WF_FWD] = NAN;
    output[O_WF_SIDE] = NAN;
    output[O_ACCEL_X] = state_der[VEL_X];
    output[O_ACCEL_Y] = 0.0f;
    output[O_OMEGA_Z] = state_der[YAW];
    output[O_UNC_VEL_X] = next_state[UNC_VEL_X];
    output[O_UNC_YAW_VEL_X] = next_state[UNC_YAW_VEL_X];
    output[O_UNC_POS_X_VEL_X] = next_state[UNC_POS_X_VEL_X];
    output[O_UNC_POS_Y_VEL_X] = next_state[UNC_POS_Y_VEL_X];
    output[O_UNC_YAW] = next_state[UNC_YAW];
    output[O_UNC_POS_X_YAW] = next_state[UNC_POS_X_YAW];
    output[O_UNC_POS_Y_YAW] = next_state[UNC_POS_Y_YAW];
    output[O_UNC_POS_X] = next_state[UNC_POS_X];
    output[O_UNC_POS_X_Y] = next_state[UNC_POS_X_Y];
    output[O_UNC_POS_Y] = next_state[UNC_POS_Y];
    output[O_TOTAL_VELOCITY] = fabsf(next_state[VEL_X]);
  }

  __device__ static __forceinline__ float pick3(const float (&a)[3], int index)
  {
    return index == 0 ? a[0] : (index == 1 ? a[1] : a[2]);
  }

  // what the step's later pieces take from the parametric derivative
  struct Kinematics
  {
    int index;  // speed bin of |VEL_X|: 0 (<= 0.2), 1 (<= 3), 2
    float brake_state, c_v, sin_yaw, cos_yaw;
  };
  // computeParametricDelayDeriv (device) + computeParametricAccelDeriv (device) with the kinematic rows: state_der's VEL_X,
  // YAW, POS_X, POS_Y and BRAKE_STATE
  __device__ static __forceinline__ Kinematics parametricDeriv(const mppib_racer_lstm_dyn_params& p, const float* state,
                                                               const float* control, float* state_der)
  {
    const float vx = state[VEL_X];
    const float linear_brake_slope = 0.2f;
    const int index = (fabsf(vx) > linear_brake_slope && fabsf(vx) <= 3.0f) + (fabsf(vx) > 3.0f) * 2;
    const bool enable_brake = control[0] < 0.0f;
    // computeParametricDelayDeriv, racer_dubins.cu:281-293
    {
      const float brake_error = (enable_brake * -control[0] - state[BRAKE_STATE]);
      state_der[BRAKE_STATE] = fminf(fmaxf((brake_error > 0) * brake_error * p.brake_delay_constant +
                                               (brake_error < 0) * brake_error * p.brake_delay_constant_neg,
                                           -p.max_brake_rate_neg),
                                     p.max_brake_rate_pos);
    }
    const float brake_state = fminf(fmaxf(state[BRAKE_STATE], 0.0f), 0.25f);
    const float c_t = pick3(p.c_t, index), c_b = pick3(p.c_b, index), c_v = pick3(p.c_v, index);
    // computeParametricAccelDeriv (device), racer_dubins_elevation.cu:767-806
    {
      float throttle = c_t * control[0];
      float brake = c_b * brake_state * (vx >= 0.0f ? -1.0f : 1.0f);
      if (fabsf(vx) <= linear_brake_slope)
      {
        throttle = c_t * fmaxf(control[0] - p.low_min_throttle, 0.0f);
        brake = c_b * brake_state * -vx;
      }
      state_der[VEL_X] = (!enable_brake) * throttle * p.gear_sign + brake - c_v * vx + p.c_0;
      state_der[VEL_X] = fminf(fmaxf(state_der[VEL_X], -p.clamp_ax), p.clamp_ax);
      if (fabsf(state[PITCH]) < 1.57079632679489661923f)
        state_der[VEL_X] -= p.gravity * __sinf(normalizeAngle(state[PITCH]));
      state_der[YAW] = (vx / p.wheel_base) * __tanf(normalizeAngle(state[STEER_ANGLE] / p.steer_angle_scale));
    }
    const float yaw_norm = normalizeAngle(state[YAW]);
    float sin_yaw, cos_yaw;
    __sincosf(yaw_norm, &sin_yaw, &cos_yaw);
    state_der[POS_X] = vx * cos_yaw;
    state_der[POS_Y] = vx * sin_yaw;
    return Kinematics{ index, brake_state, c_v, sin_yaw, cos_yaw };
  }

  // the 4x4 covariance over (VEL_X, YAW, POS_X, POS_Y) one step forward: next_state's ten uncertainty entries
  __device__ static __forceinline__ void propagateUncertainty(const mppib_racer_lstm_dyn_params& p, const Kinematics& k,
                                                              const float* state, const float* state_der,
                                                              float* next_state, float dt)
  {
    const float vx = state[VEL_X];
    const int index = k.index;
    const float brake_state = k.brake_state, c_v = k.c_v, sin_yaw = k.sin_yaw, cos_yaw = k.cos_yaw;
    // computeUncertaintyPropagation (device), racer_dubins_elevation.cu:662-741
    {
      float A[16], Sa[16], Sb[16];
      const float delta = state[STEER_ANGLE] / p.steer_angle_scale;
      const float tan_steer_angle = __tanf(delta);
      const float cos_2_delta = MPPIB_SQ(__cosf(delta));
      // computeUncertaintyJacobian :336-425
      A[cm(U_VEL_X, U_VEL_X)] = -c_v - p.K_vel_x - (index == 0 ? 1.0f : 0.0f) * p.c_b[0] * brake_state;
      A[cm(U_VEL_X, U_YAW)] = 0.0f;
      A[cm(U_VEL_X, U_POS_X)] = -p.K_x * cos_yaw;
      A[cm(U_VEL_X, U_POS_Y)] = -p.K_x * sin_yaw;
      A[cm(U_YAW, U_VEL_X)] = tan_steer_angle / (p.wheel_base);
      A[cm(U_YAW, U_YAW)] = -fabsf(vx) * p.K_yaw / (p.wheel_base * cos_2_delta);
      A[cm(U_YAW, U_POS_X)] = vx * p.K_y * sin_yaw / (p.wheel_base * cos_2_delta);
      A[cm(U_YAW, U_POS_Y)] = -vx * p.K_y * cos_yaw / (p.wheel_base * cos_2_delta);
      A[cm(U_POS_X, U_VEL_X)] = cos_yaw;
      A[cm(U_POS_X, U_YAW)] = -sin_yaw * vx;
      A[cm(U_POS_X, U_POS_X)] = 0.0f;
      A[cm(U_POS_X, U_POS_Y)] = 0.0f;
      A[cm(U_POS_Y, U_VEL_X)] = sin_yaw;
      A[cm(U_POS_Y, U_YAW)] = cos_yaw * vx;
      A[cm(U_POS_Y, U_POS_Y)] = 0.0f;
      A[cm(U_POS_Y, U_POS_X)] = 0.0f;
      // uncertaintyStateToMatrix :517-577
      Sa[cm(U_VEL_X, U_VEL_X)] = state[UNC_VEL_X];
      Sa[cm(U_YAW, U_VEL_X)] = Sa[cm(U_VEL_X, U_YAW)] = state[UNC_YAW_VEL_X];
      Sa[cm(U_POS_X, U_VEL_X)] = Sa[cm(U_VEL_X, U_POS_X)] = state[UNC_POS_X_VEL_X];
      Sa[cm(U_POS_Y, U_VEL_X)] = Sa[cm(U_VEL_X, U_POS_Y)] = state[UNC_POS_Y_VEL_X];
      Sa[cm(U_YAW, U_YAW)] = state[UNC_YAW];
      Sa[cm(U_POS_X, U_YAW)] = Sa[cm(U_YAW, U_POS_X)] = state[UNC_POS_X_YAW];
      Sa[cm(U_POS_Y, U_YAW)] = Sa[cm(U_YAW, U_POS_Y)] = state[UNC_POS_Y_YAW];
      Sa[cm(U_POS_X, U_POS_X)] = state[UNC_POS_X];
      Sa[cm(U_POS_Y, U_POS_X)] = Sa[cm(U_POS_X, U_POS_Y)] = state[UNC_POS_X_Y];
      Sa[cm(U_POS_Y, U_POS_Y)] = state[UNC_POS_Y];
#pragma unroll
      for (int i = 0; i < 16; i++)
        A[i] = (i % 5 == 0) + A[i] * dt;  // I + A dt
      // Sigma_b = A Sigma_a ; Sigma_a = Sigma_b A^T   (mm::gemm1, k ascending)
#pragma unroll
      for (int col = 0; col < 4; col++)
#pragma unroll
        for (int row = 0; row < 4; row++)
        {
          float acc = 0.0f;
#pragma unroll
          for (int q = 0; q < 4; q++)
            acc += A[cm(row, q)] * Sa[cm(q, col)];
          Sb[cm(row, col)] = acc;
        }
#pragma unroll
      for (int col = 0; col < 4; col++)
#pragma unroll
        for (int row = 0; row < 4; row++)
        {
          float acc = 0.0f;
#pragma unroll
          for (int q = 0; q < 4; q++)
            acc += Sb[cm(row, q)] * A[cm(col, q)];
          Sa[cm(row, col)] = acc;
        }
      // computeQ :427-515 (device branch), added as Q dt
      const float abs_vx = fabsf(vx);
      const float abs_acc_x = fabsf(state_der[VEL_X]);
      const float sin_roll = __sinf(normalizeAngle(state[ROLL]));
      const float side_force = MPPIB_SQ(abs_vx) * tan_steer_angle / p.wheel_base + p.gravity * sin_roll;
      const float Q_11 = fabsf(p.Q_y_f * fabsf(side_force) * fmaxf(abs_vx - 2, 0.0f));
      Sa[cm(U_VEL_X, U_VEL_X)] += (p.Q_x_acc * abs_acc_x + pick3(p.Q_x_v, index) * abs_vx) * dt;
      Sa[cm(U_YAW, U_YAW)] += (abs_vx * (p.Q_omega_steering * fabsf(delta) + p.Q_omega_v)) * dt;
      Sa[cm(U_POS_X, U_POS_X)] += (Q_11 * sin_yaw * sin_yaw) * dt;
      Sa[cm(U_POS_X, U_POS_Y)] += (-Q_11 * sin_yaw * cos_yaw) * dt;
      Sa[cm(U_POS_Y, U_POS_Y)] += (Q_11 * cos_yaw * cos_yaw) * dt;
      Sa[cm(U_POS_Y, U_POS_X)] += (-Q_11 * sin_yaw * cos_yaw) * dt;
      // uncertaintyMatrixToState :579-621
      next_state[UNC_VEL_X] = Sa[cm(U_VEL_X, U_VEL_X)];
      next_state[UNC_YAW_VEL_X] = Sa[cm(U_YAW, U_VEL_X)];
      next_state[UNC_POS_X_VEL_X] = Sa[cm(U_POS_X, U_VEL_X)];
      next_state[UNC_POS_Y_VEL_X] = Sa[cm(U_POS_Y, U_VEL_X)];
      next_state[UNC_YAW] = Sa[cm(U_YAW, U_YAW)];
      next_state[UNC_POS_X_YAW] = Sa[cm(U_POS_X, U_YAW)];
      next_state[UNC_POS_Y_YAW] = Sa[cm(U_POS_Y, U_YAW)];
      next_state[UNC_POS_X] = Sa[cm(U_POS_X, U_POS_X)];
      next_state[UNC_POS_X_Y] = Sa[cm(U_POS_Y, U_POS_X)];
      next_state[UNC_POS_Y] = Sa[cm(U_POS_Y, U_POS_Y)];
    }
  }

  // computeLSTMSteering (device), lstm_steering.cu:131-166, with the steering network's evaluation handed in
  // (NET(in) -> head output): state_der's STEER_ANGLE_RATE and STEER_ANGLE
  template <class NET>
  __device__ static __forceinline__ void lstmSteering(const mppib_racer_lstm_dyn_params& p, const float* state,
                                                      const float* control, float* state_der, NET&& net)
  {
    const float parametric_accel = (control[1] * p.steer_command_angle_scale - state[STEER_ANGLE]) * p.steering_constant;
    state_der[STEER_ANGLE_RATE] = fmaxf(fminf((parametric_accel - state[STEER_ANGLE_RATE]) * p.steer_accel_constant -
                                                  state[STEER_ANGLE_RATE] * p.steer_accel_drag_constant,
                                              p.max_steer_rate),
                                        -p.max_steer_rate);
    float in[MPPIB_RACER_LSTM_INPUT_DIM];
    in[0] = state[STEER_ANGLE] * 0.2f;
    in[1] = state[STEER_ANGLE_RATE] * 0.2f;
    in[2] = control[1];
    in[3] = state_der[STEER_ANGLE_RATE] * 0.2f;
    const float nn_output = net(in);
    state_der[STEER_ANGLE_RATE] += nn_output * 5.0f;
    state_der[STEER_ANGLE] = state[STEER_ANGLE_RATE];
  }

  // roll, pitch and height over the elevation map, then the outputs
  __device__ static __forceinline__ void settleAndOutput(const ElevationMap& elev, const float* state,
                                                         const float* state_der, float* next_state, float* output)
  {
    // static settling (lstm_steering.cu:105-112 -> racer_dubins.cu:359-434); flat ground without a map (:427-432)
    float roll = state[ROLL], pitch = state[PITCH], height;
    racer_static_settling(elev, next_state[YAW], next_state[POS_X], next_state[POS_Y], roll, pitch, height);
    output[O_POS_I_Z] = height;
    next_state[PITCH] = pitch;
    next_state[ROLL] = roll;
    setOutputs(state_der, next_state, output);
  }
};
using RacerElevationParts = RacerElevationPartsT<8, 9>;  // racer_dubins_elevation.cuh:18-39

struct RacerLSTMDynamics : public Dynamics<RacerLSTMDynamics, mppib_racer_lstm_dyn_params, 19, 2, 28>, RacerElevationParts
{
  static constexpr int I = MPPIB_RACER_LSTM_INPUT_DIM;
  static constexpr int MAX_BLOCK_THREADS = 128;
  static constexpr int MAX_DISTRIBUTIONS = 1;  // the per-sample LSTM state is keyed by thread only
  static constexpr bool UNROLL_STEPS = false;
  static constexpr int MAX_HIDDEN = 64, MAX_HEAD = 64;
  struct Aux
  {
    const float* theta_d;  // MPPIB_BLOB_LSTM_WEIGHTS: LSTM block then head block (params.h)
    int H, L1;
    ElevationMap elev;     // MPPIB_BLOB_ELEVATION_MAP (hdr.use == 0: flat ground)
  };
  // compile-time fast path: the reference's test architecture (racer_dubins_elevation_lstm_steering_model_test.cu:26-32)
  // keeps h and c in registers and runs fully unrolled; any other (H, L1) takes the run-time loops over shared memory
  static constexpr int FAST_H = 4, FAST_L1 = 20;
  struct Carry
  {
    float h[FAST_H], c[FAST_H];
  };
  struct Layout
  {
    int gate, w1t, b1, w2, b2, per_thread, L1p, total;
  };
  __host__ __device__ static Layout layout(int H, int L1, int bx)
  {
    Layout l;
    l.L1p = (L1 + 3) & ~3;
    l.gate = 0;
    l.w1t = l.gate + 4 * H * (I + H + 1);
    l.b1 = l.w1t + (H + I) * l.L1p;
    l.w2 = l.b1 + l.L1p;
    l.b2 = l.w2 + l.L1p;
    l.per_thread = l.b2 + 4;
    l.total = l.per_thread + ((H == FAST_H && L1 == FAST_L1) ? 0 : 3 * H * bx);
    return l;
  }
  static int sharedFloats(const int* model_dims, int bx)
  {
    return layout(model_dims[0], model_dims[1], bx).total;
  }
  // lstm_steering.cu:115-128 (initializeDynamics: LSTMHelper::initialize copies the weights to shared memory and the
  // initial hidden / cell state into the sample's slice; outputs from the initial state)
  __device__ static __forceinline__ void initializeDynamics(const Params&, const Aux& aux, float* theta_s, Carry& carry,
                                                            const float* x, float* y)
  {
    initializeNetwork(aux, theta_s, carry);
    setOutputs(x, x, y);  // lstm_steering.cu:128
  }
  // the network part of initializeDynamics, shared with the suspension model
  __device__ static __forceinline__ void initializeNetwork(const Aux& aux, float* theta_s, Carry& carry)
  {
    const int H = aux.H, L1 = aux.L1, bx = blockDim.x, tid = threadIdx.x;
    const Layout l = layout(H, L1, bx);
    const float* g = aux.theta_d;
    const int HH = H * H, IH = H * I;
    const float* gb = g + 4 * HH + 4 * IH;  // b_i b_f b_o b_c
    // gate rows
    const int row_f4 = I + H + 1;
    for (int q = tid; q < H * row_f4; q += bx)
    {
      const int i = q / row_f4, j = q - i * row_f4;
      float4 v;
      if (j < I)
      {  // (W_ii, W_fi, W_oi, W_ci)[i][j]
        const float* w = g + 4 * HH + i * I + j;
        v = make_float4(w[0], w[IH], w[2 * IH], w[3 * IH]);
      }
      else if (j < I + H)
      {  // (W_im, W_fm, W_om, W_cm)[i][j - I]
        const float* w = g + i * H + (j - I);
        v = make_float4(w[0], w[HH], w[2 * HH], w[3 * HH]);
      }
      else
        v = make_float4(gb[i], gb[H + i], gb[2 * H + i], gb[3 * H + i]);
      reinterpret_cast<float4*>(theta_s + l.gate)[q] = v;
    }
    // head {H+I, L1, 1}: W1 (L1 x (H+I) row-major) | b1 | W2 (1 x L1) | b2   (fnn_helper.cu:176-183)
    const float* hd = g + 4 * HH + 4 * IH + 6 * H;
    const int IN = H + I;
    for (int q = tid; q < IN * l.L1p; q += bx)
    {
      const int j = q / l.L1p, k = q - j * l.L1p;
      theta_s[l.w1t + q] = (k < L1) ? hd[k * IN + j] : 0.0f;
    }
    for (int k = tid; k < l.L1p; k += bx)
    {
      theta_s[l.b1 + k] = (k < L1) ? hd[L1 * IN + k] : 0.0f;
      theta_s[l.w2 + k] = (k < L1) ? hd[L1 * IN + L1 + k] : 0.0f;
    }
    if (tid == 0)
      theta_s[l.b2] = hd[L1 * IN + L1 + L1];
    // per-sample hidden / cell state <- initial_hidden_, initial_cell_ (lstm_helper.cu:86-87)
    const float* init = gb + 4 * H;
    if (H == FAST_H && L1 == FAST_L1)
    {
#pragma unroll
      for (int j = 0; j < FAST_H; j++)
      {
        carry.h[j] = init[j];
        carry.c[j] = init[FAST_H + j];
      }
    }
    else
    {
      float* pt = theta_s + l.per_thread;
      for (int j = 0; j < H; j++)
      {
        pt[j * bx + tid] = init[j];               // hA
        pt[(2 * H + j) * bx + tid] = init[H + j];  // c
      }
    }
  }

  __device__ static __forceinline__ float sigmoid_dev(float v)
  {
    return (1.0f + tanh_fast(v * 0.5f)) * 0.5f;  // activation_functions.cuh:49-59, device branch
  }


  // Same arithmetic and summation order as lstm_forward below with H, L1 known at compile time: every weight access is
  // a broadcast LDS.128 at a constant offset, so ptxas batches the loads ahead of the FMA chains.
  template <int HC, int L1C>
  __device__ static __forceinline__ float lstm_forward_ct(const float* theta_s, const float (&in)[I], Carry& k)
  {
    constexpr int row_f4 = I + HC + 1, L1p = (L1C + 3) & ~3;
    constexpr int off_w1t = 4 * HC * row_f4, off_b1 = off_w1t + (HC + I) * L1p, off_w2 = off_b1 + L1p,
                  off_b2 = off_w2 + L1p;
    const float4* G = reinterpret_cast<const float4*>(theta_s);
    float hn[HC];
    // the four gate sums of a row and the four neurons of a head group as two packed FFMA2 each: every lane is the same
    // IEEE fma in the same order as the scalar form (lstm_forward), so the results are identical; the kernel is issue-bound
    // (66 % issue active) and the packed form removed ~140 of its ~1060 instructions per warp-step on packed-FMA hardware.
    float2 in2[I], h2[HC];
#pragma unroll
    for (int j = 0; j < I; j++)
      in2[j] = make_float2(in[j], in[j]);
#pragma unroll
    for (int j = 0; j < HC; j++)
      h2[j] = make_float2(k.h[j], k.h[j]);
#pragma unroll
    for (int i = 0; i < HC; i++)
    {
      const float4* row = G + i * row_f4;
      float2 g_if = make_float2(0.0f, 0.0f), g_oc = make_float2(0.0f, 0.0f);
#pragma unroll
      for (int j = 0; j < I; j++)
      {
        const float4 w = row[j];
        g_if = fma2_rn(make_float2(w.x, w.y), in2[j], g_if);
        g_oc = fma2_rn(make_float2(w.z, w.w), in2[j], g_oc);
      }
#pragma unroll
      for (int j = 0; j < HC; j++)
      {
        const float4 w = row[I + j];
        g_if = fma2_rn(make_float2(w.x, w.y), h2[j], g_if);
        g_oc = fma2_rn(make_float2(w.z, w.w), h2[j], g_oc);
      }
      const float4 b = row[I + HC];
      const float gi = sigmoid_dev(g_if.x + b.x), gf = sigmoid_dev(g_if.y + b.y), go = sigmoid_dev(g_oc.x + b.z),
                  gc = tanh_fast(g_oc.y + b.w);
      k.c[i] = gi * gc + gf * k.c[i];
      hn[i] = tanh_fast(k.c[i]) * go;
    }
#pragma unroll
    for (int i = 0; i < HC; i++)
      k.h[i] = hn[i];
    const float* W1T = theta_s + off_w1t;
    float out = 0.0f;
    float2 hn2[HC];
#pragma unroll
    for (int j = 0; j < HC; j++)
      hn2[j] = make_float2(hn[j], hn[j]);
#pragma unroll
    for (int k4 = 0; k4 < L1p; k4 += 4)
    {
      float2 acc_xy = make_float2(0.0f, 0.0f), acc_zw = make_float2(0.0f, 0.0f);
#pragma unroll
      for (int j = 0; j < HC + I; j++)
      {
        const float4 w = *reinterpret_cast<const float4*>(W1T + j * L1p + k4);
        const float2 a = j < HC ? hn2[j < HC ? j : 0] : in2[j < HC ? 0 : j - HC];
        acc_xy = fma2_rn(make_float2(w.x, w.y), a, acc_xy);
        acc_zw = fma2_rn(make_float2(w.z, w.w), a, acc_zw);
      }
      const float4 b = *reinterpret_cast<const float4*>(theta_s + off_b1 + k4);
      const float4 w2 = *reinterpret_cast<const float4*>(theta_s + off_w2 + k4);
      out = fmaf(w2.x, tanh_fast(acc_xy.x + b.x), out);
      out = fmaf(w2.y, tanh_fast(acc_xy.y + b.y), out);
      out = fmaf(w2.z, tanh_fast(acc_zw.x + b.z), out);
      out = fmaf(w2.w, tanh_fast(acc_zw.y + b.w), out);
    }
    return out + theta_s[off_b2];
  }

  // LSTMHelper::forward (device) + head; returns the head's single output. h is read from the buffer of parity
  // (t & 1) and written to the other one.
  __device__ static __forceinline__ float lstm_forward(const Aux& aux, float* theta_s, const float (&in)[I], int t)
  {
    const int H = aux.H, bx = blockDim.x, tid = threadIdx.x;
    const Layout l = layout(H, aux.L1, bx);
    float* pt = theta_s + l.per_thread + tid;
    const float* h_old = pt + ((t & 1) ? H * bx : 0);
    float* h_new = pt + ((t & 1) ? 0 : H * bx);
    float* cell = pt + 2 * H * bx;
    const int row_f4 = I + H + 1;
    const float4* G = reinterpret_cast<const float4*>(theta_s + l.gate);
    for (int i = 0; i < H; i++)
    {
      const float4* row = G + i * row_f4;
      float gi = 0.0f, gf = 0.0f, go = 0.0f, gc = 0.0f;
#pragma unroll
      for (int j = 0; j < I; j++)
      {
        const float4 w = row[j];
        gi = fmaf(w.x, in[j], gi);
        gf = fmaf(w.y, in[j], gf);
        go = fmaf(w.z, in[j], go);
        gc = fmaf(w.w, in[j], gc);
      }
#pragma unroll 4
      for (int j = 0; j < H; j++)
      {
        const float4 w = row[I + j];
        const float hj = h_old[j * bx];
        gi = fmaf(w.x, hj, gi);
        gf = fmaf(w.y, hj, gf);
        go = fmaf(w.z, hj, go);
        gc = fmaf(w.w, hj, gc);
      }
      const float4 b = row[I + H];
      gi = sigmoid_dev(gi + b.x);
      gf = sigmoid_dev(gf + b.y);
      go = sigmoid_dev(go + b.z);
      gc = tanh_fast(gc + b.w);
      const float c_next = gi * gc + gf * cell[i * bx];
      cell[i * bx] = c_next;
      h_new[i * bx] = tanh_fast(c_next) * go;
    }
    // head on [h_new ; input]: layer 1 (tanh) four neurons at a time, layer 2 (linear, one output) folded in
    const int L1p = l.L1p;
    const float* W1T = theta_s + l.w1t;
    float out = 0.0f;
    for (int k4 = 0; k4 < L1p; k4 += 4)
    {
      float4 acc = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
#pragma unroll 4
      for (int j = 0; j < H; j++)
      {
        const float4 w = *reinterpret_cast<const float4*>(W1T + j * L1p + k4);
        const float a = h_new[j * bx];
        acc.x = fmaf(w.x, a, acc.x);
        acc.y = fmaf(w.y, a, acc.y);
        acc.z = fmaf(w.z, a, acc.z);
        acc.w = fmaf(w.w, a, acc.w);
      }
#pragma unroll
      for (int j = 0; j < I; j++)
      {
        const float4 w = *reinterpret_cast<const float4*>(W1T + (H + j) * L1p + k4);
        acc.x = fmaf(w.x, in[j], acc.x);
        acc.y = fmaf(w.y, in[j], acc.y);
        acc.z = fmaf(w.z, in[j], acc.z);
        acc.w = fmaf(w.w, in[j], acc.w);
      }
      const float4 b = *reinterpret_cast<const float4*>(theta_s + l.b1 + k4);
      const float4 w2 = *reinterpret_cast<const float4*>(theta_s + l.w2 + k4);  // zero for the padding neurons
      out = fmaf(w2.x, tanh_fast(acc.x + b.x), out);
      out = fmaf(w2.y, tanh_fast(acc.y + b.y), out);
      out = fmaf(w2.z, tanh_fast(acc.z + b.z), out);
      out = fmaf(w2.w, tanh_fast(acc.w + b.w), out);
    }
    return out + theta_s[l.b2];
  }

  __device__ static __forceinline__ void step(const Params& p, const Aux& aux, float* theta_s, Carry& carry,
                                              const float* state, float* next_state, float* state_der,
                                              const float* control, float* output, int t, float dt)
  {
    stepWith(p, aux.elev, state, next_state, state_der, control, output, dt,
             [&](const float(&in)[I]) { return forward(aux, theta_s, carry, in, t); });
  }
  // the steering network on one input: the compile-time path at (FAST_H, FAST_L1), the run-time loops otherwise
  __device__ static __forceinline__ float forward(const Aux& aux, float* theta_s, Carry& carry, const float (&in)[I], int t)
  {
    return (aux.H == FAST_H && aux.L1 == FAST_L1) ? lstm_forward_ct<FAST_H, FAST_L1>(theta_s, in, carry) :
                                                    lstm_forward(aux, theta_s, in, t);
  }
  // the step with the steering network's evaluation handed in (NET(in) -> head output): shared with the tensor-core form
  template <class NET>
  __device__ static __forceinline__ void stepWith(const Params& p, const ElevationMap& elev, const float* state,
                                                  float* next_state, float* state_der, const float* control,
                                                  float* output, float dt, NET&& net)
  {
    const Kinematics k = parametricDeriv(p, state, control, state_der);
    lstmSteering(p, state, control, state_der, net);
    // updateState (device), lstm_steering.cu:240-262
#pragma unroll
    for (int i = 0; i < 6; i++)
      next_state[i] = state[i] + state_der[i] * dt;
    next_state[YAW] = normalizeAngle(next_state[YAW]);
    next_state[STEER_ANGLE] = fmaxf(fminf(next_state[STEER_ANGLE], p.max_steer_angle), -p.max_steer_angle);
    next_state[STEER_ANGLE_RATE] = state[STEER_ANGLE_RATE] + state_der[STEER_ANGLE_RATE] * dt;
    next_state[BRAKE_STATE] = fminf(fmaxf(next_state[BRAKE_STATE], 0.0f), 1.0f);
    propagateUncertainty(p, k, state, state_der, next_state, dt);
    settleAndOutput(elev, state, state_der, next_state, output);
  }
};

// ---- RacerDubinsElevationLSTMSteering with the steering LSTM on tensor cores (plugins/lstm_mma.cuh): hidden_dim 32, head
//      width <= 24. A warp carries 16 samples (lanes l and l + 16 the same one, rollout_kernel.cuh: SAMPLES_PER_WARP); the LSTM's
//      hidden and cell state live in mma fragment layout in the warp's registers across the whole horizon. Everything around
//      the network is RacerLSTMDynamics'. Chosen by engine.cu from mppib_desc.model_dims. ------------------------------------
struct RacerLSTMMmaDynamics : public Dynamics<RacerLSTMMmaDynamics, mppib_racer_lstm_dyn_params, 19, 2, 28>
{
  using Base = RacerLSTMDynamics;
  static constexpr int I = Base::I;
  static constexpr int SAMPLES_PER_WARP = 16;
  using AuxDyn = RacerLSTMDynamics;  // the one-thread-per-rollout auxiliary kernels keep the one-thread-per-sample network
  static constexpr int MAX_BLOCK_THREADS = 256;
  static constexpr int MAX_DISTRIBUTIONS = 1;
  static constexpr bool UNROLL_STEPS = false;
  using Aux = Base::Aux;
  using Carry = lstm_mma::State;
  static int sharedFloats(const int* /*model_dims*/, int bx)
  {
    return lstm_mma::sharedFloats(bx / SAMPLES_PER_WARP);
  }
  __device__ static __forceinline__ void initializeDynamics(const Params&, const Aux& aux, float* theta_s, Carry& carry,
                                                            const float* x, float* y)
  {
    lstm_mma::load_weights(aux.theta_d, aux.L1, theta_s);
    lstm_mma::init_state(aux.theta_d, carry);
    Base::setOutputs(x, x, y);  // lstm_steering.cu:128
  }
  // warp-collective: every lane of the warp calls it (the rollout kernels keep out-of-range rows running)
  __device__ static __forceinline__ void step(const Params& p, const Aux& aux, float* theta_s, Carry& carry,
                                              const float* state, float* next_state, float* state_der,
                                              const float* control, float* output, int /*t*/, float dt)
  {
    float* scratch = theta_s + lstm_mma::kFixedFloats + (threadIdx.x >> 5) * lstm_mma::kScratchPerWarp;
    Base::stepWith(p, aux.elev, state, next_state, state_der, control, output, dt,
                   [&](const float(&in)[I]) { return lstm_mma::forward(theta_s, scratch, in, carry); });
  }
};

// ---- RacerDubinsElevationSuspension: dynamics/racer_dubins/racer_dubins_elevation_suspension_lstm.cu:343-391 (device
//      step), :200-340 (computeSimpleSuspensionStep), :394-418 (updateState), :438-525 (setOutputs) -----------------------
// The LSTM-steering vehicle with roll, pitch and heave integrated from four spring-damper wheels over the elevation map and
// the normals map, instead of the static settling. State layout racer_dubins_elevation_suspension_lstm.cuh:25-52 (S = 24):
// the shared parts at STEER_ANGLE_RATE = 12 and the uncertainty entries at 13..22.
struct RacerSuspensionParams : mppib_racer_lstm_dyn_params  // mppib_racer_suspension_dyn_params with the LSTM blob as base
{
  float spring_k, drag_c, mass, I_xx, I_yy, wheel_radius, c_g[3];
};
static_assert(sizeof(RacerSuspensionParams) == sizeof(mppib_racer_suspension_dyn_params), "blob layout");

struct RacerSuspensionParts : RacerElevationPartsT<12, 13>
{
  enum
  {
    CG_POS_Z = 8, CG_VEL_I_Z, ROLL_RATE, PITCH_RATE, FILLER_1 = 23
  };
  struct Aux : RacerLSTMDynamics::Aux
  {
    NormalsMap normals;  // MPPIB_BLOB_NORMALS_MAP (hdr.use == 0: every normal (0, 0, 1))
  };
  struct WheelForces
  {
    float up, fwd, side;
  };
  // computeSimpleSuspensionStep (device): state_der's ROLL, PITCH, CG_POS_Z, CG_VEL_I_Z, ROLL_RATE and PITCH_RATE, and the
  // maxima of the wheel forces. The reference sums the wheels with atomicAdd_block in no fixed order; here in wheel order,
  // which is the host's.
  __device__ static __forceinline__ WheelForces suspensionStep(const RacerSuspensionParams& p, const ElevationMap& elev,
                                                               const NormalsMap& normals, const float* state,
                                                               float* state_der)
  {
    const float x = state[POS_X], y = state[POS_Y], roll = state[ROLL], pitch = state[PITCH], yaw = state[YAW];
    state_der[ROLL] = state[ROLL_RATE];
    state_der[PITCH] = state[PITCH_RATE];
    state_der[CG_POS_Z] = state[CG_VEL_I_Z];
    float d_vz = 0.0f, d_roll_rate = 0.0f, d_pitch_rate = 0.0f;
    // mppi::math::Euler2DCM_NWU (device branch: fast sincos of normalised angles)
    float sr, cr, sp, cp, sy, cy;
    __sincosf(normalizeAngle(roll), &sr, &cr);
    __sincosf(normalizeAngle(pitch), &sp, &cp);
    __sincosf(normalizeAngle(yaw), &sy, &cy);
    const float M00 = cp * cy, M01 = sr * sp * cy - cr * sy, M10 = cp * sy, M11 = sr * sp * sy + cr * cy, M20 = -sp,
                M21 = sr * cp;
    float wheel_height = 0.0f;
    float4 n = make_float4(0.0f, 0.0f, 1.0f, 0.0f);
    WheelForces f{ 0.0f, 0.0f, 0.0f };
    // the divisions by mass, I_xx, I_yy and the normal's z go through a Newton-refined reciprocal (within an ulp of the
    // quotient): sixteen IEEE divisions per step each carry a slow-path call, around which the rollout kernels spilled
    const float inv_mass = rcp_nr(p.mass), inv_I_xx = rcp_nr(p.I_xx), inv_I_yy = rcp_nr(p.I_yy);
#pragma unroll
    for (int i = 0; i < 4; i++)
    {  // FL, FR, BL, BR (the rear labels carry swapped y signs in the reference: :266-271)
      const float bx = (i < 2) ? 2.981f : 0.0f, by = (i == 0 || i == 3) ? 0.737f : -0.737f;
      // front wheels: yaw + S_INDEX(STEER_ANGLE) / -9.1, the constant index 4 and not the steering state (:260, :264)
      const float wheel_yaw = (i < 2) ? yaw + 4.0f / -9.1f : yaw;
      float sin_wy, cos_wy;
      __sincosf(wheel_yaw, &sin_wy, &cos_wy);
      const float cgx = bx - p.c_g[0], cgy = by - p.c_g[1];
      // bodyOffsetToWorldPoseDCM with the body pose (x, y, 0)
      const float wx = M00 * bx + M01 * by + x, wy = M10 * bx + M11 * by + y, wz = M20 * bx + M21 * by + 0.0f;
      if (elev.hdr.use)
      {
        wheel_height = elevation_at_world_pose(elev, wx, wy, wz);
        if (!isfinite(wheel_height))
          wheel_height = state[CG_POS_Z] - p.wheel_radius;
      }
      if (normals.hdr.use)
      {
        n = normal_at_world_pose(normals, wx, wy, wz);
        if (!isfinite(n.x) || !isfinite(n.y) || !isfinite(n.z))
          n = make_float4(0.0f, 0.0f, 1.0f, 0.0f);
      }
      const float wheel_pos_z = state[CG_POS_Z] + roll * cgy - pitch * cgx - p.wheel_radius;
      const float wheel_vel_z = state[CG_VEL_I_Z] + state[ROLL_RATE] * cgy - state[PITCH_RATE] * cgx;
      const float h_dot = -(state[VEL_X] * cos_wy * n.x + state[VEL_X] * sin_wy * n.y);
      const float F = -p.spring_k * (wheel_pos_z - wheel_height) - p.drag_c * (wheel_vel_z - h_dot);
      const float F_nz = F * rcp_nr(n.z);
      const float fwd = fabsf(F_nz * (n.x * cos_wy + n.y * sin_wy + n.z * (-pitch)));
      const float side = fabsf(F_nz * (-n.x * sin_wy + n.y * cos_wy + n.z * roll));
      f.up = i == 0 ? F : fmaxf(f.up, F);
      f.fwd = i == 0 ? fwd : fmaxf(f.fwd, fwd);
      f.side = i == 0 ? side : fmaxf(f.side, side);
      d_vz += F * inv_mass;
      d_roll_rate += F * cgy * inv_I_xx;
      d_pitch_rate += -F * cgx * inv_I_yy;
    }
    state_der[CG_VEL_I_Z] = d_vz;
    state_der[ROLL_RATE] = d_roll_rate;
    state_der[PITCH_RATE] = d_pitch_rate;
    return f;
  }

  // the device step after the steering network: suspension, updateState, uncertainty propagation and setOutputs
  template <class NET>
  __device__ static __forceinline__ void stepWith(const RacerSuspensionParams& p, const Aux& aux, const float* state,
                                                  float* next_state, float* state_der, const float* control,
                                                  float* output, float dt, NET&& net)
  {
    const Kinematics k = parametricDeriv(p, state, control, state_der);
    lstmSteering(p, state, control, state_der, net);
    const WheelForces f = suspensionStep(p, aux.elev, aux.normals, state, state_der);
    // updateState (device), :394-418: every index below STEER_ANGLE_RATE, roll, pitch, heave and their rates included
#pragma unroll
    for (int i = 0; i < STEER_ANGLE_RATE; i++)
      next_state[i] = state[i] + state_der[i] * dt;
    next_state[YAW] = normalizeAngle(next_state[YAW]);
    next_state[STEER_ANGLE] = fmaxf(fminf(next_state[STEER_ANGLE], p.max_steer_angle), -p.max_steer_angle);
    next_state[STEER_ANGLE_RATE] = state[STEER_ANGLE_RATE] + state_der[STEER_ANGLE_RATE] * dt;
    next_state[BRAKE_STATE] = fminf(fmaxf(next_state[BRAKE_STATE], 0.0f), 1.0f);
    next_state[FILLER_1] = state[FILLER_1];
    propagateUncertainty(p, k, state, state_der, next_state, dt);
    // setOutputs, :438-525: no static settling (the call is commented out at :373-382)
    setOutputs(state_der, next_state, output);
    output[O_POS_I_Z] = next_state[CG_POS_Z] - next_state[PITCH] * (-p.c_g[0]);
    output[O_WF_UP] = f.up;
    output[O_WF_FWD] = f.fwd;
    output[O_WF_SIDE] = f.side;
  }
};

// the one-thread-per-sample steering network of RacerLSTMDynamics: the compile-time H = 4 / L1 = 20 path and the run-time
// loops
struct RacerSuspensionLSTMDynamics : public Dynamics<RacerSuspensionLSTMDynamics, RacerSuspensionParams, 24, 2, 28>,
                                     RacerSuspensionParts
{
  using Net = RacerLSTMDynamics;
  using Aux = RacerSuspensionParts::Aux;
  using Carry = Net::Carry;
  static constexpr int I = Net::I;
  static constexpr int MAX_BLOCK_THREADS = Net::MAX_BLOCK_THREADS;
  static constexpr int MAX_DISTRIBUTIONS = 1;  // the per-sample LSTM state is keyed by thread only
  static constexpr bool UNROLL_STEPS = false;
  static int sharedFloats(const int* model_dims, int bx)
  {
    return Net::sharedFloats(model_dims, bx);
  }
  __device__ static __forceinline__ void initializeDynamics(const Params&, const Aux& aux, float* theta_s, Carry& carry,
                                                            const float* x, float* y)
  {
    Net::initializeNetwork(aux, theta_s, carry);
    setOutputs(x, x, y);  // lstm_steering.cu:128 (the inherited setOutputs)
  }
  __device__ static __forceinline__ void step(const Params& p, const Aux& aux, float* theta_s, Carry& carry,
                                              const float* state, float* next_state, float* state_der,
                                              const float* control, float* output, int t, float dt)
  {
    stepWith(p, aux, state, next_state, state_der, control, output, dt,
             [&](const float(&in)[I]) { return Net::forward(aux, theta_s, carry, in, t); });
  }
};

// the steering LSTM on tensor cores (plugins/lstm_mma.cuh) at hidden_dim 32, as RacerLSTMMmaDynamics
struct RacerSuspensionLSTMMmaDynamics : public Dynamics<RacerSuspensionLSTMMmaDynamics, RacerSuspensionParams, 24, 2, 28>
{
  using Base = RacerSuspensionLSTMDynamics;
  static constexpr int I = Base::I;
  static constexpr int SAMPLES_PER_WARP = 16;
  using AuxDyn = RacerSuspensionLSTMDynamics;
  static constexpr int MAX_BLOCK_THREADS = 256;
  static constexpr int MAX_DISTRIBUTIONS = 1;
  static constexpr bool UNROLL_STEPS = false;
  using Aux = Base::Aux;
  using Carry = lstm_mma::State;
  static int sharedFloats(const int* /*model_dims*/, int bx)
  {
    return lstm_mma::sharedFloats(bx / SAMPLES_PER_WARP);
  }
  __device__ static __forceinline__ void initializeDynamics(const Params&, const Aux& aux, float* theta_s, Carry& carry,
                                                            const float* x, float* y)
  {
    lstm_mma::load_weights(aux.theta_d, aux.L1, theta_s);
    lstm_mma::init_state(aux.theta_d, carry);
    Base::setOutputs(x, x, y);
  }
  // warp-collective: every lane of the warp calls it
  __device__ static __forceinline__ void step(const Params& p, const Aux& aux, float* theta_s, Carry& carry,
                                              const float* state, float* next_state, float* state_der,
                                              const float* control, float* output, int /*t*/, float dt)
  {
    float* scratch = theta_s + lstm_mma::kFixedFloats + (threadIdx.x >> 5) * lstm_mma::kScratchPerWarp;
    Base::stepWith(p, aux, state, next_state, state_der, control, output, dt,
                   [&](const float(&in)[I]) { return lstm_mma::forward(theta_s, scratch, in, carry); });
  }
};

// ---- RacerDubinsElevation: dynamics/racer_dubins/racer_dubins_elevation.cu:835-878 (device step), racer_dubins.cu:281-304
//      (brake delay, first-order steering), racer_dubins_elevation.cu:759-797 (parametric acceleration, device), :800-832
//      (updateState, device), :257-334 (computeGrad) -------------------------------------------------------------------
// The parametric RACER vehicle. One thread = one sample with nothing but x carried between steps, so Tube-MPPI and RMPPI
// roll two systems per thread; everything but the steering and updateState is RacerElevationParts'.
struct RacerDubinsElevationDynamics
    : public Dynamics<RacerDubinsElevationDynamics, mppib_racer_dubins_elevation_dyn_params, 19, 2, 28>, RacerElevationParts
{
  static constexpr bool UNROLL_STEPS = false;
  struct Aux
  {
    ElevationMap elev;  // MPPIB_BLOB_ELEVATION_MAP (hdr.use == 0: flat ground)
  };
  // dynamics.cuh:429-435 (racer_dubins_elevation.cu:745-756 adds only the params copy to shared memory)
  __device__ static __forceinline__ void initializeDynamics(const Params&, const Aux&, float*, Carry&, const float* x,
                                                            float* y)
  {
#pragma unroll
    for (int i = 0; i < 19; i++)
      y[i] = x[i];
  }

  // computeParametricSteerDeriv (device), racer_dubins.cu:296-304
  __device__ static __forceinline__ void steerDeriv(const Params& p, const float* state, const float* control,
                                                    float* state_der)
  {
    state_der[STEER_ANGLE] =
        fmaxf(fminf((control[1] * p.steer_command_angle_scale - state[STEER_ANGLE]) * p.steering_constant,
                    p.max_steer_rate),
              -p.max_steer_rate);
  }

  __device__ static __forceinline__ void step(const Params& p, const Aux& aux, float*, Carry&, const float* state,
                                              float* next_state, float* state_der, const float* control, float* output,
                                              int /*t*/, float dt)
  {
    const Kinematics k = parametricDeriv(p, state, control, state_der);
    steerDeriv(p, state, control, state_der);
    // updateState (device), racer_dubins_elevation.cu:800-832: the steering rate is the derivative, not integrated
#pragma unroll
    for (int i = 0; i < 6; i++)
      next_state[i] = state[i] + state_der[i] * dt;
    next_state[YAW] = normalizeAngle(next_state[YAW]);
    next_state[STEER_ANGLE] = fmaxf(fminf(next_state[STEER_ANGLE], p.max_steer_angle), -p.max_steer_angle);
    next_state[STEER_ANGLE_RATE] = state_der[STEER_ANGLE];
    next_state[BRAKE_STATE] = fminf(fmaxf(next_state[BRAKE_STATE], 0.0f), 1.0f);
    propagateUncertainty(p, k, state, state_der, next_state, dt);
    settleAndOutput(aux.elev, state, state_der, next_state, output);
  }

  // f(x, u) of DDP (ddp_kernel.cuh): the step's six derivative rows. The reference's step leaves the other rows of
  // state_der as it found them (ddp_model_wrapper.h:68-81 passes a fresh vector); here they are zero, as are their rows of
  // computeGrad.
  __device__ static __forceinline__ void computeDynamics(const Params& p, const float*, const float* state,
                                                         const float* control, float* state_der)
  {
#pragma unroll
    for (int i = 0; i < 19; i++)
      state_der[i] = 0.0f;
    parametricDeriv(p, state, control, state_der);
    steerDeriv(p, state, control, state_der);
  }

  static constexpr bool HAS_GRAD = true;
  // RacerDubinsElevationImpl::computeGrad (racer_dubins_elevation.cu:257-334) as written: an approximate Jacobian (the
  // reference's own gradient test is skipped). Kept: A(4,4) clamped to +-max_steer_rate, the 0.01 margins on the rate
  // limits, and the brake-command row reading the throttle's lower limit control_rngs_[0].x (p.lim.rng_lo[0]).
  // Rows 6 .. 18 (roll, pitch, steering rate, uncertainty) are zero.
  __device__ static bool computeGrad(const Params& p, const Aux&, const float* x, const float* u, float* A, float* B)
  {
    for (int i = 0; i < 19 * 19; i++)
      A[i] = 0.0f;
    for (int i = 0; i < 19 * 2; i++)
      B[i] = 0.0f;
    auto a = [&](int r, int c) -> float& { return A[r * 19 + c]; };
    auto b = [&](int r, int c) -> float& { return B[r * 2 + c]; };
    const float eps = 0.01f;
    const bool enable_brake = u[0] < 0.0f;
    const float vx = x[VEL_X];
    const float linear_brake_slope = 0.2f;
    const int index = (fabsf(vx) > linear_brake_slope && fabsf(vx) <= 3.0f) + (fabsf(vx) > 3.0f) * 2;
    a(VEL_X, VEL_X) = -pick3(p.c_v, index);
    if (fabsf(vx) < linear_brake_slope)
      a(VEL_X, BRAKE_STATE) = pick3(p.c_b, index) * -vx;
    else
      a(VEL_X, BRAKE_STATE) = pick3(p.c_b, index) * (vx >= 0.0f ? -1.0f : 1.0f);
    const float delta = x[STEER_ANGLE] / p.steer_angle_scale;
    a(YAW, VEL_X) = (1.0f / p.wheel_base) * tanf(delta);
    a(YAW, STEER_ANGLE) = (vx / p.wheel_base) * (1.0f / MPPIB_SQ(cosf(delta))) / p.steer_angle_scale;
    const float sy = sinf(x[YAW]), cy = cosf(x[YAW]);
    a(POS_X, VEL_X) = cy;
    a(POS_X, YAW) = -sy * vx;
    a(POS_Y, VEL_X) = sy;
    a(POS_Y, YAW) = cy * vx;
    const float steer_dot = (u[1] * p.steer_command_angle_scale - x[STEER_ANGLE]) * p.steering_constant;
    if (steer_dot - eps < -p.max_steer_rate || steer_dot + eps > p.max_steer_rate)
      a(STEER_ANGLE, STEER_ANGLE) = 0.0f;
    else
      a(STEER_ANGLE, STEER_ANGLE) = -p.steering_constant;
    a(STEER_ANGLE, STEER_ANGLE) = fmaxf(fminf(a(STEER_ANGLE, STEER_ANGLE), p.max_steer_rate), -p.max_steer_rate);
    a(VEL_X, PITCH) = -p.gravity * cosf(x[PITCH]);
    const float brake_dot = (enable_brake * -u[0] - x[BRAKE_STATE]) * p.brake_delay_constant;
    if (brake_dot - eps < -p.max_brake_rate_neg || brake_dot + eps > p.max_brake_rate_pos)
      a(BRAKE_STATE, BRAKE_STATE) = 0.0f;
    else
      a(BRAKE_STATE, BRAKE_STATE) = -p.brake_delay_constant;
    b(STEER_ANGLE, 1) = p.steer_command_angle_scale * p.steering_constant;
    b(VEL_X, 0) = pick3(p.c_t, index) * p.gear_sign * (!enable_brake);
    if ((x[BRAKE_STATE] < -p.lim.rng_lo[0] && brake_dot < 0.0f) || (x[BRAKE_STATE] > 0.0f && brake_dot > 0.0f))
      b(BRAKE_STATE, 0) = -p.brake_delay_constant * enable_brake;
    return true;
  }
};

// ---- RacerSuspension: dynamics/racer_suspension/racer_suspension.cu:55-75 (device updateState), :93-298 (computeStateDeriv),
//      :300-306 (device step) --------------------------------------------------------------------------------------------
// The 6-DoF rigid-body RACER vehicle: quaternion attitude, body rates through Euler's equations, four spring-damper
// wheels with Stribeck side friction and a traction force limited by friction. The reference's elevation query is
// commented out (:128-135), so every wheel stands on the plane z = 0 with normal (0, 0, 1), and the terms of the body that
// only a tilted normal makes non-zero (h_dot, the normal's x / y) are left out. The host twin (host_twins.cpp) keeps the
// reference's host step: ω by approximate implicit Euler through the as-written Jacobian. This is the device one: explicit
// Euler on all 14 states. Divisions use rcp_nr (within 1 ulp of the quotient): 1 / mass, 1 / J (the reference's
// 1.0 / Jxx in double, rounded to float), the contact frame's 1 / |n x w| and the quaternion's 1 / |q|.
struct RacerRigidSuspensionDynamics
    : public Dynamics<RacerRigidSuspensionDynamics, mppib_racer_rigid_suspension_dyn_params, 14, 2, 26>
{
  enum
  {
    P_I_X = 0, P_I_Y, P_I_Z, Q_W, Q_X, Q_Y, Q_Z, V_I_X, V_I_Y, V_I_Z, OMEGA_B_X, OMEGA_B_Y, OMEGA_B_Z, STEER_ANGLE
  };
  enum
  {
    O_VEL_B_X = 0, O_POS_I_X = 3, O_YAW = 6, O_ROLL, O_PITCH, O_STEER_ANGLE, O_STEER_ANGLE_RATE, O_WHEEL_POS = 11,
    O_WHEEL_FORCE = 19, O_ACCEL_X = 23, O_ACCEL_Y, O_OMEGA_Z
  };
  static constexpr bool UNROLL_STEPS = false;
  // dynamics.cuh:429-435; the outputs past the state, which the reference leaves as it finds them, start at 0
  __device__ static __forceinline__ void initializeDynamics(const Params&, const Aux&, float*, Carry&, const float* x,
                                                            float* y)
  {
#pragma unroll
    for (int i = 0; i < 26; i++)
      y[i] = i < 14 ? x[i] : 0.0f;
  }

  // computeStateDeriv on flat ground: xdot of all 14 states, and the outputs of x (not of the next state)
  __device__ static __forceinline__ void stateDerivAndOutput(const Params& p, const float* x, const float* u, float* xd,
                                                             float* y)
  {
    const float qw = x[Q_W], qx = x[Q_X], qy = x[Q_Y], qz = x[Q_Z];
    // Eigen's Quaternion::toRotationMatrix
    const float tx = 2.0f * qx, ty = 2.0f * qy, tz = 2.0f * qz;
    const float twx = tx * qw, twy = ty * qw, twz = tz * qw, txx = tx * qx, txy = ty * qx, txz = tz * qx;
    const float tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
    const float R[3][3] = { { 1.0f - (tyy + tzz), txy - twz, txz + twy },
                            { txy + twz, 1.0f - (txx + tzz), tyz - twx },
                            { txz - twy, tyz + twx, 1.0f - (txx + tyy) } };
    const float* v = x + V_I_X;
    const float* w = x + OMEGA_B_X;
    const float tan_delta = tanf(x[STEER_ANGLE]);
    // the body-frame velocity of the CG, R^T v
    float vb[3];
#pragma unroll
    for (int i = 0; i < 3; i++)
      vb[i] = R[0][i] * v[0] + R[1][i] * v[1] + R[2][i] * v[2];

    // linear engine model (:108-113); copysign keeps the sign of a zero vel_x
    const float throttle = fmaxf(0.0f, u[0]), brake = fmaxf(0.0f, -u[0]);
    const float acc = p.c_t * throttle - copysignf(p.c_b * brake, vb[0]) - p.c_v * vb[0] + p.c_0;
    const float propulsion_force = p.mass * acc;

    float f_B[3] = { 0.0f, 0.0f, 0.0f }, tau_B[3] = { 0.0f, 0.0f, 0.0f };
#pragma unroll
    for (int i = 0; i < 4; i++)
    {
      // wheel position relative to the CG, in the body and the world frame; its world velocity v + R (w x p)
      const float pb[3] = { p.wheel_pos_wrt_base_link[i][0] - p.cg_pos_wrt_base_link[0],
                            p.wheel_pos_wrt_base_link[i][1] - p.cg_pos_wrt_base_link[1],
                            p.wheel_pos_wrt_base_link[i][2] - p.cg_pos_wrt_base_link[2] };
      const float wxp[3] = { w[1] * pb[2] - w[2] * pb[1], w[2] * pb[0] - w[0] * pb[2], w[0] * pb[1] - w[1] * pb[0] };
      float pw[3], pdot[3];
#pragma unroll
      for (int r = 0; r < 3; r++)
      {
        pw[r] = x[P_I_X + r] + (R[r][0] * pb[0] + R[r][1] * pb[1] + R[r][2] * pb[2]);
        pdot[r] = v[r] + (R[r][0] * wxp[0] + R[r][1] * wxp[1] + R[r][2] * wxp[2]);
      }
      // spring-damper on the spring length above the ground z = 0, clamped at 0 (wheel lift)
      float f_n = -p.k_s[i] * (pw[2] - p.l_0[i]) - p.c_s[i] * pdot[2];
      if (f_n < 0.0f)
        f_n = 0.0f;
      // Ackermann angle of the front wheels
      float delta = 0.0f;
      if (i == 0)
        delta = atanf(p.wheel_base * tan_delta / (p.wheel_base - tan_delta * p.width / 2));
      else if (i == 1)
        delta = atanf(p.wheel_base * tan_delta / (p.wheel_base + tan_delta * p.width / 2));
      float sd, cd;
      sincosf(delta, &sd, &cd);
      // contact frame: n = R^T (0, 0, 1), s = normalised n x (cos d, sin d, 0), t = s x n
      const float n[3] = { R[2][0], R[2][1], R[2][2] };
      float s[3] = { -n[2] * sd, n[2] * cd, n[0] * sd - n[1] * cd };
      const float inv_s = rcp_nr(sqrtf(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]));
#pragma unroll
      for (int r = 0; r < 3; r++)
        s[r] *= inv_s;
      const float t[3] = { s[1] * n[2] - s[2] * n[1], s[2] * n[0] - s[0] * n[2], s[0] * n[1] - s[1] * n[0] };
      // side slip velocity s . R^T (pdot_x, pdot_y, 0), Stribeck friction, traction clamped at +-mu f_n
      float v_s = 0.0f;
#pragma unroll
      for (int r = 0; r < 3; r++)
        v_s += s[r] * (R[0][r] * pdot[0] + R[1][r] * pdot[1]);
      float mu_s = v_s / p.v_slip * p.mu;
      mu_s = mu_s > p.mu ? p.mu : (mu_s < -p.mu ? -p.mu : mu_s);
      const float f_s = -mu_s * f_n;
      const float f_t = fmaxf(-p.mu * f_n, fminf(propulsion_force / 4, p.mu * f_n));
      const float f[3] = { t[0] * f_t + s[0] * f_s + n[0] * f_n, t[1] * f_t + s[1] * f_s + n[1] * f_n,
                           t[2] * f_t + s[2] * f_s + n[2] * f_n };
      // contact point in the body frame: R^T ((pw_x, pw_y, 0) - p_I)
      const float dc[3] = { pw[0] - x[P_I_X], pw[1] - x[P_I_Y], -x[P_I_Z] };
      float pc[3];
#pragma unroll
      for (int r = 0; r < 3; r++)
        pc[r] = R[0][r] * dc[0] + R[1][r] * dc[1] + R[2][r] * dc[2];
#pragma unroll
      for (int r = 0; r < 3; r++)
        f_B[r] += f[r];
      tau_B[0] += pc[1] * f[2] - pc[2] * f[1];
      tau_B[1] += pc[2] * f[0] - pc[0] * f[2];
      tau_B[2] += pc[0] * f[1] - pc[1] * f[0];
      y[O_WHEEL_POS + 2 * i] = pw[0];
      y[O_WHEEL_POS + 2 * i + 1] = pw[1];
      y[O_WHEEL_FORCE + i] = sqrtf(f[0] * f[0] + f[1] * f[1] + f[2] * f[2]);
    }

    // v_dot = R f / m + g, q_dot = q (x) (0, w) / 2, w_dot = J^-1 (J w x w + tau)
    const float inv_mass = rcp_nr(p.mass);
#pragma unroll
    for (int r = 0; r < 3; r++)
    {
      xd[P_I_X + r] = v[r];
      xd[V_I_X + r] = inv_mass * (R[r][0] * f_B[0] + R[r][1] * f_B[1] + R[r][2] * f_B[2]);
    }
    xd[V_I_Z] += p.gravity;
    xd[Q_W] = 0.5f * (-qx * w[0] - qy * w[1] - qz * w[2]);
    xd[Q_X] = 0.5f * (qw * w[0] + qy * w[2] - qz * w[1]);
    xd[Q_Y] = 0.5f * (qw * w[1] + qz * w[0] - qx * w[2]);
    xd[Q_Z] = 0.5f * (qw * w[2] + qx * w[1] - qy * w[0]);
    const float Jw[3] = { p.Jxx * w[0], p.Jyy * w[1], p.Jzz * w[2] };
    xd[OMEGA_B_X] = rcp_nr(p.Jxx) * ((Jw[1] * w[2] - Jw[2] * w[1]) + tau_B[0]);
    xd[OMEGA_B_Y] = rcp_nr(p.Jyy) * ((Jw[2] * w[0] - Jw[0] * w[2]) + tau_B[1]);
    xd[OMEGA_B_Z] = rcp_nr(p.Jzz) * ((Jw[0] * w[1] - Jw[1] * w[0]) + tau_B[2]);
    // first-order steering lag (:253-255)
    xd[STEER_ANGLE] = p.steering_constant * (u[1] / p.steer_command_angle_scale - x[STEER_ANGLE]);

    // outputs (:257-297). BASELINK_VEL_B_Y / _Z get their own components: the reference writes all three into
    // BASELINK_VEL_B_X (DESIGN §8). ACCEL_X, ACCEL_Y and OMEGA_Z are 0.
    const float cg[3] = { p.cg_pos_wrt_base_link[0], p.cg_pos_wrt_base_link[1], p.cg_pos_wrt_base_link[2] };
    y[O_VEL_B_X + 0] = vb[0] + (w[1] * -cg[2] - w[2] * -cg[1]);
    y[O_VEL_B_X + 1] = vb[1] + (w[2] * -cg[0] - w[0] * -cg[2]);
    y[O_VEL_B_X + 2] = vb[2] + (w[0] * -cg[1] - w[1] * -cg[0]);
#pragma unroll
    for (int r = 0; r < 3; r++)
      y[O_POS_I_X + r] = x[P_I_X + r] + (R[r][0] * -cg[0] + R[r][1] * -cg[1] + R[r][2] * -cg[2]);
    quat2EulerNWU(x + Q_W, y[O_ROLL], y[O_PITCH], y[O_YAW]);
    y[O_STEER_ANGLE] = x[STEER_ANGLE];
    y[O_STEER_ANGLE_RATE] = xd[STEER_ANGLE];
    y[O_ACCEL_X] = 0.0f;
    y[O_ACCEL_Y] = 0.0f;
    y[O_OMEGA_Z] = 0.0f;
  }

  // :300-306 with :55-75: the outputs are those of the state passed in, so the cost of step t sees x_t
  // (mppi_common.cu:118-127); then explicit Euler and q / |q|
  __device__ static __forceinline__ void step(const Params& p, const Aux&, float*, Carry&, const float* x, float* x_next,
                                              float* xd, const float* u, float* y, int /*t*/, float dt)
  {
    stateDerivAndOutput(p, x, u, xd, y);
#pragma unroll
    for (int i = 0; i < 14; i++)
      x_next[i] = x[i] + xd[i] * dt;
    float* q = x_next + Q_W;
    const float inv = rcp_nr(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]));
#pragma unroll
    for (int i = 0; i < 4; i++)
      q[i] *= inv;
  }
};

// ---- Quadrotor: dynamics/quadrotor/quadrotor_dynamics.cu:124-179 (device computeDynamics + updateState) with
//      Quat2DCM / omega2edot of utils/math_utils.h:272-283,534-540 ------------------------------------------------------
// The only in-tree model with CONTROL_DIM = 4: one 16-byte noise group is one time step (rollout_kernel.cuh).
struct QuadrotorDynamics : public Dynamics<QuadrotorDynamics, mppib_quadrotor_dyn_params, 13, 4, 13>
{
  __device__ static __forceinline__ void computeDynamics(const Params& p, const float*, const float* state,
                                                         const float* control, float* state_der)
  {
    const float* v = state + 3;
    const float* q = state + 6;
    const float* w = state + 10;
    const float u_thrust = control[3];
    // third column of Quat2DCM
    const float dcm02 = 2 * (q[1] * q[3] + q[0] * q[2]);
    const float dcm12 = 2 * (q[2] * q[3] - q[0] * q[1]);
    const float dcm22 = MPPIB_SQ(q[0]) - MPPIB_SQ(q[1]) - MPPIB_SQ(q[2]) + MPPIB_SQ(q[3]);
    const float accel = u_thrust * rcp_nr(p.mass);  // u_thrust / mass
    state_der[0] = v[0];
    state_der[1] = v[1];
    state_der[2] = v[2];
    state_der[3] = accel * dcm02;
    state_der[4] = accel * dcm12;
    state_der[5] = accel * dcm22 - MPPIB_GRAVITY;
    state_der[6] = 0.5f * (-w[0] * q[1] - w[1] * q[2] - w[2] * q[3]);
    state_der[7] = 0.5f * (w[0] * q[0] - w[1] * q[3] + w[2] * q[2]);
    state_der[8] = 0.5f * (w[0] * q[3] + w[1] * q[0] - w[2] * q[1]);
    state_der[9] = 0.5f * (-w[0] * q[2] + w[1] * q[1] + w[2] * q[0]);
    state_der[10] = (control[0] - w[0]) * rcp_nr(p.tau_roll);
    state_der[11] = (control[1] - w[1]) * rcp_nr(p.tau_pitch);
    state_der[12] = (control[2] - w[2]) * rcp_nr(p.tau_yaw);
  }
  // quadrotor_dynamics.cu:168-179: Euler step, then q /= |q| * copysignf(1, q_w)
  __device__ static __forceinline__ void updateState(const float* x, float* x_next, const float* xdot, float dt)
  {
#pragma unroll
    for (int i = 0; i < 13; i++)
      x_next[i] = x[i] + xdot[i] * dt;
    float* q = x_next + 6;
    const float q_norm = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const float inv = rcp_nr(q_norm * copysignf(1.0f, q[0]));
#pragma unroll
    for (int i = 0; i < 4; i++)
      q[i] *= inv;
  }

  static constexpr bool HAS_GRAD = true;
  // The exact Jacobian of computeDynamics above. The reference's QuadrotorDynamics::computeGrad (quadrotor_dynamics.cu:
  // 35-68) leaves dv/dq and dq/d(q, w) as TODOs, puts dq/dw in B and returns false, so its DDP wrapper falls back to numeric
  // differences of f (ddp_model_wrapper.h:83-95); this is the derivative those differences approximate.
  __device__ static bool computeGrad(const Params& p, const Aux&, const float* x, const float* u, float* A, float* B)
  {
    for (int i = 0; i < 169; i++)
      A[i] = 0.0f;
    for (int i = 0; i < 52; i++)
      B[i] = 0.0f;
    const float* q = x + 6;
    const float* w = x + 10;
    const float a = u[3] / p.mass;
    for (int i = 0; i < 3; i++)
      A[i * 13 + 3 + i] = 1.0f;  // dpos/dv
    // dv/dq: a * d(third column of Quat2DCM)/dq
    const float dcm[3][4] = { { 2 * q[2], 2 * q[3], 2 * q[0], 2 * q[1] },
                              { -2 * q[1], -2 * q[0], 2 * q[3], 2 * q[2] },
                              { 2 * q[0], -2 * q[1], -2 * q[2], 2 * q[3] } };
    for (int r = 0; r < 3; r++)
      for (int j = 0; j < 4; j++)
        A[(3 + r) * 13 + 6 + j] = a * dcm[r][j];
    B[3 * 4 + 3] = 2 * (q[1] * q[3] + q[0] * q[2]) / p.mass;
    B[4 * 4 + 3] = 2 * (q[2] * q[3] - q[0] * q[1]) / p.mass;
    B[5 * 4 + 3] = (q[0] * q[0] - q[1] * q[1] - q[2] * q[2] + q[3] * q[3]) / p.mass;
    // dq/dq and dq/dw of omega2edot
    const float dqq[4][4] = { { 0, -w[0], -w[1], -w[2] }, { w[0], 0, w[2], -w[1] }, { w[1], -w[2], 0, w[0] },
                              { w[2], w[1], -w[0], 0 } };
    const float dqw[4][3] = { { -q[1], -q[2], -q[3] }, { q[0], -q[3], q[2] }, { q[3], q[0], -q[1] }, { -q[2], q[1], q[0] } };
    for (int r = 0; r < 4; r++)
    {
      for (int j = 0; j < 4; j++)
        A[(6 + r) * 13 + 6 + j] = 0.5f * dqq[r][j];
      for (int j = 0; j < 3; j++)
        A[(6 + r) * 13 + 10 + j] = 0.5f * dqw[r][j];
    }
    const float tau[3] = { p.tau_roll, p.tau_pitch, p.tau_yaw };
    for (int i = 0; i < 3; i++)
    {
      A[(10 + i) * 13 + 10 + i] = -1.0f / tau[i];
      B[(10 + i) * 4 + i] = 1.0f / tau[i];
    }
    return true;
  }
};

}  // namespace plugins
}  // namespace mppib
