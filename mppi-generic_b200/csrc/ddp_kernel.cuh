/*
 * ddp_kernel.cuh — DDPFeedback::computeFeedback (feedback_controllers/DDP/ddp.cu:80-118) on the GPU: the iLQR solve of
 * DDP::run (ddp/ddp.h:56-168) with the tracking costs of ddp/ddp_tracking_costs.h, one CTA per solve, every iteration in
 * one launch. The numbered points below are the reference's behaviours this kernel keeps; each is named where it happens.
 *
 *  (1) f(x, u) is the state_der of one model step (ddp_model_wrapper.h:68-81); x' = x + f dt with the DDP's dt — no
 *      quaternion renormalisation, no angle wrapping (not the model's updateState).
 *  (2) initial rollout (ddp.h:62-71): control columns 0 .. T-3 are clamped to the limits, column T-2 is used unclamped.
 *  (3) df = I + dt [A | B] from the model's analytic computeGrad (plugins/dynamics.cuh).
 *  (4) c = (x - x*)' Q (x - x*) + (u - u*)' R (u - u*); gradient Q (x - x*), R (u - u*) and Hessian blkdiag(Q, R) as the
 *      reference writes them (no factor 2); terminal cost with Q_f around x*[T-1]. The backward pass scales the running
 *      cost's gradient and Hessian by dt.
 *  (5) backward pass (ddp.h:94-127), k = T-2 .. 0: Q_uu solved by LDLT, Vxx symmetrised after every step, K[T-1] = 0.
 *      A failed LDLT ends the solve with status k + 1 (the reference exit(-3)s) and leaves the destination gains untouched.
 *  (6) line search (ddp.h:129-162): alpha = 1, halving; candidate cost = sum_k c(x_new, u_new) dt over k < T-1 plus the
 *      terminal value of the PREVIOUS trajectory; the first iteration always accepts, later ones when the cost does not
 *      rise or alpha < 1e-4. The accepted control's last column is 0 (unew is zero-initialised there). No box-QP.
 *  (7) gains fb_gain_traj_[t] = K_t, C x S column-major = [t][s][c], the layout mppib_set_rmppi takes.
 *
 * Work split (blockDim = kThreads):
 *   Jacobians            one thread per time step, all T at once, into the workspace ([A | B] raw, row-major).
 *   backward pass        sequential over k; the products Vxx [Phi | B], [Phi | B]' (Vxx [Phi | B]) and the value update are
 *                        spread one output element per thread; the C x C LDLT runs on thread 0.
 *   rollouts, line search  sequential over k on warp 0. The Autorally network (6-32-32-4) is evaluated warp-cooperatively,
 *                        one hidden unit per lane, the lane's weight rows held in registers for the whole launch; the light
 *                        models run the same code on every lane of the warp (identical values, lane 0 stores).
 * The workspace is global memory (ddp_ws_layout): T = 500 with S = 13 holds 440 KB of Jacobians alone.
 */
#pragma once
#include <type_traits>

#include "plugins/dynamics.cuh"

namespace mppib
{
namespace ddp
{
constexpr int kThreads = 256;
constexpr int kMaxS = 20, kMaxC = 4;

// offsets (floats) of the workspace arrays for horizon T
struct WsLayout
{
  size_t x, u, xn, un, xt, ut, jac, K, kff, total;
};
__host__ __device__ inline WsLayout ws_layout(int T, int S, int C)
{
  WsLayout l;
  size_t o = 0;
  l.x = o;   o += (size_t)T * S;            // accepted state trajectory
  l.u = o;   o += (size_t)T * C;            // accepted control trajectory (in: the initial controls)
  l.xn = o;  o += (size_t)T * S;            // line-search candidate
  l.un = o;  o += (size_t)T * C;
  l.xt = o;  o += (size_t)T * S;            // tracking targets
  l.ut = o;  o += (size_t)T * C;
  l.jac = o; o += (size_t)T * S * (S + C);  // [A | B] per step, row-major
  l.K = o;   o += (size_t)T * S * C;        // gains [t][s][c]
  l.kff = o; o += (size_t)T * C;            // feed-forward terms
  l.total = o;
  return l;
}

template <class DYN>
struct DdpArgs
{
  static constexpr int S = DYN::STATE_DIM, C = DYN::CONTROL_DIM;
  typename DYN::Params dyn;
  typename DYN::Aux aux;
  float Q[S * S], Qf[S * S], R[C * C];  // row-major
  float x0[S];
  float u_lo[C], u_hi[C];  // control_rngs_ (ddp.cu:97-101)
  float dt;
  int T, iters;
  float* ws;     // ws_layout(T, S, C)
  float* gains;  // destination [T][S][C] written on success, or null (the gains stay in ws + K)
  int* status;   // 0, or k + 1 when the LDLT of Q_uu failed at step k
};

// The lane's share of the Autorally network: hidden unit `lane` of both layers and column `lane` of the output layer.
struct WarpNet
{
  float w1[6], b1, w2[32], b2, w3[4], b3[4];
  __device__ void load(const float* g, int lane)
  {
    for (int k = 0; k < 6; k++)
      w1[k] = __ldg(g + lane * 6 + k);
    b1 = __ldg(g + 192 + lane);
    for (int k = 0; k < 32; k++)
      w2[k] = __ldg(g + 224 + lane * 32 + k);
    b2 = __ldg(g + 1248 + lane);
    for (int i = 0; i < 4; i++)
    {
      w3[i] = __ldg(g + 1280 + i * 32 + lane);
      b3[i] = __ldg(g + 1408 + i);
    }
  }
  // out[4] on every lane; the whole warp calls it
  __device__ void forward(const float (&in)[6], float (&out)[4]) const
  {
    float z = 0.0f;
    for (int k = 0; k < 6; k++)
      z = fmaf(w1[k], in[k], z);
    const float h1 = tanhf(z + b1);
    z = 0.0f;
#pragma unroll
    for (int k = 0; k < 32; k++)
      z = fmaf(w2[k], __shfl_sync(0xffffffffu, h1, k), z);
    const float h2 = tanhf(z + b2);
#pragma unroll
    for (int i = 0; i < 4; i++)
    {
      float v = w3[i] * h2;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        v += __shfl_xor_sync(0xffffffffu, v, o);
      out[i] = v + b3[i];
    }
  }
};
struct NoNet
{
};

// (1): state_der of one model step, on every lane of warp 0
template <class DYN, class NET>
__device__ __forceinline__ void ddp_f(const DdpArgs<DYN>& a, const NET& net, const float* x, const float* u, float* xdot)
{
  if constexpr (DYN::DDP_WARP_NN)
  {
    DYN::computeKinematics(a.dyn, x, xdot);
    const float in[6] = { x[3], x[4], x[5], x[6], u[0], u[1] };
    float out[4];
    net.forward(in, out);
    for (int i = 0; i < 4; i++)
      xdot[3 + i] = out[i];
  }
  else
  {
    DYN::computeStateDeriv(a.dyn, nullptr, x, u, xdot);
  }
}

// (4): running tracking cost at step k
template <int S, int C>
__device__ __forceinline__ float track_cost(const float* Q, const float* R, const float* x, const float* xt, const float* u,
                                            const float* ut)
{
  float dx[S], du[C], c = 0.0f;
  for (int i = 0; i < S; i++)
    dx[i] = x[i] - xt[i];
  for (int i = 0; i < C; i++)
    du[i] = u[i] - ut[i];
  for (int i = 0; i < S; i++)
  {
    float r = 0.0f;
    for (int j = 0; j < S; j++)
      r = fmaf(Q[i * S + j], dx[j], r);
    c = fmaf(dx[i], r, c);
  }
  float cu = 0.0f;
  for (int i = 0; i < C; i++)
  {
    float r = 0.0f;
    for (int j = 0; j < C; j++)
      r = fmaf(R[i * C + j], du[j], r);
    cu = fmaf(du[i], r, cu);
  }
  return c + cu;
}

template <class DYN>
__global__ void __launch_bounds__(kThreads, 1) ddp_kernel(const __grid_constant__ DdpArgs<DYN> a)
{
  constexpr int S = DYN::STATE_DIM, C = DYN::CONTROL_DIM, SC = S + C;
  static_assert(S <= kMaxS && C <= kMaxC, "DDP is built for STATE_DIM <= 20, CONTROL_DIM <= 4");
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, T = a.T;
  const float dt = a.dt;
  const WsLayout L = ws_layout(T, S, C);
  float* x = a.ws + L.x;
  float* u = a.ws + L.u;
  float* xn = a.ws + L.xn;
  float* un = a.ws + L.un;
  const float* xt = a.ws + L.xt;
  const float* ut = a.ws + L.ut;
  float* jac = a.ws + L.jac;
  float* K = a.ws + L.K;
  float* kff = a.ws + L.kff;

  __shared__ float Vx[S], Vxx[S * S], M[S * SC], H[SC * SC], g[SC], W[S * S], Vxn[S], Ks[C * S], ks[C];
  __shared__ float V_T;
  __shared__ int failed;

  using Net = std::conditional_t<DYN::DDP_WARP_NN, WarpNet, NoNet>;
  Net net;
  if constexpr (DYN::DDP_WARP_NN)
  {
    if (warp == 0)
      net.load(a.aux.theta_d, lane);
  }
  if (tid == 0)
    failed = 0;

  // (2) initial rollout, warp 0
  if (warp == 0)
  {
    float xk[S], uk[C], xd[S];
    for (int i = 0; i < S; i++)
      xk[i] = a.x0[i];
    if (lane == 0)
      for (int i = 0; i < S; i++)
        x[i] = xk[i];
    for (int i = 1; i < T; i++)
    {
      for (int c = 0; c < C; c++)
        uk[c] = u[(i - 1) * C + c];
      if (i < T - 1)
      {
        for (int c = 0; c < C; c++)
          uk[c] = fmaxf(fminf(uk[c], a.u_hi[c]), a.u_lo[c]);
        __syncwarp();  // every lane has read column i - 1 before lane 0 overwrites it
        if (lane == 0)
          for (int c = 0; c < C; c++)
            u[(i - 1) * C + c] = uk[c];
      }
      ddp_f<DYN>(a, net, xk, uk, xd);
      for (int s = 0; s < S; s++)
        xk[s] = xk[s] + xd[s] * dt;
      if (lane == 0)
        for (int s = 0; s < S; s++)
          x[i * S + s] = xk[s];
    }
  }
  for (int i = tid; i < T * S * C; i += blockDim.x)
    K[i] = 0.0f;  // (5) K[T-1] stays zero
  __syncthreads();

  float prev_cost = 0.0f;  // warp 0
  for (int it = 0; it < a.iters; it++)
  {
    // (3) Jacobians, one thread per step
    for (int t = tid; t < T; t += blockDim.x)
    {
      float At[S * S], Bt[S * C];
      DYN::computeGrad(a.dyn, a.aux, x + t * S, u + t * C, At, Bt);
      float* J = jac + (size_t)t * S * SC;
      for (int i = 0; i < S; i++)
      {
        for (int j = 0; j < S; j++)
          J[i * SC + j] = At[i * S + j];
        for (int j = 0; j < C; j++)
          J[i * SC + S + j] = Bt[i * C + j];
      }
    }
    // boundary condition (ddp.h:88-92)
    if (tid == 0)
    {
      const float* xT = x + (T - 1) * S;
      const float* xf = xt + (T - 1) * S;
      float vt = 0.0f;
      for (int i = 0; i < S; i++)
      {
        float r = 0.0f;
        for (int j = 0; j < S; j++)
          r = fmaf(a.Qf[i * S + j], xT[j] - xf[j], r);
        Vx[i] = r;
        vt = fmaf(xT[i] - xf[i], r, vt);
      }
      V_T = vt;
    }
    for (int e = tid; e < S * S; e += blockDim.x)
    {
      const int i = e / S, j = e % S;
      Vxx[e] = 0.5f * (a.Qf[i * S + j] + a.Qf[j * S + i]);
    }
    __syncthreads();

    // (5) backward pass
    for (int k = T - 2; k >= 0; k--)
    {
      const float* Jk = jac + (size_t)k * S * SC;
      // df = I + dt [A | B]  (3)
      auto df = [&](int l, int j) { return (l == j ? 1.0f : 0.0f) + dt * Jk[l * SC + j]; };
      for (int e = tid; e < S * SC; e += blockDim.x)
      {
        const int i = e / SC, j = e % SC;
        float r = 0.0f;
        for (int l = 0; l < S; l++)
          r = fmaf(Vxx[i * S + l], df(l, j), r);
        M[e] = r;
      }
      __syncthreads();
      for (int e = tid; e < SC * SC + SC; e += blockDim.x)
      {
        if (e < SC * SC)
        {
          const int i = e / SC, j = e % SC;
          float r = 0.0f;
          for (int l = 0; l < S; l++)
            r = fmaf(df(l, i), M[l * SC + j], r);
          // (4) d2L = blkdiag(Q, R), scaled by dt
          if (i < S && j < S)
            r += a.Q[i * S + j] * dt;
          else if (i >= S && j >= S)
            r += a.R[(i - S) * C + (j - S)] * dt;
          H[e] = r;
        }
        else
        {
          const int i = e - SC * SC;
          float r = 0.0f;
          for (int l = 0; l < S; l++)
            r = fmaf(df(l, i), Vx[l], r);
          // (4) dL = [Q (x - x*); R (u - u*)], scaled by dt
          float d = 0.0f;
          if (i < S)
            for (int j = 0; j < S; j++)
              d = fmaf(a.Q[i * S + j], x[k * S + j] - xt[k * S + j], d);
          else
            for (int j = 0; j < C; j++)
              d = fmaf(a.R[(i - S) * C + j], u[k * C + j] - ut[k * C + j], d);
          g[i] = d * dt + r;
        }
      }
      __syncthreads();
      if (tid == 0)
      {
        // (5) LDLT of Q_uu (lower triangle, no pivoting: Q_uu = R dt + B' Vxx B is symmetric positive definite for the
        // default weights; Eigen's pivoted LDLT gives the same solution up to rounding). Fails on a zero or non-finite pivot.
        float Lm[C][C], D[C];
        bool ok = true;
        for (int j = 0; j < C && ok; j++)
        {
          float d = H[(S + j) * SC + S + j];
          for (int m = 0; m < j; m++)
            d -= Lm[j][m] * Lm[j][m] * D[m];
          D[j] = d;
          ok = isfinite(d) && fabsf(d) > 1.17549435e-38f;
          for (int i = j + 1; i < C && ok; i++)
          {
            float v = H[(S + i) * SC + S + j];
            for (int m = 0; m < j; m++)
              v -= Lm[i][m] * Lm[j][m] * D[m];
            Lm[i][j] = v / d;
          }
        }
        if (!ok)
          failed = k + 1;
        else
        {
          // columns 0 .. S-1: K = -Q_uu^-1 Q_ux; column S: k = -Q_uu^-1 Q_u
          for (int col = 0; col <= S; col++)
          {
            float y[C];
            for (int i = 0; i < C; i++)
            {
              float v = -(col < S ? H[(S + i) * SC + col] : g[S + i]);
              for (int m = 0; m < i; m++)
                v -= Lm[i][m] * y[m];
              y[i] = v;
            }
            for (int i = 0; i < C; i++)
              y[i] /= D[i];
            for (int i = C - 1; i >= 0; i--)
              for (int m = i + 1; m < C; m++)
                y[i] -= Lm[m][i] * y[m];
            for (int i = 0; i < C; i++)
            {
              if (col < S)
              {
                Ks[i * S + col] = y[i];
                K[((size_t)k * S + col) * C + i] = y[i];  // (7) [t][s][c]
              }
              else
              {
                ks[i] = y[i];
                kff[k * C + i] = y[i];
              }
            }
          }
        }
      }
      __syncthreads();
      if (failed)
        break;
      // value update: Vxx = Q_xx + Q_ux' K, Vx = Q_x + Q_ux' k
      for (int e = tid; e < S * S + S; e += blockDim.x)
      {
        if (e < S * S)
        {
          const int i = e / S, j = e % S;
          float r = H[i * SC + j];
          for (int c = 0; c < C; c++)
            r = fmaf(H[(S + c) * SC + i], Ks[c * S + j], r);
          W[e] = r;
        }
        else
        {
          const int i = e - S * S;
          float r = g[i];
          for (int c = 0; c < C; c++)
            r = fmaf(H[(S + c) * SC + i], ks[c], r);
          Vxn[i] = r;
        }
      }
      __syncthreads();
      for (int e = tid; e < S * S + S; e += blockDim.x)
      {
        if (e < S * S)
        {
          const int i = e / S, j = e % S;
          Vxx[e] = 0.5f * (W[i * S + j] + W[j * S + i]);  // (5) symmetrised
        }
        else
          Vx[e - S * S] = Vxn[e - S * S];
      }
      __syncthreads();
    }
    if (failed)
      break;

    // (6) line search, warp 0
    if (warp == 0)
    {
      float alpha = 1.0f;
      for (;;)
      {
        float xk[S], uk[C], xd[S], cost = 0.0f;
        for (int i = 0; i < S; i++)
          xk[i] = x[i];
        for (int k = 0; k < T - 1; k++)
        {
          for (int c = 0; c < C; c++)
          {
            float fb = 0.0f;
            for (int s = 0; s < S; s++)
              fb = fmaf(K[((size_t)k * S + s) * C + c], xk[s] - x[k * S + s], fb);
            uk[c] = fmaxf(fminf(u[k * C + c] + alpha * kff[k * C + c] + fb, a.u_hi[c]), a.u_lo[c]);
          }
          cost += track_cost<S, C>(a.Q, a.R, xk, xt + k * S, uk, ut + k * C) * dt;
          if (lane == 0)
          {
            for (int s = 0; s < S; s++)
              xn[k * S + s] = xk[s];
            for (int c = 0; c < C; c++)
              un[k * C + c] = uk[c];
          }
          ddp_f<DYN>(a, net, xk, uk, xd);
          for (int s = 0; s < S; s++)
            xk[s] = xk[s] + xd[s] * dt;
        }
        if (lane == 0)
        {
          for (int s = 0; s < S; s++)
            xn[(T - 1) * S + s] = xk[s];
          for (int c = 0; c < C; c++)
            un[(T - 1) * C + c] = 0.0f;
        }
        cost += V_T;
        if (it == 0 || alpha < 1e-4f || cost <= prev_cost)
        {
          prev_cost = cost;
          break;
        }
        alpha *= 0.5f;
      }
    }
    __syncthreads();
    for (int i = tid; i < T * S; i += blockDim.x)
      x[i] = xn[i];
    for (int i = tid; i < T * C; i += blockDim.x)
      u[i] = un[i];
    __syncthreads();
  }

  if (failed)
  {
    if (tid == 0)
      *a.status = failed;
    return;
  }
  if (tid == 0)
    *a.status = 0;
  if (a.gains)
    for (int i = tid; i < T * S * C; i += blockDim.x)
      a.gains[i] = K[i];
}

}  // namespace ddp
}  // namespace mppib
