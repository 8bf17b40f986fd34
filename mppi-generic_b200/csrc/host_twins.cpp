/*
 * host_twins.cpp — host-side (CPU) twins of the plugins and the controller tail, exported from libmppi_b200.so.
 *
 * In the reference every Dynamics / Cost class carries Eigen host methods next to its device methods
 * (include/mppi/dynamics/dynamics.cuh:250-300, include/mppi/cost_functions/cost.cuh:136-219) and the controller
 * finishes computeControl on the host: Savitzky-Golay smoothing, nominal state roll-forward and control clamping
 * (include/mppi/controllers/controller.cuh:557-663, controllers/MPPI/mppi_controller.cu:225-231). Those stay on the
 * host here as well (north_star: "host side stays header-only C++/Eigen"); they are compiled once into the library so
 * that the header-only C++ layer (include/mppi_b200/) and the ctypes mirror (mppi-generic_b200/host.py) share one
 * implementation. These functions are host conveniences of the plugin surface, NOT a fallback for the rollout path:
 * mppib_solve has no CPU route.
 */
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/mppi_b200.h"
#include "../../include/mppi_b200/host_twins.h"
#include "host_model.h"
#include "softmin.h"

using mppib::FnnT;
using mppib::HostModel;

namespace
{
inline float sign_ref(float v)  // utils/math_utils.h:744-747
{
  return v >= 0 ? 1.0f : -1.0f;
}

void enforce(const mppib_control_limits& lim, float* u, int C)  // dynamics.cuh:250-264
{
  for (int i = 0; i < C; i++)
  {
    if (fabsf(u[i]) < lim.deadband[i])
      u[i] = lim.zero_control[i];
    else
      u[i] += lim.deadband[i] * -sign_ref(u[i]);
    u[i] = fminf(fmaxf(lim.rng_lo[i], u[i]), lim.rng_hi[i]);
  }
}

// FNNHelper::forward host twin (utils/nn_helpers/fnn_helper.cu:354-382) for the fixed 6-32-32-4 net.
// The controller calls it T times per computeControl for the nominal trajectory (controller.cuh:643-663), which next to a
// GPU solve of a few hundred microseconds is a visible share of the call (112 us of ~480 us at T = 100 with the plain
// scalar loops + tanhf). So: weights transposed once per trajectory (FnnT, host_model.h: the inner loop runs over the OUT
// neurons and vectorises without reassociating any neuron's k-ascending sum), a branch-free tanh (below), and AVX2+FMA /
// baseline clones selected at load time.

// tanh(x) = 1 - 2 / (exp(2x) + 1), exp by Cody-Waite reduction + degree-7 polynomial: |abs error| < 2e-7 over the whole
// range (the same bound as the device kernels' tanh_fast; the reference calls tanhf, activation_functions.cuh:15-26).
// Straight-line code so the loops over neurons vectorise.
static inline float exp_host(float z)
{
  z = z > 30.0f ? 30.0f : (z < -30.0f ? -30.0f : z);
  const float nf = (z * 1.44269504088896341f + 12582912.0f) - 12582912.0f;  // round to nearest integer
  float r = z - nf * 0.693145751953125f;                                    // ln2 high part
  r = r - nf * 1.42860682030941723212e-6f;                                  // ln2 low part
  float p = 1.0f / 5040.0f;
  p = p * r + 1.0f / 720.0f;
  p = p * r + 1.0f / 120.0f;
  p = p * r + 1.0f / 24.0f;
  p = p * r + 1.0f / 6.0f;
  p = p * r + 0.5f;
  p = p * r + 1.0f;
  p = p * r + 1.0f;
  int bits = ((int)nf + 127) << 23;
  float scale;
  memcpy(&scale, &bits, sizeof(scale));
  return p * scale;
}
static inline float tanh_host(float x)
{
  return 1.0f - 2.0f / (exp_host(2.0f * x) + 1.0f);
}
static inline float sigmoid_host(float x)  // activation_functions.cuh:49-59 (host branch: 1 / (1 + expf(-x)))
{
  return 1.0f / (1.0f + exp_host(-x));
}

// GCC / clang generic vectors: the same source lowers to 8-lane AVX2 + FMA in the x86-64-v3 clone and to SSE2 pairs in the
// baseline clone. Written out by hand because the auto-vectoriser keeps tanh scalar (clamp branches, float -> int -> float
// round trip): 64 scalar tanh with a vdivss each were 2/3 of the forward pass.
typedef float v8f __attribute__((vector_size(32), aligned(4)));
typedef int v8i __attribute__((vector_size(32), aligned(4)));
static inline v8f splat8(float v)
{
  return v8f{ v, v, v, v, v, v, v, v };
}
static inline v8f load8(const float* p)
{
  v8f v;
  memcpy(&v, p, sizeof(v));
  return v;
}
static inline void store8(float* p, v8f v)
{
  memcpy(p, &v, sizeof(v));
}
// exp_host / tanh_host above, eight lanes at a time (same constants, same operation order)
static inline v8f exp8(v8f z)
{
  const v8f hi = splat8(30.0f), lo = splat8(-30.0f);
  z = z > hi ? hi : (z < lo ? lo : z);
  const v8f magic = splat8(12582912.0f);
  const v8f nf = (z * splat8(1.44269504088896341f) + magic) - magic;
  v8f r = z - nf * splat8(0.693145751953125f);
  r = r - nf * splat8(1.42860682030941723212e-6f);
  v8f p = splat8(1.0f / 5040.0f);
  p = p * r + splat8(1.0f / 720.0f);
  p = p * r + splat8(1.0f / 120.0f);
  p = p * r + splat8(1.0f / 24.0f);
  p = p * r + splat8(1.0f / 6.0f);
  p = p * r + splat8(0.5f);
  p = p * r + splat8(1.0f);
  p = p * r + splat8(1.0f);
  const v8i bits = (__builtin_convertvector(nf, v8i) + 127) << 23;
  v8f scale;
  memcpy(&scale, &bits, sizeof(scale));
  return p * scale;
}
static inline v8f tanh8(v8f x)
{
  return splat8(1.0f) - splat8(2.0f) / (exp8(splat8(2.0f) * x) + splat8(1.0f));
}

__attribute__((target_clones("arch=x86-64-v3", "default"))) void fnn_6_32_32_4(const FnnT& t, const float* in6,
                                                                              float* out4)
{
  // layers 1 and 2: the 32 outputs are four 8-lane vectors, k ascending per neuron (fnn_helper.cu:354-382), bias last
  v8f acc[4], a1[4], a2[4];
  for (int v = 0; v < 4; v++)
    acc[v] = splat8(0.0f);
  for (int k = 0; k < 6; k++)
  {
    const v8f xk = splat8(in6[k]);
    for (int v = 0; v < 4; v++)
      acc[v] += load8(t.WT1 + k * 32 + 8 * v) * xk;
  }
  for (int v = 0; v < 4; v++)
    a1[v] = tanh8(acc[v] + load8(t.b1 + 8 * v));
  float a1s[32];
  for (int v = 0; v < 4; v++)
    store8(a1s + 8 * v, a1[v]);
  // layer 2: even and odd k accumulate separately (two FMA chains of 16 instead of one of 32 on the critical path) and
  // are added at the end; like layer 3 below a reassociation of a few ulp
  v8f acc_odd[4];
  for (int v = 0; v < 4; v++)
    acc[v] = acc_odd[v] = splat8(0.0f);
  for (int k = 0; k < 32; k += 2)
  {
    const v8f xa = splat8(a1s[k]), xb = splat8(a1s[k + 1]);
    for (int v = 0; v < 4; v++)
    {
      acc[v] += load8(t.WT2 + k * 32 + 8 * v) * xa;
      acc_odd[v] += load8(t.WT2 + (k + 1) * 32 + 8 * v) * xb;
    }
  }
  for (int v = 0; v < 4; v++)
    a2[v] = tanh8((acc[v] + acc_odd[v]) + load8(t.b2 + 8 * v));
  // layer 3: four 32-term dot products, eight interleaved partial sums each (one 8-lane FMA chain of length 4) — a
  // reassociation of the kind Eigen's packet products in the reference's host code make as well
  for (int j = 0; j < 4; j++)
  {
    v8f part = load8(t.W3 + j * 32) * a2[0];
    for (int v = 1; v < 4; v++)
      part += load8(t.W3 + j * 32 + 8 * v) * a2[v];
    out4[j] = (((part[0] + part[4]) + (part[1] + part[5])) + ((part[2] + part[6]) + (part[3] + part[7]))) + t.b3[j];
  }
}

// ---- RacerDubinsElevationLSTMSteering host twin ------------------------------------------------------------------
// State / output indices: racer_dubins_elevation.cuh:18-39, racer_dubins.cuh:35-76
enum
{
  R_VEL_X = 0, R_YAW, R_POS_X, R_POS_Y, R_STEER_ANGLE, R_BRAKE_STATE, R_ROLL, R_PITCH, R_STEER_ANGLE_RATE, R_UNC0
};
inline float normalize_angle(float a)  // utils/angle_utils.cuh
{
  const float two_pi = 6.283185307179586f, pi = 3.14159265358979f;
  float r = fmodf(a + pi, two_pi);
  return r <= 0.0f ? r + pi : r - pi;
}

// LSTMHelper::forward (host), utils/nn_helpers/lstm_helper.cu:267-339: gates from W_*m h + W_*i x + b, FNN head on [h; x]
// In-place activations of n values, eight lanes at a time through exp8 (the scalar exp_host per value — ~40 of them per
// step at H = 4, L1 = 20 — was most of the roll-forward): kind 0 = sigmoid 1 / (1 + exp(-x)), kind 1 = tanh.
static inline void activate_n(float* v, int n, int kind)
{
  for (int i = 0; i < n; i += 8)
  {
    float buf[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    const int m = n - i < 8 ? n - i : 8;
    memcpy(buf, v + i, sizeof(float) * m);
    const v8f x = load8(buf);
    const v8f r = kind ? tanh8(x) : splat8(1.0f) / (splat8(1.0f) + exp8(-x));
    store8(buf, r);
    memcpy(v + i, buf, sizeof(float) * m);
  }
}

__attribute__((target_clones("arch=x86-64-v3", "default"))) float lstm_head_forward(const mppib_host_lstm* net,
                                                                                   const float* in4)
{
  const int H = net->hidden_dim, I = MPPIB_RACER_LSTM_INPUT_DIM, L1 = net->head_hidden;
  const int HH = H * H, IH = H * I;
  const float* w = net->theta;
  const float* bias = w + 4 * HH + 4 * IH;
  float g[4][64];  // gate pre-activations [input, forget, output, cell-update][H], H <= 64 (engine limit)
  for (int k = 0; k < 4; k++)
    for (int i = 0; i < H; i++)
    {
      const float* Wm = w + k * HH + i * H;
      const float* Wi = w + 4 * HH + k * IH + i * I;
      float hm = 0.0f, im = 0.0f;
      for (int j = 0; j < H; j++)
        hm += Wm[j] * net->hidden[j];
      for (int j = 0; j < I; j++)
        im += Wi[j] * in4[j];
      g[k][i] = (hm + im) + bias[k * H + i];
    }
  // exp-based activations without libm calls (exp8 above; |abs error| < 2e-7 against expf / tanhf)
  activate_n(g[0], H, 0);
  activate_n(g[1], H, 0);
  activate_n(g[2], H, 0);
  activate_n(g[3], H, 1);
  float hn[64], cn[64];
  for (int i = 0; i < H; i++)
    cn[i] = hn[i] = g[0][i] * g[3][i] + g[1][i] * net->cell[i];
  activate_n(hn, H, 1);
  for (int i = 0; i < H; i++)
    hn[i] = g[2][i] * hn[i];
  memcpy(net->hidden, hn, sizeof(float) * H);
  memcpy(net->cell, cn, sizeof(float) * H);
  const float* hd = w + 4 * HH + 4 * IH + 6 * H;  // head {H+I, L1, 1}: W1 | b1 | W2 | b2 (fnn_helper.cu:176-183)
  const int IN = H + I;
  float a1[64];
  for (int k = 0; k < L1; k++)
  {
    float a = 0.0f;
    for (int j = 0; j < H; j++)
      a += hd[k * IN + j] * hn[j];
    for (int j = 0; j < I; j++)
      a += hd[k * IN + H + j] * in4[j];
    a1[k] = a + hd[L1 * IN + k];
  }
  activate_n(a1, L1, 1);
  float out = 0.0f;
  for (int k = 0; k < L1; k++)
    out += hd[L1 * IN + L1 + k] * a1[k];
  return out + hd[L1 * IN + 2 * L1];
}

// TextureHelper::worldPoseToTexCoord (texture_helper.cu:94-134) + TwoDTextureHelper::queryTextureCPU
// (two_d_texture_helper.cu:151-243) for the TextureParams defaults: clamp addressing, bilinear filter
float elevation_at_world_pose(const mppib_elevation_map_header* h, float wx, float wy, float wz)
{
  const float* data = reinterpret_cast<const float*>(h + 1);
  const float dx = wx - h->origin[0], dy = wy - h->origin[1], dz = wz - h->origin[2];
  const float mx = h->rotations[0] * dx + h->rotations[1] * dy + h->rotations[2] * dz;
  const float my = h->rotations[3] * dx + h->rotations[4] * dy + h->rotations[5] * dz;
  float qx = ((mx / h->resolution[0]) / (float)h->width) * (float)h->width - 0.5f;
  float qy = ((my / h->resolution[1]) / (float)h->height) * (float)h->height - 0.5f;
  if (qx > (float)(h->width - 1))
    qx = (float)(h->width - 1);
  else if (qx <= 0.0f)
    qx = 0.0f;
  if (qy > (float)(h->height - 1))
    qy = (float)(h->height - 1);
  else if (qy <= 0.0f)
    qy = 0.0f;
  if (std::isnan(qx) || std::isnan(qy))
    return NAN;
  const int x0 = std::min((int)std::floor(qx), h->width - 2), y0 = std::min((int)std::floor(qy), h->height - 2);
  const int w = h->width;
  const float q11 = data[(size_t)y0 * w + x0], q12 = data[(size_t)y0 * w + x0 + 1];
  const float q21 = data[(size_t)(y0 + 1) * w + x0], q22 = data[(size_t)(y0 + 1) * w + x0 + 1];
  const float lo = q11 * ((float)(x0 + 1) - qx) + q12 * (qx - (float)x0);
  const float hi = q21 * ((float)(x0 + 1) - qx) + q22 * (qx - (float)x0);
  return lo * ((float)(y0 + 1) - qy) + hi * (qy - (float)y0);
}
// RACER::computeStaticSettling, racer_dubins.cu:359-434 (host branch of math::Euler2DCM_NWU: sincosf without normalisation)
float static_settling(const mppib_elevation_map_header* map, float yaw, float x, float y, float& roll, float& pitch)
{
  if (!map || !map->use)
  {
    roll = 0.0f;
    pitch = 0.0f;
    return 0.0f;
  }
  float sr, cr, sp, cp, sy, cy;
  sincosf(roll, &sr, &cr);
  sincosf(pitch, &sp, &cp);
  sincosf(yaw, &sy, &cy);
  const float M00 = cp * cy, M01 = sr * sp * cy - cr * sy, M10 = cp * sy, M11 = sr * sp * sy + cr * cy, M20 = -sp,
              M21 = sr * cp;
  float hgt[4];
  for (int k = 0; k < 4; k++)
  {  // front left, front right, rear left, rear right (:364-367)
    const float ox = (k < 2) ? 2.981f : 0.0f, oy = (k & 1) ? -0.737f : 0.737f;
    hgt[k] = elevation_at_world_pose(map, M00 * ox + M01 * oy + x, M10 * ox + M11 * oy + y, M20 * ox + M21 * oy + 0.0f);
  }
  const float fl = hgt[0], fr = hgt[1], rl = hgt[2], rr = hgt[3];
  const float front_diff = fmaxf(fminf(fl - fr, 0.736f * 2.0f), -0.736f * 2.0f);
  const float rear_diff = fmaxf(fminf(rl - rr, 0.736f * 2.0f), -0.736f * 2.0f);
  roll = (asinf(front_diff / (0.737f * 2.0f)) + asinf(rear_diff / (0.737f * 2.0f))) / 2.0f;
  const float left_diff = fmaxf(fminf(rl - fl, 2.98f), -2.98f);
  const float right_diff = fmaxf(fminf(rr - fr, 2.98f), -2.98f);
  pitch = (asinf(left_diff / 2.981f) + asinf(right_diff / 2.981f)) / 2.0f;
  float height = (rl + rr) / 2.0f;
  if (!std::isfinite(roll) || fabsf(roll) > (float)M_PI)
    roll = 2.0f * (float)M_PI;
  if (!std::isfinite(pitch) || fabsf(pitch) > (float)M_PI)
    pitch = 2.0f * (float)M_PI;
  if (!std::isfinite(height))
    height = 0.0f;
  return height;
}

// The host methods both RACER elevation models share (racer_dubins.cu:306-319 brake delay, racer_dubins_elevation.cu:32-67
// parametric acceleration, :662-741 uncertainty propagation, RACER::computeStaticSettling and setOutputs); each model's
// step adds its own steering and updateState between them.
struct RacerKin
{
  int index;
  float vx, brake_state, delta, tan_delta, sy, cy;
};
inline RacerKin racer_parametric_deriv(const mppib_racer_lstm_dyn_params& p, const float* x, const float* u, float* xd)
{
  const float vx = x[R_VEL_X];
  const int index = (fabsf(vx) > 0.2f && fabsf(vx) <= 3.0f) + (fabsf(vx) > 3.0f) * 2;
  const bool enable_brake = u[0] < 0.0f;
  const float brake_error = (enable_brake * -u[0] - x[R_BRAKE_STATE]);  // racer_dubins.cu:306-319
  xd[R_BRAKE_STATE] = fminf(fmaxf((brake_error > 0) * brake_error * p.brake_delay_constant +
                                      (brake_error < 0) * brake_error * p.brake_delay_constant_neg,
                                  -p.max_brake_rate_neg),
                            p.max_brake_rate_pos);
  const float brake_state = fminf(fmaxf(x[R_BRAKE_STATE], 0.0f), 0.25f);  // racer_dubins_elevation.cu:32-67
  float throttle = p.c_t[index] * u[0];
  float brake = p.c_b[index] * brake_state * (vx >= 0.0f ? -1.0f : 1.0f);
  if (fabsf(vx) <= 0.2f)
  {
    throttle = p.c_t[index] * fmaxf(u[0] - p.low_min_throttle, 0.0f);
    brake = p.c_b[index] * brake_state * -vx;
  }
  xd[R_VEL_X] = (!enable_brake) * throttle * p.gear_sign + brake - p.c_v[index] * vx + p.c_0;
  xd[R_VEL_X] = fminf(fmaxf(xd[R_VEL_X], -p.clamp_ax), p.clamp_ax);
  if (fabsf(x[R_PITCH]) < 1.57079632679489661923f)
    xd[R_VEL_X] -= p.gravity * sinf(x[R_PITCH]);
  const float delta = x[R_STEER_ANGLE] / p.steer_angle_scale;
  const float tan_delta = tanf(delta);
  xd[R_YAW] = (vx / p.wheel_base) * tan_delta;
  const float sy = sinf(x[R_YAW]), cy = cosf(x[R_YAW]);
  xd[R_POS_X] = vx * cy;
  xd[R_POS_Y] = vx * sy;
  return RacerKin{ index, vx, brake_state, delta, tan_delta, sy, cy };
}

// unc0: where the ten uncertainty entries start (R_UNC0 in the 19-state models, 13 in the suspension model)
inline void racer_propagate_uncertainty(const mppib_racer_lstm_dyn_params& p, const RacerKin& k, const float* x,
                                        const float* xd, float* xn, float dt, int unc0 = R_UNC0)
{
  const int index = k.index;
  const float vx = k.vx, brake_state = k.brake_state, delta = k.delta, tan_delta = k.tan_delta, sy = k.sy, cy = k.cy;
  {  // computeUncertaintyPropagation, racer_dubins_elevation.cu:662-741; matrices column-major 4x4 over
     // (VEL_X, YAW, POS_X, POS_Y); state order of the 10 covariance entries: racer_dubins_elevation.cuh:29-38
    float A[4][4] = {}, Sg[4][4], Tm[4][4], Q[4][4] = {};  // [row][col]
    const float c2 = cosf(delta) * cosf(delta);
    A[0][0] = -p.c_v[index] - p.K_vel_x - (index == 0 ? 1.0f : 0.0f) * p.c_b[0] * brake_state;
    A[0][2] = -p.K_x * cy;
    A[0][3] = -p.K_x * sy;
    A[1][0] = tan_delta / p.wheel_base;
    A[1][1] = -fabsf(vx) * p.K_yaw / (p.wheel_base * c2);
    A[1][2] = vx * p.K_y * sy / (p.wheel_base * c2);
    A[1][3] = -vx * p.K_y * cy / (p.wheel_base * c2);
    A[2][0] = cy;
    A[2][1] = -sy * vx;
    A[3][0] = sy;
    A[3][1] = cy * vx;
    const float* s = x + unc0;  // POS_X, POS_Y, YAW, VEL_X, POS_X_Y, POS_X_YAW, POS_X_VEL_X, POS_Y_YAW, POS_Y_VEL_X, YAW_VEL_X
    Sg[0][0] = s[3], Sg[1][1] = s[2], Sg[2][2] = s[0], Sg[3][3] = s[1];
    Sg[1][0] = Sg[0][1] = s[9];
    Sg[2][0] = Sg[0][2] = s[6];
    Sg[3][0] = Sg[0][3] = s[8];
    Sg[2][1] = Sg[1][2] = s[5];
    Sg[3][1] = Sg[1][3] = s[7];
    Sg[3][2] = Sg[2][3] = s[4];
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++)
        A[r][c] = (r == c) + A[r][c] * dt;
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++)
      {
        float acc = 0.0f;
        for (int k = 0; k < 4; k++)
          acc += A[r][k] * Sg[k][c];
        Tm[r][c] = acc;
      }
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++)
      {
        float acc = 0.0f;
        for (int k = 0; k < 4; k++)
          acc += Tm[r][k] * A[c][k];
        Sg[r][c] = acc;
      }
    const float abs_vx = fabsf(vx);
    const float side_force = abs_vx * abs_vx * tan_delta / p.wheel_base + p.gravity * sinf(x[R_ROLL]);
    const float Q_11 = fabsf(p.Q_y_f * fabsf(side_force) * fmaxf(abs_vx - 2, 0.0f));
    Q[0][0] = p.Q_x_acc * fabsf(xd[R_VEL_X]) + p.Q_x_v[index] * abs_vx;
    Q[1][1] = abs_vx * (p.Q_omega_steering * fabsf(delta) + p.Q_omega_v);
    Q[2][2] = Q_11 * sy * sy;
    Q[2][3] = Q[3][2] = -Q_11 * sy * cy;
    Q[3][3] = Q_11 * cy * cy;
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++)
        Sg[r][c] += Q[r][c] * dt;
    float* o = xn + unc0;
    o[0] = Sg[2][2], o[1] = Sg[3][3], o[2] = Sg[1][1], o[3] = Sg[0][0], o[4] = Sg[3][2], o[5] = Sg[2][1], o[6] = Sg[2][0],
    o[7] = Sg[3][1], o[8] = Sg[3][0], o[9] = Sg[1][0];
  }
}

// setOutputs, racer_dubins_elevation.cu:69-227 (output order racer_dubins.cuh:35-76), with the state layout's steering
// rate and uncertainty indices; the wheel forces are NaN
inline void racer_set_outputs(const float* xd, const float* xn, float* y, float height, int steer_rate, int unc0)
{
  y[0] = xn[R_VEL_X], y[1] = 0.0f, y[2] = xn[R_POS_X], y[3] = xn[R_POS_Y], y[4] = height, y[5] = xn[R_YAW];
  y[6] = xn[R_ROLL], y[7] = xn[R_PITCH], y[8] = xn[R_STEER_ANGLE], y[9] = xn[steer_rate];
  y[10] = y[11] = y[12] = NAN;
  y[13] = xd[R_VEL_X], y[14] = 0.0f, y[15] = xd[R_YAW], y[16] = fabsf(xn[R_VEL_X]);
  for (int i = 0; i < 10; i++)
    y[17 + i] = xn[unc0 + i];
  y[27] = 0.0f;
}

inline void racer_settle_and_output(const mppib_elevation_map_header* map, const float* x, const float* xd, float* xn,
                                    float* y)
{
  // computeStaticSettling (lstm_steering.cu:105-112): current roll / pitch, next yaw and position; flat without a map
  float roll = x[R_ROLL], pitch = x[R_PITCH];
  const float height = static_settling(map, xn[R_YAW], xn[R_POS_X], xn[R_POS_Y], roll, pitch);
  xn[R_ROLL] = roll;
  xn[R_PITCH] = pitch;
  racer_set_outputs(xd, xn, y, height, R_STEER_ANGLE_RATE, R_UNC0);
}

// computeLSTMSteering, lstm_steering.cu:66-88: xd's steering rate (at index steer_rate) and STEER_ANGLE
inline void racer_lstm_steering(const mppib_racer_lstm_dyn_params& p, const mppib_host_lstm* net, const float* x,
                                const float* u, float* xd, int steer_rate)
{
  const float parametric_accel = (u[1] * p.steer_command_angle_scale - x[R_STEER_ANGLE]) * p.steering_constant;
  xd[steer_rate] = fmaxf(fminf((parametric_accel - x[steer_rate]) * p.steer_accel_constant -
                                   x[steer_rate] * p.steer_accel_drag_constant,
                               p.max_steer_rate),
                         -p.max_steer_rate);
  const float in4[4] = { x[R_STEER_ANGLE] * 0.2f, x[steer_rate] * 0.2f, u[1], xd[steer_rate] * 0.2f };
  xd[steer_rate] += lstm_head_forward(net, in4) * 5.0f;
  xd[R_STEER_ANGLE] = x[steer_rate];
}

// racer_dubins_elevation_lstm_steering.cu:90-118 (host step) and the host methods it calls
void racer_step(const mppib_racer_lstm_dyn_params& p, const mppib_host_lstm* net, const mppib_elevation_map_header* map,
                const float* x, const float* u, float dt, float* xn, float* xd, float* y)
{
  const RacerKin k = racer_parametric_deriv(p, x, u, xd);
  racer_lstm_steering(p, net, x, u, xd, R_STEER_ANGLE_RATE);
  for (int i = 0; i < 6; i++)  // updateState, lstm_steering.cu:267-285
    xn[i] = x[i] + xd[i] * dt;
  xn[R_YAW] = normalize_angle(xn[R_YAW]);
  xn[R_STEER_ANGLE] = fmaxf(fminf(xn[R_STEER_ANGLE], p.max_steer_angle), -p.max_steer_angle);
  xn[R_STEER_ANGLE_RATE] = x[R_STEER_ANGLE_RATE] + xd[R_STEER_ANGLE_RATE] * dt;
  xn[R_BRAKE_STATE] = fminf(fmaxf(xn[R_BRAKE_STATE], 0.0f), -p.lim.rng_lo[0]);
  racer_propagate_uncertainty(p, k, x, xd, xn, dt);
  racer_settle_and_output(map, x, xd, xn, y);
}

// RacerDubinsElevationImpl::step (host), racer_dubins_elevation.cu:229-255: computeParametricSteerDeriv (host,
// racer_dubins.cu:321-330) and RacerDubinsImpl::updateState (host, :43-59), whose brake clamp is
// [0, -control_rngs_[0].x] where the device body's is [0, 1]
void racer_dubins_step(const mppib_racer_dubins_elevation_dyn_params& p, const mppib_elevation_map_header* map,
                       const float* x, const float* u, float dt, float* xn, float* xd, float* y)
{
  const RacerKin k = racer_parametric_deriv(p, x, u, xd);
  xd[R_STEER_ANGLE] = fmaxf(fminf((u[1] * p.steer_command_angle_scale - x[R_STEER_ANGLE]) * p.steering_constant,
                                  p.max_steer_rate),
                            -p.max_steer_rate);
  for (int i = 0; i < 6; i++)
    xn[i] = x[i] + xd[i] * dt;
  xn[R_YAW] = normalize_angle(xn[R_YAW]);
  xn[R_STEER_ANGLE] = fmaxf(fminf(xn[R_STEER_ANGLE], p.max_steer_angle), -p.max_steer_angle);
  xn[R_STEER_ANGLE_RATE] = xd[R_STEER_ANGLE];
  xn[R_BRAKE_STATE] = fminf(fmaxf(xn[R_BRAKE_STATE], 0.0f), -p.lim.rng_lo[0]);
  racer_propagate_uncertainty(p, k, x, xd, xn, dt);
  racer_settle_and_output(map, x, xd, xn, y);
}
// TwoDTextureHelper<float4>::queryTextureAtWorldPose on the host: elevation_at_world_pose's formula channel by channel
// (two_d_texture_helper.cu:151-243 is templated on the value type)
void normals_at_world_pose(const mppib_elevation_map_header* h, float wx, float wy, float wz, float* out4)
{
  const float* data = reinterpret_cast<const float*>(h + 1);
  const float dx = wx - h->origin[0], dy = wy - h->origin[1], dz = wz - h->origin[2];
  const float mx = h->rotations[0] * dx + h->rotations[1] * dy + h->rotations[2] * dz;
  const float my = h->rotations[3] * dx + h->rotations[4] * dy + h->rotations[5] * dz;
  float qx = ((mx / h->resolution[0]) / (float)h->width) * (float)h->width - 0.5f;
  float qy = ((my / h->resolution[1]) / (float)h->height) * (float)h->height - 0.5f;
  if (qx > (float)(h->width - 1))
    qx = (float)(h->width - 1);
  else if (qx <= 0.0f)
    qx = 0.0f;
  if (qy > (float)(h->height - 1))
    qy = (float)(h->height - 1);
  else if (qy <= 0.0f)
    qy = 0.0f;
  if (std::isnan(qx) || std::isnan(qy))
  {
    for (int c = 0; c < 4; c++)
      out4[c] = NAN;
    return;
  }
  const int x0 = std::min((int)std::floor(qx), h->width - 2), y0 = std::min((int)std::floor(qy), h->height - 2);
  const size_t w = h->width;
  const float* q11 = data + 4 * ((size_t)y0 * w + x0);
  const float *q12 = q11 + 4, *q21 = q11 + 4 * w, *q22 = q21 + 4;
  for (int c = 0; c < 4; c++)
  {
    const float lo = q11[c] * ((float)(x0 + 1) - qx) + q12[c] * (qx - (float)x0);
    const float hi = q21[c] * ((float)(x0 + 1) - qx) + q22[c] * (qx - (float)x0);
    out4[c] = lo * ((float)(y0 + 1) - qy) + hi * (qy - (float)y0);
  }
}

// RacerDubinsElevationSuspension host step (racer_dubins_elevation_suspension_lstm.cu:168-197): parametric derivatives,
// LSTM steering, computeSimpleSuspensionStep (host, :59-166), updateState (host, :420-435: brake clamped to
// [0, -control_rngs_[0].x]), uncertainty propagation and setOutputs (:437-525). State layout :25-52.
enum
{
  RS_CG_POS_Z = 8, RS_CG_VEL_I_Z, RS_ROLL_RATE, RS_PITCH_RATE, RS_STEER_ANGLE_RATE, RS_UNC0, RS_FILLER_1 = 23
};
void racer_suspension_step(const mppib_racer_suspension_dyn_params& sp, const mppib_host_lstm* net,
                           const mppib_elevation_map_header* elev, const mppib_elevation_map_header* normals, const float* x,
                           const float* u, float dt, float* xn, float* xd, float* y)
{
  const mppib_racer_lstm_dyn_params& p = sp.base;
  const RacerKin k = racer_parametric_deriv(p, x, u, xd);
  racer_lstm_steering(p, net, x, u, xd, RS_STEER_ANGLE_RATE);
  float up = -FLT_MAX, fwd = -FLT_MAX, side = -FLT_MAX;
  {  // computeSimpleSuspensionStep (host): Euler2DCM_NWU's host branch, sincosf of the raw angles
    const float roll = x[R_ROLL], pitch = x[R_PITCH], yaw = x[R_YAW];
    float sr, cr, spi, cpi, sy, cy;
    sincosf(roll, &sr, &cr);
    sincosf(pitch, &spi, &cpi);
    sincosf(yaw, &sy, &cy);
    const float M00 = cpi * cy, M01 = sr * spi * cy - cr * sy, M10 = cpi * sy, M11 = sr * spi * sy + cr * cy, M20 = -spi,
                M21 = sr * cpi;
    xd[R_ROLL] = x[RS_ROLL_RATE];
    xd[R_PITCH] = x[RS_PITCH_RATE];
    xd[RS_CG_POS_Z] = x[RS_CG_VEL_I_Z];
    xd[RS_CG_VEL_I_Z] = xd[RS_ROLL_RATE] = xd[RS_PITCH_RATE] = 0.0f;
    float wheel_height = 0.0f, n[4] = { 0.0f, 0.0f, 1.0f, 0.0f };
    for (int i = 0; i < 4; i++)
    {  // FL, FR, BL, BR (:74-77)
      const float bx = (i < 2) ? 2.981f : 0.0f, by = (i == 0 || i == 3) ? 0.737f : -0.737f;
      const float cgx = bx - sp.c_g[0], cgy = by - sp.c_g[1];
      const float wx = M00 * bx + M01 * by + x[R_POS_X], wy = M10 * bx + M11 * by + x[R_POS_Y],
                  wz = M20 * bx + M21 * by + 0.0f;
      if (elev && elev->use)
      {
        wheel_height = elevation_at_world_pose(elev, wx, wy, wz);
        if (!std::isfinite(wheel_height))
          wheel_height = x[RS_CG_POS_Z] - sp.wheel_radius;
      }
      if (normals && normals->use)
      {
        normals_at_world_pose(normals, wx, wy, wz, n);
        if (!std::isfinite(n[0]) || !std::isfinite(n[1]) || !std::isfinite(n[2]))
          n[0] = 0.0f, n[1] = 0.0f, n[2] = 1.0f, n[3] = 0.0f;
      }
      // front wheels: yaw + S_INDEX(STEER_ANGLE) / -9.1, the constant index 4 (:123-126)
      const float wheel_yaw = (i < 2) ? yaw + 4 / -9.1f : yaw;
      float swy, cwy;
      sincosf(wheel_yaw, &swy, &cwy);
      const float wheel_pos_z = x[RS_CG_POS_Z] + roll * cgy - pitch * cgx - sp.wheel_radius;
      const float wheel_vel_z = x[RS_CG_VEL_I_Z] + x[RS_ROLL_RATE] * cgy - x[RS_PITCH_RATE] * cgx;
      const float h_dot = -(x[R_VEL_X] * cwy * n[0] + x[R_VEL_X] * swy * n[1]);
      const float F = -sp.spring_k * (wheel_pos_z - wheel_height) - sp.drag_c * (wheel_vel_z - h_dot);
      up = fmaxf(up, F);
      fwd = fmaxf(fwd, fabsf(F / n[2] * (n[0] * cwy + n[1] * swy + n[2] * (-pitch))));
      side = fmaxf(side, fabsf(F / n[2] * (-n[0] * swy + n[1] * cwy + n[2] * roll)));
      xd[RS_CG_VEL_I_Z] += F / sp.mass;
      xd[RS_ROLL_RATE] += F * cgy / sp.I_xx;
      xd[RS_PITCH_RATE] += -F * cgx / sp.I_yy;
    }
  }
  for (int i = 0; i < RS_STEER_ANGLE_RATE; i++)
    xn[i] = x[i] + xd[i] * dt;
  xn[R_YAW] = normalize_angle(xn[R_YAW]);
  xn[R_STEER_ANGLE] = fmaxf(fminf(xn[R_STEER_ANGLE], p.max_steer_angle), -p.max_steer_angle);
  xn[RS_STEER_ANGLE_RATE] = x[RS_STEER_ANGLE_RATE] + xd[RS_STEER_ANGLE_RATE] * dt;
  xn[R_BRAKE_STATE] = fminf(fmaxf(xn[R_BRAKE_STATE], 0.0f), -p.lim.rng_lo[0]);
  xn[RS_FILLER_1] = x[RS_FILLER_1];
  racer_propagate_uncertainty(p, k, x, xd, xn, dt, RS_UNC0);
  racer_set_outputs(xd, xn, y, xn[RS_CG_POS_Z] - xn[R_PITCH] * (-sp.c_g[0]), RS_STEER_ANGLE_RATE, RS_UNC0);
  y[10] = up, y[11] = fwd, y[12] = side;
}
// ---- RacerSuspension host twin (dynamics/racer_suspension/racer_suspension.cu) ---------------------------------------
// computeStateDeriv (:93-298) on the plane z = 0 with normal (0, 0, 1) (the map query is commented out, :128-135), in
// float as the host body evaluates it, with the 3x3 omegaJacobian when jac != NULL (row-major [3][3]). Kept as written:
// `f_r_B_i_Jac = R_C_i_to_B = f_r_C_i_Jac` (:215) is an assignment, so tau_jac takes the contact-frame Jacobian as if it
// were the body-frame one; 1.0 / J is a double quotient rounded to float. The body-z velocity goes to BASELINK_VEL_B_Z,
// not into BASELINK_VEL_B_X (DESIGN §8); ACCEL_X / ACCEL_Y / OMEGA_Z are 0.
static void rigid_suspension_deriv(const mppib_racer_rigid_suspension_dyn_params& p, const float* x, const float* u,
                                   float* xd, float* y, float* jac)
{
  typedef float M3[3][3];
  const float qw = x[3], qx = x[4], qy = x[5], qz = x[6];
  const float tx = 2.0f * qx, ty = 2.0f * qy, tz = 2.0f * qz;  // Eigen's Quaternion::toRotationMatrix
  const float twx = tx * qw, twy = ty * qw, twz = tz * qw, txx = tx * qx, txy = ty * qx, txz = tz * qx;
  const float tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  const M3 R = { { 1.0f - (tyy + tzz), txy - twz, txz + twy },
                 { txy + twz, 1.0f - (txx + tzz), tyz - twx },
                 { txz - twy, tyz + twx, 1.0f - (txx + tyy) } };
  const float* pI = x;
  const float* v = x + 7;
  const float* w = x + 10;
  auto mul = [&](const float* a, float* out) {  // R a
    for (int r = 0; r < 3; r++)
      out[r] = R[r][0] * a[0] + R[r][1] * a[1] + R[r][2] * a[2];
  };
  auto mulT = [&](const float* a, float* out) {  // R^T a
    for (int r = 0; r < 3; r++)
      out[r] = R[0][r] * a[0] + R[1][r] * a[1] + R[2][r] * a[2];
  };
  auto cross = [](const float* a, const float* b, float* out) {
    out[0] = a[1] * b[2] - a[2] * b[1];
    out[1] = a[2] * b[0] - a[0] * b[2];
    out[2] = a[0] * b[1] - a[1] * b[0];
  };
  const float tan_delta = tanf(x[13]);
  float vb[3];
  mulT(v, vb);
  const float throttle = std::max(0.0f, u[0]), brake = std::max(0.0f, -u[0]);
  const float acc = p.c_t * throttle - copysignf(p.c_b * brake, vb[0]) - p.c_v * vb[0] + p.c_0;
  const float propulsion_force = p.mass * acc;

  float f_B[3] = { 0, 0, 0 }, tau_B[3] = { 0, 0, 0 };
  M3 tau_jac = {};
  for (int i = 0; i < 4; i++)
  {
    float pb[3], Rpb[3], pw[3], wxp[3], Rwxp[3], pdot[3];
    for (int r = 0; r < 3; r++)
      pb[r] = p.wheel_pos_wrt_base_link[i][r] - p.cg_pos_wrt_base_link[r];
    mul(pb, Rpb);
    cross(w, pb, wxp);
    mul(wxp, Rwxp);
    for (int r = 0; r < 3; r++)
    {
      pw[r] = pI[r] + Rpb[r];
      pdot[r] = v[r] + Rwxp[r];
    }
    // d pdot / d omega = R [e_k x pb]: column k
    M3 pdot_jac;
    for (int k = 0; k < 3; k++)
    {
      float e[3] = { 0, 0, 0 }, c[3], Rc[3];
      e[k] = 1.0f;
      cross(e, pb, c);
      mul(c, Rc);
      for (int r = 0; r < 3; r++)
        pdot_jac[r][k] = Rc[r];
    }
    float f_k = -p.k_s[i] * (pw[2] - p.l_0[i]) - p.c_s[i] * pdot[2];
    float f_k_jac[3] = { -p.c_s[i] * pdot_jac[2][0], -p.c_s[i] * pdot_jac[2][1], -p.c_s[i] * pdot_jac[2][2] };
    if (f_k < 0)
    {
      f_k = 0;
      f_k_jac[0] = f_k_jac[1] = f_k_jac[2] = 0;
    }
    float delta = 0.0f;
    if (i == 0)
      delta = atanf(p.wheel_base * tan_delta / (p.wheel_base - tan_delta * p.width / 2));
    else if (i == 1)
      delta = atanf(p.wheel_base * tan_delta / (p.wheel_base + tan_delta * p.width / 2));
    const float n[3] = { R[2][0], R[2][1], R[2][2] };  // R^T (0, 0, 1)
    const float wd[3] = { cosf(delta), sinf(delta), 0.0f };
    float s[3], t[3];
    cross(n, wd, s);
    const float sn = sqrtf(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
    for (int r = 0; r < 3; r++)
      s[r] /= sn;
    cross(s, n, t);
    // contact velocity (pdot_x, pdot_y, 0) and its Jacobian (rows 0 and 1 of pdot_jac, row 2 zero) in the body frame
    const float pdc[3] = { pdot[0], pdot[1], 0.0f };
    float pdc_B[3];
    mulT(pdc, pdc_B);
    const float v_s = s[0] * pdc_B[0] + s[1] * pdc_B[1] + s[2] * pdc_B[2];
    float v_s_jac[3];
    for (int k = 0; k < 3; k++)
    {
      const float col[3] = { pdot_jac[0][k], pdot_jac[1][k], 0.0f };
      float colB[3];
      mulT(col, colB);
      v_s_jac[k] = s[0] * colB[0] + s[1] * colB[1] + s[2] * colB[2];
    }
    const float f_n = f_k;
    float mu_s = v_s / p.v_slip * p.mu, dmu = 0.0f;  // stribeck_friction (:77-91)
    if (mu_s > p.mu)
      mu_s = p.mu;
    else if (mu_s < -p.mu)
      mu_s = -p.mu;
    else
      dmu = p.mu / p.v_slip;
    const float f_s = -mu_s * f_n;
    const float f_t = std::max(-p.mu * f_n, std::min(propulsion_force / 4, p.mu * f_n));
    float fc_jac[3][3];  // rows t, s, n of f_r_C_i_Jac
    for (int k = 0; k < 3; k++)
    {
      fc_jac[0][k] = propulsion_force / 4 > p.mu * f_n ? p.mu * f_k_jac[k] :
                     (propulsion_force / 4 < -p.mu * f_n ? -p.mu * f_k_jac[k] : 0.0f);
      fc_jac[1][k] = -f_n * dmu * v_s_jac[k] - mu_s * f_k_jac[k];
      fc_jac[2][k] = f_k_jac[k];
    }
    float f[3], pc[3];
    for (int r = 0; r < 3; r++)
      f[r] = t[r] * f_t + s[r] * f_s + n[r] * f_n;
    const float dc[3] = { pw[0] - pI[0], pw[1] - pI[1], 0.0f - pI[2] };
    mulT(dc, pc);
    float tq[3];
    cross(pc, f, tq);
    for (int r = 0; r < 3; r++)
    {
      f_B[r] += f[r];
      tau_B[r] += tq[r];
    }
    // tau_B_jac += -(f_r_B_i_Jac.colwise().cross(p_c_B_i)) with f_r_B_i_Jac = f_r_C_i_Jac (:215, as written)
    for (int k = 0; k < 3; k++)
    {
      const float col[3] = { fc_jac[0][k], fc_jac[1][k], fc_jac[2][k] };
      float c[3];
      cross(col, pc, c);
      for (int r = 0; r < 3; r++)
        tau_jac[r][k] += -c[r];
    }
    y[11 + 2 * i] = pw[0];
    y[12 + 2 * i] = pw[1];
    y[19 + i] = sqrtf(f[0] * f[0] + f[1] * f[1] + f[2] * f[2]);
  }

  const float inv_mass = 1 / p.mass;
  float Rf[3];
  mul(f_B, Rf);
  for (int r = 0; r < 3; r++)
  {
    xd[r] = v[r];
    xd[7 + r] = inv_mass * Rf[r];
  }
  xd[9] += p.gravity;
  xd[3] = 0.5f * (-qx * w[0] - qy * w[1] - qz * w[2]);
  xd[4] = 0.5f * (qw * w[0] + qy * w[2] - qz * w[1]);
  xd[5] = 0.5f * (qw * w[1] + qz * w[0] - qx * w[2]);
  xd[6] = 0.5f * (qw * w[2] + qx * w[1] - qy * w[0]);
  const float J[3] = { p.Jxx, p.Jyy, p.Jzz };
  const float Jinv[3] = { (float)(1.0 / p.Jxx), (float)(1.0 / p.Jyy), (float)(1.0 / p.Jzz) };
  const float Jw[3] = { J[0] * w[0], J[1] * w[1], J[2] * w[2] };
  float Jwxw[3];
  cross(Jw, w, Jwxw);
  for (int r = 0; r < 3; r++)
    xd[10 + r] = Jinv[r] * (Jwxw[r] + tau_B[r]);
  if (jac)
  {
    // d(Jw x w)/dw, column k: (J e_k) x w - e_k x (J w)
    for (int k = 0; k < 3; k++)
    {
      float e[3] = { 0, 0, 0 }, a[3], b[3];
      e[k] = J[k];
      cross(e, w, a);
      e[k] = 1.0f;
      cross(e, Jw, b);
      for (int r = 0; r < 3; r++)
        jac[r * 3 + k] = Jinv[r] * ((a[r] - b[r]) + tau_jac[r][k]);
    }
  }
  xd[13] = p.steering_constant * (u[1] / p.steer_command_angle_scale - x[13]);

  const float pbl[3] = { -p.cg_pos_wrt_base_link[0], -p.cg_pos_wrt_base_link[1], -p.cg_pos_wrt_base_link[2] };
  float wxb[3], Rpbl[3];
  cross(w, pbl, wxb);
  mul(pbl, Rpbl);
  for (int r = 0; r < 3; r++)
  {
    y[r] = vb[r] + wxb[r];
    y[3 + r] = pI[r] + Rpbl[r];
  }
  // Quat2EulerNWU (math_utils.h:519-527)
  y[7] = atan2f(2.0f * qz * qy + 2.0f * qw * qx, qw * qw + qz * qz - qy * qy - qx * qx);
  y[8] = -asinf(fmaxf(-1.0f, fminf(-2.0f * qw * qy + 2.0f * qx * qz, 1.0f)));
  y[6] = atan2f(2.0f * qy * qx + 2.0f * qz * qw, qw * qw + qx * qx - qy * qy - qz * qz);
  y[9] = x[13];
  y[10] = xd[13];
  y[23] = y[24] = y[25] = 0.0f;
}

// step (host, :31-45): omega by approximate implicit Euler, (I - dt J_w)^-1 dt w_dot; the rest explicit; then q / |q|
static void rigid_suspension_step(const mppib_racer_rigid_suspension_dyn_params& p, const float* x, const float* u, float dt,
                                  float* xn, float* xd, float* y)
{
  float J[9];
  rigid_suspension_deriv(p, x, u, xd, y, J);
  float M[9];
  for (int i = 0; i < 9; i++)
    M[i] = (i % 4 == 0 ? 1.0f : 0.0f) - dt * J[i];
  // the 3x3 inverse by cofactors, as Eigen computes it
  const float c00 = M[4] * M[8] - M[5] * M[7], c01 = M[5] * M[6] - M[3] * M[8], c02 = M[3] * M[7] - M[4] * M[6];
  const float det = M[0] * c00 + M[1] * c01 + M[2] * c02;
  const float inv[9] = { c00 / det, (M[2] * M[7] - M[1] * M[8]) / det, (M[1] * M[5] - M[2] * M[4]) / det,
                         c01 / det, (M[0] * M[8] - M[2] * M[6]) / det, (M[2] * M[3] - M[0] * M[5]) / det,
                         c02 / det, (M[1] * M[6] - M[0] * M[7]) / det, (M[0] * M[4] - M[1] * M[3]) / det };
  for (int i = 0; i < 14; i++)
    xn[i] = x[i] + xd[i] * dt;
  for (int r = 0; r < 3; r++)
    xn[10 + r] = x[10 + r] + ((inv[r * 3] * dt) * xd[10] + (inv[r * 3 + 1] * dt) * xd[11] + (inv[r * 3 + 2] * dt) * xd[12]);
  const float norm = sqrtf(xn[3] * xn[3] + xn[4] * xn[4] + xn[5] * xn[5] + xn[6] * xn[6]);
  for (int i = 3; i < 7; i++)
    xn[i] /= norm;
}

// ---- one trait per built-in model -----------------------------------------------------------------------------------
// S / C / O, limits(params) and step(m, x, u, dt, xn, xd, y), the model's host step; each step zeroes xd where that
// model's host step always has. `generic`: whether mppib_host_step / _output_trajectory take the model. They carry no
// LSTM state and no map, so the RACER models that read one have entries of their own.

// Dynamics::step (dynamics.cuh:283-290) of the models that keep the base class's: computeStateDeriv, updateState, then
// y <- x on the first min(S, O) entries (:292-300)
template <class M>
struct EulerModel
{
  static constexpr bool generic = true;
  static int step(const HostModel& m, const float* x, const float* u, float dt, float* xn, float* xd, float* y)
  {
    for (int i = 0; i < M::S; i++)
      xd[i] = 0.0f;
    if (int rc = M::deriv(m, x, u, xd))
      return rc;
    M::update_state(x, xd, dt, xn);
    for (int i = 0; i < M::O && i < M::S; i++)
      y[i] = xn[i];
    return MPPIB_OK;
  }
  static void update_state(const float* x, const float* xd, float dt, float* xn)  // dynamics.cuh:277-281
  {
    for (int i = 0; i < M::S; i++)
      xn[i] = x[i] + xd[i] * dt;
  }
};

struct Cartpole : EulerModel<Cartpole>
{
  static constexpr int S = 4, C = 1, O = 4;
  static const mppib_control_limits& limits(const void* p) { return ((const mppib_cartpole_dyn_params*)p)->lim; }
  static int deriv(const HostModel& m, const float* x, const float* u, float* xdot)
  {  // dynamics/cartpole/cartpole_dynamics.cu:48-69
    const auto& q = *(const mppib_cartpole_dyn_params*)m.params;
    const float st = sinf(x[2]), ct = cosf(x[2]);
    const float m_c = q.cart_mass, m_p = q.pole_mass, l_p = q.pole_length, g = q.gravity;
    xdot[0] = x[1];
    xdot[1] = 1.0f / (m_c + m_p * st * st) * (u[0] + m_p * st * (l_p * x[3] * x[3] + g * ct));
    xdot[2] = x[3];
    xdot[3] = 1.0f / (l_p * (m_c + m_p * st * st)) *
              (-u[0] * ct - m_p * l_p * x[3] * x[3] * ct * st - (m_c + m_p) * g * st);
    return 0;
  }
};

struct DoubleIntegrator : EulerModel<DoubleIntegrator>
{
  static constexpr int S = 4, C = 2, O = 4;
  static const mppib_control_limits& limits(const void* p) { return ((const mppib_di_dyn_params*)p)->lim; }
  static int deriv(const HostModel&, const float* x, const float* u, float* xdot)
  {  // dynamics/double_integrator/di_dynamics.cu:14-22
    xdot[0] = x[2];
    xdot[1] = x[3];
    xdot[2] = u[0];
    xdot[3] = u[1];
    return 0;
  }
};

struct Autorally : EulerModel<Autorally>
{
  static constexpr int S = 7, C = 2, O = 8;
  static const mppib_control_limits& limits(const void* p) { return ((const mppib_ar_nn_dyn_params*)p)->lim; }
  static int deriv(const HostModel& m, const float* x, const float* u, float* xdot)
  {  // dynamics/autorally/ar_nn_model.cu:90-119
    if (!m.fnn)
      return MPPIB_ERR_INVALID_ARG;
    const float cs = cosf(x[2]), sn = sinf(x[2]);
    xdot[0] = cs * x[4] - sn * x[5];
    xdot[1] = sn * x[4] + cs * x[5];
    xdot[2] = -x[6];
    const float in6[6] = { x[3], x[4], x[5], x[6], u[0], u[1] };
    fnn_6_32_32_4(*m.fnn, in6, xdot + 3);
    return 0;
  }
};

struct Quadrotor : EulerModel<Quadrotor>
{
  static constexpr int S = 13, C = 4, O = 13;
  static const mppib_control_limits& limits(const void* p) { return ((const mppib_quadrotor_dyn_params*)p)->lim; }
  static int deriv(const HostModel& m, const float* x, const float* u, float* xdot)
  {  // dynamics/quadrotor/quadrotor_dynamics.cu:70-112; DCM column 2 as Eigen's toRotationMatrix evaluates it
    const auto& q = *(const mppib_quadrotor_dyn_params*)m.params;
    const float qw = x[6], qx = x[7], qy = x[8], qz = x[9];
    const float tx = 2.0f * qx, ty = 2.0f * qy, tz = 2.0f * qz;
    const float col2[3] = { tz * qx + ty * qw, tz * qy - tx * qw, 1.0f - (tx * qx + ty * qy) };
    const float tau_inv[3] = { 1 / q.tau_roll, 1 / q.tau_pitch, 1 / q.tau_yaw };
    for (int i = 0; i < 3; i++)
    {
      xdot[i] = x[3 + i];
      xdot[3 + i] = (u[3] / q.mass) * col2[i];
      xdot[10 + i] = tau_inv[i] * (u[i] - x[10 + i]);
    }
    xdot[5] -= MPPIB_GRAVITY;
    const float pp = x[10], qq = x[11], rr = x[12];
    xdot[6] = 0.5f * (-pp * qx - qq * qy - rr * qz);
    xdot[7] = 0.5f * (pp * qw - qq * qz + rr * qy);
    xdot[8] = 0.5f * (pp * qz + qq * qw - rr * qx);
    xdot[9] = 0.5f * (-pp * qy + qq * qx + rr * qw);
    return 0;
  }
  // QuadrotorDynamics::updateState renormalises the quaternion after the Euler step (quadrotor_dynamics.cu:114-122)
  static void update_state(const float* x, const float* xd, float dt, float* xn)
  {
    EulerModel::update_state(x, xd, dt, xn);
    float* q = xn + 6;
    const float norm = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const float div = (float)((double)norm * copysign(1.0, (double)q[0]));
    for (int i = 0; i < 4; i++)
      q[i] /= div;
  }
};

struct RacerLstm  // RacerDubinsElevationLSTMSteering
{
  static constexpr int S = 19, C = 2, O = 28;
  static constexpr bool generic = false;
  static const mppib_control_limits& limits(const void* p) { return ((const mppib_racer_lstm_dyn_params*)p)->lim; }
  static int step(const HostModel& m, const float* x, const float* u, float dt, float* xn, float* xd, float* y)
  {
    for (int i = 0; i < S; i++)
      xd[i] = 0.0f;
    racer_step(*(const mppib_racer_lstm_dyn_params*)m.params, m.lstm, m.elevation, x, u, dt, xn, xd, y);
    return MPPIB_OK;
  }
};

struct RacerDubinsElevation
{
  static constexpr int S = 19, C = 2, O = 28;
  static constexpr bool generic = false;
  static const mppib_control_limits& limits(const void* p)
  {
    return ((const mppib_racer_dubins_elevation_dyn_params*)p)->lim;
  }
  static int step(const HostModel& m, const float* x, const float* u, float dt, float* xn, float* xd, float* y)
  {
    for (int i = 0; i < S; i++)
      xd[i] = 0.0f;
    racer_dubins_step(*(const mppib_racer_dubins_elevation_dyn_params*)m.params, m.elevation, x, u, dt, xn, xd, y);
    return MPPIB_OK;
  }
};

struct RacerSuspensionLstm  // RacerDubinsElevationSuspension
{
  static constexpr int S = 24, C = 2, O = 28;
  static constexpr bool generic = false;
  static const mppib_control_limits& limits(const void* p)
  {
    return ((const mppib_racer_suspension_dyn_params*)p)->base.lim;
  }
  static int step(const HostModel& m, const float* x, const float* u, float dt, float* xn, float* xd, float* y)
  {
    for (int i = 0; i < S; i++)
      xd[i] = 0.0f;
    racer_suspension_step(*(const mppib_racer_suspension_dyn_params*)m.params, m.lstm, m.elevation, m.normals, x, u, dt,
                          xn, xd, y);
    return MPPIB_OK;
  }
};

struct RacerSuspension  // the rigid body; its step writes every entry of xd and of y (the outputs of x)
{
  static constexpr int S = 14, C = 2, O = 26;
  static constexpr bool generic = true;
  static const mppib_control_limits& limits(const void* p)
  {
    return ((const mppib_racer_rigid_suspension_dyn_params*)p)->lim;
  }
  static int step(const HostModel& m, const float* x, const float* u, float dt, float* xn, float* xd, float* y)
  {
    rigid_suspension_step(*(const mppib_racer_rigid_suspension_dyn_params*)m.params, x, u, dt, xn, xd, y);
    return MPPIB_OK;
  }
};

// The one switch over the dynamics ids: f(the model's trait), or `unknown` for an id that is not a built-in model
template <class F>
int with_model(int dyn_id, int unknown, F&& f)
{
  switch (dyn_id)
  {
    case MPPIB_DYN_CARTPOLE:
      return f(Cartpole{});
    case MPPIB_DYN_DOUBLE_INTEGRATOR:
      return f(DoubleIntegrator{});
    case MPPIB_DYN_AUTORALLY_NN:
      return f(Autorally{});
    case MPPIB_DYN_RACER_LSTM:
      return f(RacerLstm{});
    case MPPIB_DYN_QUADROTOR:
      return f(Quadrotor{});
    case MPPIB_DYN_RACER_DUBINS_ELEVATION:
      return f(RacerDubinsElevation{});
    case MPPIB_DYN_RACER_SUSPENSION_LSTM:
      return f(RacerSuspensionLstm{});
    case MPPIB_DYN_RACER_SUSPENSION:
      return f(RacerSuspension{});
  }
  return unknown;
}

// Controller::computeOutputTrajectoryHelper (controller.cuh:643-663) with the model's dimensions known at compile time:
// this loop runs in every computeControl. y starts as initializeDynamics leaves it (dynamics.cuh:416-423: x on the first
// min(S, O) entries, 0 after) and keeps what a step does not write (Autorally's eighth output). An LSTM starts from the
// initial hidden / cell state its weight blob carries after the biases (lstm_steering.cu:230-237, lstm_helper.cu:86-87);
// the caller's hidden / cell vectors are not touched.
template <class M>
int roll(HostModel m, const float* x0, const float* u, int T, float dt, float* states, float* outputs)
{
  constexpr int S = M::S, C = M::C, O = M::O;
  mppib_host_lstm net;
  std::vector<float> hidden_cell;
  if (m.lstm)
  {
    net = *m.lstm;
    const int H = net.hidden_dim;
    const float* init = net.theta + 4 * H * H + 4 * H * MPPIB_RACER_LSTM_INPUT_DIM + 4 * H;
    hidden_cell.assign(init, init + 2 * H);
    net.hidden = hidden_cell.data();
    net.cell = hidden_cell.data() + H;
    m.lstm = &net;
  }
  const mppib_control_limits& lim = M::limits(m.params);
  float xn[S], xd[S], y[O] = {}, ui[C];
  memcpy(states, x0, sizeof(xn));
  memcpy(y, x0, sizeof(float) * std::min(S, O));
  memcpy(outputs, y, sizeof(y));
  for (int t = 0; t < T - 1; t++)
  {
    memcpy(ui, u + (size_t)t * C, sizeof(ui));
    enforce(lim, ui, C);
    if (int rc = M::step(m, states + (size_t)t * S, ui, dt, xn, xd, y))
      return rc;
    memcpy(states + (size_t)(t + 1) * S, xn, sizeof(xn));
    memcpy(outputs + (size_t)(t + 1) * O, y, sizeof(y));
  }
  return MPPIB_OK;
}

// What the generic entries know of a model: its parameters and Autorally's network, transposed into `nn`
HostModel generic_view(int dyn_id, const void* params, const float* nn_theta, FnnT& nn)
{
  const bool fnn = dyn_id == MPPIB_DYN_AUTORALLY_NN && nn_theta;
  if (fnn)
    mppib::fnn_transpose(nn_theta, nn);
  return HostModel{ dyn_id, params, fnn ? &nn : nullptr, nullptr, nullptr, nullptr };
}

// ---- robust costs (host bodies) ----------------------------------------------------------------------------------------
// utils/math_utils.h:90-94,149-155
static inline float lin_interp(const float x, const float x_min, const float x_max, const float y_min, const float y_max)
{
  return (x - x_min) / (x_max - x_min) * (y_max - y_min) + y_min;
}
static inline float norm_dist_from_center(const float r, const float r_in, const float r_out)
{
  float r_center = (r_in + r_out) / 2.0f;
  float r_width = (r_out - r_in);
  float dist_from_center = fabsf(r - r_center);
  return dist_from_center / (r_width * 0.5f);
}
// double_integrator_robust_cost.cu:41-69 — the HOST body: steep boundary 0.75 and steep cost 0.1 * crash_cost (the device
// body, csrc/plugins/costs.cuh, uses 0.5 and 0.5 * crash_cost)
float di_robust_state_cost(const mppib_di_circle_cost_params& p, const float* s)
{
  float radial_position = s[0] * s[0] + s[1] * s[1];
  float current_velocity = sqrtf(s[2] * s[2] + s[3] * s[3]);
  float current_angular_momentum = s[0] * s[3] - s[1] * s[2];
  float cost = 0;
  float normalized_dist_from_center =
      norm_dist_from_center(std::sqrt(radial_position), std::sqrt(p.inner_path_radius2), std::sqrt(p.outer_path_radius2));
  float steep_percent_boundary = 0.75;
  float steep_cost = 0.1 * p.crash_cost;  // double product, narrowed
  if (normalized_dist_from_center <= steep_percent_boundary)
    cost += lin_interp(normalized_dist_from_center, 0, steep_percent_boundary, 0, steep_cost);
  else if (normalized_dist_from_center > steep_percent_boundary && normalized_dist_from_center <= 1.0)
    cost += lin_interp(normalized_dist_from_center, steep_percent_boundary, 1, steep_cost, p.crash_cost);
  else
    cost += p.crash_cost;
  cost += p.velocity_cost * powf(current_velocity - p.velocity_desired, 2);
  cost += p.velocity_cost * powf(current_angular_momentum - p.angular_momentum_desired, 2);
  return cost;
}
// ar_robust_cost.cu:13-38 (host and device share this body)
float ar_robust_stabilizing_cost(const mppib_ar_robust_cost_params& p, const float* s)
{
  float penalty_val = 0;
  float slip;
  if (std::fabs(s[4]) < 0.001)
    slip = 0;
  else
    slip = std::fabs(-std::atan(s[5] / std::fabs(s[4])));
  if (slip >= 0.75 * p.max_slip_ang)
  {
    float slip_val = fminf(1.0, slip / p.max_slip_ang);
    float alpha = (slip_val - 0.75) / (1.0 - 0.75);
    penalty_val = alpha * p.crash_coeff;
  }
  if (std::fabs(s[3]) >= M_PI_2)
    penalty_val = p.crash_coeff;
  return p.slip_coeff * slip + penalty_val;
}
// ar_robust_cost.cu:40-117, host branch: cosf / sinf, nearest texel by std::round after the clamps of :64-70
float ar_robust_costmap_cost(const mppib_ar_robust_cost_params& p, const float* track_costs, const float* s)
{
  float cost = 0;
  float x_front = s[0] + p.front_d * cosf(s[2]);
  float y_front = s[1] + p.front_d * sinf(s[2]);
  float x_back = s[0] + p.back_d * cosf(s[2]);
  float y_back = s[1] + p.back_d * sinf(s[2]);
  auto texel = [&](float x, float y) {
    float u = p.r_c1[0] * x + p.r_c2[0] * y + p.trs[0];
    float v = p.r_c1[1] * x + p.r_c2[1] * y + p.trs[1];
    float w = p.r_c1[2] * x + p.r_c2[2] * y + p.trs[2];
    float qx = u / w * p.map_width - 0.5f;
    float qy = v / w * p.map_height - 0.5f;
    qx = fmaxf(0.0f, fminf(p.map_width - 1, qx));
    qy = fmaxf(0.0f, fminf(p.map_height - 1, qy));
    return track_costs + 4 * ((size_t)std::round(qy) * p.map_width + (size_t)std::round(qx));
  };
  const float* front = texel(x_front, y_front);
  const float* back = texel(x_back, y_back);
  float constraint_val = fminf(1.0, fmaxf(front[0], back[0]));
  if (constraint_val >= p.boundary_threshold)
  {
    float alpha = (constraint_val - p.boundary_threshold) / (1.0 - p.boundary_threshold);
    cost += alpha * p.crash_coeff;
  }
  if (front[1] > p.track_slop)
    cost += p.track_coeff * front[1];
  if (p.desired_speed == -1)
    cost += p.speed_coeff * std::fabs(s[4] - front[2]);
  else
    cost += p.speed_coeff * std::fabs(s[4] - p.desired_speed);
  cost += p.heading_coeff * std::fabs(sinf(s[2]) + front[3]);
  return cost;
}

// ---- QuadrotorMapCost (quadrotor_map_cost.cu), the __host__ side of its __host__ __device__ terms -------------------
using QMapParams = mppib_quadrotor_map_cost_params;
// :146-152
float qmap_dist_to_waypoint(const float* s, const float* w)
{
  return std::sqrt((s[0] - w[0]) * (s[0] - w[0]) + (s[1] - w[1]) * (s[1] - w[1]) + (s[2] - w[2]) * (s[2] - w[2]));
}
// :264-323
float qmap_gate_side_cost(const QMapParams& p, const float* s)
{
  float cost = 0;
  const float gx = p.curr_gate_left[0] - p.curr_gate_right[0], gy = p.curr_gate_left[1] - p.curr_gate_right[1];
  const float rx = s[0] - p.curr_gate_right[0], ry = s[1] - p.curr_gate_right[1];
  const float perp_dist = rx * gy - ry * gx;
  const float comp = (rx * gx + ry * gy) / (gx * gx + gy * gy);
  if (std::fabs(perp_dist) < p.min_dist_to_gate_side && ((comp < 0.0f && comp >= -0.5f) || (comp > 1.0f && comp <= 1.5f)))
    cost += p.crash_coeff * std::fabs(comp);
  return cost;
}
// :325-357: double weights and interpolation narrowed to float; +400 when the squared difference exceeds gate_width
float qmap_height_cost(const QMapParams& p, const float* s)
{
  float cost = 0;
  float d1 = sqrtf((s[0] - p.prev_waypoint[0]) * (s[0] - p.prev_waypoint[0]) +
                   (s[1] - p.prev_waypoint[1]) * (s[1] - p.prev_waypoint[1]));
  float d2 = sqrtf((s[0] - p.curr_waypoint[0]) * (s[0] - p.curr_waypoint[0]) +
                   (s[1] - p.curr_waypoint[1]) * (s[1] - p.curr_waypoint[1]));
  float w1 = d1 / (d1 + d2 + 0.001);
  float w2 = d2 / (d1 + d2 + 0.001);
  float interpolated_height = (1.0 - w1) * p.prev_waypoint[2] + (1.0 - w2) * p.curr_waypoint[2];
  float dz = std::fabs(s[2] - interpolated_height);
  float height_diff = dz * dz;
  cost += p.height_coeff * height_diff;
  if (height_diff > p.gate_width)
    cost += 400;
  return cost;
}
// :210-238
float qmap_heading_cost(const QMapParams& p, const float* s)
{
  float cost = 0;
  const float* q = s + 6;
  const float vx = s[3], vy = s[4], vz = s[5];
  const float R00 = q[0] * q[0] + q[1] * q[1] - q[2] * q[2] - q[3] * q[3];
  const float R01 = 2 * (q[1] * q[2] - q[0] * q[3]);
  const float R02 = 2 * (q[1] * q[3] + q[0] * q[2]);
  const float R10 = 2 * (q[1] * q[2] + q[0] * q[3]);
  const float R11 = q[0] * q[0] - q[1] * q[1] + q[2] * q[2] - q[3] * q[3];
  const float R12 = 2 * (q[2] * q[3] - q[0] * q[1]);
  const float yaw = atan2f(R10 * vx + R11 * vy + R12 * vz, R00 * vx + R01 * vy + R02 * vz);
  const float w_heading = atan2f(p.curr_waypoint[1] - s[1], p.curr_waypoint[0] - s[0]);
  if (qmap_dist_to_waypoint(s, p.curr_waypoint) > p.gate_margin)
    cost += p.heading_coeff * powf(std::fabs(normalize_angle(yaw - w_heading)), p.heading_power);
  return cost;
}
// :240-252
float qmap_speed_cost(const QMapParams& p, const float* s)
{
  const float speed = std::sqrt(s[3] * s[3] + s[4] * s[4]);
  return p.speed_coeff * ((speed - p.desired_speed) * (speed - p.desired_speed));
}
// :199-208 with Quat2EulerNWU (math_utils.h:263-270)
float qmap_stabilizing_cost(const QMapParams& p, const float* s)
{
  const float* q = s + 6;
  const float roll = atan2f(2.0f * q[3] * q[2] + 2.0f * q[0] * q[1], q[0] * q[0] + q[3] * q[3] - q[2] * q[2] - q[1] * q[1]);
  const float temp = -2.0f * q[0] * q[2] + 2.0f * q[1] * q[3];
  const float pitch = -asinf(fmaxf(fminf(1.0f, temp), -1.0f));
  return p.attitude_coeff * (roll * roll + pitch * pitch);
}
// :254-262
float qmap_waypoint_cost(const QMapParams& p, const float* s)
{
  const float d = qmap_dist_to_waypoint(s, p.curr_waypoint);
  return p.dist_to_waypoint_coeff * (d * d);
}
// :63-90, the HOST body: no costmap term, no crash flag, and the waypoint term added (the device body is in costs.cuh)
float qmap_state_cost(const QMapParams& p, const float* s)
{
  float cost = 0;
  cost += qmap_gate_side_cost(p, s);
  cost += qmap_height_cost(p, s);
  cost += qmap_heading_cost(p, s);
  cost += qmap_speed_cost(p, s);
  cost += qmap_stabilizing_cost(p, s);
  cost += qmap_waypoint_cost(p, s);
  if (qmap_dist_to_waypoint(s, p.curr_waypoint) < p.gate_margin)
    cost += p.gate_pass_cost;
  return cost;
}

}  // namespace

void mppib::fnn_transpose(const float* theta, FnnT& t)
{
  for (int j = 0; j < 32; j++)
    for (int k = 0; k < 6; k++)
      t.WT1[k * 32 + j] = theta[j * 6 + k];
  memcpy(t.b1, theta + 192, sizeof(t.b1));
  for (int j = 0; j < 32; j++)
    for (int k = 0; k < 32; k++)
      t.WT2[k * 32 + j] = theta[224 + j * 32 + k];
  memcpy(t.b2, theta + 1248, sizeof(t.b2));
  memcpy(t.W3, theta + 1280, sizeof(t.W3));
  memcpy(t.b3, theta + 1408, sizeof(t.b3));
}

int mppib::roll_forward(const HostModel& m, const float* x0, const float* u, int T, float dt, float* states,
                        float* outputs)
{
  return with_model(m.dyn_id, MPPIB_ERR_UNSUPPORTED,
                    [&](auto model) { return roll<decltype(model)>(m, x0, u, T, dt, states, outputs); });
}

extern "C" {

int mppib_host_state_cost(int cost_id, const void* params, const float* costmap, const float* y, int t, int* crash,
                          float* cost)
{
  (void)t;
  (void)crash;  // no host body reads the time step or the crash flag
  if (!params || !y || !cost)
    return MPPIB_ERR_INVALID_ARG;
  switch (cost_id)
  {
    case MPPIB_COST_DI_ROBUST:
      *cost = di_robust_state_cost(*static_cast<const mppib_di_circle_cost_params*>(params), y);
      return MPPIB_OK;
    case MPPIB_COST_AR_ROBUST:
    {
      const auto& p = *static_cast<const mppib_ar_robust_cost_params*>(params);
      if (!costmap || p.map_width <= 0 || p.map_height <= 0)
        return MPPIB_ERR_INVALID_ARG;
      float c = ar_robust_stabilizing_cost(p, y) + ar_robust_costmap_cost(p, costmap, y);  // ar_robust_cost.cu:119-132
      if (c > 1e16f || std::isnan(c))
        c = 1e16f;  // MAX_COST_VALUE
      *cost = c;
      return MPPIB_OK;
    }
    case MPPIB_COST_QUADROTOR_MAP:
      *cost = qmap_state_cost(*static_cast<const mppib_quadrotor_map_cost_params*>(params), y);
      return MPPIB_OK;
    default:
      return MPPIB_ERR_UNSUPPORTED;
  }
}

int mppib_host_quadrotor_map_term(const mppib_quadrotor_map_cost_params* params, int term, const float* s, float* cost)
{
  if (!params || !s || !cost)
    return MPPIB_ERR_INVALID_ARG;
  const mppib_quadrotor_map_cost_params& p = *params;
  switch (term)
  {
    case MPPIB_QMAP_GATE_SIDE:
      *cost = qmap_gate_side_cost(p, s);
      return MPPIB_OK;
    case MPPIB_QMAP_HEADING:
      *cost = qmap_heading_cost(p, s);
      return MPPIB_OK;
    case MPPIB_QMAP_HEIGHT:
      *cost = qmap_height_cost(p, s);
      return MPPIB_OK;
    case MPPIB_QMAP_SPEED:
      *cost = qmap_speed_cost(p, s);
      return MPPIB_OK;
    case MPPIB_QMAP_STABILIZING:
      *cost = qmap_stabilizing_cost(p, s);
      return MPPIB_OK;
    case MPPIB_QMAP_WAYPOINT:
      *cost = qmap_waypoint_cost(p, s);
      return MPPIB_OK;
    default:
      return MPPIB_ERR_INVALID_ARG;
  }
}

int mppib_host_quadrotor_map_update_gate_boundaries(mppib_quadrotor_map_cost_params* p, float left_x, float left_y,
                                                    float left_z, float right_x, float right_y, float right_z)
{
  if (!p)
    return MPPIB_ERR_INVALID_ARG;
  if (p->curr_gate_left[0] != left_x || p->curr_gate_left[1] != left_y || p->curr_gate_left[2] != left_z ||
      p->curr_gate_right[0] != right_x || p->curr_gate_right[1] != right_y || p->curr_gate_right[2] != right_z)
  {
    memcpy(p->prev_gate_left, p->curr_gate_left, sizeof(p->prev_gate_left));
    memcpy(p->prev_gate_right, p->curr_gate_right, sizeof(p->prev_gate_right));
    p->curr_gate_left[0] = left_x, p->curr_gate_left[1] = left_y, p->curr_gate_left[2] = left_z;
    p->curr_gate_right[0] = right_x, p->curr_gate_right[1] = right_y, p->curr_gate_right[2] = right_z;
    return 1;
  }
  return 0;
}

int mppib_host_quadrotor_map_update_waypoint(mppib_quadrotor_map_cost_params* p, float x, float y, float z, float heading)
{
  if (!p)
    return MPPIB_ERR_INVALID_ARG;
  if (p->curr_waypoint[0] != x || p->curr_waypoint[1] != y || p->curr_waypoint[2] != z || p->curr_waypoint[3] != heading)
  {
    memcpy(p->prev_waypoint, p->curr_waypoint, sizeof(p->prev_waypoint));
    p->curr_waypoint[0] = x, p->curr_waypoint[1] = y, p->curr_waypoint[2] = z, p->curr_waypoint[3] = heading;
    const float w = p->gate_width;
    mppib_host_quadrotor_map_update_gate_boundaries(p, x + cosf(heading) * w, y + sinf(heading) * w, z,
                                                    x - cosf(heading) * w, y - sinf(heading) * w, z);
    return 1;
  }
  return 0;
}

float mppib_host_quadrotor_map_dist_to_waypoint(const float* s, const float* waypoint)
{
  return (s && waypoint) ? qmap_dist_to_waypoint(s, waypoint) : 0.0f;
}

int mppib_host_ar_robust_stabilizing_cost(const mppib_ar_robust_cost_params* params, const float* s, float* cost)
{
  if (!params || !s || !cost)
    return MPPIB_ERR_INVALID_ARG;
  *cost = ar_robust_stabilizing_cost(*params, s);
  return MPPIB_OK;
}

int mppib_host_ar_robust_costmap_cost(const mppib_ar_robust_cost_params* params, const float* costmap, const float* s,
                                      float* cost)
{
  if (!params || !costmap || !s || !cost || params->map_width <= 0 || params->map_height <= 0)
    return MPPIB_ERR_INVALID_ARG;
  *cost = ar_robust_costmap_cost(*params, costmap, s);
  return MPPIB_OK;
}

int mppib_host_dims(int dyn_id, int* S, int* C, int* O)
{
  return with_model(dyn_id, MPPIB_ERR_UNSUPPORTED, [&](auto model) -> int {
    using M = decltype(model);
    if (S)
      *S = M::S;
    if (C)
      *C = M::C;
    if (O)
      *O = M::O;
    return MPPIB_OK;
  });
}

int mppib_host_enforce_constraints(int dyn_id, const void* dyn_params, float* u)
{
  if (!dyn_params || !u)
    return MPPIB_ERR_INVALID_ARG;
  return with_model(dyn_id, MPPIB_ERR_INVALID_ARG, [&](auto model) -> int {
    using M = decltype(model);
    enforce(M::limits(dyn_params), u, M::C);
    return MPPIB_OK;
  });
}

int mppib_host_step(int dyn_id, const void* dyn_params, const float* nn_theta, const float* x, const float* u,
                    float dt, float* x_next, float* xdot, float* y)
{
  if (!dyn_params || !x || !u || !x_next || !xdot || !y)
    return MPPIB_ERR_INVALID_ARG;
  return with_model(dyn_id, MPPIB_ERR_INVALID_ARG, [&](auto model) -> int {
    using M = decltype(model);
    if constexpr (M::generic)
    {
      FnnT nn;
      return M::step(generic_view(dyn_id, dyn_params, nn_theta, nn), x, u, dt, x_next, xdot, y);
    }
    else
    {
      std::fill(xdot, xdot + M::S, 0.0f);  // a refused model's xdot comes back zeroed, as it always has
      return MPPIB_ERR_UNSUPPORTED;
    }
  });
}

void mppib_host_smooth_controls(float* u, const float* history, int T, int C)
{
  // controller.cuh:557-586: coefficients (-3 12 17 12 -3)/35 over [history(2) | u(T) | u_last u_last]
  const float coef[5] = { -3.0f / 35.0f, 12.0f / 35.0f, 17.0f / 35.0f, 12.0f / 35.0f, -3.0f / 35.0f };
  std::vector<float> buf((size_t)(T + 4) * C);
  for (int c = 0; c < C; c++)
  {
    buf[c] = history[c];
    buf[C + c] = history[C + c];
    for (int t = 0; t < T; t++)
      buf[(size_t)(t + 2) * C + c] = u[(size_t)t * C + c];
    buf[(size_t)(T + 2) * C + c] = u[(size_t)(T - 1) * C + c];
    buf[(size_t)(T + 3) * C + c] = u[(size_t)(T - 1) * C + c];
  }
  for (int t = 0; t < T; t++)
    for (int c = 0; c < C; c++)
    {
      float acc = 0.0f;
      for (int k = 0; k < 5; k++)
        acc += coef[k] * buf[(size_t)(t + k) * C + c];
      u[(size_t)t * C + c] = acc;
    }
}

void mppib_host_slide_controls(float* u, int steps, int T, int C, const float* zero_control, const float* scale)
{
  // controller.cuh:588-600
  for (int i = 0; i < T; ++i)
  {
    const int ind = std::min(i + steps, T - 1);
    for (int c = 0; c < C; c++)
    {
      float v = u[(size_t)ind * C + c];
      if (i + steps > T - 1)
        v = (v - zero_control[c]) * scale[c] + zero_control[c];
      u[(size_t)i * C + c] = v;
    }
  }
}

int mppib_host_output_trajectory(int dyn_id, const void* dyn_params, const float* nn_theta, const float* x0,
                                 const float* u, int T, float dt, float* states, float* outputs)
{
  if (!dyn_params || !x0 || !u || !states || !outputs || T <= 0)
    return MPPIB_ERR_INVALID_ARG;
  if (dyn_id == MPPIB_DYN_AUTORALLY_NN && !nn_theta)
    return MPPIB_ERR_INVALID_ARG;
  return with_model(dyn_id, MPPIB_ERR_UNSUPPORTED, [&](auto model) -> int {
    using M = decltype(model);
    if constexpr (M::generic)
    {
      FnnT nn;
      return roll<M>(generic_view(dyn_id, dyn_params, nn_theta, nn), x0, u, T, dt, states, outputs);
    }
    else
      return MPPIB_ERR_UNSUPPORTED;
  });
}

// LSTMLSTMHelper::initializeLSTM, lstm_lstm_helper.cu:50-73, with LSTMHelper::forward (host, lstm_helper.cu:267-339) and
// FNNHelper::forward (host: tanh between layers, linear output) for arbitrary dimensions. Runs once per re-initialisation
// (a few hundred microseconds of scalar code), not per solve.
int mppib_host_lstm_initialize(const mppib_host_init_lstm* net, const float* buffer, int cols, float* out)
{
  if (!net || !net->lstm_theta || !net->head_theta || !net->head_layers || !buffer || !out)
    return MPPIB_ERR_INVALID_ARG;
  const int I = net->input_dim, H = net->hidden_dim, L = net->head_num_layers;
  if (I <= 0 || H <= 0 || L < 2 || net->init_len <= 0 || cols < net->init_len || net->head_layers[0] != H + I)
    return MPPIB_ERR_INVALID_ARG;
  const int HH = H * H, IH = H * I;
  const float* w = net->lstm_theta;
  const float* bias = w + 4 * HH + 4 * IH;
  std::vector<float> h(bias + 4 * H, bias + 5 * H), c(bias + 5 * H, bias + 6 * H);  // resetHiddenCellCPU
  std::vector<float> hn(H), cn(H);
  for (int t = cols - net->init_len; t < cols; t++)
  {
    const float* x = buffer + (size_t)t * I;
    for (int i = 0; i < H; i++)
    {
      float g[4];
      for (int k = 0; k < 4; k++)
      {
        const float* Wm = w + k * HH + i * H;
        const float* Wi = w + 4 * HH + k * IH + i * I;
        float hm = 0.0f, im = 0.0f;
        for (int j = 0; j < H; j++)
          hm += Wm[j] * h[j];
        for (int j = 0; j < I; j++)
          im += Wi[j] * x[j];
        g[k] = (hm + im) + bias[k * H + i];
      }
      const float gi = 1.0f / (1.0f + expf(-g[0])), gf = 1.0f / (1.0f + expf(-g[1])), go = 1.0f / (1.0f + expf(-g[2]));
      cn[i] = gi * tanhf(g[3]) + gf * c[i];
      hn[i] = go * tanhf(cn[i]);
    }
    h = hn;
    c = cn;
  }
  // head on [h; x_last]
  int widest = 0;
  for (int l = 0; l < L; l++)
  {
    if (net->head_layers[l] <= 0)
      return MPPIB_ERR_INVALID_ARG;
    widest = std::max(widest, net->head_layers[l]);
  }
  std::vector<float> a(widest), b(widest);
  for (int i = 0; i < H; i++)
    a[i] = h[i];
  for (int i = 0; i < I; i++)
    a[H + i] = buffer[(size_t)(cols - 1) * I + i];
  const float* th = net->head_theta;
  for (int l = 0; l + 1 < L; l++)
  {
    const int in = net->head_layers[l], on = net->head_layers[l + 1];
    const float* W = th;
    const float* bb = th + (size_t)in * on;
    for (int o = 0; o < on; o++)
    {
      float acc = 0.0f;
      for (int j = 0; j < in; j++)
        acc += W[(size_t)o * in + j] * a[j];
      acc += bb[o];
      b[o] = (l + 2 < L) ? tanhf(acc) : acc;
    }
    std::swap(a, b);
    th += (size_t)in * on + on;
  }
  memcpy(out, a.data(), sizeof(float) * net->head_layers[L - 1]);
  return MPPIB_OK;
}

float mppib_host_elevation_at_world_pose(const mppib_elevation_map_header* map, float x, float y, float z)
{
  return map ? elevation_at_world_pose(map, x, y, z) : 0.0f;
}
float mppib_host_static_settling(const mppib_elevation_map_header* map, float yaw, float x, float y, float* roll, float* pitch)
{
  float r = roll ? *roll : 0.0f, p = pitch ? *pitch : 0.0f;
  const float h = static_settling(map, yaw, x, y, r, p);
  if (roll)
    *roll = r;
  if (pitch)
    *pitch = p;
  return h;
}

int mppib_host_step_lstm(const void* dyn_params, const mppib_host_lstm* net, const float* x, const float* u, float dt,
                         float* x_next, float* xdot, float* y)
{
  if (!dyn_params || !net || !net->theta || !net->hidden || !net->cell || !x || !u || !x_next || !xdot || !y)
    return MPPIB_ERR_INVALID_ARG;
  return RacerLstm::step({ MPPIB_DYN_RACER_LSTM, dyn_params, nullptr, net, net->map, nullptr }, x, u, dt, x_next, xdot, y);
}

int mppib_host_step_racer_dubins_elevation(const void* dyn_params, const mppib_elevation_map_header* map, const float* x,
                                           const float* u, float dt, float* x_next, float* xdot, float* y)
{
  if (!dyn_params || !x || !u || !x_next || !xdot || !y)
    return MPPIB_ERR_INVALID_ARG;
  return RacerDubinsElevation::step({ MPPIB_DYN_RACER_DUBINS_ELEVATION, dyn_params, nullptr, nullptr, map, nullptr }, x, u,
                                    dt, x_next, xdot, y);
}

// RacerDubinsElevationImpl::computeGrad (host method, racer_dubins_elevation.cu:257-334) as written: A [19][19] and
// B [19][2] row-major; 1 / cos^2 in double as the reference evaluates it
int mppib_host_grad_racer_dubins_elevation(const void* dyn_params, const float* x, const float* u, float* A, float* B)
{
  if (!dyn_params || !x || !u || !A || !B)
    return MPPIB_ERR_INVALID_ARG;
  const auto& p = *(const mppib_racer_dubins_elevation_dyn_params*)dyn_params;
  std::fill(A, A + 19 * 19, 0.0f);
  std::fill(B, B + 19 * 2, 0.0f);
  auto a = [&](int r, int c) -> float& { return A[r * 19 + c]; };
  const float eps = 0.01f;
  const bool enable_brake = u[0] < 0.0f;
  const float vx = x[R_VEL_X];
  const int index = (fabsf(vx) > 0.2f && fabsf(vx) <= 3.0f) + (fabsf(vx) > 3.0f) * 2;
  a(R_VEL_X, R_VEL_X) = -p.c_v[index];
  a(R_VEL_X, R_BRAKE_STATE) = fabsf(vx) < 0.2f ? p.c_b[index] * -vx : p.c_b[index] * (vx >= 0.0f ? -1.0f : 1.0f);
  a(R_YAW, R_VEL_X) = (1.0f / p.wheel_base) * tanf(x[R_STEER_ANGLE] / p.steer_angle_scale);
  a(R_YAW, R_STEER_ANGLE) = (float)((vx / p.wheel_base) * (1.0 / ((double)cosf(x[R_STEER_ANGLE] / p.steer_angle_scale) *
                                                                   cosf(x[R_STEER_ANGLE] / p.steer_angle_scale))) /
                                    p.steer_angle_scale);
  a(R_POS_X, R_VEL_X) = cosf(x[R_YAW]);
  a(R_POS_X, R_YAW) = -sinf(x[R_YAW]) * vx;
  a(R_POS_Y, R_VEL_X) = sinf(x[R_YAW]);
  a(R_POS_Y, R_YAW) = cosf(x[R_YAW]) * vx;
  const float steer_dot = (u[1] * p.steer_command_angle_scale - x[R_STEER_ANGLE]) * p.steering_constant;
  a(R_STEER_ANGLE, R_STEER_ANGLE) =
      (steer_dot - eps < -p.max_steer_rate || steer_dot + eps > p.max_steer_rate) ? 0.0f : -p.steering_constant;
  a(R_STEER_ANGLE, R_STEER_ANGLE) = fmaxf(fminf(a(R_STEER_ANGLE, R_STEER_ANGLE), p.max_steer_rate), -p.max_steer_rate);
  a(R_VEL_X, R_PITCH) = -p.gravity * cosf(x[R_PITCH]);
  const float brake_dot = (enable_brake * -u[0] - x[R_BRAKE_STATE]) * p.brake_delay_constant;
  a(R_BRAKE_STATE, R_BRAKE_STATE) =
      (brake_dot - eps < -p.max_brake_rate_neg || brake_dot + eps > p.max_brake_rate_pos) ? 0.0f : -p.brake_delay_constant;
  B[R_STEER_ANGLE * 2 + 1] = p.steer_command_angle_scale * p.steering_constant;
  B[R_VEL_X * 2 + 0] = p.c_t[index] * p.gear_sign * (!enable_brake);
  if ((x[R_BRAKE_STATE] < -p.lim.rng_lo[0] && brake_dot < 0.0f) || (x[R_BRAKE_STATE] > 0.0f && brake_dot > 0.0f))
    B[R_BRAKE_STATE * 2 + 0] = -p.brake_delay_constant * enable_brake;
  return MPPIB_OK;
}

int mppib_host_output_trajectory_racer_dubins_elevation(const void* dyn_params, const mppib_elevation_map_header* map,
                                                        const float* x0, const float* u, int T, float dt, float* states,
                                                        float* outputs)
{
  if (!dyn_params || !x0 || !u || !states || !outputs || T <= 0)
    return MPPIB_ERR_INVALID_ARG;
  return roll<RacerDubinsElevation>({ MPPIB_DYN_RACER_DUBINS_ELEVATION, dyn_params, nullptr, nullptr, map, nullptr }, x0,
                                    u, T, dt, states, outputs);
}

void mppib_host_normals_at_world_pose(const mppib_elevation_map_header* map, float x, float y, float z, float* out4)
{
  if (!out4)
    return;
  if (map)
    return normals_at_world_pose(map, x, y, z, out4);
  out4[0] = out4[1] = out4[3] = 0.0f;
  out4[2] = 1.0f;
}

int mppib_host_step_racer_suspension(const void* dyn_params, const mppib_host_lstm* net,
                                     const mppib_elevation_map_header* normals, const float* x, const float* u, float dt,
                                     float* x_next, float* xdot, float* y)
{
  if (!dyn_params || !net || !net->theta || !net->hidden || !net->cell || !x || !u || !x_next || !xdot || !y)
    return MPPIB_ERR_INVALID_ARG;
  return RacerSuspensionLstm::step({ MPPIB_DYN_RACER_SUSPENSION_LSTM, dyn_params, nullptr, net, net->map, normals }, x, u,
                                   dt, x_next, xdot, y);
}

int mppib_host_output_trajectory_racer_suspension(const void* dyn_params, const mppib_host_lstm* net,
                                                  const mppib_elevation_map_header* normals, const float* x0,
                                                  const float* u, int T, float dt, float* states, float* outputs)
{
  if (!dyn_params || !net || !net->theta || !x0 || !u || !states || !outputs || T <= 0)
    return MPPIB_ERR_INVALID_ARG;
  return roll<RacerSuspensionLstm>({ MPPIB_DYN_RACER_SUSPENSION_LSTM, dyn_params, nullptr, net, net->map, normals }, x0,
                                   u, T, dt, states, outputs);
}

int mppib_host_output_trajectory_lstm(const void* dyn_params, const mppib_host_lstm* net, const float* x0,
                                      const float* u, int T, float dt, float* states, float* outputs)
{
  if (!dyn_params || !net || !net->theta || !x0 || !u || !states || !outputs || T <= 0)
    return MPPIB_ERR_INVALID_ARG;
  return roll<RacerLstm>({ MPPIB_DYN_RACER_LSTM, dyn_params, nullptr, net, net->map, nullptr }, x0, u, T, dt, states,
                         outputs);
}

int mppib_host_state_deriv_racer_rigid_suspension(const void* dyn_params, const float* x, const float* u, float* xdot,
                                                  float* y, float* omega_jacobian)
{
  if (!dyn_params || !x || !u || !xdot || !y)
    return MPPIB_ERR_INVALID_ARG;
  rigid_suspension_deriv(*(const mppib_racer_rigid_suspension_dyn_params*)dyn_params, x, u, xdot, y, omega_jacobian);
  return MPPIB_OK;
}

int mppib_host_step_racer_rigid_suspension(const void* dyn_params, const float* x, const float* u, float dt, float* x_next,
                                           float* xdot, float* y)
{
  if (!dyn_params || !x || !u || !x_next || !xdot || !y)
    return MPPIB_ERR_INVALID_ARG;
  return RacerSuspension::step({ MPPIB_DYN_RACER_SUSPENSION, dyn_params, nullptr, nullptr, nullptr, nullptr }, x, u, dt,
                               x_next, xdot, y);
}

int mppib_host_output_trajectory_racer_rigid_suspension(const void* dyn_params, const float* x0, const float* u, int T,
                                                        float dt, float* states, float* outputs)
{
  if (!dyn_params || !x0 || !u || !states || !outputs || T <= 0)
    return MPPIB_ERR_INVALID_ARG;
  return roll<RacerSuspension>({ MPPIB_DYN_RACER_SUSPENSION, dyn_params, nullptr, nullptr, nullptr, nullptr }, x0, u, T,
                               dt, states, outputs);
}

// ---- RobustMPPI host logic (controllers/R-MPPI/robust_mppi_controller.cu) --------------------------------------------
void mppib_host_rmppi_line_search_weights(int num_candidates, float* out /*[3][K]*/)
{  // computeLineSearchWeights, :472-491
  const int K = num_candidates, h = K / 2;
  for (int i = 0; i < 3 * K; i++)
    out[i] = 0.0f;
  for (int i = 0; i < h + 1; i++)
  {
    out[0 * K + i] = 1 - i / float(h);
    out[1 * K + i] = i / float(h);
    out[2 * K + i] = 0.0;
  }
  for (int i = 1; i < h + 1; i++)
  {
    out[0 * K + h + i] = 0.0;
    out[1 * K + h + i] = 1 - i / float(h);
    out[2 * K + h + i] = i / float(h);
  }
}

void mppib_host_rmppi_candidates(int num_candidates, int S, const float* nominal_x_k, const float* nominal_x_kp1,
                                 const float* real_x_kp1, int stride, float* candidates /*[K][S]*/, int* strides /*[K]*/)
{  // getInitNominalStateCandidates :351-362 (points * line_search_weights) and computeImportanceSamplerStride :493-503
  std::vector<float> w(3 * (size_t)num_candidates);
  mppib_host_rmppi_line_search_weights(num_candidates, w.data());
  const int K = num_candidates;
  for (int k = 0; k < K; k++)
  {
    for (int i = 0; i < S; i++)
      candidates[(size_t)k * S + i] = nominal_x_k[i] * w[k] + nominal_x_kp1[i] * w[K + k] + real_x_kp1[i] * w[2 * K + k];
    strides[k] = (int)roundf(0.0f * w[k] + (float)stride * w[K + k] + (float)stride * w[2 * K + k]);
  }
}

int mppib_host_rmppi_best_index(const float* costs, int num_candidates, int samples_per_candidate, float lambda,
                                float value_func_threshold, int previous_best, float* free_energy /*[K] or NULL*/)
{  // computeCandidateBaseline + computeBestIndex, :505-537 (the LAST candidate under the threshold wins; if none does
   // best_index_ keeps its previous value)
  const int n = num_candidates * samples_per_candidate;
  float baseline = costs[0];
  for (int i = 1; i < n; i++)
    if (costs[i] < baseline)
      baseline = costs[i];
  int best = previous_best;
  for (int i = 0; i < num_candidates; i++)
  {
    float fe = 0.0f;
    for (int j = 0; j < samples_per_candidate; j++)
      fe += expf(-1.0 / lambda * (costs[i * samples_per_candidate + j] - baseline));
    fe /= (1.0 * samples_per_candidate);
    fe = -lambda * logf(fe) + baseline;
    if (free_energy)
      free_energy[i] = fe;
    if (fe < value_func_threshold)
      best = i;
  }
  return best;
}

void mppib_host_free_energy(const mppib_solve_stats* st, int num_rollouts, float lambda, float* out3)
{
  // core/mppi_common.cu:1065-1081 from (eta, sum w^2): norm = eta/N, var = sum w^2
  const float norm = st->normalizer / num_rollouts;
  out3[0] = -lambda * logf(norm) + st->baseline;
  out3[1] = lambda * (st->sum_w2 / num_rollouts - norm * norm);
  const float weird_term = out3[1] / (norm * sqrtf(1.0f * num_rollouts));
  out3[2] = lambda * (weird_term + 0.5f * weird_term * weird_term);
}


int mppib_host_merge_records(const float* records, int nrec, int D, int TC, int pstride, float lambda, int normalize,
                             float* out)
{
  // CPU twin of combine_kernel (csrc/combine_kernel.cuh): merges per-block or per-rank records
  // [beta_b, eta_b, sum w^2_b, -, V_b[TC]] with s_b = expf(-(beta_b - beta)/lambda). Used by launchers and tests that
  // reason about rollout sharding without a GPU; the engine itself always merges on the device.
  if (!records || !out || nrec <= 0 || D <= 0 || TC <= 0 || pstride < 4 + TC || !(lambda > 0.0f))
    return MPPIB_ERR_INVALID_ARG;
  const float lambda_inv = (float)(1.0 / lambda);
  for (int d = 0; d < D; d++)
  {
    const float* rec = records + (size_t)d * pstride;
    const size_t rstride = (size_t)D * pstride;
    float beta = rec[0];
    for (int b = 1; b < nrec; b++)
      beta = fminf(beta, rec[b * rstride]);
    double eta = 0.0, w2 = 0.0;
    std::vector<float> acc(TC, 0.0f);
    for (int b = 0; b < nrec; b++)
    {
      const float* r = rec + b * rstride;
      const float s = mppib::softmin_weight(r[0], beta, lambda_inv);  // 0 for an empty record (baseline +inf)
      eta += (double)s * (double)r[1];
      w2 += (double)s * (double)s * (double)r[2];
      for (int c = 0; c < TC; c++)
        acc[c] = fmaf(s, r[4 + c], acc[c]);
    }
    float* o = out + (size_t)d * pstride;
    o[0] = beta;
    o[1] = (float)eta;
    o[2] = (float)w2;
    o[3] = 0.0f;
    for (int c = 0; c < TC; c++)
      o[4 + c] = normalize ? acc[c] / (float)eta : acc[c];
  }
  return MPPIB_OK;
}

}  // extern "C"
