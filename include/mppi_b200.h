/*
 * mppi_b200.h — C ABI of libmppi_b200.so, the Hopper (sm_90a) MPPI rollout-and-reduce engine.
 *
 * This is the drop-in boundary for the reference's hot path (SURVEY.md §8b). The reference has no ABI: its
 * controllers call the templated launchers of include/mppi/core/mppi_common.cuh:206-247 plus the sampler methods of
 * include/mppi/sampling_distributions/sampling_distribution.cuh:367-401 directly. Templates cannot cross a C ABI, so
 * each entry point below names the reference interface it replaces; the header-only host layer
 * (the .hpp files under include/mppi_b200/, same class / method names as the reference) and the ctypes mirror
 * (mppi-generic_b200/host.py) are the only callers. INTEGRATION.md shows the binding a reference maintainer adds.
 *
 * Conventions: every function returns 0 on success or a negative mppib_status; nothing exit()s or throws across the
 * boundary (the reference's HANDLE_ERROR -> exit behaviour, include/mppi/utils/gpu_err_chk.cuh:32-40, is restored by
 * the host layer). Host arrays are caller-owned, plain float/int pointers; device memory, the cuRAND generator, streams
 * and the NCCL communicator are owned by the opaque engine. One engine = one caller thread at a time (same rule as
 * the reference: include/mppi/core/base_plant.hpp:464-468 serialises access with a mutex).
 *
 * Layouts (identical to the reference, SURVEY.md Appendix A):
 *   samples  [D][N][T][C]  ((N*d + n)*T + t)*C + c        sampling_distribution.cu:175-177
 *   costs    [D][N]        n + N*d                        mppi_common.cu:850
 *   means/U  [D][T][C]     (T*d + t)*C + c  == Eigen C x T column-major   gaussian.cu:494
 *   x0       [D][S]        S*d + i                        mppi_common.cu:781
 */
#ifndef MPPI_B200_H_
#define MPPI_B200_H_

#include <stddef.h>
#include "mppi_b200/params.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mppib_engine mppib_engine; /* opaque */

enum mppib_status
{
  MPPIB_OK = 0,
  MPPIB_ERR_INVALID_ARG = -1,
  MPPIB_ERR_UNSUPPORTED = -2, /* no kernel registered for (dynamics, cost, sampler, D) */
  MPPIB_ERR_CUDA = -3,        /* a CUDA runtime call failed; mppib_last_error() has the text */
  MPPIB_ERR_CURAND = -4,
  MPPIB_ERR_NO_DEVICE = -5, /* no CUDA device / driver: the engine never falls back to the CPU */
  MPPIB_ERR_NCCL = -6,
  MPPIB_ERR_SMEM = -7, /* horizon tile does not fit in shared memory (mirrors mppi_controller.cu:64-76 runtime_error) */
  MPPIB_ERR_CUFFT = -8,
  MPPIB_ERR_STATE = -9 /* call order violated (e.g. solve before blobs were set) */
};

enum mppib_blob
{
  MPPIB_BLOB_DYN_PARAMS = 0,  /* Dynamics::setParams + control ranges   dynamics.cuh:147-175 */
  MPPIB_BLOB_COST_PARAMS = 1, /* Cost::setParams                         cost.cuh:97-105      */
  MPPIB_BLOB_SAMPLER_PARAMS = 2, /* SamplingDistribution::setParams      sampling_distribution.cuh */
  MPPIB_BLOB_NN_WEIGHTS = 3,  /* NeuralNetModel::updateModel             ar_nn_model.cu:40-45 (packed W,b per layer) */
  MPPIB_BLOB_COSTMAP = 4,     /* ARStandardCost::costmapToTexture        ar_standard_cost.cu:145-184 (float4 texels) */
  MPPIB_BLOB_LSTM_WEIGHTS = 5, /* LSTMHelper weights                     lstm_helper.cu:72-88 */
  MPPIB_BLOB_ELEVATION_MAP = 6, /* RACER models: TwoDTextureHelper<float> map 0 (mppib_elevation_map_header + floats,
                                  params.h); optional — without it the ground is flat  racer_dubins.cu:359-434 */
  MPPIB_BLOB_COST_TEXTURE = 7,  /* QuadrotorMapCost: its tex_helper_ map 0, same format as MPPIB_BLOB_ELEVATION_MAP;
                                   optional — without it the costmap term is 0  quadrotor_map_cost.cu:359-395 */
  MPPIB_BLOB_NORMALS_MAP = 8    /* RacerDubinsElevationSuspension: normals_tex_helper_ map 0 (mppib_elevation_map_header +
                                   float4, params.h); optional — without it every normal is (0, 0, 1)
                                   racer_dubins_elevation_suspension_lstm.cu:288-295 */
};

/* Flags for mppib_desc.flags */
#define MPPIB_FLAG_WRITEBACK_CONTROLS 1u /* keep the constrained sampled controls in HBM like the reference does    \
                                            (mppi_common.cu:117); needed by mppib_get_samples */
#define MPPIB_FLAG_NO_TMA 2u             /* stage noise tiles with plain loads instead of cp.async.bulk.tensor */
#define MPPIB_FLAG_NO_PREFETCH 8u         /* draw each solve's noise inline instead of one solve ahead on a side stream */
#define MPPIB_FLAG_RMPPI 32u             /* RobustMPPI rollout semantics (core/rmppi_kernels.cu:665-866): requires                \
                                            num_distributions == 2 with distribution 0 = nominal, 1 = real system */
#define MPPIB_FLAG_NN_TENSOR 16u         /* Autorally NN: forward pass on wgmma tensor cores (3xTF32) */
#define MPPIB_FLAG_NN_MMA 64u            /* Autorally NN: forward pass with register-level mma.sync (FP16 hi/lo split, 3      \
                                            products, FP32 accumulate) — the default for that model */
#define MPPIB_FLAG_NN_FFMA2 128u         /* Autorally NN: forward pass as FP32 FFMA2s fed from shared memory (the round-1 form) */
#define MPPIB_FLAG_NO_WARP_SPEC 256u     /* Autorally pair: keep the generic one-thread-per-sample K1 instead of the warp-   \
                                            specialised producer / consumer kernel (rollout_kernel_ar_ws.cuh) */
#define MPPIB_FLAG_LSTM_SIMT 512u         /* RacerDubinsElevationLSTMSteering at hidden_dim 32: keep the one-thread-per-sample    \
                                            LSTM instead of the tensor-core form (plugins/lstm_mma.cuh) */
#define MPPIB_FLAG_CURAND_HOST_API 4u    /* draw with curandGenerateNormal (library) instead of the engine's own     \
                                            bit-identical XORWOW kernel */

typedef struct mppib_desc
{
  int dynamics_id;       /* enum mppib_dynamics_id */
  int cost_id;           /* enum mppib_cost_id */
  int sampler_id;        /* enum mppib_sampler_id */
  int num_rollouts;      /* N  (template NUM_ROLLOUTS in the reference) — GLOBAL count across all ranks */
  int num_timesteps;     /* T  (<= MAX_TIMESTEPS in the reference) */
  int num_distributions; /* D: 1 = VanillaMPPI, 2 = Tube-MPPI / RMPPI (blockDim.z in the reference) */
  int device;            /* CUDA device ordinal (the reference hard-codes 0, mppi_controller.cu:48) */
  unsigned flags;
  void* stream; /* cudaStream_t to run on (Controller::setCUDAStream, controller.cuh:901); NULL = engine-owned */
  /* rollout sharding across GPUs (SURVEY §8e). rank r owns samples [r*N/W, (r+1)*N/W). */
  int rank;
  int world_size;
  /* architecture arguments of the dynamics' constructor (not parameters): MPPIB_DYN_RACER_LSTM and
   * MPPIB_DYN_RACER_SUSPENSION_LSTM = { hidden_dim H, head hidden width L1 } (racer_dubins_elevation_lstm_steering.cu:11-22);
   * all zero for the other models. */
  int model_dims[8];
} mppib_desc;

/* Per-solve statistics for one distribution (getBaselineCost / getNormalizerCost, controller.cuh:510-517, and the
 * inputs of computeFreeEnergy, mppi_common.cu:1065-1081). */
typedef struct mppib_solve_stats
{
  float baseline;   /* beta = min_n cost */
  float normalizer; /* eta  = sum_n w_n */
  float sum_w2;     /* sum_n w_n^2 */
  float pad;
} mppib_solve_stats;

/* ---- lifetime ---------------------------------------------------------------------------------- */
/* Replaces Controller::Controller + allocateCUDAMemoryHelper + createAndSeedCUDARandomNumberGen
 * (controller.cuh:111-152, controller.cu:192-236) and the plugins' GPUSetup() (managed.cuh:121-131). */
int mppib_create(mppib_engine** out, const mppib_desc* desc);
/* Replaces Controller::~Controller / freeCudaMem (controller.cuh:194-216). */
int mppib_destroy(mppib_engine* e);

/* ---- configuration ----------------------------------------------------------------------------- */
/* Replaces <plugin>::setParams -> paramsToDevice (dynamics.cu:36-58, cost.cu:5-13, sampling_distribution.cu:52-70). */
int mppib_set_blob(mppib_engine* e, int which, const void* host, size_t nbytes);
/* Replaces Controller::setParams for the fields the device path uses (dt_, lambda_, alpha_; controller.cuh:46-68). */
int mppib_set_solver(mppib_engine* e, float dt, float lambda, float alpha);
/* Replaces Controller::setSeedCUDARandomNumberGen: seed and absolute offset (controller.cu:200-207 resets offset to 0). */
int mppib_seed(mppib_engine* e, unsigned long long seed, unsigned long long offset);
/* Consume n_generate_calls noise draws without using them — mirrors the draw made by
 * VanillaMPPIController::chooseAppropriateKernel (mppi_controller.cu:95) so RNG offsets stay in lock-step. */
int mppib_burn_draws(mppib_engine* e, int n_generate_calls);
/* Current absolute RNG offset in normals (checkpoint/resume: SURVEY §5). */
int mppib_get_rng_offset(mppib_engine* e, unsigned long long* offset);
/* MPPIB_SAMPLER_SMOOTH_MPPI: the rate mean [T][C] the sampler carries from solve to solve (deriv_action_mean_d_,
 * smooth-MPPI.cuh), zero at mppib_create. Each solve samples its rates around row min(optimization_stride, T - 1) and its
 * merge replaces the whole array; mppib_burn_draws broadcasts row min(1, T - 1). get returns it once the solves enqueued
 * so far are done; set while a solve is pending returns MPPIB_ERR_STATE. Other samplers: MPPIB_ERR_INVALID_ARG. */
int mppib_get_derivative_mean(mppib_engine* e, float* host);
int mppib_set_derivative_mean(mppib_engine* e, const float* host);
/* Join an NCCL communicator for world_size > 1. unique_id = the 128-byte ncclUniqueId created on rank 0 and
 * distributed by the caller (torch.distributed / MPI / a file). No reference counterpart (single GPU only). */
int mppib_comm_unique_id(void* unique_id_128);
int mppib_comm_init(mppib_engine* e, const void* unique_id_128);

/* ---- the hot path ------------------------------------------------------------------------------ */
/* One optimisation iteration of Controller::computeControl up to the new mean — replaces, in one call:
 *   cudaMemcpyAsync(initial_state_d_), copyNominalControlToDevice      mppi_controller.cu:157-165
 *   SAMPLING_T::generateSamples                                        gaussian.cu:375-431
 *   launchRolloutKernel / launchSplitRolloutKernel                     mppi_common.cu:1259-1325
 *   D2H costs, computeBaselineCost, launchNormExpKernel, computeNormalizer   mppi_controller.cu:187-208
 *   updateDistributionParamsFromDevice -> launchWeightedReductionKernel      gaussian.cu:434-457
 *   setHostOptimalControlSequence                                      gaussian.cu:460-478
 * x0 [D][S], U_in [D][T][C], U_out [D][T][C], stats [D] are host arrays. iteration_num scales std_dev by
 * std_dev_decay^iteration_num (gaussian.cu:423). Blocks until U_out is valid. */
/* Optional peer-memory exchange (world_size <= 8, one node): every rank exports the handle of its gather buffer
 * (64 bytes, a cudaIpcMemHandle_t), the launcher distributes all of them and every rank opens them. From then on a solve
 * merges the ranks' records with ONE kernel that stores to / polls NVLink peer memory instead of ncclAllGather + two
 * launches. Call after mppib_comm_init (NCCL stays the fallback if peer access is not possible). */
int mppib_comm_p2p_handle(mppib_engine* e, void* handle_64);
int mppib_comm_p2p_open(mppib_engine* e, const void* handles_world_x_64);

int mppib_solve(mppib_engine* e, const float* x0, const float* U_in, int optimization_stride, int iteration_num,
                float* U_out, mppib_solve_stats* stats);

/* Pipelined variant: mppib_solve_async enqueues the same work (x0 / U_in are captured into the kernel parameter bank at
 * call time, so the host arrays may be reused immediately) and returns without waiting; mppib_solve_wait blocks until
 * everything enqueued so far is done and returns the result of the LAST solve. mppib_solve == async + wait. */
int mppib_solve_async(mppib_engine* e, const float* x0, const float* U_in, int optimization_stride, int iteration_num);
int mppib_solve_wait(mppib_engine* e, float* U_out, mppib_solve_stats* stats);

/* Kernel-level parity hooks (the reference tests kernels in isolation: tests/mppi_core/rollout_kernel_tests.cu). */
/* mppib_set_noise: overwrite the raw N(0,1) buffer [N_local][T][C] from the host (tests with hand-made noise).
 * mppib_draw_noise: one generateSamples-equivalent draw into the buffer, advancing the RNG offset.
 * mppib_rollout_only: launchRolloutKernel on the current buffer; no draw. costs -> mppib_get_costs. */
int mppib_set_noise(mppib_engine* e, const float* host_eps, size_t count);
int mppib_draw_noise(mppib_engine* e);
int mppib_rollout_only(mppib_engine* e, const float* x0, const float* U_in, int optimization_stride,
                       int iteration_num);
/* mppib_reduce_only: baseline / weights / weighted average over the costs and samples of the last rollout. */
int mppib_reduce_only(mppib_engine* e, float* U_out, mppib_solve_stats* stats);

/* ---- read-backs (getSampledCostSeq controller.cuh:431-436, getSampledNoise :778) ---------------- */
int mppib_get_costs(mppib_engine* e, float* host_costs /*[D][N_local]*/);
int mppib_get_noise(mppib_engine* e, float* host_eps /*[N_local][T][C] raw N(0,1)*/);
int mppib_get_samples(mppib_engine* e, float* host_samples /*[D][N_local][T][C]; needs WRITEBACK_CONTROLS*/);
/* importance-sampling weights w_n = exp(-(c_n - beta)/lambda) of the last solve (trajectory_costs_d_ after
 * launchNormExpKernel in the reference). */
int mppib_get_weights(mppib_engine* e, float* host_weights /*[D][N_local]*/);

/* ---- introspection / timing -------------------------------------------------------------------- */
typedef struct mppib_timing
{
  float noise_ms;   /* K0 draw */
  float rollout_ms; /* K1 fused rollout */
  float reduce_ms;  /* K2 combine (+ collective) */
  float total_ms;   /* first launch to last kernel end, device time */
  int samples;      /* synchronous solves averaged */
} mppib_timing;
/* Enable CUDA-event timestamps around each stage of subsequent solves (adds ~us; off by default); mppib_get_timing
 * returns the averages since the last enable call over the solves enqueued while timing was on, each counted when it is
 * waited for with timing still on (with several solves in flight, only the last). */
int mppib_enable_timing(mppib_engine* e, int enable);
int mppib_get_timing(mppib_engine* e, mppib_timing* out);
/* Launch geometry actually used by K1 (for bench.py / DESIGN.md). */
int mppib_get_launch_info(mppib_engine* e, int* grid, int* block, int* smem_bytes, int* uses_tma,
                          int* kernels_per_solve);
/* 1 if the engine's own XORWOW kernel draws the noise, 0 if curandGenerateNormal does (sizes / flag); chunks = K. */
int mppib_get_rng_info(mppib_engine* e, int* own_kernel, int* chunks, int* rounds_per_chunk);
int mppib_local_rollouts(mppib_engine* e, int* n_local, int* n_offset);

/* Measurement options. MPPIB_OPT_L2_FLUSH_BYTES: if > 0, a buffer of that many bytes is overwritten between the noise
 * draw and the rollout so K1 reads its tile from HBM instead of the L2 lines K0 just wrote (roofline measurements). */
enum mppib_option
{
  MPPIB_OPT_L2_FLUSH_BYTES = 1,
  /* ColoredNoise: the optimization_stride (rearrangeNoise's offset_t, colored_noise.cu:39-56) assumed by draws that
   * are issued before a solve names its own: mppib_draw_noise and the one-solve-ahead prefetch. Default 1. */
  MPPIB_OPT_COLORED_OFFSET_T = 2,
  /* 0 = go back to the NCCL all-gather after mppib_comm_p2p_open (a launcher sets it on EVERY rank when any rank failed
   * to open its peers' buffers: the two exchange paths cannot be mixed), 1 = use the peer-memory exchange again. */
  MPPIB_OPT_P2P_ENABLE = 3
};
int mppib_set_option(mppib_engine* e, int option, long long value);

/* ColoredMPPIController's alternative weighting (ColoredMPPI/colored_mppi_controller.cu:199-209): when gamma and r are
 * both non-zero the exp weights are replaced by TsallisTransform (core/mppi_common.cu:968-985). Needs an engine created
 * with MPPIB_FLAG_WRITEBACK_CONTROLS on one rank; gamma = 0 or r = 0 switches back to the exponential weights. */
int mppib_set_tsallis(mppib_engine* e, float gamma, float r);

/* ---- RMPPI (engines created with MPPIB_FLAG_RMPPI) ------------------------------------------------------------- */
/* RobustMPPIController::setValueFunctionThreshold + fb_controller_->copyToDevice (robust_mppi_controller.cu:630-633):
 * feedback_gains = the DDP gain trajectory, T matrices C x S column-major ([t][s][c]), or NULL for no feedback. */
int mppib_set_rmppi(mppib_engine* e, float value_func_threshold, const float* feedback_gains);
/* computeNominalStateAndStride's device part (robust_mppi_controller.cu:581-617): draws one noise block with
 * `optimization_stride` (generateSamples) and evaluates num_candidates nominal-state candidates x samples_per_candidate
 * rollouts of the nominal control U_nominal [T][C], candidate k replaying the controls shifted by strides[k]
 * (launchInitEvalKernel, core/rmppi_kernels.cu:230-356). costs_out [num_candidates * samples_per_candidate]. A negative
 * stride is refused with MPPIB_ERR_INVALID_ARG before any noise is drawn. */
int mppib_init_eval(mppib_engine* e, const float* candidates, const int* strides, int num_candidates,
                    int samples_per_candidate, const float* U_nominal, int optimization_stride, float* costs_out);

/* ---- DDP feedback (Tube-MPPI / RMPPI ancillary controller) ----------------------------------------------------- */
/* DDPFeedback::setParams (feedback_controllers/DDP/ddp.cu:69-76) with DDPParams (DDP/ddp.cuh:16-26): tracking weights
 * Q [S][S], Q_f [S][S], R [C][C] (row-major) and the iteration count. Until called: Q = Q_f = I, R = I, 1 iteration. */
int mppib_set_ddp(mppib_engine* e, const float* Q, const float* Q_f, const float* R, int num_iterations);
/* DDPFeedback::computeFeedback (ddp.cu:80-118): DDP::run (ddp/ddp.h:56-168) from x0 [S] around the targets x_target [T][S],
 * u_target [T][C] (also the initial controls), with the engine's dt, the model's control ranges and the weights of
 * mppib_set_ddp. One CTA on the engine's stream; T is independent of the engine's horizon. Outputs (each may be NULL):
 *   gains [T][S][C]         fb_gain_traj_: K_t, C x S column-major per step; K_{T-1} = 0
 *   x_out [T][S], u_out [T][C]   the final state / control trajectory (result_.state_trajectory / control_trajectory)
 *   jac_out [T][S][S+C]     [A | B] = d f / d(x, u) of the model's computeGrad at the trajectory the last backward pass
 *                           linearised around (df = I + dt [A | B])
 * to_rmppi = 1 (engines with MPPIB_FLAG_RMPPI, T == the horizon): the kernel also writes the gains into the engine's
 * feedback-gain buffer, so the next RMPPI solve applies them with no host copy (robust_mppi_controller.cu:629-632).
 * MPPIB_ERR_UNSUPPORTED for dynamics without an analytic Jacobian (the RACER LSTM pair, plugins). A failed LDLT of Q_uu
 * (the reference exits, ddp.h:112-116) returns MPPIB_ERR_INVALID_ARG and leaves every gain buffer untouched. */
int mppib_ddp_feedback(mppib_engine* e, int T, const float* x0, const float* x_target, const float* u_target, int to_rmppi,
                       float* gains, float* x_out, float* u_out, float* jac_out);

/* ---- sampled (visualisation) trajectories ---------------------------------------------------------------------- */
/* VanillaMPPIController::calculateSampledStateTrajectories (controllers/MPPI/mppi_controller.cu:262-298) /
 * launchVisualizeKernel (core/mppi_common.cu:364-520, 1376-1420): after a solve, re-rolls the rollouts the host picked
 * (controllers/controller.cu:55-179: the optimised sequence, a random subset, the top-n by weight) and returns every
 * step's output, cost and crash flag. Needs MPPIB_FLAG_WRITEBACK_CONTROLS (the constrained controls of the last solve
 * are the input) and no solve in flight; not available on RMPPI engines.
 *   x0 [S], U_nominal [T][C]   what that solve was called with, for system `distribution`
 *   sample_idx [n]             rank-local rollout indices in [0, n_local), or -1 = roll out U_opt [T][C]
 *                              (the optimised sequence; control constraints are applied to it)
 *   outputs [n][T][O]          y after step t (the reference keeps the first T - 1 rows)
 *   costs   [n][T + 1]         [t] = (state cost + likelihood-ratio cost of step t) / T, [T] = terminal cost / T: a row
 *                              of a stored rollout sums to its trajectory cost (mppib_get_costs)
 *   crash   [n][T]             the sticky crash flag after step t */
int mppib_sample_trajectories(mppib_engine* e, const float* x0, const float* U_nominal, int distribution,
                              const int* sample_idx, int n, const float* U_opt, float* outputs, float* costs, int* crash);

/* One iteration of Controller::computeControl (controllers/MPPI/mppi_controller.cu:151-241) as ONE call: mppib_solve, then the
 * host tail on the result with the parameter blobs the engine holds — smoothControlTrajectory (controllers/controller.cuh:
 * 557-586) and computeStateTrajectory (:643-663) through the library's host twins (host_twins.h).
 *   U_inout [D][T][C]          in: nominal control, out: the optimised (and, with a history, smoothed) control
 *   control_history [2][C]     or NULL = no smoothing
 *   states [D][T][S], outputs [D][T][O]   the nominal roll-forward; both NULL = skip it (user dynamics registered by a plugin
 *                              have no host twin here: MPPIB_ERR_UNSUPPORTED unless both are NULL)
 * The header-only controllers keep calling mppib_solve and the host twins separately (their virtual hooks sit in between);
 * this entry point is for C callers and language bindings, where every call across the boundary costs. */
int mppib_compute_control(mppib_engine* e, const float* x0, float* U_inout, int optimization_stride, int iteration_num,
                          const float* control_history, float* states, float* outputs, mppib_solve_stats* stats);

/* Device-side host tail (SURVEY §8 f2): Controller::smoothControlTrajectoryHelper (controllers/controller.cuh:557-586) and
 * computeOutputTrajectoryHelper (:643-663) as one kernel on the solve's stream — Savitzky-Golay smoothing of the control
 * sequence and the nominal state / output roll-forward (T - 1 step() calls with the constrained controls).
 *   x0 [D][S]
 *   U  [D][T][C] host, or NULL = the optimised sequence of the last solve, read on the device from the result record
 *                (may be called right after mppib_solve_async: the kernel is ordered behind the solve, and this call's
 *                single wait then covers the whole computeControl; mppib_solve_wait afterwards returns at once)
 *   control_history [2][C], or NULL = no smoothing (the controls are only copied)
 *   U_smoothed [D][T][C] (may be NULL), states [D][T][S], outputs [D][T][O]   row 0 = x0 / the initial output
 * A T-step dependent chain on ONE thread per system: slower than the library's vectorised host twins
 * (mppib_host_output_trajectory), which stay the default of the controller mirrors; see DESIGN.md §9. */
int mppib_nominal_trajectory(mppib_engine* e, const float* x0, const float* U, const float* control_history,
                             float* U_smoothed, float* states, float* outputs);

/* ---- user plugins ----------------------------------------------------------------------------------------------------
 * The reference's plugin contract is "compile your Dynamics / Cost class against the templates" (dynamics.cuh:67-76,
 * cost.cuh:34-35, utils/managed.cuh:109-135). Here a user pair is compiled into a SECOND shared library from
 * mppi-generic_b200/csrc/engine_internal.cuh (device twins with the static methods of csrc/plugins/dynamics.cuh / costs.cuh;
 * see plugins_example/ and INTEGRATION.md E) whose `int mppib_plugin_init(void)` registers it; engines are then created with
 * its ids (>= MPPIB_USER_ID_BASE) and its POD parameter structs go through mppib_set_blob like the built-in ones.
 * mppib_load_plugin = dlopen + mppib_plugin_init. mppib_register_pair is what the plugin calls (through register_pair<>). */
#define MPPIB_USER_ID_BASE 1000
int mppib_load_plugin(const char* path);
int mppib_register_pair(const void* pair_entry, size_t entry_bytes, unsigned abi);

const char* mppib_strerror(int status);
const char* mppib_last_error(void); /* thread-local text of the last failure */
int mppib_version(void);

#ifdef __cplusplus
}
#endif
#endif /* MPPI_B200_H_ */
