// SPDX-License-Identifier: Apache-2.0
//
// upkie_b200.cu -- sm_90a kernels and the C ABI of include/upkie_b200.h.
//
// Kernels (one thread = one robot, state struct-of-arrays, model in the kernel
// parameter constant bank):
//   k_step<MODE>   one 5 ms env tick: action front-end, 5 x (moteus torque law,
//                  articulated-body dynamics, wheel-ground contact solve,
//                  semi-implicit integration), observation, termination; optional
//                  fused auto-reset.
//   k_reset        masked reset: set state, one physics substep, observe; the randomisations' per-env state restarts.
//   k_spine_obs    spine observations of the state, or of the same-step auto-resets' terminal step from the stash.
//   k_ring_copy    rows <-> struct-of-arrays columns of every per-env buffer, and the delay histories.
//   k_history_read / k_history_fill   the observation history's entries of each env / its ring filled from the state.
// The servo dropouts' held rows take no kernel of their own: k_reset latches, k_ring_copy copies them for checkpoints,
// and a new spec or set_state latches the state with device copies of its rows (servo_dropout_latch).
// The IMU misalignment takes none either: k_reset draws, k_ring_copy copies its quaternions for checkpoints, and
// k_spine_obs, k_reset_obs and k_history_fill read the orientation through it (imu_misalign_observed). Neither do the
// encoder offsets: k_reset draws and shifts the leg targets, and the same three kernels read the servo positions
// through them (encoder_offset_observed). Nor does the servo noise: k_reset draws, noises the leg targets, the latch
// and the history refill, and the same three kernels read the servo replies through it (servo_noise_observed). The
// servo velocity limits touch the torque law only: k_reset draws, and the step kernels' substeps derate. The attitude
// filter has one, k_attitude_init (a new filter, set_state): k_reset draws and initialises, and k_spine_obs,
// k_reset_obs and k_history_fill report the estimate (attitude_observed). The torque scales touch the physics only:
// k_reset draws, and the step kernels' substeps scale the torque integrated.
// MPC kernels live in mpc.cuh, the UpkieBaseVelocity epilogue (k_base_velocity_post) in base_velocity.cu.
//
// There is deliberately NO CPU path in this library: every entry point needs a
// CUDA device and fails with UPKIE_B200_ECUDA otherwise.

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "mpc.cuh"
#include "base_velocity.cuh"
#include "controllers.cuh"
#include "observers.cuh"
#include "kernel_common.cuh"
#include "params.h"

using namespace upkie_b200;

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

#define CUDA_TRY(expr)                                                                        \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) return fail(UPKIE_B200_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

struct Handle {
  uint32_t magic;
  int n, n_pad, device;
  SimParams P;
  UpkieModel model;            // kept for upkie_b200_set_config
  float* state = nullptr;      // [STATE_DIM][n_pad]
  float* eps = nullptr;        // [n][6] or null
  float* mu = nullptr;         // [n] or null
  uint32_t* err = nullptr;     // [n]
  uint8_t* done_prev = nullptr;  // [n]
  uint32_t* episode = nullptr;   // [n]
  uint32_t* bv_episode = nullptr;  // [n] episode as of the last upkie_b200_base_velocity_post: which envs reset since
  uint32_t* tick = nullptr;      // [n] env ticks since create: counter of the noise generator
  uint32_t* elapsed = nullptr;   // [n] agent steps since the env's last reset (config.max_episode_steps)
  float* ext = nullptr;          // [7 * 3][n_pad] external forces, null = none
  float* lag = nullptr;          // [UPKIE_LAG_DIM][n_pad] spine-mode lag records (config.spine_mode), else null
  float* body_rec = nullptr;     // [UPKIE_BODY_REC_DIM][n_pad] body-ground contacts of the last substep (config.body_contacts)
  float* env_params = nullptr;   // [UPKIE_EP_DIM][n_pad] per-env parameter table (upkie_b200_set_env_params), else null
  uint32_t env_param_flags = 0;  // env_row_flags of the table, OR-ed over its rows
  uint32_t config_flags = 0;     // noise_flags of the config (restored when the table is dropped)
  uint32_t* ep_check = nullptr;  // [1] device word of the table validation
  uint32_t ext_local = 0;
  int autoreset = AUTORESET_DISABLED;
  uint64_t seed = 0, env_offset = 0;
  int block = UPKIE_DEFAULT_BLOCK;
  int num_sms = 0;               // cudaDevAttrMultiProcessorCount, read at create
  int host_chunks = 2;           // chunks of the pipelined host-buffer step (tools/e2e_parts.py sweeps 2..16)
  uint64_t step_launches = 0;    // step kernels launched (upkie_b200_launch_count)
  int host_block = 128;          // zero-copy step: persistent blocks of 4 warps, one per SM: ~3.5 tiles per block at
  int host_blocks_per_sm = 1;    // 65536 envs, so PCIe reads of tile k+1 overlap the compute of tile k
  int zero_copy = 2;             // pinned host buffers: 0 staged copies, 1 kernel reads+writes host memory, 2 hybrid
  int smem_carveout = cudaSharedmemCarveoutMaxL1;  // step kernels' preferred carveout, % (-1: the driver's choice)
  // host-buffer staging (allocated on first use)
  float *h_act = nullptr, *h_obs = nullptr, *h_rew = nullptr;
  uint8_t *h_term = nullptr, *h_trunc = nullptr;
  float *d_act = nullptr, *d_obs = nullptr, *d_rew = nullptr;
  uint8_t *d_term = nullptr, *d_trunc = nullptr;
  float* h_fin = nullptr;        // pinned copy of a pageable final_obs buffer (allocated on first use)
  // same-step terminal spine observations (UpkieStepOutputs.final_state, upkie_b200_final_spine_obs): the stash
  // [kFinalRows or kFinalRowsSpine][n_pad] (allocated on the first request), the number of the last step that asked for
  // it, and whether that step is the last call that advanced or reset the simulator
  float* final_state = nullptr;
  int final_rows = 0;            // rows of the stash allocated (kFinalParamCols more with reset randomisation)
  uint32_t final_gen = 0;
  bool final_valid = false;
  bool final_params = false;     // the stashing step ran with reset randomisation: the stash holds the table columns
  // reset randomisation (upkie_b200_set_reset_randomization): the device block P.reset_rand points to while a spec is
  // set, the per-env draw counters (allocated on the first spec or set_draws), and the noise flags the spec implies
  ResetRand* rr_dev = nullptr;
  uint32_t* draws = nullptr;
  uint32_t rr_flags = 0;
  // push randomisation (upkie_b200_set_push_randomization): the device block P.push points to while a spec is set, and
  // the per-env schedule state (allocated on the first spec or set_push_state)
  PushRand* push_dev = nullptr;
  uint32_t* push_count = nullptr;
  uint32_t* push_timer = nullptr;
  int push_body = 0;             // the body of the spec in force
  // action-delay randomisation (upkie_b200_set_action_delay): the device block P.action_delay points to while a spec
  // is set, and the per-env state (allocated on the first spec or set_action_delay_state)
  ActionDelay* delay_dev = nullptr;
  uint32_t* delay_count = nullptr;
  uint32_t* delay_delay = nullptr;
  float* delay_command = nullptr;  // [delay_ticks][UPKIE_ACT_DIM][n_pad], a ring of the last delay_ticks commands
  uint32_t* delay_head = nullptr;  // the ring row each env's next tick writes
  uint32_t delay_high = 0;         // substeps_high of the spec in force
  int delay_ticks = 1;             // the history depth (upkie_b200_set_action_delay_ticks)
  // observation-delay randomisation (upkie_b200_set_observation_delay): the device block P.obs_delay points to while a
  // spec is set, and the per-env state (allocated on the first spec or set_observation_delay_state)
  ObsDelay* sense_dev = nullptr;
  uint32_t* sense_count = nullptr;
  uint32_t* sense_delay = nullptr;
  float* sense_rows = nullptr;     // [UPKIE_STATE_DIM][n_pad] sensed states
  uint32_t sense_high = 0;         // substeps_high of the spec in force
  int sense_ticks = 1;             // the history depth (upkie_b200_set_observation_delay_ticks)
  float* sense_hist = nullptr;     // sense_ticks > 1: [sense_ticks][UPKIE_STATE_DIM][n_pad], a ring of snapshots
  uint32_t* sense_head = nullptr;  // the ring row each env's next tick writes
  // spine-rate observation history (upkie_b200_set_history): the device block P.history points to while a spec is set,
  // and its ring [hist_ticks][spec.count][n_pad] and per-env heads (allocated with the spec, freed when it is turned off)
  History* hist_dev = nullptr;
  UpkieHistory hist_spec = {};
  int hist_ticks = 0;
  float* hist_ring = nullptr;
  uint32_t* hist_head = nullptr;
  // servo reply dropouts (upkie_b200_set_servo_dropout): the device block P.servo_dropout points to while a spec is set,
  // and the per-env state it points to (allocated with the first spec, freed when it is turned off)
  ServoDropout* drop_dev = nullptr;
  uint32_t* drop_count = nullptr;
  float* drop_prob = nullptr;
  float* drop_held = nullptr;  // [kServoHeldRows][n_pad]
  uint32_t drop_mask = 0;      // joint_mask of the spec in force
  // IMU mounting misalignment (upkie_b200_set_imu_misalignment): the device block P.imu_misalign points to while a spec
  // is set, and the per-env state it points to (allocated with the first spec, freed when it is turned off)
  ImuMisalign* tilt_dev = nullptr;
  uint32_t* tilt_count = nullptr;
  float* tilt_quat = nullptr;  // [4][n_pad], e_i (w, x, y, z)
  // servo encoder zero offsets (upkie_b200_set_encoder_offset): the device block P.encoder_offset points to while a spec
  // is set, and the per-env state it points to (allocated with the first spec, freed when it is turned off)
  EncoderOffset* enc_dev = nullptr;
  uint32_t* enc_count = nullptr;
  float* enc_offset = nullptr;  // [UPKIE_NJ][n_pad], delta_i
  uint32_t enc_mask = 0;        // joint_mask of the spec in force
  // servo measurement noise (upkie_b200_set_servo_noise): the device block P.servo_noise points to while a spec is set,
  // and the per-env state it points to (allocated with the first spec, freed when it is turned off)
  ServoNoise* noise_dev = nullptr;
  uint32_t* noise_count = nullptr;
  float* noise_sigma = nullptr;  // [12][n_pad], sigma_i
  uint8_t* noise_fresh = nullptr;
  UpkieServoNoise noise_spec{};  // the spec in force
  // servo velocity limits (upkie_b200_set_velocity_derate): the device block P.velocity_derate points to while a spec
  // is set, and the per-env state it points to (allocated with the first spec, freed when it is turned off)
  VelocityDerate* vlim_dev = nullptr;
  uint32_t* vlim_count = nullptr;
  float* vlim_max = nullptr;  // [UPKIE_NJ][n_pad], v_i
  uint32_t vlim_mask = 0;     // joint_mask of the spec in force
  // IMU attitude estimation (upkie_b200_set_attitude_filter): the device block P.attitude_filter points to while a spec
  // is set, and the per-env state it points to (allocated with the first spec, freed when it is turned off)
  AttitudeFilter* att_dev = nullptr;
  uint32_t* att_count = nullptr;
  float* att_gains = nullptr;  // [2][n_pad] kp, ki
  float* att_quat = nullptr;   // [4][n_pad] q_i
  float* att_bias = nullptr;   // [3][n_pad] b_i
  float* att_rep = nullptr;    // [4][n_pad] the estimate the observation reports under an observation delay
  float* att_vel = nullptr;    // [3][n_pad] the step kernels' last-substep IMU velocity
  UpkieAttitudeFilter att_spec{};  // the spec in force
  // servo torque-constant errors (upkie_b200_set_torque_scale): the device block P.torque_scale points to while a spec
  // is set, and the per-env state it points to (allocated with the first spec, freed when it is turned off)
  TorqueScale* tsc_dev = nullptr;
  uint32_t* tsc_count = nullptr;
  float* tsc_scale = nullptr;  // [UPKIE_NJ][n_pad], s_i
  uint32_t tsc_mask = 0;       // joint_mask of the spec in force
  cudaStream_t host_streams[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t host_events[64] = {};
  int host_kernel_streams = 1;
  double host_split[8] = {};
  int host_split_n = 0;   // hybrid host step: kernels of successive chunks alternate over this many streams
};
constexpr int kHostStreams = 3;  // H2D, kernel and D2H of different chunks overlap
constexpr uint32_t kMagic = 0x55504B42u;  // "UPKB"

Handle* as_handle(void* h) {
  Handle* p = static_cast<Handle*>(h);
  return (p && p->magic == kMagic) ? p : nullptr;
}

// ---- masked reset ------------------------------------------------------------------
// The envs the reset takes (mask, NULL = all) restart from `init_state` rows or from a sampled state (keyed on `seed`,
// `env_offset`), and the per-env state of every randomisation the handle runs restarts with them, in the per-lane
// functions of the step kernels' fused resets. Those draws are keyed on the auto-reset's seed and env offset
// (`rand_seed`, `rand_offset`), whatever init rows the reset takes.
__device__ void attitude_history_observed(const SimParams& P, int i, const History& H);

__global__ void __launch_bounds__(128)
k_reset(const __grid_constant__ SimParams P, int n, int n_pad, float* __restrict__ state,
        const uint8_t* __restrict__ mask, const float* __restrict__ init_state, const float* __restrict__ eps_all,
        const float* __restrict__ mu_all, uint32_t* __restrict__ err, uint8_t* __restrict__ done_prev,
        uint32_t* __restrict__ episode, uint64_t seed, uint64_t env_offset, float* __restrict__ lag,
        uint64_t rand_seed, uint64_t rand_offset, const uint32_t* __restrict__ tick) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mask && !mask[i]) return;
  const uint64_t g = rand_offset + uint64_t(i);
  RobotState S;
  load_state(state, n_pad, i, S);
  float epsv[6];
  const float* eps = nullptr;
  if (eps_all) {
#pragma unroll
    for (int k = 0; k < 6; ++k) epsv[k] = eps_all[size_t(i) * 6 + k];
    eps = epsv;
  }
  float mu = mu_all ? mu_all[i] : P.friction;
  // reset randomisation (the handle then holds eps_all and mu_all): the reset substep runs with the drawn epsilons and
  // friction, taken from the draw in registers and not read back from eps_all and mu_all (the reset substep reads no
  // parameter table)
  if (P.reset_rand) {
    const ResetRand& R = *P.reset_rand;
    float v[UPKIE_RR_DIM];
    reset_rand_draw(R.spec, rand_seed, g, R.draws[i] + 1u, v);
    const uint64_t cols = R.spec.columns;
#pragma unroll
    for (int b = 0; b < 6; ++b)
      if ((cols >> (UPKIE_RR_INERTIA + b)) & 1u) epsv[b] = v[UPKIE_RR_INERTIA + b];
    if ((cols >> UPKIE_RR_FRICTION) & 1u) mu = v[UPKIE_RR_FRICTION];
    reset_rand_store(R, i, v);
  }
  if (P.push) push_reset(*P.push, rand_seed, g, i);  // a new schedule
  if (P.action_delay) {  // the next delay, and the stop row as every previous command (the ring head stays)
    action_delay_reset(*P.action_delay, rand_seed, g, i);
    action_delay_fill_history(*P.action_delay, i);
  }
  float init[UPKIE_INIT_DIM];
  if (init_state) {
#pragma unroll
    for (int k = 0; k < UPKIE_INIT_DIM; ++k) init[k] = init_state[size_t(i) * UPKIE_INIT_DIM + k];
  } else {
    const uint32_t ep = episode[i] + 1u;
    episode[i] = ep;
    sample_init_state(P, seed, env_offset + uint64_t(i), uint64_t(ep), init);
  }
  const BodyRecOut br{P.body_rec ? P.body_rec + i : nullptr, size_t(P.body_rec_stride)};
  if (P.spine_mode && lag) {
    SpineLag L;
    reset_robot_spine(P, S, L, init, eps, mu, WarpAny(), P.joint_limits, br);
    float lr[UPKIE_LAG_DIM];
    lag_to_row(L, lr);
    for (int k = 0; k < UPKIE_LAG_DIM; ++k) lag[size_t(k) * n_pad + i] = lr[k];
  } else {
    reset_robot(P, S, init, eps, mu, WarpAny(), P.joint_limits, br);
  }
  // the servo noise's and the encoder offsets' next draws: the new episode's leg targets are its reported leg
  // positions, the reset observation's (the noise, then the offsets)
  Noise12 nd;
  uint64_t rcyc = 0;  // the reset observation's cycle, keyed on the new draw
  if (P.servo_noise) {
    const ServoNoise& N = *P.servo_noise;
    rcyc = servo_noise_reset_cycle(servo_noise_reset(N, rand_seed, g, i));
    nd = servo_noise_increments([&](int c) { return N.sigma[size_t(c) * size_t(N.stride) + size_t(i)]; }, rand_seed, g,
                                rcyc);
    servo_noise_leg_targets(S, nd);
  }
  if (P.velocity_derate) velocity_derate_reset(*P.velocity_derate, rand_seed, g, i);  // the new episode's v_i
  if (P.torque_scale) torque_scale_reset(*P.torque_scale, rand_seed, g, i);           // and s_i
  Offset6 d{{0.f, 0.f, 0.f, 0.f, 0.f, 0.f}};
  if (P.encoder_offset) {
    d = encoder_offset_reset(*P.encoder_offset, rand_seed, g, i);
    encoder_offset_leg_targets(S, d);
  }
  store_state(state, n_pad, i, S);
  err[i] = 0;
  done_prev[i] = 0;
  P.elapsed[i] = 0;
  if (P.obs_delay) {
    // the next delay, and the post-reset state as the sensed row and every snapshot: the reset is observed undelayed
    const ObsDelay& O = *P.obs_delay;
    obs_delay_reset(O, rand_seed, g, i);
    float r[UPKIE_STATE_DIM];
    state_to_row(S, r);
    float* const col = O.rows + size_t(i);
    for (int k = 0; k < UPKIE_STATE_DIM; ++k) col[size_t(k) * size_t(O.stride)] = r[k];
    if (O.ticks > 1) obs_delay_fill_history(O, i, r);
  }
  // the misalignment's next draw, before the history: the new episode is observed through it
  Quat4 e{{1.f, 0.f, 0.f, 0.f}};
  if (P.imu_misalign) e = imu_misalign_reset(*P.imu_misalign, rand_seed, g, i);
  if (P.attitude_filter) {  // the attitude filter's next draw and the new episode's estimate, before the history
    RobotState V = S;
    imu_misalign_view(V, e);
    attitude_filter_reset(*P.attitude_filter, rand_seed, g, i, V);
  }
  if (P.history) {  // a new episode's history starts from its post-reset columns
    const History& H = *P.history;
    if (P.servo_noise) {  // each entry with the noise of its cycle, the newest the reset observation's
      const ServoNoise& N = *P.servo_noise;
      history_fill_noise(
          H, P, S, H.head[i], [&](int c) { return N.sigma[size_t(c) * size_t(N.stride) + size_t(i)]; }, rand_seed, g,
          rcyc, tick[i],
          [&](RobotState& V) {
            imu_misalign_view(V, e);
            encoder_offset_view(V, d);
          },
          [&](uint32_t en, int c, float v) {
            H.ring[(size_t(en) * size_t(H.count) + size_t(c)) * size_t(H.stride) + size_t(i)] = v;
          });
    } else {
      RobotState V = S;
      imu_misalign_view(V, e);
      encoder_offset_view(V, d);
      history_fill(H, P, V, i);
    }
    attitude_history_observed(P, i, H);
  }
  if (P.servo_dropout) {  // a new p_i, the reset latched (its replies as the reset observation reports them)
    RobotState V = S;
    if (P.servo_noise) servo_noise_view(V, nd);
    servo_dropout_reset(*P.servo_dropout, rand_seed, g, i, V);
  }
}

// The attitude filter: the orientation-derived columns of env i's spine observation o reported from its estimate (`q`:
// rows [4][n_pad] of estimates, the block's own by default: the report under an observation delay, the estimate
// otherwise), and those columns of every entry of its history
__device__ void attitude_observed(const SimParams& P, int i, float* o, const float* q = nullptr, int n_pad = 0) {
  if (!P.attitude_filter) return;
  const AttitudeFilter& A = *P.attitude_filter;
  size_t stride = size_t(n_pad);
  if (!q) {
    q = P.obs_delay ? A.rep : A.quat;
    stride = size_t(A.stride);
  }
  float e[4], qb[4];
  for (int r = 0; r < 4; ++r) e[r] = q[size_t(r) * stride + size_t(i)];
  attitude_filter_base(A, e, qb);
  attitude_filter_observation(P, qb, o);
}
__device__ void attitude_history_observed(const SimParams& P, int i, const History& H) {
  if (!P.attitude_filter) return;
  float o[UPKIE_SP_IMU_ANGVEL];
  attitude_observed(P, i, o);
  for (int c = 0; c < H.count; ++c) {
    if (!attitude_filter_column(H.columns[c])) continue;
    for (int en = 0; en < H.ticks; ++en)
      H.ring[(size_t(en) * size_t(H.count) + size_t(c)) * size_t(H.stride) + size_t(i)] = o[H.columns[c]];
  }
}

// The IMU misalignment: the observed orientation of S, read through env i's e_i (the state or a sensed row: under an
// observation delay the misalignment is applied to the snapshot when the observation is built)
__device__ void imu_misalign_observed(const SimParams& P, int i, RobotState& S) {
  if (!P.imu_misalign) return;
  const ImuMisalign& M = *P.imu_misalign;
  imu_misalign_view(S, imu_misalign_load([&](int r) { return M.quat[size_t(r) * size_t(M.stride) + size_t(i)]; }));
}

// The encoder offsets: the reported servo positions of S, read through env i's delta_i (the state or a sensed row, as
// imu_misalign_observed)
__device__ void encoder_offset_observed(const SimParams& P, int i, RobotState& S) {
  if (!P.encoder_offset) return;
  const EncoderOffset& E = *P.encoder_offset;
  encoder_offset_view(S, encoder_offset_load([&](int j) { return E.offset[size_t(j) * size_t(E.stride) + size_t(i)]; }));
}

// The servo noise: the replies of S with the noise of the cycle env i reports, its reset observation's (fresh) or the
// cycle d before the last step's last cycle (d its observation delay, as the step kernels clamp it; the state or a
// sensed row), before the other views
__device__ uint64_t servo_noise_reported_cycle(const SimParams& P, int i, const uint32_t* tick) {
  const ServoNoise& N = *P.servo_noise;
  if (N.fresh[i]) return servo_noise_reset_cycle(N.count[i]);
  uint32_t d = 0;
  if (P.obs_delay) {
    const uint32_t cap = uint32_t(P.obs_delay->ticks > 1 ? P.obs_delay->ticks : 1) * uint32_t(P.nb_substeps);
    d = min(P.obs_delay->delay[i], cap);
  }
  return servo_noise_cycle_before(tick[i], uint32_t(P.nb_substeps), d);
}
__device__ void servo_noise_observed(const SimParams& P, int i, RobotState& S, const uint32_t* tick,
                                     uint64_t seed, uint64_t g) {
  if (!P.servo_noise) return;
  const ServoNoise& N = *P.servo_noise;
  servo_noise_view(S, servo_noise_increments([&](int c) { return N.sigma[size_t(c) * size_t(N.stride) + size_t(i)]; },
                                             seed, g, servo_noise_reported_cycle(P, i, tick)));
}

// Servo dropouts without an observation delay: the observed state of S, every servo of the mask reporting its held
// triple (the held rows latch every servo after a tick's last substep that received it, so this is the state for them)
__device__ void servo_dropout_observed(const SimParams& P, int i, RobotState& S) {
  if (!P.servo_dropout || P.obs_delay) return;
  const ServoDropout& D = *P.servo_dropout;
  servo_dropout_view(S, D.spec.joint_mask, [&](int r) { return D.held[size_t(r) * size_t(D.stride) + size_t(i)]; });
}

// The observation history of every env, out[n][size][count], entries newest first: the window ends `d` substeps
// before the end of the tick, the env's observation delay when one is set (clamped as the step kernels clamp it)
__global__ void k_history_read(const __grid_constant__ SimParams P, const History* __restrict__ H, int n,
                               float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t ticks = uint32_t(H->ticks), size = uint32_t(H->size), count = uint32_t(H->count);
  uint32_t d = 0;
  if (P.obs_delay) {
    const uint32_t cap = uint32_t(P.obs_delay->ticks > 1 ? P.obs_delay->ticks : 1) * uint32_t(P.nb_substeps);
    d = min(P.obs_delay->delay[i], cap);
    d = min(d, ticks - size);
  }
  const uint32_t head = H->head[i];
  for (uint32_t k = 0; k < size; ++k) {
    const float* const e = H->ring + size_t(history_entry(head, ticks, d, k)) * count * size_t(H->stride) + size_t(i);
    for (uint32_t c = 0; c < count; ++c) out[(size_t(i) * size + k) * count + c] = e[size_t(c) * size_t(H->stride)];
  }
}

// Every env's history filled from its state (a new spec, set_state, a new ring size)
__global__ void k_history_fill(const __grid_constant__ SimParams P, const History* __restrict__ H, int n, int n_pad,
                               const float* __restrict__ state, const uint32_t* __restrict__ tick,
                               uint64_t seed, uint64_t env_offset) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  RobotState S;
  load_state(state, n_pad, i, S);
  if (P.servo_noise) {  // each entry with the noise of its cycle, the newest the one the env reports
    const ServoNoise& N = *P.servo_noise;
    const uint64_t g = env_offset + uint64_t(i);
    history_fill_noise(
        *H, P, S, H->head[i], [&](int c) { return N.sigma[size_t(c) * size_t(N.stride) + size_t(i)]; },
        seed, g, servo_noise_reported_cycle(P, i, tick), tick[i],
        [&](RobotState& V) {
          imu_misalign_observed(P, i, V);
          encoder_offset_observed(P, i, V);
        },
        [&](uint32_t e, int c, float v) {
          H->ring[(size_t(e) * size_t(H->count) + size_t(c)) * size_t(H->stride) + size_t(i)] = v;
        });
    attitude_history_observed(P, i, *H);
    return;
  }
  imu_misalign_observed(P, i, S);
  encoder_offset_observed(P, i, S);
  history_fill(*H, P, S, i);
  attitude_history_observed(P, i, *H);
}

// The spine observation rows of the states `state` (and in spine mode the lag records `lag`), with the noise keys of
// the step that produced them (tick[i]). `mark` set: the envs whose mark is `gen` only, the rows of the others are left
// as they are (upkie_b200_final_spine_obs: the pre-reset states that the same-step auto-resets of step `gen` stashed,
// store_final_state; neither the reset nor the rest of the step writes tick[i]).
__global__ void k_spine_obs(const __grid_constant__ SimParams P, int n, int n_pad, const float* __restrict__ state,
                            const float* __restrict__ lag, const uint32_t* __restrict__ mark, uint32_t gen,
                            const uint32_t* __restrict__ tick, uint64_t env_offset, float* __restrict__ out,
                            uint64_t seed, const float* __restrict__ att = nullptr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mark && mark[i] != gen) return;
  float o[UPKIE_SPINE_DIM];
  const NoiseCtx nz{env_offset + uint64_t(i), tick[i]};  // same draw as the step that produced this state
  if (P.spine_mode && lag) {
    // the observation the spine assembled in the first cycle of the last step / the last cycle of the reset
    float lr[UPKIE_LAG_DIM];
    for (int k = 0; k < UPKIE_LAG_DIM; ++k) lr[k] = lag[size_t(k) * n_pad + i];
    SpineLag L;
    lag_from_row(lr, L);
    spine_observation_from_lag(P, L, o);
  } else {
    RobotState S;
    load_state(state, n_pad, i, S);
    if (!mark) {  // (the stash holds the terminal step's observed state)
      servo_noise_observed(P, i, S, tick, seed, env_offset + uint64_t(i));
      servo_dropout_observed(P, i, S);
      imu_misalign_observed(P, i, S);
      encoder_offset_observed(P, i, S);
    }
    float tq[6];
    measured_torques(P, S, &nz, tq, i);
    spine_observation(P, S, o, tq);
    attitude_observed(P, i, o, att, n_pad);  // (`att`: the stash's rows of the terminal estimates)
  }
  apply_imu_uncertainty(P, nz, o, i);
#pragma unroll
  for (int k = 0; k < UPKIE_SPINE_DIM; ++k) out[size_t(i) * UPKIE_SPINE_DIM + k] = o[k];
}

__global__ void k_reset_obs(const __grid_constant__ SimParams P, int n, int n_pad, const float* __restrict__ state,
                            const uint32_t* __restrict__ tick, uint64_t env_offset, int obs_dim,
                            float* __restrict__ out, const float* __restrict__ lag, uint64_t seed) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  RobotState S;
  load_state(state, n_pad, i, S);
  servo_noise_observed(P, i, S, tick, seed, env_offset + uint64_t(i));
  servo_dropout_observed(P, i, S);
  imu_misalign_observed(P, i, S);
  encoder_offset_observed(P, i, S);
  if (obs_dim == UPKIE_OBS_DIM && P.spine_mode && lag) {
    for (int j = 0; j < 6; ++j) {
      float* o = out + size_t(i) * UPKIE_OBS_DIM + j * 5;
      for (int k = 0; k < 3; ++k) o[k] = lag[size_t(UPKIE_LAG_OBS_REPLY + 3 * j + k) * n_pad + i];
      o[3] = 20.0f; o[4] = 18.0f;
    }
    return;
  }
  if (obs_dim == UPKIE_OBS_DIM) {
    float tq[6];
    const NoiseCtx nz{env_offset + uint64_t(i), tick[i]};
    measured_torques(P, S, &nz, tq, i);
    for (int j = 0; j < 6; ++j) {
      float* o = out + size_t(i) * UPKIE_OBS_DIM + j * 5;
      o[0] = S.q[j]; o[1] = S.qd[j]; o[2] = tq[j]; o[3] = 42.0f; o[4] = 18.0f;
    }
    return;
  }
  float o6[6];
  gyropod_obs(P, S, o6);
  if (P.attitude_filter) {  // the pitch of the estimate the env reports
    float o[UPKIE_SP_IMU_ANGVEL];
    attitude_observed(P, i, o);
    o6[1] = o[UPKIE_SP_PITCH];
  }
  if (obs_dim == 6) {
    for (int k = 0; k < 6; ++k) out[size_t(i) * 6 + k] = o6[k];
  } else {
    out[size_t(i) * 4 + 0] = o6[1]; out[size_t(i) * 4 + 1] = o6[0];
    out[size_t(i) * 4 + 2] = o6[4]; out[size_t(i) * 4 + 3] = o6[3];
  }
}

// The attitude filter of every env from its state (set_state, a first filter): the estimate of the observed (misaligned)
// orientation without an error, stored as the estimate and the report, b = 0; `gains` (a first filter) also stores
// kp, ki
__global__ void k_attitude_init(const __grid_constant__ SimParams P, int n, int n_pad, const float* __restrict__ state,
                                bool gains, float kp, float ki) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  RobotState S;
  load_state(state, n_pad, i, S);
  imu_misalign_observed(P, i, S);
  const AttitudeFilter& A = *P.attitude_filter;
  const size_t stride = size_t(A.stride);
  float q[4];
  attitude_filter_initial(A, S.quat, 0.f, 0.f, q);
  for (int r = 0; r < 4; ++r) {
    A.quat[size_t(r) * stride + size_t(i)] = q[r];
    A.rep[size_t(r) * stride + size_t(i)] = q[r];
  }
  for (int r = 0; r < 3; ++r) A.bias[size_t(r) * stride + size_t(i)] = 0.f;
  if (gains) {
    A.gains[size_t(i)] = kp;
    A.gains[stride + size_t(i)] = ki;
  }
}

// validation of the caller's rows [n][UPKIE_EP_DIM] of a per-env parameter table (env_row_flags OR-ed into *flags)
__global__ void k_env_params_check(int n, const float* __restrict__ rows, uint32_t* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t f = env_row_flags(rows + size_t(i) * UPKIE_EP_DIM);
  if (f) atomicOr(flags, f);
}

// Every env's row of the config's parameter values (what the envs run without a table), as out[i * istride + k *
// kstride]: a table [UPKIE_EP_DIM][n_pad] (1, n_pad) or rows [n][UPKIE_EP_DIM] (UPKIE_EP_DIM, 1)
__global__ void k_env_params_from_config(const __grid_constant__ SimParams P, int n, int istride, int kstride,
                                         float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int k = 0; k < UPKIE_EP_DIM; ++k) out[size_t(i) * istride + size_t(k) * kstride] = config_env_param(P, k);
}

// The action delay's stop row as every env's command, out[i * istride + c * cstride]: the columns of the command buffer
// [UPKIE_ACT_DIM][n_pad] (1, n_pad) or rows [n][UPKIE_ACT_DIM] (UPKIE_ACT_DIM, 1)
__global__ void k_stop_rows(int n, int istride, int cstride, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int c = 0; c < UPKIE_ACT_DIM; ++c) out[size_t(i) * istride + size_t(c) * cstride] = action_delay_stop_value(c);
}

__global__ void k_fill(int n, float* __restrict__ out, float v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = v;
}

// Rows [ages][n][dim] <-> ages 0 .. ages - 1 (0 the newest) of the rings [ticks][dim][stride] whose next write is row
// head[i] (head null: row 0). At ticks = ages = 1, the transpose of rows [n][dim] and the struct-of-arrays columns
// [dim][stride] of every per-env buffer.
__global__ void k_ring_copy(float* __restrict__ ring, const uint32_t* __restrict__ head, int ticks, int dim, int n,
                            int stride, int ages, float* __restrict__ rows, int to_rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t h = head ? head[i] : 0u;
  for (int a = 0; a < ages; ++a) {
    float* const col = ring + size_t(delay_ring_row(h, uint32_t(ticks), uint32_t(a))) * dim * stride + size_t(i);
    float* const row = rows + (size_t(a) * n + i) * dim;
    for (int k = 0; k < dim; ++k) {
      if (to_rows) row[k] = col[size_t(k) * stride];
      else col[size_t(k) * stride] = row[k];
    }
  }
}

// the rings `src` [src_ticks][dim][stride] (next write head[i], null: 0) into `dst` [dst_ticks][dim][stride] in age
// order, with row 0 of dst the next write: the ages beyond src_ticks are stop rows (stop) or copies of the oldest;
// columns = a mask of the columns copied (bit k, 64 bits at most), all of them for ~0
__global__ void k_ring_resize(const float* __restrict__ src, const uint32_t* __restrict__ head, int src_ticks,
                              float* __restrict__ dst, int dst_ticks, int dim, int n, int stride, int stop,
                              uint64_t columns) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t h = head ? head[i] : 0u;
  for (int a = 0; a < dst_ticks; ++a) {
    const int sa = a < src_ticks ? a : src_ticks - 1;
    const float* const s = src + size_t(delay_ring_row(h, uint32_t(src_ticks), uint32_t(sa))) * dim * stride + i;
    float* const d = dst + size_t(delay_ring_row(0u, uint32_t(dst_ticks), uint32_t(a))) * dim * stride + i;
    for (int k = 0; k < dim; ++k)
      if ((columns >> k) & 1u) d[size_t(k) * stride] = (stop && a >= src_ticks) ? action_delay_stop_value(k) : s[size_t(k) * stride];
  }
}

// the push force of each env's last step, from its schedule state (R null: no spec, zeros)
__global__ void k_push_forces(const PushRand* __restrict__ R, int n, uint64_t seed, uint64_t env_offset,
                              float* __restrict__ force) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float f[3] = {0.f, 0.f, 0.f};
  if (R) push_last_force(R->spec, seed, env_offset + uint64_t(i), R->count[i], R->timer[i], f);
  for (int k = 0; k < 3; ++k) force[size_t(i) * 3 + k] = f[k];
}

int grid_of(int n) { return (n + 127) / 128; }

// rows [ages][n][dim] of the rings `ring` (ring_rows) or the other way (ring_cols), k_ring_copy; the defaults are the
// plain transpose of rows [n][dim] and columns [dim][stride]
cudaError_t ring_rows(const float* ring, int dim, int n, int stride, float* rows, cudaStream_t s,
                      const uint32_t* head = nullptr, int ticks = 1, int ages = 1) {
  k_ring_copy<<<grid_of(n), 128, 0, s>>>(const_cast<float*>(ring), head, ticks, dim, n, stride, ages, rows, 1);
  return cudaGetLastError();
}
cudaError_t ring_cols(const float* rows, int dim, int n, int stride, float* ring, cudaStream_t s,
                      const uint32_t* head = nullptr, int ticks = 1, int ages = 1) {
  k_ring_copy<<<grid_of(n), 128, 0, s>>>(ring, head, ticks, dim, n, stride, ages, const_cast<float*>(rows), 0);
  return cudaGetLastError();
}

cudaError_t ring_resize(const float* src, const uint32_t* head, int src_ticks, float* dst, int dst_ticks, int dim,
                        int n, int stride, int stop, uint64_t columns, cudaStream_t s) {
  k_ring_resize<<<grid_of(n), 128, 0, s>>>(src, head, src_ticks, dst, dst_ticks, dim, n, stride, stop, columns);
  return cudaGetLastError();
}

cudaError_t stop_rows(int n, int istride, int cstride, float* out, cudaStream_t s) {
  k_stop_rows<<<grid_of(n), 128, 0, s>>>(n, istride, cstride, out);
  return cudaGetLastError();
}

cudaError_t env_params_from_config(const SimParams& P, int n, int istride, int kstride, float* out, cudaStream_t s) {
  k_env_params_from_config<<<grid_of(n), 128, 0, s>>>(P, n, istride, kstride, out);
  return cudaGetLastError();
}

cudaError_t fill(int n, float* out, float v, cudaStream_t s) {
  k_fill<<<grid_of(n), 128, 0, s>>>(n, out, v);
  return cudaGetLastError();
}

// a per-env buffer the handle may never have allocated, copied into `dst` (src null: zeros)
cudaError_t copy_or_zero(void* dst, const void* src, size_t bytes, cudaStream_t s) {
  return src ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s) : cudaMemsetAsync(dst, 0, bytes, s);
}

// Per-env buffers {&pointer, bytes}, allocated and zeroed, all of them or none: on a failure the ones allocated are
// freed and every pointer is null again
cudaError_t alloc_zeroed(std::initializer_list<std::pair<void**, size_t>> bufs) {
  cudaError_t e = cudaSuccess;
  for (const auto& b : bufs) {
    if (e == cudaSuccess) e = cudaMalloc(b.first, b.second);
    if (e == cudaSuccess) e = cudaMemset(*b.first, 0, b.second);
  }
  if (e != cudaSuccess)
    for (const auto& b : bufs) {
      cudaFree(*b.first);
      *b.first = nullptr;
    }
  return e;
}

__global__ void k_init_state(const __grid_constant__ SimParams P, int n, int n_pad, float* __restrict__ state) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pad) return;
  for (int k = 0; k < UPKIE_STATE_DIM; ++k) state[size_t(k) * n_pad + i] = 0.f;
  for (int k = 0; k < 3; ++k) state[size_t(UPKIE_ST_POS + k) * n_pad + i] = P.init_pos[k];
  for (int k = 0; k < 4; ++k) state[size_t(UPKIE_ST_QUAT + k) * n_pad + i] = P.init_quat[k];
  (void)n;
}

// Block size per launch. (1) The warps of a block run the substep body in lock-step (one barrier per substep) and
// share its instruction fetches, so larger blocks fetch less per warp; (2) with 255 registers/thread one 256-thread
// block fills an SM, so a fixed block size leaves a partial last wave (65 536 envs in 256-thread blocks on 132 SMs:
// 1.94 waves). Pick the number of waves k first, then the block size (multiple of 32) that makes the grid
// k * num_sms blocks: every SM gets the same number of equally sized blocks.
int pick_block(const Handle* h, int cnt) {
  if (h->block > 0) return h->block;
  const int per_wave = h->num_sms * UPKIE_MAX_THREADS;
  const int waves = (cnt + per_wave - 1) / per_wave;
  int block = (cnt + waves * h->num_sms - 1) / (waves * h->num_sms);
  block = (block + 31) / 32 * 32;
  if (block < 32) block = 32;
  if (block > UPKIE_MAX_THREADS) block = UPKIE_MAX_THREADS;
  return block;
}

// The step kernels of (TILE, family): a compile-time walk over the pairs that step_instantiated names, the others
// cudaErrorNotSupported.
template <int TILE = 0, int FAMILY = 0>
cudaError_t dispatch_step(int tile, const StepArgs& a) {
  if constexpr (TILE == kNumTiles) {
    return cudaErrorNotSupported;
  } else if constexpr (FAMILY == kNumFamilies) {
    return dispatch_step<TILE + 1, 0>(tile, a);
  } else {
    if constexpr (step_instantiated(TILE, FAMILY)) {
      if (tile == TILE && a.family == FAMILY) return launch_step<TILE, FAMILY>(a);
    }
    return dispatch_step<TILE, FAMILY + 1>(tile, a);
  }
}

// envs [i0, i0 + cnt): all buffers are indexed by the env index of the handle. `tile` selects the
// shared-memory-tile instantiation (host buffers), see kernel_common.cuh.
// `final_obs`: rows of the same-step auto-resets' terminal observations (null = not requested): it travels in a copy of
// the parameter block made for this launch only, as does the stash of the pre-reset states when `final_state` is set
// (prepare_final_state allocated it and numbered the step).
int step_range(Handle* h, int mode, int i0, int cnt, const float* action, float* obs, float* reward, uint8_t* term,
               uint8_t* trunc, cudaStream_t s, bool tile = false, bool persistent = true, bool compact = false,
               bool multicast = false, const PeerPtrs* peers = nullptr, float* final_obs = nullptr,
               bool final_state = false) {
  h->final_valid = false;  // the simulator moves on: the caller marks the stash valid once the whole step is enqueued
  if (multicast && final_state)
    return fail(UPKIE_B200_EINVAL, "final_state has no in-kernel rollout transport (use upkie_b200_step)");
  const int transport = multicast ? 2 : (tile ? 1 : 0);  // the TILE of the step kernels
  const char* why = nullptr;
  const int family = step_family(h->P, h->ext != nullptr, mode, transport, &why);
  if (family < 0) return fail(UPKIE_B200_EINVAL, why);
  StepArgs a;
  std::memset(&a.peers, 0, sizeof(a.peers));
  if (peers) a.peers = *peers;
  a.history = (h->P.action_delay && h->delay_ticks > 1) || (h->P.obs_delay && h->sense_ticks > 1);
  SimParams P_launch;
  const bool stash = final_state && h->final_state && h->autoreset == AUTORESET_SAME_STEP;
  if ((final_obs || stash) && h->autoreset == AUTORESET_SAME_STEP) {
    P_launch = h->P;
    P_launch.final_obs = final_obs;
    if (stash) {
      P_launch.final_state = h->final_state;
      P_launch.final_gen = h->final_gen;
    }
    a.P = &P_launch;
  } else {
    a.P = &h->P;
  }
  a.mode = mode;
  a.autoreset = h->autoreset;
  a.family = family;
  a.lag = h->P.spine_mode ? h->lag : nullptr;
  a.ext = h->ext;
  a.ext_local = h->ext_local;
  a.i0 = i0;
  a.cnt = cnt;
  a.n_pad = h->n_pad;
  // Only the persistent launch keeps its fixed block (one small block per SM that walks tiles while the next tile's
  // rows cross PCIe). Every other launch, tile path included, takes pick_block's size: at 65 536 envs that is one
  // 256-thread block per SM instead of two 128-thread ones, all 8 warps of an SM share each substep's barrier and so
  // its instruction fetches (H100 80GB HBM3 at 700 W: 0.164 / 0.171 / 0.191 / 0.216 ms per tick at 256 / 128 / 64 /
  // 32 threads per block, DESIGN.md section 4).
  a.block = (tile && persistent) ? h->host_block : pick_block(h, cnt);
  a.grid = (tile && persistent) ? h->num_sms * h->host_blocks_per_sm : 0;
  a.compact_obs = compact ? 1 : 0;
  a.smem_carveout = h->smem_carveout;
  a.state = h->state;
  a.action = action;
  a.obs = obs;
  a.reward = reward;
  a.terminated = term;
  a.truncated = trunc;
  a.eps = h->eps;
  a.mu = h->mu;
  a.err = h->err;
  a.done_prev = h->done_prev;
  a.episode = h->episode;
  a.tick = h->tick;
  a.seed = h->seed;
  a.env_offset = h->env_offset;
  a.stream = s;
  CUDA_TRY(dispatch_step(transport, a));
  h->step_launches += 1;
  return UPKIE_B200_OK;
}

// UpkieStepOutputs.final_state: whether this step stashes the pre-reset states (same-step mode only; the flag is
// ignored in the other modes). The stash is allocated on the first request, so that a handle that never asks holds no
// memory for it, and each such step gets a new number: the mark a resetting env leaves in its column of the stash.
int prepare_final_state(Handle* h, int32_t flag, bool& stash) {
  stash = flag != 0 && h->autoreset == AUTORESET_SAME_STEP;
  if (!stash) return UPKIE_B200_OK;
  // reset randomisation: the pre-reset parameter-table columns go to kFinalParamCols more rows
  const bool params = h->P.reset_rand != nullptr;
  // the attitude filter: the terminal estimates go to 4 more rows after those (no spine mode with a filter)
  const int rows = (h->lag ? kFinalRowsSpine : kFinalRows) + (params ? kFinalParamCols : 0) +
                   (h->P.attitude_filter ? 4 : 0);
  if (h->final_state && h->final_rows < rows) {
    CUDA_TRY(cudaSetDevice(h->device));
    CUDA_TRY(cudaDeviceSynchronize());  // steps in flight may still write the smaller stash
    cudaFree(h->final_state);
    h->final_state = nullptr;
  }
  h->final_params = params;
  if (!h->final_state) {
    const size_t bytes = size_t(rows) * h->n_pad * sizeof(float);
    h->final_rows = rows;
    CUDA_TRY(cudaSetDevice(h->device));
    CUDA_TRY(cudaMalloc(&h->final_state, bytes));
    CUDA_TRY(cudaMemset(h->final_state, 0, bytes));
    CUDA_TRY(cudaDeviceSynchronize());  // the marks are 0 before any stream's step reads them
  }
  if (++h->final_gen == 0) h->final_gen = 1;  // 0 is the mark of a column that no step has written
  return UPKIE_B200_OK;
}

int step_any(Handle* h, int mode, const float* action, float* obs, float* reward, uint8_t* term, uint8_t* trunc,
             cudaStream_t s) {
  if (!action || !obs || !term) return fail(UPKIE_B200_EINVAL, "step: null buffer");
  CUDA_TRY(cudaSetDevice(h->device));
  return step_range(h, mode, 0, h->n, action, obs, reward, term, trunc, s);
}

int ensure_staging(Handle* h) {
  if (h->d_act) return UPKIE_B200_OK;
  const size_t n = size_t(h->n);
  CUDA_TRY(cudaSetDevice(h->device));
  for (int k = 0; k < kHostStreams; ++k) CUDA_TRY(cudaStreamCreateWithFlags(&h->host_streams[k], cudaStreamNonBlocking));
  for (int k = 0; k < 64; ++k) CUDA_TRY(cudaEventCreateWithFlags(&h->host_events[k], cudaEventDisableTiming));
  CUDA_TRY(cudaMallocHost(&h->h_act, n * UPKIE_ACT_DIM * sizeof(float)));
  CUDA_TRY(cudaMallocHost(&h->h_obs, n * UPKIE_OBS_DIM * sizeof(float)));
  CUDA_TRY(cudaMallocHost(&h->h_rew, n * sizeof(float)));
  CUDA_TRY(cudaMallocHost(&h->h_term, n));
  CUDA_TRY(cudaMallocHost(&h->h_trunc, n));
  CUDA_TRY(cudaMalloc(&h->d_act, n * UPKIE_ACT_DIM * sizeof(float)));
  CUDA_TRY(cudaMalloc(&h->d_obs, n * UPKIE_OBS_DIM * sizeof(float)));
  CUDA_TRY(cudaMalloc(&h->d_rew, n * sizeof(float)));
  CUDA_TRY(cudaMalloc(&h->d_term, n));
  CUDA_TRY(cudaMalloc(&h->d_trunc, n));
  return UPKIE_B200_OK;
}

// device-side alias of a pinned host buffer (nullptr when the buffer is pageable or not mapped)
template <typename T>
T* mapped(T* p) {
  if (!p) return nullptr;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  if (at.type != cudaMemoryTypeHost || !at.devicePointer) return nullptr;
  return static_cast<T*>(at.devicePointer);
}

// Host-buffer step. Pageable caller buffers are first staged through the handle's pinned buffers; on
// pinned (mapped) buffers one of three pipelines runs, `zero_copy` selecting it:
//   2 (default, servos)  hybrid: the copy engine streams the action rows in, chunk by chunk on one stream; each
//                        chunk's TILE=1 kernel waits for its rows only and writes observations / flags straight
//                        to host memory. Copy-engine reads overlap SM writes on the link, SM reads and writes
//                        share it (tools/micro/pcie_duplex.cu measures both).
//   1                    one persistent TILE=1 launch reading actions from and writing observations to host memory.
//   0                    H2D copy -> TILE=0 kernel -> D2H copies per chunk on rotating streams.
// `compact` (servos): observation rows [6][3] = position, velocity, torque (TILE=1 kernels).
// `final_obs` (same-step auto-reset): its rows are sparse, so in every pipeline the kernel stores them straight into
// host memory through the mapped alias; a pageable buffer goes through a pinned copy of the caller's rows, so that
// the rows of the envs that do not reset keep their values.
int step_host(Handle* h, int mode, const float* action, float* obs, float* reward, uint8_t* term, uint8_t* trunc,
              bool compact = false, float* final_obs = nullptr, bool final_state = false) {
  if (!action || !obs || !term) return fail(UPKIE_B200_EINVAL, "step_host: null buffer");
  int rc = ensure_staging(h);
  if (rc) return rc;
  CUDA_TRY(cudaSetDevice(h->device));
  const size_t n = size_t(h->n);
  const size_t act_dim = mode == MODE_SERVOS ? UPKIE_ACT_DIM : (mode == MODE_GYROPOD ? 2 : 1);
  const size_t obs_dim = mode == MODE_SERVOS ? (compact ? 18 : UPKIE_OBS_DIM) : (mode == MODE_GYROPOD ? 6 : 4);
  // The kernels move a row with vector accesses: the servo action row as float4 and the gyropod one as float2, the
  // observation rows as float2 and the pendulum's as float4. A pinned buffer short of that alignment (a float32 view
  // that starts 4 bytes into its allocation, say) is staged like a pageable one rather than used in place.
  auto aligned_to = [](const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; };
  const uintptr_t act_align = mode == MODE_SERVOS ? 16 : (mode == MODE_GYROPOD ? 8 : 4);
  const uintptr_t obs_align = mode == MODE_PENDULUM ? 16 : 8;
  // reward / truncated are constants of the reference (0.0 and false): callers may pass NULL for them
  const bool pin_in = mapped(action) != nullptr && aligned_to(action, act_align);
  const bool pin_out = mapped(obs) && aligned_to(obs, obs_align) && (!reward || mapped(reward)) && mapped(term) &&
                       (!trunc || mapped(trunc));
  if (!pin_in) std::memcpy(h->h_act, action, n * act_dim * sizeof(float));
  const float* src_act = pin_in ? action : h->h_act;
  float* dst_obs = pin_out ? obs : h->h_obs;
  float* dst_rew = reward ? (pin_out ? reward : h->h_rew) : nullptr;
  uint8_t* dst_term = pin_out ? term : h->h_term;
  uint8_t* dst_trunc = trunc ? (pin_out ? trunc : h->h_trunc) : nullptr;
  if (h->autoreset != AUTORESET_SAME_STEP) final_obs = nullptr;
  const bool fin_staged = final_obs && !mapped(final_obs);
  if (fin_staged) {
    if (!h->h_fin) CUDA_TRY(cudaMallocHost(&h->h_fin, n * UPKIE_OBS_DIM * sizeof(float)));
    std::memcpy(h->h_fin, final_obs, n * obs_dim * sizeof(float));
  }
  float* fin = final_obs ? mapped(fin_staged ? h->h_fin : final_obs) : nullptr;

  // Order the private (non-blocking) streams after whatever the caller enqueued on the default stream - reset(),
  // set_state(), set_counters() through PyTorch's default current stream: without this a step_*_host() right after
  // an asynchronous reset raced with it (round-1 advisor finding). Callers on other streams synchronise themselves.
  CUDA_TRY(cudaEventRecord(h->host_events[63], cudaStreamLegacy));
  for (int k = 0; k < kHostStreams; ++k) CUDA_TRY(cudaStreamWaitEvent(h->host_streams[k], h->host_events[63], 0));

  int pipeline = h->zero_copy;
  if (pipeline == 2 && mode != MODE_SERVOS) pipeline = 1;  // tiny rows: nothing to stream
  // chunk boundaries (multiples of 256 envs). Default: host_chunks equal chunks; UPKIE_B200_HOST_SPLIT gives the
  // fractions explicitly (a small last chunk shortens the exposed tail: last kernel + its write drain).
  int start[65];
  int chunks = 0;
  start[0] = 0;
  if (h->host_split_n > 0 && h->n >= 4 * 8192) {
    double acc = 0.0;
    for (int c = 0; c < h->host_split_n && chunks < 62; ++c) {
      acc += h->host_split[c];
      int end = c + 1 == h->host_split_n ? h->n : int(acc * h->n + 0.5);
      end = (end + 255) / 256 * 256;
      if (end > h->n) end = h->n;
      if (end > start[chunks]) start[++chunks] = end;
    }
    if (start[chunks] < h->n) start[++chunks] = h->n;
  } else {
    const int want = h->n >= 4 * 8192 ? h->host_chunks : (h->n >= 2 * 8192 ? 2 : 1);
    int per = (h->n + want - 1) / want;
    per = (per + 255) / 256 * 256;
    for (int i0 = 0; i0 < h->n && chunks < 63; i0 += per) start[++chunks] = (i0 + per < h->n) ? i0 + per : h->n;
  }
  auto chunk_count = [&](int c) { return start[c + 1] - start[c]; };

  if (pipeline == 2) {
    cudaStream_t sc = h->host_streams[0];
    for (int c = 0; c < chunks; ++c) {
      const size_t i0 = size_t(start[c]);
      CUDA_TRY(cudaMemcpyAsync(h->d_act + i0 * act_dim, src_act + i0 * act_dim, size_t(chunk_count(c)) * act_dim * sizeof(float),
                               cudaMemcpyHostToDevice, sc));
      CUDA_TRY(cudaEventRecord(h->host_events[c], sc));
    }
    for (int c = 0; c < chunks; ++c) {
      cudaStream_t sk = h->host_streams[1 + (c % h->host_kernel_streams)];
      CUDA_TRY(cudaStreamWaitEvent(sk, h->host_events[c], 0));
      rc = step_range(h, mode, start[c], chunk_count(c), h->d_act, mapped(dst_obs), mapped(dst_rew), mapped(dst_term),
                      mapped(dst_trunc), sk, /*tile=*/true, /*persistent=*/false, compact, false, nullptr, fin,
                      final_state);
      if (rc) return rc;
    }
    for (int k = 0; k < h->host_kernel_streams; ++k) CUDA_TRY(cudaStreamSynchronize(h->host_streams[1 + k]));
  } else if (pipeline == 1) {
    cudaStream_t s = h->host_streams[0];
    rc = step_range(h, mode, 0, h->n, mapped(src_act), mapped(dst_obs), mapped(dst_rew), mapped(dst_term),
                    mapped(dst_trunc), s, /*tile=*/true, /*persistent=*/true, compact, false, nullptr, fin, final_state);
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(s));
  } else {
    for (int c = 0; c < chunks; ++c) {
      const int i0 = start[c];
      const int cnt = chunk_count(c);
      cudaStream_t s = h->host_streams[c % kHostStreams];
      CUDA_TRY(cudaMemcpyAsync(h->d_act + size_t(i0) * act_dim, src_act + size_t(i0) * act_dim,
                               size_t(cnt) * act_dim * sizeof(float), cudaMemcpyHostToDevice, s));
      // compact rows exist in the TILE=1 kernels only; device staging buffers either way
      rc = step_range(h, mode, i0, cnt, h->d_act, h->d_obs, h->d_rew, h->d_term, h->d_trunc, s, /*tile=*/compact,
                      /*persistent=*/false, compact, false, nullptr, fin, final_state);
      if (rc) return rc;
      CUDA_TRY(cudaMemcpyAsync(dst_obs + size_t(i0) * obs_dim, h->d_obs + size_t(i0) * obs_dim,
                               size_t(cnt) * obs_dim * sizeof(float), cudaMemcpyDeviceToHost, s));
      if (dst_rew) CUDA_TRY(cudaMemcpyAsync(dst_rew + i0, h->d_rew + i0, size_t(cnt) * sizeof(float), cudaMemcpyDeviceToHost, s));
      CUDA_TRY(cudaMemcpyAsync(dst_term + i0, h->d_term + i0, size_t(cnt), cudaMemcpyDeviceToHost, s));
      if (dst_trunc) CUDA_TRY(cudaMemcpyAsync(dst_trunc + i0, h->d_trunc + i0, size_t(cnt), cudaMemcpyDeviceToHost, s));
    }
    for (int k = 0; k < kHostStreams; ++k) CUDA_TRY(cudaStreamSynchronize(h->host_streams[k]));
  }
  if (!pin_out) {
    std::memcpy(obs, h->h_obs, n * obs_dim * sizeof(float));
    if (reward) std::memcpy(reward, h->h_rew, n * sizeof(float));
    std::memcpy(term, h->h_term, n);
    if (trunc) std::memcpy(trunc, h->h_trunc, n);
  }
  if (fin_staged) std::memcpy(final_obs, h->h_fin, n * obs_dim * sizeof(float));
  return UPKIE_B200_OK;
}

// The entries the observation history's ring holds: K, and the deepest observation delay the handle may draw
int history_ticks(const Handle* h) {
  return int(h->hist_spec.size) + (h->sense_ticks > 1 ? h->sense_ticks : 1) * h->P.nb_substeps;
}

// The observation history of the spec h->hist_spec: its device block, ring (history_ticks entries) and heads, every
// entry filled from the current state. Waits for the device.
int history_build(Handle* h) {
  const UpkieHistory& spec = h->hist_spec;
  const int ticks = history_ticks(h);
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may use the ring
  h->P.history = nullptr;
  cudaFree(h->hist_ring);
  h->hist_ring = nullptr;
  CUDA_TRY(cudaMalloc(&h->hist_ring, size_t(ticks) * spec.count * h->n_pad * sizeof(float)));
  if (!h->hist_head) CUDA_TRY(cudaMalloc(&h->hist_head, size_t(h->n) * sizeof(uint32_t)));
  CUDA_TRY(cudaMemset(h->hist_head, 0, size_t(h->n) * sizeof(uint32_t)));
  if (!h->hist_dev) CUDA_TRY(cudaMalloc(&h->hist_dev, sizeof(History)));
  History H;
  std::memset(&H, 0, sizeof(H));
  H.size = int(spec.size);
  H.count = int(spec.count);
  H.ticks = ticks;
  H.stride = h->n_pad;
  for (uint32_t c = 0; c < spec.count; ++c) {
    H.columns[c] = spec.columns[c];
    if (history_acc_column(spec.columns[c])) H.acc = 1;
  }
  H.ring = h->hist_ring;
  H.head = h->hist_head;
  CUDA_TRY(cudaMemcpy(h->hist_dev, &H, sizeof(H), cudaMemcpyHostToDevice));
  h->hist_ticks = ticks;
  h->P.history = h->hist_dev;
  k_history_fill<<<grid_of(h->n), 128>>>(h->P, h->hist_dev, h->n, h->n_pad, h->state, h->tick, h->seed, h->env_offset);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  return UPKIE_B200_OK;
}

// Servo dropouts: the held rows of the servos of `joints` (bit j) latch every env's current state (a new spec, a mask
// that gains servos, set_state): the state's position, velocity and torque rows of joint j into held rows 3j, 3j + 1,
// 3j + 2
cudaError_t servo_dropout_latch(Handle* h, uint32_t joints, cudaStream_t s) {
  const int src[3] = {UPKIE_ST_Q, UPKIE_ST_QD, UPKIE_ST_TORQUE};
  const size_t row = size_t(h->n_pad) * sizeof(float);
  for (int j = 0; j < UPKIE_NJ; ++j) {
    if (!((joints >> j) & 1u)) continue;
    for (int k = 0; k < 3; ++k) {
      const cudaError_t e = cudaMemcpyAsync(h->drop_held + size_t(3 * j + k) * h->n_pad,
                                            h->state + size_t(src[k] + j) * h->n_pad, row, cudaMemcpyDeviceToDevice, s);
      if (e != cudaSuccess) return e;
    }
  }
  return cudaSuccess;
}

// After a change of nb_substeps or of the observation delay's depth: a ring of the new size, filled from the state
int history_resize(Handle* h) {
  if (!h->P.history || history_ticks(h) == h->hist_ticks) return UPKIE_B200_OK;
  return history_build(h);
}

}  // namespace

// ---- C ABI ----------------------------------------------------------------------------

extern "C" {

int upkie_b200_abi_version(void) { return UPKIE_B200_ABI_VERSION; }
const char* upkie_b200_last_error(void) { return g_last_error.c_str(); }

int upkie_b200_default_config(UpkieSimConfig* config) {
  if (!config) return fail(UPKIE_B200_EINVAL, "default_config: null");
  default_sim_config(config);
  return UPKIE_B200_OK;
}
int upkie_b200_default_mpc_config(UpkieMpcConfig* config) {
  if (!config) return fail(UPKIE_B200_EINVAL, "default_mpc_config: null");
  default_mpc_config(config);
  return UPKIE_B200_OK;
}

int upkie_b200_create(const UpkieModel* model, const UpkieSimConfig* config, int n_envs, int device, void** handle) {
  if (!model || !config || !handle) return fail(UPKIE_B200_EINVAL, "create: null argument");
  if (n_envs < 1) return fail(UPKIE_B200_EINVAL, "create: n_envs must be >= 1");
  int count = 0;
  cudaError_t ce = cudaGetDeviceCount(&count);
  if (ce != cudaSuccess || count == 0)
    return fail(UPKIE_B200_ECUDA, "create: no CUDA device available (this library has no CPU path)");
  if (device < 0 || device >= count) return fail(UPKIE_B200_EINVAL, "create: invalid device index");
  Handle* h = new (std::nothrow) Handle();
  if (!h) return fail(UPKIE_B200_ENOMEM, "create: out of host memory");
  std::memset(&h->P, 0, sizeof(h->P));
  std::string err;
  int rc = make_sim_params(*model, *config, h->P, err);
  if (rc) { delete h; return fail(rc, err); }
  h->magic = kMagic;
  h->model = *model;
  h->config_flags = noise_flags(h->P);
  h->n = n_envs;
  h->n_pad = (n_envs + 31) / 32 * 32;
  h->device = device;
  if (const char* b = std::getenv("UPKIE_B200_BLOCK")) {
    const int v = std::atoi(b);
    if (v >= 32 && v <= UPKIE_MAX_THREADS && v % 32 == 0) h->block = v;
  }
  if (const char* b = std::getenv("UPKIE_B200_HOST_BLOCK")) {  // developer knob
    const int v = std::atoi(b);
    if (v >= 32 && v <= 160 && v % 32 == 0) h->host_block = v;  // 2 x 4608 B of tile per warp: <= 48 KB
  }
  if (const char* b = std::getenv("UPKIE_B200_HOST_BLOCKS_PER_SM")) {  // developer knob
    const int v = std::atoi(b);
    if (v >= 1 && v <= 8) h->host_blocks_per_sm = v;
  }
  if (const char* b = std::getenv("UPKIE_B200_ZERO_COPY")) h->zero_copy = std::atoi(b);  // developer knob: 0, 1, 2
  // developer knob (tools/l1_budget.py): the step kernels' preferred shared-memory carveout, a percentage of the
  // maximum, or -1 to leave it to the driver. The attribute belongs to the kernel: it outlives the handle in the process
  if (const char* b = std::getenv("UPKIE_STEP_SMEM_CARVEOUT")) {
    const int v = std::atoi(b);
    if (v >= -1 && v <= 100) h->smem_carveout = v;
  }
  if (const char* b = std::getenv("UPKIE_B200_HOST_SPLIT")) {  // developer knob: "0.4,0.4,0.2"
    h->host_split_n = 0;
    const char* p = b;
    while (*p && h->host_split_n < 8) {
      char* end = nullptr;
      const double v = std::strtod(p, &end);
      if (end == p) break;
      if (v > 0.0) h->host_split[h->host_split_n++] = v;
      p = (*end == ',') ? end + 1 : end;
    }
  }
  if (const char* b = std::getenv("UPKIE_B200_HOST_KERNEL_STREAMS")) {  // developer knob
    const int v = std::atoi(b);
    if (v >= 1 && v <= 2) h->host_kernel_streams = v;
  }
  if (const char* b = std::getenv("UPKIE_B200_HOST_CHUNKS")) {  // developer knob
    const int v = std::atoi(b);
    if (v >= 1 && v <= 62) h->host_chunks = v;
  }
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, device);
  if (e == cudaSuccess) e = cudaMalloc(&h->state, size_t(UPKIE_STATE_DIM) * h->n_pad * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->err, size_t(n_envs) * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->done_prev, size_t(n_envs));
  if (e == cudaSuccess) e = cudaMalloc(&h->episode, size_t(n_envs) * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMemset(h->err, 0, size_t(n_envs) * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMemset(h->done_prev, 0, size_t(n_envs));
  if (e == cudaSuccess) e = cudaMemset(h->episode, 0, size_t(n_envs) * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->bv_episode, size_t(n_envs) * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMemset(h->bv_episode, 0, size_t(n_envs) * sizeof(uint32_t));
  if (e == cudaSuccess && h->P.spine_mode) {
    e = cudaMalloc(&h->lag, size_t(UPKIE_LAG_DIM) * h->n_pad * sizeof(float));
    if (e == cudaSuccess) e = cudaMemset(h->lag, 0, size_t(UPKIE_LAG_DIM) * h->n_pad * sizeof(float));
  }
  if (e == cudaSuccess && h->P.body_contacts) {
    e = cudaMalloc(&h->body_rec, size_t(UPKIE_BODY_REC_DIM) * h->n_pad * sizeof(float));
    if (e == cudaSuccess) e = cudaMemset(h->body_rec, 0, size_t(UPKIE_BODY_REC_DIM) * h->n_pad * sizeof(float));
    h->P.body_rec = h->body_rec;
    h->P.body_rec_stride = h->n_pad;
  }
  if (e == cudaSuccess) e = cudaMalloc(&h->tick, size_t(n_envs) * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMemset(h->tick, 0, size_t(n_envs) * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->elapsed, size_t(n_envs) * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMemset(h->elapsed, 0, size_t(n_envs) * sizeof(uint32_t));
  h->P.elapsed = h->elapsed;
  if (e == cudaSuccess) {
    k_init_state<<<(h->n_pad + 127) / 128, 128>>>(h->P, h->n, h->n_pad, h->state);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    std::string msg = std::string("create: ") + cudaGetErrorString(e);
    upkie_b200_destroy(h);
    return fail(UPKIE_B200_ECUDA, msg);
  }
  *handle = h;
  return UPKIE_B200_OK;
}

void upkie_b200_destroy(void* handle) {
  Handle* h = as_handle(handle);
  if (!h) return;
  cudaSetDevice(h->device);
  cudaFree(h->state); cudaFree(h->eps); cudaFree(h->mu); cudaFree(h->err); cudaFree(h->done_prev); cudaFree(h->episode);
  cudaFree(h->bv_episode);
  cudaFree(h->tick); cudaFree(h->elapsed); cudaFree(h->ext); cudaFree(h->lag); cudaFree(h->body_rec);
  cudaFree(h->env_params); cudaFree(h->ep_check); cudaFree(h->final_state); cudaFree(h->rr_dev); cudaFree(h->draws);
  cudaFree(h->push_dev); cudaFree(h->push_count); cudaFree(h->push_timer);
  cudaFree(h->delay_dev); cudaFree(h->delay_count); cudaFree(h->delay_delay); cudaFree(h->delay_command);
  cudaFree(h->delay_head);
  cudaFree(h->sense_dev); cudaFree(h->sense_count); cudaFree(h->sense_delay); cudaFree(h->sense_rows);
  cudaFree(h->sense_hist); cudaFree(h->sense_head);
  cudaFree(h->hist_dev); cudaFree(h->hist_ring); cudaFree(h->hist_head);
  cudaFree(h->drop_dev); cudaFree(h->drop_count); cudaFree(h->drop_prob); cudaFree(h->drop_held);
  cudaFree(h->tilt_dev); cudaFree(h->tilt_count); cudaFree(h->tilt_quat);
  cudaFree(h->enc_dev); cudaFree(h->enc_count); cudaFree(h->enc_offset);
  cudaFree(h->noise_dev); cudaFree(h->noise_count); cudaFree(h->noise_sigma); cudaFree(h->noise_fresh);
  cudaFree(h->vlim_dev); cudaFree(h->vlim_count); cudaFree(h->vlim_max);
  cudaFree(h->tsc_dev); cudaFree(h->tsc_count); cudaFree(h->tsc_scale);
  cudaFree(h->att_dev); cudaFree(h->att_count); cudaFree(h->att_gains); cudaFree(h->att_quat); cudaFree(h->att_bias);
  cudaFree(h->att_rep); cudaFree(h->att_vel);
  cudaFreeHost(h->h_fin); cudaFreeHost(h->h_act); cudaFreeHost(h->h_obs); cudaFreeHost(h->h_rew); cudaFreeHost(h->h_term); cudaFreeHost(h->h_trunc);
  cudaFree(h->d_act); cudaFree(h->d_obs); cudaFree(h->d_rew); cudaFree(h->d_term); cudaFree(h->d_trunc);
  for (int k = 0; k < kHostStreams; ++k)
    if (h->host_streams[k]) cudaStreamDestroy(h->host_streams[k]);
  for (int k = 0; k < 64; ++k)
    if (h->host_events[k]) cudaEventDestroy(h->host_events[k]);
  h->magic = 0;
  delete h;
}

int upkie_b200_num_envs(void* handle) {
  Handle* h = as_handle(handle);
  return h ? h->n : fail(UPKIE_B200_EINVAL, "invalid handle");
}

int upkie_b200_set_config(void* handle, const UpkieSimConfig* config) {
  Handle* h = as_handle(handle);
  if (!h || !config) return fail(UPKIE_B200_EINVAL, "set_config: invalid argument");
  h->final_valid = false;  // the stashed states no longer belong to the last step
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  std::string err;
  int rc = make_sim_params(h->model, *config, P, err);
  if (rc) return fail(rc, err);
  if (P.spine_mode != h->P.spine_mode) return fail(UPKIE_B200_EINVAL, "set_config: spine_mode is fixed at creation");
  if (h->P.reset_rand && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: reset randomisation needs joint_limits != 0");
  if (h->P.push && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: push randomisation needs joint_limits != 0");
  if (h->P.action_delay && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: action delay needs joint_limits != 0");
  if (h->P.action_delay && uint64_t(P.nb_substeps) * uint32_t(h->delay_ticks) < h->delay_high)
    return fail(UPKIE_B200_EINVAL, "set_config: nb_substeps below the action delay's substeps_high");
  if (h->P.obs_delay && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: observation delay needs joint_limits != 0");
  if (h->P.obs_delay && uint64_t(P.nb_substeps) * uint32_t(h->sense_ticks) < h->sense_high)
    return fail(UPKIE_B200_EINVAL, "set_config: nb_substeps below the observation delay's substeps_high");
  if (h->P.obs_delay && P.body_contacts)
    return fail(UPKIE_B200_EINVAL, "set_config: body_contacts has no observation-delay kernels");
  if (h->P.history && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: the observation history needs joint_limits != 0");
  if (h->P.history && P.body_contacts)
    return fail(UPKIE_B200_EINVAL, "set_config: body_contacts has no observation-history kernels");
  if (h->P.servo_dropout && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: servo dropouts need joint_limits != 0");
  if (h->P.servo_dropout && P.body_contacts)
    return fail(UPKIE_B200_EINVAL, "set_config: body_contacts has no servo-dropout kernels");
  if (h->P.imu_misalign && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: IMU misalignment needs joint_limits != 0");
  if (h->P.imu_misalign && P.body_contacts)
    return fail(UPKIE_B200_EINVAL, "set_config: body_contacts has no IMU-misalignment kernels");
  if (h->P.encoder_offset && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: encoder offsets need joint_limits != 0");
  if (h->P.encoder_offset && P.body_contacts)
    return fail(UPKIE_B200_EINVAL, "set_config: body_contacts has no encoder-offset kernels");
  if (h->P.servo_noise && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: servo noise needs joint_limits != 0");
  if (h->P.servo_noise && P.body_contacts)
    return fail(UPKIE_B200_EINVAL, "set_config: body_contacts has no servo-noise kernels");
  if (h->P.velocity_derate && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: velocity limits need joint_limits != 0");
  if (h->P.velocity_derate && P.body_contacts)
    return fail(UPKIE_B200_EINVAL, "set_config: body_contacts has no velocity-limit kernels");
  if (h->P.attitude_filter && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: the attitude filter needs joint_limits != 0");
  if (h->P.attitude_filter && P.body_contacts)
    return fail(UPKIE_B200_EINVAL, "set_config: body_contacts has no attitude-filter kernels");
  if (h->P.torque_scale && P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_config: torque scales need joint_limits != 0");
  if (h->P.torque_scale && P.body_contacts)
    return fail(UPKIE_B200_EINVAL, "set_config: body_contacts has no torque-scale kernels");
  if (h->P.attitude_filter) {
    // the bound holds for the gains every env holds (a narrower spec keeps each env's gains until its next reset, and
    // set_attitude_filter_state may set others) and for those the spec in force draws
    CUDA_TRY(cudaSetDevice(h->device));
    CUDA_TRY(cudaDeviceSynchronize());  // resets in flight may draw new gains
    std::vector<float> kp(size_t(h->n));
    CUDA_TRY(cudaMemcpy(kp.data(), h->att_gains, kp.size() * sizeof(float), cudaMemcpyDeviceToHost));
    float kp_max = h->att_spec.kp_high;
    for (float k : kp) kp_max = std::max(kp_max, k);
    if (!(double(kp_max) * double(P.h) <= 0.5))
      return fail(UPKIE_B200_EINVAL, "set_config: the attitude filter's largest kp (held by an env or the spec's "
                                     "kp_high) times dt / nb_substeps must stay <= 0.5");
  }
  if (P.body_contacts && !h->body_rec) {  // switched on after creation: the record buffer is allocated now
    CUDA_TRY(cudaSetDevice(h->device));
    CUDA_TRY(cudaMalloc(&h->body_rec, size_t(UPKIE_BODY_REC_DIM) * h->n_pad * sizeof(float)));
    CUDA_TRY(cudaMemset(h->body_rec, 0, size_t(UPKIE_BODY_REC_DIM) * h->n_pad * sizeof(float)));
  }
  P.body_rec = P.body_contacts ? h->body_rec : nullptr;
  P.body_rec_stride = h->n_pad;
  P.elapsed = h->elapsed;
  // the per-env parameter table stays: its values and its noise flags override the config's
  const uint32_t config_flags = noise_flags(P);
  if (h->env_params) {
    P.env_params = h->env_params;
    P.env_params_stride = h->n_pad;
    set_noise_flags(P, h->env_param_flags | h->rr_flags);
  }
  P.reset_rand = h->P.reset_rand;  // so does the reset randomisation
  P.push = h->P.push;              // and the push randomisation
  P.action_delay = h->P.action_delay;  // and the action delay
  P.obs_delay = h->P.obs_delay;        // and the observation delay
  P.history = h->P.history;            // and the observation history
  P.servo_dropout = h->P.servo_dropout;  // and the servo dropouts
  P.imu_misalign = h->P.imu_misalign;    // and the IMU misalignment
  P.encoder_offset = h->P.encoder_offset;  // and the encoder offsets
  P.servo_noise = h->P.servo_noise;        // and the servo noise
  P.velocity_derate = h->P.velocity_derate;  // and the velocity limits
  P.attitude_filter = h->P.attitude_filter;  // and the attitude filter
  P.torque_scale = h->P.torque_scale;        // and the torque scales
  if (P.max_episode_steps > 0 && P.max_episode_steps != h->P.max_episode_steps) {
    // a limit switched on or changed: episodes are timed from this call. The counts were not kept (no limit) or
    // were kept against another limit; steps enqueued before the call finish first.
    CUDA_TRY(cudaSetDevice(h->device));
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemset(h->elapsed, 0, size_t(h->n) * sizeof(uint32_t)));
    CUDA_TRY(cudaDeviceSynchronize());
  }
  // kernels read the parameter block by value at launch: steps already enqueued keep the old one
  h->P = P;
  h->config_flags = config_flags;
  return history_resize(h);  // a new nb_substeps changes the ring's size
}

int upkie_b200_set_env_params(void* handle, const float* rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  h->final_valid = false;  // the stashed states no longer belong to the last step
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaSetDevice(h->device));
  if (!rows) {
    if (h->P.reset_rand)
      return fail(UPKIE_B200_EINVAL, "set_env_params: reset randomisation writes into the table; turn it off first "
                                     "(upkie_b200_set_reset_randomization(NULL))");
    if (h->env_params) {
      CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may still read the table
      cudaFree(h->env_params);
      h->env_params = nullptr;
    }
    h->P.env_params = nullptr;
    h->P.env_params_stride = 0;
    set_noise_flags(h->P, h->config_flags);
    return UPKIE_B200_OK;
  }
  // validate first: a rejected table leaves the previous one (or none) in force
  if (!h->ep_check) CUDA_TRY(cudaMalloc(&h->ep_check, sizeof(uint32_t)));
  CUDA_TRY(cudaMemsetAsync(h->ep_check, 0, sizeof(uint32_t), s));
  k_env_params_check<<<(h->n + 127) / 128, 128, 0, s>>>(h->n, rows, h->ep_check);
  CUDA_TRY(cudaGetLastError());
  uint32_t flags = 0;
  CUDA_TRY(cudaMemcpyAsync(&flags, h->ep_check, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  if (flags & kEpInvalid)
    return fail(UPKIE_B200_EINVAL, "set_env_params: every value must be finite, and gains, friction and noise standard "
                                   "deviations >= 0");
  const size_t bytes = size_t(UPKIE_EP_DIM) * h->n_pad * sizeof(float);
  if (!h->env_params) {
    CUDA_TRY(cudaMalloc(&h->env_params, bytes));
    CUDA_TRY(cudaMemsetAsync(h->env_params, 0, bytes, s));
  }
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight on other streams may still read the previous table
  CUDA_TRY(ring_cols(rows, UPKIE_EP_DIM, h->n, h->n_pad, h->env_params, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  h->env_param_flags = flags;
  h->P.env_params = h->env_params;
  h->P.env_params_stride = h->n_pad;
  set_noise_flags(h->P, flags | h->rr_flags);
  return UPKIE_B200_OK;
}

int upkie_b200_set_reset_randomization(void* handle, const UpkieResetRandomization* spec) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  h->final_valid = false;  // the stash's layout follows the spec
  if (!spec) {
    // off: the kernels enqueued before keep the block they were launched with, which stays allocated; the values
    // in force and the noise flags they needed stay
    h->P.reset_rand = nullptr;
    return UPKIE_B200_OK;
  }
  if (h->P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_reset_randomization: needs joint_limits != 0 (the table kernels carry it)");
  const uint32_t flags = reset_rand_flags(*spec);
  if (flags & kEpInvalid)
    return fail(UPKIE_B200_EINVAL, "set_reset_randomization: every bound must be finite with low <= high, low >= 0 on "
                                   "gains, joint friction, noise standard deviations and the floor friction, and "
                                   "inertia bounds > -1; columns < UPKIE_RR_DIM");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the block
  if (!h->env_params) {
    CUDA_TRY(cudaMalloc(&h->env_params, size_t(UPKIE_EP_DIM) * h->n_pad * sizeof(float)));
    CUDA_TRY(cudaMemset(h->env_params, 0, size_t(UPKIE_EP_DIM) * h->n_pad * sizeof(float)));
    CUDA_TRY(env_params_from_config(h->P, h->n, 1, h->n_pad, h->env_params, nullptr));
    h->env_param_flags = h->config_flags;
    h->P.env_params = h->env_params;
    h->P.env_params_stride = h->n_pad;
  }
  if (!h->eps) {
    CUDA_TRY(cudaMalloc(&h->eps, size_t(h->n) * 6 * sizeof(float)));
    CUDA_TRY(cudaMemset(h->eps, 0, size_t(h->n) * 6 * sizeof(float)));
  }
  if (!h->mu) {
    CUDA_TRY(cudaMalloc(&h->mu, size_t(h->n) * sizeof(float)));
    CUDA_TRY(fill(h->n, h->mu, h->P.friction, nullptr));
  }
  if (!h->draws) {
    CUDA_TRY(cudaMalloc(&h->draws, size_t(h->n) * sizeof(uint32_t)));
    CUDA_TRY(cudaMemset(h->draws, 0, size_t(h->n) * sizeof(uint32_t)));
  }
  if (!h->rr_dev) CUDA_TRY(cudaMalloc(&h->rr_dev, sizeof(ResetRand)));
  ResetRand R;
  std::memset(&R, 0, sizeof(R));
  R.spec = *spec;
  R.draws = h->draws;
  R.table = h->env_params;
  R.stride = h->n_pad;
  R.eps = h->eps;
  R.mu = h->mu;
  CUDA_TRY(cudaMemcpy(h->rr_dev, &R, sizeof(R), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaDeviceSynchronize());
  // the noise models some drawn level may need; a spec that is replaced or turned off leaves its flags on (the levels
  // it drew stay in force)
  h->rr_flags |= flags;
  set_noise_flags(h->P, h->env_param_flags | h->rr_flags);
  h->P.reset_rand = h->rr_dev;
  return UPKIE_B200_OK;
}

int upkie_b200_get_draws(void* handle, uint32_t* draws, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !draws) return fail(UPKIE_B200_EINVAL, "get_draws: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(copy_or_zero(draws, h->draws, size_t(h->n) * sizeof(uint32_t), static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

int upkie_b200_set_draws(void* handle, const uint32_t* draws, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !draws) return fail(UPKIE_B200_EINVAL, "set_draws: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (!h->draws) CUDA_TRY(cudaMalloc(&h->draws, size_t(h->n) * sizeof(uint32_t)));
  CUDA_TRY(cudaMemcpyAsync(h->draws, draws, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                           static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

int upkie_b200_get_randomization(void* handle, float* friction, float* inertia_eps, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!friction && !inertia_eps) return UPKIE_B200_OK;
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // without buffers, the nominal values: the config's friction and zero epsilons
  if (friction && h->mu) CUDA_TRY(cudaMemcpyAsync(friction, h->mu, size_t(h->n) * sizeof(float), cudaMemcpyDeviceToDevice, s));
  else if (friction) CUDA_TRY(fill(h->n, friction, h->P.friction, s));
  if (inertia_eps) CUDA_TRY(copy_or_zero(inertia_eps, h->eps, size_t(h->n) * 6 * sizeof(float), s));
  return UPKIE_B200_OK;
}

int upkie_b200_get_env_params(void* handle, float* rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !rows) return fail(UPKIE_B200_EINVAL, "get_env_params: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // without a table, the config's values
  if (h->env_params) CUDA_TRY(ring_rows(h->env_params, UPKIE_EP_DIM, h->n, h->n_pad, rows, s));
  else CUDA_TRY(env_params_from_config(h->P, h->n, UPKIE_EP_DIM, 1, rows, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_autoreset(void* handle, int mode, uint64_t seed, uint64_t env_offset) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (mode < 0 || mode > 2) return fail(UPKIE_B200_EINVAL, "set_autoreset: mode must be 0 (disabled), 1 (next step) or 2 (same step)");
  h->final_valid = false;  // the stashed states no longer belong to the last step
  h->autoreset = mode;
  h->seed = seed;
  h->env_offset = env_offset;
  return UPKIE_B200_OK;
}

int upkie_b200_set_randomization(void* handle, const float* friction, const float* inertia_eps, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (h->P.reset_rand && (!friction || !inertia_eps))
    return fail(UPKIE_B200_EINVAL, "set_randomization: reset randomisation writes into both buffers; turn it off "
                                   "first (upkie_b200_set_reset_randomization(NULL)) to drop one");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaSetDevice(h->device));
  if (friction) {
    if (!h->mu) CUDA_TRY(cudaMalloc(&h->mu, size_t(h->n) * sizeof(float)));
    CUDA_TRY(cudaMemcpyAsync(h->mu, friction, size_t(h->n) * sizeof(float), cudaMemcpyDeviceToDevice, s));
  } else if (h->mu) {
    CUDA_TRY(cudaStreamSynchronize(s));
    cudaFree(h->mu);
    h->mu = nullptr;
  }
  if (inertia_eps) {
    if (!h->eps) CUDA_TRY(cudaMalloc(&h->eps, size_t(h->n) * 6 * sizeof(float)));
    CUDA_TRY(cudaMemcpyAsync(h->eps, inertia_eps, size_t(h->n) * 6 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  } else if (h->eps) {
    CUDA_TRY(cudaStreamSynchronize(s));
    cudaFree(h->eps);
    h->eps = nullptr;
  }
  return UPKIE_B200_OK;
}

int upkie_b200_reset(void* handle, const uint8_t* mask, const float* init_state, uint64_t seed, uint64_t env_offset,
                     void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  h->final_valid = false;  // the stashed states no longer belong to the last step
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  k_reset<<<grid_of(h->n), 128, 0, s>>>(h->P, h->n, h->n_pad, h->state, mask, init_state, h->eps, h->mu, h->err,
                                        h->done_prev, h->episode, seed, env_offset, h->lag, h->seed, h->env_offset,
                                        h->tick);
  CUDA_TRY(cudaGetLastError());
  // a reset sampled on the device counts an episode: it is not one the base-velocity post step has to carry out
  if (!init_state)
    CUDA_TRY(cudaMemcpyAsync(h->bv_episode, h->episode, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  return UPKIE_B200_OK;
}

int upkie_b200_step_servos(void* handle, const float* action, float* obs, float* reward, uint8_t* terminated,
                           uint8_t* truncated, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  return step_any(h, MODE_SERVOS, action, obs, reward, terminated, truncated, static_cast<cudaStream_t>(stream));
}

int upkie_b200_step_servos_compact(void* handle, const float* action, float* obs, uint8_t* terminated, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!action || !obs || !terminated) return fail(UPKIE_B200_EINVAL, "step_servos_compact: null buffer");
  CUDA_TRY(cudaSetDevice(h->device));
  return step_range(h, MODE_SERVOS, 0, h->n, action, obs, nullptr, terminated, nullptr, static_cast<cudaStream_t>(stream),
                    /*tile=*/true, /*persistent=*/false, /*compact=*/true);
}

int upkie_b200_step_servos_multicast(void* handle, const float* action, float* obs_mc, uint8_t* terminated_mc, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!action || !obs_mc || !terminated_mc) return fail(UPKIE_B200_EINVAL, "step_servos_multicast: null buffer");
  if (h->n % 32 != 0) return fail(UPKIE_B200_EINVAL, "step_servos_multicast: the number of envs must be a multiple of 32");
  if (((reinterpret_cast<uintptr_t>(action) | reinterpret_cast<uintptr_t>(obs_mc)) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(terminated_mc) & 3) != 0)
    return fail(UPKIE_B200_EINVAL, "step_servos_multicast: action / obs rows must be 16-byte, terminated 4-byte aligned");
  CUDA_TRY(cudaSetDevice(h->device));
  return step_range(h, MODE_SERVOS, 0, h->n, action, obs_mc, nullptr, terminated_mc, nullptr, static_cast<cudaStream_t>(stream),
                    /*tile=*/true, /*persistent=*/false, /*compact=*/true, /*multicast=*/true);
}

int upkie_b200_step_servos_peers(void* handle, const float* action, float* const* obs_ptrs,
                                 uint8_t* const* terminated_ptrs, int n_peers, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!action || !obs_ptrs || !terminated_ptrs) return fail(UPKIE_B200_EINVAL, "step_servos_peers: null buffer");
  if (n_peers < 1 || n_peers > UPKIE_MAX_PEERS) return fail(UPKIE_B200_EINVAL, "step_servos_peers: 1 <= n_peers <= UPKIE_MAX_PEERS");
  if (h->n % 32 != 0) return fail(UPKIE_B200_EINVAL, "step_servos_peers: the number of envs must be a multiple of 32");
  PeerPtrs pp;
  std::memset(&pp, 0, sizeof(pp));
  pp.n = n_peers;
  for (int p = 0; p < UPKIE_MAX_PEERS; ++p) {
    pp.obs[p] = p < n_peers ? obs_ptrs[p] : nullptr;
    pp.term[p] = p < n_peers ? terminated_ptrs[p] : nullptr;
    if (p < n_peers && (!pp.obs[p] || !pp.term[p] || (reinterpret_cast<uintptr_t>(pp.obs[p]) & 15) != 0 ||
                        (reinterpret_cast<uintptr_t>(pp.term[p]) & 3) != 0))
      return fail(UPKIE_B200_EINVAL, "step_servos_peers: slot pointers must be non-null, obs 16-byte and terminated 4-byte aligned");
  }
  if ((reinterpret_cast<uintptr_t>(action) & 15) != 0) return fail(UPKIE_B200_EINVAL, "step_servos_peers: action rows must be 16-byte aligned");
  CUDA_TRY(cudaSetDevice(h->device));
  return step_range(h, MODE_SERVOS, 0, h->n, action, pp.obs[0], nullptr, pp.term[0], nullptr, static_cast<cudaStream_t>(stream),
                    /*tile=*/true, /*persistent=*/false, /*compact=*/true, /*multicast=*/true, &pp);
}

namespace {
int fill_push(const Handle* h, const UpkiePush* push, PeerPtrs& pp, const char* who) {
  std::memset(&pp, 0, sizeof(pp));
  pp.deferred = 1;
  if (!push) return UPKIE_B200_OK;  // nothing to send
  if (push->n_peers < 0 || push->n_peers > UPKIE_MAX_PEERS) return fail(UPKIE_B200_EINVAL, std::string(who) + ": 0 <= n_peers <= UPKIE_MAX_PEERS");
  if (h->n % 32 != 0) return fail(UPKIE_B200_EINVAL, std::string(who) + ": the number of envs must be a multiple of 32");
  auto bad = [](const void* q, uintptr_t mask) { return !q || (reinterpret_cast<uintptr_t>(q) & mask) != 0; };
  if (push->src_obs) {
    if (bad(push->src_obs, 15) || bad(push->src_terminated, 3)) return fail(UPKIE_B200_EINVAL, std::string(who) + ": source slot misaligned or null");
    pp.src_obs = push->src_obs;
    pp.src_term = push->src_terminated;
    pp.n = push->n_peers;
    if (pp.n == 0) {
      if (bad(push->mc_obs, 15) || bad(push->mc_terminated, 3)) return fail(UPKIE_B200_EINVAL, std::string(who) + ": multicast slot misaligned or null");
      pp.mc_obs = push->mc_obs;
      pp.mc_term = push->mc_terminated;
    }
    for (int p = 0; p < pp.n; ++p) {
      if (bad(push->peer_obs[p], 15) || bad(push->peer_terminated[p], 3)) return fail(UPKIE_B200_EINVAL, std::string(who) + ": peer slot misaligned or null");
      pp.obs[p] = push->peer_obs[p];
      pp.term[p] = push->peer_terminated[p];
    }
  }
  return UPKIE_B200_OK;
}
}  // namespace

int upkie_b200_step_servos_push(void* handle, const float* action, float* obs, uint8_t* terminated,
                                const UpkiePush* push, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!action || !obs || !terminated) return fail(UPKIE_B200_EINVAL, "step_servos_push: null buffer");
  if (h->n % 32 != 0) return fail(UPKIE_B200_EINVAL, "step_servos_push: the number of envs must be a multiple of 32");
  if (((reinterpret_cast<uintptr_t>(action) | reinterpret_cast<uintptr_t>(obs)) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(terminated) & 3) != 0)
    return fail(UPKIE_B200_EINVAL, "step_servos_push: action / obs rows must be 16-byte, terminated 4-byte aligned");
  PeerPtrs pp;
  int rc = fill_push(h, push, pp, "step_servos_push");
  if (rc) return rc;
  CUDA_TRY(cudaSetDevice(h->device));
  return step_range(h, MODE_SERVOS, 0, h->n, action, obs, nullptr, terminated, nullptr, static_cast<cudaStream_t>(stream),
                    /*tile=*/true, /*persistent=*/false, /*compact=*/true, /*multicast=*/true, &pp);
}

int upkie_b200_push_rows(void* handle, const UpkiePush* push, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !push || !push->src_obs) return fail(UPKIE_B200_EINVAL, "push_rows: invalid argument");
  PeerPtrs pp;
  int rc = fill_push(h, push, pp, "push_rows");
  if (rc) return rc;
  CUDA_TRY(cudaSetDevice(h->device));
#if UPKIE_EXACT_BUILD
  CUDA_TRY(cudaErrorNotSupported);  // the exact-arithmetic library has no in-kernel rollout transport (build.py)
#else
  CUDA_TRY(launch_push_rows(pp, h->n, static_cast<cudaStream_t>(stream)));
#endif
  return UPKIE_B200_OK;
}

int upkie_b200_step_gyropod(void* handle, const float* action, int act_dim, float* obs, float* reward,
                            uint8_t* terminated, uint8_t* truncated, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (act_dim != 1 && act_dim != 2) return fail(UPKIE_B200_EINVAL, "step_gyropod: act_dim must be 1 (pendulum) or 2 (gyropod)");
  return step_any(h, act_dim == 2 ? MODE_GYROPOD : MODE_PENDULUM, action, obs, reward, terminated, truncated,
                  static_cast<cudaStream_t>(stream));
}

int upkie_b200_step_servos_host(void* handle, const float* action, float* obs, float* reward, uint8_t* terminated,
                                uint8_t* truncated) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  return step_host(h, MODE_SERVOS, action, obs, reward, terminated, truncated);
}
int upkie_b200_step_servos_host_compact(void* handle, const float* action, float* obs, uint8_t* terminated) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "step_servos_host_compact: bad handle");
  return step_host(h, MODE_SERVOS, action, obs, nullptr, terminated, nullptr, /*compact=*/true);
}

namespace {
int step_mode_of(int act_dim) {
  return act_dim == UPKIE_ACT_DIM ? MODE_SERVOS : (act_dim == 2 ? MODE_GYROPOD : (act_dim == 1 ? MODE_PENDULUM : -1));
}
}  // namespace

int upkie_b200_step(void* handle, int act_dim, const float* action, const UpkieStepOutputs* out, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  const int mode = step_mode_of(act_dim);
  if (mode < 0) return fail(UPKIE_B200_EINVAL, "step: act_dim must be 36 (servos), 2 (gyropod) or 1 (pendulum)");
  if (!out || !action || !out->obs || !out->terminated) return fail(UPKIE_B200_EINVAL, "step: null buffer");
  const bool compact = out->compact != 0;
  if (compact && mode != MODE_SERVOS) return fail(UPKIE_B200_EINVAL, "step: compact rows exist for servos only");
  CUDA_TRY(cudaSetDevice(h->device));
  bool stash = false;
  int rc = prepare_final_state(h, out->final_state, stash);
  if (rc) return rc;
  // compact rows: the TILE=1 kernels on device buffers, as upkie_b200_step_servos_compact
  rc = step_range(h, mode, 0, h->n, action, out->obs, out->reward, out->terminated, out->truncated,
                  static_cast<cudaStream_t>(stream), /*tile=*/compact, /*persistent=*/false, compact, false, nullptr,
                  out->final_obs, stash);
  h->final_valid = rc == UPKIE_B200_OK && stash;
  return rc;
}

int upkie_b200_step_host(void* handle, int act_dim, const float* action, const UpkieStepOutputs* out) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  const int mode = step_mode_of(act_dim);
  if (mode < 0) return fail(UPKIE_B200_EINVAL, "step_host: act_dim must be 36 (servos), 2 (gyropod) or 1 (pendulum)");
  if (!out) return fail(UPKIE_B200_EINVAL, "step_host: null outputs");
  const bool compact = out->compact != 0;
  if (compact && mode != MODE_SERVOS) return fail(UPKIE_B200_EINVAL, "step_host: compact rows exist for servos only");
  bool stash = false;
  int rc = prepare_final_state(h, out->final_state, stash);
  if (rc) return rc;
  rc = step_host(h, mode, action, out->obs, out->reward, out->terminated, out->truncated, compact, out->final_obs, stash);
  h->final_valid = rc == UPKIE_B200_OK && stash;
  return rc;
}

int upkie_b200_step_gyropod_host(void* handle, const float* action, int act_dim, float* obs, float* reward,
                                 uint8_t* terminated, uint8_t* truncated) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (act_dim != 1 && act_dim != 2) return fail(UPKIE_B200_EINVAL, "step_gyropod_host: act_dim must be 1 or 2");
  return step_host(h, act_dim == 2 ? MODE_GYROPOD : MODE_PENDULUM, action, obs, reward, terminated, truncated);
}

int upkie_b200_spine_obs(void* handle, float* out, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !out) return fail(UPKIE_B200_EINVAL, "spine_obs: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  // observation delay: the spine observation of the sensed states
  const float* state = h->P.obs_delay ? h->sense_rows : h->state;
  k_spine_obs<<<grid_of(h->n), 128, 0, static_cast<cudaStream_t>(stream)>>>(h->P, h->n, h->n_pad, state, h->lag, nullptr,
                                                                            0u, h->tick, h->env_offset, out, h->seed);
  CUDA_TRY(cudaGetLastError());
  return UPKIE_B200_OK;
}

int upkie_b200_final_spine_obs(void* handle, float* out, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !out) return fail(UPKIE_B200_EINVAL, "final_spine_obs: invalid argument");
  if (!h->final_valid)
    return fail(UPKIE_B200_EINVAL, "final_spine_obs: the last call that advanced or reset the simulator was not a "
                                   "same-step auto-reset step with final_state = 1");
  CUDA_TRY(cudaSetDevice(h->device));
  SimParams P = h->P;
  if (h->final_params) {
    // reset randomisation: the resets of that step redrew the table, the stash holds its pre-reset columns
    // UPKIE_EP_MEAS_NOISE .. UPKIE_EP_DIM - 1 (the only ones k_spine_obs reads): the launch's table is the stash,
    // shifted so that column k of env i is stash row (first parameter row + k - UPKIE_EP_MEAS_NOISE)
    const int row0 = h->lag ? kFinalRowsSpine : kFinalRows;
    P.env_params = h->final_state + size_t(row0 - UPKIE_EP_MEAS_NOISE) * h->n_pad;
    P.env_params_stride = h->n_pad;
  }
  const float* stash = h->final_state;
  k_spine_obs<<<grid_of(h->n), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      P, h->n, h->n_pad, stash + size_t(kFinalStateRow) * h->n_pad,
      h->lag ? stash + size_t(kFinalLagRow) * h->n_pad : nullptr,
      reinterpret_cast<const uint32_t*>(stash + size_t(kFinalMarkRow) * h->n_pad), h->final_gen, h->tick,
      h->env_offset, out, h->seed,
      h->P.attitude_filter ? stash + size_t(kFinalRows + (h->final_params ? kFinalParamCols : 0)) * h->n_pad : nullptr);
  CUDA_TRY(cudaGetLastError());
  return UPKIE_B200_OK;
}

int upkie_b200_reset_obs(void* handle, int obs_dim, float* obs, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !obs) return fail(UPKIE_B200_EINVAL, "reset_obs: invalid argument");
  if (obs_dim != 4 && obs_dim != 6 && obs_dim != UPKIE_OBS_DIM) return fail(UPKIE_B200_EINVAL, "reset_obs: obs_dim must be 4, 6 or 30");
  CUDA_TRY(cudaSetDevice(h->device));
  // observation delay: the observation of the sensed states (those of the envs a reset took are the post-reset state;
  // the others report their robot as the last step observed it)
  const float* state = h->P.obs_delay ? h->sense_rows : h->state;
  k_reset_obs<<<(h->n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(h->P, h->n, h->n_pad, state, h->tick, h->env_offset, obs_dim, obs, h->lag, h->seed);
  CUDA_TRY(cudaGetLastError());
  return UPKIE_B200_OK;
}

int upkie_b200_get_state(void* handle, float* state, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !state) return fail(UPKIE_B200_EINVAL, "get_state: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(ring_rows(h->state, UPKIE_STATE_DIM, h->n, h->n_pad, state, static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

int upkie_b200_set_state(void* handle, const float* state, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !state) return fail(UPKIE_B200_EINVAL, "set_state: invalid argument");
  h->final_valid = false;  // the stashed states no longer belong to the last step
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(ring_cols(state, UPKIE_STATE_DIM, h->n, h->n_pad, h->state, static_cast<cudaStream_t>(stream)));
  // observation delay: the sensors see the state set, without a lag behind it (every snapshot of a history too)
  if (h->P.obs_delay) {
    CUDA_TRY(cudaMemcpyAsync(h->sense_rows, h->state, size_t(UPKIE_STATE_DIM) * h->n_pad * sizeof(float),
                             cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
    if (h->sense_hist)
      CUDA_TRY(ring_resize(h->state, nullptr, 1, h->sense_hist, h->sense_ticks, UPKIE_STATE_DIM, h->n, h->n_pad, 0,
                           ~uint64_t(0), static_cast<cudaStream_t>(stream)));
  }
  // the servo dropouts latch the state set
  if (h->P.servo_dropout) CUDA_TRY(servo_dropout_latch(h, ~0u, static_cast<cudaStream_t>(stream)));
  // the attitude filter starts from the state set, without an error (before the history, which reports it)
  if (h->P.attitude_filter) {
    k_attitude_init<<<grid_of(h->n), 128, 0, static_cast<cudaStream_t>(stream)>>>(h->P, h->n, h->n_pad, h->state,
                                                                                 false, 0.f, 0.f);
    CUDA_TRY(cudaGetLastError());
  }
  // the observation history restarts from the state set
  if (h->P.history) {
    k_history_fill<<<grid_of(h->n), 128, 0, static_cast<cudaStream_t>(stream)>>>(
        h->P, h->P.history, h->n, h->n_pad, h->state, h->tick, h->seed, h->env_offset);
    CUDA_TRY(cudaGetLastError());
  }
  return UPKIE_B200_OK;
}

int upkie_b200_get_body_contacts(void* handle, float* rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !rows) return fail(UPKIE_B200_EINVAL, "get_body_contacts: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // without body contacts, zeros
  if (h->P.body_rec) CUDA_TRY(ring_rows(h->P.body_rec, UPKIE_BODY_REC_DIM, h->n, h->n_pad, rows, s));
  else CUDA_TRY(cudaMemsetAsync(rows, 0, size_t(h->n) * UPKIE_BODY_REC_DIM * sizeof(float), s));
  return UPKIE_B200_OK;
}

int upkie_b200_get_lag(void* handle, float* lag_rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !lag_rows) return fail(UPKIE_B200_EINVAL, "get_lag: invalid argument");
  if (!h->lag) return fail(UPKIE_B200_EINVAL, "get_lag: the handle was not created with spine_mode");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(ring_rows(h->lag, UPKIE_LAG_DIM, h->n, h->n_pad, lag_rows, static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}
int upkie_b200_set_lag(void* handle, const float* lag_rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !lag_rows) return fail(UPKIE_B200_EINVAL, "set_lag: invalid argument");
  if (!h->lag) return fail(UPKIE_B200_EINVAL, "set_lag: the handle was not created with spine_mode");
  h->final_valid = false;  // the stashed states no longer belong to the last step
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(ring_cols(lag_rows, UPKIE_LAG_DIM, h->n, h->n_pad, h->lag, static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

int upkie_b200_set_external_forces(void* handle, const float* force, uint32_t local_mask, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "set_external_forces: invalid handle");
  if (h->P.push && ((local_mask >> h->push_body) & 1u))
    return fail(UPKIE_B200_EINVAL, "set_external_forces: the push randomisation pushes this body in the world frame; "
                                   "its bit of local_mask must be 0");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  h->ext_local = local_mask;
  if (!force) {
    if (h->ext) {
      CUDA_TRY(cudaStreamSynchronize(s));
      cudaFree(h->ext);
      h->ext = nullptr;
    }
    return UPKIE_B200_OK;
  }
  if (!h->ext) {
    CUDA_TRY(cudaMalloc(&h->ext, size_t(3 * UPKIE_NB) * h->n_pad * sizeof(float)));
    CUDA_TRY(cudaMemsetAsync(h->ext, 0, size_t(3 * UPKIE_NB) * h->n_pad * sizeof(float), s));
  }
  CUDA_TRY(ring_cols(force, 3 * UPKIE_NB, h->n, h->n_pad, h->ext, s));
  return UPKIE_B200_OK;
}

namespace {
// the per-env push state, zeros on a handle that has none yet
int alloc_push_state(Handle* h) {
  if (h->push_count) return UPKIE_B200_OK;
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  CUDA_TRY(alloc_zeroed({{reinterpret_cast<void**>(&h->push_count), bytes},
                         {reinterpret_cast<void**>(&h->push_timer), bytes}}));
  return UPKIE_B200_OK;
}
}  // namespace

int upkie_b200_set_push_randomization(void* handle, const UpkiePushRandomization* spec) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!spec) {
    // off: the kernels enqueued before keep the block they were launched with, which stays allocated
    h->P.push = nullptr;
    return UPKIE_B200_OK;
  }
  const UpkiePushRandomization& s = *spec;
  if (!push_spec_valid(s))
    return fail(UPKIE_B200_EINVAL, "set_push_randomization: body must be 0 .. UPKIE_NB - 1, step bounds low <= high <= "
                                   "UPKIE_PUSH_MAX_STEPS with duration_low >= 1, force bounds finite with low <= high");
  if (h->P.joint_limits == 0)
    return fail(UPKIE_B200_EINVAL, "set_push_randomization: needs joint_limits != 0 (the pushes run in the table and "
                                   "body-contact kernels)");
  if (h->P.spine_mode)
    return fail(UPKIE_B200_EINVAL, "set_push_randomization: spine_mode cycles take no external forces");
  if ((h->ext_local >> s.body) & 1u)
    return fail(UPKIE_B200_EINVAL, "set_push_randomization: the forces of set_external_forces on this body are in its "
                                   "body frame (local_mask); pushes are world-frame");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the block
  if (alloc_push_state(h)) return UPKIE_B200_ECUDA;
  if (!h->push_dev) CUDA_TRY(cudaMalloc(&h->push_dev, sizeof(PushRand)));
  PushRand R;
  std::memset(&R, 0, sizeof(R));
  R.spec = s;
  R.count = h->push_count;
  R.timer = h->push_timer;
  CUDA_TRY(cudaMemcpy(h->push_dev, &R, sizeof(R), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaDeviceSynchronize());
  h->push_body = s.body;
  h->P.push = h->push_dev;
  return UPKIE_B200_OK;
}

int upkie_b200_get_push_forces(void* handle, float* force, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !force) return fail(UPKIE_B200_EINVAL, "get_push_forces: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  k_push_forces<<<grid_of(h->n), 128, 0, static_cast<cudaStream_t>(stream)>>>(h->P.push, h->n, h->seed, h->env_offset,
                                                                              force);
  CUDA_TRY(cudaGetLastError());
  return UPKIE_B200_OK;
}

int upkie_b200_get_push_state(void* handle, uint32_t* count, uint32_t* timer, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !timer) return fail(UPKIE_B200_EINVAL, "get_push_state: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  CUDA_TRY(copy_or_zero(count, h->push_count, bytes, s));
  CUDA_TRY(copy_or_zero(timer, h->push_timer, bytes, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_push_state(void* handle, const uint32_t* count, const uint32_t* timer, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !timer) return fail(UPKIE_B200_EINVAL, "set_push_state: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (alloc_push_state(h)) return UPKIE_B200_ECUDA;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  CUDA_TRY(cudaMemcpyAsync(h->push_count, count, bytes, cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(h->push_timer, timer, bytes, cudaMemcpyDeviceToDevice, s));
  return UPKIE_B200_OK;
}

namespace {
// the per-env action-delay state: counters 0, delays 0 and stop rows on a handle that has none yet
// (the three buffers are set together: a failure frees what was allocated, so that a handle holds all or none)
int alloc_delay_state(Handle* h) {
  if (h->delay_count) return UPKIE_B200_OK;
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  cudaError_t e = alloc_zeroed({{reinterpret_cast<void**>(&h->delay_count), bytes},
                                {reinterpret_cast<void**>(&h->delay_delay), bytes},
                                {reinterpret_cast<void**>(&h->delay_head), bytes},
                                {reinterpret_cast<void**>(&h->delay_command),
                                 size_t(UPKIE_ACT_DIM) * h->n_pad * sizeof(float)}});
  if (e == cudaSuccess) e = stop_rows(h->n, 1, h->n_pad, h->delay_command, nullptr);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(UPKIE_B200_ECUDA, std::string("action delay state: ") + cudaGetErrorString(e));
  h->delay_ticks = 1;
  return UPKIE_B200_OK;
}
}  // namespace

namespace {
// a history of `ticks` rows [ticks][dim][n_pad] in place of `*ring` ([*cur][dim][n_pad], next writes *head): the newest
// min(ticks, *cur) rows in age order, the ages added stop rows (stop) or copies of the oldest, every next write row 0
int resize_ring(Handle* h, float** ring, uint32_t* head, int* cur, int ticks, int dim, int stop, const char* what) {
  if (ticks == *cur) return UPKIE_B200_OK;
  float* next = nullptr;
  cudaError_t e = cudaMalloc(&next, size_t(ticks) * dim * h->n_pad * sizeof(float));
  if (e == cudaSuccess)
    e = ring_resize(*ring, head, *cur, next, ticks, dim, h->n, h->n_pad, stop, ~uint64_t(0), nullptr);
  if (e == cudaSuccess) e = cudaMemset(head, 0, size_t(h->n) * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    cudaFree(next);
    return fail(UPKIE_B200_ECUDA, std::string(what) + cudaGetErrorString(e));
  }
  cudaFree(*ring);
  *ring = next;
  *cur = ticks;
  return UPKIE_B200_OK;
}
}  // namespace

int upkie_b200_set_action_delay(void* handle, const UpkieActionDelay* spec) {
  return upkie_b200_set_action_delay_ticks(handle, spec, 1);
}

int upkie_b200_set_action_delay_ticks(void* handle, const UpkieActionDelay* spec, uint32_t max_ticks) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!spec) {
    // off: the kernels enqueued before keep the block they were launched with, which stays allocated
    h->P.action_delay = nullptr;
    h->delay_high = 0;
    return UPKIE_B200_OK;
  }
  if (max_ticks == 0 || max_ticks > UPKIE_MAX_DELAY_TICKS)
    return fail(UPKIE_B200_EINVAL, "set_action_delay: max_ticks outside 1 .. UPKIE_MAX_DELAY_TICKS");
  if (const char* why = action_delay_spec_error(*spec, h->P, max_ticks)) return fail(UPKIE_B200_EINVAL, why);
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the block
  if (alloc_delay_state(h)) return UPKIE_B200_ECUDA;
  if (resize_ring(h, &h->delay_command, h->delay_head, &h->delay_ticks, int(max_ticks), UPKIE_ACT_DIM, 1,
                  "action delay history: "))
    return UPKIE_B200_ECUDA;
  if (!h->delay_dev) CUDA_TRY(cudaMalloc(&h->delay_dev, sizeof(ActionDelay)));
  ActionDelay A;
  std::memset(&A, 0, sizeof(A));
  A.spec = *spec;
  A.count = h->delay_count;
  A.delay = h->delay_delay;
  A.command = h->delay_command;
  A.stride = h->n_pad;
  A.ticks = h->delay_ticks;
  A.head = h->delay_head;
  CUDA_TRY(cudaMemcpy(h->delay_dev, &A, sizeof(A), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaDeviceSynchronize());
  h->delay_high = spec->substeps_high;
  h->P.action_delay = h->delay_dev;
  return UPKIE_B200_OK;
}

int upkie_b200_get_action_delay_state(void* handle, uint32_t* count, uint32_t* delay, float* command, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !delay || !command) return fail(UPKIE_B200_EINVAL, "get_action_delay_state: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  CUDA_TRY(copy_or_zero(count, h->delay_count, bytes, s));
  CUDA_TRY(copy_or_zero(delay, h->delay_delay, bytes, s));
  if (h->delay_command)  // the previous tick's command: age 0 of the history
    CUDA_TRY(ring_rows(h->delay_command, UPKIE_ACT_DIM, h->n, h->n_pad, command, s, h->delay_head, h->delay_ticks, 1));
  else
    CUDA_TRY(stop_rows(h->n, UPKIE_ACT_DIM, 1, command, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_action_delay_state(void* handle, const uint32_t* count, const uint32_t* delay, const float* command,
                                      void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !delay || !command) return fail(UPKIE_B200_EINVAL, "set_action_delay_state: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (alloc_delay_state(h)) return UPKIE_B200_ECUDA;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  CUDA_TRY(cudaMemcpyAsync(h->delay_count, count, bytes, cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(h->delay_delay, delay, bytes, cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_cols(command, UPKIE_ACT_DIM, h->n, h->n_pad, h->delay_command, s, h->delay_head, h->delay_ticks, 1));
  return UPKIE_B200_OK;
}

int upkie_b200_get_action_delay_history(void* handle, float* commands, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !commands) return fail(UPKIE_B200_EINVAL, "get_action_delay_history: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (h->delay_command)
    CUDA_TRY(ring_rows(h->delay_command, UPKIE_ACT_DIM, h->n, h->n_pad, commands, s, h->delay_head, h->delay_ticks,
                       h->delay_ticks));
  else
    CUDA_TRY(stop_rows(h->n, UPKIE_ACT_DIM, 1, commands, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_action_delay_history(void* handle, const float* commands, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !commands) return fail(UPKIE_B200_EINVAL, "set_action_delay_history: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (alloc_delay_state(h)) return UPKIE_B200_ECUDA;
  CUDA_TRY(ring_cols(commands, UPKIE_ACT_DIM, h->n, h->n_pad, h->delay_command, static_cast<cudaStream_t>(stream),
                     h->delay_head, h->delay_ticks, h->delay_ticks));
  return UPKIE_B200_OK;
}

namespace {
// the per-env observation-delay state: counters 0, delays 0 and the sensed rows filled from the current state on a
// handle that has none yet (the three buffers are set together: a failure frees what was allocated)
int alloc_sense_state(Handle* h) {
  if (h->sense_count) return UPKIE_B200_OK;
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  const size_t row_bytes = size_t(UPKIE_STATE_DIM) * h->n_pad * sizeof(float);
  cudaError_t e = cudaDeviceSynchronize();  // the state of the steps in flight
  if (e == cudaSuccess)
    e = alloc_zeroed({{reinterpret_cast<void**>(&h->sense_count), bytes},
                      {reinterpret_cast<void**>(&h->sense_delay), bytes},
                      {reinterpret_cast<void**>(&h->sense_head), bytes},
                      {reinterpret_cast<void**>(&h->sense_rows), row_bytes}});
  if (e == cudaSuccess) e = cudaMemcpy(h->sense_rows, h->state, row_bytes, cudaMemcpyDeviceToDevice);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(UPKIE_B200_ECUDA, std::string("observation delay state: ") + cudaGetErrorString(e));
  h->sense_ticks = 1;
  return UPKIE_B200_OK;
}
}  // namespace

int upkie_b200_set_observation_delay(void* handle, const UpkieObservationDelay* spec) {
  return upkie_b200_set_observation_delay_ticks(handle, spec, 1);
}

namespace {
// the snapshot history of depth `ticks` (1: none, the sensed rows are the newest snapshot): the newest min(ticks, K)
// snapshots in age order, the ages added copies of the oldest
int resize_sense_history(Handle* h, int ticks) {
  if (ticks == h->sense_ticks) return UPKIE_B200_OK;
  const char* what = "observation delay history: ";
  if (ticks == 1) {  // the newest snapshot's sensed columns become the sensed rows
    uint64_t sensed = 0;
    for (int k = 0; k < UPKIE_STATE_DIM; ++k)
      if (obs_delay_sensed(k)) sensed |= uint64_t(1) << k;
    cudaError_t e = ring_resize(h->sense_hist, h->sense_head, h->sense_ticks, h->sense_rows, 1, UPKIE_STATE_DIM, h->n,
                                h->n_pad, 0, sensed, nullptr);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return fail(UPKIE_B200_ECUDA, std::string(what) + cudaGetErrorString(e));
    cudaFree(h->sense_hist);
    h->sense_hist = nullptr;
    h->sense_ticks = 1;
    return UPKIE_B200_OK;
  }
  if (h->sense_ticks == 1) {  // every snapshot of the new ring starts as a copy of the sensed rows
    float* hist = nullptr;
    cudaError_t e = cudaMalloc(&hist, size_t(ticks) * UPKIE_STATE_DIM * h->n_pad * sizeof(float));
    if (e == cudaSuccess)
      e = ring_resize(h->sense_rows, nullptr, 1, hist, ticks, UPKIE_STATE_DIM, h->n, h->n_pad, 0, ~uint64_t(0), nullptr);
    if (e == cudaSuccess) e = cudaMemset(h->sense_head, 0, size_t(h->n) * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
      cudaFree(hist);
      return fail(UPKIE_B200_ECUDA, std::string(what) + cudaGetErrorString(e));
    }
    h->sense_hist = hist;
    h->sense_ticks = ticks;
    return UPKIE_B200_OK;
  }
  return resize_ring(h, &h->sense_hist, h->sense_head, &h->sense_ticks, ticks, UPKIE_STATE_DIM, 0, what);
}
}  // namespace

int upkie_b200_set_observation_delay_ticks(void* handle, const UpkieObservationDelay* spec, uint32_t max_ticks) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!spec) {
    // off: the kernels enqueued before keep the block they were launched with, which stays allocated
    h->P.obs_delay = nullptr;
    h->sense_high = 0;
    return UPKIE_B200_OK;
  }
  if (max_ticks == 0 || max_ticks > UPKIE_MAX_DELAY_TICKS)
    return fail(UPKIE_B200_EINVAL, "set_observation_delay: max_ticks outside 1 .. UPKIE_MAX_DELAY_TICKS");
  if (const char* why = obs_delay_spec_error(*spec, h->P, max_ticks)) return fail(UPKIE_B200_EINVAL, why);
  if (h->P.servo_noise && h->P.servo_dropout)
    return fail(UPKIE_B200_EINVAL, "set_observation_delay: not with both servo noise and servo dropouts (a delayed "
                                   "snapshot does not record which of its replies were held)");
  if (h->P.attitude_filter && max_ticks > 1)
    return fail(UPKIE_B200_EINVAL, "set_observation_delay_ticks: not more than one tick with an attitude filter (the "
                                   "report of a deeper delay would need a ring of estimates)");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the block
  // the attitude filter: the sensed rows start from the state (below), and the report from the estimate
  if (h->P.attitude_filter && !h->P.obs_delay)
    CUDA_TRY(cudaMemcpy(h->att_rep, h->att_quat, size_t(4) * h->n_pad * sizeof(float), cudaMemcpyDeviceToDevice));
  const bool allocated = h->sense_rows != nullptr;
  if (alloc_sense_state(h)) return UPKIE_B200_ECUDA;  // a first allocation fills the rows from the state
  if (resize_sense_history(h, int(max_ticks))) return UPKIE_B200_ECUDA;
  if (allocated && !h->P.obs_delay) {
    // turned on again: the sensors did not follow the robot while the delay was off, so the rows (and every snapshot
    // of a history) start from the current state (its IMU velocity is what the next snapshot differentiates against);
    // counters and delays stay
    CUDA_TRY(cudaMemcpy(h->sense_rows, h->state, size_t(UPKIE_STATE_DIM) * h->n_pad * sizeof(float),
                        cudaMemcpyDeviceToDevice));
    if (h->sense_hist)
      CUDA_TRY(ring_resize(h->state, nullptr, 1, h->sense_hist, h->sense_ticks, UPKIE_STATE_DIM, h->n, h->n_pad, 0,
                           ~uint64_t(0), nullptr));
  }
  if (!h->sense_dev) CUDA_TRY(cudaMalloc(&h->sense_dev, sizeof(ObsDelay)));
  ObsDelay O;
  std::memset(&O, 0, sizeof(O));
  O.spec = *spec;
  O.count = h->sense_count;
  O.delay = h->sense_delay;
  O.rows = h->sense_rows;
  O.stride = h->n_pad;
  O.ticks = h->sense_ticks;
  O.hist = h->sense_hist;
  O.head = h->sense_head;
  CUDA_TRY(cudaMemcpy(h->sense_dev, &O, sizeof(O), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaDeviceSynchronize());
  h->sense_high = spec->substeps_high;
  h->P.obs_delay = h->sense_dev;
  return history_resize(h);  // a new depth changes the observation history's ring
}

int upkie_b200_get_observation_delay_state(void* handle, uint32_t* count, uint32_t* delay, float* rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !delay || !rows)
    return fail(UPKIE_B200_EINVAL, "get_observation_delay_state: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  CUDA_TRY(copy_or_zero(count, h->sense_count, bytes, s));
  CUDA_TRY(copy_or_zero(delay, h->sense_delay, bytes, s));
  // a handle without a state: the current state, what its first spec would fill the rows with
  CUDA_TRY(ring_rows(h->sense_rows ? h->sense_rows : h->state, UPKIE_STATE_DIM, h->n, h->n_pad, rows, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_observation_delay_state(void* handle, const uint32_t* count, const uint32_t* delay,
                                           const float* rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !delay || !rows)
    return fail(UPKIE_B200_EINVAL, "set_observation_delay_state: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (alloc_sense_state(h)) return UPKIE_B200_ECUDA;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  CUDA_TRY(cudaMemcpyAsync(h->sense_count, count, bytes, cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(h->sense_delay, delay, bytes, cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_cols(rows, UPKIE_STATE_DIM, h->n, h->n_pad, h->sense_rows, s));
  return UPKIE_B200_OK;
}

int upkie_b200_get_observation_delay_history(void* handle, float* rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !rows) return fail(UPKIE_B200_EINVAL, "get_observation_delay_history: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (h->sense_hist)
    CUDA_TRY(ring_rows(h->sense_hist, UPKIE_STATE_DIM, h->n, h->n_pad, rows, s, h->sense_head, h->sense_ticks,
                       h->sense_ticks));
  else  // depth 1: the sensed rows are the newest snapshot (as get_observation_delay_state)
    CUDA_TRY(ring_rows(h->sense_rows ? h->sense_rows : h->state, UPKIE_STATE_DIM, h->n, h->n_pad, rows, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_observation_delay_history(void* handle, const float* rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !rows) return fail(UPKIE_B200_EINVAL, "set_observation_delay_history: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (alloc_sense_state(h)) return UPKIE_B200_ECUDA;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (h->sense_hist)
    CUDA_TRY(ring_cols(rows, UPKIE_STATE_DIM, h->n, h->n_pad, h->sense_hist, s, h->sense_head, h->sense_ticks,
                       h->sense_ticks));
  else
    CUDA_TRY(ring_cols(rows, UPKIE_STATE_DIM, h->n, h->n_pad, h->sense_rows, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_servo_dropout(void* handle, const UpkieServoDropout* spec) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!spec) {
    if (h->P.servo_dropout) {
      CUDA_TRY(cudaSetDevice(h->device));
      CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may use the per-env state
      h->P.servo_dropout = nullptr;
      cudaFree(h->drop_count);
      cudaFree(h->drop_prob);
      cudaFree(h->drop_held);
      h->drop_count = nullptr;
      h->drop_prob = nullptr;
      h->drop_held = nullptr;
    }
    return UPKIE_B200_OK;
  }
  if (const char* why = servo_dropout_spec_error(*spec, h->P)) return fail(UPKIE_B200_EINVAL, why);
  if (h->P.servo_noise && h->P.obs_delay)
    return fail(UPKIE_B200_EINVAL, "set_servo_dropout: not with both servo noise and an observation delay (a delayed "
                                   "snapshot does not record which of its replies were held)");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the device block
  // the servos the held rows have not followed latch the current state: every servo when the feature is switched on
  // (zero counters and probabilities), the servos a replaced spec adds to the mask (the kernels latch masked servos
  // only, so an unmasked servo's rows hold its last reset)
  uint32_t latch = ~0u;
  if (!h->P.servo_dropout) {
    const size_t bytes = size_t(h->n) * sizeof(uint32_t);
    CUDA_TRY(alloc_zeroed({{reinterpret_cast<void**>(&h->drop_count), bytes},
                           {reinterpret_cast<void**>(&h->drop_prob), bytes},
                           {reinterpret_cast<void**>(&h->drop_held), size_t(kServoHeldRows) * h->n_pad * sizeof(float)}}));
  } else {
    latch = spec->joint_mask & ~h->drop_mask;
  }
  CUDA_TRY(servo_dropout_latch(h, latch, nullptr));
  h->drop_mask = spec->joint_mask;
  if (!h->drop_dev) CUDA_TRY(cudaMalloc(&h->drop_dev, sizeof(ServoDropout)));
  ServoDropout D;
  std::memset(&D, 0, sizeof(D));
  D.spec = *spec;
  D.count = h->drop_count;
  D.prob = h->drop_prob;
  D.held = h->drop_held;
  D.stride = h->n_pad;
  CUDA_TRY(cudaMemcpy(h->drop_dev, &D, sizeof(D), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaDeviceSynchronize());
  h->P.servo_dropout = h->drop_dev;
  return UPKIE_B200_OK;
}

int upkie_b200_get_servo_dropout_state(void* handle, uint32_t* count, float* prob, float* held, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !prob || !held) return fail(UPKIE_B200_EINVAL, "get_servo_dropout_state: invalid argument");
  if (!h->P.servo_dropout)
    return fail(UPKIE_B200_EINVAL, "get_servo_dropout_state: no servo dropouts are set (upkie_b200_set_servo_dropout)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  CUDA_TRY(cudaMemcpyAsync(count, h->drop_count, bytes, cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(prob, h->drop_prob, bytes, cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_rows(h->drop_held, kServoHeldRows, h->n, h->n_pad, held, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_servo_dropout_state(void* handle, const uint32_t* count, const float* prob, const float* held,
                                       void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !prob || !held) return fail(UPKIE_B200_EINVAL, "set_servo_dropout_state: invalid argument");
  if (!h->P.servo_dropout)
    return fail(UPKIE_B200_EINVAL, "set_servo_dropout_state: no servo dropouts are set (upkie_b200_set_servo_dropout)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t bytes = size_t(h->n) * sizeof(uint32_t);
  CUDA_TRY(cudaMemcpyAsync(h->drop_count, count, bytes, cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(h->drop_prob, prob, bytes, cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_cols(held, kServoHeldRows, h->n, h->n_pad, h->drop_held, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_imu_misalignment(void* handle, const UpkieImuMisalignment* spec) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!spec) {
    if (h->P.imu_misalign) {
      CUDA_TRY(cudaSetDevice(h->device));
      CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may use the per-env state
      h->P.imu_misalign = nullptr;
      cudaFree(h->tilt_count);
      cudaFree(h->tilt_quat);
      h->tilt_count = nullptr;
      h->tilt_quat = nullptr;
    }
    return UPKIE_B200_OK;
  }
  if (const char* why = imu_misalignment_spec_error(*spec, h->P)) return fail(UPKIE_B200_EINVAL, why);
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the device block
  if (!h->P.imu_misalign) {
    // switched on: zero counters, and the identity as every env's misalignment until its next reset
    CUDA_TRY(alloc_zeroed({{reinterpret_cast<void**>(&h->tilt_count), size_t(h->n) * sizeof(uint32_t)},
                           {reinterpret_cast<void**>(&h->tilt_quat), size_t(4) * h->n_pad * sizeof(float)}}));
    CUDA_TRY(fill(h->n, h->tilt_quat, 1.f, nullptr));
  }
  if (!h->tilt_dev) CUDA_TRY(cudaMalloc(&h->tilt_dev, sizeof(ImuMisalign)));
  ImuMisalign M;
  std::memset(&M, 0, sizeof(M));
  M.spec = *spec;
  M.count = h->tilt_count;
  M.quat = h->tilt_quat;
  M.stride = h->n_pad;
  CUDA_TRY(cudaMemcpy(h->tilt_dev, &M, sizeof(M), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaDeviceSynchronize());
  h->P.imu_misalign = h->tilt_dev;
  return UPKIE_B200_OK;
}

int upkie_b200_get_imu_misalignment_state(void* handle, uint32_t* count, float* quat, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !quat) return fail(UPKIE_B200_EINVAL, "get_imu_misalignment_state: invalid argument");
  if (!h->P.imu_misalign)
    return fail(UPKIE_B200_EINVAL,
                "get_imu_misalignment_state: no IMU misalignment is set (upkie_b200_set_imu_misalignment)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemcpyAsync(count, h->tilt_count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_rows(h->tilt_quat, 4, h->n, h->n_pad, quat, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_imu_misalignment_state(void* handle, const uint32_t* count, const float* quat, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !quat) return fail(UPKIE_B200_EINVAL, "set_imu_misalignment_state: invalid argument");
  if (!h->P.imu_misalign)
    return fail(UPKIE_B200_EINVAL,
                "set_imu_misalignment_state: no IMU misalignment is set (upkie_b200_set_imu_misalignment)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // every quaternion must be a rotation: read back (after the caller's work on the stream) and checked here
  std::vector<float> q(size_t(h->n) * 4);
  CUDA_TRY(cudaMemcpyAsync(q.data(), quat, q.size() * sizeof(float), cudaMemcpyDefault, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (int i = 0; i < h->n; ++i) {
    const double w = q[4 * i], x = q[4 * i + 1], y = q[4 * i + 2], z = q[4 * i + 3];
    const double norm = std::sqrt(w * w + x * x + y * y + z * z);
    if (!(std::fabs(norm - 1.0) <= 1e-5))
      return fail(UPKIE_B200_EINVAL, "set_imu_misalignment_state: every quaternion must be unit (within 1e-5)");
  }
  CUDA_TRY(cudaMemcpyAsync(h->tilt_count, count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_cols(quat, 4, h->n, h->n_pad, h->tilt_quat, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_encoder_offset(void* handle, const UpkieEncoderOffset* spec) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!spec) {
    if (h->P.encoder_offset) {
      CUDA_TRY(cudaSetDevice(h->device));
      CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may use the per-env state
      h->P.encoder_offset = nullptr;
      cudaFree(h->enc_count);
      cudaFree(h->enc_offset);
      h->enc_count = nullptr;
      h->enc_offset = nullptr;
      h->enc_mask = 0;
    }
    return UPKIE_B200_OK;
  }
  if (const char* why = encoder_offset_spec_error(*spec, h->P)) return fail(UPKIE_B200_EINVAL, why);
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the device block
  if (!h->P.encoder_offset) {
    // switched on: zero counters, and zero offsets until each env's next reset
    CUDA_TRY(alloc_zeroed({{reinterpret_cast<void**>(&h->enc_count), size_t(h->n) * sizeof(uint32_t)},
                           {reinterpret_cast<void**>(&h->enc_offset), size_t(UPKIE_NJ) * h->n_pad * sizeof(float)}}));
  } else {
    // a replacement: the joints it drops from the mask have no offset from now on
    for (int j = 0; j < UPKIE_NJ; ++j)
      if (((h->enc_mask & ~spec->joint_mask) >> j) & 1u)
        CUDA_TRY(cudaMemset(h->enc_offset + size_t(j) * h->n_pad, 0, size_t(h->n_pad) * sizeof(float)));
  }
  if (!h->enc_dev) CUDA_TRY(cudaMalloc(&h->enc_dev, sizeof(EncoderOffset)));
  EncoderOffset E;
  std::memset(&E, 0, sizeof(E));
  E.spec = *spec;
  E.count = h->enc_count;
  E.offset = h->enc_offset;
  E.stride = h->n_pad;
  CUDA_TRY(cudaMemcpy(h->enc_dev, &E, sizeof(E), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaDeviceSynchronize());
  h->P.encoder_offset = h->enc_dev;
  h->enc_mask = spec->joint_mask;
  return UPKIE_B200_OK;
}

int upkie_b200_get_encoder_offset_state(void* handle, uint32_t* count, float* offset, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !offset) return fail(UPKIE_B200_EINVAL, "get_encoder_offset_state: invalid argument");
  if (!h->P.encoder_offset)
    return fail(UPKIE_B200_EINVAL, "get_encoder_offset_state: no encoder offsets are set (upkie_b200_set_encoder_offset)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemcpyAsync(count, h->enc_count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_rows(h->enc_offset, UPKIE_NJ, h->n, h->n_pad, offset, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_encoder_offset_state(void* handle, const uint32_t* count, const float* offset, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !offset) return fail(UPKIE_B200_EINVAL, "set_encoder_offset_state: invalid argument");
  if (!h->P.encoder_offset)
    return fail(UPKIE_B200_EINVAL, "set_encoder_offset_state: no encoder offsets are set (upkie_b200_set_encoder_offset)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // every offset must be a calibration error of a joint of the mask: read back (after the caller's work on the
  // stream) and checked here
  std::vector<float> d(size_t(h->n) * UPKIE_NJ);
  CUDA_TRY(cudaMemcpyAsync(d.data(), offset, d.size() * sizeof(float), cudaMemcpyDefault, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (size_t k = 0; k < d.size(); ++k) {
    if (!(std::fabs(d[k]) <= 0.5f))
      return fail(UPKIE_B200_EINVAL, "set_encoder_offset_state: every offset must be finite and within [-0.5, 0.5] "
                                     "radians");
    if (d[k] != 0.f && !((h->enc_mask >> (k % UPKIE_NJ)) & 1u))
      return fail(UPKIE_B200_EINVAL, "set_encoder_offset_state: a joint outside joint_mask must have a zero offset");
  }
  CUDA_TRY(cudaMemcpyAsync(h->enc_count, count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_cols(offset, UPKIE_NJ, h->n, h->n_pad, h->enc_offset, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_servo_noise(void* handle, const UpkieServoNoise* spec) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!spec) {
    if (h->P.servo_noise) {
      CUDA_TRY(cudaSetDevice(h->device));
      CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may use the per-env state
      h->P.servo_noise = nullptr;
      cudaFree(h->noise_count);
      cudaFree(h->noise_sigma);
      cudaFree(h->noise_fresh);
      h->noise_count = nullptr;
      h->noise_sigma = nullptr;
      h->noise_fresh = nullptr;
      h->noise_spec = UpkieServoNoise{};
    }
    return UPKIE_B200_OK;
  }
  if (const char* why = servo_noise_spec_error(*spec, h->P)) return fail(UPKIE_B200_EINVAL, why);
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the device block
  if (!h->P.servo_noise) {
    // switched on: zero counters, and zero sigmas until each env's next reset
    CUDA_TRY(alloc_zeroed({{reinterpret_cast<void**>(&h->noise_count), size_t(h->n) * sizeof(uint32_t)},
                           {reinterpret_cast<void**>(&h->noise_sigma), size_t(kServoNoiseCols) * h->n_pad * sizeof(float)},
                           {reinterpret_cast<void**>(&h->noise_fresh), size_t(h->n_pad)}}));
  } else {
    // a replacement: the columns whose high bound is 0 have no noise from now on
    for (int c = 0; c < kServoNoiseCols; ++c) {
      const float hi = c < UPKIE_NJ ? spec->position_high[c] : spec->velocity_high[c - UPKIE_NJ];
      if (hi == 0.f) CUDA_TRY(cudaMemset(h->noise_sigma + size_t(c) * h->n_pad, 0, size_t(h->n_pad) * sizeof(float)));
    }
  }
  if (!h->noise_dev) CUDA_TRY(cudaMalloc(&h->noise_dev, sizeof(ServoNoise)));
  ServoNoise N;
  std::memset(&N, 0, sizeof(N));
  N.spec = *spec;
  N.count = h->noise_count;
  N.sigma = h->noise_sigma;
  N.fresh = h->noise_fresh;
  N.stride = h->n_pad;
  CUDA_TRY(cudaMemcpy(h->noise_dev, &N, sizeof(N), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaDeviceSynchronize());
  h->P.servo_noise = h->noise_dev;
  h->noise_spec = *spec;
  return UPKIE_B200_OK;
}

int upkie_b200_get_servo_noise_state(void* handle, uint32_t* count, float* sigma, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !sigma) return fail(UPKIE_B200_EINVAL, "get_servo_noise_state: invalid argument");
  if (!h->P.servo_noise)
    return fail(UPKIE_B200_EINVAL, "get_servo_noise_state: no servo noise is set (upkie_b200_set_servo_noise)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemcpyAsync(count, h->noise_count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_rows(h->noise_sigma, kServoNoiseCols, h->n, h->n_pad, sigma, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_servo_noise_state(void* handle, const uint32_t* count, const float* sigma, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !sigma) return fail(UPKIE_B200_EINVAL, "set_servo_noise_state: invalid argument");
  if (!h->P.servo_noise)
    return fail(UPKIE_B200_EINVAL, "set_servo_noise_state: no servo noise is set (upkie_b200_set_servo_noise)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // every sigma must be a sensor noise (the fixed caps of a spec's bounds, not the spec in force: a narrower spec
  // leaves each env's sigmas until its next reset, and a checkpoint taken before then must load), and zero in the
  // columns the spec in force turns off: read back (after the caller's work on the stream) and checked here
  std::vector<float> v(size_t(h->n) * kServoNoiseCols);
  CUDA_TRY(cudaMemcpyAsync(v.data(), sigma, v.size() * sizeof(float), cudaMemcpyDefault, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  const UpkieServoNoise& sp = h->noise_spec;
  for (size_t k = 0; k < v.size(); ++k) {
    const int c = int(k % kServoNoiseCols);
    const float hi = c < UPKIE_NJ ? sp.position_high[c] : sp.velocity_high[c - UPKIE_NJ];
    if (!(v[k] >= 0.f && v[k] <= (c < UPKIE_NJ ? 0.1f : 5.f)))
      return fail(UPKIE_B200_EINVAL, "set_servo_noise_state: every sigma must be finite, >= 0, at most 0.1 rad for a "
                                     "position and 5 rad/s for a velocity");
    if (v[k] != 0.f && hi == 0.f)
      return fail(UPKIE_B200_EINVAL, "set_servo_noise_state: a column whose high bound is zero must have a zero sigma");
  }
  CUDA_TRY(cudaMemcpyAsync(h->noise_count, count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_cols(sigma, kServoNoiseCols, h->n, h->n_pad, h->noise_sigma, s));
  return UPKIE_B200_OK;
}

int upkie_b200_get_servo_noise_mark(void* handle, uint8_t* mark, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !mark) return fail(UPKIE_B200_EINVAL, "get_servo_noise_mark: invalid argument");
  if (!h->P.servo_noise)
    return fail(UPKIE_B200_EINVAL, "get_servo_noise_mark: no servo noise is set (upkie_b200_set_servo_noise)");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaMemcpyAsync(mark, h->noise_fresh, size_t(h->n), cudaMemcpyDeviceToDevice,
                           static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

int upkie_b200_set_servo_noise_mark(void* handle, const uint8_t* mark, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !mark) return fail(UPKIE_B200_EINVAL, "set_servo_noise_mark: invalid argument");
  if (!h->P.servo_noise)
    return fail(UPKIE_B200_EINVAL, "set_servo_noise_mark: no servo noise is set (upkie_b200_set_servo_noise)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  std::vector<uint8_t> m(size_t(h->n));
  CUDA_TRY(cudaMemcpyAsync(m.data(), mark, m.size(), cudaMemcpyDefault, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (uint8_t x : m)
    if (x > 1) return fail(UPKIE_B200_EINVAL, "set_servo_noise_mark: every mark must be 0 or 1");
  CUDA_TRY(cudaMemcpyAsync(h->noise_fresh, mark, m.size(), cudaMemcpyDefault, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_velocity_derate(void* handle, const UpkieVelocityDerate* spec) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!spec) {
    if (h->P.velocity_derate) {
      CUDA_TRY(cudaSetDevice(h->device));
      CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may use the per-env state
      h->P.velocity_derate = nullptr;
      cudaFree(h->vlim_count);
      cudaFree(h->vlim_max);
      h->vlim_count = nullptr;
      h->vlim_max = nullptr;
      h->vlim_mask = 0;
    }
    return UPKIE_B200_OK;
  }
  if (const char* why = velocity_derate_spec_error(*spec, h->P)) return fail(UPKIE_B200_EINVAL, why);
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the device block
  if (!h->P.velocity_derate) {
    // switched on: zero counters; every joint of the mask is filled below
    CUDA_TRY(alloc_zeroed({{reinterpret_cast<void**>(&h->vlim_count), size_t(h->n) * sizeof(uint32_t)},
                           {reinterpret_cast<void**>(&h->vlim_max), size_t(UPKIE_NJ) * h->n_pad * sizeof(float)}}));
  }
  // the joints the spec drops from the mask have no limit from now on, and those it adds take the range's upper bound
  // until each env's next reset (a joint of the mask always holds a limit > 0)
  for (int j = 0; j < UPKIE_NJ; ++j) {
    float* const col = h->vlim_max + size_t(j) * h->n_pad;
    if (((h->vlim_mask & ~spec->joint_mask) >> j) & 1u)
      CUDA_TRY(cudaMemset(col, 0, size_t(h->n_pad) * sizeof(float)));
    if (((spec->joint_mask & ~h->vlim_mask) >> j) & 1u) {
      k_fill<<<grid_of(h->n), 128>>>(h->n, col, spec->max_velocity_high[j]);
      CUDA_TRY(cudaGetLastError());
    }
  }
  if (!h->vlim_dev) CUDA_TRY(cudaMalloc(&h->vlim_dev, sizeof(VelocityDerate)));
  VelocityDerate V;
  std::memset(&V, 0, sizeof(V));
  V.spec = *spec;
  V.count = h->vlim_count;
  V.max_velocity = h->vlim_max;
  V.stride = h->n_pad;
  CUDA_TRY(cudaMemcpy(h->vlim_dev, &V, sizeof(V), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaDeviceSynchronize());
  h->P.velocity_derate = h->vlim_dev;
  h->vlim_mask = spec->joint_mask;
  return UPKIE_B200_OK;
}

int upkie_b200_get_velocity_derate_state(void* handle, uint32_t* count, float* max_velocity, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !max_velocity) return fail(UPKIE_B200_EINVAL, "get_velocity_derate_state: invalid argument");
  if (!h->P.velocity_derate)
    return fail(UPKIE_B200_EINVAL,
                "get_velocity_derate_state: no velocity limits are set (upkie_b200_set_velocity_derate)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemcpyAsync(count, h->vlim_count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_rows(h->vlim_max, UPKIE_NJ, h->n, h->n_pad, max_velocity, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_velocity_derate_state(void* handle, const uint32_t* count, const float* max_velocity, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !max_velocity) return fail(UPKIE_B200_EINVAL, "set_velocity_derate_state: invalid argument");
  if (!h->P.velocity_derate)
    return fail(UPKIE_B200_EINVAL,
                "set_velocity_derate_state: no velocity limits are set (upkie_b200_set_velocity_derate)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // every joint of the mask in force must hold a limit, every other joint none: read back (after the caller's work on
  // the stream) and checked here
  std::vector<float> v(size_t(h->n) * UPKIE_NJ);
  CUDA_TRY(cudaMemcpyAsync(v.data(), max_velocity, v.size() * sizeof(float), cudaMemcpyDefault, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (size_t k = 0; k < v.size(); ++k) {
    if ((h->vlim_mask >> (k % UPKIE_NJ)) & 1u) {
      if (!(v[k] > 0.f && std::isfinite(v[k])))
        return fail(UPKIE_B200_EINVAL, "set_velocity_derate_state: every limit of a joint of joint_mask must be finite "
                                       "and > 0");
    } else if (v[k] != 0.f) {
      return fail(UPKIE_B200_EINVAL, "set_velocity_derate_state: a joint outside joint_mask must have a zero limit");
    }
  }
  CUDA_TRY(cudaMemcpyAsync(h->vlim_count, count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_cols(max_velocity, UPKIE_NJ, h->n, h->n_pad, h->vlim_max, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_attitude_filter(void* handle, const UpkieAttitudeFilter* spec) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  h->final_valid = false;  // the stash's layout follows the spec (the terminal estimates' rows)
  if (!spec) {
    if (h->P.attitude_filter) {
      CUDA_TRY(cudaSetDevice(h->device));
      CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may use the per-env state
      h->P.attitude_filter = nullptr;
      float** bufs[] = {&h->att_gains, &h->att_quat, &h->att_bias, &h->att_rep, &h->att_vel};
      for (float** b : bufs) {
        cudaFree(*b);
        *b = nullptr;
      }
      cudaFree(h->att_count);
      h->att_count = nullptr;
    }
    return UPKIE_B200_OK;
  }
  if (const char* why = attitude_filter_spec_error(*spec, h->P)) return fail(UPKIE_B200_EINVAL, why);
  if (h->P.obs_delay && h->sense_ticks > 1)
    return fail(UPKIE_B200_EINVAL, "set_attitude_filter: not with an observation delay of more than one tick (its "
                                   "report would need a ring of estimates)");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the device block
  const bool first = !h->P.attitude_filter;
  if (first) {
    const size_t col = size_t(h->n_pad) * sizeof(float);
    CUDA_TRY(alloc_zeroed({{reinterpret_cast<void**>(&h->att_count), size_t(h->n) * sizeof(uint32_t)},
                           {reinterpret_cast<void**>(&h->att_gains), 2 * col},
                           {reinterpret_cast<void**>(&h->att_quat), 4 * col},
                           {reinterpret_cast<void**>(&h->att_bias), 3 * col},
                           {reinterpret_cast<void**>(&h->att_rep), 4 * col},
                           {reinterpret_cast<void**>(&h->att_vel), 3 * col}}));
  }
  if (!h->att_dev) CUDA_TRY(cudaMalloc(&h->att_dev, sizeof(AttitudeFilter)));
  AttitudeFilter A;
  std::memset(&A, 0, sizeof(A));
  A.spec = *spec;
  quat_from_rot(h->P.Rbi, A.qbi);
  A.count = h->att_count;
  A.gains = h->att_gains;
  A.quat = h->att_quat;
  A.bias = h->att_bias;
  A.rep = h->att_rep;
  A.vel = h->att_vel;
  A.stride = h->n_pad;
  CUDA_TRY(cudaMemcpy(h->att_dev, &A, sizeof(A), cudaMemcpyHostToDevice));
  h->P.attitude_filter = h->att_dev;
  h->att_spec = *spec;
  if (first) {  // every env: the upper gains, the true orientation and b = 0 until its next reset
    k_attitude_init<<<grid_of(h->n), 128>>>(h->P, h->n, h->n_pad, h->state, true, spec->kp_high, spec->ki_high);
    CUDA_TRY(cudaGetLastError());
  }
  CUDA_TRY(cudaDeviceSynchronize());
  return UPKIE_B200_OK;
}

int upkie_b200_get_attitude_filter_state(void* handle, uint32_t* count, float* gains, float* quat, float* bias,
                                         void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !gains || !quat || !bias)
    return fail(UPKIE_B200_EINVAL, "get_attitude_filter_state: invalid argument");
  if (!h->P.attitude_filter)
    return fail(UPKIE_B200_EINVAL, "get_attitude_filter_state: no attitude filter is set (upkie_b200_set_attitude_filter)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemcpyAsync(count, h->att_count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_rows(h->att_gains, 2, h->n, h->n_pad, gains, s));
  CUDA_TRY(ring_rows(h->att_quat, 4, h->n, h->n_pad, quat, s));
  CUDA_TRY(ring_rows(h->att_bias, 3, h->n, h->n_pad, bias, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_attitude_filter_state(void* handle, const uint32_t* count, const float* gains, const float* quat,
                                         const float* bias, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !gains || !quat || !bias)
    return fail(UPKIE_B200_EINVAL, "set_attitude_filter_state: invalid argument");
  if (!h->P.attitude_filter)
    return fail(UPKIE_B200_EINVAL, "set_attitude_filter_state: no attitude filter is set (upkie_b200_set_attitude_filter)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // read back (after the caller's work on the stream) and checked here: finite values, unit quaternions, gains within
  // the caps of a spec (not the spec in force: a narrower spec keeps each env's gains until its next reset)
  const size_t n = size_t(h->n);
  std::vector<float> g(n * 2), q(n * 4), b(n * 3);
  CUDA_TRY(cudaMemcpyAsync(g.data(), gains, g.size() * sizeof(float), cudaMemcpyDefault, s));
  CUDA_TRY(cudaMemcpyAsync(q.data(), quat, q.size() * sizeof(float), cudaMemcpyDefault, s));
  CUDA_TRY(cudaMemcpyAsync(b.data(), bias, b.size() * sizeof(float), cudaMemcpyDefault, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (size_t i = 0; i < n; ++i) {
    const float kp = g[2 * i], ki = g[2 * i + 1];
    if (!std::isfinite(kp) || !std::isfinite(ki) || !(kp >= 0.f) || !(double(kp) * double(h->P.h) <= 0.5) ||
        !(ki >= 0.f) || !(ki <= 10.f))
      return fail(UPKIE_B200_EINVAL, "set_attitude_filter_state: every gain must be finite, 0 <= kp with "
                                     "kp * (dt / nb_substeps) <= 0.5, and 0 <= ki <= 10");
    double norm2 = 0.0;
    for (int r = 0; r < 4; ++r) {
      const float v = q[4 * i + r];
      if (!std::isfinite(v)) return fail(UPKIE_B200_EINVAL, "set_attitude_filter_state: every value must be finite");
      norm2 += double(v) * double(v);
    }
    if (!(std::fabs(std::sqrt(norm2) - 1.0) <= 1e-5))
      return fail(UPKIE_B200_EINVAL, "set_attitude_filter_state: every quaternion must be unit (within 1e-5)");
    for (int r = 0; r < 3; ++r)
      if (!std::isfinite(b[3 * i + r]))
        return fail(UPKIE_B200_EINVAL, "set_attitude_filter_state: every value must be finite");
  }
  CUDA_TRY(cudaMemcpyAsync(h->att_count, count, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_cols(gains, 2, h->n, h->n_pad, h->att_gains, s));
  CUDA_TRY(ring_cols(quat, 4, h->n, h->n_pad, h->att_quat, s));
  CUDA_TRY(ring_cols(bias, 3, h->n, h->n_pad, h->att_bias, s));
  return UPKIE_B200_OK;
}

int upkie_b200_get_attitude_filter_report(void* handle, float* quat, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !quat) return fail(UPKIE_B200_EINVAL, "get_attitude_filter_report: invalid argument");
  if (!h->P.attitude_filter)
    return fail(UPKIE_B200_EINVAL, "get_attitude_filter_report: no attitude filter is set (upkie_b200_set_attitude_filter)");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(ring_rows(h->att_rep, 4, h->n, h->n_pad, quat, static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

int upkie_b200_set_attitude_filter_report(void* handle, const float* quat, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !quat) return fail(UPKIE_B200_EINVAL, "set_attitude_filter_report: invalid argument");
  if (!h->P.attitude_filter)
    return fail(UPKIE_B200_EINVAL, "set_attitude_filter_report: no attitude filter is set (upkie_b200_set_attitude_filter)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  std::vector<float> q(size_t(h->n) * 4);
  CUDA_TRY(cudaMemcpyAsync(q.data(), quat, q.size() * sizeof(float), cudaMemcpyDefault, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (int i = 0; i < h->n; ++i) {
    double norm2 = 0.0;
    for (int r = 0; r < 4; ++r) norm2 += double(q[4 * size_t(i) + r]) * double(q[4 * size_t(i) + r]);
    if (!(std::fabs(std::sqrt(norm2) - 1.0) <= 1e-5))  // (NaN fails too)
      return fail(UPKIE_B200_EINVAL, "set_attitude_filter_report: every quaternion must be unit (within 1e-5)");
  }
  CUDA_TRY(ring_cols(quat, 4, h->n, h->n_pad, h->att_rep, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_torque_scale(void* handle, const UpkieTorqueScale* spec) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!spec) {
    if (h->P.torque_scale) {
      CUDA_TRY(cudaSetDevice(h->device));
      CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may use the per-env state
      h->P.torque_scale = nullptr;
      cudaFree(h->tsc_count);
      cudaFree(h->tsc_scale);
      h->tsc_count = nullptr;
      h->tsc_scale = nullptr;
      h->tsc_mask = 0;
    }
    return UPKIE_B200_OK;
  }
  if (const char* why = torque_scale_spec_error(*spec, h->P)) return fail(UPKIE_B200_EINVAL, why);
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may read the device block
  // the joints the spec adds to the mask hold 1 until each env's next reset, and those it drops store 1: on a handle
  // that had no spec every joint starts at 1, and a replacement resets the joints whose membership changes
  uint32_t fill = (h->tsc_mask ^ spec->joint_mask) & ((1u << UPKIE_NJ) - 1u);
  if (!h->P.torque_scale) {  // switched on: zero counters
    CUDA_TRY(alloc_zeroed({{reinterpret_cast<void**>(&h->tsc_count), size_t(h->n) * sizeof(uint32_t)},
                           {reinterpret_cast<void**>(&h->tsc_scale), size_t(UPKIE_NJ) * h->n_pad * sizeof(float)}}));
    fill = (1u << UPKIE_NJ) - 1u;
  }
  for (int j = 0; j < UPKIE_NJ; ++j) {
    if (!((fill >> j) & 1u)) continue;
    k_fill<<<grid_of(h->n), 128>>>(h->n, h->tsc_scale + size_t(j) * h->n_pad, 1.f);
    CUDA_TRY(cudaGetLastError());
  }
  if (!h->tsc_dev) CUDA_TRY(cudaMalloc(&h->tsc_dev, sizeof(TorqueScale)));
  TorqueScale T;
  std::memset(&T, 0, sizeof(T));
  T.spec = *spec;
  T.count = h->tsc_count;
  T.scale = h->tsc_scale;
  T.stride = h->n_pad;
  CUDA_TRY(cudaMemcpy(h->tsc_dev, &T, sizeof(T), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaDeviceSynchronize());
  h->P.torque_scale = h->tsc_dev;
  h->tsc_mask = spec->joint_mask;
  return UPKIE_B200_OK;
}

int upkie_b200_get_torque_scale_state(void* handle, uint32_t* count, float* scale, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !scale) return fail(UPKIE_B200_EINVAL, "get_torque_scale_state: invalid argument");
  if (!h->P.torque_scale)
    return fail(UPKIE_B200_EINVAL, "get_torque_scale_state: no torque scales are set (upkie_b200_set_torque_scale)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemcpyAsync(count, h->tsc_count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_rows(h->tsc_scale, UPKIE_NJ, h->n, h->n_pad, scale, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_torque_scale_state(void* handle, const uint32_t* count, const float* scale, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !count || !scale) return fail(UPKIE_B200_EINVAL, "set_torque_scale_state: invalid argument");
  if (!h->P.torque_scale)
    return fail(UPKIE_B200_EINVAL, "set_torque_scale_state: no torque scales are set (upkie_b200_set_torque_scale)");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // every joint of the mask in force must hold a scale in (0, 2], every other joint exactly 1: read back (after the
  // caller's work on the stream) and checked here
  std::vector<float> v(size_t(h->n) * UPKIE_NJ);
  CUDA_TRY(cudaMemcpyAsync(v.data(), scale, v.size() * sizeof(float), cudaMemcpyDefault, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  if (const char* why = torque_scale_state_error(h->tsc_mask, v.data(), size_t(h->n))) return fail(UPKIE_B200_EINVAL, why);
  CUDA_TRY(cudaMemcpyAsync(h->tsc_count, count, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CUDA_TRY(ring_cols(scale, UPKIE_NJ, h->n, h->n_pad, h->tsc_scale, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_history(void* handle, const UpkieHistory* spec) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "invalid handle");
  if (!spec) {
    if (h->P.history) {
      CUDA_TRY(cudaSetDevice(h->device));
      CUDA_TRY(cudaDeviceSynchronize());  // launches in flight may use the ring
      h->P.history = nullptr;
      cudaFree(h->hist_ring);
      cudaFree(h->hist_head);
      h->hist_ring = nullptr;
      h->hist_head = nullptr;
      h->hist_ticks = 0;
    }
    return UPKIE_B200_OK;
  }
  if (const char* why = history_spec_error(*spec, h->P)) return fail(UPKIE_B200_EINVAL, why);
  h->hist_spec = *spec;
  return history_build(h);
}

int upkie_b200_get_history(void* handle, float* out, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !out) return fail(UPKIE_B200_EINVAL, "get_history: invalid argument");
  if (!h->P.history) return fail(UPKIE_B200_EINVAL, "get_history: no history is set (upkie_b200_set_history)");
  CUDA_TRY(cudaSetDevice(h->device));
  k_history_read<<<grid_of(h->n), 128, 0, static_cast<cudaStream_t>(stream)>>>(h->P, h->P.history, h->n, out);
  CUDA_TRY(cudaGetLastError());
  return UPKIE_B200_OK;
}

int upkie_b200_history_entries(void* handle, int* ticks) {
  Handle* h = as_handle(handle);
  if (!h || !ticks) return fail(UPKIE_B200_EINVAL, "history_entries: invalid argument");
  *ticks = h->P.history ? h->hist_ticks : 0;
  return UPKIE_B200_OK;
}

int upkie_b200_get_history_state(void* handle, float* rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !rows) return fail(UPKIE_B200_EINVAL, "get_history_state: invalid argument");
  if (!h->P.history) return fail(UPKIE_B200_EINVAL, "get_history_state: no history is set (upkie_b200_set_history)");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(ring_rows(h->hist_ring, int(h->hist_spec.count), h->n, h->n_pad, rows, static_cast<cudaStream_t>(stream),
                     h->hist_head, h->hist_ticks, h->hist_ticks));
  return UPKIE_B200_OK;
}

int upkie_b200_set_history_state(void* handle, const float* rows, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !rows) return fail(UPKIE_B200_EINVAL, "set_history_state: invalid argument");
  if (!h->P.history) return fail(UPKIE_B200_EINVAL, "set_history_state: no history is set (upkie_b200_set_history)");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(ring_cols(rows, int(h->hist_spec.count), h->n, h->n_pad, h->hist_ring, static_cast<cudaStream_t>(stream),
                     h->hist_head, h->hist_ticks, h->hist_ticks));
  return UPKIE_B200_OK;
}

int upkie_b200_launch_count(void* handle, uint64_t* count) {
  Handle* h = as_handle(handle);
  if (!h || !count) return fail(UPKIE_B200_EINVAL, "launch_count: bad argument");
  *count = h->step_launches;
  return UPKIE_B200_OK;
}

int upkie_b200_error_flags(void* handle, uint32_t* flags, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !flags) return fail(UPKIE_B200_EINVAL, "error_flags: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaMemcpyAsync(flags, h->err, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                           static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

int upkie_b200_get_counters(void* handle, uint32_t* episode, uint32_t* tick, uint8_t* pending_reset,
                            uint32_t* error_flags, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "get_counters: invalid handle");
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t n = size_t(h->n);
  if (episode) CUDA_TRY(cudaMemcpyAsync(episode, h->episode, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  if (tick) CUDA_TRY(cudaMemcpyAsync(tick, h->tick, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  if (pending_reset) CUDA_TRY(cudaMemcpyAsync(pending_reset, h->done_prev, n, cudaMemcpyDeviceToDevice, s));
  if (error_flags) CUDA_TRY(cudaMemcpyAsync(error_flags, h->err, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  return UPKIE_B200_OK;
}

int upkie_b200_set_counters(void* handle, const uint32_t* episode, const uint32_t* tick, const uint8_t* pending_reset,
                            const uint32_t* error_flags, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "set_counters: invalid handle");
  h->final_valid = false;  // the stashed states no longer belong to the last step
  CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t n = size_t(h->n);
  if (episode) {
    CUDA_TRY(cudaMemcpyAsync(h->episode, episode, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
    // restored counters are not resets for the base-velocity post step
    CUDA_TRY(cudaMemcpyAsync(h->bv_episode, episode, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  }
  if (tick) CUDA_TRY(cudaMemcpyAsync(h->tick, tick, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  if (pending_reset) CUDA_TRY(cudaMemcpyAsync(h->done_prev, pending_reset, n, cudaMemcpyDeviceToDevice, s));
  if (error_flags) CUDA_TRY(cudaMemcpyAsync(h->err, error_flags, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  return UPKIE_B200_OK;
}

int upkie_b200_get_elapsed(void* handle, uint32_t* elapsed, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !elapsed) return fail(UPKIE_B200_EINVAL, "get_elapsed: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaMemcpyAsync(elapsed, h->elapsed, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                           static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

int upkie_b200_set_elapsed(void* handle, const uint32_t* elapsed, void* stream) {
  Handle* h = as_handle(handle);
  if (!h || !elapsed) return fail(UPKIE_B200_EINVAL, "set_elapsed: invalid argument");
  h->final_valid = false;  // the stashed states no longer belong to the last step
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaMemcpyAsync(h->elapsed, elapsed, size_t(h->n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                           static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

// ---- MPC ---------------------------------------------------------------------------------

int upkie_b200_mpc_create(const UpkieMpcConfig* config, int n_robots, int device, void** mpc) {
  if (!config || !mpc) return fail(UPKIE_B200_EINVAL, "mpc_create: null argument");
  std::string err;
  int rc = mpc_create_impl(*config, n_robots, device, mpc, err);
  return rc ? fail(rc, err) : UPKIE_B200_OK;
}
void upkie_b200_mpc_destroy(void* mpc) { mpc_destroy_impl(mpc); }
int upkie_b200_mpc_reset(void* mpc, const uint8_t* mask, void* stream) {
  std::string err;
  int rc = mpc_reset_impl(mpc, mask, static_cast<cudaStream_t>(stream), err);
  return rc ? fail(rc, err) : UPKIE_B200_OK;
}
int upkie_b200_mpc_step(void* mpc, const float* x0, const float* v_target, const uint8_t* floor_contact, float dt,
                        float* v_cmd, float* first_input, uint8_t* found, void* stream) {
  std::string err;
  int rc = mpc_step_impl(mpc, x0, v_target, floor_contact, dt, v_cmd, first_input, found,
                         static_cast<cudaStream_t>(stream), err);
  return rc ? fail(rc, err) : UPKIE_B200_OK;
}
int upkie_b200_mpc_plan(void* mpc, float* plan, void* stream) {
  std::string err;
  int rc = mpc_plan_impl(mpc, plan, static_cast<cudaStream_t>(stream), err);
  return rc ? fail(rc, err) : UPKIE_B200_OK;
}

// ---- UpkieBaseVelocity epilogue -------------------------------------------------------------

int upkie_b200_base_velocity_post(void* handle, void* mpc, const UpkieBaseVelocityPost* args, void* stream) {
  Handle* h = as_handle(handle);
  if (!h) return fail(UPKIE_B200_EINVAL, "base_velocity_post: invalid sim handle");
  MpcHandle* m = as_mpc(mpc);
  if (!m) return fail(UPKIE_B200_EINVAL, "base_velocity_post: invalid mpc handle");
  if (!args) return fail(UPKIE_B200_EINVAL, "base_velocity_post: null arguments");
  if (m->n != h->n || m->device != h->device)
    return fail(UPKIE_B200_EINVAL, "base_velocity_post: the mpc handle must hold as many robots as the sim handle has "
                                   "envs, on the same device");
  const UpkieBaseVelocityPost& a = *args;
  if (!a.action || !a.gyropod_obs || !a.xy || !a.commanded_velocity || !a.obs)
    return fail(UPKIE_B200_EINVAL, "base_velocity_post: null buffer");
  if (!(a.dt > 0.f) || !std::isfinite(a.dt)) return fail(UPKIE_B200_EINVAL, "base_velocity_post: dt must be > 0 and finite");
  if (a.autoreset_mode != h->autoreset)
    return fail(UPKIE_B200_EINVAL, "base_velocity_post: autoreset_mode differs from the sim handle's "
                                   "(upkie_b200_set_autoreset)");
  const bool same_step = a.autoreset_mode == AUTORESET_SAME_STEP;
  if (same_step && (!a.gyropod_final_obs || !a.final_obs))
    return fail(UPKIE_B200_EINVAL, "base_velocity_post: same-step mode needs gyropod_final_obs and final_obs");
  BaseVelocityPostArgs k;
  k.n = h->n;
  k.detect_resets = a.autoreset_mode != AUTORESET_DISABLED;
  k.same_step = same_step;
  k.dt = a.dt;
  k.action = a.action;
  k.gyro_obs = a.gyropod_obs;
  k.gyro_final_obs = same_step ? a.gyropod_final_obs : nullptr;
  k.episode = h->episode;
  k.seen_episode = h->bv_episode;
  k.xy = a.xy;
  k.v_cmd = a.commanded_velocity;
  k.active = m->active;
  k.obs = a.obs;
  k.final_obs = same_step ? a.final_obs : nullptr;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(launch_base_velocity_post(k, static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

// ---- observer pipeline --------------------------------------------------------------------

int upkie_b200_default_observer_config(const UpkieModel* model, UpkieObserverConfig* config) {
  if (!model || !config) return fail(UPKIE_B200_EINVAL, "default_observer_config: null");
  default_observer_config(*model, config);
  return UPKIE_B200_OK;
}
int upkie_b200_default_wheel_balancer_config(UpkieWheelBalancerConfig* config) {
  if (!config) return fail(UPKIE_B200_EINVAL, "default_wheel_balancer_config: null");
  default_wheel_balancer_config(config);
  return UPKIE_B200_OK;
}
int upkie_b200_wheel_balancer_create(const UpkieWheelBalancerConfig* config, int n_robots, int device, void** balancer) {
  if (!config || !balancer) return fail(UPKIE_B200_EINVAL, "wheel_balancer_create: null argument");
  std::string err;
  int rc = wheel_balancer_create_impl(*config, n_robots, device, balancer, err);
  return rc ? fail(rc, err) : UPKIE_B200_OK;
}
void upkie_b200_wheel_balancer_destroy(void* balancer) { wheel_balancer_destroy_impl(balancer); }
int upkie_b200_wheel_balancer_reset(void* balancer, const uint8_t* mask, void* stream) {
  WheelBalancerHandle* h = as_wheel_balancer(balancer);
  if (!h) return fail(UPKIE_B200_EINVAL, "wheel_balancer_reset: invalid handle");
  CUDA_TRY(cudaSetDevice(h->device));
  k_wheel_balancer_reset<<<(h->n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(h->n, mask, h->state);
  CUDA_TRY(cudaGetLastError());
  return UPKIE_B200_OK;
}
int upkie_b200_wheel_balancer_step(void* balancer, const float* obs, int obs_layout, const float* target, float* action,
                                   void* stream) {
  WheelBalancerHandle* h = as_wheel_balancer(balancer);
  if (!h || !obs || !action) return fail(UPKIE_B200_EINVAL, "wheel_balancer_step: invalid argument");
  int stride, pitch, contact, odom;
  if (obs_layout == UPKIE_OBS_LAYOUT_SPINE) {
    stride = UPKIE_SPINE_DIM; pitch = UPKIE_SP_PITCH; contact = UPKIE_SP_CONTACT; odom = UPKIE_SP_ODOM_POS;
  } else if (obs_layout == UPKIE_OBS_LAYOUT_OBSERVERS) {
    stride = UPKIE_OBSV_DIM; pitch = UPKIE_OBSV_PITCH; contact = UPKIE_OBSV_CONTACT; odom = UPKIE_OBSV_ODOM_POS;
  } else {
    return fail(UPKIE_B200_EINVAL, "wheel_balancer_step: unknown observation layout");
  }
  CUDA_TRY(cudaSetDevice(h->device));
  k_wheel_balancer_step<<<(h->n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      h->P, h->n, h->state, obs, stride, pitch, contact, odom, target, action);
  CUDA_TRY(cudaGetLastError());
  return UPKIE_B200_OK;
}
int upkie_b200_wheel_balancer_state(void* balancer, float* state, void* stream) {
  WheelBalancerHandle* h = as_wheel_balancer(balancer);
  if (!h || !state) return fail(UPKIE_B200_EINVAL, "wheel_balancer_state: invalid argument");
  CUDA_TRY(cudaSetDevice(h->device));
  // [4][n] -> [n][4]
  for (int k = 0; k < 4; ++k)
    CUDA_TRY(cudaMemcpy2DAsync(state + k, 4 * sizeof(float), h->state + size_t(k) * h->n, sizeof(float), sizeof(float), h->n,
                               cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
  return UPKIE_B200_OK;
}

int upkie_b200_observers_create(const UpkieObserverConfig* config, int n_robots, int device, void** observers) {
  if (!config || !observers) return fail(UPKIE_B200_EINVAL, "observers_create: null argument");
  std::string err;
  int rc = observers_create_impl(*config, n_robots, device, observers, err);
  return rc ? fail(rc, err) : UPKIE_B200_OK;
}
void upkie_b200_observers_destroy(void* observers) { observers_destroy_impl(observers); }
int upkie_b200_observers_reset(void* observers, const uint8_t* mask, void* stream) {
  std::string err;
  int rc = observers_reset_impl(observers, mask, static_cast<cudaStream_t>(stream), err);
  return rc ? fail(rc, err) : UPKIE_B200_OK;
}
int upkie_b200_observers_step(void* observers, const float* spine_obs, float* out, void* stream) {
  std::string err;
  int rc = observers_step_impl(observers, spine_obs, out, static_cast<cudaStream_t>(stream), err);
  return rc ? fail(rc, err) : UPKIE_B200_OK;
}

}  // extern "C"
