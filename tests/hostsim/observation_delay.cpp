// SPDX-License-Identifier: Apache-2.0
//
// observation_delay.cpp -- TEST INFRASTRUCTURE. The CPU build of the observation delay's draw, snapshot and sensed
// state (sim_core.cuh obs_delay_draw / obs_delay_reset, params.h obs_delay_snapshot / obs_delay_sensed_state, the code
// the step kernels and observation_delay.cu inline), of its spec's validation and of the family choice with a spec set
// (step_family.h). Built by tests/test_observation_delay_cpu.py; never loaded by the product.
#include "hostsim.cpp"
#include "../../upkie_b200/csrc/step_family.h"

extern "C" {

uint32_t hostsim_obs_delay_draw(const UpkieObservationDelay* spec, uint64_t seed, uint64_t g, uint32_t k) {
  return obs_delay_draw(*spec, seed, g, k);
}

// the draw of an explicit reset of the envs [0, n) selected by mask (NULL = all)
void hostsim_obs_delay_reset(const UpkieObservationDelay* spec, uint64_t seed, uint64_t env_offset, int n,
                             const uint8_t* mask, uint32_t* count, uint32_t* delay) {
  ObsDelay O;
  std::memset(&O, 0, sizeof(O));
  O.spec = *spec;
  O.count = count;
  O.delay = delay;
  for (int i = 0; i < n; ++i)
    if (!mask || mask[i]) obs_delay_reset(O, seed, env_offset + uint64_t(i), i);
}

// One UpkieServos tick of each env [0, n) under the command rows command[n][36] as given (no clamps, no reset), with
// the snapshots of the step kernels (step_env): the state at the start of the tick for delay nb_substeps, the end of
// substep nb_substeps - d - 1 for 0 < d < nb_substeps, the end of the tick after the observation update for d = 0.
// state[n][UPKIE_STATE_DIM]: the true state (in and out); sensed[n][UPKIE_STATE_DIM]: the sensed rows (in: the previous
// snapshot, out: this tick's, with the true state's other fields); obs[n][UPKIE_OBS_DIM]: the observation built from
// the sensed state (measured torques without noise).
void hostsim_obs_delay_tick(void* hv, int n, float* state, float* sensed, const float* command, const uint32_t* delay,
                            float* obs) {
  HostSim* h = static_cast<HostSim*>(hv);
  const SimParams& P = h->P;
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float* row = sensed + size_t(i) * UPKIE_STATE_DIM;
    auto load = [&](int k) { return row[k]; };
    auto store = [&](int k, float v) { row[k] = v; };
    const uint32_t nb = uint32_t(P.nb_substeps);
    const uint32_t d = delay[i] < nb ? delay[i] : nb;
    if (d == nb) {
      float v[3];
      imu_velocity(P, S, v);
      obs_delay_snapshot(P, S, v, load, store);
    }
    for (int sub = 0; sub < P.nb_substeps; ++sub) {
      servo_substep(P, S, command + size_t(i) * UPKIE_ACT_DIM, false, nullptr, P.friction, any_fn, NoSync(), nullptr,
                    sub, nullptr, P.joint_limits);
      if (d != 0 && uint32_t(sub) + d + 1u == nb) {
        float v[3];
        imu_velocity(P, S, v);
        obs_delay_snapshot(P, S, v, load, store);
      }
    }
    observe_update(P, S);
    if (d == 0) obs_delay_snapshot(P, S, S.prev_imu_vel, load, store);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
    for (int k = 0; k < UPKIE_STATE_DIM; ++k)
      if (!obs_delay_sensed(k)) row[k] = state[size_t(i) * UPKIE_STATE_DIM + k];
    obs_delay_sensed_state(S, load);
    float tq[6];
    measured_torques(P, S, nullptr, tq);
    for (int j = 0; j < 6; ++j) {
      float* o = obs + size_t(i) * UPKIE_OBS_DIM + 5 * j;
      o[0] = S.q[j]; o[1] = S.qd[j]; o[2] = tq[j]; o[3] = 42.0f; o[4] = 18.0f;
    }
  }
}

// Substeps sub0 .. sub1 - 1 of each env under the command rows as given; `observe`: then the observation update
void hostsim_obs_substeps(void* hv, int n, float* state, const float* command, int sub0, int sub1, int observe) {
  HostSim* h = static_cast<HostSim*>(hv);
  const SimParams& P = h->P;
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    for (int sub = sub0; sub < sub1; ++sub)
      servo_substep(P, S, command + size_t(i) * UPKIE_ACT_DIM, false, nullptr, P.friction, any_fn, NoSync(), nullptr,
                    sub, nullptr, P.joint_limits);
    if (observe) observe_update(P, S);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// the IMU velocity of each state row (imu_velocity)
void hostsim_imu_velocity(void* hv, int n, const float* state, float* v) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    imu_velocity(h->P, S, v + 3 * i);
  }
}

// obs_delay_sensed of every column of a state row
void hostsim_obs_delay_sensed_columns(uint8_t* out) {
  for (int k = 0; k < UPKIE_STATE_DIM; ++k) out[k] = obs_delay_sensed(k) ? 1 : 0;
}

// obs_delay_spec_error of a handle with the given config values; the message to why[why_len], 0 when accepted
int hostsim_obs_delay_spec_error(const UpkieObservationDelay* spec, int nb_substeps, int joint_limits, int spine_mode,
                                 int body_contacts, char* why, int why_len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.nb_substeps = nb_substeps;
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  const char* msg = obs_delay_spec_error(*spec, P);
  why[0] = '\0';
  if (msg) {
    std::strncpy(why, msg, why_len - 1);
    why[why_len - 1] = '\0';
  }
  return msg ? 1 : 0;
}

// step_family of a handle with the given features, `sense` the observation delay (tests/hostsim/step_family.cpp's
// hostsim_step_family with one more feature); the reason of a rejection goes to why[why_len]
int hostsim_step_family_sense(int joint_limits, int ctrl_noise, int meas_noise, int ext, int table, int body_contacts,
                              int push, int delay, int spine_mode, int max_episode_steps, int sense, int mode,
                              int transport, char* why, int why_len) {
  static float table_storage[1];
  static char push_storage[1], delay_storage[1], sense_storage[1];
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.joint_limits = joint_limits;
  P.any_ctrl_noise = ctrl_noise;
  P.any_meas_noise = meas_noise;
  P.env_params = table ? table_storage : nullptr;
  P.body_contacts = body_contacts;
  P.push = push ? reinterpret_cast<const PushRand*>(push_storage) : nullptr;
  P.action_delay = delay ? reinterpret_cast<const ActionDelay*>(delay_storage) : nullptr;
  P.obs_delay = sense ? reinterpret_cast<const ObsDelay*>(sense_storage) : nullptr;
  P.spine_mode = spine_mode;
  P.max_episode_steps = max_episode_steps;
  const char* msg = nullptr;
  const int family = step_family(P, ext != 0, mode, transport, &msg);
  why[0] = '\0';
  if (msg) {
    std::strncpy(why, msg, why_len - 1);
    why[why_len - 1] = '\0';
  }
  return family;
}

// what `family` compiles in: extras, limits, table, reset_rand, spine, body, push, delay, sense
void hostsim_family_traits_sense(int family, uint8_t* out) {
  const StepFamily f = step_family_traits(family);
  const bool v[9] = {f.extras, f.limits, f.table, f.reset_rand, f.spine, f.body, f.push, f.delay, f.sense};
  for (int k = 0; k < 9; ++k) out[k] = v[k] ? 1 : 0;
}

int hostsim_step_instantiated_sense(int tile, int family) { return step_instantiated(tile, family) ? 1 : 0; }

}  // extern "C"
