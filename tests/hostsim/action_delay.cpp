// SPDX-License-Identifier: Apache-2.0
//
// action_delay.cpp -- TEST INFRASTRUCTURE. The CPU build of the action delay's draw, reset and delayed tick
// (sim_core.cuh action_delay_draw / action_delay_reset / action_delay_substep, the code the step kernels and
// action_delay.cu inline), and of the step kernels' family choice with a delay (step_family.h). Built by
// tests/test_action_delay_cpu.py; never loaded by the product.
#include "hostsim.cpp"
#include "../../upkie_b200/csrc/step_family.h"

extern "C" {

uint32_t hostsim_action_delay_draw(const UpkieActionDelay* spec, uint64_t seed, uint64_t g, uint32_t k) {
  return action_delay_draw(*spec, seed, g, k);
}

// an explicit reset of the envs [0, n) selected by mask (NULL = all); command [UPKIE_ACT_DIM][stride]
void hostsim_action_delay_reset(const UpkieActionDelay* spec, uint64_t seed, uint64_t env_offset, int n,
                                const uint8_t* mask, uint32_t* count, uint32_t* delay, float* command, int stride) {
  ActionDelay A;
  std::memset(&A, 0, sizeof(A));
  A.spec = *spec;
  A.count = count;
  A.delay = delay;
  A.command = command;
  A.stride = stride;
  for (int i = 0; i < n; ++i)
    if (!mask || mask[i]) action_delay_reset(A, seed, env_offset + uint64_t(i), i);
}

// One delayed tick of each env [0, n) in the order of the step kernels (step_env, no reset): the action front end
// (mode 0 servos: action[n][36]; 1 gyropod: action[n][2]), the clamps, the swap of this tick's command into the
// command buffer prev[n][36] (in: the previous command, out: this tick's), the substeps with action_delay_substep
// switching at delay[i], the observation update and the wrapper's yaw integration. `noise`: the torque-control noise of
// tick `tick` (NoiseCtx of env env_offset + i).
void hostsim_action_delay_tick(void* hv, int n, int mode, float* state, float* prev, const float* action,
                               const uint32_t* delay, int noise, uint32_t tick, uint64_t env_offset, uint32_t* err) {
  HostSim* h = static_cast<HostSim*>(hv);
  const SimParams& P = h->P;
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    uint32_t e = 0;
    float a1 = 0.f;
    if (mode == 0) {
      std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    } else {
      a1 = action[2 * i + 1];
      e |= gyropod_action(P, S, action[2 * i], a1, a);
    }
    e |= clamp_servo_action(P, a);
    float* row = prev + size_t(i) * UPKIE_ACT_DIM;
    for (int c = 0; c < UPKIE_ACT_DIM; ++c) {
      const float p = row[c];
      row[c] = a[c];
      a[c] = p;
    }
    const NoiseCtx nz{env_offset + uint64_t(i), tick};
    for (int sub = 0; sub < P.nb_substeps; ++sub) {
      action_delay_substep(sub, delay[i], a, [&](int c) { return row[c]; });
      servo_substep(P, S, a, false, nullptr, P.friction, any_fn, NoSync(), noise ? &nz : nullptr, sub, nullptr,
                    P.joint_limits);
    }
    observe_update(P, S);
    e |= state_sanity(S);
    if (mode != 0) {
      S.yaw += a1 * P.dt;
      S.yaw_vel = a1;
    }
    if (err) err[i] = e;
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// Substeps sub0 .. sub1 - 1 of each env under the command rows command[n][36] as given (no clamps), through
// servo_substep, the single substep of every tick; `observe`: then the tick's observation update
void hostsim_servo_substeps(void* hv, int n, float* state, const float* command, int sub0, int sub1, int noise,
                            uint32_t tick, uint64_t env_offset, int observe) {
  HostSim* h = static_cast<HostSim*>(hv);
  const SimParams& P = h->P;
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    const NoiseCtx nz{env_offset + uint64_t(i), tick};
    for (int sub = sub0; sub < sub1; ++sub)
      servo_substep(P, S, command + size_t(i) * UPKIE_ACT_DIM, false, nullptr, P.friction, any_fn, NoSync(),
                    noise ? &nz : nullptr, sub, nullptr, P.joint_limits);
    if (observe) observe_update(P, S);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// the stop row, as action_delay_reset writes it
void hostsim_action_delay_stop_row(float* row) {
  for (int c = 0; c < UPKIE_ACT_DIM; ++c) row[c] = action_delay_stop_value(c);
}

// gyropod front end and clamps of one tick: the servo command row[n][36] the tick computes (the leg filter advances)
void hostsim_gyropod_command(void* hv, int n, float* state, const float* action, float* row) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    gyropod_action(h->P, S, action[2 * i], action[2 * i + 1], row + size_t(i) * UPKIE_ACT_DIM);
    clamp_servo_action(h->P, row + size_t(i) * UPKIE_ACT_DIM);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// action_delay_spec_error of a handle with the given config values; the message to why[why_len], 0 when accepted
int hostsim_action_delay_spec_error(const UpkieActionDelay* spec, int nb_substeps, int joint_limits, int spine_mode,
                                    char* why, int why_len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.nb_substeps = nb_substeps;
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  const char* msg = action_delay_spec_error(*spec, P);
  why[0] = '\0';
  if (msg) {
    std::strncpy(why, msg, why_len - 1);
    why[why_len - 1] = '\0';
  }
  return msg ? 1 : 0;
}

// what `family` compiles in: extras, limits, table, reset_rand, spine, body, push, delay
void hostsim_family_traits_delay(int family, uint8_t* out) {
  const StepFamily f = step_family_traits(family);
  const bool v[8] = {f.extras, f.limits, f.table, f.reset_rand, f.spine, f.body, f.push, f.delay};
  for (int k = 0; k < 8; ++k) out[k] = v[k] ? 1 : 0;
}

// step_family of a handle with the given features, an action delay among them
int hostsim_step_family_delay(int joint_limits, int table, int body_contacts, int push, int delay, int spine_mode,
                              int max_episode_steps, int mode, int transport, char* why, int why_len) {
  static float table_storage[1];
  static char push_storage[1], delay_storage[1];
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.joint_limits = joint_limits;
  P.env_params = table ? table_storage : nullptr;
  P.body_contacts = body_contacts;
  P.push = push ? reinterpret_cast<const PushRand*>(push_storage) : nullptr;
  P.action_delay = delay ? reinterpret_cast<const ActionDelay*>(delay_storage) : nullptr;
  P.spine_mode = spine_mode;
  P.max_episode_steps = max_episode_steps;
  const char* msg = nullptr;
  const int family = step_family(P, false, mode, transport, &msg);
  why[0] = '\0';
  if (msg) {
    std::strncpy(why, msg, why_len - 1);
    why[why_len - 1] = '\0';
  }
  return family;
}

}  // extern "C"
