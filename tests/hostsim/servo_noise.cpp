// SPDX-License-Identifier: Apache-2.0
//
// servo_noise.cpp -- TEST INFRASTRUCTURE. The CPU build of the servo noise's draws, cycle counters, normals, view and
// reset leg targets (sim_core.cuh servo_noise_draw / servo_noise_cycle / servo_noise_normals / servo_noise_increments /
// servo_noise_view / servo_noise_leg_targets, the code the FAM_SENSE step kernels and the handle-side kernels inline),
// of its spec's validation (params.h servo_noise_spec_error) and of the family choice with noise set (step_family.h).
// Built by tests/test_servo_noise_cpu.py; never loaded by the product.
#include "hostsim.cpp"
#include "../../upkie_b200/csrc/step_family.h"

extern "C" {

// servo_noise_draw of draw k of the env of global index g: s[12]
void hostsim_servo_noise_draw(const UpkieServoNoise* spec, uint64_t seed, uint64_t g, uint32_t k, float* s) {
  const Sigma12 o = servo_noise_draw(*spec, seed, g, k);
  for (int c = 0; c < kServoNoiseCols; ++c) s[c] = o.s[c];
}

// The reset of the envs [0, n): count, sigma [12][n] and fresh of servo_noise_reset
void hostsim_servo_noise_reset(int n, const UpkieServoNoise* spec, uint64_t seed, uint64_t env_offset, uint32_t* count,
                               float* sigma, uint8_t* fresh) {
  ServoNoise N;
  std::memset(&N, 0, sizeof(N));
  N.spec = *spec;
  N.count = count;
  N.sigma = sigma;
  N.fresh = fresh;
  N.stride = n;
  for (int i = 0; i < n; ++i) servo_noise_reset(N, seed, env_offset + uint64_t(i), i);
}

uint64_t hostsim_servo_noise_cycle(uint32_t t, uint32_t s) { return servo_noise_cycle(t, s); }
uint64_t hostsim_servo_noise_reset_cycle(uint32_t ep) { return servo_noise_reset_cycle(ep); }
uint64_t hostsim_servo_noise_cycle_before(uint32_t t, uint32_t nb, uint32_t age) {
  return servo_noise_cycle_before(t, nb, age);
}

// The twelve normals of cycle `cycle` of the env of global index g
void hostsim_servo_noise_normals(uint64_t seed, uint64_t g, uint64_t cycle, float* n) {
  servo_noise_normals(seed, g, cycle, n);
}

// The view of the state rows [n][UPKIE_STATE_DIM] of the envs g0 + i with sigmas [n][12] in cycle `cycle`: the rows
// read through it, in place, and changed[i] = the view's result (a wheel value changed)
void hostsim_servo_noise_view(int n, float* state, const float* sigma, uint64_t seed, uint64_t g0, uint64_t cycle,
                              int* changed) {
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    const float* s = sigma + size_t(i) * kServoNoiseCols;
    const Noise12 d = servo_noise_increments([&](int c) { return s[c]; }, seed, g0 + uint64_t(i), cycle);
    changed[i] = servo_noise_view(S, d) ? 1 : 0;
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// The gyropod row [n][6] of the states viewed as above (the order of the step kernels: the view, then gyropod_obs
// again when a wheel changed), and the leg targets a reset sets from them (reset_wrapper_state, then the reset
// observation's noise), in `state` in place
void hostsim_servo_noise_gyropod_obs(void* hv, int n, float* state, const float* sigma, uint64_t seed, uint64_t g0,
                                     uint64_t cycle, float* obs6) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    const float* s = sigma + size_t(i) * kServoNoiseCols;
    const Noise12 d = servo_noise_increments([&](int c) { return s[c]; }, seed, g0 + uint64_t(i), cycle);
    reset_wrapper_state(S);
    servo_noise_leg_targets(S, d);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
    gyropod_obs(h->P, S, obs6 + size_t(i) * 6);
    if (servo_noise_view(S, d)) gyropod_obs(h->P, S, obs6 + size_t(i) * 6);
  }
}

// servo_noise_spec_error of a handle with these settings: 1 and the message in `why`, or 0
int hostsim_servo_noise_spec_error(const UpkieServoNoise* spec, int joint_limits, int spine_mode, int body_contacts,
                                   int obs_delay, int servo_dropout, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  static ObsDelay O;
  static ServoDropout D;
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  P.obs_delay = obs_delay ? &O : nullptr;
  P.servo_dropout = servo_dropout ? &D : nullptr;
  const char* w = servo_noise_spec_error(*spec, P);
  if (!w) return 0;
  std::snprintf(why, size_t(len), "%s", w);
  return 1;
}

// step_family with noise set (a non-null P.servo_noise) and the other settings given
int hostsim_step_family_servo_noise(int joint_limits, int spine_mode, int body_contacts, int obs_delay, int mode,
                                    int transport, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  static ServoNoise N;
  static ObsDelay O;
  P.servo_noise = &N;
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  P.obs_delay = obs_delay ? &O : nullptr;
  const char* w = nullptr;
  const int f = step_family(P, false, mode, transport, &w);
  if (f < 0) std::snprintf(why, size_t(len), "%s", w);
  return f;
}

}  // extern "C"
