// SPDX-License-Identifier: Apache-2.0
//
// encoder_offset.cpp -- TEST INFRASTRUCTURE. The CPU build of the encoder offsets' draws, reset, view, executed
// targets and reset leg targets (sim_core.cuh encoder_offset_draw / encoder_offset_reset / encoder_offset_view /
// encoder_offset_command / encoder_offset_leg_targets, the code the FAM_SENSE step kernels and k_reset inline), in the
// order the step kernels run them, of its spec's validation (params.h encoder_offset_spec_error) and of the family
// choice with offsets set (step_family.h). Built by tests/test_encoder_offset_cpu.py; never loaded by the product.
#include "hostsim.cpp"
#include "../../upkie_b200/csrc/step_family.h"

extern "C" {

// encoder_offset_draw of draw k of the env of global index g: d[6]
void hostsim_encoder_offset_draw(const UpkieEncoderOffset* spec, uint64_t seed, uint64_t g, uint32_t k, float* d) {
  const Offset6 o = encoder_offset_draw(*spec, seed, g, k);
  for (int j = 0; j < UPKIE_NJ; ++j) d[j] = o.d[j];
}

// The reset of the envs [0, n): count and offset [6][n] of encoder_offset_reset
void hostsim_encoder_offset_reset(int n, const UpkieEncoderOffset* spec, uint64_t seed, uint64_t env_offset,
                                  uint32_t* count, float* offset) {
  EncoderOffset E;
  std::memset(&E, 0, sizeof(E));
  E.spec = *spec;
  E.count = count;
  E.offset = offset;
  E.stride = n;
  for (int i = 0; i < n; ++i) encoder_offset_reset(E, seed, env_offset + uint64_t(i), i);
}

static Offset6 offsets_of(const float* d, int i) {
  Offset6 o;
  for (int j = 0; j < UPKIE_NJ; ++j) o.d[j] = d ? d[size_t(i) * UPKIE_NJ + j] : 0.f;
  return o;
}

// One UpkieServos tick of the step kernels under the offsets d[n][6] (null: none): the clamps, the executed targets
// target - delta, the substeps, and the [6][5] rows built from a copy of the state read through the offsets
void hostsim_encoder_offset_servo_tick(void* hv, int n, float* state, const float* action, const float* d, float* obs) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    const Offset6 o = offsets_of(d, i);
    clamp_servo_action(h->P, a);
    encoder_offset_command(a, o);
    step_servo_action<false>(h->P, S, a, nullptr, h->P.friction, any_fn);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
    encoder_offset_view(S, o);
    for (int j = 0; j < 6; ++j) {
      float* r = obs + size_t(i) * UPKIE_OBS_DIM + j * 5;
      r[0] = S.q[j]; r[1] = S.qd[j]; r[2] = S.torque[j]; r[3] = 42.0f; r[4] = 18.0f;
    }
  }
}

// One gyropod tick of the step kernels under the offsets d[n][6]: the wrapper's servo action (leg targets decayed
// toward the servo zero), the clamps, the executed targets, the substeps, and the row built through the offsets.
// `servo` [n][36] receives the servo action before the shift.
void hostsim_encoder_offset_gyropod_tick(void* hv, int n, float* state, const float* action, const float* d,
                                         float* obs6, float* servo) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    const float a0 = action[size_t(i) * 2], a1 = action[size_t(i) * 2 + 1];
    const Offset6 o = offsets_of(d, i);
    gyropod_action(h->P, S, a0, a1, a);
    clamp_servo_action(h->P, a);
    std::memcpy(servo + size_t(i) * UPKIE_ACT_DIM, a, sizeof(a));
    encoder_offset_command(a, o);
    step_servo_action<false>(h->P, S, a, nullptr, h->P.friction, any_fn);
    S.yaw += a1 * h->P.dt;
    S.yaw_vel = a1;
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
    gyropod_obs(h->P, S, obs6 + size_t(i) * 6);
    if (encoder_offset_view(S, o)) gyropod_obs(h->P, S, obs6 + size_t(i) * 6);
  }
}

// A reset of the step kernels and k_reset under the offsets d[n][6]: reset_robot, then the leg targets made the
// reported positions
void hostsim_encoder_offset_reset_robot(void* hv, int n, float* state, const float* init, const float* d) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    reset_robot(h->P, S, init + size_t(i) * UPKIE_INIT_DIM, nullptr, h->P.friction, any_fn, h->P.joint_limits);
    encoder_offset_leg_targets(S, offsets_of(d, i));
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// The view of the state rows [n][UPKIE_STATE_DIM] through d[n][6]: the rows read through it, in place, and
// changed[i] = the view's result (a wheel position changed)
void hostsim_encoder_offset_view(int n, float* state, const float* d, int* changed) {
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    changed[i] = encoder_offset_view(S, offsets_of(d, i)) ? 1 : 0;
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// encoder_offset_spec_error of a handle with these settings: 1 and the message in `why`, or 0
int hostsim_encoder_offset_spec_error(const UpkieEncoderOffset* spec, int joint_limits, int spine_mode,
                                      int body_contacts, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  const char* w = encoder_offset_spec_error(*spec, P);
  if (!w) return 0;
  std::snprintf(why, size_t(len), "%s", w);
  return 1;
}

// step_family with offsets set (a non-null P.encoder_offset) and the other settings given
int hostsim_step_family_encoder_offset(int joint_limits, int spine_mode, int body_contacts, int obs_delay, int mode,
                                       int transport, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  static EncoderOffset E;
  static ObsDelay O;
  P.encoder_offset = &E;
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
