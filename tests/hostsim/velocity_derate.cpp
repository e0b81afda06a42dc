// SPDX-License-Identifier: Apache-2.0
//
// velocity_derate.cpp -- TEST INFRASTRUCTURE. The CPU build of the servo velocity limits' draws, reset and torque law
// (sim_core.cuh velocity_derate_draw / velocity_derate_reset / velocity_derate_torque, and servo_substep with a
// VelocityDerate block: the code the FAM_SENSE step kernels and k_reset inline), of its spec's validation (params.h
// velocity_derate_spec_error) and of the family choice with limits set (step_family.h). Built by
// tests/test_velocity_derate_cpu.py; never loaded by the product.
#include "hostsim.cpp"
#include "../../upkie_b200/csrc/step_family.h"

extern "C" {

// velocity_derate_draw of draw k of the env of global index g: v[6]
void hostsim_velocity_derate_draw(const UpkieVelocityDerate* spec, uint64_t seed, uint64_t g, uint32_t k, float* v) {
  const Vmax6 o = velocity_derate_draw(*spec, seed, g, k);
  for (int j = 0; j < UPKIE_NJ; ++j) v[j] = o.v[j];
}

// The reset of the envs [0, n): count and max_velocity [6][n] of velocity_derate_reset
void hostsim_velocity_derate_reset(int n, const UpkieVelocityDerate* spec, uint64_t seed, uint64_t env_offset,
                                   uint32_t* count, float* max_velocity) {
  VelocityDerate V;
  std::memset(&V, 0, sizeof(V));
  V.spec = *spec;
  V.count = count;
  V.max_velocity = max_velocity;
  V.stride = n;
  for (int i = 0; i < n; ++i) velocity_derate_reset(V, seed, env_offset + uint64_t(i), i);
}

// velocity_derate_torque elementwise over n values
void hostsim_velocity_derate_torque(int n, const float* t, const float* qd, const float* v, const float* derate,
                                    const float* tau_max, float* out) {
  for (int k = 0; k < n; ++k) out[k] = velocity_derate_torque(t[k], qd[k], v[k], derate[k], tau_max[k]);
}

// One UpkieServos tick of the step kernels: the clamps, then nb_substeps servo_substep calls under the limits
// max_velocity [6][n] of `spec` (spec null: none), and the [6][5] rows. peak [n][6] (may be null) receives the largest
// |qd| of each joint at the end of a substep.
void hostsim_velocity_derate_servo_tick(void* hv, int n, float* state, const float* action,
                                        const UpkieVelocityDerate* spec, float* max_velocity, float* obs,
                                        float* peak) {
  HostSim* h = static_cast<HostSim*>(hv);
  VelocityDerate V;
  std::memset(&V, 0, sizeof(V));
  if (spec) V.spec = *spec;
  V.max_velocity = max_velocity;
  V.stride = n;
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    clamp_servo_action(h->P, a);
    float pk[UPKIE_NJ] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int sub = 0; sub < h->P.nb_substeps; ++sub) {
      servo_substep(h->P, S, a, false, nullptr, h->P.friction, any_fn, NoSync(), nullptr, sub, nullptr,
                    h->P.joint_limits, BodyRecOut{nullptr, 0}, -1, nullptr, spec ? &V : nullptr, i);
      for (int j = 0; j < UPKIE_NJ; ++j) pk[j] = std::fmax(pk[j], std::fabs(S.qd[j]));
    }
    observe_update(h->P, S);
    if (peak)
      for (int j = 0; j < UPKIE_NJ; ++j) peak[size_t(i) * UPKIE_NJ + j] = pk[j];
    for (int j = 0; j < 6; ++j) {
      float* r = obs + size_t(i) * UPKIE_OBS_DIM + j * 5;
      r[0] = S.q[j]; r[1] = S.qd[j]; r[2] = S.torque[j]; r[3] = 42.0f; r[4] = 18.0f;
    }
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// velocity_derate_spec_error of a handle with these settings: 1 and the message in `why`, or 0
int hostsim_velocity_derate_spec_error(const UpkieVelocityDerate* spec, int joint_limits, int spine_mode,
                                       int body_contacts, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  const char* w = velocity_derate_spec_error(*spec, P);
  if (!w) return 0;
  std::snprintf(why, size_t(len), "%s", w);
  return 1;
}

// step_family with limits set (a non-null P.velocity_derate) and the other settings given
int hostsim_step_family_velocity_derate(int joint_limits, int spine_mode, int body_contacts, int mode, int transport,
                                        char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  static VelocityDerate V;
  P.velocity_derate = &V;
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  const char* w = nullptr;
  const int f = step_family(P, false, mode, transport, &w);
  if (f < 0) std::snprintf(why, size_t(len), "%s", w);
  return f;
}

}  // extern "C"
