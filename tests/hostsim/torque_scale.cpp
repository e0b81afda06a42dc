// SPDX-License-Identifier: Apache-2.0
//
// torque_scale.cpp -- TEST INFRASTRUCTURE. The CPU build of the servo torque scales' draws, reset and law
// (sim_core.cuh torque_scale_draw / torque_scale_reset / torque_scale_load, and servo_substep with an env's scales:
// the code the FAM_SENSE step kernels and k_reset inline), of its spec's and state's validation (params.h
// torque_scale_spec_error / torque_scale_state_error) and of the family choice with scales set (step_family.h). Built
// by tests/test_torque_scale_cpu.py; never loaded by the product.
#include "hostsim.cpp"
#include "../../upkie_b200/csrc/step_family.h"

extern "C" {

// torque_scale_draw of draw k of the env of global index g: s[6]
void hostsim_torque_scale_draw(const UpkieTorqueScale* spec, uint64_t seed, uint64_t g, uint32_t k, float* s) {
  const Scale6 o = torque_scale_draw(*spec, seed, g, k);
  for (int j = 0; j < UPKIE_NJ; ++j) s[j] = o.s[j];
}

// The reset of the envs [0, n): count and scale [6][n] of torque_scale_reset
void hostsim_torque_scale_reset(int n, const UpkieTorqueScale* spec, uint64_t seed, uint64_t env_offset,
                                uint32_t* count, float* scale) {
  TorqueScale T;
  std::memset(&T, 0, sizeof(T));
  T.spec = *spec;
  T.count = count;
  T.scale = scale;
  T.stride = n;
  for (int i = 0; i < n; ++i) torque_scale_reset(T, seed, env_offset + uint64_t(i), i);
}

// One UpkieServos tick of the step kernels: the clamps, then nb_substeps servo_substep calls under the scales
// scale [6][n] of `spec` (spec null: none), loaded once per env as torque_scale_load does, with external forces
// ext[n][7][3] (null: none) and, when `zero_torque`, as a reset's zero-torque substeps; the [6][5] rows.
void hostsim_torque_scale_servo_tick(void* hv, int n, float* state, const float* action, const UpkieTorqueScale* spec,
                                     float* scale, const float* ext, int zero_torque, float* obs) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    // the env's scales, as the step kernels load them once per tick
    const Scale6 s6 = torque_scale_load([&](int j) { return scale ? scale[size_t(j) * size_t(n) + size_t(i)] : 1.f; });
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    clamp_servo_action(h->P, a);
    const ExtForces X{ext ? ext + size_t(i) * 21 : nullptr, 1, 0u};
    for (int sub = 0; sub < h->P.nb_substeps; ++sub)
      servo_substep(h->P, S, a, zero_torque != 0, nullptr, h->P.friction, any_fn, NoSync(), nullptr, sub,
                    ext ? &X : nullptr, h->P.joint_limits, BodyRecOut{nullptr, 0}, -1, nullptr, nullptr, i,
                    spec ? &s6 : nullptr);
    observe_update(h->P, S);
    for (int j = 0; j < 6; ++j) {
      float* r = obs + size_t(i) * UPKIE_OBS_DIM + j * 5;
      r[0] = S.q[j]; r[1] = S.qd[j]; r[2] = S.torque[j]; r[3] = 42.0f; r[4] = 18.0f;
    }
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// torque_scale_apply elementwise over n values: the delivered torque fl(s t)
void hostsim_torque_scale_apply(int n, const float* s, const float* t, float* out) {
  for (int k = 0; k < n; ++k) out[k] = torque_scale_apply(s[k], t[k]);
}

// torque_scale_spec_error of a handle with these settings: 1 and the message in `why`, or 0
int hostsim_torque_scale_spec_error(const UpkieTorqueScale* spec, int joint_limits, int spine_mode, int body_contacts,
                                    char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  const char* w = torque_scale_spec_error(*spec, P);
  if (!w) return 0;
  std::snprintf(why, size_t(len), "%s", w);
  return 1;
}

// torque_scale_state_error of scales v[n][6] under joint_mask: 1 and the message in `why`, or 0
int hostsim_torque_scale_state_error(uint32_t joint_mask, const float* v, int n, char* why, int len) {
  const char* w = torque_scale_state_error(joint_mask, v, size_t(n));
  if (!w) return 0;
  std::snprintf(why, size_t(len), "%s", w);
  return 1;
}

// step_family with scales set (a non-null P.torque_scale) and the other settings given
int hostsim_step_family_torque_scale(int joint_limits, int spine_mode, int body_contacts, int mode, int transport,
                                     char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  static TorqueScale T;
  P.torque_scale = &T;
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  const char* w = nullptr;
  const int f = step_family(P, false, mode, transport, &w);
  if (f < 0) std::snprintf(why, size_t(len), "%s", w);
  return f;
}

}  // extern "C"
