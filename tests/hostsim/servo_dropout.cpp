// SPDX-License-Identifier: Apache-2.0
//
// servo_dropout.cpp -- TEST INFRASTRUCTURE. The CPU build of the servo dropouts' draws, loss rule, holds and latched
// view (sim_core.cuh servo_dropout_draw / servo_dropout_lost / servo_dropout_hold / servo_dropout_view /
// servo_dropout_reset, the code the FAM_SENSE step kernels and k_reset inline), of its spec's validation (params.h
// servo_dropout_spec_error) and of the family choice with dropouts set (step_family.h). Built by
// tests/test_servo_dropout_cpu.py; never loaded by the product.
#include "hostsim.cpp"
#include "../../upkie_b200/csrc/step_family.h"

namespace {
ServoDropout make_dropout(int n, uint32_t mask, uint32_t* count, float* prob, float* held) {
  ServoDropout D;
  std::memset(&D, 0, sizeof(D));
  D.spec.joint_mask = mask;
  D.count = count;
  D.prob = prob;
  D.held = held;
  D.stride = n;
  return D;
}
}  // namespace

extern "C" {

// `nticks` UpkieServos ticks of each env [0, n) under the command rows command[n][36] as given (no clamps, no reset),
// with the step kernels' dropout rule: at the end of each substep its losses, and the triples of the masked servos
// received latched into held[18][n]. Tick t of env i is tick0[i] + 1 + t, its
// probability prob[i], its global index env_offset + i. truth / seen [nticks * nb][n][18]: the true
// [joint][q, qd, torque] after each substep and the latched view of it, what an observation at that instant reports.
void hostsim_servo_dropout_run(void* hv, int n, float* state, const float* command, uint32_t mask, const float* prob,
                               const uint32_t* tick0, uint64_t seed, uint64_t env_offset, int nticks, float* held,
                               float* truth, float* seen) {
  HostSim* h = static_cast<HostSim*>(hv);
  const SimParams& P = h->P;
  const int nb = P.nb_substeps;
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    const uint64_t g = env_offset + uint64_t(i);
    auto load = [&](int r) { return held[size_t(r) * n + i]; };
    auto store = [&](int r, float v) { held[size_t(r) * n + i] = v; };
    for (int t = 0; t < nticks; ++t) {
      const uint32_t tick = tick0[i] + 1u + uint32_t(t);
      for (int sub = 0; sub < nb; ++sub) {
        servo_substep(P, S, command + size_t(i) * UPKIE_ACT_DIM, false, nullptr, P.friction, any_fn, NoSync(), nullptr,
                      sub, nullptr, P.joint_limits);
        const uint32_t lost = servo_dropout_lost(mask, prob[i], seed, g, tick, uint32_t(sub));
        RobotState V = S;
        servo_dropout_view(V, lost, load);
        float* const tr = truth + (size_t(t * nb + sub) * n + i) * kServoHeldRows;
        float* const se = seen + (size_t(t * nb + sub) * n + i) * kServoHeldRows;
        for (int j = 0; j < UPKIE_NJ; ++j) {
          tr[3 * j] = S.q[j]; tr[3 * j + 1] = S.qd[j]; tr[3 * j + 2] = S.torque[j];
          se[3 * j] = V.q[j]; se[3 * j + 1] = V.qd[j]; se[3 * j + 2] = V.torque[j];
        }
        servo_dropout_hold(S, mask, lost, store);
      }
      observe_update(P, S);
    }
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// servo_dropout_lost of one (env, tick, substep)
uint32_t hostsim_servo_dropout_lost(uint32_t mask, float p, uint64_t seed, uint64_t g, uint32_t tick, uint32_t sub) {
  return servo_dropout_lost(mask, p, seed, g, tick, sub);
}

// The reset of the envs [0, n) from their state rows: count, prob and held of servo_dropout_reset
void hostsim_servo_dropout_reset(int n, const float* state, const UpkieServoDropout* spec, uint64_t seed,
                                 uint64_t env_offset, uint32_t* count, float* prob, float* held) {
  ServoDropout D = make_dropout(n, spec->joint_mask, count, prob, held);
  D.spec = *spec;
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    servo_dropout_reset(D, seed, env_offset + uint64_t(i), i, S);
  }
}

// servo_dropout_spec_error of a handle with these settings: 1 and the message in `why`, or 0
int hostsim_servo_dropout_spec_error(const UpkieServoDropout* spec, int joint_limits, int spine_mode,
                                     int body_contacts, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  const char* e = servo_dropout_spec_error(*spec, P);
  if (!e) return 0;
  std::snprintf(why, size_t(len), "%s", e);
  return 1;
}

// step_family with servo dropouts set (a non-null P.servo_dropout) and the other settings given
int hostsim_step_family_servo_dropout(int joint_limits, int spine_mode, int body_contacts, int obs_delay, int mode,
                                      int transport, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  static ServoDropout D;
  static ObsDelay O;
  P.servo_dropout = &D;
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
