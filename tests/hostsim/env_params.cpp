// SPDX-License-Identifier: Apache-2.0
//
// env_params.cpp -- TEST INFRASTRUCTURE. The CPU build of the kernels' arithmetic (hostsim.cpp) with the per-env
// parameter table of upkie_b200_set_env_params: the table as the handle installs it, and the entry points that pass
// each robot's column to the table readers (servo_substep, spine_cycle, measured_torques, apply_imu_uncertainty), in
// the order the step kernels call them. Built by tests/test_env_params_config.py; never loaded by the product.
#include "hostsim.cpp"

extern "C" {

// rows[n][UPKIE_EP_DIM] -> soa[UPKIE_EP_DIM][n] (caller-owned, kept alive while the handle runs), installed as the
// handle's table with the "some env has it" noise flags. Returns env_row_flags OR-ed over the rows; an invalid table
// (kEpInvalid) is not installed.
uint32_t hostsim_ep_set_env_params(void* hv, int n, const float* rows, float* soa) {
  HostSim* h = static_cast<HostSim*>(hv);
  uint32_t f = 0;
  for (int i = 0; i < n; ++i) f |= env_row_flags(rows + size_t(i) * UPKIE_EP_DIM);
  if (f & kEpInvalid) return f;
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < UPKIE_EP_DIM; ++k) soa[size_t(k) * n + i] = rows[size_t(i) * UPKIE_EP_DIM + k];
  h->P.env_params = soa;
  h->P.env_params_stride = n;
  set_noise_flags(h->P, f);
  return f;
}

// one env tick with the torque noise models, env i reading column i (k_step<.., NOISE=1/5>'s sequence)
void hostsim_ep_step_servos_noise(void* hv, int n, float* state, const float* action, uint32_t tick,
                                  uint64_t env_offset, float* obs) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    clamp_servo_action(h->P, a);
    const NoiseCtx nz{env_offset + uint64_t(i), tick};
    for (int sub = 0; sub < h->P.nb_substeps; ++sub)
      servo_substep(h->P, S, a, false, nullptr, h->P.friction, any_fn, NoSync(), &nz, sub, nullptr, h->P.joint_limits,
                    BodyRecOut{nullptr, 0}, i);
    observe_update(h->P, S);
    float tq[6];
    measured_torques(h->P, S, &nz, tq, i);
    for (int j = 0; j < 6; ++j) {
      float* o = obs + size_t(i) * UPKIE_OBS_DIM + j * 5;
      o[0] = S.q[j]; o[1] = S.qd[j]; o[2] = tq[j]; o[3] = 42.0f; o[4] = 18.0f;
    }
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// the spine observation as k_spine_obs assembles it, env i reading column i
void hostsim_ep_spine_obs_with_uncertainty(void* hv, int n, const float* state, uint32_t tick, uint64_t env_offset,
                                           float* out) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    const NoiseCtx nz{env_offset + uint64_t(i), tick};
    float tq[6];
    measured_torques(h->P, S, &nz, tq, i);
    float* o = out + size_t(i) * UPKIE_SPINE_DIM;
    spine_observation(h->P, S, o, tq);
    apply_imu_uncertainty(h->P, nz, o, i);
  }
}

// spine mode: one step (observation of the first cycle + nb_substeps cycles), env i reading column i
void hostsim_ep_step_servos_spine(void* hv, int n, float* state, float* lag, const float* action, float* spine) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    SpineLag L;
    lag_from_row(lag + size_t(i) * UPKIE_LAG_DIM, L);
    float a[UPKIE_ACT_DIM];
    std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    clamp_servo_action(h->P, a);
    spine_assemble_observation(S, L);
    for (int sub = 0; sub < h->P.nb_substeps; ++sub)
      spine_cycle(h->P, S, L, a, false, nullptr, h->P.friction, any_fn, NoSync(), h->P.joint_limits,
                  BodyRecOut{nullptr, 0}, i);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
    lag_to_row(L, lag + size_t(i) * UPKIE_LAG_DIM);
    spine_observation_from_lag(h->P, L, spine + size_t(i) * UPKIE_SPINE_DIM);
  }
}

}  // extern "C"
