// SPDX-License-Identifier: Apache-2.0
//
// imu_misalignment.cpp -- TEST INFRASTRUCTURE. The CPU build of the IMU misalignment's draws, reset and view
// (sim_core.cuh imu_misalign_draw / imu_misalign_reset / imu_misalign_view, the code the FAM_SENSE step kernels,
// k_reset, k_spine_obs and k_reset_obs inline), of the observations built through it (spine_observation,
// gyropod_obs), of its spec's validation (params.h imu_misalignment_spec_error) and of the family choice with a
// misalignment set (step_family.h). Built by tests/test_imu_misalignment_cpu.py; never loaded by the product.
#include "hostsim.cpp"
#include "../../upkie_b200/csrc/step_family.h"

extern "C" {

// imu_misalign_draw of draw k of the env of global index g: e (w, x, y, z)
void hostsim_imu_misalign_draw(const UpkieImuMisalignment* spec, uint64_t seed, uint64_t g, uint32_t k, float* e) {
  const Quat4 q = imu_misalign_draw(*spec, seed, g, k);
  for (int r = 0; r < 4; ++r) e[r] = q.q[r];
}

// The reset of the envs [0, n): count and quat [4][n] of imu_misalign_reset
void hostsim_imu_misalign_reset(int n, const UpkieImuMisalignment* spec, uint64_t seed, uint64_t env_offset,
                                uint32_t* count, float* quat) {
  ImuMisalign M;
  std::memset(&M, 0, sizeof(M));
  M.spec = *spec;
  M.count = count;
  M.quat = quat;
  M.stride = n;
  for (int i = 0; i < n; ++i) imu_misalign_reset(M, seed, env_offset + uint64_t(i), i);
}

// The observations of the state rows [n][UPKIE_STATE_DIM] through the misalignments e [n][4]: the spine observation
// spine[n][UPKIE_SPINE_DIM] (commanded torques, no noise) and the gyropod row o6[n][6]; changed[i] = the view's result
void hostsim_imu_misalign_obs(void* hv, int n, const float* state, const float* e, float* spine, float* o6,
                              int* changed) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    Quat4 q;
    for (int r = 0; r < 4; ++r) q.q[r] = e[size_t(i) * 4 + r];
    changed[i] = imu_misalign_view(S, q) ? 1 : 0;
    spine_observation(h->P, S, spine + size_t(i) * UPKIE_SPINE_DIM);
    gyropod_obs(h->P, S, o6 + size_t(i) * 6);
  }
}

// imu_misalignment_spec_error of a handle with these settings: 1 and the message in `why`, or 0
int hostsim_imu_misalign_spec_error(const UpkieImuMisalignment* spec, int joint_limits, int spine_mode,
                                    int body_contacts, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  const char* w = imu_misalignment_spec_error(*spec, P);
  if (!w) return 0;
  std::snprintf(why, size_t(len), "%s", w);
  return 1;
}

// step_family with a misalignment set (a non-null P.imu_misalign) and the other settings given
int hostsim_step_family_imu_misalign(int joint_limits, int spine_mode, int body_contacts, int obs_delay, int mode,
                                     int transport, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  static ImuMisalign M;
  static ObsDelay O;
  P.imu_misalign = &M;
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
