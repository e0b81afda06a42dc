// SPDX-License-Identifier: Apache-2.0
//
// attitude_filter.cpp -- TEST INFRASTRUCTURE. The CPU build of the attitude filter's draws, step, inputs and initial
// estimate (sim_core.cuh attitude_filter_draw / attitude_filter_step / attitude_filter_inputs /
// attitude_filter_initial, the code the FAM_SENSE step kernels and k_reset call), of the observation read from an
// estimate (attitude_filter_observation), of its spec's validation (params.h attitude_filter_spec_error) and of the
// family choice with a filter set (step_family.h). Built by tests/test_attitude_filter_cpu.py; never loaded by the
// product.
#include "hostsim.cpp"
#include "../../upkie_b200/csrc/step_family.h"

namespace {
AttitudeFilter host_filter() {
  AttitudeFilter A;
  std::memset(&A, 0, sizeof(A));
  return A;
}
}  // namespace

extern "C" {

// attitude_filter_draw of draw k of the env of global index g: (kp, ki, roll, pitch)
void hostsim_att_draw(const UpkieAttitudeFilter* spec, uint64_t seed, uint64_t g, uint32_t k, float* out) {
  const AttitudeDraw d = attitude_filter_draw(*spec, seed, g, k);
  out[0] = d.kp;
  out[1] = d.ki;
  out[2] = d.roll;
  out[3] = d.pitch;
}

// `steps` filter steps of one filter from q[4], b[3] with gains kp, ki over a substep h, step s taking the rate
// wm[s][3] and the specific force am[s][3] (an input stride of 0 repeats the first); the estimate after every step
// into qs[steps][4] and the bias estimate into bs[steps][3] (either may be null). q and b are updated in place.
void hostsim_att_run(int steps, float* q, float* b, float kp, float ki, float h, const float* wm, const float* am,
                     int stride, float* qs, float* bs) {
  for (int s = 0; s < steps; ++s) {
    attitude_filter_step(q, b, kp, ki, h, wm + size_t(s) * size_t(stride), am + size_t(s) * size_t(stride));
    if (qs)
      for (int r = 0; r < 4; ++r) qs[size_t(s) * 4 + r] = q[r];
    if (bs)
      for (int r = 0; r < 3; ++r) bs[size_t(s) * 3 + r] = b[r];
  }
}

// The filter inputs of the state rows [n][UPKIE_STATE_DIM] (their orientation the observed one) with the previous
// IMU velocities vp[n][3] and the biases gb, ab [3]: the IMU velocities v[n][3], w_m[n][3] and a_m[n][3]
void hostsim_att_inputs(void* hv, int n, const float* state, const float* vp, const float* gb, const float* ab,
                        float* v, float* wm, float* am) {
  HostSim* h = static_cast<HostSim*>(hv);
  AttitudeFilter A = host_filter();
  quat_from_rot(h->P.Rbi, A.qbi);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    imu_velocity(h->P, S, v + size_t(i) * 3);
    attitude_filter_inputs(h->P, A, S, v + size_t(i) * 3, vp + size_t(i) * 3, gb, ab, wm + size_t(i) * 3,
                           am + size_t(i) * 3);
  }
}

// The initial estimate of a base observed with orientation qb[n][4] and errors roll[n], pitch[n]: q[n][4]
void hostsim_att_initial(void* hv, int n, const float* qb, const float* roll, const float* pitch, float* q) {
  HostSim* h = static_cast<HostSim*>(hv);
  AttitudeFilter A = host_filter();
  quat_from_rot(h->P.Rbi, A.qbi);
  for (int i = 0; i < n; ++i) attitude_filter_initial(A, qb + size_t(i) * 4, roll[i], pitch[i], q + size_t(i) * 4);
}

// The orientation-derived columns of the spine observation of estimates q[n][4] into o[n][UPKIE_SPINE_DIM] (the
// other columns untouched), and the gyropod pitch into pitch[n]
void hostsim_att_observation(void* hv, int n, const float* q, float* o, float* pitch) {
  HostSim* h = static_cast<HostSim*>(hv);
  AttitudeFilter A = host_filter();
  quat_from_rot(h->P.Rbi, A.qbi);
  for (int i = 0; i < n; ++i) {
    float qb[4];
    attitude_filter_base(A, q + size_t(i) * 4, qb);
    attitude_filter_observation(h->P, qb, o + size_t(i) * UPKIE_SPINE_DIM);
    pitch[i] = attitude_filter_pitch(qb);
  }
}

// attitude_filter_spec_error of a handle with these settings (h: the substep): 1 and the message in `why`, or 0
int hostsim_att_spec_error(const UpkieAttitudeFilter* spec, int joint_limits, int spine_mode, int body_contacts,
                           float h, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  P.h = h;
  const char* w = attitude_filter_spec_error(*spec, P);
  if (!w) return 0;
  std::snprintf(why, size_t(len), "%s", w);
  return 1;
}

// step_family with a filter set (a non-null P.attitude_filter) and the other settings given
int hostsim_step_family_att(int joint_limits, int spine_mode, int body_contacts, int mode, int transport, char* why,
                            int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  static AttitudeFilter A;
  P.attitude_filter = &A;
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  const char* w = nullptr;
  const int f = step_family(P, false, mode, transport, &w);
  if (f < 0) std::snprintf(why, size_t(len), "%s", w);
  return f;
}

}  // extern "C"
