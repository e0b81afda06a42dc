// SPDX-License-Identifier: Apache-2.0
//
// history.cpp -- TEST INFRASTRUCTURE. The CPU build of the observation history's column arithmetic, ring fill and
// ring indexing (sim_core.cuh history_value / history_fill / history_entry, the code the FAM_SENSE step kernels,
// k_reset and k_history_read inline), of its spec's validation (params.h history_spec_error) and of the family choice
// with a history set (step_family.h). Built by tests/test_history_cpu.py; never loaded by the product.
#include "hostsim.cpp"
#include "../../upkie_b200/csrc/step_family.h"

namespace {
History make_history(int n, int count, const int* cols, int size, int ticks, float* ring, uint32_t* head) {
  History H;
  std::memset(&H, 0, sizeof(H));
  H.size = size;
  H.count = count;
  H.ticks = ticks;
  H.stride = n;
  for (int c = 0; c < count; ++c) {
    H.columns[c] = cols[c];
    if (history_acc_column(cols[c])) H.acc = 1;
  }
  H.ring = ring;
  H.head = head;
  return H;
}
}  // namespace

extern "C" {

// `nticks` UpkieServos ticks of each env [0, n) under the command rows command[n][36] as given (no clamps, no reset),
// recording the history as the step kernels do: after every substep, the columns of the state with the IMU velocity
// differentiated over the substep, into ring entry (head + sub) % ticks; the heads move on by nb_substeps per tick.
// ring[ticks][count][n], head[n] in and out. spine[nticks * nb][n][UPKIE_SPINE_DIM]: the full spine observation
// (spine_observation) of the state after each substep, its IMU acceleration the same substep difference.
void hostsim_history_run(void* hv, int n, float* state, const float* command, int count, const int* cols, int size,
                         int ticks, int nticks, float* ring, uint32_t* head, float* spine) {
  HostSim* h = static_cast<HostSim*>(hv);
  const SimParams& P = h->P;
  const History H = make_history(n, count, cols, size, ticks, ring, head);
  const int nb = P.nb_substeps;
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    for (int t = 0; t < nticks; ++t) {
      float hv3[3] = {S.prev_imu_vel[0], S.prev_imu_vel[1], S.prev_imu_vel[2]};
      const uint32_t h0 = head[i];
      for (int sub = 0; sub < nb; ++sub) {
        servo_substep(P, S, command + size_t(i) * UPKIE_ACT_DIM, false, nullptr, P.friction, any_fn, NoSync(), nullptr,
                      sub, nullptr, P.joint_limits);
        float v[3], acc[3];
        imu_velocity(P, S, v);
        for (int k = 0; k < 3; ++k) {
          acc[k] = (v[k] - hv3[k]) * P.inv_h;
          hv3[k] = v[k];
        }
        history_store(H, P, S, acc, (h0 + uint32_t(sub)) % uint32_t(ticks), i, [&](int c) { return H.columns[c]; });
        RobotState So = S;
        for (int k = 0; k < 3; ++k) So.imu_acc[k] = acc[k];
        spine_observation(P, So, spine + (size_t(t * nb + sub) * n + i) * UPKIE_SPINE_DIM);
      }
      observe_update(P, S);
      head[i] = (h0 + uint32_t(nb)) % uint32_t(ticks);
    }
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// The fill of a reset / new spec of the envs selected by mask (NULL = all): every entry the columns of the state
void hostsim_history_fill(void* hv, int n, const float* state, int count, const int* cols, int size, int ticks,
                          float* ring, const uint8_t* mask) {
  HostSim* h = static_cast<HostSim*>(hv);
  const History H = make_history(n, count, cols, size, ticks, ring, nullptr);
  for (int i = 0; i < n; ++i) {
    if (mask && !mask[i]) continue;
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    history_fill(H, h->P, S, i);
  }
}

// k_history_read's indexing: out[n][size][count], env i's window ending d[i] substeps before the end of the tick
void hostsim_history_read(int n, int count, int size, int ticks, const float* ring, const uint32_t* head,
                          const uint32_t* d, float* out) {
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < size; ++k)
      for (int c = 0; c < count; ++c)
        out[(size_t(i) * size + k) * count + c] =
            ring[(size_t(history_entry(head[i], uint32_t(ticks), d[i], uint32_t(k))) * count + c) * n + i];
}

// history_spec_error of a handle with these settings: 1 and the message in `why`, or 0
int hostsim_history_spec_error(const UpkieHistory* spec, int joint_limits, int spine_mode, int body_contacts,
                               char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  const char* e = history_spec_error(*spec, P);
  if (!e) return 0;
  std::snprintf(why, size_t(len), "%s", e);
  return 1;
}

// step_family with a history set (a non-null P.history) and the other settings given
int hostsim_step_family_history(int joint_limits, int spine_mode, int body_contacts, int obs_delay, int action_delay,
                                int mode, int transport, char* why, int len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  static History H;
  static ObsDelay O;
  static ActionDelay A;
  P.history = &H;
  P.joint_limits = joint_limits;
  P.spine_mode = spine_mode;
  P.body_contacts = body_contacts;
  P.obs_delay = obs_delay ? &O : nullptr;
  P.action_delay = action_delay ? &A : nullptr;
  const char* w = nullptr;
  const int f = step_family(P, false, mode, transport, &w);
  if (f < 0) std::snprintf(why, size_t(len), "%s", w);
  return f;
}

}  // extern "C"
