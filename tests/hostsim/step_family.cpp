// SPDX-License-Identifier: Apache-2.0
//
// step_family.cpp -- TEST INFRASTRUCTURE. The CPU build of the step kernels' family table, of the host's choice of a
// launch's family and of the (TILE, family) pairs the library instantiates (upkie_b200/csrc/step_family.h:
// step_family_traits, step_family, step_instantiated). Built by tests/test_step_family_cpu.py, also with
// -DUPKIE_EXACT_BUILD=1; never loaded by the product.
#include <cstdint>
#include <cstring>

#include "../../upkie_b200/csrc/step_family.h"

using namespace upkie_b200;

extern "C" {

// what `family` compiles in: extras, limits, table, reset_rand, spine, body, push, delay
void hostsim_family_traits(int family, uint8_t* out) {
  const StepFamily f = step_family_traits(family);
  const bool v[8] = {f.extras, f.limits, f.table, f.reset_rand, f.spine, f.body, f.push, f.delay};
  for (int k = 0; k < 8; ++k) out[k] = v[k] ? 1 : 0;
}

// step_family of a handle with the given features; the reason of a rejection goes to why[why_len]
int hostsim_step_family(int joint_limits, int ctrl_noise, int meas_noise, int ext, int table, int body_contacts,
                        int push, int delay, int spine_mode, int max_episode_steps, int mode, int transport, char* why,
                        int why_len) {
  static float table_storage[1];
  static char push_storage[1], delay_storage[1];
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.joint_limits = joint_limits;
  P.any_ctrl_noise = ctrl_noise;
  P.any_meas_noise = meas_noise;
  P.env_params = table ? table_storage : nullptr;
  P.body_contacts = body_contacts;
  P.push = push ? reinterpret_cast<const PushRand*>(push_storage) : nullptr;
  P.action_delay = delay ? reinterpret_cast<const ActionDelay*>(delay_storage) : nullptr;
  P.spine_mode = spine_mode;
  P.max_episode_steps = max_episode_steps;
  const char* msg = nullptr;
  const int family = step_family(P, ext != 0, mode, transport, &msg);
  why[0] = '\0';
  if (msg) {
    std::strncpy(why, msg, why_len - 1);
    why[why_len - 1] = '\0';
  }
  return family;
}

int hostsim_step_instantiated(int tile, int family) { return step_instantiated(tile, family) ? 1 : 0; }

}  // extern "C"
