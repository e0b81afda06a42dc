// SPDX-License-Identifier: Apache-2.0
//
// base_velocity_post.cpp -- TEST INFRASTRUCTURE. The CPU build of k_base_velocity_post's per-env arithmetic
// (upkie_b200/csrc/base_velocity_core.cuh, the __host__ __device__ function the kernel inlines), driven over a batch
// the way the kernel drives it. Built by tests/test_base_velocity_post.py; never loaded by the product.
#include <cstddef>
#include <cstdint>

#include "../../upkie_b200/csrc/base_velocity_core.cuh"

using namespace upkie_b200;

extern "C" {

// mode 0 disabled, 1 next step, 2 same step; reset[i] = 1: env i reset in this tick (ignored in mode 0).
// final_obs rows are written for the resetting envs of mode 2 only.
void hostsim_bv_post(int n, int mode, float dt, const uint8_t* reset, const float* action, const float* gyro_obs,
                     const float* gyro_final_obs, float* xy, float* v_cmd, float* obs, float* final_obs) {
  for (int i = 0; i < n; ++i) {
    const bool r = mode != 0 && reset[i] != 0;
    const float final_yaw = (r && mode == 2) ? gyro_final_obs[size_t(i) * 6 + 2] : 0.f;
    float v = v_cmd[i];
    float f[3];
    const bool fin = base_velocity_post_env(mode == 2, r, action[size_t(i) * 2], gyro_obs[size_t(i) * 6 + 2],
                                            final_yaw, dt, xy + size_t(i) * 2, v, obs + size_t(i) * 3, f);
    if (r) v_cmd[i] = v;
    if (fin)
      for (int k = 0; k < 3; ++k) final_obs[size_t(i) * 3 + k] = f[k];
  }
}

}  // extern "C"
