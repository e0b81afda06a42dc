// SPDX-License-Identifier: Apache-2.0
//
// base_velocity.cu -- k_base_velocity_post: the UpkieBaseVelocity layer of one tick, after the gyropod step and
// k_spine_obs (upkie_b200_base_velocity_post, include/upkie_b200.h). One thread per env.
//
// Built WITHOUT --use_fast_math (upkie_b200/build.py): the dead reckoning must give the bits of the torch statement
// of the tick (upkie_b200/base_velocity.py), whose cos / sin are the IEEE routines (base_velocity_core.cuh).
//
// Which envs reset in this tick: every reset the step kernels sample on the device (both fused auto-resets) adds 1 to
// the sim handle's episode[i]; the handle keeps a copy of the counters as of the last post step (seen_episode). An
// env reset in this tick iff the two differ. Explicit resets from host rows (B200VectorEnv.reset) do not touch the
// counter, and cancel a pending next-step reset by clearing done_prev, so the step kernel neither resets nor counts.
#include <cuda_runtime.h>

#include "base_velocity.cuh"
#include "base_velocity_core.cuh"

namespace upkie_b200 {

__global__ void __launch_bounds__(128)
k_base_velocity_post(const BaseVelocityPostArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  bool reset = false;
  if (a.detect_resets) {
    const uint32_t ep = a.episode[i];
    reset = ep != a.seen_episode[i];
    if (reset) a.seen_episode[i] = ep;
  }
  const float v = a.action[size_t(i) * 2];  // commanded linear velocity (scalar loads: views need not be 8 B aligned)
  const float yaw = a.gyro_obs[size_t(i) * 6 + 2];
  const float final_yaw = (reset && a.same_step) ? a.gyro_final_obs[size_t(i) * 6 + 2] : 0.f;
  float p[2] = {a.xy[size_t(i) * 2], a.xy[size_t(i) * 2 + 1]};
  float v_cmd = 0.f;
  float o[3], f[3];
  const bool fin = base_velocity_post_env(a.same_step, reset, v, yaw, final_yaw, a.dt, p, v_cmd, o, f);
  a.xy[size_t(i) * 2] = p[0];
  a.xy[size_t(i) * 2 + 1] = p[1];
  a.obs[size_t(i) * 3 + 0] = o[0];
  a.obs[size_t(i) * 3 + 1] = o[1];
  a.obs[size_t(i) * 3 + 2] = o[2];
  if (fin) {
    a.final_obs[size_t(i) * 3 + 0] = f[0];
    a.final_obs[size_t(i) * 3 + 1] = f[1];
    a.final_obs[size_t(i) * 3 + 2] = f[2];
  }
  if (reset) {
    // MPCBalancer.reset: commanded velocity 0 and no warm start (k_mpc_reset's effect for this env). In next-step
    // mode the MPC of this tick ran on the terminal spine observation; its result for env i is discarded here.
    a.v_cmd[i] = v_cmd;
    a.active[i] = 0ull;
    a.active[size_t(a.n) + i] = 0ull;
  }
}

cudaError_t launch_base_velocity_post(const BaseVelocityPostArgs& a, cudaStream_t s) {
  k_base_velocity_post<<<(a.n + 127) / 128, 128, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace upkie_b200
