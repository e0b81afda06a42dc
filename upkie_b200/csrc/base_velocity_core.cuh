// SPDX-License-Identifier: Apache-2.0
//
// base_velocity_core.cuh -- per-env arithmetic of the UpkieBaseVelocity epilogue (k_base_velocity_post,
// base_velocity.cu), shared by the sm_90a kernel and the CPU test build (tests/hostsim/base_velocity_post.cpp).
//
// One env after the tick's gyropod step (upkie/envs/upkie_base_velocity.py:164-202) and, when it reset in this tick,
// UpkieBaseVelocity.reset (upkie_base_velocity.py:138-162):
//   - no reset: x += v cos(yaw) dt, y += v sin(yaw) dt along the POST-step yaw, observation [x, y, yaw];
//   - reset in same-step mode: the step the env ended in is dead-reckoned first (along the gyropod's pre-reset yaw),
//     that [x, y, yaw] is the final observation; then x = y = 0, observation [0, 0, 0], commanded velocity 0;
//   - reset in next-step mode: the reset step has no agent step to dead-reckon: x = y = 0, [0, 0, 0], velocity 0.
//
// Exactness: the product expression of the device-agnostic statement (upkie_b200/base_velocity.py) is
// `xy[:, 0] += linear_velocity * torch.cos(yaw) * dt`: (v * cos(yaw)) * float(dt), then the add, each rounded to
// nearest and never contracted into an FMA, with the IEEE cosf / sinf. bv_mul / bv_add spell that out; the device
// build of this header must come from a translation unit compiled WITHOUT --use_fast_math (which would turn cosf /
// sinf into __cosf / __sinf and flush subnormals).
#pragma once

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define UPKIE_BV_HD __host__ __device__ __forceinline__
#else
#define UPKIE_BV_HD inline
#endif

#if defined(__CUDA_ARCH__) && defined(__USE_FAST_MATH__)
#error "base_velocity_core.cuh needs the IEEE cosf / sinf: compile its translation unit without --use_fast_math"
#endif

namespace upkie_b200 {

UPKIE_BV_HD float bv_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;  // ISO C++ mode: g++ does not contract across statements or expressions into an FMA
#endif
}

UPKIE_BV_HD float bv_add(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}

// x + (v * cos(yaw)) * dt and y + (v * sin(yaw)) * dt, in base_velocity_tick's order of operations
UPKIE_BV_HD void bv_dead_reckon(float v, float yaw, float dt, float& x, float& y) {
  x = bv_add(x, bv_mul(bv_mul(v, cosf(yaw)), dt));
  y = bv_add(y, bv_mul(bv_mul(v, sinf(yaw)), dt));
}

// One env. `reset`: the env reset in this tick (same_step: its gyropod step ended the episode and reset it; next_step:
// the step kernel ran its pending reset instead of a step). `yaw`: column 2 of the gyropod observation of this tick;
// `final_yaw`: column 2 of the gyropod step's final-observation row (read in same-step mode on reset only).
// Updates xy and v_cmd in place, writes obs[3]; returns true when fin[3] holds a final-observation row.
UPKIE_BV_HD bool base_velocity_post_env(bool same_step, bool reset, float v, float yaw, float final_yaw, float dt,
                                        float xy[2], float& v_cmd, float obs[3], float fin[3]) {
  if (!reset) {
    bv_dead_reckon(v, yaw, dt, xy[0], xy[1]);
    obs[0] = xy[0];
    obs[1] = xy[1];
    obs[2] = yaw;
    return false;
  }
  bool wrote = false;
  if (same_step) {
    float x = xy[0], y = xy[1];
    bv_dead_reckon(v, final_yaw, dt, x, y);
    fin[0] = x;
    fin[1] = y;
    fin[2] = final_yaw;
    wrote = true;
  }
  xy[0] = xy[1] = 0.f;  // UpkieBaseVelocity.reset: x = y = 0 (upkie_base_velocity.py:157-158)
  obs[0] = obs[1] = obs[2] = 0.f;
  v_cmd = 0.f;  // MPCBalancer.reset (mpc_balancer.py:228-235); the caller drops the warm start
  return wrote;
}

}  // namespace upkie_b200
