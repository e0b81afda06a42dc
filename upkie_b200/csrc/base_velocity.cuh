// SPDX-License-Identifier: Apache-2.0
//
// base_velocity.cuh -- launcher of k_base_velocity_post (base_velocity.cu, a translation unit built without
// --use_fast_math, see base_velocity_core.cuh). Called by upkie_b200_base_velocity_post (upkie_b200.cu).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

namespace upkie_b200 {

struct BaseVelocityPostArgs {
  int n;
  bool detect_resets;             // next-step and same-step modes: the sim's episode counters tell which envs reset
  bool same_step;                 // same-step mode: the envs that reset write a final-observation row
  float dt;
  const float* action;            // [n][2]
  const float* gyro_obs;          // [n][6]
  const float* gyro_final_obs;    // [n][6], same-step mode only
  const uint32_t* episode;        // [n] the sim handle's episode counters
  uint32_t* seen_episode;         // [n] the counters as of the last post step (the sim handle's copy)
  float* xy;                      // [n][2]
  float* v_cmd;                   // [n]
  uint64_t* active;               // [2][n] the MPC handle's warm-start active sets
  float* obs;                     // [n][3]
  float* final_obs;               // [n][3], same-step mode only
};

cudaError_t launch_base_velocity_post(const BaseVelocityPostArgs& a, cudaStream_t s);

}  // namespace upkie_b200
