// SPDX-License-Identifier: Apache-2.0
//
// pushes.cu -- the handle-side kernels of push randomisation (upkie_b200_set_push_randomization; the step kernels run
// the schedule inside their ticks, step_kernel.cuh). In a translation unit of their own, so that the kernels of
// upkie_b200.cu (k_reset among them) keep their code whether or not a handle ever sets a spec: an explicit
// upkie_b200_reset restarts the schedules in k_push_reset, launched right before k_reset on the same stream.
#include "kernel_common.cuh"

namespace upkie_b200 {
namespace {

// the envs the reset takes (mask, NULL = all) start their next draw
__global__ void k_push_reset(const PushRand* __restrict__ R, int n, const uint8_t* __restrict__ mask, uint64_t seed,
                             uint64_t env_offset) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mask && !mask[i]) return;
  push_reset(*R, seed, env_offset + uint64_t(i), i);
}

// the push force of each env's last step, from its schedule state (R null: no spec, zeros)
__global__ void k_push_forces(const PushRand* __restrict__ R, int n, uint64_t seed, uint64_t env_offset,
                              float* __restrict__ force) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float f[3] = {0.f, 0.f, 0.f};
  if (R) push_last_force(R->spec, seed, env_offset + uint64_t(i), R->count[i], R->timer[i], f);
  for (int k = 0; k < 3; ++k) force[size_t(i) * 3 + k] = f[k];
}

int grid_of(int n) { return (n + 127) / 128; }

}  // namespace

cudaError_t launch_push_reset(const PushRand* R, int n, const uint8_t* mask, uint64_t seed, uint64_t env_offset,
                              cudaStream_t stream) {
  k_push_reset<<<grid_of(n), 128, 0, stream>>>(R, n, mask, seed, env_offset);
  return cudaGetLastError();
}

cudaError_t launch_push_forces(const PushRand* R, int n, uint64_t seed, uint64_t env_offset, float* force,
                               cudaStream_t stream) {
  k_push_forces<<<grid_of(n), 128, 0, stream>>>(R, n, seed, env_offset, force);
  return cudaGetLastError();
}

}  // namespace upkie_b200
