// SPDX-License-Identifier: Apache-2.0
//
// action_delay.cu -- the handle-side kernels of action-delay randomisation (upkie_b200_set_action_delay; the step
// kernels apply the delay inside their ticks, step_kernel.cuh). In a translation unit of their own, so that the kernels
// of upkie_b200.cu (k_reset among them) keep their code whether or not a handle ever sets a spec: an explicit
// upkie_b200_reset draws and stops the previous commands in k_action_delay_reset, launched right before k_reset on the
// same stream.
#include "kernel_common.cuh"

namespace upkie_b200 {
namespace {

// the envs the reset takes (mask, NULL = all) draw their next delay and hold the stop row
__global__ void k_action_delay_reset(const ActionDelay* __restrict__ A, int n, const uint8_t* __restrict__ mask,
                                     uint64_t seed, uint64_t env_offset) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mask && !mask[i]) return;
  action_delay_reset(*A, seed, env_offset + uint64_t(i), i);
}

// command rows [n][UPKIE_ACT_DIM] of the columns [UPKIE_ACT_DIM][stride] (cols null: stop rows)
__global__ void k_command_rows(const float* __restrict__ cols, int n, int stride, float* __restrict__ rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int c = 0; c < UPKIE_ACT_DIM; ++c)
    rows[size_t(i) * UPKIE_ACT_DIM + c] = cols ? cols[size_t(c) * stride + i] : action_delay_stop_value(c);
}

// the columns of command rows (rows null: stop rows)
__global__ void k_command_cols(const float* __restrict__ rows, int n, int stride, float* __restrict__ cols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int c = 0; c < UPKIE_ACT_DIM; ++c)
    cols[size_t(c) * stride + i] = rows ? rows[size_t(i) * UPKIE_ACT_DIM + c] : action_delay_stop_value(c);
}

int grid_of(int n) { return (n + 127) / 128; }

}  // namespace

cudaError_t launch_action_delay_reset(const ActionDelay* A, int n, const uint8_t* mask, uint64_t seed,
                                      uint64_t env_offset, cudaStream_t stream) {
  k_action_delay_reset<<<grid_of(n), 128, 0, stream>>>(A, n, mask, seed, env_offset);
  return cudaGetLastError();
}

cudaError_t launch_command_rows(const float* cols, int n, int stride, float* rows, cudaStream_t stream) {
  k_command_rows<<<grid_of(n), 128, 0, stream>>>(cols, n, stride, rows);
  return cudaGetLastError();
}

cudaError_t launch_command_cols(const float* rows, int n, int stride, float* cols, cudaStream_t stream) {
  k_command_cols<<<grid_of(n), 128, 0, stream>>>(rows, n, stride, cols);
  return cudaGetLastError();
}

}  // namespace upkie_b200
