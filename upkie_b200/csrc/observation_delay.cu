// SPDX-License-Identifier: Apache-2.0
//
// observation_delay.cu -- the handle-side kernels of observation-delay randomisation (upkie_b200_set_observation_delay;
// the step kernels of FAM_SENSE take the snapshots inside their ticks, step_kernel.cuh). In a translation unit of their
// own, so that the kernels of upkie_b200.cu (k_reset among them) keep their code whether or not a handle ever sets a
// spec: an explicit upkie_b200_reset draws and copies the post-reset states in k_obs_delay_reset, launched right after
// k_reset on the same stream.
#include "kernel_common.cuh"

namespace upkie_b200 {
namespace {

// the envs the reset takes (mask, NULL = all) draw their next delay, and their sensed rows become the post-reset state
__global__ void k_obs_delay_reset(const ObsDelay* __restrict__ O, int n, int n_pad, const float* __restrict__ state,
                                  const uint8_t* __restrict__ mask, uint64_t seed, uint64_t env_offset) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mask && !mask[i]) return;
  obs_delay_reset(*O, seed, env_offset + uint64_t(i), i);
  float* const col = O->rows + size_t(i);
  const size_t stride = size_t(O->stride);
  float r[UPKIE_STATE_DIM];
  for (int k = 0; k < UPKIE_STATE_DIM; ++k) r[k] = state[size_t(k) * n_pad + i];
  for (int k = 0; k < UPKIE_STATE_DIM; ++k) col[size_t(k) * stride] = r[k];
  if (O->ticks > 1) obs_delay_fill_history(*O, i, r);  // and so does every snapshot of the history
}

// rows [n][UPKIE_STATE_DIM] <-> columns [UPKIE_STATE_DIM][stride]
__global__ void k_sensed_copy(const float* __restrict__ src, int n, int stride, float* __restrict__ dst, int to_rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int k = 0; k < UPKIE_STATE_DIM; ++k) {
    if (to_rows) dst[size_t(i) * UPKIE_STATE_DIM + k] = src[size_t(k) * stride + i];
    else dst[size_t(k) * stride + i] = src[size_t(i) * UPKIE_STATE_DIM + k];
  }
}

int grid_of(int n) { return (n + 127) / 128; }

}  // namespace

cudaError_t launch_obs_delay_reset(const ObsDelay* O, int n, int n_pad, const float* state, const uint8_t* mask,
                                   uint64_t seed, uint64_t env_offset, cudaStream_t stream) {
  k_obs_delay_reset<<<grid_of(n), 128, 0, stream>>>(O, n, n_pad, state, mask, seed, env_offset);
  return cudaGetLastError();
}

cudaError_t launch_sensed_rows(const float* cols, int n, int stride, float* rows, cudaStream_t stream) {
  k_sensed_copy<<<grid_of(n), 128, 0, stream>>>(cols, n, stride, rows, 1);
  return cudaGetLastError();
}

cudaError_t launch_sensed_cols(const float* rows, int n, int stride, float* cols, cudaStream_t stream) {
  k_sensed_copy<<<grid_of(n), 128, 0, stream>>>(rows, n, stride, cols, 0);
  return cudaGetLastError();
}

}  // namespace upkie_b200
