// SPDX-License-Identifier: Apache-2.0
//
// reset_randomization.cu -- the handle-side kernels of reset randomisation (upkie_b200_set_reset_randomization; the
// step kernels draw inside their reset branches, step_kernel.cuh). In a translation unit of their own, so that the
// kernels of upkie_b200.cu (k_reset among them) keep their code whether or not a handle ever sets a spec: the reset of
// an explicit upkie_b200_reset draws in k_reset_rand, launched right before k_reset on the same stream.
#include "kernel_common.cuh"

namespace upkie_b200 {
namespace {

// The draw of every env the reset takes (mask, NULL = all), stored into the handle's buffers; k_reset then runs the
// reset substep with the stored epsilons and friction, as with values set from the host before the reset
__global__ void k_reset_rand(const ResetRand* __restrict__ R, int n, const uint8_t* __restrict__ mask, uint64_t seed,
                             uint64_t env_offset) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mask && !mask[i]) return;
  float v[UPKIE_RR_DIM];
  reset_randomize(*R, seed, env_offset + uint64_t(i), i, true, v);
}

// the randomisation in force (upkie_b200_get_randomization): the buffers, or the nominal values without one
__global__ void k_get_randomization(const __grid_constant__ SimParams P, int n, const float* __restrict__ mu,
                                    const float* __restrict__ eps, float* __restrict__ friction,
                                    float* __restrict__ inertia_eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (friction) friction[i] = mu ? mu[i] : P.friction;
  if (inertia_eps)
    for (int k = 0; k < 6; ++k) inertia_eps[size_t(i) * 6 + k] = eps ? eps[size_t(i) * 6 + k] : 0.f;
}

__global__ void k_fill(int n, float* __restrict__ out, float v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = v;
}

// a new table holding the config's values in every column (the table a spec writes into when the handle has none)
__global__ void k_env_params_from_config(const __grid_constant__ SimParams P, int n, int n_pad,
                                         float* __restrict__ table) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int k = 0; k < UPKIE_EP_DIM; ++k) table[size_t(k) * n_pad + i] = config_env_param(P, k);
}

int grid_of(int n) { return (n + 127) / 128; }

}  // namespace

cudaError_t launch_reset_rand(const ResetRand* R, int n, const uint8_t* mask, uint64_t seed, uint64_t env_offset,
                              cudaStream_t stream) {
  k_reset_rand<<<grid_of(n), 128, 0, stream>>>(R, n, mask, seed, env_offset);
  return cudaGetLastError();
}

cudaError_t launch_get_randomization(const SimParams& P, int n, const float* mu, const float* eps, float* friction,
                                     float* inertia_eps, cudaStream_t stream) {
  k_get_randomization<<<grid_of(n), 128, 0, stream>>>(P, n, mu, eps, friction, inertia_eps);
  return cudaGetLastError();
}

cudaError_t launch_fill(int n, float* out, float v, cudaStream_t stream) {
  k_fill<<<grid_of(n), 128, 0, stream>>>(n, out, v);
  return cudaGetLastError();
}

cudaError_t launch_env_params_from_config(const SimParams& P, int n, int n_pad, float* table, cudaStream_t stream) {
  k_env_params_from_config<<<grid_of(n), 128, 0, stream>>>(P, n, n_pad, table);
  return cudaGetLastError();
}

}  // namespace upkie_b200
