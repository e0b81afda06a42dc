// SPDX-License-Identifier: Apache-2.0
//
// reset_randomization.cpp -- TEST INFRASTRUCTURE. The CPU build of the reset randomisation's draw (sim_core.cuh
// reset_rand_draw / reset_randomize, the code the step kernels and k_reset inline) and of the spec's validation
// (params.h reset_rand_flags). Built by tests/test_reset_randomization_cpu.py; never loaded by the product.
#include "hostsim.cpp"

extern "C" {

// draw `draw` of the env of global index `env_index`: all UPKIE_RR_DIM values
void hostsim_rr_draw(const UpkieResetRandomization* spec, uint64_t seed, uint64_t env_index, uint32_t draw, float* v) {
  reset_rand_draw(*spec, seed, env_index, draw, v);
}

// one reset of the envs [0, n) selected by mask (NULL = all) into host buffers laid out as the handle's:
// draws[n], table[UPKIE_EP_DIM][n], eps[n][6], mu[n]
void hostsim_rr_reset(const UpkieResetRandomization* spec, uint64_t seed, uint64_t env_offset, int n,
                      const uint8_t* mask, uint32_t* draws, float* table, float* eps, float* mu) {
  ResetRand R;
  std::memset(&R, 0, sizeof(R));
  R.spec = *spec;
  R.draws = draws;
  R.table = table;
  R.stride = n;
  R.eps = eps;
  R.mu = mu;
  for (int i = 0; i < n; ++i) {
    if (mask && !mask[i]) continue;
    float v[UPKIE_RR_DIM];
    reset_randomize(R, seed, env_offset + uint64_t(i), i, true, v);
  }
}

uint32_t hostsim_rr_flags(const UpkieResetRandomization* spec) { return reset_rand_flags(*spec); }

}  // extern "C"
