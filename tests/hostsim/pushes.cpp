// SPDX-License-Identifier: Apache-2.0
//
// pushes.cpp -- TEST INFRASTRUCTURE. The CPU build of the push randomisation's draw and schedule (sim_core.cuh
// push_draw / push_force / push_step / push_restart / push_last_force / push_reset, the code the step kernels and
// pushes.cu inline). Built by tests/test_push_randomization_cpu.py; never loaded by the product.
#include "hostsim.cpp"

extern "C" {

// draw k of the env of global index g: gap, duration and force
void hostsim_push_draw(const UpkiePushRandomization* spec, uint64_t seed, uint64_t g, uint32_t k, uint32_t* steps,
                       float* force) {
  const PushDraw d = push_draw(*spec, seed, g, k);
  steps[0] = d.gap;
  steps[1] = d.duration;
  push_force(*spec, seed, g, k, d, force);
}

// `ticks` ticks of one env as the step kernels run them: reset[t] = 0 a counted step, 1 a next-step reset (an
// uncounted step), 2 a counted step followed by a same-step reset; force[t][3] the push of each step (what the physics
// took), count / timer the state after each step. count0 / timer0 the state before the first.
void hostsim_push_run(const UpkiePushRandomization* spec, uint64_t seed, uint64_t g, int ticks, const uint8_t* reset,
                      uint32_t count0, uint32_t timer0, float* force, uint32_t* count, uint32_t* timer) {
  uint32_t k = count0, t = timer0;
  for (int s = 0; s < ticks; ++s) {
    float f[3] = {0.f, 0.f, 0.f};
    if (reset[s] == 1) {
      const PushDraw d = push_draw(*spec, seed, g, k);
      push_restart(k, t, d.gap + d.duration);
    } else {
      uint32_t end = 0;
      push_step(*spec, seed, g, k, t, end, f);
      if (reset[s] == 2) push_restart(k, t, end);
    }
    for (int a = 0; a < 3; ++a) force[3 * s + a] = f[a];
    count[s] = k;
    timer[s] = t;
  }
}

// the force upkie_b200_get_push_forces reports for state (k, t)
void hostsim_push_last_force(const UpkiePushRandomization* spec, uint64_t seed, uint64_t g, uint32_t k, uint32_t t,
                             float* force) {
  push_last_force(*spec, seed, g, k, t, force);
}

// an explicit reset of the envs [0, n) selected by mask (NULL = all)
void hostsim_push_reset(const UpkiePushRandomization* spec, uint64_t seed, uint64_t env_offset, int n,
                        const uint8_t* mask, uint32_t* count, uint32_t* timer) {
  PushRand R;
  std::memset(&R, 0, sizeof(R));
  R.spec = *spec;
  R.count = count;
  R.timer = timer;
  for (int i = 0; i < n; ++i)
    if (!mask || mask[i]) push_reset(R, seed, env_offset + uint64_t(i), i);
}

int hostsim_push_spec_valid(const UpkiePushRandomization* spec) { return push_spec_valid(*spec) ? 1 : 0; }

}  // extern "C"
