// SPDX-License-Identifier: Apache-2.0
//
// delay_ticks.cpp -- TEST INFRASTRUCTURE. The CPU build of the history helpers of delays of more than one tick
// (sim_core.cuh delay_split / delay_ring_row / action_delay_rows / obs_delay_rows / action_delay_reset /
// obs_delay_fill_history, params.h *_delay_spec_error, the code the step kernels and the delay kernels inline). Built
// by tests/test_delay_ticks_cpu.py; never loaded by the product.
#include "hostsim.cpp"

extern "C" {

// {q, r} of delay_split
void hostsim_delay_split(uint32_t d, uint32_t nb, uint32_t ticks, uint32_t* out) {
  const DelaySplit s = delay_split(d, nb, ticks);
  out[0] = s.q;
  out[1] = s.r;
}

uint32_t hostsim_delay_ring_row(uint32_t head, uint32_t ticks, uint32_t age) { return delay_ring_row(head, ticks, age); }

// {first, second, r} of action_delay_rows
void hostsim_action_delay_rows(uint32_t d, uint32_t nb, uint32_t ticks, uint32_t head, uint32_t* out) {
  const ActionDelayRows r = action_delay_rows(d, nb, ticks, head);
  out[0] = r.first;
  out[1] = r.second;
  out[2] = r.r;
}

// {newest, report, r} of obs_delay_rows
void hostsim_obs_delay_rows(uint32_t d, uint32_t nb, uint32_t ticks, uint32_t head, uint32_t* out) {
  const ObsDelayRows r = obs_delay_rows(d, nb, ticks, head);
  out[0] = r.newest;
  out[1] = r.report;
  out[2] = r.r;
}

// an explicit reset of the envs [0, n) with a history of `ticks` commands [ticks][UPKIE_ACT_DIM][stride]
void hostsim_action_delay_reset_ticks(const UpkieActionDelay* spec, uint64_t seed, int n, uint32_t* count,
                                      uint32_t* delay, float* command, int stride, int ticks) {
  ActionDelay A;
  std::memset(&A, 0, sizeof(A));
  A.spec = *spec;
  A.count = count;
  A.delay = delay;
  A.command = command;
  A.stride = stride;
  A.ticks = ticks;
  for (int i = 0; i < n; ++i) {
    action_delay_reset(A, seed, uint64_t(i), i);
    action_delay_fill_history(A, i);
  }
}

// the snapshots [ticks][UPKIE_STATE_DIM][stride] of env i after a reset to the state row r
void hostsim_obs_delay_fill_history(float* hist, int stride, int ticks, int i, const float* r) {
  ObsDelay O;
  std::memset(&O, 0, sizeof(O));
  O.hist = hist;
  O.stride = stride;
  O.ticks = ticks;
  obs_delay_fill_history(O, i, r);
}

// the *_delay_spec_error of a handle with nb_substeps and a history of `ticks` (action: 0, observation: 1)
int hostsim_delay_ticks_spec_error(int which, uint32_t low, uint32_t high, int nb_substeps, uint32_t ticks, char* why,
                                   int why_len) {
  SimParams P;
  std::memset(&P, 0, sizeof(P));
  P.nb_substeps = nb_substeps;
  P.joint_limits = 3;
  const char* msg = which == 0 ? action_delay_spec_error(UpkieActionDelay{low, high}, P, ticks)
                               : obs_delay_spec_error(UpkieObservationDelay{low, high}, P, ticks);
  why[0] = '\0';
  if (msg) {
    std::strncpy(why, msg, why_len - 1);
    why[why_len - 1] = '\0';
  }
  return msg ? 1 : 0;
}

}  // extern "C"
