// SPDX-License-Identifier: Apache-2.0
//
// kernel_common.cuh -- what the translation units of libupkie_b200.so share: build-time knobs, the
// state load/store helpers, and the launch descriptor of the env-step kernel. The step kernel itself
// (step_kernel.cuh) is instantiated in the step units, step_unit.cu compiled once per TILE and one or two families,
// that nvcc compiles in parallel (build.py, step_family.h, DESIGN.md section 4). TILE is how the rows travel:
//   0  per-thread action loads / observation stores (device buffers)
//   1  per-warp shared-memory tile with coalesced 16 B accesses, the variant whose warps read actions from and
//      write observations to mapped pinned HOST memory
//   2  the TILE=1 tile path whose compact rows leave through the in-kernel rollout transport (UpkieServos only)
#pragma once

#include <cuda_runtime.h>

#include "params.h"
#include "step_family.h"

namespace upkie_b200 {

// build-time tuning knobs (tools/variants.py explores them)
#ifndef UPKIE_MAX_THREADS
#define UPKIE_MAX_THREADS 256
#endif
#ifndef UPKIE_MIN_BLOCKS
#define UPKIE_MIN_BLOCKS 1
#endif
#ifndef UPKIE_DEFAULT_BLOCK
#define UPKIE_DEFAULT_BLOCK 0  // 0 = pick per launch (pick_block)
#endif
#ifndef UPKIE_PHASE_SYNC_LEVEL  // 0 none, 1 one barrier per substep, 2 also six barriers inside the substep
#define UPKIE_PHASE_SYNC_LEVEL 1
#endif

enum { AUTORESET_DISABLED = 0, AUTORESET_NEXT_STEP = 1, AUTORESET_SAME_STEP = 2 };

// CTA-wide barrier that tolerates intra-warp divergence (non-.aligned form): every
// thread of the block arrives exactly kPhaseSyncs times per substep. It buys no
// data exchange: it keeps the block's warps within the same instruction-cache
// window of the ~100 KB substep body (ncu: stall_no_instruction was the top stall).
struct PhaseSync {
  __device__ __forceinline__ void operator()() const {
#if UPKIE_PHASE_SYNC_LEVEL >= 2
    asm volatile("barrier.sync 0;" ::: "memory");
#endif
  }
};

struct WarpAny {
  __device__ __forceinline__ bool operator()(bool p) const { return __any_sync(__activemask(), p); }
};

__device__ __forceinline__ void load_state(const float* __restrict__ st, int n_pad, int i, RobotState& S) {
  float r[UPKIE_STATE_DIM];
#pragma unroll
  for (int k = 0; k < UPKIE_STATE_DIM; ++k) r[k] = st[size_t(k) * n_pad + i];
  state_from_row(r, S);
}

__device__ __forceinline__ void store_state(float* __restrict__ st, int n_pad, int i, const RobotState& S) {
  float r[UPKIE_STATE_DIM];
  state_to_row(S, r);
#pragma unroll
  for (int k = 0; k < UPKIE_STATE_DIM; ++k) st[size_t(k) * n_pad + i] = r[k];
}

// Stash of the same-step auto-reset's pre-reset states (SimParams.final_state, upkie_b200_final_spine_obs), rows of
// n_pad floats: the step number that last wrote the env's column (uint32 bits), the state (store_state layout), and in
// spine mode the lag record (lag_to_row layout)
constexpr int kFinalMarkRow = 0, kFinalStateRow = 1, kFinalLagRow = 1 + UPKIE_STATE_DIM;
constexpr int kFinalRows = kFinalLagRow, kFinalRowsSpine = kFinalLagRow + UPKIE_LAG_DIM;
// with reset randomisation, kFinalParamCols more rows after those: the pre-reset values of the parameter-table columns
// UPKIE_EP_MEAS_NOISE .. UPKIE_EP_DIM - 1 (torque measurement noise, IMU uncertainty)
constexpr int kFinalParamCols = UPKIE_EP_DIM - UPKIE_EP_MEAS_NOISE;

// TILE=2 (rollout rows leave the GPU from inside the step kernel): n = 0 -> `obs` / `terminated` are NVSwitch multicast
// addresses (multimem.st, the switch replicates the store into every GPU's buffer); n > 0 -> plain stores into the n
// peer buffers listed here (peer-mapped symmetric memory over NVLink; the list includes this rank's own buffer).
//
// `deferred` (round 2, the default of bench.py): the rows this launch sends are those of an EARLIER step - read from
// `src_obs` / `src_term` (this rank's local slot of that step) and sent in the PROLOGUE of the kernel, so that their
// NVLink latency hides under the ~0.1 ms of simulation instead of holding up the completion of the launch - while this
// step's rows go to the local slot (`obs` / `terminated` of the launch) with plain stores.
struct PeerPtrs {
  float* obs[UPKIE_MAX_PEERS];
  uint8_t* term[UPKIE_MAX_PEERS];
  int n;
  int deferred;
  float* mc_obs;          // deferred + multicast: multicast address of the earlier step's slot (null with peer stores)
  uint8_t* mc_term;
  const float* src_obs;   // deferred: local rows of the earlier step, null = nothing to send in this launch
  const uint8_t* src_term;
};

// One launch of the env-step kernel over the envs [i0, i0 + cnt) of a handle.
struct StepArgs {
  const SimParams* P;
  int mode, autoreset, family;  // family: FAM_* of step_family.h
  int i0, cnt, n_pad, block;
  int compact_obs;      // TILE=1, servos: observation rows [6][3] (position, velocity, torque) instead of [6][5]
  int grid;             // TILE=1: number of persistent blocks (0 = one block per tile)
  int smem_carveout;    // preferred shared-memory carveout of the kernel, % of the maximum (-1: the driver's choice)
  float* state;
  const float* action;
  float* obs;
  float* reward;        // may be null
  uint8_t* terminated;
  uint8_t* truncated;   // may be null
  const float* eps;
  const float* mu;
  uint32_t* err;
  uint8_t* done_prev;
  uint32_t* episode;
  uint32_t* tick;
  uint64_t seed, env_offset;
  const float* ext;     // external forces [21][n_pad] or null (the family has `extras` when set)
  uint32_t ext_local;
  cudaStream_t stream;
  PeerPtrs peers;       // TILE=2 only
  int history;          // the delay families: a delay keeps more than one tick (the k_step_hist kernels)
  float* lag;           // spine mode: [UPKIE_LAG_DIM][n_pad] lag records, else null
};

// The step kernels of one (TILE, FAMILY) pair (step_kernel.cuh), explicitly instantiated in its step unit (step_unit.cu)
template <int TILE, int FAMILY>
cudaError_t launch_step(const StepArgs& a);
cudaError_t launch_push_rows(const PeerPtrs& pp, int n, cudaStream_t stream);  // step_unit.cu, TILE=2: flush of a rollout's last rows

}  // namespace upkie_b200
