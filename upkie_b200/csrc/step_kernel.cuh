// SPDX-License-Identifier: Apache-2.0
//
// step_kernel.cuh -- the env-step kernel (one thread = one robot) and its launcher template.
//   k_step<MODE, AUTORESET, FAMILY, TILE>   one 5 ms env tick: action front-end, 5 x (moteus torque law,
//       articulated-body dynamics, wheel-ground contact solve, semi-implicit integration), observation,
//       termination; optional fused auto-reset; the optional features of FAMILY (step_family.h).
//   launch_step<TILE, FAMILY>   the launcher of a (TILE, FAMILY) pair, explicitly instantiated in its step unit
//       (step_unit.cu, build.py, DESIGN.md section 4).
#pragma once

#include <map>
#include <mutex>
#include <utility>

#include "kernel_common.cuh"

namespace upkie_b200 {
namespace {

// NVSwitch multicast stores (TILE=2): one store to the multicast address of a symmetric buffer is replicated by the
// switch into the same offset of every GPU's buffer -- the rollout "all-gather" without any collective kernel or copy.
__device__ __forceinline__ void mc_store4(float4* addr, const float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void mc_store_u32(uint32_t* addr, uint32_t v) {
  asm volatile("multimem.st.relaxed.sys.global.b32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}

// The observation row env `i` would return if it did not reset in this step, stored at its row of P.final_obs before
// the same-step auto-reset overwrites the state. Same layout as the step's own rows: servos [6][5] or compact [6][3]
// (spine mode: the rows the spine assembled), gyropod o6, pendulum [4]. Per-thread stores: only resetting lanes write.
template <int MODE, bool SPINE>
__device__ __forceinline__ void store_final_obs(const SimParams& P, const RobotState& S, const SpineLag& L,
                                                const float* o6, const NoiseCtx* nz, bool compact, int i, int env_col) {
  if (MODE == MODE_SERVOS) {
    float tq[6];
    measured_torques(P, S, nz, tq, env_col);
    const int dim = compact ? 18 : UPKIE_OBS_DIM;
    float* o = P.final_obs + size_t(i) * dim;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const float q = SPINE ? L.obs_rep[3 * j] : S.q[j];
      const float qd = SPINE ? L.obs_rep[3 * j + 1] : S.qd[j];
      const float t = SPINE ? L.obs_rep[3 * j + 2] : tq[j];
      if (compact) {
        o[3 * j] = q; o[3 * j + 1] = qd; o[3 * j + 2] = t;
      } else {
        o[5 * j] = q; o[5 * j + 1] = qd; o[5 * j + 2] = t;
        o[5 * j + 3] = SPINE ? 20.0f : 42.0f;  // BulletInterface.cpp:70 / pybullet_backend.py:471
        o[5 * j + 4] = 18.0f;                  // pybullet_backend.py:472
      }
    }
  } else if (MODE == MODE_GYROPOD) {
#pragma unroll
    for (int k = 0; k < 6; ++k) P.final_obs[size_t(i) * 6 + k] = o6[k];
  } else {
    float* o = P.final_obs + size_t(i) * 4;
    o[0] = o6[1]; o[1] = o6[0]; o[2] = o6[4]; o[3] = o6[3];  // upkie_pendulum.py:17
  }
}

// The pre-reset state of env `i`, stashed before the same-step auto-reset overwrites it (upkie_b200_final_spine_obs
// turns it into the spine observation the env would have returned, k_spine_obs): the step's number in the mark
// row, the state, and in spine mode the lag record. Per-thread stores on the reset branch only.
template <bool SPINE>
__device__ __forceinline__ void store_final_state(const SimParams& P, const RobotState& S, const SpineLag& L, int n_pad,
                                                  int i) {
  reinterpret_cast<uint32_t*>(P.final_state + size_t(kFinalMarkRow) * n_pad)[i] = P.final_gen;
  store_state(P.final_state + size_t(kFinalStateRow) * n_pad, n_pad, i, S);
  if (SPINE) {
    float lr[UPKIE_LAG_DIM];
    lag_to_row(L, lr);
#pragma unroll
    for (int k = 0; k < UPKIE_LAG_DIM; ++k) P.final_state[size_t(kFinalLagRow + k) * n_pad + i] = lr[k];
  }
}

// Reset randomisation, same-step auto-reset with the stash requested: the pre-reset values of the parameter-table
// columns k_spine_obs reads (torque measurement noise and IMU uncertainty), read before the reset's draw
// overwrites them, in the stash rows after the state (and lag) rows
template <bool SPINE>
__device__ __forceinline__ void store_final_params(const SimParams& P, int n_pad, int i) {
  constexpr int row0 = SPINE ? kFinalRowsSpine : kFinalRows;
#pragma unroll
  for (int k = 0; k < kFinalParamCols; ++k)
    P.final_state[size_t(row0 + k) * n_pad + i] = env_param(P, i, UPKIE_EP_MEAS_NOISE + k);
}

// Reset randomisation of a resetting lane (P.reset_rand set): env i's next draw into v, and in registers the values
// the rest of this launch uses from it: the inertia epsilons, the floor friction and the torque measurement-noise
// levels of the observation (an unselected column keeps the table's value). The draw is stored at the end of the
// tick (reset_rand_store), after every read of the lane's row: the read-only path the table is read through need not
// see a lane's own stores of the same launch.
__device__ __forceinline__ void reset_rand_lane(const SimParams& P, uint64_t seed, uint64_t env_index, int i,
                                                float v[UPKIE_RR_DIM], float eps[6], float& mu, float meas_sd[6]) {
  const ResetRand& R = *P.reset_rand;
#pragma unroll
  for (int j = 0; j < 6; ++j) meas_sd[j] = env_param(P, i, UPKIE_EP_MEAS_NOISE + j);
  reset_rand_draw(R.spec, seed, env_index, R.draws[i] + 1u, v);
  const uint64_t cols = R.spec.columns;
#pragma unroll
  for (int b = 0; b < 6; ++b)
    if ((cols >> (UPKIE_RR_INERTIA + b)) & 1u) eps[b] = v[UPKIE_RR_INERTIA + b];
  if ((cols >> UPKIE_RR_FRICTION) & 1u) mu = v[UPKIE_RR_FRICTION];
#pragma unroll
  for (int j = 0; j < 6; ++j)
    if ((cols >> (UPKIE_EP_MEAS_NOISE + j)) & 1u) meas_sd[j] = v[UPKIE_EP_MEAS_NOISE + j];
}

// A history of K > 1 ticks: the env's ring moves on by one row. Every step advances every env's ring, a resetting lane
// included (its reset refills the whole ring, so the row it lands on does not matter to it), and nothing else moves
// them: the rings of all envs stay on the same row, and a warp's history loads and stores stay coalesced rows.
__device__ __forceinline__ void delay_ring_advance(uint32_t* head, int ticks, int i) {
  if (ticks > 1) __stcg(head + i, (__ldcg(head + i) + 1u) % uint32_t(ticks));
}

// Observation delay with a history of K > 1 ticks: the sensed columns of ring row `srep` (the snapshot the step
// reports) into env i's sensed row, stored by live lanes; the sensed row's address
__device__ __forceinline__ float* obs_delay_report(const ObsDelay& O, uint32_t srep, int i, bool live) {
  const size_t stride = size_t(O.stride);
  float* const row = O.rows + size_t(i);
  const float* const src = O.hist + size_t(i) + size_t(srep) * UPKIE_STATE_DIM * stride;
  if (live) {
#pragma unroll
    for (int k = 0; k < UPKIE_STATE_DIM; ++k)
      if (obs_delay_sensed(k)) __stcg(row + size_t(k) * stride, __ldcg(src + size_t(k) * stride));
  }
  return row;
}

// ---- one env tick of the robot `tid` --------------------------------------------------
// `tile4` is this warp's staging tile (TILE >= 1): on entry it holds the warp's 32 action rows when
// `full` (prefetched by the caller), during the substeps each lane's clamped row, and it is reused to transpose the
// observation rows on the way out.
// HIST (the delay families' k_step_hist kernels): a delay keeps a history of more than one tick; compiled out of k_step
template <int MODE, int AUTORESET, int FAMILY, int TILE, bool HIST = false>
__device__ __forceinline__ void step_env(
    const SimParams& P, int tid, int n, int n_pad, float* __restrict__ state, const float* __restrict__ action,
    float* __restrict__ obs, float* __restrict__ reward, uint8_t* __restrict__ terminated,
    uint8_t* __restrict__ truncated, const float* __restrict__ eps_all, const float* __restrict__ mu_all,
    uint32_t* __restrict__ err, uint8_t* __restrict__ done_prev, uint32_t* __restrict__ episode,
    uint32_t* __restrict__ tick, uint64_t seed, uint64_t env_offset, const float* __restrict__ ext,
    uint32_t ext_local, float4* tile4, bool full, bool compact, const PeerPtrs* peers = nullptr,
    float* __restrict__ lag = nullptr) {
  const bool live = tid < n;
  const int i = live ? tid : n - 1;  // tail lanes shadow the last robot, stores masked
  const int lane = threadIdx.x & 31;
  const int wb = tid - lane;  // first env of this warp
  constexpr StepFamily F = step_family_traits(FAMILY);

  RobotState S;
  load_state(state, n_pad, i, S);
  float epsv[6];
  const float* eps = nullptr;
  if (eps_all) {
#pragma unroll
    for (int k = 0; k < 6; ++k) epsv[k] = eps_all[size_t(i) * 6 + k];
    eps = epsv;
  }
  float mu = mu_all ? mu_all[i] : P.friction;
  // reset randomisation (F.reset_rand kernels, P.reset_rand set; the handle gives it eps_all and mu_all, so that `eps`
  // is epsv): whether this lane drew in this launch, its draw, and the measurement-noise levels of its observation
  bool drawn = false;
  float rr_v[UPKIE_RR_DIM];
  float meas_sd[6];

  bool resetting = false;
  if (AUTORESET == AUTORESET_NEXT_STEP) resetting = done_prev[i] != 0;

  // push randomisation (F.push kernels, P.push set: a uniform branch): this tick's push, in registers, and the
  // env's schedule state after the tick (stored at its end). The step of a next-step reset is not counted.
  const bool pushing = F.push && P.push;
  ExtPush pu{0, {0.f, 0.f, 0.f}};
  uint32_t push_k = 0, push_t = 0, push_end = 0;
  if (pushing) {
    const PushRand& R = *P.push;
    pu.body = R.spec.body;
    push_k = R.count[i];
    push_t = R.timer[i];
    if (resetting) {
      const PushDraw d = push_draw(R.spec, seed, env_offset + uint64_t(i), push_k);
      push_restart(push_k, push_t, d.gap + d.duration);
    } else {
      push_step(R.spec, seed, env_offset + uint64_t(i), push_k, push_t, push_end, pu.f);
    }
  }

  uint32_t e = 0;
  float a[UPKIE_ACT_DIM];
  float a0 = 0.f, a1 = 0.f;
  if (MODE == MODE_SERVOS) {
    if (TILE && full) {
#pragma unroll
      for (int k = 0; k < UPKIE_ACT_DIM / 4; ++k) {
        const float4 v = tile4[lane * (UPKIE_ACT_DIM / 4) + k];
        a[4 * k + 0] = v.x; a[4 * k + 1] = v.y; a[4 * k + 2] = v.z; a[4 * k + 3] = v.w;
      }
      __syncwarp();
    } else {
      const float4* ap = reinterpret_cast<const float4*>(action + size_t(i) * UPKIE_ACT_DIM);
#pragma unroll
      for (int k = 0; k < UPKIE_ACT_DIM / 4; ++k) {
        const float4 v = __ldg(ap + k);
        a[4 * k + 0] = v.x; a[4 * k + 1] = v.y; a[4 * k + 2] = v.z; a[4 * k + 3] = v.w;
      }
    }
  } else if (MODE == MODE_GYROPOD) {
    const float2 v = __ldg(reinterpret_cast<const float2*>(action) + i);
    a0 = v.x; a1 = v.y;
  } else {
    a0 = __ldg(action + i);
    a1 = 0.f;  // upkie_pendulum.py:137
  }

  // One inlined copy of the physics serves both the regular tick (nb_substeps
  // substeps under the torque law) and the fused auto-reset (new initial state,
  // ONE zero-torque substep, pybullet_backend.py:227-228): resetting lanes run a
  // single iteration of the same loop, which keeps the kernel's code small
  // (instruction-cache footprint) and the warp converged.
  NoiseCtx nz{env_offset + uint64_t(i), 0u};
  if (F.extras) {
    nz.tick = tick[i] + 1u;
    if (live) tick[i] = nz.tick;
  }
  // external forces ride on the F.extras instantiations so the plain kernels stay untouched
  const ExtForces xf{ext ? ext + i : nullptr, size_t(n_pad), ext_local};
  // this robot's column of the per-env parameter table. The FAM_LIMITS kernels (the headline's family) never run with
  // a table, the host picks their FAM_TABLE copy then: -1 compiles the table reads out of them, so that their register
  // allocation is the one they have without the feature
  const int env_col = F.table ? i : -1;
  int nsub = P.nb_substeps;
  // spine mode (config.spine_mode, UpkieServos): every substep is one cycle of the Bullet spine (FAM_SPINE: its own
  // step units, step_*_spine, so that the other kernels do not carry the lag record)
  constexpr bool spine = F.spine && MODE == MODE_SERVOS;
  SpineLag L;
  if (spine) {
    float lr[UPKIE_LAG_DIM];
#pragma unroll
    for (int k = 0; k < UPKIE_LAG_DIM; ++k) lr[k] = lag[size_t(k) * n_pad + i];
    lag_from_row(lr, L);
  }
  if (resetting) {
    const uint32_t ep = episode[i] + 1u;
    if (live) episode[i] = ep;
    float init[UPKIE_INIT_DIM];
    sample_init_state(P, seed, env_offset + uint64_t(i), uint64_t(ep), init);
    if (F.reset_rand && P.reset_rand) {
      reset_rand_lane(P, seed, env_offset + uint64_t(i), i, rr_v, epsv, mu, meas_sd);
      drawn = true;
    }
    if (spine) {
      reset_pose_spine(P, S, init, L);
      nsub = 3;  // three cycles with the servos stopped (Spine.cpp:119-125)
    } else {
      reset_pose(S, init);
      nsub = 1;
    }
  } else {
    if (MODE != MODE_SERVOS) e |= gyropod_action(P, S, a0, a1, a);
    e |= clamp_servo_action(P, a);
  }
  // action delay (F.delay kernels, P.action_delay set: a uniform branch). A tick swaps this tick's command into the
  // env's column of the command buffer and enters its substeps with the previous one in `a`; substep `dly` loads the
  // new one back (action_delay_substep) into the row the substeps read (the tile row for TILE >= 1, below), so that one
  // row is held per lane. A next-step reset draws and holds the
  // stop row instead; its reset substep never switches.
  // The buffer's address and stride are read into registers once and the row goes through global-space accesses:
  // reached through the generic pointers of the device block, every store of the row could alias the block, and each
  // of the 36 elements then re-read the pointer and waited for it (a chain of dependent loads per env that made the
  // tick 2.2 times as long). The previous row is read whole before the new one is written. The loads are coherent
  // (ld.global.cg), not the read-only path, which need not return a thread's own stores of the same launch.
  // A history of K > 1 ticks (A.ticks, a uniform branch; delay_split): the buffer is a ring of K rows, and a delay of
  // q whole ticks and r substeps enters the tick with the command of age q (tick t - q - 1), stores this tick's into the
  // oldest row (age K - 1, read before it is overwritten when q = K - 1), and substep r loads the command of tick t - q
  // from row `dsec` (this tick's own for q = 0).
  const bool delaying = F.delay && P.action_delay;
  uint32_t dly = 0xffffffffu;
  size_t dsec = 0;  // the ring row substep dly loads, in floats (0 for K = 1)
  if (delaying) {
    const ActionDelay& A = *P.action_delay;
    if (resetting) {
      if (live) {
        action_delay_reset(A, seed, env_offset + uint64_t(i), i);
        if (HIST) {
          action_delay_fill_history(A, i);
          delay_ring_advance(A.head, A.ticks, i);
        }
      }
    } else {
      float* col = A.command + size_t(i);
      const size_t stride = size_t(A.stride);
      dly = __ldcg(A.delay + i);
      const float* first = col;
      if (HIST && A.ticks > 1) {
        const uint32_t K = uint32_t(A.ticks), h = __ldcg(A.head + i);
        const ActionDelayRows dr = action_delay_rows(dly, uint32_t(P.nb_substeps), K, h);
        const size_t row = size_t(UPKIE_ACT_DIM) * stride;
        dly = dr.r;
        first = col + dr.first * row;
        dsec = dr.second * row;
        col += h * row;
        if (live) __stcg(A.head + i, (h + 1u) % K);
      }
      float prev[UPKIE_ACT_DIM];
#pragma unroll
      for (int c = 0; c < UPKIE_ACT_DIM; ++c) prev[c] = __ldcg(first + size_t(c) * stride);
      if (live) {
#pragma unroll
        for (int c = 0; c < UPKIE_ACT_DIM; ++c) __stcg(col + size_t(c) * stride, a[c]);
      }
#pragma unroll
      for (int c = 0; c < UPKIE_ACT_DIM; ++c) a[c] = prev[c];
    }
  }
  // TILE >= 1: the row the substeps read (torque law, action delay, spine cycle) is the lane's own row of the warp's
  // tile, written here whole (9 x 16 B at a stride of 9 float4: conflict-free) whether the row came from the tile or
  // from global memory, instead of a 36-float register array that ptxas spills to the local-memory frame and reloads in
  // every substep. The tile is next used by the observation transpose after the substep loop. TILE = 0: the registers.
  float* arow = a;
  if (TILE) {
    float4* row = tile4 + lane * (UPKIE_ACT_DIM / 4);
#pragma unroll
    for (int k = 0; k < UPKIE_ACT_DIM / 4; ++k) row[k] = make_float4(a[4 * k], a[4 * k + 1], a[4 * k + 2], a[4 * k + 3]);
    arow = reinterpret_cast<float*>(row);
  }
  // observation delay (F.sense kernels, P.obs_delay set: a uniform branch). A lane with delay `sdl` stores the sensed
  // fields of its state at the end of substep nb_substeps - sdl - 1 (before the loop for sdl = nb_substeps, after the
  // observation update for sdl = 0) into the env's column of the sensed rows, and builds its observation from them
  // after the tick (obs_delay_snapshot, obs_delay_sensed_state). A resetting lane draws its next delay, and its row
  // becomes a copy of the post-reset state at the end of the tick. As for the action delay, the column's address and
  // stride are read into registers once and the row goes through global-space coherent accesses (ld/st.global.cg):
  // the loads read back this thread's own stores of the same launch.
  const bool sensing = F.sense && P.obs_delay;
  float* scol = nullptr;
  size_t sstride = 0;
  uint32_t sdl = 0xffffffffu;  // resetting lanes: no snapshot
  uint32_t srep = 0;           // K > 1: the ring row of the snapshot the step reports
  // A history of K > 1 ticks (O.ticks, a uniform branch; delay_split): a delay of q whole ticks and r substeps takes
  // this tick's snapshot at substep nb - r into the oldest row of the ring (`scol` points there for the substeps; it
  // first takes the newest snapshot's IMU velocity, which the snapshot differentiates against), and the step reports
  // the snapshot of age q, copied into the sensed row after the substeps (obs_delay_report).
  if (sensing) {
    const ObsDelay& O = *P.obs_delay;
    scol = O.rows + size_t(i);
    sstride = size_t(O.stride);
    if (resetting) {
      if (live) {
        obs_delay_reset(O, seed, env_offset + uint64_t(i), i);
        if (HIST) delay_ring_advance(O.head, O.ticks, i);
      }
    } else if (HIST && O.ticks > 1) {
      const uint32_t K = uint32_t(O.ticks), h = __ldcg(O.head + i);
      const ObsDelayRows dr = obs_delay_rows(__ldcg(O.delay + i), uint32_t(P.nb_substeps), K, h);
      sdl = dr.r;
      srep = dr.report;
      const size_t row = size_t(UPKIE_STATE_DIM) * sstride;
      float* const hcol = O.hist + size_t(i);
      scol = hcol + h * row;
      const float* const newest = hcol + dr.newest * row;
      if (live) {
#pragma unroll
        for (int k = 0; k < 3; ++k)
          __stcg(scol + size_t(UPKIE_ST_PREV_IMU_VEL + k) * sstride,
                 __ldcg(newest + size_t(UPKIE_ST_PREV_IMU_VEL + k) * sstride));
        __stcg(O.head + i, (h + 1u) % K);
      }
    } else {
      sdl = min(__ldcg(O.delay + i), uint32_t(P.nb_substeps));
    }
  }
  auto sense_load = [&](int k) { return __ldcg(scol + size_t(k) * sstride); };
  auto sense_store = [&](int k, float v) { __stcg(scol + size_t(k) * sstride, v); };
  if (sensing && live && sdl == uint32_t(P.nb_substeps)) {  // the state at the start of the tick
    float v[3];
    imu_velocity(P, S, v);
    obs_delay_snapshot(P, S, v, sense_load, sense_store);
  }
  if (spine && !resetting) spine_assemble_observation(S, L);  // the first cycle's observation (Spine.cpp:126-131)
  const int nloop = (AUTORESET == AUTORESET_NEXT_STEP && spine && P.nb_substeps < 3) ? 3 : P.nb_substeps;
  for (int sub = 0; sub < nloop; ++sub) {
#if UPKIE_PHASE_SYNC_LEVEL >= 1
    __syncthreads();  // once per substep: all threads are converged here
#endif
    if (sub < nsub) {
      if (delaying) {
        action_delay_substep(sub, dly, arow, [&](int c) {
          const ActionDelay& A = *P.action_delay;
          return __ldcg(A.command + dsec + size_t(c) * size_t(A.stride) + size_t(i));
        });
      }
      // the body-ground contacts of the tick's last substep go to the handle's record (F.body kernels)
      const BodyRecOut br{(F.body && P.body_rec && live && sub == nsub - 1) ? P.body_rec + i : nullptr,
                          size_t(P.body_rec_stride)};
      if (spine) {
        if (resetting && sub == 2) spine_assemble_observation(S, L);
        spine_cycle(P, S, L, arow, resetting, eps, mu, WarpAny(), PhaseSync(), P.joint_limits >= 1 ? P.joint_limits : 1, br,
                    i);
      } else {
        // F.limits: the device's two limit modes (1 and 0 alias to 3 there, see physics_substep_paired), spelled as
        // a choice between two nonzero constants so that the compiler drops servo_substep's limits == 0 branches, a
        // second and third inlined copy of the substep that these kernels never run
        servo_substep(P, S, arow, resetting, eps, mu, WarpAny(), PhaseSync(), F.extras ? &nz : nullptr, sub,
                      (F.extras && ext) ? &xf : nullptr, F.limits ? (P.joint_limits == 2 ? 2 : 3) : 0, br, env_col,
                      pushing ? &pu : nullptr);
      }
      // the end of substep nb_substeps - sdl - 1 (0 < sdl < nb_substeps)
      if (sensing && live && sdl != 0 && uint32_t(sub) + sdl + 1u == uint32_t(P.nb_substeps)) {
        float v[3];
        imu_velocity(P, S, v);
        obs_delay_snapshot(P, S, v, sense_load, sense_store);
      }
    } else {
#pragma unroll
      for (int k = 0; k < kPhaseSyncs; ++k) PhaseSync()();
    }
  }
  if (!spine) observe_update(P, S);  // spine mode: the cycles read the IMU
  // sdl = 0: the end of the tick, with the IMU velocity observe_update just computed
  if (sensing && live && sdl == 0) obs_delay_snapshot(P, S, S.prev_imu_vel, sense_load, sense_store);
  if (resetting) {
    reset_wrapper_state(S);
  } else {
    e |= state_sanity(S);
    if (MODE != MODE_SERVOS) {
      S.yaw += a1 * P.dt;  // integrates the unclamped action[1], upkie_gyropod.py:383-385
      S.yaw_vel = a1;
    }
  }

  // observation, reward, termination
  bool term = false;
  float o6[6];
  if (MODE == MODE_SERVOS) {
    if (P.servos_fall_termination) term = (fabsf(base_pitch(S)) > P.fall_pitch) || (S.pos[2] < P.min_base_height);
  } else {
    gyropod_obs(P, S, o6);
    term = fabsf(o6[1]) > P.fall_pitch;  // strict, upkie_gyropod.py:345
  }
  if (resetting) term = false;

  // Episode time limit (config.max_episode_steps): a uniform branch, no counter traffic without a limit. Every step
  // adds 1 to the env's count elapsed[i]; the step of a next-step auto-reset is not counted: a lane that will reset
  // at the next step leaves 0xffffffff, which that step's +1 turns into 0. The in-kernel transports (TILE=2) do not
  // carry `truncated`: the host rejects a limit there. Same-step mode needs the flag before its reset; the other
  // modes count in a block of their own after the stores of the tick (below).
  const bool timed = TILE != 2 && P.max_episode_steps > 0;
  bool trunc = false;
  uint32_t elapsed = 0;
  if (AUTORESET == AUTORESET_SAME_STEP && timed) {
    elapsed = P.elapsed[i] + 1u;
    trunc = elapsed >= uint32_t(P.max_episode_steps);
  }

  bool fin_pending = false;  // F.sense, same-step reset: the terminal observation is stashed after the tick
  float fin_o6[6], fin_yaw = 0.f, fin_yaw_vel = 0.f;
  if (AUTORESET == AUTORESET_SAME_STEP) {
    if (term || trunc) {
      if constexpr (F.sense) {
        // the terminal step's observation is delayed: it is stashed from the env's sensed row after the tick (below);
        // what the reset overwrites and the stash needs is kept here, the gyropod observation and the wrapper's yaw
        fin_pending = sensing;
        if (MODE != MODE_SERVOS) {  // (UpkieServos rows hold no gyropod observation)
#pragma unroll
          for (int k = 0; k < 6; ++k) fin_o6[k] = o6[k];
        }
        fin_yaw = S.yaw;
        fin_yaw_vel = S.yaw_vel;
      }
      if (!(F.sense && sensing)) {
        if (P.final_obs && live)
          store_final_obs<MODE, spine>(P, S, L, o6, F.extras ? &nz : nullptr, TILE && compact, i, env_col);
        // neither the reset below nor the rest of the tick writes tick[i] (written above, before the physics) or the
        // parameter table, so the stash and those give the rows k_spine_obs would have returned without the reset (a
        // reset randomisation draw overwrites the table at the end of the tick, and the stash then also holds the
        // pre-reset columns k_spine_obs reads, store_final_params)
        if (P.final_state && live) store_final_state<spine>(P, S, L, n_pad, i);
      }
      if (F.reset_rand && P.reset_rand && P.final_state && live) store_final_params<spine>(P, n_pad, i);
      if (pushing) push_restart(push_k, push_t, push_end);  // the terminal step ran under its push; a new schedule
      // the terminal step ran under its delay; the next tick starts from the stop row with a new one
      if (delaying && live) {
        action_delay_reset(*P.action_delay, seed, env_offset + uint64_t(i), i);
        if (HIST) action_delay_fill_history(*P.action_delay, i);
      }
      // the terminal step was observed under its delay; the reset is observed undelayed, with a new draw
      if (sensing && live) obs_delay_reset(*P.obs_delay, seed, env_offset + uint64_t(i), i);
      elapsed = 0;
      const uint32_t ep = episode[i] + 1u;
      if (live) episode[i] = ep;
      float init[UPKIE_INIT_DIM];
      sample_init_state(P, seed, env_offset + uint64_t(i), uint64_t(ep), init);
      if (F.reset_rand && P.reset_rand) {
        reset_rand_lane(P, seed, env_offset + uint64_t(i), i, rr_v, epsv, mu, meas_sd);
        drawn = true;
      }
      const BodyRecOut br{(F.body && P.body_rec && live) ? P.body_rec + i : nullptr,
                          size_t(P.body_rec_stride)};
      if (spine) reset_robot_spine(P, S, L, init, eps, mu, WarpAny(), P.joint_limits, br);
      else reset_robot(P, S, init, eps, mu, WarpAny(), F.limits ? P.joint_limits : 0, br);
      if (MODE != MODE_SERVOS) gyropod_obs(P, S, o6);
    }
  }

  if (live) store_state(state, n_pad, i, S);
  if (sensing) {
    // K > 1: the sensed row becomes the report, and the end of the tick works on it as for one tick
    if (HIST && !resetting && P.obs_delay->ticks > 1) scol = obs_delay_report(*P.obs_delay, srep, i, live);
    if (fin_pending) {
      // the terminal step's sensed state: its snapshot, with the terminal step's wrapper yaw, built in S (the post-reset
      // state is stored, and read back below). sdl = 0: the snapshot is the true state, whose gyropod observation fin_o6
      // already holds (computed again, the pitch could round differently: fast-math contracts the products of another
      // inlined copy differently). Neither the reset nor the rest of the tick writes tick[i] or the parameter table
      // (see the stash above).
      S.yaw = fin_yaw;
      S.yaw_vel = fin_yaw_vel;
      obs_delay_sensed_state(S, sense_load);
      if (MODE != MODE_SERVOS && sdl != 0) gyropod_obs(P, S, fin_o6);
      if (P.final_obs && live)
        store_final_obs<MODE, spine>(P, S, L, fin_o6, F.extras ? &nz : nullptr, TILE && compact, i, env_col);
      if (P.final_state && live) store_final_state<spine>(P, S, L, n_pad, i);
      load_state(state, n_pad, i, S);  // the post-reset state, which this thread stored (plain coherent loads)
    } else if (!resetting) {
      // the row's wrapper fields and contact impulses are the true state's; the observation is built from the snapshot,
      // reloaded into S in place (the true state is stored). sdl = 0: the snapshot is the true state, whose gyropod
      // observation o6 already holds (as above)
      if (live) {
        float r[UPKIE_STATE_DIM];
        state_to_row(S, r);
#pragma unroll
        for (int k = 0; k < UPKIE_STATE_DIM; ++k)
          if (!obs_delay_sensed(k)) sense_store(k, r[k]);
      }
      obs_delay_sensed_state(S, sense_load);
      if (MODE != MODE_SERVOS && sdl != 0) gyropod_obs(P, S, o6);
    }
    if ((resetting || fin_pending) && live) {
      // a reset in this tick: the sensed row becomes a copy of the post-reset state, the observation is undelayed
      float r[UPKIE_STATE_DIM];
      state_to_row(S, r);
#pragma unroll
      for (int k = 0; k < UPKIE_STATE_DIM; ++k) sense_store(k, r[k]);
      if (HIST && P.obs_delay->ticks > 1) obs_delay_fill_history(*P.obs_delay, i, r);  // and so does every snapshot
    }
  }
  if (spine && live) {
    float lr[UPKIE_LAG_DIM];
    lag_to_row(L, lr);
#pragma unroll
    for (int k = 0; k < UPKIE_LAG_DIM; ++k) lag[size_t(k) * n_pad + i] = lr[k];
  }
  // TILE >= 1: every lane is past its last read of its action row before the observation rows overwrite the tile
  if (TILE) __syncwarp();
  if (MODE == MODE_SERVOS) {
    float o[UPKIE_OBS_DIM];
    float tq[6];
    measured_torques(P, S, F.extras ? &nz : nullptr, tq, env_col, meas_sd, F.reset_rand && drawn);
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      o[j * 5 + 0] = S.q[j]; o[j * 5 + 1] = S.qd[j]; o[j * 5 + 2] = tq[j];
      o[j * 5 + 3] = 42.0f;  // pybullet_backend.py:471
      o[j * 5 + 4] = 18.0f;  // pybullet_backend.py:472
    }
    if (spine) {  // the replies of two cycles ago, as the spine's observation reports them
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        o[j * 5 + 0] = L.obs_rep[3 * j]; o[j * 5 + 1] = L.obs_rep[3 * j + 1]; o[j * 5 + 2] = L.obs_rep[3 * j + 2];
        o[j * 5 + 3] = 20.0f;  // BulletInterface.cpp:70
      }
    }
    if (TILE && compact) {
      // compact rows [6 joints][position, velocity, torque]: temperature / voltage are constants the
      // host fills once (pybullet_backend.py:471-472), 72 B per env instead of 120 B over PCIe
      float c[18];
#pragma unroll
      for (int j = 0; j < 6; ++j) { c[3 * j] = o[5 * j]; c[3 * j + 1] = o[5 * j + 1]; c[3 * j + 2] = o[5 * j + 2]; }
      if (full) {
        float2* t2 = reinterpret_cast<float2*>(tile4) + lane * 9;
#pragma unroll
        for (int k = 0; k < 9; ++k) t2[k] = make_float2(c[2 * k], c[2 * k + 1]);
        __syncwarp();
        float4* op = reinterpret_cast<float4*>(obs + size_t(wb) * 18);
#pragma unroll
        for (int k = 0; k < 5; ++k) {
          const int idx = k * 32 + lane;
          if (idx < 32 * 18 / 4) {
            if (TILE == 2 && !peers->deferred) {
              const float4 v = tile4[idx];
              if (peers->n == 0) {
                mc_store4(op + idx, v);
              } else {
                // `obs` is unused here: the row offset of this step's slot is already in every peer pointer
                for (int p = 0; p < peers->n; ++p) reinterpret_cast<float4*>(peers->obs[p] + size_t(wb) * 18)[idx] = v;
              }
            } else {
              op[idx] = tile4[idx];
            }
          }
        }
      } else if (live) {
        float2* op = reinterpret_cast<float2*>(obs + size_t(i) * 18);
#pragma unroll
        for (int k = 0; k < 9; ++k) op[k] = make_float2(c[2 * k], c[2 * k + 1]);
      }
    } else if (TILE && full) {
      float2* t2 = reinterpret_cast<float2*>(tile4) + lane * (UPKIE_OBS_DIM / 2);
#pragma unroll
      for (int k = 0; k < UPKIE_OBS_DIM / 2; ++k) t2[k] = make_float2(o[2 * k], o[2 * k + 1]);
      __syncwarp();
      float4* op = reinterpret_cast<float4*>(obs + size_t(wb) * UPKIE_OBS_DIM);
#pragma unroll
      for (int k = 0; k < (32 * UPKIE_OBS_DIM / 4 + 31) / 32; ++k) {
        const int idx = k * 32 + lane;
        if (idx < 32 * UPKIE_OBS_DIM / 4) op[idx] = tile4[idx];
      }
    } else if (live) {
      float2* op = reinterpret_cast<float2*>(obs + size_t(i) * UPKIE_OBS_DIM);
#pragma unroll
      for (int k = 0; k < UPKIE_OBS_DIM / 2; ++k) op[k] = make_float2(o[2 * k], o[2 * k + 1]);
    }
  } else if (MODE == MODE_GYROPOD) {
    if (TILE && full) {
      float2* t2 = reinterpret_cast<float2*>(tile4) + lane * 3;
      t2[0] = make_float2(o6[0], o6[1]);
      t2[1] = make_float2(o6[2], o6[3]);
      t2[2] = make_float2(o6[4], o6[5]);
      __syncwarp();
      float4* op = reinterpret_cast<float4*>(obs + size_t(wb) * 6);
      op[lane] = tile4[lane];
      if (lane < 16) op[32 + lane] = tile4[32 + lane];
    } else if (live) {
      float2* op = reinterpret_cast<float2*>(obs + size_t(i) * 6);
      op[0] = make_float2(o6[0], o6[1]);
      op[1] = make_float2(o6[2], o6[3]);
      op[2] = make_float2(o6[4], o6[5]);
    }
  } else if (live) {
    // upkie_pendulum.py:17 _PENDULUM_OBS_INDICES = [1, 0, 4, 3]
    reinterpret_cast<float4*>(obs)[i] = make_float4(o6[1], o6[0], o6[4], o6[3]);
  }
  if (TILE == 2) {
    // the host only launches this variant on full, aligned warps (n % 32 == 0): the warp's 32 `terminated` bytes go
    // out as eight words built from the ballot (multimem.st has no byte form)
    const unsigned m = __ballot_sync(0xffffffffu, term);
    if (lane < 8) {
      const unsigned nib = (m >> (4 * lane)) & 0xFu;
      const uint32_t word = (nib & 1u) | ((nib & 2u) << 7) | ((nib & 4u) << 14) | ((nib & 8u) << 21);
      if (peers->deferred) {
        reinterpret_cast<uint32_t*>(terminated + wb)[lane] = word;  // local slot; sent by a later launch's prologue
      } else if (peers->n == 0) {
        mc_store_u32(reinterpret_cast<uint32_t*>(terminated + wb) + lane, word);
      } else {
        for (int p = 0; p < peers->n; ++p) reinterpret_cast<uint32_t*>(peers->term[p] + wb)[lane] = word;
      }
    }
  }
  if (!live) return;
  if (F.reset_rand && drawn) reset_rand_store(*P.reset_rand, i, rr_v);  // after the last read of the lane's row
  if (pushing) {
    P.push->count[i] = push_k;
    P.push->timer[i] = push_t;
  }
  if (reward) reward[i] = 0.0f;  // upkie_env.py:230
  if (TILE != 2) terminated[i] = term ? 1 : 0;
  if (truncated) truncated[i] = trunc ? 1 : 0;
  if (AUTORESET == AUTORESET_SAME_STEP && timed) P.elapsed[i] = elapsed;
  if (e) err[i] |= e;
  if (AUTORESET == AUTORESET_NEXT_STEP) done_prev[i] = term ? 1 : 0;
  if (AUTORESET != AUTORESET_SAME_STEP && timed) {
    uint32_t el = P.elapsed[i] + 1u;
    const bool tr = el >= uint32_t(P.max_episode_steps);
    if (AUTORESET == AUTORESET_NEXT_STEP && (term || tr)) el = 0xffffffffu;  // reset pending: the next step is not counted
    P.elapsed[i] = el;
    if (truncated) truncated[i] = tr ? 1 : 0;
    if (AUTORESET == AUTORESET_NEXT_STEP && tr) done_prev[i] = 1;
  }
}

// Deferred rollout transport: send the warp's 32 compact rows (and `terminated` bytes) of an EARLIER step, read from
// this rank's local slot of that step, to every GPU - NVSwitch multicast store or plain stores into the peers'
// buffers. Called at the top of a tile, before its physics: the stores drain while the warp simulates.
__device__ __forceinline__ void push_rows(const PeerPtrs& pp, int wb, int lane) {
  const float4* src = reinterpret_cast<const float4*>(pp.src_obs + size_t(wb) * 18);
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const int idx = k * 32 + lane;
    if (idx < 32 * 18 / 4) {
      const float4 v = src[idx];
      if (pp.n == 0) {
        mc_store4(reinterpret_cast<float4*>(pp.mc_obs + size_t(wb) * 18) + idx, v);
      } else {
        for (int p = 0; p < pp.n; ++p) reinterpret_cast<float4*>(pp.obs[p] + size_t(wb) * 18)[idx] = v;
      }
    }
  }
  if (lane < 8) {
    const uint32_t word = reinterpret_cast<const uint32_t*>(pp.src_term + wb)[lane];
    if (pp.n == 0) {
      mc_store_u32(reinterpret_cast<uint32_t*>(pp.mc_term + wb) + lane, word);
    } else {
      for (int p = 0; p < pp.n; ++p) reinterpret_cast<uint32_t*>(pp.term[p] + wb)[lane] = word;
    }
  }
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(uint32_t(__cvta_generic_to_shared(smem_dst))),
               "l"(gmem_src)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ---- the env-step kernel ------------------------------------------------------------
// TILE=0 (device buffers): one env per thread, grid = ceil(cnt / block).
// TILE=1 (host buffers, zero-copy): persistent blocks walk the tiles of `blockDim.x` envs with stride
// gridDim.x. The action rows of the NEXT tile are fetched over PCIe with cp.async into the second
// shared-memory buffer while the current tile computes, and observation rows leave through coalesced
// 16 B stores, so the link streams in both directions for the whole launch instead of in bursts
// between compute phases.
template <int MODE, int AUTORESET, int FAMILY, int TILE, bool HIST>
__device__ __forceinline__ void step_tiles(const SimParams& P, int i0, int n, int n_pad, float* __restrict__ state,
       const float* __restrict__ action, float* __restrict__ obs, float* __restrict__ reward,
       uint8_t* __restrict__ terminated, uint8_t* __restrict__ truncated, const float* __restrict__ eps_all,
       const float* __restrict__ mu_all, uint32_t* __restrict__ err, uint8_t* __restrict__ done_prev,
       uint32_t* __restrict__ episode, uint32_t* __restrict__ tick, uint64_t seed, uint64_t env_offset,
       const float* __restrict__ ext, uint32_t ext_local, int coalesce, const PeerPtrs& peers,
       float* __restrict__ lag) {
  // this launch covers the envs [i0, n)
  if (!TILE) {
    step_env<MODE, AUTORESET, FAMILY, 0, HIST>(P, i0 + blockIdx.x * blockDim.x + threadIdx.x, n, n_pad, state, action, obs,
                                         reward, terminated, truncated, eps_all, mu_all, err, done_prev, episode, tick,
                                         seed, env_offset, ext, ext_local, nullptr, false, false, nullptr, lag);
    return;
  }
  extern __shared__ float4 s_tile[];
  constexpr int kRow4 = 32 * UPKIE_ACT_DIM / 4;  // float4 per warp tile
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  // the warp's tile of buffer b, computed from the shared-memory symbol where it is used so that the compiler sees
  // shared-memory accesses (LDS / STS) and not generic ones
  auto buf = [&](int b) { return s_tile + (b * nwarps + warp) * kRow4; };
  const int ntiles = (n - i0 + blockDim.x - 1) / blockDim.x;
  // a warp's rows are prefetched when all 32 envs exist and the rows are 16 B aligned
  auto warp_full = [&](int t) { return (coalesce & 1) && (i0 + t * int(blockDim.x) + warp * 32 + 32 <= n); };
  auto prefetch = [&](int t, float4* dst) {
    if (MODE == MODE_SERVOS && warp_full(t)) {
      const float4* src =
          reinterpret_cast<const float4*>(action + size_t(i0 + t * int(blockDim.x) + warp * 32) * UPKIE_ACT_DIM);
#pragma unroll
      for (int k = 0; k < UPKIE_ACT_DIM / 4; ++k) cp_async16(dst + k * 32 + lane, src + k * 32 + lane);
    }
    cp_async_commit();
  };
  int t = blockIdx.x, it = 0;
  if (t < ntiles) prefetch(t, buf(0));
  for (; t < ntiles; t += gridDim.x, ++it) {
    const int nt = t + gridDim.x;
    if (nt < ntiles) {
      prefetch(nt, buf((it + 1) & 1));
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncwarp();
    if (TILE == 2) {
      if (peers.deferred && peers.src_obs) push_rows(peers, i0 + t * int(blockDim.x) + warp * 32, lane);
    }
    step_env<MODE, AUTORESET, FAMILY, TILE, HIST>(P, i0 + t * blockDim.x + threadIdx.x, n, n_pad, state, action, obs,
                                         reward, terminated, truncated, eps_all, mu_all, err, done_prev, episode, tick,
                                         seed, env_offset, ext, ext_local, buf(it & 1), warp_full(t),
                                         (coalesce & 2) != 0, TILE == 2 ? &peers : nullptr, lag);
    __syncwarp();  // the tile is free again before the next prefetch lands in it
  }
}


template <int MODE, int AUTORESET, int FAMILY, int TILE>
#ifdef UPKIE_MAXNREG
__global__ void __maxnreg__(UPKIE_MAXNREG)
#else
__global__ void __launch_bounds__(UPKIE_MAX_THREADS, UPKIE_MIN_BLOCKS)
#endif
k_step(const __grid_constant__ SimParams P, int i0, int n, int n_pad, float* __restrict__ state,
       const float* __restrict__ action, float* __restrict__ obs, float* __restrict__ reward,
       uint8_t* __restrict__ terminated, uint8_t* __restrict__ truncated, const float* __restrict__ eps_all,
       const float* __restrict__ mu_all, uint32_t* __restrict__ err, uint8_t* __restrict__ done_prev,
       uint32_t* __restrict__ episode, uint32_t* __restrict__ tick, uint64_t seed, uint64_t env_offset,
       const float* __restrict__ ext, uint32_t ext_local, int coalesce, const __grid_constant__ PeerPtrs peers,
       float* __restrict__ lag) {
  step_tiles<MODE, AUTORESET, FAMILY, TILE, false>(P, i0, n, n_pad, state, action, obs, reward, terminated, truncated,
                                                 eps_all, mu_all, err, done_prev, episode, tick, seed, env_offset, ext,
                                                 ext_local, coalesce, peers, lag);
}

// the delay families with a history of more than one tick (StepArgs::history): their own kernels, so that k_step keeps
// the one-tick code
template <int MODE, int AUTORESET, int FAMILY, int TILE>
#ifdef UPKIE_MAXNREG
__global__ void __maxnreg__(UPKIE_MAXNREG)
#else
__global__ void __launch_bounds__(UPKIE_MAX_THREADS, UPKIE_MIN_BLOCKS)
#endif
k_step_hist(const __grid_constant__ SimParams P, int i0, int n, int n_pad, float* __restrict__ state,
       const float* __restrict__ action, float* __restrict__ obs, float* __restrict__ reward,
       uint8_t* __restrict__ terminated, uint8_t* __restrict__ truncated, const float* __restrict__ eps_all,
       const float* __restrict__ mu_all, uint32_t* __restrict__ err, uint8_t* __restrict__ done_prev,
       uint32_t* __restrict__ episode, uint32_t* __restrict__ tick, uint64_t seed, uint64_t env_offset,
       const float* __restrict__ ext, uint32_t ext_local, int coalesce, const __grid_constant__ PeerPtrs peers,
       float* __restrict__ lag) {
  step_tiles<MODE, AUTORESET, FAMILY, TILE, true>(P, i0, n, n_pad, state, action, obs, reward, terminated, truncated,
                                                 eps_all, mu_all, err, done_prev, episode, tick, seed, env_offset, ext,
                                                 ext_local, coalesce, peers, lag);
}

// The shared-memory attributes of a step kernel on the current device: the opt-in above 48 KB of dynamic shared memory,
// and the preferred carveout (a percentage of the maximum; < 0 leaves the choice to the driver). They belong to a
// kernel on a device, so each is set on the first launch of the kernel there and again only when it changes: a
// cudaFuncSetAttribute per launch would be a driver call on every tick.
inline cudaError_t step_kernel_attributes(const void* kernel, int smem, int carveout) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  static std::mutex m;
  static std::map<std::pair<const void*, int>, std::pair<int, int>> set;  // (kernel, device) -> (smem, carveout)
  const std::lock_guard<std::mutex> lock(m);
  const auto key = std::make_pair(kernel, dev);
  const auto it = set.find(key);
  if (it != set.end() && it->second == std::make_pair(smem, carveout)) return cudaSuccess;
  if (smem > 48 * 1024) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e == cudaSuccess && carveout >= 0)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carveout);
  if (e == cudaSuccess) set[key] = std::make_pair(smem, carveout);
  return e;
}

template <int TILE, int MODE, int AUTORESET, int FAMILY>
cudaError_t launch_k_step(const StepArgs& a) {
  const int tiles = (a.cnt + a.block - 1) / a.block;
  const int grid = (TILE && a.grid > 0 && a.grid < tiles) ? a.grid : tiles;
  // One tile buffer per warp when every block steps one tile (grid == tiles: the headline and every launch that is not
  // persistent), two when blocks walk several tiles (the persistent host-buffer launch), for the cp.async prefetch of
  // the next tile. step_tiles touches the second buffer only for a tile t + gridDim.x < ntiles, which exists exactly
  // when grid < tiles. One buffer of a 256-thread block is 36 KB, so the block fits the 64 KB carveout and leaves 192 KB
  // of L1 to the kernel's local-memory frame (DESIGN.md section 4).
  const int nbuf = grid < tiles ? 2 : 1;
  const int smem = TILE ? nbuf * (a.block / 32) * 32 * UPKIE_ACT_DIM * int(sizeof(float)) : 0;
  // the tile path needs 16 B aligned rows of 32 envs
  const int aligned =
      ((reinterpret_cast<uintptr_t>(a.action) | reinterpret_cast<uintptr_t>(a.obs)) & 15) == 0 && (a.i0 % 32) == 0;
  const int coalesce = (aligned ? 1 : 0) | ((TILE && a.compact_obs) ? 2 : 0);  // bit 0 tile path, bit 1 compact rows
  auto kernel = k_step<MODE, AUTORESET, FAMILY, TILE>;
  if constexpr (step_family_traits(FAMILY).delay && TILE != 2) {
    if (a.history) kernel = k_step_hist<MODE, AUTORESET, FAMILY, TILE>;
  }
  // the carveout: a.smem_carveout, by default cudaSharedmemCarveoutMaxL1 (the driver then rounds up only as far as the
  // block's shared memory needs, and the rest of the SM's 256 KB stays L1)
  const cudaError_t e = step_kernel_attributes(reinterpret_cast<const void*>(kernel), smem, a.smem_carveout);
  if (e != cudaSuccess) return e;
  kernel<<<grid, a.block, smem, a.stream>>>(
      *a.P, a.i0, a.i0 + a.cnt, a.n_pad, a.state, a.action, a.obs, a.reward, a.terminated, a.truncated, a.eps, a.mu,
      a.err, a.done_prev, a.episode, a.tick, a.seed, a.env_offset, a.ext, a.ext_local, coalesce, a.peers, a.lag);
  return cudaGetLastError();
}

template <int TILE, int MODE, int FAMILY>
cudaError_t launch_step_mode(const StepArgs& a) {
  if (a.autoreset == AUTORESET_NEXT_STEP) return launch_k_step<TILE, MODE, AUTORESET_NEXT_STEP, FAMILY>(a);
  if (a.autoreset == AUTORESET_SAME_STEP) return launch_k_step<TILE, MODE, AUTORESET_SAME_STEP, FAMILY>(a);
  return launch_k_step<TILE, MODE, AUTORESET_DISABLED, FAMILY>(a);
}

}  // namespace

template <int TILE, int FAMILY>
cudaError_t launch_step(const StepArgs& a) {
  static_assert(bool(UPKIE_BODY_CONTACTS_BUILD) == step_family_traits(FAMILY).body,
                "a unit's UPKIE_BODY_CONTACTS_BUILD is 1 exactly when its families carry body-contact rows");
  // the spine family and the in-kernel transport (TILE=2) are instantiated for UpkieServos only
  if (a.mode == MODE_SERVOS) return launch_step_mode<TILE, MODE_SERVOS, FAMILY>(a);
  if constexpr (TILE == 2 || step_family_traits(FAMILY).spine) {
    return cudaErrorNotSupported;
  } else {
    if (a.mode == MODE_GYROPOD) return launch_step_mode<TILE, MODE_GYROPOD, FAMILY>(a);
    return launch_step_mode<TILE, MODE_PENDULUM, FAMILY>(a);
  }
}

}  // namespace upkie_b200
