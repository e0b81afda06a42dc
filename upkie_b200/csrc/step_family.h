// SPDX-License-Identifier: Apache-2.0
//
// step_family.h -- the kernel families of the env-step kernel k_step<MODE, AUTORESET, FAMILY, TILE> (step_kernel.cuh):
// what each family compiles in, and which family a step launch runs. Every feature that costs the kernels code,
// registers or stack is compiled into the families that need it only, so that the others keep their code; each family
// has translation units of its own (step_unit.cu, DESIGN.md section 4). Compiles with nvcc and with g++ (the CPU test of
// the choice).
#pragma once

#include "sim_core.cuh"

namespace upkie_b200 {

enum { MODE_SERVOS = 0, MODE_GYROPOD = 1, MODE_PENDULUM = 2 };

// The values are part of the kernel symbols: k_stepILi0ELi1ELi2ELi1E is MODE 0, AUTORESET 1, FAMILY 2, TILE 1.
enum {
  FAM_PLAIN = 0,      // nothing optional: no noise, no external forces, no joint-limit rows
  FAM_EXTRAS = 1,     // torque noise models, external forces
  FAM_LIMITS = 2,     // extras + joint-limit rows, no table reads: the headline family
  FAM_SPINE = 3,      // FAM_BODY + the Bullet spine's timing (UpkieServos only)
  FAM_BODY = 4,       // extras + limits + table + reset randomisation + body-ground contact rows
  FAM_TABLE = 5,      // extras + limits + the per-env parameter table + reset randomisation
  FAM_PUSH = 6,       // FAM_TABLE + push randomisation
  FAM_BODY_PUSH = 7,  // FAM_BODY + push randomisation
  FAM_DELAY = 8,      // FAM_PUSH + action delay
  FAM_BODY_DELAY = 9, // FAM_BODY_PUSH + action delay
  FAM_SENSE = 10,     // FAM_DELAY + observation delay + observation history + servo reply dropouts + IMU misalignment
                      // + encoder offsets + servo measurement noise + servo velocity limits + attitude filter
                      // + servo torque scales
  kNumFamilies = 11
};

// What a family's kernels compile in
struct StepFamily {
  bool extras;      // noise context and per-env tick counter, external forces (nz, xf, measured_torques)
  bool limits;      // the device's joint-limit modes 2 / 3 (servo_substep, reset_robot); else mode 0
  bool table;       // per-env parameter table reads (env_col = i); else compiled out (env_col = -1)
  bool reset_rand;  // reset randomisation draws (reset_rand_lane, store_final_params, reset_rand_store)
  bool spine;       // spine timing, UpkieServos: the lag record, spine_cycle
  bool body;        // body-contact record (BodyRecOut); units built with UPKIE_BODY_CONTACTS_BUILD 1
  bool push;        // the push schedule
  bool delay;       // the action delay: previous command rows, per-env delays
  bool sense;       // the observation delay: sensed state rows, per-env delays; the observation history's ring; the
                    // servo dropouts' held rows
};

UPKIE_HD constexpr StepFamily step_family_traits(int family) {
  constexpr StepFamily t[kNumFamilies] = {
      // extras limits table  reset_rand spine  body   push   delay  sense
      {false, false, true, false, false, false, false, false, false},  // FAM_PLAIN
      {true, false, true, false, false, false, false, false, false},   // FAM_EXTRAS
      {true, true, false, false, false, false, false, false, false},   // FAM_LIMITS
      {true, true, true, true, true, true, false, false, false},       // FAM_SPINE
      {true, true, true, true, false, true, false, false, false},      // FAM_BODY
      {true, true, true, true, false, false, false, false, false},     // FAM_TABLE
      {true, true, true, true, false, false, true, false, false},      // FAM_PUSH
      {true, true, true, true, false, true, true, false, false},       // FAM_BODY_PUSH
      {true, true, true, true, false, false, true, true, false},       // FAM_DELAY
      {true, true, true, true, false, true, true, true, false},        // FAM_BODY_DELAY
      {true, true, true, true, false, false, true, true, true},        // FAM_SENSE
  };
  return t[family];
}

// The TILEs of k_step: 0 device buffers, 1 host-buffer tiles, 2 in-kernel rollout transport
constexpr int kNumTiles = 3;

// Whether the library holds the step kernels of (tile, family): every family on TILE 0 and 1, families 0-2 on TILE 2,
// and in the exact-arithmetic library (build.py: build_exact) TILE 0, families 0-2 only. Each pair is instantiated by one
// row of build.py's unit table; the step dispatch (upkie_b200.cu) launches exactly these pairs.
UPKIE_HD constexpr bool step_instantiated(int tile, int family) {
  if (tile < 0 || tile >= kNumTiles || family < 0 || family >= kNumFamilies) return false;
#if UPKIE_EXACT_BUILD
  return tile == 0 && family <= FAM_LIMITS;
#else
  return tile < 2 || family <= FAM_LIMITS;
#endif
}

// The family of a step launch of `mode` on `transport` (the TILE of k_step: 0 device buffers, 1 host-buffer tiles,
// 2 in-kernel rollout transport) for a handle with parameters P (`ext`: external forces set), or -1 with the reason in
// *why when no instantiation serves it. The in-kernel transport has families 0-2 only, and no `truncated`.
inline int step_family(const SimParams& P, bool ext, int mode, int transport, const char** why) {
  const bool in_kernel = transport == 2;
  const char* no = nullptr;
  if (in_kernel && P.env_params)
    no = "the per-env parameter table has no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.push)
    no = "push randomisation has no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.action_delay)
    no = "action delay has no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.obs_delay)
    no = "observation delay has no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.history)
    no = "the observation history has no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.servo_dropout)
    no = "servo dropouts have no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.imu_misalign)
    no = "IMU misalignment has no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.encoder_offset)
    no = "encoder offsets have no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.servo_noise)
    no = "servo noise has no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.velocity_derate)
    no = "velocity limits have no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.attitude_filter)
    no = "the attitude filter has no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.torque_scale)
    no = "torque scales have no in-kernel rollout transport (use upkie_b200_step with compact rows)";
  else if (in_kernel && P.max_episode_steps > 0)
    no = "max_episode_steps has no in-kernel rollout transport: it does not carry truncated (use upkie_b200_step with "
         "compact rows)";
  else if (in_kernel && P.body_contacts)
    no = "body_contacts has no in-kernel rollout transport (use upkie_b200_step_servos_compact)";
  else if (P.spine_mode && mode != MODE_SERVOS)
    no = "spine_mode supports UpkieServos steps only";
  else if (P.spine_mode && in_kernel)
    no = "spine_mode has no in-kernel rollout transport";
  else if (P.obs_delay && P.spine_mode)
    no = "observation delay: spine_mode models the spine's own lag";
  else if (P.obs_delay && P.joint_limits == 0)
    no = "observation delay needs joint_limits != 0";
  else if (P.obs_delay && P.body_contacts)
    no = "observation delay has no body-contact kernels";
  else if (P.history && P.spine_mode)
    no = "observation history: spine_mode reports the spine's lagged replies";
  else if (P.history && P.joint_limits == 0)
    no = "observation history needs joint_limits != 0";
  else if (P.history && P.body_contacts)
    no = "observation history has no body-contact kernels";
  else if (P.servo_dropout && P.spine_mode)
    no = "servo dropouts: spine_mode reports the spine's own servo replies";
  else if (P.servo_dropout && P.joint_limits == 0)
    no = "servo dropouts need joint_limits != 0";
  else if (P.servo_dropout && P.body_contacts)
    no = "servo dropouts have no body-contact kernels";
  else if (P.imu_misalign && P.spine_mode)
    no = "IMU misalignment: spine_mode models its spine's own IMU";
  else if (P.imu_misalign && P.joint_limits == 0)
    no = "IMU misalignment needs joint_limits != 0";
  else if (P.imu_misalign && P.body_contacts)
    no = "IMU misalignment has no body-contact kernels";
  else if (P.encoder_offset && P.spine_mode)
    no = "encoder offsets: spine_mode reports the spine's own servos";
  else if (P.encoder_offset && P.joint_limits == 0)
    no = "encoder offsets need joint_limits != 0";
  else if (P.encoder_offset && P.body_contacts)
    no = "encoder offsets have no body-contact kernels";
  else if (P.servo_noise && P.spine_mode)
    no = "servo noise: spine_mode reports the spine's own servos";
  else if (P.servo_noise && P.joint_limits == 0)
    no = "servo noise needs joint_limits != 0";
  else if (P.servo_noise && P.body_contacts)
    no = "servo noise has no body-contact kernels";
  else if (P.velocity_derate && P.spine_mode)
    no = "velocity limits: spine_mode applies the spine's own torque law";
  else if (P.velocity_derate && P.joint_limits == 0)
    no = "velocity limits need joint_limits != 0";
  else if (P.velocity_derate && P.body_contacts)
    no = "velocity limits have no body-contact kernels";
  else if (P.attitude_filter && P.spine_mode)
    no = "the attitude filter: spine_mode models its spine's own IMU";
  else if (P.attitude_filter && P.joint_limits == 0)
    no = "the attitude filter needs joint_limits != 0";
  else if (P.attitude_filter && P.body_contacts)
    no = "the attitude filter has no body-contact kernels";
  else if (P.torque_scale && P.spine_mode)
    no = "torque scales: spine_mode applies the spine's own torque law";
  else if (P.torque_scale && P.joint_limits == 0)
    no = "torque scales need joint_limits != 0";
  else if (P.torque_scale && P.body_contacts)
    no = "torque scales have no body-contact kernels";
  if (no) {
    *why = no;
    return -1;
  }
  if (P.spine_mode) return FAM_SPINE;
  // the observation-delay family carries the action delay and the pushes too (runtime-uniform branches on
  // P.action_delay and P.push), the observation history (P.history), the servo dropouts (P.servo_dropout), the IMU
  // misalignment (P.imu_misalign), the encoder offsets (P.encoder_offset), the servo noise (P.servo_noise) and the
  // servo velocity limits (P.velocity_derate), the attitude filter (P.attitude_filter) and the torque scales
  // (P.torque_scale), by the same rule; the set calls reject spine mode, no limits and body contacts
  if (P.obs_delay || P.history || P.servo_dropout || P.imu_misalign || P.encoder_offset || P.servo_noise ||
      P.velocity_derate || P.attitude_filter || P.torque_scale)
    return FAM_SENSE;
  // the delay families carry the pushes too (a runtime-uniform branch on P.push); the set calls reject spine mode and
  // no limits
  if (P.action_delay) return P.body_contacts ? FAM_BODY_DELAY : FAM_DELAY;
  if (P.push) return P.body_contacts ? FAM_BODY_PUSH : FAM_PUSH;  // the set call rejects spine mode and no limits
  if (P.body_contacts) return FAM_BODY;  // the model's collision points hold contact rows
  if (P.joint_limits) return P.env_params ? FAM_TABLE : FAM_LIMITS;
  return (P.any_ctrl_noise || P.any_meas_noise || ext) ? FAM_EXTRAS : FAM_PLAIN;
}

}  // namespace upkie_b200
