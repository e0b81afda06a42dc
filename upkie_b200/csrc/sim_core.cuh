// SPDX-License-Identifier: Apache-2.0
//
// sim_core.cuh -- per-robot simulation arithmetic of the sm_90a kernels.
//
// One CUDA thread advances one robot (lane = robot): the path is bound by fp32
// issue rate, not by HBM (DESIGN.md "Roofline"), so the layout keeps all 32
// lanes of a warp busy with independent robots, state arrays are
// struct-of-arrays for coalesced loads, and the model lives in the kernel
// parameter constant bank (uniform operands, no register or LDS cost).
//
// Formulation (different from the oracle's on purpose): every spatial quantity
// of the 7-body tree is expressed in ONE frame, the base frame at the current
// instant, so parent/child propagation needs no Pluecker transforms; the legs
// are planar chains about the base y-axis (all Upkie joint axes are +-y), which
// makes every motion subspace S = s * [0 1 0 | -oz 0 ox] with three non-zeros.
//
// What it replaces, per env-step (reference file:line):
//   UpkieServos.get_spine_action clamps        upkie/envs/upkie_servos.py:316-344
//   PyBulletBackend.step substep loop          upkie/envs/backends/pybullet_backend.py:269-311
//   compute_joint_torque (moteus law)          pybullet_backend.py:492-553
//   pybullet.stepSimulation (Bullet, 3rd-party) pybullet_backend.py:306
//   get_spine_observation                      pybullet_backend.py:313-490
//   UpkieGyropod / UpkiePendulum front-end      upkie/envs/upkie_gyropod.py:246-392, upkie_pendulum.py:124-142
#pragma once

#include <math.h>
#include <stdint.h>

#include "../../include/upkie_b200.h"

#if defined(__CUDACC__)
#define UPKIE_HD __host__ __device__ __forceinline__
#else
#define UPKIE_HD inline
#endif

namespace upkie_b200 {

#ifndef UPKIE_PAIRED_LEGS
#define UPKIE_PAIRED_LEGS 1  // left/right leg arithmetic on (left, right) pairs (sim_pair.cuh)
#endif

// (left leg, right leg) pair; maps onto one 64-bit register pair
struct alignas(8) f2 {
  float x, y;
};

// ---- kernel parameters (constant bank) ----------------------------------------
struct SimParams {
  // model (upkie.model.Model + URDF inertials)
  float sgn[6];            // joint axis = sgn * y
  float jo[6][3];          // joint origin in parent body frame
  float mass[7];
  float com[7][3];
  float inertia[7][6];     // xx yy zz xy xz yz about the CoM
  float q_lower[6], q_upper[6], qd_max[6], tau_max[6];
  float wheel_radius;
  float half_wheel_base;
  float left_sign;         // +1 left-wheeled
  float imu_pos[3];
  float Rbi[9];            // rotation_base_to_imu
  int wheel_symmetric;     // wheel CoM on its axis and inertia axisymmetric: skip wheel-angle trig
  // the per-leg constants again as (left, right) pairs, k = hip, knee, wheel (64-bit constant operands)
  f2 sgn2[3];
  f2 jo2[3][3];
  f2 oy2[3];               // y of the body origin (sum of joint-origin y's down the chain)
  f2 mass2[3];
  f2 com2[3][3];
  f2 inertia2[3][6];
  // backend
  float dt, inv_dt, h, inv_h;
  int nb_substeps, pgs_iterations;
  float res_thr;           // Bullet's m_leastSquaresResidualThreshold: a robot's solve ends once the largest squared
                           // velocity-level row change of a sweep is at or below it (0 = all sweeps)
  float warm;              // warm-starting factor of the normal contact impulses (Bullet: 0.85)
  int skip_action_clamps;
  float gravity, kp, kd;
  float joint_friction[6];
  float ctrl_noise[6], meas_noise[6];  // JointProperties noise standard deviations
  int any_ctrl_noise, any_meas_noise;
  float imu_acc_bias[3], imu_gyro_bias[3], imu_acc_noise, imu_gyro_noise;  // ImuUncertainty.h:29-69
  int any_imu_uncertainty;
  uint64_t noise_seed;
  float lin_damp, ang_damp, vmax;
  float cfm, erp;          // from contact stiffness/damping and h (Bullet formulas)
  float breaking_threshold;
  float friction;
  // envs
  float max_gain_scale, fall_pitch, leg_gain_scale, max_ground_velocity, max_yaw_velocity;
  int servos_fall_termination;
  float min_base_height;
  // init-state sampling (RobotStateRandomization)
  float init_pos[3], init_quat[4];
  float rand_roll, rand_pitch, rand_x, rand_z, rand_omega_x, rand_omega_y, rand_linvel[3];
  // joint-limit rows (btMultiBodyJointLimitConstraint; "extras" instantiations only). Kept at the end of the
  // struct so that the constant-bank offsets of everything above stay where the GPU-validated kernels read them.
  int joint_limits;        // 0 off, 1 scalar slow path, 2 packed ten-row solver (sim_pair.cuh)
  float limit_erp, limit_max_impulse;
  // nominal joint configuration / base velocities of the initial state (RobotState.sample_state keeps / adds them)
  float init_q[6], init_angvel[3], init_linvel[3];
  int spine_mode;  // 1: timing of the C++ Bullet spine in simulate() mode (include/upkie_b200.h: spine_mode)
  // body-ground contacts (config.body_contacts; the families with the body trait). Collision points of the model:
  int body_contacts;       // 1: on AND the model has collision points
  int n_bp;
  int bp_body[UPKIE_MAX_COLLISION_POINTS];
  float bp_pos[UPKIE_MAX_COLLISION_POINTS][3];
  float bp_radius[UPKIE_MAX_COLLISION_POINTS];
  // the per-substep gate of the packed solvers (sim_pair.cuh body_points_near_ground): base-body points exactly
  // (x, y, z, radius), leg bodies through the height of the body origin minus a bound on |point| + radius
  int n_gate_base;
  float gate_base[UPKIE_MAX_COLLISION_POINTS][4];
  f2 gate_leg_bound[3];    // (left, right) per level hip / knee / wheel body; -1e30 = no collision point on that body
  float body_erp, body_mu_scale;
  // device buffer [UPKIE_BODY_REC_DIM][body_rec_stride] the step kernels write the body contacts of a tick's last
  // substep to (upkie_b200_get_body_contacts); null in the host build and when the handle has no body contacts
  float* body_rec;
  int body_rec_stride;
  // episode time limit (config.max_episode_steps, 0 = none): elapsed[n] counts each env's agent steps since its last
  // reset (the handle's buffer; null in the host build), final_obs receives the rows of the same-step auto-resets'
  // terminal observations (set per launch, null = not requested)
  int max_episode_steps;
  uint32_t* elapsed;
  float* final_obs;
  // per-env parameter table (upkie_b200_set_env_params): [UPKIE_EP_DIM][env_params_stride], env i in column i; null =
  // every env runs the values above (kp, kd, joint_friction, ctrl_noise, meas_noise, imu_*). While a table is set the
  // any_* flags above say whether SOME env of the table has that noise.
  const float* env_params;
  int env_params_stride;
  // same-step auto-reset, terminal spine observation (UpkieStepOutputs.final_state; set per launch, null = not
  // requested): a resetting env stashes its pre-reset state in the handle's buffer final_state (rows kFinal* of
  // kernel_common.cuh, n_pad floats each) and marks its column with final_gen, the number of the step.
  // Appended after every other field, so that their offsets stay where the kernels read them.
  uint32_t final_gen;
  float* final_state;
  // reset randomisation (upkie_b200_set_reset_randomization): the handle's device block, null = off. Read by the
  // step kernels of the reset_rand families (step_family.h) and k_reset only. Appended last, as final_state above.
  const struct ResetRand* reset_rand;
  // push randomisation (upkie_b200_set_push_randomization): the handle's device block, null = off. Read by the
  // step kernels of the push families (step_family.h) only. Appended last, as reset_rand above.
  const struct PushRand* push;
  // action-delay randomisation (upkie_b200_set_action_delay): the handle's device block, null = off. Read by the step
  // kernels of the delay families (step_family.h) only. Appended last, as push above.
  const struct ActionDelay* action_delay;
  // observation-delay randomisation (upkie_b200_set_observation_delay): the handle's device block, null = off. Read by
  // the step kernels of FAM_SENSE (step_family.h) only. Appended last, as action_delay above.
  const struct ObsDelay* obs_delay;
  // spine-rate observation history (upkie_b200_set_history): the handle's device block, null = off. Read by the step
  // kernels of FAM_SENSE (step_family.h) and k_reset only. Appended last, as obs_delay above.
  const struct History* history;
  // servo reply dropouts (upkie_b200_set_servo_dropout): the handle's device block, null = off. Read by the step kernels
  // of FAM_SENSE (step_family.h), k_reset, k_spine_obs and k_reset_obs only. Appended last, as history above.
  const struct ServoDropout* servo_dropout;
  // IMU mounting misalignment (upkie_b200_set_imu_misalignment): the handle's device block, null = off. Read by the step
  // kernels of FAM_SENSE (step_family.h), k_reset, k_spine_obs, k_reset_obs and k_history_fill only. Appended last.
  const struct ImuMisalign* imu_misalign;
  // servo encoder zero offsets (upkie_b200_set_encoder_offset): the handle's device block, null = off. Read by the step
  // kernels of FAM_SENSE (step_family.h), k_reset, k_spine_obs, k_reset_obs and k_history_fill only. Appended last.
  const struct EncoderOffset* encoder_offset;
  // servo measurement noise (upkie_b200_set_servo_noise): the handle's device block, null = off. Read by the step kernels
  // of FAM_SENSE (step_family.h), k_reset, k_spine_obs, k_reset_obs and k_history_fill only. Appended last.
  const struct ServoNoise* servo_noise;
  // servo velocity limits (upkie_b200_set_velocity_derate): the handle's device block, null = off. Read by the step
  // kernels of FAM_SENSE (step_family.h) and k_reset only. Appended last.
  const struct VelocityDerate* velocity_derate;
  // IMU attitude estimation (upkie_b200_set_attitude_filter): the handle's device block, null = off. Read by the step
  // kernels of FAM_SENSE (step_family.h), k_reset, k_spine_obs, k_reset_obs, k_history_fill and k_attitude_init only.
  // Appended last.
  const struct AttitudeFilter* attitude_filter;
  // servo torque-constant errors (upkie_b200_set_torque_scale): the handle's device block, null = off. Read by the step
  // kernels of FAM_SENSE (step_family.h) and k_reset only. Appended last.
  const struct TorqueScale* torque_scale;
};

// Column k of env i's row of the per-env parameter table (read where it is used, through the read-only cache: the
// table stays in L2 next to the state)
UPKIE_HD float env_param(const SimParams& P, int i, int k) {
#if defined(__CUDA_ARCH__)
  return __ldg(P.env_params + size_t(k) * size_t(P.env_params_stride) + size_t(i));
#else
  return P.env_params[size_t(k) * size_t(P.env_params_stride) + size_t(i)];
#endif
}

// per-robot state in registers
struct RobotState {
  float pos[3], quat[4], linvel[3], angvel[3];
  float q[6], qd[6];
  float prev_imu_vel[3];
  float torque[6];
  float leg_target[4];
  float yaw, yaw_vel;
  float contact;
  float imu_acc[3];  // world-frame IMU acceleration of the last observation
  float lam_n[2];    // normal contact impulses of the last substep (warm start)
  float lam_t[4];    // friction impulses of the last substep: (rolling, lateral) of the left wheel, of the right wheel
};

// packed upper-triangular index of a symmetric 6x6
UPKIE_HD constexpr int SI(int i, int j) { return i <= j ? (i * (11 - i)) / 2 + j : (j * (11 - j)) / 2 + i; }

struct LegCache {
  float ox[3], oz[3];  // body origins (x, z) in base coordinates
  float U[3][6];
  float invD[3];
};

UPKIE_HD float clampf(float v, float lo, float hi) { return fminf(fmaxf(v, lo), hi); }

// clamp of upkie/utils/clamp.py:15-30: NaN passes through
UPKIE_HD float clamp_ref(float v, float lo, float hi) {
  if (v < lo) return lo;
  if (v > hi) return hi;
  return v;
}

UPKIE_HD void quat_to_rot(const float q[4], float R[9]) {
  // upkie/utils/rotations.py:36-71
  const float qw = q[0], qx = q[1], qy = q[2], qz = q[3];
  R[0] = 1.f - 2.f * (qy * qy + qz * qz);
  R[1] = 2.f * (qx * qy - qz * qw);
  R[2] = 2.f * (qw * qy + qx * qz);
  R[3] = 2.f * (qx * qy + qz * qw);
  R[4] = 1.f - 2.f * (qx * qx + qz * qz);
  R[5] = 2.f * (qy * qz - qx * qw);
  R[6] = 2.f * (qx * qz - qy * qw);
  R[7] = 2.f * (qy * qz + qx * qw);
  R[8] = 1.f - 2.f * (qx * qx + qy * qy);
}

// y = R x, y = R^T x
UPKIE_HD void rot_mul(const float R[9], const float x[3], float y[3]) {
  y[0] = R[0] * x[0] + R[1] * x[1] + R[2] * x[2];
  y[1] = R[3] * x[0] + R[4] * x[1] + R[5] * x[2];
  y[2] = R[6] * x[0] + R[7] * x[1] + R[8] * x[2];
}
UPKIE_HD void rot_tmul(const float R[9], const float x[3], float y[3]) {
  y[0] = R[0] * x[0] + R[3] * x[1] + R[6] * x[2];
  y[1] = R[1] * x[0] + R[4] * x[1] + R[7] * x[2];
  y[2] = R[2] * x[0] + R[5] * x[1] + R[8] * x[2];
}
UPKIE_HD void cross3(const float a[3], const float b[3], float c[3]) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// S^T x for S = s * [0 1 0 | -oz 0 ox]
UPKIE_HD float sdot(float s, float ox, float oz, const float x[6]) { return s * (x[1] - oz * x[3] + ox * x[5]); }

// LDL^T of a symmetric positive definite 6x6 (packed upper triangle, in place):
// on exit A[SI(i,i)] = 1/d_i and A[SI(j,i)] (j < i) = L_ij.
UPKIE_HD void ldl6(float A[21]) {
  float d[6];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    float dj = A[SI(j, j)];
#pragma unroll
    for (int k = 0; k < j; ++k) dj -= A[SI(k, j)] * A[SI(k, j)] * d[k];
    d[j] = dj;
    const float invd = 1.f / dj;
    A[SI(j, j)] = invd;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      float v = A[SI(j, i)];
#pragma unroll
      for (int k = 0; k < j; ++k) v -= A[SI(k, i)] * A[SI(k, j)] * d[k];
      A[SI(j, i)] = v * invd;
    }
  }
}

// x <- A^-1 x with the factors of ldl6
UPKIE_HD void ldl6_solve(const float A[21], float x[6]) {
#pragma unroll
  for (int i = 1; i < 6; ++i) {
#pragma unroll
    for (int k = 0; k < i; ++k) x[i] -= A[SI(k, i)] * x[k];
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) x[i] *= A[SI(i, i)];
#pragma unroll
  for (int i = 4; i >= 0; --i) {
#pragma unroll
    for (int k = i + 1; k < 6; ++k) x[i] -= A[SI(i, k)] * x[k];
  }
}

// ---- one leg of the articulated-body algorithm -----------------------------------
// Forward kinematics + velocities down the leg, then articulated inertias and
// bias forces back up to the hip. Adds the hip's reduced articulated inertia
// and bias force into the base accumulators IA0 / pA0, keeps (U, 1/D, origins)
// in `lc` and (c, u) in cc/uu for the acceleration pass.
template <int LEG>
UPKIE_HD void leg_pass12(const SimParams& P, const float q[6], const float qd[6], const float tau[6],
                         const float V0[6], const float* eps, LegCache& lc, float cc[3][6], float uu[3],
                         float IA0[21], float pA0[6]) {
  constexpr int J0 = 3 * LEG;
  float cphi[3], sphi[3];
  float V[3][6];
  {
    float phi = 0.f, cp = 1.f, sp = 0.f;
    float ox = 0.f, oz = 0.f;
    float Vc[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) Vc[i] = V0[i];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int j = J0 + k;
      const float s = P.sgn[j];
      // origin of body k: parent origin + Ry(phi_parent) * joint origin
      ox += cp * P.jo[j][0] + sp * P.jo[j][2];
      oz += -sp * P.jo[j][0] + cp * P.jo[j][2];
      lc.ox[k] = ox;
      lc.oz[k] = oz;
      phi += s * q[j];
      if (k < 2 || !P.wheel_symmetric) {
        // explicit range reduction: the fast-math sincos of the device build is only accurate on [-pi, pi]
        const float red = phi - 6.28318530718f * rintf(phi * 0.15915494309f);
        sincosf(red, &sp, &cp);
      }
      cphi[k] = cp;
      sphi[k] = sp;
      const float w = s * qd[j];
      Vc[1] += w;
      Vc[3] -= oz * w;
      Vc[5] += ox * w;
#pragma unroll
      for (int i = 0; i < 6; ++i) V[k][i] = Vc[i];
    }
  }
  float IA[21], pA[6];
#pragma unroll
  for (int k = 2; k >= 0; --k) {
    const int j = J0 + k;
    const int b = j + 1;
    const float s = P.sgn[j];
    const float ox = lc.ox[k], oz = lc.oz[k];
    const float scale = eps ? 1.f + eps[j] : 1.f;
    const float m = P.mass[b] * scale;
    // CoM and rotated inertia in base coordinates
    float C[3], Ib[6];
    if (k == 2 && P.wheel_symmetric) {
      C[0] = ox; C[1] = 0.f; C[2] = oz;  // y of the origin is irrelevant below only through C[1]
      Ib[0] = P.inertia[b][0] * scale; Ib[1] = P.inertia[b][1] * scale; Ib[2] = P.inertia[b][2] * scale;
      Ib[3] = 0.f; Ib[4] = 0.f; Ib[5] = 0.f;
    } else {
      const float c = cphi[k], sn = sphi[k];
      C[0] = ox + c * P.com[b][0] + sn * P.com[b][2];
      C[1] = P.com[b][1];
      C[2] = oz - sn * P.com[b][0] + c * P.com[b][2];
      const float a = P.inertia[b][0] * scale, bb = P.inertia[b][1] * scale, cz = P.inertia[b][2] * scale;
      const float d = P.inertia[b][3] * scale, e = P.inertia[b][4] * scale, f = P.inertia[b][5] * scale;
      Ib[0] = c * c * a + 2.f * c * sn * e + sn * sn * cz;
      Ib[1] = bb;
      Ib[2] = sn * sn * a - 2.f * c * sn * e + c * c * cz;
      Ib[3] = c * d + sn * f;
      Ib[4] = c * sn * (cz - a) + (c * c - sn * sn) * e;
      Ib[5] = -sn * d + c * f;
    }
    // the y coordinate of the body origin: sum of joint-origin y's down the chain
    {
      float oy = 0.f;
#pragma unroll
      for (int kk = 0; kk <= k; ++kk) oy += P.jo[J0 + kk][1];
      C[1] += oy;
    }
    // spatial inertia about the base origin
    float I[21];
    {
      const float cc2 = C[0] * C[0] + C[1] * C[1] + C[2] * C[2];
      I[SI(0, 0)] = Ib[0] + m * (cc2 - C[0] * C[0]);
      I[SI(1, 1)] = Ib[1] + m * (cc2 - C[1] * C[1]);
      I[SI(2, 2)] = Ib[2] + m * (cc2 - C[2] * C[2]);
      I[SI(0, 1)] = Ib[3] - m * C[0] * C[1];
      I[SI(0, 2)] = Ib[4] - m * C[0] * C[2];
      I[SI(1, 2)] = Ib[5] - m * C[1] * C[2];
      const float hx = m * C[0], hy = m * C[1], hz = m * C[2];
      I[SI(0, 3)] = 0.f; I[SI(0, 4)] = -hz; I[SI(0, 5)] = hy;
      I[SI(1, 3)] = hz;  I[SI(1, 4)] = 0.f; I[SI(1, 5)] = -hx;
      I[SI(2, 3)] = -hy; I[SI(2, 4)] = hx;  I[SI(2, 5)] = 0.f;
      I[SI(3, 3)] = m; I[SI(4, 4)] = m; I[SI(5, 5)] = m;
      I[SI(3, 4)] = 0.f; I[SI(3, 5)] = 0.f; I[SI(4, 5)] = 0.f;
    }
    // momentum, bias force p = V x* (I V) - damping wrench
    float p[6];
    float spin_damp = 0.f;  // damping moment about the body's own y axis (closed-form wheel leaf below)
    {
      const float* om = &V[k][0];
      const float* v = &V[k][3];
      float vC[3], t[3];
      cross3(om, C, t);
      vC[0] = v[0] + t[0]; vC[1] = v[1] + t[1]; vC[2] = v[2] + t[2];
      float f[3] = {m * vC[0], m * vC[1], m * vC[2]};
      float nC[3] = {Ib[0] * om[0] + Ib[3] * om[1] + Ib[4] * om[2], Ib[3] * om[0] + Ib[1] * om[1] + Ib[5] * om[2],
                     Ib[4] * om[0] + Ib[5] * om[1] + Ib[2] * om[2]};
      float n[3];
      cross3(C, f, n);
      n[0] += nC[0]; n[1] += nC[1]; n[2] += nC[2];
      float a1[3], a2[3], a3[3];
      cross3(om, n, a1);
      cross3(v, f, a2);
      cross3(om, f, a3);
      // Bullet-style damping: F = -m vC (k + k|vC|), N = -Ic om (k + k|om|)
      const float gl = P.lin_damp * (1.f + sqrtf(vC[0] * vC[0] + vC[1] * vC[1] + vC[2] * vC[2]));
      const float ga = P.ang_damp * (1.f + sqrtf(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]));
      float F[3] = {f[0] * gl, f[1] * gl, f[2] * gl};  // = -damping force
      float cF[3];
      cross3(C, F, cF);
      p[0] = a1[0] + a2[0] + nC[0] * ga + cF[0];
      p[1] = a1[1] + a2[1] + nC[1] * ga + cF[1];
      p[2] = a1[2] + a2[2] + nC[2] * ga + cF[2];
      p[3] = a3[0] + F[0];
      p[4] = a3[1] + F[1];
      p[5] = a3[2] + F[2];
      spin_damp = nC[1] * ga;
    }
    if (k == 2) {
#pragma unroll
      for (int i = 0; i < 21; ++i) IA[i] = I[i];
#pragma unroll
      for (int i = 0; i < 6; ++i) pA[i] = p[i];
    } else {
#pragma unroll
      for (int i = 0; i < 21; ++i) IA[i] += I[i];
#pragma unroll
      for (int i = 0; i < 6; ++i) pA[i] += p[i];
    }
    // velocity-product acceleration c = V x (S qd)
    {
      const float w = s * qd[j];
      const float* om = &V[k][0];
      const float* v = &V[k][3];
      cc[k][0] = -om[2] * w;
      cc[k][1] = 0.f;
      cc[k][2] = om[0] * w;
      cc[k][3] = (om[1] * ox - v[2]) * w;
      cc[k][4] = -(om[2] * oz + om[0] * ox) * w;
      cc[k][5] = (om[1] * oz + v[0]) * w;
    }
    // U = IA S, D = S^T U, u = tau - S^T pA
    float U[6], invD, u;
    if (k == 2 && P.wheel_symmetric) {
      // closed-form leaf (see legs_pass12 in sim_pair.cuh): U = (0, s Iyy, 0 | 0), D = Iyy, S^T pA = s * damping_y
      const float Iyy = Ib[1];
#pragma unroll
      for (int r = 0; r < 6; ++r) U[r] = 0.f;
      U[1] = s * Iyy;
      invD = 1.f / Iyy;
      u = tau[j] - s * spin_damp;
      IA[SI(1, 1)] -= Iyy;
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        float acc = pA[r];
#pragma unroll
        for (int c2 = 0; c2 < 6; ++c2) {
          if (c2 != 1) acc += IA[SI(r, c2)] * cc[k][c2];
        }
        p[r] = acc;
      }
      p[1] += s * u;
    } else {
#pragma unroll
      for (int r = 0; r < 6; ++r) U[r] = s * (IA[SI(r, 1)] - oz * IA[SI(r, 3)] + ox * IA[SI(r, 5)]);
      const float D = sdot(s, ox, oz, U);
      invD = 1.f / D;
      u = tau[j] - sdot(s, ox, oz, pA);
      // Ia = IA - U U^T / D ; pa = pA + Ia c + U u / D
      float Ud[6];
#pragma unroll
      for (int r = 0; r < 6; ++r) Ud[r] = U[r] * invD;
#pragma unroll
      for (int r = 0; r < 6; ++r) {
#pragma unroll
        for (int c2 = r; c2 < 6; ++c2) IA[SI(r, c2)] -= Ud[r] * U[c2];
      }
      const float ud = u * invD;
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        float acc = pA[r] + U[r] * ud;
#pragma unroll
        for (int c2 = 0; c2 < 6; ++c2) acc += IA[SI(r, c2)] * cc[k][c2];
        p[r] = acc;
      }
    }
#pragma unroll
    for (int r = 0; r < 6; ++r) lc.U[k][r] = U[r];
    lc.invD[k] = invD;
    uu[k] = u;
#pragma unroll
    for (int r = 0; r < 6; ++r) pA[r] = p[r];
  }
#pragma unroll
  for (int i = 0; i < 21; ++i) IA0[i] += IA[i];
#pragma unroll
  for (int i = 0; i < 6; ++i) pA0[i] += pA[i];
}

// base body spatial inertia about its origin + bias force
UPKIE_HD void base_inertia_bias(const SimParams& P, const float V0[6], float IA0[21], float pA0[6]) {
  const float m = P.mass[0];
  const float C[3] = {P.com[0][0], P.com[0][1], P.com[0][2]};
  const float* Ib = P.inertia[0];
  const float cc2 = C[0] * C[0] + C[1] * C[1] + C[2] * C[2];
  IA0[SI(0, 0)] = Ib[0] + m * (cc2 - C[0] * C[0]);
  IA0[SI(1, 1)] = Ib[1] + m * (cc2 - C[1] * C[1]);
  IA0[SI(2, 2)] = Ib[2] + m * (cc2 - C[2] * C[2]);
  IA0[SI(0, 1)] = Ib[3] - m * C[0] * C[1];
  IA0[SI(0, 2)] = Ib[4] - m * C[0] * C[2];
  IA0[SI(1, 2)] = Ib[5] - m * C[1] * C[2];
  const float hx = m * C[0], hy = m * C[1], hz = m * C[2];
  IA0[SI(0, 3)] = 0.f; IA0[SI(0, 4)] = -hz; IA0[SI(0, 5)] = hy;
  IA0[SI(1, 3)] = hz;  IA0[SI(1, 4)] = 0.f; IA0[SI(1, 5)] = -hx;
  IA0[SI(2, 3)] = -hy; IA0[SI(2, 4)] = hx;  IA0[SI(2, 5)] = 0.f;
  IA0[SI(3, 3)] = m; IA0[SI(4, 4)] = m; IA0[SI(5, 5)] = m;
  IA0[SI(3, 4)] = 0.f; IA0[SI(3, 5)] = 0.f; IA0[SI(4, 5)] = 0.f;
  const float* om = &V0[0];
  const float* v = &V0[3];
  float vC[3], t[3];
  cross3(om, C, t);
  vC[0] = v[0] + t[0]; vC[1] = v[1] + t[1]; vC[2] = v[2] + t[2];
  float f[3] = {m * vC[0], m * vC[1], m * vC[2]};
  float nC[3] = {Ib[0] * om[0] + Ib[3] * om[1] + Ib[4] * om[2], Ib[3] * om[0] + Ib[1] * om[1] + Ib[5] * om[2],
                 Ib[4] * om[0] + Ib[5] * om[1] + Ib[2] * om[2]};
  float n[3];
  cross3(C, f, n);
  n[0] += nC[0]; n[1] += nC[1]; n[2] += nC[2];
  float a1[3], a2[3], a3[3];
  cross3(om, n, a1);
  cross3(v, f, a2);
  cross3(om, f, a3);
  const float gl = P.lin_damp * (1.f + sqrtf(vC[0] * vC[0] + vC[1] * vC[1] + vC[2] * vC[2]));
  const float ga = P.ang_damp * (1.f + sqrtf(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]));
  float F[3] = {f[0] * gl, f[1] * gl, f[2] * gl};
  float cF[3];
  cross3(C, F, cF);
  pA0[0] = a1[0] + a2[0] + nC[0] * ga + cF[0];
  pA0[1] = a1[1] + a2[1] + nC[1] * ga + cF[1];
  pA0[2] = a1[2] + a2[2] + nC[2] * ga + cF[2];
  pA0[3] = a3[0] + F[0];
  pA0[4] = a3[1] + F[1];
  pA0[5] = a3[2] + F[2];
}

// joint accelerations down one leg given the base acceleration
template <int LEG>
UPKIE_HD void leg_pass3(const SimParams& P, const LegCache& lc, const float cc[3][6], const float uu[3],
                        const float a0[6], float qdd[6]) {
  float a[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) a[i] = a0[i];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int j = 3 * LEG + k;
    const float s = P.sgn[j];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      a[i] += cc[k][i];
      dot += lc.U[k][i] * a[i];
    }
    const float dd = (uu[k] - dot) * lc.invD[k];
    qdd[j] = dd;
    const float w = s * dd;
    a[1] += w;
    a[3] -= lc.oz[k] * w;
    a[5] += lc.ox[k] * w;
  }
}

// Propagate a spatial impulse applied on the wheel of one leg up to the base:
// returns the per-joint u's and adds the residual to p0.
UPKIE_HD void leg_impulse_up(const SimParams& P, int J0, const LegCache& lc, const float f[6], float uu[3], float p0[6]) {
  float p[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) p[i] = -f[i];
#pragma unroll
  for (int k = 2; k >= 0; --k) {
    const float s = P.sgn[J0 + k];
    const float u = -sdot(s, lc.ox[k], lc.oz[k], p);
    uu[k] = u;
    const float ud = u * lc.invD[k];
#pragma unroll
    for (int i = 0; i < 6; ++i) p[i] += lc.U[k][i] * ud;
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) p0[i] += p[i];
}

// velocity changes down one leg given the base velocity change; returns the
// wheel body's spatial velocity change in aw and the joint velocity changes.
UPKIE_HD void leg_impulse_down(const SimParams& P, int J0, const LegCache& lc, const float uu[3], const float a0[6],
                               float aw[6], float dqd[3]) {
#pragma unroll
  for (int i = 0; i < 6; ++i) aw[i] = a0[i];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float s = P.sgn[J0 + k];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < 6; ++i) dot += lc.U[k][i] * aw[i];
    const float dd = (uu[k] - dot) * lc.invD[k];
    dqd[k] = dd;
    const float w = s * dd;
    aw[1] += w;
    aw[3] -= lc.oz[k] * w;
    aw[5] += lc.ox[k] * w;
  }
}

// ---- one physics substep ------------------------------------------------------
// Restates one pybullet.stepSimulation() (pybullet_backend.py:306): collision
// detection at the current configuration, ABA velocity update, PGS contact
// solve on velocities, semi-implicit position integration. `any_contact_hint`
// lets a warp skip the contact solve when no lane touches the ground.
// `phase_sync` is called exactly kPhaseSyncs times per substep by every lane,
// whatever its path: on the device it is a CTA-wide barrier that keeps the
// block's warps on the same stretch of this (instruction-cache-sized) code.
struct NoSync {
  UPKIE_HD void operator()() const {}
};
constexpr int kPhaseSyncs = 6;

// Projected Gauss-Seidel over the six contact rows in Bullet's order (nL nR t1L t2L t1R t2R), residual form:
// r_k = rhs_k + sum_l G_kl lam_l is kept up to date for every row, so a row update is clamp(r_k) and the change
// delta = lam_k' - lam_k is pushed into all six residuals with independent FMAs (r_m += G_mk delta). Same
// iterates as the textbook sweep that re-sums each row, but the dependent chain per row is clamp -> delta -> one
// FMA instead of a six-term sum (the solver is latency-bound), and the six updates pair into three fma2 calls in the
// paired build (sim_pair.cuh).
//
// Exit rule (Bullet's, btSequentialImpulseConstraintSolver::solveGroupCacheFriendlyIterations): after every sweep the
// largest squared velocity-level change of a row, (delta_k * dinv_k)^2 with dinv_k = 1 / jacDiagABInv_k, is compared with
// m_leastSquaresResidualThreshold (P.res_thr; PyBullet: 1e-7); at or below it the robot's solve is over. A lane that
// has met it is frozen (its updates become no-ops) while the other lanes of the warp finish, so that every robot keeps
// exactly the impulses Bullet would have left it with.
template <typename AnyFn>
UPKIE_HD void pgs_solve(const SimParams& P, const float G[6][6], const float rhs[6], float lam[6], float mu,
                        float hiL, float hiR, const float dinv[6], AnyFn warp_any) {
  float r[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    r[k] = rhs[k];
#pragma unroll
    for (int l = 0; l < 2; ++l) r[k] += G[k][l] * lam[l];  // warm-started normals; frictions start from 0
  }
  bool frozen = false;
  for (int it = 0; it < P.pgs_iterations; ++it) {
    float res = 0.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      float lo, hi;
      if (k == 0) { lo = 0.f; hi = hiL; }
      else if (k == 1) { lo = 0.f; hi = hiR; }
      else { hi = mu * lam[(k < 4) ? 0 : 1]; lo = -hi; }
      const float nl = frozen ? lam[k] : fminf(fmaxf(r[k], lo), hi);
      const float delta = nl - lam[k];
      res = fmaxf(res, fabsf(delta) * dinv[k]);
      lam[k] = nl;
#pragma unroll
      for (int m = 0; m < 6; ++m) r[m] += G[m][k] * delta;
    }
    const bool was_frozen = frozen;
    frozen = frozen || (res * res <= P.res_thr);
#ifdef UPKIE_PGS_STATS
    if (frozen && !was_frozen) upkie_pgs_stats(it + 1);
    else if (!frozen && it + 1 == P.pgs_iterations) upkie_pgs_stats(it + 1);
#else
    (void)was_frozen;
#endif
    if (!warp_any(!frozen)) break;
  }
}

template <typename AnyFn, typename SyncFn = NoSync>
UPKIE_HD void physics_substep(const SimParams& P, RobotState& S, const float tau[6], const float* eps, float mu,
                              AnyFn warp_any, SyncFn phase_sync = SyncFn(), const float* wext = nullptr) {
  float R[9];
  quat_to_rot(S.quat, R);
  float V0[6];
  rot_tmul(R, S.angvel, &V0[0]);
  rot_tmul(R, S.linvel, &V0[3]);

  float IA0[21], pA0[6];
  base_inertia_bias(P, V0, IA0, pA0);
  LegCache lcL, lcR;
  float ccL[3][6], ccR[3][6], uuL[3], uuR[3];
  leg_pass12<0>(P, S.q, S.qd, tau, V0, eps, lcL, ccL, uuL, IA0, pA0);
  phase_sync();  // 1
  leg_pass12<1>(P, S.q, S.qd, tau, V0, eps, lcR, ccR, uuR, IA0, pA0);
  ldl6(IA0);
  float a0[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) a0[i] = wext ? wext[i] - pA0[i] : -pA0[i];
  ldl6_solve(IA0, a0);
  float qdd[6];
  leg_pass3<0>(P, lcL, ccL, uuL, a0, qdd);
  leg_pass3<1>(P, lcR, ccR, uuR, a0, qdd);

  // gravity as a uniform frame acceleration, classical acceleration of the origin
  const float zb[3] = {R[6], R[7], R[8]};  // world z axis in base coordinates
  {
    float lin[3], wxv[3], dw[3], dv[3];
    cross3(&V0[0], &V0[3], wxv);
    lin[0] = a0[3] - P.gravity * zb[0] + wxv[0];
    lin[1] = a0[4] - P.gravity * zb[1] + wxv[1];
    lin[2] = a0[5] - P.gravity * zb[2] + wxv[2];
    rot_mul(R, &a0[0], dw);
    rot_mul(R, lin, dv);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      S.angvel[i] = clampf(S.angvel[i] + P.h * dw[i], -P.vmax, P.vmax);
      S.linvel[i] = clampf(S.linvel[i] + P.h * dv[i], -P.vmax, P.vmax);
    }
#pragma unroll
    for (int j = 0; j < 6; ++j) S.qd[j] = clampf(S.qd[j] + P.h * qdd[j], -P.vmax, P.vmax);
  }

  // -- collision detection: tire circle vs the plane z = 0 (base coordinates)
  const float nxz = sqrtf(zb[0] * zb[0] + zb[2] * zb[2]);
  const bool rim_ok = nxz > 1e-6f;
  const float inv_n = rim_ok ? 1.f / nxz : 0.f;
  // lowest rim point relative to the wheel centre
  const float dB[3] = {-zb[0] * inv_n * P.wheel_radius, 0.f, -zb[2] * inv_n * P.wheel_radius};
  float oyL = P.jo[0][1] + P.jo[1][1] + P.jo[2][1];
  float oyR = P.jo[3][1] + P.jo[4][1] + P.jo[5][1];
  const float PL[3] = {lcL.ox[2] + dB[0], oyL, lcL.oz[2] + dB[2]};
  const float PR[3] = {lcR.ox[2] + dB[0], oyR, lcR.oz[2] + dB[2]};
  const float distL = S.pos[2] + zb[0] * PL[0] + zb[1] * PL[1] + zb[2] * PL[2];
  const float distR = S.pos[2] + zb[0] * PR[0] + zb[1] * PR[1] + zb[2] * PR[2];
  const bool actL = rim_ok && (distL < P.breaking_threshold);
  const bool actR = rim_ok && (distR < P.breaking_threshold);
  S.contact = (actL || actR) ? 1.f : 0.f;
  phase_sync();  // 2

  if (!warp_any(actL || actR)) {
    S.lam_n[0] = 0.f;
    S.lam_n[1] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) S.lam_t[k] = 0.f;
    phase_sync();  // 3
    phase_sync();  // 4
    phase_sync();  // 5
    phase_sync();  // 6
  } else {
    // contact directions in base coordinates: normal, rolling, lateral
    const float nB[3] = {zb[0], zb[1], zb[2]};
    float dirs[2][3][3];
    {
      // t1 = a x z / |.| with a = sgn * y: s * (zb.z, 0, -zb.x) / n
      const float sL = P.sgn[2], sR = P.sgn[5];
      const float t1[3] = {zb[2] * inv_n, 0.f, -zb[0] * inv_n};
      float t2[3];
      cross3(nB, t1, t2);
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        dirs[0][0][i] = nB[i]; dirs[1][0][i] = nB[i];
        dirs[0][1][i] = sL * t1[i]; dirs[1][1][i] = sR * t1[i];
        dirs[0][2][i] = sL * t2[i]; dirs[1][2][i] = sR * t2[i];
      }
    }
    // row order (Bullet: normals first, then friction): nL nR t1L t2L t1R t2R
    // J rows as spatial forces about the base origin
    float J[6][6];
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      const float* Pc = side == 0 ? PL : PR;
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        const int r = d == 0 ? side : 2 + 2 * side + (d - 1);
        cross3(Pc, dirs[side][d], &J[r][0]);
        J[r][3] = dirs[side][d][0]; J[r][4] = dirs[side][d][1]; J[r][5] = dirs[side][d][2];
      }
    }
    // wheel spatial velocities at the predicted generalized velocity
    float VL[6], VR[6];
    rot_tmul(R, S.angvel, &VL[0]);
    rot_tmul(R, S.linvel, &VL[3]);
#pragma unroll
    for (int i = 0; i < 6; ++i) VR[i] = VL[i];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float wl = P.sgn[k] * S.qd[k], wr = P.sgn[3 + k] * S.qd[3 + k];
      VL[1] += wl; VL[3] -= lcL.oz[k] * wl; VL[5] += lcL.ox[k] * wl;
      VR[1] += wr; VR[3] -= lcR.oz[k] * wr; VR[5] += lcR.ox[k] * wr;
    }
    // Delassus matrix W = J M^-1 J^T through impulse responses
    float W[6][6];
#pragma unroll
    for (int l = 0; l < 6; ++l) {
      const bool left = (l == 0) || (l == 2) || (l == 3);
      float uL[3] = {0.f, 0.f, 0.f}, uR[3] = {0.f, 0.f, 0.f};
      float p0[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (left) leg_impulse_up(P, 0, lcL, J[l], uL, p0);
      else leg_impulse_up(P, 3, lcR, J[l], uR, p0);
      float da0[6];
#pragma unroll
      for (int i = 0; i < 6; ++i) da0[i] = -p0[i];
      ldl6_solve(IA0, da0);
      float aL[6], aR[6], dq[3];
      leg_impulse_down(P, 0, lcL, uL, da0, aL, dq);
      leg_impulse_down(P, 3, lcR, uR, da0, aR, dq);
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        const bool kleft = (k == 0) || (k == 2) || (k == 3);
        const float* a = kleft ? aL : aR;
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) acc += J[k][i] * a[i];
        W[k][l] = acc;
      }
      if (l & 1) phase_sync();  // 3, 4, 5
    }
    // right-hand sides (btMultiBodyConstraintSolver::setupMultiBodyContactConstraint)
    float rhs[6], jdi[6], lam[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const bool kleft = (k == 0) || (k == 2) || (k == 3);
      const float* Vw = kleft ? VL : VR;
      float rel = 0.f;
#pragma unroll
      for (int i = 0; i < 6; ++i) rel += J[k][i] * Vw[i];
      // warm start (Bullet SOLVER_USE_WARMSTARTING): normals from the previous substep, frictions from 0
      lam[k] = k == 0 ? (actL ? P.warm * S.lam_n[0] : 0.f) : (k == 1 ? (actR ? P.warm * S.lam_n[1] : 0.f) : 0.f);
      if (k < 2) {
        const float pen = k == 0 ? distL : distR;
        jdi[k] = 1.f / (W[k][k] + P.cfm);
        float pos_err = 0.f, vel_err = -rel;
        if (pen > 0.f) vel_err -= pen * P.inv_h;
        else pos_err = -pen * P.erp * P.inv_h;
        rhs[k] = (pos_err + vel_err) * jdi[k];
      } else {
        jdi[k] = W[k][k] > 0.f ? 1.f / W[k][k] : 0.f;
        rhs[k] = -rel * jdi[k];
      }
    }
    const float cfmrow = P.cfm;  // m_cfm = cfm * jacDiagABInv
    const float hiL = actL ? 1e10f : 0.f, hiR = actR ? 1e10f : 0.f;
    // Projected Gauss-Seidel, at most Bullet's iteration count, with Bullet's residual exit rule (pgs_solve)
    float dinv[6];  // 1 / jacDiagABInv: turns an impulse change into the row's velocity change
#pragma unroll
    for (int k = 0; k < 6; ++k) dinv[k] = W[k][k] + (k < 2 ? P.cfm : 0.f);
    // row update lam_k <- clamp(lam_k + rhs_k - cfm_k lam_k - jdi_k sum_l W_kl lam_l) with the
    // row pre-scaled: G_kl = -jdi_k W_kl (l != k), G_kk = 1 - cfm_k - jdi_k W_kk
#pragma unroll
    for (int k = 0; k < 6; ++k) {
#pragma unroll
      for (int l = 0; l < 6; ++l) W[k][l] = -jdi[k] * W[k][l];
      W[k][k] += 1.f - (k < 2 ? cfmrow * jdi[k] : 0.f);
    }
    pgs_solve(P, W, rhs, lam, mu, hiL, hiR, dinv, warp_any);
    S.lam_n[0] = lam[0];
    S.lam_n[1] = lam[1];
#pragma unroll
    for (int k = 0; k < 4; ++k) S.lam_t[k] = lam[2 + k];
    // apply the total wheel impulses
    float fL[6], fR[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      fL[i] = lam[0] * J[0][i] + lam[2] * J[2][i] + lam[3] * J[3][i];
      fR[i] = lam[1] * J[1][i] + lam[4] * J[4][i] + lam[5] * J[5][i];
    }
    float uL[3], uR[3];
    float p0[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    leg_impulse_up(P, 0, lcL, fL, uL, p0);
    leg_impulse_up(P, 3, lcR, fR, uR, p0);
    float da0[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) da0[i] = -p0[i];
    ldl6_solve(IA0, da0);
    float aL[6], aR[6], dqL[3], dqR[3];
    leg_impulse_down(P, 0, lcL, uL, da0, aL, dqL);
    leg_impulse_down(P, 3, lcR, uR, da0, aR, dqR);
    float dw[3], dv[3];
    rot_mul(R, &da0[0], dw);
    rot_mul(R, &da0[3], dv);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      S.angvel[i] = clampf(S.angvel[i] + dw[i], -P.vmax, P.vmax);
      S.linvel[i] = clampf(S.linvel[i] + dv[i], -P.vmax, P.vmax);
      S.qd[i] = clampf(S.qd[i] + dqL[i], -P.vmax, P.vmax);
      S.qd[3 + i] = clampf(S.qd[3 + i] + dqR[i], -P.vmax, P.vmax);
    }
    phase_sync();  // 6
  }

  // -- position integration with the new velocities
#pragma unroll
  for (int i = 0; i < 3; ++i) S.pos[i] += P.h * S.linvel[i];
  {
    // rotation increment exp(w h / 2): the even Taylor polynomials of sin(x) / x and cos(x) to degree 6, x = |w| h / 2.
    // make_sim_params bounds h * max_coordinate_velocity by 0.6, so x <= 0.52 and the truncation stays below 1.4e-7
    // (defaults, h = 1 ms and the clamp at 100: x <= 0.087, ~1e-14). Not sinf / cosf: under --use_fast_math they
    // carry an absolute error of up to 3.6e-7, as large as the increment itself at slow rates
    const float* om = S.angvel;
    const float hh = 0.5f * P.h;
    const float x2 = (om[0] * om[0] + om[1] * om[1] + om[2] * om[2]) * hh * hh;
    const float sc = hh * (1.f + x2 * (-1.f / 6.f + x2 * (1.f / 120.f - x2 * (1.f / 5040.f))));
    const float ax = om[0] * sc, ay = om[1] * sc, az = om[2] * sc;
    const float dqw = 1.f + x2 * (-0.5f + x2 * (1.f / 24.f - x2 * (1.f / 720.f)));
    const float qw = S.quat[0], qx = S.quat[1], qy = S.quat[2], qz = S.quat[3];
    const float nw = dqw * qw - ax * qx - ay * qy - az * qz;
    const float nx = dqw * qx + ax * qw + ay * qz - az * qy;
    const float ny = dqw * qy - ax * qz + ay * qw + az * qx;
    const float nz = dqw * qz + ax * qy - ay * qx + az * qw;
    const float inv = 1.f / sqrtf(nw * nw + nx * nx + ny * ny + nz * nz);
    S.quat[0] = nw * inv; S.quat[1] = nx * inv; S.quat[2] = ny * inv; S.quat[3] = nz * inv;
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) S.q[j] += P.h * S.qd[j];
}

}  // namespace upkie_b200
#include "sim_pair.cuh"
namespace upkie_b200 {

// the substep the env-level functions below use
// `wext`: external wrench on the base (moment about the base origin, force; base coordinates) or null
template <typename AnyFn, typename SyncFn = NoSync>
UPKIE_HD void substep(const SimParams& P, RobotState& S, const float tau[6], const float* eps, float mu, AnyFn warp_any,
                      SyncFn phase_sync = SyncFn(), const float* wext = nullptr, int limits = 0, bool locked = false,
                      BodyRecOut rec = BodyRecOut{nullptr, 0}) {
#if UPKIE_PAIRED_LEGS
  physics_substep_paired(P, S, tau, eps, mu, warp_any, phase_sync, wext, limits, locked, rec);
#else
  (void)limits;  // the scalar-leg build has no joint-limit rows
  (void)locked;
  (void)rec;
  physics_substep(P, S, tau, eps, mu, warp_any, phase_sync, wext);
#endif
}

// External forces (PyBulletBackend.set_external_forces / __apply_external_forces,
// pybullet_backend.py:603-658): one force per body acting at the body's centre of mass, expressed in the
// world frame or (bit i of `local`) in the body frame, constant over the substeps of a tick. A wrench on
// body i enters the equations of motion only through the generalized force J_i^T w, so it is applied as
// joint torques on the ancestors of the body plus a wrench on the base, outside the ABA core.
struct ExtForces {
  const float* f;  // this env's forces, element (body b, axis k) at f[(3 * b + k) * stride]
  size_t stride;
  uint32_t local;
};

// The push of push randomisation (PushRand below) in force in this tick: a world-frame force on one body, zero when
// the env is not being pushed
struct ExtPush {
  int body;
  float f[3];
};

// PUSH (the push families' kernels with a push spec set): `push` is added to the force of X on its body, and X.f may
// be null (no forces of upkie_b200_set_external_forces). A push body is never in X.local (the handle rejects it).
template <bool PUSH = false>
UPKIE_HD void external_generalized_forces(const SimParams& P, const RobotState& S, const ExtForces& X,
                                          float tau_add[6], float wbase[6], const ExtPush* push = nullptr) {
  float R[9];
  quat_to_rot(S.quat, R);
#pragma unroll
  for (int k = 0; k < 6; ++k) { tau_add[k] = 0.f; wbase[k] = 0.f; }
  auto body_force = [&](int b, float out[3]) {
    if (!PUSH || X.f) {
      out[0] = X.f[(3 * b + 0) * X.stride];
      out[1] = X.f[(3 * b + 1) * X.stride];
      out[2] = X.f[(3 * b + 2) * X.stride];
    } else {
      out[0] = 0.f; out[1] = 0.f; out[2] = 0.f;
    }
    if (PUSH && b == push->body) {
      // the sum a host-written force of (user force + push) would hold; the push alone without user forces
#pragma unroll
      for (int k = 0; k < 3; ++k) out[k] = X.f ? out[k] + push->f[k] : push->f[k];
    }
  };
  auto add_base = [&](const float c[3], const float f[3]) {
    wbase[0] += c[1] * f[2] - c[2] * f[1];
    wbase[1] += c[2] * f[0] - c[0] * f[2];
    wbase[2] += c[0] * f[1] - c[1] * f[0];
    wbase[3] += f[0]; wbase[4] += f[1]; wbase[5] += f[2];
  };
  {
    float F[3], fb[3];
    body_force(0, F);
    if (X.local & 1u) { fb[0] = F[0]; fb[1] = F[1]; fb[2] = F[2]; }
    else rot_tmul(R, F, fb);
    add_base(P.com[0], fb);
  }
#pragma unroll
  for (int side = 0; side < 2; ++side) {
    float th = 0.f, o[3][3], cs = 1.f, sn = 0.f;  // rotation of the parent body about +y, joint origins
    float prev[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int j = 3 * side + k, b = j + 1;
      // joint origin: parent origin + R_y(theta_parent) * joint offset
      o[k][0] = prev[0] + cs * P.jo[j][0] + sn * P.jo[j][2];
      o[k][1] = prev[1] + P.jo[j][1];
      o[k][2] = prev[2] - sn * P.jo[j][0] + cs * P.jo[j][2];
      th += P.sgn[j] * S.q[j];
      sincosf(th - 6.28318530718f * rintf(th * 0.15915494309f), &sn, &cs);  // fast-math sincos: reduce to [-pi, pi]
      prev[0] = o[k][0]; prev[1] = o[k][1]; prev[2] = o[k][2];
      float F[3], fb[3], c[3];
      body_force(b, F);
      if ((X.local >> b) & 1u) {
        fb[0] = cs * F[0] + sn * F[2]; fb[1] = F[1]; fb[2] = -sn * F[0] + cs * F[2];
      } else {
        rot_tmul(R, F, fb);
      }
      c[0] = o[k][0] + cs * P.com[b][0] + sn * P.com[b][2];
      c[1] = o[k][1] + P.com[b][1];
      c[2] = o[k][2] - sn * P.com[b][0] + cs * P.com[b][2];
      add_base(c, fb);
#pragma unroll
      for (int m = 0; m <= k; ++m)  // torque of the force about every ancestor joint axis (+-y)
        tau_add[3 * side + m] += P.sgn[3 * side + m] * ((c[2] - o[m][2]) * fb[0] - (c[0] - o[m][0]) * fb[2]);
    }
  }
}

// pybullet_backend.py:492-553 compute_joint_torque. torque_control_kp / kd and the joint's friction come from the
// config or from the env's row of the parameter table (the caller picks; the arithmetic is the same either way).
UPKIE_HD float joint_torque(float torque_control_kp, float torque_control_kd, float friction, float q, float qd,
                            float ff, float target_position, float target_velocity, float kp_scale, float kd_scale,
                            float maximum_torque, float control_noise = 0.f) {
  const float kp = kp_scale * torque_control_kp;
  const float kd = kd_scale * torque_control_kd;
  float torque = ff;
  torque += kd * (target_velocity - qd);
  if (!(target_position != target_position)) torque += kp * (target_position - q);
  if (fabsf(qd) > 1e-3f) {
    const float sign = qd > 0.f ? 1.f : -1.f;
    torque += -friction * sign;
  }
  torque += control_noise;  // torque-control Gaussian white noise, before the clip (pybullet_backend.py:545-552)
  // np.clip(x, lo, hi) = minimum(maximum(x, lo), hi)
  return fminf(fmaxf(torque, -maximum_torque), maximum_torque);
}

// ---- Servo velocity limits (upkie_b200_set_velocity_derate, tools/configure_servos:99-104) ----
// The handle's device block: the spec and the per-env state (include/upkie_b200.h): count[i] = k, the number of the
// env's last draw, and max_velocity = v_i, each joint's limit in rad/s (0 outside the mask), [UPKIE_NJ][stride]
// structure-of-arrays like the state, env i in column i. The draws are at the end of this file.
struct VelocityDerate {
  UpkieVelocityDerate spec;
  uint32_t* count;
  float* max_velocity;
  int stride;
};

// The moteus derate of the torque t of a joint at velocity qd under the limit v, the band `derate` and the effort limit
// tau_max: past v, the torque that drives the joint faster in its direction of motion is capped by f * tau_max, f
// falling linearly from 1 at v to 0 at v + derate. A braking torque, and any torque at |qd| <= v, is t bit for bit.
UPKIE_HD float velocity_derate_torque(float t, float qd, float v, float derate, float tau_max) {
  const float s = fabsf(qd);
  if (!(s > v)) return t;
  const float cap = clampf((v + derate - s) / derate, 0.f, 1.f) * tau_max;
  return qd > 0.f ? fminf(t, cap) : fmaxf(t, -cap);
}

// Joint j's torque t of env i (its column of V) at velocity qd: derated on a joint of the mask, t otherwise
UPKIE_HD float velocity_derate_joint(const VelocityDerate& V, int i, int j, float qd, float t, float tau_max) {
  if (!((V.spec.joint_mask >> j) & 1u)) return t;
  return velocity_derate_torque(t, qd, V.max_velocity[size_t(j) * size_t(V.stride) + size_t(i)], V.spec.derate[j],
                                tau_max);
}

// ---- Servo torque-constant errors (upkie_b200_set_torque_scale, pybullet_backend.py:457-459) ----
// The handle's device block: the spec and the per-env state (include/upkie_b200.h): count[i] = k, the number of the
// env's last draw, and scale = s_i, each joint's delivered-torque scale (exactly 1 outside the mask), [UPKIE_NJ][stride]
// structure-of-arrays like the state, env i in column i. The draws are at the end of this file.
struct TorqueScale {
  UpkieTorqueScale spec;
  uint32_t* count;
  float* scale;
  int stride;
};

// An env's six scales, as the substeps of a tick hold them
struct Scale6 {
  float s[UPKIE_NJ];
};

// Env i's scales through load(j) (its column of the per-env state)
template <typename Load>
UPKIE_HD Scale6 torque_scale_load(Load load) {
  Scale6 o;
#pragma unroll
  for (int j = 0; j < UPKIE_NJ; ++j) o.s[j] = load(j);
  return o;
}

// The torque a joint receives when its servo applies t under the scale s: fl(s * t), one rounding. On the device the
// product is __fmul_rn, which fast-math contraction never folds into the substep's next add.
UPKIE_HD float torque_scale_apply(float s, float t) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(s, t);
#else
  return s * t;
#endif
}

// Derived observation quantities (pybullet_backend.py:333-490). Updates the
// IMU finite-difference state exactly once per call, as get_spine_observation.
UPKIE_HD void observe_update(const SimParams& P, RobotState& S) {
  float R[9];
  quat_to_rot(S.quat, R);
  float rp[3], w[3];
  rot_mul(R, P.imu_pos, rp);
  cross3(S.angvel, rp, w);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float v = S.linvel[i] + w[i];
    S.imu_acc[i] = (v - S.prev_imu_vel[i]) * P.inv_dt;  // dt, not the substep (pybullet_backend.py:405-408)
    S.prev_imu_vel[i] = v;
  }
}

UPKIE_HD float base_pitch(const RobotState& S) {
  // pybullet_backend.py:350-352. The argument is sin(pitch) of a unit quaternion; clamped because round-off can put
  // it an ulp beyond 1 when the torso lies flat on the floor (np.arcsin would hand out nan there)
  return asinf(clampf(2.f * (S.quat[0] * S.quat[2] - S.quat[3] * S.quat[1]), -1.f, 1.f));
}

// scipy Rotation.from_matrix(...).as_quat(scalar_first=True) (rotations.py:14-33)
UPKIE_HD void quat_from_rot(const float M[9], float q_wxyz[4]) {
  const float tr = M[0] + M[4] + M[8];
  float dec[4] = {M[0], M[4], M[8], tr};
  int choice = 0;
#pragma unroll
  for (int i = 1; i < 4; ++i)
    if (dec[i] > dec[choice]) choice = i;
  float x, y, z, w;
  if (choice == 0) {
    x = 1.f - tr + 2.f * M[0]; y = M[3] + M[1]; z = M[6] + M[2]; w = M[7] - M[5];
  } else if (choice == 1) {
    y = 1.f - tr + 2.f * M[4]; z = M[7] + M[5]; x = M[1] + M[3]; w = M[2] - M[6];
  } else if (choice == 2) {
    z = 1.f - tr + 2.f * M[8]; x = M[2] + M[6]; y = M[5] + M[7]; w = M[3] - M[1];
  } else {
    x = M[7] - M[5]; y = M[2] - M[6]; z = M[3] - M[1]; w = 1.f + tr;
  }
  const float inv = 1.f / sqrtf(x * x + y * y + z * z + w * w);
  q_wxyz[0] = w * inv; q_wxyz[1] = x * inv; q_wxyz[2] = y * inv; q_wxyz[3] = z * inv;
}

// full spine observation dictionary from the state (no side effects)
UPKIE_HD void spine_observation(const SimParams& P, const RobotState& S, float* o, const float* torque_obs = nullptr) {
  float R[9];
  quat_to_rot(S.quat, R);
  float om_b[3];
  rot_tmul(R, S.angvel, om_b);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    o[UPKIE_SP_BASE_ANGVEL + i] = om_b[i];
    o[UPKIE_SP_BASE_LINVEL + i] = S.linvel[i];
  }
  o[UPKIE_SP_PITCH] = base_pitch(S);
#pragma unroll
  for (int i = 0; i < 9; ++i) o[UPKIE_SP_ROT + i] = R[i];
  // rotation_imu_to_world = R * Rbi^T ; rotation_imu_to_ars = diag(1,-1,-1) * that
  float Riw[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      Riw[3 * i + j] = R[3 * i + 0] * P.Rbi[3 * j + 0] + R[3 * i + 1] * P.Rbi[3 * j + 1] + R[3 * i + 2] * P.Rbi[3 * j + 2];
  float Ria[9];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    Ria[j] = Riw[j];
    Ria[3 + j] = -Riw[3 + j];
    Ria[6 + j] = -Riw[6 + j];
  }
  quat_from_rot(Ria, &o[UPKIE_SP_IMU_QUAT]);
  float t[3];
  rot_tmul(Riw, S.angvel, t);
#pragma unroll
  for (int i = 0; i < 3; ++i) o[UPKIE_SP_IMU_ANGVEL + i] = t[i];
  rot_tmul(Riw, S.imu_acc, t);
#pragma unroll
  for (int i = 0; i < 3; ++i) o[UPKIE_SP_IMU_LINACC + i] = t[i];
  const float praw[3] = {S.imu_acc[0], S.imu_acc[1], S.imu_acc[2] + 9.81f};
  rot_tmul(Riw, praw, t);
#pragma unroll
  for (int i = 0; i < 3; ++i) o[UPKIE_SP_IMU_RAWACC + i] = t[i];
  o[UPKIE_SP_CONTACT] = S.contact;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    float* so = o + UPKIE_SP_SERVO + j * UPKIE_OBS_KEYS;
    so[UPKIE_OBS_POSITION] = S.q[j];
    so[UPKIE_OBS_VELOCITY] = S.qd[j];
    so[UPKIE_OBS_TORQUE] = torque_obs ? torque_obs[j] : S.torque[j];
    so[UPKIE_OBS_TEMPERATURE] = 42.0f;
    so[UPKIE_OBS_VOLTAGE] = 18.0f;
  }
  const float signed_radius = P.left_sign * P.wheel_radius;
  o[UPKIE_SP_ODOM_POS] = 0.5f * (S.q[2] - S.q[5]) * signed_radius;
  o[UPKIE_SP_ODOM_VEL] = 0.5f * (S.qd[2] - S.qd[5]) * signed_radius;
}

// ---- env-level steps -----------------------------------------------------------

// UpkieServos.get_spine_action clamps + PyBulletBackend.step + observation update.
// `a` is the 6x6 servo action (modified in place by the clamps).
// UpkieServos.get_spine_action clamps (upkie_servos.py:316-344), in place.
UPKIE_HD uint32_t clamp_servo_action(const SimParams& P, float a[UPKIE_ACT_DIM]) {
  uint32_t err = 0;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const float lo[6] = {P.q_lower[j], -P.qd_max[j], -P.tau_max[j], 0.f, 0.f, 0.f};
    const float hi[6] = {P.q_upper[j], P.qd_max[j], P.tau_max[j], P.max_gain_scale, P.max_gain_scale, P.tau_max[j]};
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const float v = a[j * 6 + k];
      const float c = P.skip_action_clamps ? v : clamp_ref(v, lo[k], hi[k]);
      if (c != v && !(c != c && v != v)) err |= UPKIE_ERR_CLAMPED;
      a[j * 6 + k] = c;
    }
    if (a[j * 6 + UPKIE_ACT_VELOCITY] != a[j * 6 + UPKIE_ACT_VELOCITY]) err |= UPKIE_ERR_NAN_VELOCITY;
  }
  return err;
}

// One substep of PyBulletBackend.step (pybullet_backend.py:276-306): torque law on
// the live joint state, then one stepSimulation. `store_torque` is false for the
// zero-torque substep of a reset (the reference keeps __joint_torques across resets).
// Counter-based Gaussian noise: (seed, global env index, per-env tick, slot) -> 8 standard normals
// (Philox4x32-10 + Box-Muller). Slots 0..nb_substeps-1 feed the torque-control noise of the substeps,
// slot 255 the torque-measurement noise of the observation.
struct Philox4;
UPKIE_HD Philox4 philox4x32_10(uint64_t counter_lo, uint64_t counter_hi, uint64_t key);
struct NoiseCtx {
  uint64_t env;   // global env index
  uint32_t tick;  // per-env step counter
};
UPKIE_HD void gaussian8(uint64_t seed, const NoiseCtx& nz, uint32_t slot, float out[8]);

template <typename AnyFn, typename SyncFn = NoSync>
UPKIE_HD void servo_substep(const SimParams& P, RobotState& S, const float a[UPKIE_ACT_DIM], bool zero_torque,
                            const float* eps, float mu, AnyFn warp_any, SyncFn phase_sync = SyncFn(),
                            const NoiseCtx* nz = nullptr, int sub = 0, const ExtForces* ext = nullptr,
                            int limits = 0, BodyRecOut rec = BodyRecOut{nullptr, 0}, int env = -1,
                            const ExtPush* push = nullptr, const VelocityDerate* derate = nullptr,
                            int derate_env = 0, const Scale6* tscale = nullptr) {
  // `env`: this robot's column of the per-env parameter table; env < 0 (the default, and a constant in the
  // instantiations that never run with a table) compiles the table reads out. Its values are read where they are used, under a uniform branch
  // on the table pointer; the arithmetic is the same for the config's values and the table's.
  // `derate` (non-null in every lane of a FAM_SENSE launch with velocity limits; a null constant elsewhere, which
  // compiles the law out): the servo velocity limits of env `derate_env`, read from its column in every substep.
  // `tscale` (likewise, for a FAM_SENSE launch with torque scales): the env's six delivered-torque scales, loaded once
  // per tick (exactly 1 outside the mask, and fl(1 t) = t). The reply S.torque stays the servo's t; the physics
  // integrates fl(s t).
  const bool table = env >= 0 && P.env_params != nullptr;
  float tau[6];
  float noise[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (P.any_ctrl_noise && nz) {
    gaussian8(P.noise_seed, *nz, uint32_t(sub), noise);
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const float sd = table ? env_param(P, env, UPKIE_EP_CTRL_NOISE + j) : P.ctrl_noise[j];
      noise[j] = sd > 1e-10f ? noise[j] * sd : 0.f;
    }
  }
  const float kp = table ? env_param(P, env, UPKIE_EP_KP) : P.kp;
  const float kd = table ? env_param(P, env, UPKIE_EP_KD) : P.kd;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const float* aj = a + j * 6;
    const float fr = table ? env_param(P, env, UPKIE_EP_FRICTION + j) : P.joint_friction[j];
    float t = joint_torque(kp, kd, fr, S.q[j], S.qd[j], aj[UPKIE_ACT_FEEDFORWARD_TORQUE], aj[UPKIE_ACT_POSITION],
                           aj[UPKIE_ACT_VELOCITY], aj[UPKIE_ACT_KP_SCALE], aj[UPKIE_ACT_KD_SCALE],
                           aj[UPKIE_ACT_MAXIMUM_TORQUE], noise[j]);
    if (derate) t = velocity_derate_joint(*derate, derate_env, j, S.qd[j], t, P.tau_max[j]);
    tau[j] = zero_torque ? 0.f : (tscale ? torque_scale_apply(tscale->s[j], t) : t);
    if (!zero_torque) S.torque[j] = t;
  }
  if (limits != 0) {
    // joint-limit instantiations: ONE inlined copy of the substep (its code is twice as long there), the external
    // wrench passed through a nullable pointer. `push` (non-null in every lane of a launch with a push spec, the
    // push families' kernels) adds the lane's push to `ext`, which may then be null.
    float tau_add[6], wbase[6];
    const bool forced = (ext || push) && !zero_torque;
    if (forced) {
      if (push) external_generalized_forces<true>(P, S, ext ? *ext : ExtForces{nullptr, 0, 0u}, tau_add, wbase, push);
      else external_generalized_forces(P, S, *ext, tau_add, wbase);
#pragma unroll
      for (int j = 0; j < 6; ++j) tau[j] += tau_add[j];
    }
    substep(P, S, tau, eps, mu, warp_any, phase_sync, forced ? wbase : nullptr, limits, false, rec);
  } else if (ext && !zero_torque) {  // the substep of a reset runs without external forces (pybullet_backend.py:227-228)
    float tau_add[6], wbase[6];
    external_generalized_forces(P, S, *ext, tau_add, wbase);
#pragma unroll
    for (int j = 0; j < 6; ++j) tau[j] += tau_add[j];
    substep(P, S, tau, eps, mu, warp_any, phase_sync, wbase, 0);
  } else {
    substep(P, S, tau, eps, mu, warp_any, phase_sync, nullptr, 0);
  }
}

UPKIE_HD uint32_t state_sanity(const RobotState& S) {
  const float chk = S.quat[0] + S.quat[1] + S.quat[2] + S.quat[3] + S.pos[2] + S.linvel[0];
  return (fabsf(chk) <= 3.0e38f) ? 0u : UPKIE_ERR_NAN_STATE;
}

// Host-side test entry (tests/hostsim): one env tick from a servo action. SCALAR_LEGS = false runs the substep the
// kernels run (substep(): the paired legs unless UPKIE_PAIRED_LEGS is 0), true the scalar-leg variant.
template <bool SCALAR_LEGS = false, typename AnyFn>
UPKIE_HD uint32_t step_servo_action(const SimParams& P, RobotState& S, float a[UPKIE_ACT_DIM], const float* eps, float mu,
                                    AnyFn warp_any, float* body_rec = nullptr) {
  uint32_t err = 0;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const float lo[6] = {P.q_lower[j], -P.qd_max[j], -P.tau_max[j], 0.f, 0.f, 0.f};
    const float hi[6] = {P.q_upper[j], P.qd_max[j], P.tau_max[j], P.max_gain_scale, P.max_gain_scale, P.tau_max[j]};
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const float v = a[j * 6 + k];
      const float c = clamp_ref(v, lo[k], hi[k]);
      if (c != v && !(c != c && v != v)) err |= UPKIE_ERR_CLAMPED;
      a[j * 6 + k] = c;
    }
    if (a[j * 6 + UPKIE_ACT_VELOCITY] != a[j * 6 + UPKIE_ACT_VELOCITY]) err |= UPKIE_ERR_NAN_VELOCITY;
  }
  for (int sub = 0; sub < P.nb_substeps; ++sub) {
    float tau[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const float* aj = a + j * 6;
      tau[j] = joint_torque(P.kp, P.kd, P.joint_friction[j], S.q[j], S.qd[j], aj[UPKIE_ACT_FEEDFORWARD_TORQUE], aj[UPKIE_ACT_POSITION],
                            aj[UPKIE_ACT_VELOCITY], aj[UPKIE_ACT_KP_SCALE], aj[UPKIE_ACT_KD_SCALE],
                            aj[UPKIE_ACT_MAXIMUM_TORQUE]);
      S.torque[j] = tau[j];
    }
    if (SCALAR_LEGS) physics_substep(P, S, tau, eps, mu, warp_any);  // no joint-limit rows in the scalar-leg variant
    else substep(P, S, tau, eps, mu, warp_any, NoSync(), nullptr, P.joint_limits, false,
                 BodyRecOut{sub + 1 == P.nb_substeps ? body_rec : nullptr, 1});
  }
  observe_update(P, S);
  const float chk = S.quat[0] + S.quat[1] + S.quat[2] + S.quat[3] + S.pos[2] + S.linvel[0];
  if (!(fabsf(chk) <= 3.0e38f)) err |= UPKIE_ERR_NAN_STATE;
  return err;
}

// UpkieGyropod.__get_spine_action (upkie_gyropod.py:246-331): builds the servo
// action from [ground velocity, yaw velocity], advancing the leg low-pass filter.
UPKIE_HD uint32_t gyropod_action(const SimParams& P, RobotState& S, float a0, float a1, float a[UPKIE_ACT_DIM]) {
  uint32_t err = 0;
  const float gv = clamp_ref(a0, -P.max_ground_velocity, P.max_ground_velocity);
  const float yv = clamp_ref(a1, -P.max_yaw_velocity, P.max_yaw_velocity);
  if (gv != a0 || yv != a1) err |= UPKIE_ERR_CLAMPED;
  const float wheel_velocity = gv / P.wheel_radius;
  float left = P.left_sign * wheel_velocity;
  float right = -P.left_sign * wheel_velocity;
  const float yaw_to_wheel = P.left_sign * P.half_wheel_base / P.wheel_radius;
  left += yaw_to_wheel * yv;
  right += yaw_to_wheel * yv;
  const float alpha = P.dt / 1.0f;  // low_pass_filter(cutoff_period=1.0), filters.py:63-80
#pragma unroll
  for (int k = 0; k < 4; ++k) S.leg_target[k] = S.leg_target[k] + alpha * (0.0f - S.leg_target[k]);
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    a[j * 6 + UPKIE_ACT_POSITION] = nanf("");
    a[j * 6 + UPKIE_ACT_VELOCITY] = 0.f;
    a[j * 6 + UPKIE_ACT_FEEDFORWARD_TORQUE] = 0.f;
    a[j * 6 + UPKIE_ACT_KP_SCALE] = 1.f;
    a[j * 6 + UPKIE_ACT_KD_SCALE] = 1.f;
    a[j * 6 + UPKIE_ACT_MAXIMUM_TORQUE] = P.tau_max[j];
  }
  const int leg_joint[4] = {0, 1, 3, 4};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int j = leg_joint[k];
    a[j * 6 + UPKIE_ACT_POSITION] = S.leg_target[k];
    a[j * 6 + UPKIE_ACT_KP_SCALE] = P.leg_gain_scale;
    a[j * 6 + UPKIE_ACT_KD_SCALE] = P.leg_gain_scale;
  }
  a[2 * 6 + UPKIE_ACT_VELOCITY] = left;
  a[5 * 6 + UPKIE_ACT_VELOCITY] = right;
  return err;
}

// gyropod observation vector (upkie_gyropod.py:186-214)
UPKIE_HD void gyropod_obs(const SimParams& P, const RobotState& S, float o6[6]) {
  float R[9];
  quat_to_rot(S.quat, R);
  const float signed_radius = P.left_sign * P.wheel_radius;
  o6[0] = 0.5f * (S.q[2] - S.q[5]) * signed_radius;
  o6[1] = base_pitch(S);
  o6[2] = S.yaw;
  o6[3] = 0.5f * (S.qd[2] - S.qd[5]) * signed_radius;
  o6[4] = R[1] * S.angvel[0] + R[4] * S.angvel[1] + R[7] * S.angvel[2];  // (R^T w).y
  o6[5] = S.yaw_vel;
}

// _reset_robot_state (pybullet_backend.py:234-267): pose and velocities only
UPKIE_HD void reset_pose(RobotState& S, const float init[UPKIE_INIT_DIM]) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    S.pos[i] = init[UPKIE_INIT_POS + i];
    S.linvel[i] = init[UPKIE_INIT_LINVEL + i];
    S.angvel[i] = init[UPKIE_INIT_ANGVEL + i];  // body-frame vector used as world-frame (:253-258)
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) S.quat[i] = init[UPKIE_INIT_QUAT + i];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    S.q[j] = init[UPKIE_INIT_Q + j];
    S.qd[j] = 0.f;
  }
  S.lam_n[0] = 0.f;  // new contact points carry no cached impulse
  S.lam_n[1] = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) S.lam_t[k] = 0.f;
}

// UpkieGyropod.reset (upkie_gyropod.py:216-244), after the reset's stepSimulation + observation
UPKIE_HD void reset_wrapper_state(RobotState& S) {
  S.leg_target[0] = S.q[0]; S.leg_target[1] = S.q[1]; S.leg_target[2] = S.q[3]; S.leg_target[3] = S.q[4];
  S.yaw = 0.f;
  S.yaw_vel = 0.f;
}

// PyBulletBackend.reset (pybullet_backend.py:220-267) + UpkieGyropod.reset (upkie_gyropod.py:216-244)
template <typename AnyFn>
UPKIE_HD void reset_robot(const SimParams& P, RobotState& S, const float init[UPKIE_INIT_DIM], const float* eps, float mu,
                          AnyFn warp_any, int limits, BodyRecOut rec = BodyRecOut{nullptr, 0}) {
  reset_pose(S, init);
  const float zero[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  substep(P, S, zero, eps, mu, warp_any, NoSync(), nullptr, limits, false, rec);  // one stepSimulation (:228)
  observe_update(P, S);
  reset_wrapper_state(S);
}

// ---- spine mode: the timing of the C++ Bullet spine in simulate() mode ----------------------------------------------
// What the spine's actuation interface holds between cycles (layout UPKIE_LAG_*, include/upkie_b200.h), plus the last
// observation the spine assembled (what get_spine_observation / the env observation report).
struct SpineLag {
  float rep1[18], rep2[18];  // servo replies of the latest cycle and of the one before: [6][position, velocity, torque]
  float imu[13];             // latest IMU reading: orientation_imu_in_ars wxyz, angular velocity, acceleration, raw
  float obs_rep[18], obs_imu[13];  // the assembled observation: replies of two cycles ago, IMU of the last cycle
  float obs_base[10];        // "sim" ground truth at that instant: base quaternion wxyz, linear, angular velocity (world)
  float obs_contact;
};

// bullet::read_imu_data (upkie/cpp/interfaces/bullet/read_imu_data.h:25-89) on the current state; the acceleration is
// differentiated against the IMU velocity of the previous cycle over one cycle (inv_h)
UPKIE_HD void spine_read_imu(const SimParams& P, RobotState& S, float imu[13]) {
  float R[9];
  quat_to_rot(S.quat, R);
  float rp[3], w[3], acc[3];
  rot_mul(R, P.imu_pos, rp);
  cross3(S.angvel, rp, w);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float v = S.linvel[i] + w[i];
    acc[i] = (v - S.prev_imu_vel[i]) * P.inv_h;
    S.prev_imu_vel[i] = v;
    S.imu_acc[i] = acc[i];
  }
  float Riw[9], Ria[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      Riw[3 * i + j] = R[3 * i + 0] * P.Rbi[3 * j + 0] + R[3 * i + 1] * P.Rbi[3 * j + 1] + R[3 * i + 2] * P.Rbi[3 * j + 2];
#pragma unroll
  for (int j = 0; j < 3; ++j) { Ria[j] = Riw[j]; Ria[3 + j] = -Riw[3 + j]; Ria[6 + j] = -Riw[6 + j]; }
  quat_from_rot(Ria, &imu[0]);
  rot_tmul(Riw, S.angvel, &imu[4]);
  rot_tmul(Riw, acc, &imu[7]);
  const float praw[3] = {acc[0], acc[1], acc[2] + 9.81f};
  rot_tmul(Riw, praw, &imu[10]);
}

// BulletInterface::cycle (BulletInterface.cpp:228-250): read_joint_sensors, read_imu, send_commands - torques from the
// readings just taken, tau_max = min(maximum_torque, URDF effort), no joint friction (:278-352) - and one
// stepSimulation. `stopped`: the servos are in moteus kStopped mode (locked joints, zero torque).
template <typename AnyFn, typename SyncFn>
UPKIE_HD void spine_cycle(const SimParams& P, RobotState& S, SpineLag& L, const float a[UPKIE_ACT_DIM], bool stopped,
                          const float* eps, float mu, AnyFn warp_any, SyncFn phase_sync, int limits,
                          BodyRecOut rec = BodyRecOut{nullptr, 0}, int env = -1) {
#pragma unroll
  for (int k = 0; k < 18; ++k) L.rep2[k] = L.rep1[k];
  spine_read_imu(P, S, L.imu);
  // torque_control_kp / kd of the config or of the env's row of the parameter table (env < 0: no table reads, as in
  // servo_substep)
  const bool table = env >= 0 && P.env_params != nullptr;
  const float kp_env = table ? env_param(P, env, UPKIE_EP_KP) : P.kp;
  const float kd_env = table ? env_param(P, env, UPKIE_EP_KD) : P.kd;
  float tau[6];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const float* aj = a + j * 6;
    const float kp = aj[UPKIE_ACT_KP_SCALE] * kp_env, kd = aj[UPKIE_ACT_KD_SCALE] * kd_env;
    const float tau_max = fminf(aj[UPKIE_ACT_MAXIMUM_TORQUE], P.tau_max[j]);
    float t = aj[UPKIE_ACT_FEEDFORWARD_TORQUE] + kd * (aj[UPKIE_ACT_VELOCITY] - S.qd[j]);
    const float tp = aj[UPKIE_ACT_POSITION];
    if (!(tp != tp)) t += kp * (tp - S.q[j]);
    t = fmaxf(fminf(t, tau_max), -tau_max);
    if (stopped) t = 0.f;
    tau[j] = t;
    S.torque[j] = t;
    L.rep1[3 * j + 0] = S.q[j];
    L.rep1[3 * j + 1] = S.qd[j];
    L.rep1[3 * j + 2] = t;
  }
  substep(P, S, tau, eps, mu, warp_any, phase_sync, nullptr, limits, stopped, rec);
}

// the observation cycle_actuation assembles before it cycles the simulator (Spine.cpp:185-200)
UPKIE_HD void spine_assemble_observation(const RobotState& S, SpineLag& L) {
#pragma unroll
  for (int k = 0; k < 18; ++k) L.obs_rep[k] = L.rep2[k];
#pragma unroll
  for (int k = 0; k < 13; ++k) L.obs_imu[k] = L.imu[k];
#pragma unroll
  for (int k = 0; k < 4; ++k) L.obs_base[k] = S.quat[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) { L.obs_base[4 + k] = S.linvel[k]; L.obs_base[7 + k] = S.angvel[k]; }
  L.obs_contact = S.contact;
}

// BulletInterface::reset (BulletInterface.cpp:129-163): base pose, velocities (the body-frame angular velocity rotated
// to the world frame), joint angles; the IMU's previous velocity restarts from the reset state; no simulation step
UPKIE_HD void reset_pose_spine(const SimParams& P, RobotState& S, const float init[UPKIE_INIT_DIM], SpineLag& L) {
  reset_pose(S, init);
  float R[9], wb[3] = {S.angvel[0], S.angvel[1], S.angvel[2]}, rp[3], w[3];
  quat_to_rot(S.quat, R);
  rot_mul(R, wb, S.angvel);
  rot_mul(R, P.imu_pos, rp);
  cross3(S.angvel, rp, w);
#pragma unroll
  for (int i = 0; i < 3; ++i) S.prev_imu_vel[i] = S.linvel[i] + w[i];
#pragma unroll
  for (int j = 0; j < 6; ++j) S.torque[j] = 0.f;
#pragma unroll
  for (int k = 0; k < 18; ++k) { L.rep1[k] = 0.f; L.rep2[k] = 0.f; L.obs_rep[k] = 0.f; }
#pragma unroll
  for (int k = 0; k < 13; ++k) { L.imu[k] = 0.f; L.obs_imu[k] = 0.f; }
#pragma unroll
  for (int k = 0; k < 10; ++k) L.obs_base[k] = 0.f;
  L.obs_contact = 0.f;
}

// Spine::simulate in State::kReset (Spine.cpp:119-125): three cycles with the servos stopped (zero torques, so no
// env's gains enter and spine_cycle reads no parameter table); the observation handed to the agent is the one the
// third cycle assembled
template <typename AnyFn>
UPKIE_HD void reset_robot_spine(const SimParams& P, RobotState& S, SpineLag& L, const float init[UPKIE_INIT_DIM],
                                const float* eps, float mu, AnyFn warp_any, int limits,
                                BodyRecOut rec = BodyRecOut{nullptr, 0}) {
  reset_pose_spine(P, S, init, L);
  float a[UPKIE_ACT_DIM];
#pragma unroll
  for (int k = 0; k < UPKIE_ACT_DIM; ++k) a[k] = 0.f;
  for (int c = 0; c < 3; ++c) {
    if (c == 2) spine_assemble_observation(S, L);
    spine_cycle(P, S, L, a, true, eps, mu, warp_any, NoSync(), limits, c == 2 ? rec : BodyRecOut{nullptr, 0});
  }
  reset_wrapper_state(S);
}

// spine observation row [UPKIE_SPINE_DIM] from the assembled observation of the lag record
UPKIE_HD void spine_observation_from_lag(const SimParams& P, const SpineLag& L, float* o) {
  float R[9];
  quat_to_rot(L.obs_base, R);
  float om_b[3];
  rot_tmul(R, &L.obs_base[7], om_b);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    o[UPKIE_SP_BASE_ANGVEL + i] = om_b[i];
    o[UPKIE_SP_BASE_LINVEL + i] = L.obs_base[4 + i];
  }
  o[UPKIE_SP_PITCH] = asinf(clampf(2.f * (L.obs_base[0] * L.obs_base[2] - L.obs_base[3] * L.obs_base[1]), -1.f, 1.f));
#pragma unroll
  for (int i = 0; i < 9; ++i) o[UPKIE_SP_ROT + i] = R[i];
#pragma unroll
  for (int k = 0; k < 4; ++k) o[UPKIE_SP_IMU_QUAT + k] = L.obs_imu[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    o[UPKIE_SP_IMU_ANGVEL + k] = L.obs_imu[4 + k];
    o[UPKIE_SP_IMU_LINACC + k] = L.obs_imu[7 + k];
    o[UPKIE_SP_IMU_RAWACC + k] = L.obs_imu[10 + k];
  }
  o[UPKIE_SP_CONTACT] = L.obs_contact;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    float* so = o + UPKIE_SP_SERVO + j * UPKIE_OBS_KEYS;
    so[UPKIE_OBS_POSITION] = L.obs_rep[3 * j];
    so[UPKIE_OBS_VELOCITY] = L.obs_rep[3 * j + 1];
    so[UPKIE_OBS_TORQUE] = L.obs_rep[3 * j + 2];
    so[UPKIE_OBS_TEMPERATURE] = 20.0f;  // BulletInterface.cpp:70
    so[UPKIE_OBS_VOLTAGE] = 18.0f;
  }
  const float signed_radius = P.left_sign * P.wheel_radius;
  o[UPKIE_SP_ODOM_POS] = 0.5f * (L.obs_rep[3 * 2] - L.obs_rep[3 * 5]) * signed_radius;
  o[UPKIE_SP_ODOM_VEL] = 0.5f * (L.obs_rep[3 * 2 + 1] - L.obs_rep[3 * 5 + 1]) * signed_radius;
}

UPKIE_HD void lag_from_row(const float* r, SpineLag& L) {
#pragma unroll
  for (int k = 0; k < 18; ++k) { L.rep1[k] = r[UPKIE_LAG_REPLY1 + k]; L.rep2[k] = r[UPKIE_LAG_REPLY2 + k]; L.obs_rep[k] = r[UPKIE_LAG_OBS_REPLY + k]; }
#pragma unroll
  for (int k = 0; k < 13; ++k) { L.imu[k] = r[UPKIE_LAG_IMU + k]; L.obs_imu[k] = r[UPKIE_LAG_OBS_IMU + k]; }
#pragma unroll
  for (int k = 0; k < 10; ++k) L.obs_base[k] = r[UPKIE_LAG_OBS_BASE + k];
  L.obs_contact = r[UPKIE_LAG_OBS_CONTACT];
}
UPKIE_HD void lag_to_row(const SpineLag& L, float* r) {
#pragma unroll
  for (int k = 0; k < 18; ++k) { r[UPKIE_LAG_REPLY1 + k] = L.rep1[k]; r[UPKIE_LAG_REPLY2 + k] = L.rep2[k]; r[UPKIE_LAG_OBS_REPLY + k] = L.obs_rep[k]; }
#pragma unroll
  for (int k = 0; k < 13; ++k) { r[UPKIE_LAG_IMU + k] = L.imu[k]; r[UPKIE_LAG_OBS_IMU + k] = L.obs_imu[k]; }
#pragma unroll
  for (int k = 0; k < 10; ++k) r[UPKIE_LAG_OBS_BASE + k] = L.obs_base[k];
  r[UPKIE_LAG_OBS_CONTACT] = L.obs_contact;
}

// ---- counter-based RNG (Philox4x32-10) for on-device init-state sampling and noise ----
struct Philox4 { uint32_t v[4]; };

UPKIE_HD void mulhilo32(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
  const uint64_t p = uint64_t(a) * uint64_t(b);
  hi = uint32_t(p >> 32);
  lo = uint32_t(p);
}

UPKIE_HD Philox4 philox4x32_10(uint64_t counter_lo, uint64_t counter_hi, uint64_t key) {
  uint32_t c0 = uint32_t(counter_lo), c1 = uint32_t(counter_lo >> 32), c2 = uint32_t(counter_hi), c3 = uint32_t(counter_hi >> 32);
  uint32_t k0 = uint32_t(key), k1 = uint32_t(key >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, lo0, hi1, lo1;
    mulhilo32(0xD2511F53u, c0, hi0, lo0);
    mulhilo32(0xCD9E8D57u, c2, hi1, lo1);
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  Philox4 out;
  out.v[0] = c0; out.v[1] = c1; out.v[2] = c2; out.v[3] = c3;
  return out;
}

// uniform in [0, 1) with 24 bits
UPKIE_HD float u01(uint32_t x) { return float(x >> 8) * (1.0f / 16777216.0f); }

UPKIE_HD void gaussian8(uint64_t seed, const NoiseCtx& nz, uint32_t slot, float out[8]) {
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const Philox4 r = philox4x32_10(nz.env, (uint64_t(nz.tick) << 10) | (uint64_t(slot) << 1) | uint64_t(b),
                                    seed ^ 0x6E6F697365ull);
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const float u1 = (float(r.v[2 * p] >> 8) + 1.0f) * (1.0f / 16777216.0f);  // (0, 1]
      const float u2 = u01(r.v[2 * p + 1]);
      const float rad = sqrtf(-2.0f * logf(u1));
      float sn, cs;
      sincosf(6.28318530718f * u2, &sn, &cs);
      out[4 * b + 2 * p] = rad * cs;
      out[4 * b + 2 * p + 1] = rad * sn;
    }
  }
}

// ImuUncertainty::apply on the IMU part of a spine observation (BulletInterface.cpp:252-258): bias plus
// white noise on the filtered acceleration and the angular velocity, and with independent draws on the
// raw acceleration. One draw per env tick, repeatable (slots 254 / 253 of the tick's generator). `env`: the robot's
// column of the per-env parameter table, whose IMU columns replace the config's when it is set (env < 0: no table
// reads, as in servo_substep).
UPKIE_HD void apply_imu_uncertainty(const SimParams& P, const NoiseCtx& nz, float* o, int env = -1) {
  if (!P.any_imu_uncertainty) return;
  float g1[8], g2[8];
  gaussian8(P.noise_seed, nz, 254u, g1);
  gaussian8(P.noise_seed, nz, 253u, g2);
  const bool table = env >= 0 && P.env_params != nullptr;
  const float acc_noise = table ? env_param(P, env, UPKIE_EP_IMU_ACC_NOISE) : P.imu_acc_noise;
  const float gyro_noise = table ? env_param(P, env, UPKIE_EP_IMU_GYRO_NOISE) : P.imu_gyro_noise;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float acc_bias = table ? env_param(P, env, UPKIE_EP_IMU_ACC_BIAS + k) : P.imu_acc_bias[k];
    const float gyro_bias = table ? env_param(P, env, UPKIE_EP_IMU_GYRO_BIAS + k) : P.imu_gyro_bias[k];
    o[UPKIE_SP_IMU_LINACC + k] += acc_bias + acc_noise * g1[k];
    o[UPKIE_SP_IMU_ANGVEL + k] += gyro_bias + gyro_noise * g1[3 + k];
    o[UPKIE_SP_IMU_RAWACC + k] += acc_bias + acc_noise * g2[k];
  }
}

// observed torques: commanded torque + measurement noise (pybullet_backend.py:457-466); the standard deviations of
// the config or of the env's row (`env`, < 0: never a table, see servo_substep) of the parameter table, or `meas_sd`
// when `own` (a lane that redrew its row in this launch: the values in force, in registers)
UPKIE_HD void measured_torques(const SimParams& P, const RobotState& S, const NoiseCtx* nz, float out[6],
                               int env = -1, const float* meas_sd = nullptr, bool own = false) {
  float noise[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const bool draw = P.any_meas_noise && nz;
  if (draw) gaussian8(P.noise_seed, *nz, 255u, noise);
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const float sd = (draw && own) ? meas_sd[j]
                     : (draw && env >= 0 && P.env_params) ? env_param(P, env, UPKIE_EP_MEAS_NOISE + j)
                                                          : P.meas_noise[j];
    out[j] = S.torque[j] + (sd > 1e-10f ? noise[j] * sd : 0.f);
  }
}

// RobotState.sample_state (robot_state.py:175-196) with a counter-based
// generator keyed on (seed, global env index, episode): same draw order as the
// reference (angular velocity, linear velocity, ZYX euler, position).
UPKIE_HD void sample_init_state(const SimParams& P, uint64_t seed, uint64_t env_index, uint64_t episode,
                                float init[UPKIE_INIT_DIM]) {
  float u[12];
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    const Philox4 r = philox4x32_10(env_index, (episode << 2) | uint64_t(b), seed);
#pragma unroll
    for (int i = 0; i < 4; ++i) u[4 * b + i] = u01(r.v[i]);
  }
  auto uni = [](float x, float lo, float hi) { return lo + (hi - lo) * x; };
  const float om[3] = {uni(u[0], -P.rand_omega_x, P.rand_omega_x), uni(u[1], -P.rand_omega_y, P.rand_omega_y), 0.f};
  const float v[3] = {uni(u[3], -P.rand_linvel[0], P.rand_linvel[0]), uni(u[4], -P.rand_linvel[1], P.rand_linvel[1]),
                      uni(u[5], -P.rand_linvel[2], P.rand_linvel[2])};
  const float pitch = uni(u[7], -P.rand_pitch, P.rand_pitch);
  const float roll = uni(u[8], -P.rand_roll, P.rand_roll);
  const float px = uni(u[9], -P.rand_x, P.rand_x);
  const float pz = uni(u[11], 0.f, P.rand_z);
  // ZYX euler [0, pitch, roll] -> quaternion qy(pitch) * qx(roll)
  float sp, cp, sr, cr;
  sincosf(0.5f * pitch, &sp, &cp);
  sincosf(0.5f * roll, &sr, &cr);
  const float qr[4] = {cp * cr, cp * sr, sp * cr, -sp * sr};
  const float* a = P.init_quat;
  init[UPKIE_INIT_QUAT + 0] = a[0] * qr[0] - a[1] * qr[1] - a[2] * qr[2] - a[3] * qr[3];
  init[UPKIE_INIT_QUAT + 1] = a[0] * qr[1] + a[1] * qr[0] + a[2] * qr[3] - a[3] * qr[2];
  init[UPKIE_INIT_QUAT + 2] = a[0] * qr[2] - a[1] * qr[3] + a[2] * qr[0] + a[3] * qr[1];
  init[UPKIE_INIT_QUAT + 3] = a[0] * qr[3] + a[1] * qr[2] - a[2] * qr[1] + a[3] * qr[0];
  init[UPKIE_INIT_POS + 0] = P.init_pos[0] + px;
  init[UPKIE_INIT_POS + 1] = P.init_pos[1];
  init[UPKIE_INIT_POS + 2] = P.init_pos[2] + pz;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    // nominal + random part (robot_state.py:113-135 sample_angular_velocity / sample_linear_velocity)
    init[UPKIE_INIT_LINVEL + i] = P.init_linvel[i] + v[i];
    init[UPKIE_INIT_ANGVEL + i] = P.init_angvel[i] + om[i];
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    init[UPKIE_INIT_Q + j] = P.init_q[j];  // joint configuration is not randomised (robot_state.py:183)
    init[UPKIE_INIT_QD + j] = 0.f;         // resetJointState zeroes the rates (pybullet_backend.py:262-267)
  }
}

// ---- reset randomisation (upkie_b200_set_reset_randomization) ----
// The handle's device block: the spec and the buffers a reset writes its draw to. Its pointers stay valid while the
// spec is set (the handle refuses to drop those buffers then).
struct ResetRand {
  UpkieResetRandomization spec;
  uint32_t* draws;  // [n] draws so far per env
  float* table;     // [UPKIE_EP_DIM][stride] the per-env parameter table
  int stride;
  float* eps;       // [n][6] inertia epsilons
  float* mu;        // [n] floor friction
};

// bit 63 of the high counter word: never set by sample_init_state ((episode << 2) | b, episode < 2^32) or the noise
// ((tick << 10) | (slot << 1) | b, tick < 2^32)
constexpr uint64_t kResetRandTag = uint64_t(1) << 63;

// Draw `draw` (1, 2, ...) of the env of global index `env_index`: all UPKIE_RR_DIM columns, whatever is selected, so
// that selecting a column never changes another one's value. The product is rounded on its own (no FMA), so that a
// NumPy statement in fp32 reproduces it bit for bit.
UPKIE_HD void reset_rand_draw(const UpkieResetRandomization& R, uint64_t seed, uint64_t env_index, uint32_t draw,
                              float v[UPKIE_RR_DIM]) {
#pragma unroll 1
  for (int b = 0; b < (UPKIE_RR_DIM + 3) / 4; ++b) {
    const Philox4 r = philox4x32_10(env_index, kResetRandTag | (uint64_t(draw) << 4) | uint64_t(b), seed);
    for (int k = 0; k < 4 && 4 * b + k < UPKIE_RR_DIM; ++k) {
      const int c = 4 * b + k;
      const float lo = R.low[c], hi = R.high[c];
#if defined(__CUDA_ARCH__)
      const float span = __fmul_rn(hi - lo, u01(r.v[k]));
#else
      const float span = (hi - lo) * u01(r.v[k]);  // ISO C++ mode: g++ does not contract this into an FMA
#endif
      v[c] = fminf(lo + span, hi);
    }
  }
}

// Env i's draw `v`, stored into the selected columns of the table / eps / mu, and its number into the counter
UPKIE_HD void reset_rand_store(const ResetRand& R, int i, const float v[UPKIE_RR_DIM]) {
  R.draws[i] += 1u;
  const uint64_t cols = R.spec.columns;
  for (int k = 0; k < UPKIE_EP_DIM; ++k)
    if ((cols >> k) & 1u) R.table[size_t(k) * size_t(R.stride) + size_t(i)] = v[k];
  for (int b = 0; b < 6; ++b)
    if ((cols >> (UPKIE_RR_INERTIA + b)) & 1u) R.eps[size_t(i) * 6 + b] = v[UPKIE_RR_INERTIA + b];
  if ((cols >> UPKIE_RR_FRICTION) & 1u) R.mu[i] = v[UPKIE_RR_FRICTION];
}

// Env i's next draw (number draws[i] + 1) into v, then stored (`store` false: a tail lane shadowing another env,
// which stores nothing). A caller that reads the buffers again in the same launch keeps the values it uses from v
// instead (the step kernels: reset_rand_draw, then reset_rand_store at the end of the tick).
UPKIE_HD void reset_randomize(const ResetRand& R, uint64_t seed, uint64_t env_index, int i, bool store,
                              float v[UPKIE_RR_DIM]) {
  reset_rand_draw(R.spec, seed, env_index, R.draws[i] + 1u, v);
  if (store) reset_rand_store(R, i, v);
}

// ---- push randomisation (upkie_b200_set_push_randomization) ----
// The handle's device block: the spec and the per-env schedule state (include/upkie_b200.h): count[i] = k, the draw in
// force, and timer[i] = steps taken since it was made, 0 .. gap + duration.
struct PushRand {
  UpkiePushRandomization spec;
  uint32_t* count;
  uint32_t* timer;
};

// bit 62 of the high counter word: never set by sample_init_state ((episode << 2) | b, episode < 2^32), the noise
// ((tick << 10) | (slot << 1) | b) or the reset randomisation (bit 63 set)
constexpr uint64_t kPushTag = uint64_t(1) << 62;

// an integer of [lo, hi] from the top 24 bits of a word, exact (hi - lo <= UPKIE_PUSH_MAX_STEPS, so no overflow)
UPKIE_HD uint32_t push_steps(uint32_t w, uint32_t lo, uint32_t hi) {
  return lo + uint32_t((uint64_t(w >> 8) * uint64_t(hi - lo + 1u)) >> 24);
}

// a value of [lo, hi] as reset_rand_draw draws one: the product rounded on its own (no FMA)
UPKIE_HD float push_value(uint32_t w, float lo, float hi) {
#if defined(__CUDA_ARCH__)
  const float span = __fmul_rn(hi - lo, u01(w));
#else
  const float span = (hi - lo) * u01(w);  // ISO C++ mode: g++ does not contract this into an FMA
#endif
  return fminf(lo + span, hi);
}

// Draw k of the env of global index g: its gap and duration, and block 0, which also holds words 2 and 3 of the force
struct PushDraw {
  uint32_t gap, duration;
  Philox4 r0;
};
UPKIE_HD PushDraw push_draw(const UpkiePushRandomization& s, uint64_t seed, uint64_t g, uint32_t k) {
  PushDraw d;
  d.r0 = philox4x32_10(g, kPushTag | (uint64_t(k) << 4), seed);
  d.gap = push_steps(d.r0.v[0], s.gap_low, s.gap_high);
  d.duration = push_steps(d.r0.v[1], s.duration_low, s.duration_high);
  return d;
}

// the force of draw k (words 2, 3 of block 0 and word 0 of block 1)
UPKIE_HD void push_force(const UpkiePushRandomization& s, uint64_t seed, uint64_t g, uint32_t k, const PushDraw& d,
                         float f[3]) {
  const Philox4 r1 = philox4x32_10(g, kPushTag | (uint64_t(k) << 4) | 1u, seed);
  f[0] = push_value(d.r0.v[2], s.force_low[0], s.force_high[0]);
  f[1] = push_value(d.r0.v[3], s.force_low[1], s.force_high[1]);
  f[2] = push_value(r1.v[0], s.force_low[2], s.force_high[2]);
}

// One counted step of an env's schedule: (k, t) before the step -> after it, the push of the step in f (zero when not
// pushed), and `end` = gap + duration of the draw in force after the step. A push that ran out at the last step
// (t = gap + duration) starts draw k + 1 here.
UPKIE_HD void push_step(const UpkiePushRandomization& s, uint64_t seed, uint64_t g, uint32_t& k, uint32_t& t,
                        uint32_t& end, float f[3]) {
  PushDraw d = push_draw(s, seed, g, k);
  if (t >= d.gap + d.duration) {
    k += 1u;
    t = 0u;
    d = push_draw(s, seed, g, k);
  }
  t += 1u;
  end = d.gap + d.duration;
  f[0] = 0.f; f[1] = 0.f; f[2] = 0.f;
  if (t > d.gap) push_force(s, seed, g, k, d, f);
}

// A reset of an env whose draw in force has gap + duration = end: the next draw, after the +1 of a push that ran out
UPKIE_HD void push_restart(uint32_t& k, uint32_t& t, uint32_t end) {
  k += t >= end ? 2u : 1u;
  t = 0u;
}

// The push force env state (k, t) says was applied in the last step (upkie_b200_get_push_forces)
UPKIE_HD void push_last_force(const UpkiePushRandomization& s, uint64_t seed, uint64_t g, uint32_t k, uint32_t t,
                              float f[3]) {
  const PushDraw d = push_draw(s, seed, g, k);
  f[0] = 0.f; f[1] = 0.f; f[2] = 0.f;
  if (t > d.gap && t <= d.gap + d.duration) push_force(s, seed, g, k, d, f);
}

// An explicit reset of env i (k_reset, upkie_b200_reset)
UPKIE_HD void push_reset(const PushRand& R, uint64_t seed, uint64_t g, int i) {
  const PushDraw d = push_draw(R.spec, seed, g, R.count[i]);
  uint32_t k = R.count[i], t = R.timer[i];
  push_restart(k, t, d.gap + d.duration);
  R.count[i] = k;
  R.timer[i] = t;
}

// ---- action-delay randomisation (upkie_b200_set_action_delay) ----
// The handle's device block: the spec and the per-env state (include/upkie_b200.h): count[i] = k, the number of the
// env's last draw, delay[i] = d_i in substeps, and command = the servo command of each env's previous tick,
// [UPKIE_ACT_DIM][stride] structure-of-arrays like the state, env i in column i.
struct ActionDelay {
  UpkieActionDelay spec;
  uint32_t* count;
  uint32_t* delay;
  float* command;
  int stride;
  // the history depth K (upkie_b200_set_action_delay_ticks; 0 acts as 1): command holds K rows [K][UPKIE_ACT_DIM][stride]
  // of the env's last K ticks, a ring whose next write is row head[i] (read by the K > 1 branch only)
  int ticks;
  uint32_t* head;
};

// bit 61 of the high counter word: never set by sample_init_state ((episode << 2) | b, episode < 2^32), the noise
// ((tick << 10) | (slot << 1) | b, tick < 2^32), the reset randomisation (bit 63 set) or the pushes (bit 62 set)
constexpr uint64_t kActionDelayTag = uint64_t(1) << 61;

// Draw k of the env of global index g: its delay in substeps, push_steps' exact integer form
UPKIE_HD uint32_t action_delay_draw(const UpkieActionDelay& s, uint64_t seed, uint64_t g, uint32_t k) {
  const Philox4 r = philox4x32_10(g, kActionDelayTag | (uint64_t(k) << 4), seed);
  return push_steps(r.v[0], s.substeps_low, s.substeps_high);
}

// The previous command an env holds after a reset: servos stopped, {position NaN, velocity 0, feedforward 0, kp_scale 0,
// kd_scale 0, maximum_torque 0} per joint. joint_torque clips last, to [-0, 0]: the torque is exactly zero whatever
// the state, friction and torque-control noise.
UPKIE_HD float action_delay_stop_value(int k) { return (k % UPKIE_ACT_KEYS) == UPKIE_ACT_POSITION ? nanf("") : 0.f; }

// The command of substep `sub` of a tick with delay d, in `a`: the tick enters its substeps with the previous command in
// `a`, and substep d (never reached for d >= nb_substeps) first replaces it with this tick's, load(c) for c = 0 ..
// UPKIE_ACT_DIM - 1. The step kernels load it back from the command buffer, so that only one row is held in registers.
template <typename Load>
UPKIE_HD void action_delay_substep(int sub, uint32_t d, float a[UPKIE_ACT_DIM], Load load) {
  if (uint32_t(sub) == d) {
#pragma unroll
    for (int c = 0; c < UPKIE_ACT_DIM; ++c) a[c] = load(c);
  }
}

// ---- delays of more than one tick (a history of K ticks, upkie_b200_set_*_delay_ticks) ----
// A delay of d substeps, clamped to K * nb, as whole ticks q and a part r of a tick: d = q * nb + r with 0 <= q < K and
// 1 <= r <= nb (q = r = 0 for d = 0). r = nb is the whole tick, which the one-tick kernels already run (the action
// delay switches at no substep, the observation delay snapshots the start of the tick), so a delay of at most nb
// substeps is q = 0 and the one-tick rule itself.
struct DelaySplit {
  uint32_t q, r;
};
UPKIE_HD DelaySplit delay_split(uint32_t d, uint32_t nb, uint32_t ticks) {
  const uint32_t cap = ticks * nb;
  const uint32_t dd = d < cap ? d : cap;
  const uint32_t q = dd ? (dd - 1u) / nb : 0u;
  return {q, dd - q * nb};
}

// The ring row of age `age` (0 the newest) of a history of K rows whose next write is row `head`
UPKIE_HD uint32_t delay_ring_row(uint32_t head, uint32_t ticks, uint32_t age) { return (head + ticks - 1u - age) % ticks; }

// The ring rows of one tick of an action delay d with a history of K ticks whose next write is row `head`: the tick
// enters its substeps with the command of row `first` (age q: tick t - q - 1), then stores this tick's command into row
// `head` (age K - 1, the oldest, read first when q = K - 1), and substep r loads the command of tick t - q from row
// `second` (the row just stored for q = 0). The next tick writes row (head + 1) % K.
struct ActionDelayRows {
  uint32_t first, second, r;
};
UPKIE_HD ActionDelayRows action_delay_rows(uint32_t d, uint32_t nb, uint32_t ticks, uint32_t head) {
  const DelaySplit s = delay_split(d, nb, ticks);
  return {delay_ring_row(head, ticks, s.q), (head + ticks - s.q) % ticks, s.r};
}

// The ring rows of one tick of an observation delay d with a history of K ticks whose next write is row `head`: the
// snapshot of substep nb - r goes into row `head` and differentiates its IMU velocity against row `newest` (age 0, the
// last tick's), and after the tick the step reports row `report` (age q of the ring with this tick's snapshot in it).
struct ObsDelayRows {
  uint32_t newest, report, r;
};
UPKIE_HD ObsDelayRows obs_delay_rows(uint32_t d, uint32_t nb, uint32_t ticks, uint32_t head) {
  const DelaySplit s = delay_split(d, nb, ticks);
  return {delay_ring_row(head, ticks, 0u), (head + ticks - s.q) % ticks, s.r};
}

// A reset of env i (the step kernels' fused resets, k_reset): the next draw, and the stop row as the
// previous command. The block's fields are copied before the first store, which the compiler cannot tell apart from
// the block itself.
UPKIE_HD void action_delay_reset(const ActionDelay& A, uint64_t seed, uint64_t g, int i) {
  const UpkieActionDelay spec = A.spec;
  uint32_t* const count = A.count;
  uint32_t* const delay = A.delay;
  float* const col = A.command + size_t(i);
  const size_t stride = size_t(A.stride);
  const uint32_t k = count[i] + 1u;
  count[i] = k;
  delay[i] = action_delay_draw(spec, seed, g, k);
  for (int c = 0; c < UPKIE_ACT_DIM; ++c) col[size_t(c) * stride] = action_delay_stop_value(c);
}

// With a history of K > 1 ticks, after action_delay_reset: the stop row as the other K - 1 commands too
UPKIE_HD void action_delay_fill_history(const ActionDelay& A, int i) {
  float* const col = A.command + size_t(i);
  const size_t stride = size_t(A.stride);
  for (int c = UPKIE_ACT_DIM; c < A.ticks * UPKIE_ACT_DIM; ++c) col[size_t(c) * stride] = action_delay_stop_value(c);
}

// ---- observation-delay randomisation (upkie_b200_set_observation_delay) ----
// The handle's device block: the spec and the per-env state (include/upkie_b200.h): count[i] = k, the number of the
// env's last draw, delay[i] = d_i in substeps, and rows = the sensed state of each env, [UPKIE_STATE_DIM][stride]
// structure-of-arrays like the state, env i in column i: what the env's sensors report, the state whose observation
// the step returns and upkie_b200_spine_obs reads.
struct ObsDelay {
  UpkieObservationDelay spec;
  uint32_t* count;
  uint32_t* delay;
  float* rows;
  int stride;
  // the history depth K (upkie_b200_set_observation_delay_ticks; 0 acts as 1). K > 1: hist holds the snapshots of the
  // env's last K ticks [K][UPKIE_STATE_DIM][stride], a ring whose next write is row head[i]; `rows` is then a copy of
  // the sensed columns of the snapshot the last step reported
  int ticks;
  float* hist;
  uint32_t* head;
};

// bit 60 of the high counter word: never set by sample_init_state ((episode << 2) | b, episode < 2^32), the noise
// ((tick << 10) | (slot << 1) | b, tick < 2^32), the reset randomisation (bit 63), the pushes (bit 62) or the action
// delay (bit 61)
constexpr uint64_t kObsDelayTag = uint64_t(1) << 60;

// Draw k of the env of global index g: its delay in substeps, push_steps' exact integer form
UPKIE_HD uint32_t obs_delay_draw(const UpkieObservationDelay& s, uint64_t seed, uint64_t g, uint32_t k) {
  const Philox4 r = philox4x32_10(g, kObsDelayTag | (uint64_t(k) << 4), seed);
  return push_steps(r.v[0], s.substeps_low, s.substeps_high);
}

// Whether column k of a state row is sensed (delayed): base pose and twist, joint positions and velocities, the IMU
// velocity of the last snapshot, the commanded torques, the floor contact and the IMU acceleration. The others (leg
// targets, yaw, yaw velocity: the gyropod wrapper's software state; the contact impulses) are the true state's.
UPKIE_HD constexpr bool obs_delay_sensed(int k) {
  return k < UPKIE_ST_LEG_TARGET || k == UPKIE_ST_CONTACT || (k >= UPKIE_ST_IMU_ACC && k < UPKIE_ST_IMU_ACC + 3);
}

// The world-frame velocity of the IMU of state S (what observe_update differentiates)
UPKIE_HD void imu_velocity(const SimParams& P, const RobotState& S, float v[3]) {
  float R[9];
  quat_to_rot(S.quat, R);
  float rp[3], w[3];
  rot_mul(R, P.imu_pos, rp);
  cross3(S.angvel, rp, w);
#pragma unroll
  for (int i = 0; i < 3; ++i) v[i] = S.linvel[i] + w[i];
}

// A reset of env i (the step kernels' fused resets, k_reset): the next draw. The caller then copies the
// post-reset state into the sensed row. The block's fields are copied before the first store, as action_delay_reset.
UPKIE_HD void obs_delay_reset(const ObsDelay& O, uint64_t seed, uint64_t g, int i) {
  const UpkieObservationDelay spec = O.spec;
  uint32_t* const count = O.count;
  uint32_t* const delay = O.delay;
  const uint32_t k = count[i] + 1u;
  count[i] = k;
  delay[i] = obs_delay_draw(spec, seed, g, k);
}

// A reset of env i with a history of K > 1 ticks: every snapshot of the ring becomes the post-reset state row r
UPKIE_HD void obs_delay_fill_history(const ObsDelay& O, int i, const float r[UPKIE_STATE_DIM]) {
  float* const col = O.hist + size_t(i);
  const size_t stride = size_t(O.stride);
  for (int s = 0; s < O.ticks; ++s)
    for (int k = 0; k < UPKIE_STATE_DIM; ++k) col[(size_t(s) * UPKIE_STATE_DIM + k) * stride] = r[k];
}

// ---- spine-rate observation history (upkie_b200_set_history, HistoryObserver.h) ----
// The handle's device block: the spec and the ring. ring [ticks][count][stride], env i in column i: each entry holds
// the `count` selected columns of the env's spine observation after one substep, and head[i] is the entry the env's
// next substep writes. Every step moves every env's head on by nb_substeps, a resetting env's included (its reset
// refills the whole ring), and nothing else moves them: all envs sit on the same entry, and a warp's stores are
// coalesced rows (the rule of delay_ring_advance).
struct History {
  int size;    // K, the entries a read reports
  int count;   // C, the columns of an entry
  int ticks;   // entries of the ring: K + (the observation delay's depth) * nb_substeps
  int stride;
  int acc;     // 1: some column is an IMU acceleration, which the substeps differentiate
  int columns[UPKIE_MAX_HISTORY_CHANNELS];
  float* ring;
  uint32_t* head;
};

// Whether spine column `col` is an IMU acceleration (linear or raw)
UPKIE_HD constexpr bool history_acc_column(int col) {
  return col >= UPKIE_SP_IMU_LINACC && col < UPKIE_SP_IMU_RAWACC + 3;
}

// t[k] of a short array for a runtime k, as unrolled selects (an indexed read would put the array in local memory)
template <int N>
UPKIE_HD float history_pick(const float (&t)[N], int k) {
  float v = t[0];
#pragma unroll
  for (int j = 1; j < N; ++j) v = k == j ? t[j] : v;
  return v;
}

// Column `col` of the spine observation of S (spine_observation's arithmetic, that column only), with `acc` as the
// IMU acceleration and the commanded torques without measurement noise
UPKIE_HD float history_value(const SimParams& P, const RobotState& S, const float acc[3], int col) {
  if (col >= UPKIE_SP_BASE_LINVEL && col < UPKIE_SP_PITCH) return history_pick(S.linvel, col - UPKIE_SP_BASE_LINVEL);
  if (col == UPKIE_SP_PITCH) return base_pitch(S);
  if (col == UPKIE_SP_CONTACT) return S.contact;
  if (col >= UPKIE_SP_SERVO && col < UPKIE_SP_ODOM_POS) {
    const int j = (col - UPKIE_SP_SERVO) / UPKIE_OBS_KEYS, key = (col - UPKIE_SP_SERVO) % UPKIE_OBS_KEYS;
    if (key == UPKIE_OBS_POSITION) return history_pick(S.q, j);
    if (key == UPKIE_OBS_VELOCITY) return history_pick(S.qd, j);
    if (key == UPKIE_OBS_TORQUE) return history_pick(S.torque, j);
    return key == UPKIE_OBS_TEMPERATURE ? 42.0f : 18.0f;
  }
  const float signed_radius = P.left_sign * P.wheel_radius;
  if (col == UPKIE_SP_ODOM_POS) return 0.5f * (S.q[2] - S.q[5]) * signed_radius;
  if (col == UPKIE_SP_ODOM_VEL) return 0.5f * (S.qd[2] - S.qd[5]) * signed_radius;
  float R[9];
  quat_to_rot(S.quat, R);
  if (col < UPKIE_SP_BASE_LINVEL) {
    float om_b[3];
    rot_tmul(R, S.angvel, om_b);
    return history_pick(om_b, col - UPKIE_SP_BASE_ANGVEL);
  }
  if (col < UPKIE_SP_IMU_QUAT) return history_pick(R, col - UPKIE_SP_ROT);
  float Riw[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      Riw[3 * i + j] = R[3 * i + 0] * P.Rbi[3 * j + 0] + R[3 * i + 1] * P.Rbi[3 * j + 1] + R[3 * i + 2] * P.Rbi[3 * j + 2];
  if (col < UPKIE_SP_IMU_ANGVEL) {
    float Ria[9];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      Ria[j] = Riw[j];
      Ria[3 + j] = -Riw[3 + j];
      Ria[6 + j] = -Riw[6 + j];
    }
    float q[4];
    quat_from_rot(Ria, q);
    return history_pick(q, col - UPKIE_SP_IMU_QUAT);
  }
  float t[3];
  if (col < UPKIE_SP_IMU_LINACC) {
    rot_tmul(Riw, S.angvel, t);
    return history_pick(t, col - UPKIE_SP_IMU_ANGVEL);
  }
  if (col < UPKIE_SP_IMU_RAWACC) {
    rot_tmul(Riw, acc, t);
    return history_pick(t, col - UPKIE_SP_IMU_LINACC);
  }
  const float praw[3] = {acc[0], acc[1], acc[2] + 9.81f};
  rot_tmul(Riw, praw, t);
  return history_pick(t, col - UPKIE_SP_IMU_RAWACC);
}

// One entry of env i's ring, `e`: the columns of S with IMU acceleration `acc`, column(c) the spine column of channel c
// (the CPU build's record of a substep; the step kernels' history_substep stores the same values)
template <typename Column>
UPKIE_HD void history_store(const History& H, const SimParams& P, const RobotState& S, const float acc[3], uint32_t e,
                            int i, Column column) {
  float* const col = H.ring + size_t(e) * size_t(H.count) * size_t(H.stride) + size_t(i);
  for (int c = 0; c < H.count; ++c) col[size_t(c) * size_t(H.stride)] = history_value(P, S, acc, column(c));
}

// A reset of env i (both fused auto-resets, k_reset), a new spec or a state set: every entry of the ring becomes the
// columns of S, the IMU acceleration that of the state (what the observation of S reports)
UPKIE_HD void history_fill(const History& H, const SimParams& P, const RobotState& S, int i) {
  float* const col = H.ring + size_t(i);
  const size_t stride = size_t(H.stride), entry = size_t(H.count) * stride;
  for (int c = 0; c < H.count; ++c) {
    const float v = history_value(P, S, S.imu_acc, H.columns[c]);
    for (int e = 0; e < H.ticks; ++e) col[size_t(e) * entry + size_t(c) * stride] = v;
  }
}

// The ring entry of history entry k (0 the newest) of an env whose next write is entry `head`, observed `d` substeps
// before the end of the tick (the observation delay in force; 0 without one)
UPKIE_HD uint32_t history_entry(uint32_t head, uint32_t ticks, uint32_t d, uint32_t k) {
  return (head + 2u * ticks - 1u - d - k) % ticks;
}

// ---- servo reply dropouts (upkie_b200_set_servo_dropout, observe_servos.cpp:32-52) ----
// The handle's device block: the spec and the per-env state (include/upkie_b200.h): count[i] = k, the number of the
// env's last draw, prob[i] = p_i, and held = the latched [joint][position, velocity, torque] of each env,
// [kServoHeldRows][stride] structure-of-arrays like the state, env i in column i.
constexpr int kServoHeldRows = 18;
struct ServoDropout {
  UpkieServoDropout spec;
  uint32_t* count;
  float* prob;
  float* held;
  int stride;
};

// bit 59 of the high counter word, the per-reset draws of p_i: never set by sample_init_state ((episode << 2) | b,
// episode < 2^32), the noise ((tick << 10) | (slot << 1) | b, tick < 2^32), the reset randomisation (bit 63), the
// pushes (bit 62), the action delay (bit 61) or the observation delay (bit 60), whose draw numbers stay below bit 36.
// Bits 59 and 58 together: the per-cycle losses, (tick << 20) | (sub << 1) | b below bit 52.
constexpr uint64_t kServoDropoutTag = uint64_t(1) << 59;
constexpr uint64_t kServoLossTag = kServoDropoutTag | (uint64_t(1) << 58);

// Draw k of the env of global index g: its loss probability, push_value's exact form
UPKIE_HD float servo_dropout_draw(const UpkieServoDropout& s, uint64_t seed, uint64_t g, uint32_t k) {
  const Philox4 r = philox4x32_10(g, kServoDropoutTag | (uint64_t(k) << 4), seed);
  return push_value(r.v[0], s.prob_low, s.prob_high);
}

// The servos of `mask` whose reply is lost in substep `sub` of the env's tick `tick` (bit j: servo j), each with
// probability p. A block of four servos none of which may lose a reply, or p <= 0, draws nothing.
UPKIE_HD uint32_t servo_dropout_lost(uint32_t mask, float p, uint64_t seed, uint64_t g, uint32_t tick, uint32_t sub) {
  uint32_t lost = 0;
  if (!(p > 0.f)) return lost;
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    if (!((mask >> (4 * b)) & 0xFu)) continue;
    const Philox4 r = philox4x32_10(g, kServoLossTag | (uint64_t(tick) << 20) | (uint64_t(sub) << 1) | uint64_t(b), seed);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = 4 * b + k;
      if (j < UPKIE_NJ && ((mask >> j) & 1u) && u01(r.v[k]) < p) lost |= 1u << j;
    }
  }
  return lost;
}

// One spine cycle: the servos of `mask` whose reply was not lost (`lost`) latch their triple after the substep,
// store(row, value). The held rows then always hold each masked servo's last received triple.
template <typename Store>
UPKIE_HD void servo_dropout_hold(const RobotState& S, uint32_t mask, uint32_t lost, Store store) {
#pragma unroll
  for (int j = 0; j < UPKIE_NJ; ++j) {
    if (!((mask >> j) & 1u) || ((lost >> j) & 1u)) continue;
    store(3 * j, S.q[j]);
    store(3 * j + 1, S.qd[j]);
    store(3 * j + 2, S.torque[j]);
  }
}

// The observed state of S at an instant whose replies `lost` lost: those servos report their held triple, load(row)
template <typename Load>
UPKIE_HD void servo_dropout_view(RobotState& S, uint32_t lost, Load load) {
#pragma unroll
  for (int j = 0; j < UPKIE_NJ; ++j) {
    if (!((lost >> j) & 1u)) continue;
    S.q[j] = load(3 * j);
    S.qd[j] = load(3 * j + 1);
    S.torque[j] = load(3 * j + 2);
  }
}

// A reset of env i (the step kernels' fused resets, k_reset): the next draw, and the post-reset state S latched. The
// block's fields are copied before the first store, as action_delay_reset.
UPKIE_HD void servo_dropout_reset(const ServoDropout& D, uint64_t seed, uint64_t g, int i, const RobotState& S) {
  const UpkieServoDropout spec = D.spec;
  uint32_t* const count = D.count;
  float* const prob = D.prob;
  float* const col = D.held + size_t(i);
  const size_t stride = size_t(D.stride);
  const uint32_t k = count[i] + 1u;
  count[i] = k;
  prob[i] = servo_dropout_draw(spec, seed, g, k);
  servo_dropout_hold(S, ~0u, 0u, [&](int r, float v) { col[size_t(r) * stride] = v; });
}

// ---- IMU mounting misalignment (upkie_b200_set_imu_misalignment, BaseOrientation.h:29-35,106-112) ----
// The handle's device block: the spec and the per-env state (include/upkie_b200.h): count[i] = k, the number of the
// env's last draw, and quat = the unit quaternion e_i (w, x, y, z) of the env's misalignment, a rotation in the base
// frame, [4][stride] structure-of-arrays like the state, env i in column i.
struct ImuMisalign {
  UpkieImuMisalignment spec;
  uint32_t* count;
  float* quat;
  int stride;
};

// bit 57 of the high counter word, the per-reset draws of e_i: never set by sample_init_state (below 2^34), the noise
// (below bit 42), the reset randomisation (bit 63), the pushes (62), the action delay (61), the observation delay (60)
// or the servo dropouts (59, and 59 | 58), whose draw numbers stay below bit 36
constexpr uint64_t kImuMisalignTag = uint64_t(1) << 57;

struct Quat4 {
  float q[4];  // w, x, y, z
};

// The unit quaternion of Rz(yaw) Ry(pitch) Rx(roll)
UPKIE_HD Quat4 imu_misalign_quat(float roll, float pitch, float yaw) {
  const float cr = cosf(0.5f * roll), sr = sinf(0.5f * roll);
  const float cp = cosf(0.5f * pitch), sp = sinf(0.5f * pitch);
  const float cy = cosf(0.5f * yaw), sy = sinf(0.5f * yaw);
  Quat4 e;
  e.q[0] = cr * cp * cy + sr * sp * sy;
  e.q[1] = sr * cp * cy - cr * sp * sy;
  e.q[2] = cr * sp * cy + sr * cp * sy;
  e.q[3] = cr * cp * sy - sr * sp * cy;
  return e;
}

// Draw k of the env of global index g: words 0, 1, 2 give roll, pitch and yaw, push_value's exact form (the map of the
// servo dropouts), and the result is the quaternion of the misalignment they make
UPKIE_HD Quat4 imu_misalign_draw(const UpkieImuMisalignment& s, uint64_t seed, uint64_t g, uint32_t k) {
  const Philox4 r = philox4x32_10(g, kImuMisalignTag | (uint64_t(k) << 4), seed);
  return imu_misalign_quat(push_value(r.v[0], s.roll_low, s.roll_high), push_value(r.v[1], s.pitch_low, s.pitch_high),
                           push_value(r.v[2], s.yaw_low, s.yaw_high));
}

// The observed state of S under the misalignment e: its base orientation becomes R E (quat <- quat (x) e), so that
// every orientation-derived observation is that of an IMU tilted by E while the pipeline assumes the nominal mounting.
// Nothing else changes: the twist is world-frame and the IMU acceleration of the state is world-frame too. The identity
// leaves S bit for bit (the product would turn a -0 component into +0); returns whether S changed.
UPKIE_HD bool imu_misalign_view(RobotState& S, const Quat4& e) {
  if (e.q[1] == 0.f && e.q[2] == 0.f && e.q[3] == 0.f) return false;
  const float w = S.quat[0], x = S.quat[1], y = S.quat[2], z = S.quat[3];
  S.quat[0] = w * e.q[0] - x * e.q[1] - y * e.q[2] - z * e.q[3];
  S.quat[1] = w * e.q[1] + x * e.q[0] + y * e.q[3] - z * e.q[2];
  S.quat[2] = w * e.q[2] - x * e.q[3] + y * e.q[0] + z * e.q[1];
  S.quat[3] = w * e.q[3] + x * e.q[2] - y * e.q[1] + z * e.q[0];
  return true;
}

// Env i's misalignment, load(row) of its column
template <typename Load>
UPKIE_HD Quat4 imu_misalign_load(Load load) {
  Quat4 e;
#pragma unroll
  for (int r = 0; r < 4; ++r) e.q[r] = load(r);
  return e;
}

// A reset of env i (the step kernels' fused resets, k_reset): the next draw, stored; the new e_i. The block's fields
// are copied before the first store, as servo_dropout_reset.
UPKIE_HD Quat4 imu_misalign_reset(const ImuMisalign& M, uint64_t seed, uint64_t g, int i) {
  const UpkieImuMisalignment spec = M.spec;
  uint32_t* const count = M.count;
  float* const col = M.quat + size_t(i);
  const size_t stride = size_t(M.stride);
  const uint32_t k = count[i] + 1u;
  count[i] = k;
  const Quat4 e = imu_misalign_draw(spec, seed, g, k);
#pragma unroll
  for (int r = 0; r < 4; ++r) col[size_t(r) * stride] = e.q[r];
  return e;
}

// ---- Servo encoder zero offsets (upkie_b200_set_encoder_offset, pi3hat_spine.cpp:181-236) ----
// The handle's device block: the spec and the per-env state (include/upkie_b200.h): count[i] = k, the number of the
// env's last draw, and offset = delta_i, the encoder zero offset of each joint in radians, [UPKIE_NJ][stride]
// structure-of-arrays like the state, env i in column i.
struct EncoderOffset {
  UpkieEncoderOffset spec;
  uint32_t* count;
  float* offset;
  int stride;
};

// bit 56 of the high counter word, the per-reset draws of delta_i, (k << 4) | b below bit 36: never set by
// sample_init_state (below 2^34), the noise (below bit 42), the reset randomisation (bit 63), the pushes (62), the
// action delay (61), the observation delay (60), the servo dropouts (59, and 59 | 58, below bit 52 otherwise) or the
// IMU misalignment (57)
constexpr uint64_t kEncoderOffsetTag = uint64_t(1) << 56;

struct Offset6 {
  float d[UPKIE_NJ];
};

// Draw k of the env of global index g: word j % 4 of the block of counter j / 4 gives joint j's offset, push_value's
// exact form (the map of the servo dropouts). Every joint's word is drawn whatever the mask, and a joint outside it
// gets 0, so that the mask changes no other joint's draw.
UPKIE_HD Offset6 encoder_offset_draw(const UpkieEncoderOffset& s, uint64_t seed, uint64_t g, uint32_t k) {
  Offset6 o;
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const Philox4 r = philox4x32_10(g, kEncoderOffsetTag | (uint64_t(k) << 4) | uint64_t(b), seed);
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const int j = 4 * b + w;
      if (j < UPKIE_NJ) o.d[j] = ((s.joint_mask >> j) & 1u) ? push_value(r.v[w], s.low, s.high) : 0.f;
    }
  }
  return o;
}

// The observed state of S under the offsets d: every servo reports its position in its own frame, q_j + delta_j.
// A zero offset leaves q_j bit for bit (the sum would turn a -0 into +0). Returns whether a wheel position changed (the
// odometry that the gyropod and pendulum rows report).
UPKIE_HD bool encoder_offset_view(RobotState& S, const Offset6& d) {
#pragma unroll
  for (int j = 0; j < UPKIE_NJ; ++j)
    if (d.d[j] != 0.f) S.q[j] += d.d[j];
  return d.d[2] != 0.f || d.d[5] != 0.f;
}

// The position targets of the servo command `a` (servo frame, after clamp_servo_action) as the joints execute them,
// target - delta_j. A NaN target stays NaN; a zero offset leaves the target as it is.
UPKIE_HD void encoder_offset_command(float a[UPKIE_ACT_DIM], const Offset6& d) {
#pragma unroll
  for (int j = 0; j < UPKIE_NJ; ++j)
    if (d.d[j] != 0.f) a[j * UPKIE_ACT_KEYS + UPKIE_ACT_POSITION] -= d.d[j];
}

// The gyropod and pendulum leg targets a reset sets (reset_wrapper_state: the true hip and knee positions) made the
// reported ones, q + delta: the wrapper holds servo-frame targets
UPKIE_HD void encoder_offset_leg_targets(RobotState& S, const Offset6& d) {
  const int leg_joint[4] = {0, 1, 3, 4};
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (d.d[leg_joint[k]] != 0.f) S.leg_target[k] += d.d[leg_joint[k]];
}

// Env i's offsets, load(row) of its column
template <typename Load>
UPKIE_HD Offset6 encoder_offset_load(Load load) {
  Offset6 o;
#pragma unroll
  for (int j = 0; j < UPKIE_NJ; ++j) o.d[j] = load(j);
  return o;
}

// A reset of env i (the step kernels' fused resets, k_reset): the next draw, stored; the new delta_i. The block's
// fields are copied before the first store, as servo_dropout_reset.
UPKIE_HD Offset6 encoder_offset_reset(const EncoderOffset& E, uint64_t seed, uint64_t g, int i) {
  const UpkieEncoderOffset spec = E.spec;
  uint32_t* const count = E.count;
  float* const col = E.offset + size_t(i);
  const size_t stride = size_t(E.stride);
  const uint32_t k = count[i] + 1u;
  count[i] = k;
  const Offset6 o = encoder_offset_draw(spec, seed, g, k);
#pragma unroll
  for (int j = 0; j < UPKIE_NJ; ++j) col[size_t(j) * stride] = o.d[j];
  return o;
}

// ---- Servo measurement noise (upkie_b200_set_servo_noise, observe_servos.cpp:62-75) ----
// The handle's device block: the spec and the per-env state (include/upkie_b200.h): count[i] = k, the number of the
// env's last draw; sigma = the standard deviations of env i, [12][stride] structure-of-arrays like the state (rows 0-5
// position, 6-11 velocity), env i in column i; fresh[i] = 1 while the observation env i reports is its reset
// observation (set by a reset, cleared by a step that does not reset), which k_spine_obs and k_reset_obs key on.
constexpr int kServoNoiseCols = 2 * UPKIE_NJ;
struct ServoNoise {
  UpkieServoNoise spec;
  uint32_t* count;
  float* sigma;
  uint8_t* fresh;
  int stride;
};

// bit 55 of the high counter word: the per-reset draws of sigma_i, (k << 4) | b below bit 36; with bit 54, the cycles
// of a step, (t << 20) | (s << 2) | b below bit 52; with bits 54 and 53, the reset observations, (k << 2) | b with the
// env's draw counter k after the reset (every reset advances it, whether it samples its state or takes host rows).
// Never set by sample_init_state (below 2^34), the noise (below bit 42), the reset randomisation (bit 63), the pushes
// (62), the action delay (61), the observation delay (60), the servo dropouts (59, and 59 | 58 below bit 52), the IMU
// misalignment (57), the encoder offsets (56) or the velocity limits (52).
constexpr uint64_t kServoNoiseTag = uint64_t(1) << 55;
constexpr uint64_t kServoNoiseCycleTag = kServoNoiseTag | (uint64_t(1) << 54);
constexpr uint64_t kServoNoiseResetTag = kServoNoiseCycleTag | (uint64_t(1) << 53);

// The counter word (b = 0) of cycle s of tick t, and of the observation of the reset that made draw k
UPKIE_HD uint64_t servo_noise_cycle(uint32_t t, uint32_t s) {
  return kServoNoiseCycleTag | (uint64_t(t) << 20) | (uint64_t(s) << 2);
}
UPKIE_HD uint64_t servo_noise_reset_cycle(uint32_t k) { return kServoNoiseResetTag | (uint64_t(k) << 2); }

// The cycle `age` cycles before cycle nb - 1 of tick t (an observation delay of `age` substeps, an older history entry):
// cycle t * nb + nb - 1 - age of the env's count of cycles, floored into its tick (modulo 2^32 ticks)
UPKIE_HD uint64_t servo_noise_cycle_before(uint32_t t, uint32_t nb, uint32_t age) {
  const uint32_t back = age / nb, s = nb - 1u - age % nb;  // cycle s of tick t - back
  return servo_noise_cycle(t - back, s);
}

// Draw k of the env of global index g: column c from word c % 4 of the block of counter c / 4 (push_value's exact form,
// the map of the servo dropouts). Every column is drawn whatever the ranges.
struct Sigma12 {
  float s[kServoNoiseCols];
};
UPKIE_HD Sigma12 servo_noise_draw(const UpkieServoNoise& spec, uint64_t seed, uint64_t g, uint32_t k) {
  Sigma12 o;
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    const Philox4 r = philox4x32_10(g, kServoNoiseTag | (uint64_t(k) << 4) | uint64_t(b), seed);
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const int c = 4 * b + w;
      const float lo = c < UPKIE_NJ ? spec.position_low[c] : spec.velocity_low[c - UPKIE_NJ];
      const float hi = c < UPKIE_NJ ? spec.position_high[c] : spec.velocity_high[c - UPKIE_NJ];
      o.s[c] = push_value(r.v[w], lo, hi);
    }
  }
  return o;
}

// The twelve standard normals of the cycle of counter word `cycle`: gaussian8's Box-Muller transform on the words of
// three Philox blocks, normal c from block c / 4
UPKIE_HD void servo_noise_normals(uint64_t seed, uint64_t g, uint64_t cycle, float n[kServoNoiseCols]) {
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    const Philox4 r = philox4x32_10(g, cycle | uint64_t(b), seed);
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const float u1 = (float(r.v[2 * p] >> 8) + 1.0f) * (1.0f / 16777216.0f);  // (0, 1]
      const float u2 = u01(r.v[2 * p + 1]);
      const float rad = sqrtf(-2.0f * logf(u1));
      float sn, cs;
      sincosf(6.28318530718f * u2, &sn, &cs);
      n[4 * b + 2 * p] = rad * cs;
      n[4 * b + 2 * p + 1] = rad * sn;
    }
  }
}

// What the noise adds to each reported value of one cycle, sigma * n rounded on its own (never contracted into the
// sum it enters); exactly 0 where sigma is 0. An env whose sigmas are all zero draws nothing.
struct Noise12 {
  float d[kServoNoiseCols];
};
UPKIE_HD float servo_noise_mul(float s, float n) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(s, n);
#else
  return s * n;  // ISO C++ mode: g++ does not contract this into an FMA
#endif
}
template <typename Load>
UPKIE_HD Noise12 servo_noise_increments(Load sigma, uint64_t seed, uint64_t g, uint64_t cycle) {
  Noise12 o;
  bool any = false;
#pragma unroll
  for (int c = 0; c < kServoNoiseCols; ++c) {
    o.d[c] = sigma(c);
    any = any || o.d[c] != 0.f;
  }
  if (!any) return o;
  float n[kServoNoiseCols];
  servo_noise_normals(seed, g, cycle, n);
#pragma unroll
  for (int c = 0; c < kServoNoiseCols; ++c) o.d[c] = o.d[c] != 0.f ? servo_noise_mul(o.d[c], n[c]) : 0.f;
  return o;
}

// The reported state of S under the increments d: q_j + d_j, qd_j + d_{6+j}. A zero increment leaves the value bit for
// bit. Returns whether a wheel's position or velocity changed (the odometry that the gyropod and pendulum rows report).
UPKIE_HD bool servo_noise_view(RobotState& S, const Noise12& d) {
#pragma unroll
  for (int j = 0; j < UPKIE_NJ; ++j) {
    if (d.d[j] != 0.f) S.q[j] += d.d[j];
    if (d.d[UPKIE_NJ + j] != 0.f) S.qd[j] += d.d[UPKIE_NJ + j];
  }
  return d.d[2] != 0.f || d.d[5] != 0.f || d.d[UPKIE_NJ + 2] != 0.f || d.d[UPKIE_NJ + 5] != 0.f;
}

// The gyropod and pendulum leg targets a reset sets (reset_wrapper_state: the true hip and knee positions) made the
// reported ones of the reset observation: applied before encoder_offset_leg_targets, in the order of the view
UPKIE_HD void servo_noise_leg_targets(RobotState& S, const Noise12& d) {
  const int leg_joint[4] = {0, 1, 3, 4};
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (d.d[leg_joint[k]] != 0.f) S.leg_target[k] += d.d[leg_joint[k]];
}

// A reset of env i (the step kernels' fused resets, k_reset): the next draw, stored, and the env marked as reporting
// its reset observation; returns the draw's number k, which keys that observation's cycle. The block's fields are
// copied before the first store, as servo_dropout_reset.
UPKIE_HD uint32_t servo_noise_reset(const ServoNoise& N, uint64_t seed, uint64_t g, int i) {
  const UpkieServoNoise spec = N.spec;
  uint32_t* const count = N.count;
  float* const col = N.sigma + size_t(i);
  uint8_t* const fresh = N.fresh;
  const size_t stride = size_t(N.stride);
  const uint32_t k = count[i] + 1u;
  count[i] = k;
  const Sigma12 o = servo_noise_draw(spec, seed, g, k);
#pragma unroll
  for (int c = 0; c < kServoNoiseCols; ++c) col[size_t(c) * stride] = o.s[c];
  fresh[i] = 1;
  return k;
}

// Whether spine column `col` reports a servo position or velocity, or the wheel odometry built from them
UPKIE_HD constexpr bool history_noise_column(int col) {
  return (col >= UPKIE_SP_SERVO && col < UPKIE_SP_ODOM_POS &&
          ((col - UPKIE_SP_SERVO) % UPKIE_OBS_KEYS == UPKIE_OBS_POSITION ||
           (col - UPKIE_SP_SERVO) % UPKIE_OBS_KEYS == UPKIE_OBS_VELOCITY)) ||
         col == UPKIE_SP_ODOM_POS || col == UPKIE_SP_ODOM_VEL;
}

// A ring filled under servo noise (a reset, a new spec or a state set): every entry holds the columns of S with the
// noise of the cycle it stands for, the newest (age 0) cycle `newest`, the entry of age a >= 1 the cycle a substeps
// before cycle nb - 1 of tick t; `view` then reads the copy through the other views. `head` is the env's next write.
template <typename Sigma, typename View, typename Store>
UPKIE_HD void history_fill_noise(const History& H, const SimParams& P, const RobotState& S, uint32_t head, Sigma sigma,
                                 uint64_t seed, uint64_t g, uint64_t newest, uint32_t t, View view, Store store) {
  const uint32_t ticks = uint32_t(H.ticks);
  for (uint32_t a = 0; a < ticks; ++a) {
    RobotState V = S;
    const uint64_t cyc = a == 0 ? newest : servo_noise_cycle_before(t, uint32_t(P.nb_substeps), a);
    servo_noise_view(V, servo_noise_increments(sigma, seed, g, cyc));
    view(V);
    const uint32_t e = (head + 2u * ticks - 1u - a) % ticks;
    for (int c = 0; c < H.count; ++c) store(e, c, history_value(P, V, V.imu_acc, H.columns[c]));
  }
}

// ---- Servo velocity limits: the draws (upkie_b200_set_velocity_derate; the block and the law above servo_substep) ----
// bit 52 of the high counter word, the per-reset draws of v_i, (k << 4) | b below bit 36: never set by
// sample_init_state (below 2^34), the noise (below bit 42), the reset randomisation (bit 63), the pushes (62), the
// action delay (61), the observation delay (60), the servo dropouts (59, and 59 | 58, below bit 52 otherwise), the IMU
// misalignment (57), the encoder offsets (56), the servo noise (55, 55 | 54 below bit 52, and 55 | 54 | 53), the
// attitude filter (51 alone) or the torque scales (50 alone)
constexpr uint64_t kVelocityDerateTag = uint64_t(1) << 52;

struct Vmax6 {
  float v[UPKIE_NJ];
};

// Draw k of the env of global index g: word j % 4 of the block of counter j / 4 gives joint j's limit, push_value's
// exact form (the map of the servo dropouts). Every joint's word is drawn whatever the mask, and a joint outside it
// gets 0, so that the mask changes no other joint's draw.
UPKIE_HD Vmax6 velocity_derate_draw(const UpkieVelocityDerate& s, uint64_t seed, uint64_t g, uint32_t k) {
  Vmax6 o;
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const Philox4 r = philox4x32_10(g, kVelocityDerateTag | (uint64_t(k) << 4) | uint64_t(b), seed);
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const int j = 4 * b + w;
      if (j < UPKIE_NJ)
        o.v[j] = ((s.joint_mask >> j) & 1u) ? push_value(r.v[w], s.max_velocity_low[j], s.max_velocity_high[j]) : 0.f;
    }
  }
  return o;
}

// A reset of env i (the step kernels' fused resets, k_reset): the next draw, stored. The block's fields are copied
// before the first store, as servo_dropout_reset.
UPKIE_HD void velocity_derate_reset(const VelocityDerate& V, uint64_t seed, uint64_t g, int i) {
  const UpkieVelocityDerate spec = V.spec;
  uint32_t* const count = V.count;
  float* const col = V.max_velocity + size_t(i);
  const size_t stride = size_t(V.stride);
  const uint32_t k = count[i] + 1u;
  count[i] = k;
  const Vmax6 o = velocity_derate_draw(spec, seed, g, k);
#pragma unroll
  for (int j = 0; j < UPKIE_NJ; ++j) col[size_t(j) * stride] = o.v[j];
}

// ---- Servo torque-constant errors: the draws (upkie_b200_set_torque_scale; the block and the law above servo_substep) ----
// bit 50 of the high counter word alone, the per-reset draws of s_i, (k << 4) | b below bit 36: never set by
// sample_init_state (below 2^34) or the noise (below bit 42); every other tag sets a bit above 50 (the reset
// randomisation 63, the pushes 62, the action delay 61, the observation delay 60, the servo dropouts 59 and 59 | 58, the
// IMU misalignment 57, the encoder offsets 56, the servo noise 55, 55 | 54 and 55 | 54 | 53, the velocity limits 52,
// the attitude filter 51)
constexpr uint64_t kTorqueScaleTag = uint64_t(1) << 50;

// Draw k of the env of global index g: word j % 4 of the block of counter j / 4 gives joint j's scale, push_value's
// exact form (the map of the servo dropouts). Every joint's word is drawn whatever the mask, and a joint outside it
// gets exactly 1, so that the mask changes no other joint's draw.
UPKIE_HD Scale6 torque_scale_draw(const UpkieTorqueScale& s, uint64_t seed, uint64_t g, uint32_t k) {
  Scale6 o;
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const Philox4 r = philox4x32_10(g, kTorqueScaleTag | (uint64_t(k) << 4) | uint64_t(b), seed);
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const int j = 4 * b + w;
      if (j < UPKIE_NJ)
        o.s[j] = ((s.joint_mask >> j) & 1u) ? push_value(r.v[w], s.scale_low[j], s.scale_high[j]) : 1.f;
    }
  }
  return o;
}

// A reset of env i (the step kernels' fused resets, k_reset): the next draw, stored. The block's fields are copied
// before the first store, as servo_dropout_reset.
UPKIE_HD void torque_scale_reset(const TorqueScale& T, uint64_t seed, uint64_t g, int i) {
  const UpkieTorqueScale spec = T.spec;
  uint32_t* const count = T.count;
  float* const col = T.scale + size_t(i);
  const size_t stride = size_t(T.stride);
  const uint32_t k = count[i] + 1u;
  count[i] = k;
  const Scale6 o = torque_scale_draw(spec, seed, g, k);
#pragma unroll
  for (int j = 0; j < UPKIE_NJ; ++j) col[size_t(j) * stride] = o.s[j];
}

// ---- IMU attitude estimation (upkie_b200_set_attitude_filter, Pi3HatInterface.cpp:151-169) ----
// The handle's device block: the spec and the per-env state (include/upkie_b200.h), [rows][stride] structure-of-arrays
// like the state, env i in column i: count[i] = k, the number of the env's last draw; gains (kp, ki); quat, the
// estimate q_i (w, x, y, z) of the IMU-to-world rotation; bias, the gyro-bias estimate b_i. `rep` is the estimate the
// env's observation reports under an observation delay (that of the cycle observed), `vel` the world-frame IMU velocity
// of the env's last substep (scratch of the step kernels), and qbi the quaternion of rotation_base_to_imu.
struct AttitudeFilter {
  UpkieAttitudeFilter spec;
  float qbi[4];
  uint32_t* count;
  float* gains;
  float* quat;
  float* bias;
  float* rep;
  float* vel;
  int stride;
};

// bit 51 of the high counter word alone, the per-reset draws, (k << 4) below bit 36: never set by sample_init_state
// (below 2^34) or the noise (below bit 42); every other tag sets a bit above 51 (the reset randomisation 63, the pushes
// 62, the action delay 61, the observation delay 60, the servo dropouts 59 and 59 | 58, the IMU misalignment 57, the
// encoder offsets 56, the servo noise 55, 55 | 54 and 55 | 54 | 53, the velocity limits 52), except the torque
// scales' bit 50 alone, below it
constexpr uint64_t kAttitudeFilterTag = uint64_t(1) << 51;

struct AttitudeDraw {
  float kp, ki, roll, pitch;
};

// Draw k of the env of global index g: words 0 .. 3 of one block give kp, ki, roll and pitch, push_value's exact form
// (the map of the servo dropouts)
UPKIE_HD AttitudeDraw attitude_filter_draw(const UpkieAttitudeFilter& s, uint64_t seed, uint64_t g, uint32_t k) {
  const Philox4 r = philox4x32_10(g, kAttitudeFilterTag | (uint64_t(k) << 4), seed);
  return AttitudeDraw{push_value(r.v[0], s.kp_low, s.kp_high), push_value(r.v[1], s.ki_low, s.ki_high),
                      push_value(r.v[2], s.roll_low, s.roll_high), push_value(r.v[3], s.pitch_low, s.pitch_high)};
}

// p (x) q, quaternions (w, x, y, z)
UPKIE_HD void quat_mul(const float p[4], const float q[4], float r[4]) {
  r[0] = p[0] * q[0] - p[1] * q[1] - p[2] * q[2] - p[3] * q[3];
  r[1] = p[0] * q[1] + p[1] * q[0] + p[2] * q[3] - p[3] * q[2];
  r[2] = p[0] * q[2] - p[1] * q[3] + p[2] * q[0] + p[3] * q[1];
  r[3] = p[0] * q[3] + p[1] * q[2] - p[2] * q[1] + p[3] * q[0];
}

// One step of the filter (include/upkie_b200.h: the law, in this order): the estimate q and the bias estimate b of a
// filter of gains kp, ki, updated in place over a substep h from the gyro rate w_m and the specific force a_m of the
// IMU frame
UPKIE_HD void attitude_filter_step(float q[4], float b[3], float kp, float ki, float h, const float wm[3],
                                   const float am[3]) {
  const float vx = 2.f * (q[1] * q[3] - q[2] * q[0]);
  const float vy = 2.f * (q[2] * q[3] + q[1] * q[0]);
  const float vz = 1.f - 2.f * (q[1] * q[1] + q[2] * q[2]);
  float e[3] = {0.f, 0.f, 0.f};
  const float n = sqrtf(am[0] * am[0] + am[1] * am[1] + am[2] * am[2]);
  if (n > 1e-3f) {
    const float inv = 1.f / n;
    const float ux = am[0] * inv, uy = am[1] * inv, uz = am[2] * inv;
    e[0] = uy * vz - uz * vy;
    e[1] = uz * vx - ux * vz;
    e[2] = ux * vy - uy * vx;
  }
  float w[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    b[k] = b[k] - (ki * e[k]) * h;
    w[k] = (wm[k] - b[k]) + kp * e[k];
  }
  const float nw = sqrtf(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (!(nw > 0.f)) return;
  const float t = 0.5f * nw * h;
  float c, s;
  if (t < 0.25f) {
    // the series of cos t and sin t / t (truncation below 1e-8 here), free of the approximate sin / cos of fast math
    // at the small angles of one substep
    const float t2 = t * t;
    c = 1.f - t2 * (0.5f - t2 * (1.f / 24.f - t2 * (1.f / 720.f)));
    s = 0.5f * h * (1.f - t2 * (1.f / 6.f - t2 * (1.f / 120.f - t2 * (1.f / 5040.f))));
  } else {
    c = cosf(t);
    s = sinf(t) / nw;
  }
  const float d[4] = {c, s * w[0], s * w[1], s * w[2]};
  float r[4];
  quat_mul(q, d, r);
  const float inv = 1.f / sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]);
#pragma unroll
  for (int k = 0; k < 4; ++k) q[k] = r[k] * inv;
}

// The filter's inputs of the state S, whose orientation is the observed one (the IMU misalignment's view applied):
// the gyro rate w_m and the specific force a_m of the IMU frame, from the IMU velocities v (after the substep) and vp
// (after the previous one), with the env's gyro and accelerometer biases gb, ab
UPKIE_HD void attitude_filter_inputs(const SimParams& P, const AttitudeFilter& A, const RobotState& S, const float v[3],
                                     const float vp[3], const float gb[3], const float ab[3], float wm[3],
                                     float am[3]) {
  const float qbc[4] = {A.qbi[0], -A.qbi[1], -A.qbi[2], -A.qbi[3]};
  float qi[4];
  quat_mul(S.quat, qbc, qi);
  float R[9];
  quat_to_rot(qi, R);
  float f[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) f[k] = (v[k] - vp[k]) * P.inv_h;
  f[2] += 9.81f;
  rot_tmul(R, S.angvel, wm);
  rot_tmul(R, f, am);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    wm[k] += gb[k];
    am[k] += ab[k];
  }
}

// The env's IMU biases (the parameter table's columns, or the config's; zero without IMU uncertainty)
UPKIE_HD void attitude_filter_biases(const SimParams& P, int env, float gb[3], float ab[3]) {
  const bool table = env >= 0 && P.env_params != nullptr;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    gb[k] = 0.f;
    ab[k] = 0.f;
    if (P.any_imu_uncertainty) {
      gb[k] = table ? env_param(P, env, UPKIE_EP_IMU_GYRO_BIAS + k) : P.imu_gyro_bias[k];
      ab[k] = table ? env_param(P, env, UPKIE_EP_IMU_ACC_BIAS + k) : P.imu_acc_bias[k];
    }
  }
}

// The estimate of a base observed with orientation qb (the misalignment's view applied) and an estimate error
// E = Ry(pitch) Rx(roll) in the base frame: qb (x) E (x) qbi^-1
UPKIE_HD void attitude_filter_initial(const AttitudeFilter& A, const float qb[4], float roll, float pitch, float q[4]) {
  const Quat4 E = imu_misalign_quat(roll, pitch, 0.f);
  float t[4];
  quat_mul(qb, E.q, t);
  const float qbc[4] = {A.qbi[0], -A.qbi[1], -A.qbi[2], -A.qbi[3]};
  quat_mul(t, qbc, q);
}

// The estimate q taken back to the base: q (x) qbi, the orientation every orientation-derived observation reports
UPKIE_HD void attitude_filter_base(const AttitudeFilter& A, const float q[4], float qb[4]) { quat_mul(q, A.qbi, qb); }

// The base pitch of the base orientation qb (base_pitch's arithmetic)
UPKIE_HD float attitude_filter_pitch(const float qb[4]) {
  return asinf(clampf(2.f * (qb[0] * qb[2] - qb[3] * qb[1]), -1.f, 1.f));
}

// Whether spine column `col` is orientation-derived (the estimate replaces it)
UPKIE_HD constexpr bool attitude_filter_column(int col) {
  return col == UPKIE_SP_PITCH || (col >= UPKIE_SP_ROT && col < UPKIE_SP_IMU_ANGVEL);
}

// The orientation-derived columns of a spine observation o, from the base orientation qb (spine_observation's
// arithmetic, those columns only)
UPKIE_HD void attitude_filter_observation(const SimParams& P, const float qb[4], float* o) {
  RobotState T;
#pragma unroll
  for (int k = 0; k < 4; ++k) T.quat[k] = qb[k];
  o[UPKIE_SP_PITCH] = base_pitch(T);
  const float zero[3] = {0.f, 0.f, 0.f};
  for (int c = UPKIE_SP_ROT; c < UPKIE_SP_IMU_ANGVEL; ++c) o[c] = history_value(P, T, zero, c);
}

// A reset of env i (the step kernels' fused resets, k_reset): the next draw, stored, and the new episode's estimate of
// the observed post-reset state S (misalignment view applied), stored as the estimate and the report, b = 0. The
// block's fields are copied before the first store, as servo_dropout_reset.
UPKIE_HD void attitude_filter_reset(const AttitudeFilter& A, uint64_t seed, uint64_t g, int i, const RobotState& S) {
  const AttitudeFilter B = A;
  const size_t stride = size_t(B.stride);
  const uint32_t k = B.count[i] + 1u;
  B.count[i] = k;
  const AttitudeDraw d = attitude_filter_draw(B.spec, seed, g, k);
  float q[4];
  attitude_filter_initial(B, S.quat, d.roll, d.pitch, q);
  B.gains[size_t(i)] = d.kp;
  B.gains[stride + size_t(i)] = d.ki;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    B.quat[size_t(r) * stride + size_t(i)] = q[r];
    B.rep[size_t(r) * stride + size_t(i)] = q[r];
  }
#pragma unroll
  for (int r = 0; r < 3; ++r) B.bias[size_t(r) * stride + size_t(i)] = 0.f;
}

}  // namespace upkie_b200
