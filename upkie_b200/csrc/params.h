// SPDX-License-Identifier: Apache-2.0
//
// params.h -- host-side conversion of the public UpkieModel / UpkieSimConfig
// (double precision, include/upkie_b200.h) into the fp32 kernel parameter block.
#pragma once

#include <cmath>
#include <string>

#include "sim_core.cuh"

namespace upkie_b200 {

inline void default_sim_config(UpkieSimConfig* c) {
  // PyBulletBackend.__init__ defaults (upkie/envs/backends/pybullet_backend.py:55-112)
  c->dt = 1.0 / 200.0;          // UpkieServos frequency=200 (upkie/envs/upkie_servos.py:118)
  c->nb_substeps = 5;           // int(1000 * dt), pybullet_backend.py:85-87
  c->pgs_iterations = 50;       // Bullet numSolverIterations default
  c->gravity = 9.81;            // pybullet_backend.py:110
  c->torque_control_kp = 20.0;  // pybullet_backend.py:65
  c->torque_control_kd = 1.0;   // pybullet_backend.py:64
  for (int j = 0; j < UPKIE_NJ; ++j) {
    c->joint_friction[j] = 0.0;
    c->torque_control_noise[j] = 0.0;
    c->torque_measurement_noise[j] = 0.0;
  }
  for (int k = 0; k < 3; ++k) c->imu_accelerometer_bias[k] = c->imu_gyroscope_bias[k] = 0.0;
  c->imu_accelerometer_noise = c->imu_gyroscope_noise = 0.0;
  c->noise_seed = 0;
  c->linear_damping = 0.04;     // Bullet btMultiBody default
  c->angular_damping = 0.04;
  c->max_coordinate_velocity = 100.0;
  c->contact_stiffness = 30000.0;
  c->contact_damping = 1000.0;
  c->contact_breaking_threshold = 0.02;
  c->friction = 1.0;            // plane.urdf lateral_friction=1 (upkie/cpp/interfaces/bullet/plane/plane.urdf:5) x tire
  c->max_gain_scale = 5.0;      // upkie_servos.py:120
  c->fall_pitch = 1.0;          // upkie_gyropod.py:108
  c->leg_gain_scale = 1.0;
  c->max_ground_velocity = 3.0;
  c->max_yaw_velocity = 1.0;
  c->servos_fall_termination = 0;
  c->skip_action_clamps = 0;
  c->min_base_height = 0.0;
  c->pgs_tolerance = 0.0;  // deprecated, ignored (see solver_residual_threshold)
  c->warmstarting_factor = 0.0;  // off by default (Bullet's m_warmstartingFactor is 0.85; see DESIGN.md)
  c->joint_limits = 3;  // Bullet's hip / knee limit constraints ON (pybullet_backend.py:121 loadURDF): ten-row solver for warps with a robot on a bound
  c->reserved_joint_limits = 0;
  c->joint_limit_erp = 0.2;
  c->joint_limit_max_impulse = 100.0;
  c->init_position[0] = 0.0; c->init_position[1] = 0.0; c->init_position[2] = 0.6;  // upkie_env.py:87-90
  c->init_quat[0] = 1.0; c->init_quat[1] = 0.0; c->init_quat[2] = 0.0; c->init_quat[3] = 0.0;
  c->rand_roll = c->rand_pitch = c->rand_x = c->rand_z = 0.0;
  c->rand_omega_x = c->rand_omega_y = 0.0;
  for (int k = 0; k < 3; ++k) c->rand_linear_velocity[k] = 0.0;
  for (int j = 0; j < UPKIE_NJ; ++j) c->init_joint_configuration[j] = 0.0;
  for (int k = 0; k < 3; ++k) c->init_angular_velocity[k] = c->init_linear_velocity[k] = 0.0;
  c->spine_mode = 0;
  c->reserved_spine_mode = 0;
  c->body_contacts = 0;  // opt-in for batched handles (B200Backend, the single-env drop-in, turns it on): see include/upkie_b200.h
  c->reserved_body_contacts = 0;
  c->body_contact_erp = 0.2;  // btContactSolverInfo::m_erp2
  c->body_friction = 0.5;     // URDF importer default lateral friction of a link without <contact>
  c->solver_residual_threshold = 1e-7;  // PyBullet: getSolverInfo().m_leastSquaresResidualThreshold = 1e-7
  c->max_episode_steps = 0;  // no time limit (the reference leaves it to a TimeLimit wrapper, upkie_env.py:232)
  c->reserved_max_episode_steps = 0;
}

inline void default_mpc_config(UpkieMpcConfig* c) {
  // MPCBalancer.__init__ defaults (upkie/controllers/mpc_balancer.py:168-181)
  c->fall_pitch = 1.0;
  c->leg_length = 0.58;
  c->max_ground_accel = 10.0;
  c->max_ground_velocity = 3.0;
  c->nb_timesteps = 50;
  c->max_iterations = 30;
  c->sampling_period = 0.02;
  c->stage_input_cost_weight = 1e-3;
  c->stage_state_cost_weight = 1e-3;
  c->terminal_cost_weight = 1.0;
  c->gravity = 9.81;
}

// Returns 0 on success; fills `err` otherwise.
inline int make_sim_params(const UpkieModel& m, const UpkieSimConfig& c, SimParams& P, std::string& err) {
  const int expect_parent[UPKIE_NB] = {-1, 0, 1, 2, 0, 4, 5};
  for (int i = 0; i < UPKIE_NB; ++i)
    if (m.parent[i] != expect_parent[i]) {
      err = "model: kinematic tree must be base -> (hip, knee, wheel) x 2 in URDF joint order";
      return UPKIE_B200_EMODEL;
    }
  P.any_ctrl_noise = 0;
  P.any_meas_noise = 0;
  for (int j = 0; j < UPKIE_NJ; ++j) {
    const double ax = m.joint_axis[j][0], ay = m.joint_axis[j][1], az = m.joint_axis[j][2];
    if (std::fabs(ax) > 1e-9 || std::fabs(az) > 1e-9 || std::fabs(std::fabs(ay) - 1.0) > 1e-9) {
      err = "model: the kernels specialise on joint axes along +-y of the base frame (Upkie, Cookie)";
      return UPKIE_B200_EMODEL;
    }
    P.sgn[j] = ay > 0 ? 1.f : -1.f;
    for (int k = 0; k < 3; ++k) P.jo[j][k] = float(m.joint_origin[j][k]);
    P.q_lower[j] = float(m.q_lower[j]);
    P.q_upper[j] = float(m.q_upper[j]);
    P.qd_max[j] = float(m.qd_max[j]);
    P.tau_max[j] = float(m.tau_max[j]);
    P.joint_friction[j] = float(c.joint_friction[j]);
    P.ctrl_noise[j] = float(c.torque_control_noise[j]);
    P.meas_noise[j] = float(c.torque_measurement_noise[j]);
    // thresholds of the reference: noise is drawn only when sigma > 1e-10 (pybullet_backend.py:464,548)
    if (c.torque_control_noise[j] > 1e-10) P.any_ctrl_noise = 1;
    if (c.torque_measurement_noise[j] > 1e-10) P.any_meas_noise = 1;
  }
  for (int i = 0; i < UPKIE_NB; ++i) {
    if (!(m.mass[i] > 0.0)) { err = "model: body masses must be positive"; return UPKIE_B200_EMODEL; }
    P.mass[i] = float(m.mass[i]);
    for (int k = 0; k < 3; ++k) P.com[i][k] = float(m.com[i][k]);
    for (int k = 0; k < 6; ++k) P.inertia[i][k] = float(m.inertia[i][k]);
  }
  auto wheel_sym = [&](int b) {
    const double* I = m.inertia[b];
    const double* cm = m.com[b];
    return std::fabs(cm[0]) < 1e-12 && std::fabs(cm[2]) < 1e-12 && std::fabs(I[0] - I[2]) < 1e-12 &&
           std::fabs(I[3]) < 1e-12 && std::fabs(I[4]) < 1e-12 && std::fabs(I[5]) < 1e-12;
  };
  P.wheel_symmetric = (wheel_sym(3) && wheel_sym(6)) ? 1 : 0;
  P.noise_seed = c.noise_seed;
  P.any_imu_uncertainty = 0;
  for (int k = 0; k < 3; ++k) {
    P.imu_acc_bias[k] = float(c.imu_accelerometer_bias[k]);
    P.imu_gyro_bias[k] = float(c.imu_gyroscope_bias[k]);
    if (c.imu_accelerometer_bias[k] != 0.0 || c.imu_gyroscope_bias[k] != 0.0) P.any_imu_uncertainty = 1;
  }
  P.imu_acc_noise = float(c.imu_accelerometer_noise);
  P.imu_gyro_noise = float(c.imu_gyroscope_noise);
  if (c.imu_accelerometer_noise > 0.0 || c.imu_gyroscope_noise > 0.0) P.any_imu_uncertainty = 1;
  for (int k = 0; k < 3; ++k) {
    P.sgn2[k].x = P.sgn[k]; P.sgn2[k].y = P.sgn[k + 3];
    P.mass2[k].x = P.mass[k + 1]; P.mass2[k].y = P.mass[k + 4];
    float oyl = 0.f, oyr = 0.f;
    for (int kk = 0; kk <= k; ++kk) { oyl += P.jo[kk][1]; oyr += P.jo[kk + 3][1]; }
    P.oy2[k].x = oyl; P.oy2[k].y = oyr;
    for (int i = 0; i < 3; ++i) {
      P.jo2[k][i].x = P.jo[k][i]; P.jo2[k][i].y = P.jo[k + 3][i];
      P.com2[k][i].x = P.com[k + 1][i]; P.com2[k][i].y = P.com[k + 4][i];
    }
    for (int i = 0; i < 6; ++i) { P.inertia2[k][i].x = P.inertia[k + 1][i]; P.inertia2[k][i].y = P.inertia[k + 4][i]; }
  }
  if (!(m.wheel_radius > 0.0)) { err = "model: wheel_radius must be positive"; return UPKIE_B200_EMODEL; }
  P.wheel_radius = float(m.wheel_radius);
  P.half_wheel_base = float(0.5 * m.wheel_base);
  P.left_sign = m.left_wheeled ? 1.f : -1.f;
  for (int k = 0; k < 3; ++k) P.imu_pos[k] = float(m.imu_position[k]);
  for (int k = 0; k < 9; ++k) P.Rbi[k] = float(m.rotation_base_to_imu[k]);

  if (!(c.dt > 0.0) || c.nb_substeps < 1 || c.pgs_iterations < 0) {
    err = "config: dt > 0, nb_substeps >= 1, pgs_iterations >= 0 required";
    return UPKIE_B200_EINVAL;
  }
  const double h = c.dt / c.nb_substeps;
  // the base-orientation integrator's polynomials of sin(x) / x and cos(x) (sim_pair.cuh) are fp32-exact for
  // x = |w| h / 2 <= 0.6 sqrt(3) / 2: truncation below 1.4e-7 with every angular velocity component at the clamp
  if (!(h * c.max_coordinate_velocity <= 0.6)) {
    err = "config: dt / nb_substeps * max_coordinate_velocity <= 0.6 required (substep rotation of the base)";
    return UPKIE_B200_EINVAL;
  }
  P.dt = float(c.dt);
  P.inv_dt = float(1.0 / c.dt);
  P.h = float(h);
  P.inv_h = float(1.0 / h);
  P.nb_substeps = c.nb_substeps;
  P.pgs_iterations = c.pgs_iterations;
  P.res_thr = float(c.solver_residual_threshold);
  P.warm = float(c.warmstarting_factor);
  P.joint_limits = c.joint_limits < 0 ? 0 : (c.joint_limits > 3 ? 3 : c.joint_limits);
  P.limit_erp = float(c.joint_limit_erp);
  P.limit_max_impulse = float(c.joint_limit_max_impulse);
  P.skip_action_clamps = c.skip_action_clamps;
  P.gravity = float(c.gravity);
  P.kp = float(c.torque_control_kp);
  P.kd = float(c.torque_control_kd);
  P.lin_damp = float(c.linear_damping);
  P.ang_damp = float(c.angular_damping);
  P.vmax = float(c.max_coordinate_velocity);
  // Bullet btMultiBodyConstraintSolver: cfm = 1/(h k + d), erp = h k/(h k + d), cfm *= 1/h
  double denom = h * c.contact_stiffness + c.contact_damping;
  if (denom < 1.1920929e-7) denom = 1.1920929e-7;
  P.cfm = float((1.0 / denom) / h);
  P.erp = float(h * c.contact_stiffness / denom);
  P.breaking_threshold = float(c.contact_breaking_threshold);
  P.friction = float(c.friction);
  P.max_gain_scale = float(c.max_gain_scale);
  P.fall_pitch = float(c.fall_pitch);
  P.leg_gain_scale = float(c.leg_gain_scale);
  P.max_ground_velocity = float(c.max_ground_velocity);
  P.max_yaw_velocity = float(c.max_yaw_velocity);
  P.servos_fall_termination = c.servos_fall_termination;
  P.min_base_height = float(c.min_base_height);
  for (int k = 0; k < 3; ++k) P.init_pos[k] = float(c.init_position[k]);
  for (int k = 0; k < 4; ++k) P.init_quat[k] = float(c.init_quat[k]);
  P.rand_roll = float(c.rand_roll);
  P.rand_pitch = float(c.rand_pitch);
  P.rand_x = float(c.rand_x);
  P.rand_z = float(c.rand_z);
  P.rand_omega_x = float(c.rand_omega_x);
  P.rand_omega_y = float(c.rand_omega_y);
  for (int k = 0; k < 3; ++k) P.rand_linvel[k] = float(c.rand_linear_velocity[k]);
  P.spine_mode = c.spine_mode ? 1 : 0;
  if (P.spine_mode && P.joint_limits == 0) {
    err = "config: spine_mode needs joint_limits != 0 (it lives in the extras + limits kernels)";
    return UPKIE_B200_EINVAL;
  }
  // body-ground contacts: the model's collision points and the gate constants of the packed solvers
  if (m.n_collision_points < 0 || m.n_collision_points > UPKIE_MAX_COLLISION_POINTS) {
    err = "model: n_collision_points must be in [0, UPKIE_MAX_COLLISION_POINTS]";
    return UPKIE_B200_EMODEL;
  }
  P.n_bp = m.n_collision_points;
  P.n_gate_base = 0;
  for (int k = 0; k < 3; ++k) { P.gate_leg_bound[k].x = -1e30f; P.gate_leg_bound[k].y = -1e30f; }
  for (int p = 0; p < UPKIE_MAX_COLLISION_POINTS; ++p) {
    P.bp_body[p] = 0; P.bp_radius[p] = 0.f;
    for (int k = 0; k < 3; ++k) P.bp_pos[p][k] = 0.f;
    for (int k = 0; k < 4; ++k) P.gate_base[p][k] = 0.f;
  }
  for (int p = 0; p < P.n_bp; ++p) {
    const int b = m.collision_body[p];
    if (b < 0 || b >= UPKIE_NB || !(m.collision_radius[p] >= 0.0)) {
      err = "model: collision point on an unknown body or with a negative radius";
      return UPKIE_B200_EMODEL;
    }
    P.bp_body[p] = b;
    for (int k = 0; k < 3; ++k) P.bp_pos[p][k] = float(m.collision_point[p][k]);
    P.bp_radius[p] = float(m.collision_radius[p]);
    const double* cp = m.collision_point[p];
    if (b == 0) {
      float* g = P.gate_base[P.n_gate_base++];
      g[0] = P.bp_pos[p][0]; g[1] = P.bp_pos[p][1]; g[2] = P.bp_pos[p][2]; g[3] = P.bp_radius[p];
    } else {
      // a point on a leg body can be at most |point| + radius below that body's origin (1 mm of slack for fp32)
      const float bound = float(std::sqrt(cp[0] * cp[0] + cp[1] * cp[1] + cp[2] * cp[2]) + m.collision_radius[p] + 1e-3);
      const int leg = (b - 1) / 3, k = (b - 1) % 3;
      float& slot = leg == 0 ? P.gate_leg_bound[k].x : P.gate_leg_bound[k].y;
      if (bound > slot) slot = bound;
    }
  }
  P.body_contacts = (c.body_contacts != 0 && P.n_bp > 0 && P.joint_limits != 0) ? 1 : 0;
  P.body_erp = float(c.body_contact_erp);
  P.body_mu_scale = float(c.body_friction);
  for (int j = 0; j < 6; ++j) P.init_q[j] = float(c.init_joint_configuration[j]);
  for (int k = 0; k < 3; ++k) {
    P.init_angvel[k] = float(c.init_angular_velocity[k]);
    P.init_linvel[k] = float(c.init_linear_velocity[k]);
  }
  if (c.max_episode_steps < 0) {
    err = "config: max_episode_steps must be >= 0 (0 = no time limit)";
    return UPKIE_B200_EINVAL;
  }
  P.max_episode_steps = c.max_episode_steps;
  P.elapsed = nullptr;
  P.final_obs = nullptr;
  P.env_params = nullptr;
  P.env_params_stride = 0;
  P.final_gen = 0;
  P.final_state = nullptr;
  P.reset_rand = nullptr;
  P.push = nullptr;
  P.action_delay = nullptr;
  P.obs_delay = nullptr;
  P.history = nullptr;
  P.servo_dropout = nullptr;
  P.imu_misalign = nullptr;
  P.encoder_offset = nullptr;
  P.servo_noise = nullptr;
  P.velocity_derate = nullptr;
  P.attitude_filter = nullptr;
  P.torque_scale = nullptr;
  return 0;
}

// ---- per-env parameter table (upkie_b200_set_env_params) ----------------------------------------------------------
// What a row of the table (or the config) holds besides plain values: bad input, and which noise models some env needs
constexpr uint32_t kEpInvalid = 1u, kEpCtrlNoise = 2u, kEpMeasNoise = 4u, kEpImuUncertainty = 8u;

UPKIE_HD uint32_t env_row_flags(const float* r) {
  uint32_t f = 0;
  for (int k = 0; k < UPKIE_EP_DIM; ++k) {
    const bool bias = (k >= UPKIE_EP_IMU_ACC_BIAS && k < UPKIE_EP_IMU_ACC_BIAS + 3) ||
                      (k >= UPKIE_EP_IMU_GYRO_BIAS && k < UPKIE_EP_IMU_GYRO_BIAS + 3);
    if (!(fabsf(r[k]) <= 3.402823466e38f)) f |= kEpInvalid;  // NaN or infinite
    if (!bias && !(r[k] >= 0.f)) f |= kEpInvalid;           // gains, friction, standard deviations
    if (bias && r[k] != 0.f) f |= kEpImuUncertainty;
  }
  for (int j = 0; j < UPKIE_NJ; ++j) {
    // the reference's thresholds: noise is drawn only when sigma > 1e-10 (pybullet_backend.py:464,548)
    if (r[UPKIE_EP_CTRL_NOISE + j] > 1e-10f) f |= kEpCtrlNoise;
    if (r[UPKIE_EP_MEAS_NOISE + j] > 1e-10f) f |= kEpMeasNoise;
  }
  if (r[UPKIE_EP_IMU_ACC_NOISE] > 0.f || r[UPKIE_EP_IMU_GYRO_NOISE] > 0.f) f |= kEpImuUncertainty;
  return f;
}

// the config's value of column k (what every env runs without a table)
UPKIE_HD float config_env_param(const SimParams& P, int k) {
  if (k == UPKIE_EP_KP) return P.kp;
  if (k == UPKIE_EP_KD) return P.kd;
  if (k < UPKIE_EP_CTRL_NOISE) return P.joint_friction[k - UPKIE_EP_FRICTION];
  if (k < UPKIE_EP_MEAS_NOISE) return P.ctrl_noise[k - UPKIE_EP_CTRL_NOISE];
  if (k < UPKIE_EP_IMU_ACC_BIAS) return P.meas_noise[k - UPKIE_EP_MEAS_NOISE];
  if (k < UPKIE_EP_IMU_ACC_NOISE) return P.imu_acc_bias[k - UPKIE_EP_IMU_ACC_BIAS];
  if (k == UPKIE_EP_IMU_ACC_NOISE) return P.imu_acc_noise;
  if (k < UPKIE_EP_IMU_GYRO_NOISE) return P.imu_gyro_bias[k - UPKIE_EP_IMU_GYRO_BIAS];
  return P.imu_gyro_noise;
}

// the "some env has this noise" flags of a parameter block as env_row_flags bits, and back
inline uint32_t noise_flags(const SimParams& P) {
  return (P.any_ctrl_noise ? kEpCtrlNoise : 0u) | (P.any_meas_noise ? kEpMeasNoise : 0u) |
         (P.any_imu_uncertainty ? kEpImuUncertainty : 0u);
}
// The noise models a reset randomisation spec can switch on in some env: a selected noise column whose range reaches
// above 0, a selected IMU bias column with a nonzero bound. kEpInvalid: a range the spec must not hold (a bound not
// finite, low > high, low < 0 where the table needs >= 0, an inertia bound <= -1, a floor friction low < 0).
inline uint32_t reset_rand_flags(const UpkieResetRandomization& R) {
  uint32_t f = 0;
  for (int k = 0; k < UPKIE_RR_DIM; ++k) {
    const float lo = R.low[k], hi = R.high[k];
    const bool bias = (k >= UPKIE_EP_IMU_ACC_BIAS && k < UPKIE_EP_IMU_ACC_BIAS + 3) ||
                      (k >= UPKIE_EP_IMU_GYRO_BIAS && k < UPKIE_EP_IMU_GYRO_BIAS + 3);
    if (!(std::fabs(lo) <= 3.402823466e38f) || !(std::fabs(hi) <= 3.402823466e38f) || lo > hi) f |= kEpInvalid;
    if (k < UPKIE_EP_DIM && !bias && lo < 0.f) f |= kEpInvalid;
    if (k >= UPKIE_RR_INERTIA && k < UPKIE_RR_FRICTION && lo <= -1.f) f |= kEpInvalid;
    if (k == UPKIE_RR_FRICTION && lo < 0.f) f |= kEpInvalid;
    if (!((R.columns >> k) & 1u)) continue;
    if (k >= UPKIE_EP_CTRL_NOISE && k < UPKIE_EP_MEAS_NOISE && hi > 0.f) f |= kEpCtrlNoise;
    if (k >= UPKIE_EP_MEAS_NOISE && k < UPKIE_EP_IMU_ACC_BIAS && hi > 0.f) f |= kEpMeasNoise;
    if ((k == UPKIE_EP_IMU_ACC_NOISE || k == UPKIE_EP_IMU_GYRO_NOISE) && hi > 0.f) f |= kEpImuUncertainty;
    if (bias && (lo != 0.f || hi != 0.f)) f |= kEpImuUncertainty;
  }
  if (R.columns >> UPKIE_RR_DIM) f |= kEpInvalid;  // no such column
  return f;
}

// Whether a push randomisation spec holds valid ranges: a body of the model, low <= high everywhere, step bounds up to
// UPKIE_PUSH_MAX_STEPS with at least one step of push, finite forces. (The handle's own conditions, joint_limits,
// spine_mode and local_mask, are checked by upkie_b200_set_push_randomization.)
inline bool push_spec_valid(const UpkiePushRandomization& s) {
  if (s.body < 0 || s.body >= UPKIE_NB) return false;
  if (s.gap_low > s.gap_high || s.duration_low > s.duration_high || s.duration_low == 0) return false;
  if (s.gap_high > UPKIE_PUSH_MAX_STEPS || s.duration_high > UPKIE_PUSH_MAX_STEPS) return false;
  for (int a = 0; a < 3; ++a) {
    const float lo = s.force_low[a], hi = s.force_high[a];
    if (!(std::fabs(lo) <= 3.402823466e38f) || !(std::fabs(hi) <= 3.402823466e38f) || lo > hi) return false;
  }
  return true;
}

// Why a handle with parameters P refuses an action-delay spec (upkie_b200_set_action_delay), null when it takes it
// (with a history of `ticks` whole ticks, upkie_b200_set_action_delay_ticks: one tick is the call without it)
inline const char* action_delay_spec_error(const UpkieActionDelay& s, const SimParams& P, uint32_t ticks = 1) {
  if (s.substeps_low > s.substeps_high) return "set_action_delay: substeps_low > substeps_high";
  if (ticks == 1 && s.substeps_high > uint32_t(P.nb_substeps))
    return "set_action_delay: substeps_high above nb_substeps (the delay is at most one tick)";
  if (s.substeps_high > uint64_t(ticks) * uint32_t(P.nb_substeps))
    return "set_action_delay: substeps_high above max_ticks * nb_substeps (the delay is at most max_ticks ticks)";
  if (P.joint_limits == 0)
    return "set_action_delay: needs joint_limits != 0 (the delay runs in the table and body-contact kernels)";
  if (P.spine_mode) return "set_action_delay: spine_mode models the spine's own lag";
  return nullptr;
}

// Why a handle with parameters P refuses an observation-delay spec (upkie_b200_set_observation_delay), null when it
// takes it
// (with a history of `ticks` whole ticks, upkie_b200_set_observation_delay_ticks: one tick is the call without it)
inline const char* obs_delay_spec_error(const UpkieObservationDelay& s, const SimParams& P, uint32_t ticks = 1) {
  if (s.substeps_low > s.substeps_high) return "set_observation_delay: substeps_low > substeps_high";
  if (ticks == 1 && s.substeps_high > uint32_t(P.nb_substeps))
    return "set_observation_delay: substeps_high above nb_substeps (the delay is at most one tick)";
  if (s.substeps_high > uint64_t(ticks) * uint32_t(P.nb_substeps))
    return "set_observation_delay: substeps_high above max_ticks * nb_substeps (the delay is at most max_ticks ticks)";
  if (P.joint_limits == 0)
    return "set_observation_delay: needs joint_limits != 0 (the delay runs in a copy of the table kernels)";
  if (P.spine_mode) return "set_observation_delay: spine_mode models the spine's own lag";
  if (P.body_contacts) return "set_observation_delay: body_contacts has no observation-delay kernels";
  return nullptr;
}

// Why a handle with parameters P refuses a history spec (upkie_b200_set_history), null when it takes it
inline const char* history_spec_error(const UpkieHistory& s, const SimParams& P) {
  if (s.count < 1 || s.count > UPKIE_MAX_HISTORY_CHANNELS)
    return "set_history: count outside 1 .. UPKIE_MAX_HISTORY_CHANNELS";
  if (s.size < 1 || s.size > UPKIE_MAX_HISTORY) return "set_history: size outside 1 .. UPKIE_MAX_HISTORY";
  for (uint32_t c = 0; c < s.count; ++c)
    if (s.columns[c] < 0 || s.columns[c] >= UPKIE_SPINE_DIM)
      return "set_history: a column outside 0 .. UPKIE_SPINE_DIM - 1";
  if (P.joint_limits == 0)
    return "set_history: needs joint_limits != 0 (the history runs in the observation-delay kernels)";
  if (P.spine_mode) return "set_history: spine_mode reports the spine's lagged replies, which the history does not record";
  if (P.body_contacts) return "set_history: body_contacts has no observation-history kernels";
  return nullptr;
}

// Why a handle with parameters P refuses a servo-dropout spec (upkie_b200_set_servo_dropout), null when it takes it
inline const char* servo_dropout_spec_error(const UpkieServoDropout& s, const SimParams& P) {
  if (!(s.prob_low >= 0.f) || !(s.prob_low <= s.prob_high) || !(s.prob_high <= 1.f))
    return "set_servo_dropout: 0 <= prob_low <= prob_high <= 1 required";
  if (s.joint_mask == 0 || (s.joint_mask >> UPKIE_NJ) != 0)
    return "set_servo_dropout: joint_mask must select servos of bits 0 .. 5, at least one";
  if (P.joint_limits == 0)
    return "set_servo_dropout: needs joint_limits != 0 (the dropouts run in the observation-delay kernels)";
  if (P.spine_mode) return "set_servo_dropout: spine_mode reports the spine's own servo replies";
  if (P.body_contacts) return "set_servo_dropout: body_contacts has no servo-dropout kernels";
  return nullptr;
}

// Why a handle with parameters P refuses an IMU-misalignment spec (upkie_b200_set_imu_misalignment), null when it takes
// it: every bound finite, low <= high and |bound| <= pi/4 (a misalignment, not a remount)
inline const char* imu_misalignment_spec_error(const UpkieImuMisalignment& s, const SimParams& P) {
  const float b[6] = {s.roll_low, s.roll_high, s.pitch_low, s.pitch_high, s.yaw_low, s.yaw_high};
  for (int k = 0; k < 6; ++k)
    if (!(b[k] >= -0.78539816f && b[k] <= 0.78539816f))
      return "set_imu_misalignment: every bound must be finite and within [-pi/4, pi/4] radians";
  for (int k = 0; k < 6; k += 2)
    if (!(b[k] <= b[k + 1])) return "set_imu_misalignment: low <= high required for roll, pitch and yaw";
  if (P.joint_limits == 0)
    return "set_imu_misalignment: needs joint_limits != 0 (the misalignment runs in the observation-delay kernels)";
  if (P.spine_mode) return "set_imu_misalignment: spine_mode models its spine's own IMU";
  if (P.body_contacts) return "set_imu_misalignment: body_contacts has no IMU-misalignment kernels";
  return nullptr;
}

// Why a handle with parameters P refuses an encoder-offset spec (upkie_b200_set_encoder_offset), null when it takes it:
// both bounds finite, low <= high and |bound| <= 0.5 rad (a calibration error, not a remount), and a mask of joints
inline const char* encoder_offset_spec_error(const UpkieEncoderOffset& s, const SimParams& P) {
  if (!(s.low >= -0.5f && s.low <= 0.5f) || !(s.high >= -0.5f && s.high <= 0.5f))
    return "set_encoder_offset: both bounds must be finite and within [-0.5, 0.5] radians";
  if (!(s.low <= s.high)) return "set_encoder_offset: low <= high required";
  if (s.joint_mask == 0 || (s.joint_mask >> UPKIE_NJ) != 0)
    return "set_encoder_offset: joint_mask must select joints of bits 0 .. 5, at least one";
  if (P.joint_limits == 0)
    return "set_encoder_offset: needs joint_limits != 0 (the offsets run in the observation-delay kernels)";
  if (P.spine_mode) return "set_encoder_offset: spine_mode reports the spine's own servos";
  if (P.body_contacts) return "set_encoder_offset: body_contacts has no encoder-offset kernels";
  return nullptr;
}

// Why a handle with parameters P refuses a servo-noise spec (upkie_b200_set_servo_noise), null when it takes it: every
// bound finite, 0 <= low <= high, a position high of at most 0.1 rad and a velocity high of at most 5 rad/s (a sensor
// noise, not a broken encoder)
inline const char* servo_noise_spec_error(const UpkieServoNoise& s, const SimParams& P) {
  for (int j = 0; j < UPKIE_NJ; ++j) {
    if (!(s.position_low[j] >= 0.f && s.position_low[j] <= s.position_high[j] && s.position_high[j] <= 0.1f) ||
        !(s.velocity_low[j] >= 0.f && s.velocity_low[j] <= s.velocity_high[j] && s.velocity_high[j] <= 5.f))
      return "set_servo_noise: every range must be finite with 0 <= low <= high, position high <= 0.1 rad and "
             "velocity high <= 5 rad/s";
  }
  if (P.joint_limits == 0)
    return "set_servo_noise: needs joint_limits != 0 (the noise runs in the observation-delay kernels)";
  if (P.spine_mode) return "set_servo_noise: spine_mode reports the spine's own servos";
  if (P.body_contacts) return "set_servo_noise: body_contacts has no servo-noise kernels";
  if (P.obs_delay && P.servo_dropout)
    return "set_servo_noise: not with both an observation delay and servo dropouts (a delayed snapshot does not "
           "record which of its replies were held)";
  return nullptr;
}

// Why a handle with parameters P refuses a velocity-limit spec (upkie_b200_set_velocity_derate), null when it takes it:
// every bound finite, and on a joint of the mask 0 < low <= high and derate > 0
inline const char* velocity_derate_spec_error(const UpkieVelocityDerate& s, const SimParams& P) {
  if (s.joint_mask == 0 || (s.joint_mask >> UPKIE_NJ) != 0)
    return "set_velocity_derate: joint_mask must select joints of bits 0 .. 5, at least one";
  if (s.reserved != 0) return "set_velocity_derate: reserved must be 0";
  for (int j = 0; j < UPKIE_NJ; ++j) {
    if (!std::isfinite(s.max_velocity_low[j]) || !std::isfinite(s.max_velocity_high[j]) || !std::isfinite(s.derate[j]))
      return "set_velocity_derate: every bound must be finite";
    if (!((s.joint_mask >> j) & 1u)) continue;
    if (!(s.max_velocity_low[j] > 0.f && s.max_velocity_low[j] <= s.max_velocity_high[j]))
      return "set_velocity_derate: 0 < max_velocity_low <= max_velocity_high required on every joint of the mask";
    if (!(s.derate[j] > 0.f)) return "set_velocity_derate: derate > 0 required on every joint of the mask";
  }
  if (P.joint_limits == 0)
    return "set_velocity_derate: needs joint_limits != 0 (the limits run in the observation-delay kernels)";
  if (P.spine_mode) return "set_velocity_derate: spine_mode applies the spine's own torque law";
  if (P.body_contacts) return "set_velocity_derate: body_contacts has no velocity-limit kernels";
  return nullptr;
}

// Why a handle with parameters P refuses a torque-scale spec (upkie_b200_set_torque_scale), null when it takes it: every
// bound finite, and on a joint of the mask 0 < low <= high <= 2
inline const char* torque_scale_spec_error(const UpkieTorqueScale& s, const SimParams& P) {
  if (s.joint_mask == 0 || (s.joint_mask >> UPKIE_NJ) != 0)
    return "set_torque_scale: joint_mask must select joints of bits 0 .. 5, at least one";
  if (s.reserved != 0) return "set_torque_scale: reserved must be 0";
  for (int j = 0; j < UPKIE_NJ; ++j) {
    if (!std::isfinite(s.scale_low[j]) || !std::isfinite(s.scale_high[j]))
      return "set_torque_scale: every bound must be finite";
    if (!((s.joint_mask >> j) & 1u)) continue;
    if (!(s.scale_low[j] > 0.f && s.scale_low[j] <= s.scale_high[j] && s.scale_high[j] <= 2.f))
      return "set_torque_scale: 0 < scale_low <= scale_high <= 2 required on every joint of the mask";
  }
  if (P.joint_limits == 0)
    return "set_torque_scale: needs joint_limits != 0 (the scale runs in the observation-delay kernels)";
  if (P.spine_mode) return "set_torque_scale: spine_mode applies the spine's own torque law";
  if (P.body_contacts) return "set_torque_scale: body_contacts has no torque-scale kernels";
  return nullptr;
}

// Why per-env torque scales v[n][UPKIE_NJ] are refused under the mask in force (upkie_b200_set_torque_scale_state),
// null when they are taken: a scale in (0, 2] on every joint of the mask, exactly 1 on every other joint
inline const char* torque_scale_state_error(uint32_t joint_mask, const float* v, size_t n) {
  for (size_t k = 0; k < n * UPKIE_NJ; ++k) {
    if ((joint_mask >> (k % UPKIE_NJ)) & 1u) {
      if (!(v[k] > 0.f && v[k] <= 2.f))  // (NaN fails too)
        return "set_torque_scale_state: every scale of a joint of joint_mask must be in (0, 2]";
    } else if (v[k] != 1.f) {
      return "set_torque_scale_state: a joint outside joint_mask must have a scale of exactly 1";
    }
  }
  return nullptr;
}

// Why a handle with parameters P refuses an attitude-filter spec (upkie_b200_set_attitude_filter), null when it takes
// it: every bound finite, low <= high, 0 <= kp with kp_high * h <= 0.5, 0 <= ki <= 10, and |roll|, |pitch| <= pi/4
inline const char* attitude_filter_spec_error(const UpkieAttitudeFilter& s, const SimParams& P) {
  const float b[8] = {s.kp_low, s.kp_high, s.ki_low, s.ki_high, s.roll_low, s.roll_high, s.pitch_low, s.pitch_high};
  for (int k = 0; k < 8; ++k)
    if (!std::isfinite(b[k])) return "set_attitude_filter: every bound must be finite";
  for (int k = 0; k < 8; k += 2)
    if (!(b[k] <= b[k + 1])) return "set_attitude_filter: low <= high required for kp, ki, roll and pitch";
  if (!(s.kp_low >= 0.f)) return "set_attitude_filter: kp_low >= 0 required";
  if (!(double(s.kp_high) * double(P.h) <= 0.5))
    return "set_attitude_filter: kp_high * (dt / nb_substeps) <= 0.5 required (the correction must not overshoot)";
  if (!(s.ki_low >= 0.f) || !(s.ki_high <= 10.f)) return "set_attitude_filter: 0 <= ki_low and ki_high <= 10 required";
  for (int k = 4; k < 8; ++k)
    if (!(b[k] >= -0.78539816f && b[k] <= 0.78539816f))
      return "set_attitude_filter: roll and pitch bounds must be within [-pi/4, pi/4] radians";
  if (P.joint_limits == 0)
    return "set_attitude_filter: needs joint_limits != 0 (the filter runs in the observation-delay kernels)";
  if (P.spine_mode) return "set_attitude_filter: spine_mode models its spine's own IMU";
  if (P.body_contacts) return "set_attitude_filter: body_contacts has no attitude-filter kernels";
  return nullptr;
}

inline void set_noise_flags(SimParams& P, uint32_t f) {
  P.any_ctrl_noise = (f & kEpCtrlNoise) ? 1 : 0;
  P.any_meas_noise = (f & kEpMeasNoise) ? 1 : 0;
  P.any_imu_uncertainty = (f & kEpImuUncertainty) ? 1 : 0;
}

// AoS state row <-> registers
UPKIE_HD void state_from_row(const float* r, RobotState& S) {
  for (int i = 0; i < 3; ++i) {
    S.pos[i] = r[UPKIE_ST_POS + i];
    S.linvel[i] = r[UPKIE_ST_LINVEL + i];
    S.angvel[i] = r[UPKIE_ST_ANGVEL + i];
    S.prev_imu_vel[i] = r[UPKIE_ST_PREV_IMU_VEL + i];
    S.imu_acc[i] = r[UPKIE_ST_IMU_ACC + i];
  }
  for (int i = 0; i < 4; ++i) {
    S.quat[i] = r[UPKIE_ST_QUAT + i];
    S.leg_target[i] = r[UPKIE_ST_LEG_TARGET + i];
  }
  for (int j = 0; j < 6; ++j) {
    S.q[j] = r[UPKIE_ST_Q + j];
    S.qd[j] = r[UPKIE_ST_QD + j];
    S.torque[j] = r[UPKIE_ST_TORQUE + j];
  }
  S.yaw = r[UPKIE_ST_YAW];
  S.yaw_vel = r[UPKIE_ST_YAW_VEL];
  S.contact = r[UPKIE_ST_CONTACT];
  S.lam_n[0] = r[UPKIE_ST_CONTACT_IMPULSE];
  S.lam_n[1] = r[UPKIE_ST_CONTACT_IMPULSE + 1];
  for (int k = 0; k < 4; ++k) S.lam_t[k] = r[UPKIE_ST_FRICTION_IMPULSE + k];
}

UPKIE_HD void state_to_row(const RobotState& S, float* r) {
  for (int i = 0; i < 3; ++i) {
    r[UPKIE_ST_POS + i] = S.pos[i];
    r[UPKIE_ST_LINVEL + i] = S.linvel[i];
    r[UPKIE_ST_ANGVEL + i] = S.angvel[i];
    r[UPKIE_ST_PREV_IMU_VEL + i] = S.prev_imu_vel[i];
    r[UPKIE_ST_IMU_ACC + i] = S.imu_acc[i];
  }
  for (int i = 0; i < 4; ++i) {
    r[UPKIE_ST_QUAT + i] = S.quat[i];
    r[UPKIE_ST_LEG_TARGET + i] = S.leg_target[i];
  }
  for (int j = 0; j < 6; ++j) {
    r[UPKIE_ST_Q + j] = S.q[j];
    r[UPKIE_ST_QD + j] = S.qd[j];
    r[UPKIE_ST_TORQUE + j] = S.torque[j];
  }
  r[UPKIE_ST_YAW] = S.yaw;
  r[UPKIE_ST_YAW_VEL] = S.yaw_vel;
  r[UPKIE_ST_CONTACT] = S.contact;
  r[UPKIE_ST_CONTACT_IMPULSE] = S.lam_n[0];
  r[UPKIE_ST_CONTACT_IMPULSE + 1] = S.lam_n[1];
  for (int k = 0; k < 4; ++k) r[UPKIE_ST_FRICTION_IMPULSE + k] = S.lam_t[k];
}

// ---- observation delay: the sensed rows (sim_core.cuh ObsDelay) ----
// A snapshot of S into an env's sensed row: store(k, value) for every sensed column k. The IMU pair is differentiated
// against the row's previous snapshot, load(k) of its UPKIE_ST_PREV_IMU_VEL columns (read before any store), over dt as
// observe_update does: acceleration (v - previous) / dt, then v becomes the previous velocity. `v` is the IMU velocity
// of S (imu_velocity, or observe_update's S.prev_imu_vel right after it ran).
template <typename Load, typename Store>
UPKIE_HD void obs_delay_snapshot(const SimParams& P, const RobotState& S, const float v[3], Load load, Store store) {
  float r[UPKIE_STATE_DIM];
  state_to_row(S, r);
  float prev[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) prev[k] = load(UPKIE_ST_PREV_IMU_VEL + k);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    r[UPKIE_ST_IMU_ACC + k] = (v[k] - prev[k]) * P.inv_dt;  // dt, not the substep (pybullet_backend.py:405-408)
    r[UPKIE_ST_PREV_IMU_VEL + k] = v[k];
  }
#pragma unroll
  for (int k = 0; k < UPKIE_STATE_DIM; ++k)
    if (obs_delay_sensed(k)) store(k, r[k]);
}

// S with its sensed fields replaced by load(k) of the env's sensed row: the state the observation is built from
template <typename Load>
UPKIE_HD void obs_delay_sensed_state(RobotState& S, Load load) {
  float r[UPKIE_STATE_DIM];
  state_to_row(S, r);
#pragma unroll
  for (int k = 0; k < UPKIE_STATE_DIM; ++k)
    if (obs_delay_sensed(k)) r[k] = load(k);
  state_from_row(r, S);
}

}  // namespace upkie_b200
