/* SPDX-License-Identifier: Apache-2.0
 *
 * upkie_b200.h -- C ABI of the H100-native vectorised Upkie simulation and
 * balance-control path (libupkie_b200.so).
 *
 * This is the drop-in boundary of SURVEY.md section 8(b). The reference has no
 * FFI for this path (it is Python calling the pybullet C extension); the entry
 * points below are what a binding of the reference's `Backend` ABC
 * (upkie/envs/backends/backend.py:11-50) and of `MPCBalancer.step`
 * (upkie/controllers/mpc_balancer.py:237-312) would call, vectorised over N
 * independent robots. Plain pointers and sizes only: no torch types.
 *
 * Conventions
 *  - every `const float*` / `float*` / `uint8_t*` argument of the non-`_host`
 *    functions is a DEVICE pointer on the handle's device; the caller owns all
 *    buffers, the library owns only the handle's internal state;
 *  - `stream` is a `cudaStream_t` passed as `void*` (NULL = legacy default
 *    stream); all launches are asynchronous on that stream;
 *  - every function returns 0 on success and a negative UPKIE_B200_E* code on
 *    failure, in which case `upkie_b200_last_error()` describes the failure
 *    (thread-local string). Nothing throws across the boundary.
 *  - joint order everywhere: left_hip, left_knee, left_wheel, right_hip,
 *    right_knee, right_wheel (URDF order, upkie/cpp/interfaces/static_config.h:64-69).
 */
#ifndef UPKIE_B200_H_
#define UPKIE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UPKIE_B200_ABI_VERSION 8

#define UPKIE_NJ 6 /* actuated joints */
#define UPKIE_NB 7 /* moving bodies: base lump + 2 x (upper leg, lower leg, wheel) */
#define UPKIE_MAX_COLLISION_POINTS 16 /* body-ground collision points a model may carry (UpkieModel) */
#define UPKIE_MAX_BODY_CONTACTS 4    /* of which at most this many (the deepest) hold contact rows in one substep:
                                      * Bullet's persistent manifold keeps 4 points per pair (MANIFOLD_CACHE_SIZE) */

/* ---- flat tensor layouts (all row-major, last index fastest) ------------- */

/* action[N][6 joints][6 keys], keys in UpkieServos.ACTION_KEYS order
 * (upkie/envs/upkie_servos.py:98-105). */
#define UPKIE_ACT_POSITION 0
#define UPKIE_ACT_VELOCITY 1
#define UPKIE_ACT_FEEDFORWARD_TORQUE 2
#define UPKIE_ACT_KP_SCALE 3
#define UPKIE_ACT_KD_SCALE 4
#define UPKIE_ACT_MAXIMUM_TORQUE 5
#define UPKIE_ACT_KEYS 6
#define UPKIE_ACT_DIM (UPKIE_NJ * UPKIE_ACT_KEYS) /* 36 */

/* obs[N][6 joints][5 keys], keys in the servo observation space order
 * (upkie/envs/upkie_servos.py:221-253). */
#define UPKIE_OBS_POSITION 0
#define UPKIE_OBS_VELOCITY 1
#define UPKIE_OBS_TORQUE 2
#define UPKIE_OBS_TEMPERATURE 3
#define UPKIE_OBS_VOLTAGE 4
#define UPKIE_OBS_KEYS 5
#define UPKIE_OBS_DIM (UPKIE_NJ * UPKIE_OBS_KEYS) /* 30 */

/* init_state[N][25]: what RobotState carries (upkie/utils/robot_state.py:37-92) */
#define UPKIE_INIT_POS 0     /* position_base_in_world[3] */
#define UPKIE_INIT_QUAT 3    /* orientation_base_in_world as (w, x, y, z) */
#define UPKIE_INIT_LINVEL 7  /* linear_velocity_base_to_world_in_world[3] */
#define UPKIE_INIT_ANGVEL 10 /* angular_velocity_base_in_base[3] */
#define UPKIE_INIT_Q 13      /* joint_configuration[6] */
#define UPKIE_INIT_QD 19     /* joint_velocity[6] (ignored by the PyBullet-mode reset, pybullet_backend.py:260-267) */
#define UPKIE_INIT_DIM 25

/* state[N][UPKIE_STATE_DIM]: full per-robot simulator + wrapper state
 * (get_state / set_state; internally stored struct-of-arrays). */
#define UPKIE_ST_POS 0          /* base position in world [3] */
#define UPKIE_ST_QUAT 3         /* base orientation (w, x, y, z) */
#define UPKIE_ST_LINVEL 7       /* base linear velocity, world frame [3] */
#define UPKIE_ST_ANGVEL 10      /* base angular velocity, world frame [3] */
#define UPKIE_ST_Q 13           /* joint angles [6] */
#define UPKIE_ST_QD 19          /* joint velocities [6] */
#define UPKIE_ST_PREV_IMU_VEL 25 /* __previous_imu_linear_velocity, pybullet_backend.py:157,405-408 */
#define UPKIE_ST_TORQUE 28      /* __joint_torques: last commanded torques [6], pybullet_backend.py:163,294 */
#define UPKIE_ST_LEG_TARGET 34  /* UpkieGyropod leg position targets: lh, lk, rh, rk (upkie_gyropod.py:246-267) */
#define UPKIE_ST_YAW 38         /* UpkieGyropod commanded-yaw integral (upkie_gyropod.py:383-385) */
#define UPKIE_ST_YAW_VEL 39
#define UPKIE_ST_CONTACT 40     /* floor contact seen by the last collision pass (0/1) */
#define UPKIE_ST_IMU_ACC 41     /* world-frame IMU linear acceleration of the last observation [3] (pybullet_backend.py:405-408) */
#define UPKIE_ST_CONTACT_IMPULSE 44 /* normal contact impulses of the last substep (left, right wheel): PGS warm start */
#define UPKIE_ST_FRICTION_IMPULSE 46 /* friction impulses of the last substep: rolling / lateral direction of the left wheel, then of the right wheel [4] (what getContactPoints reports as lateralFriction1 / 2, pybullet_backend.py:696-709) */
#define UPKIE_STATE_DIM 50

/* spine_obs[N][UPKIE_SPINE_DIM]: the observation dictionary of
 * PyBulletBackend.get_spine_observation (pybullet_backend.py:313-331), flattened. */
#define UPKIE_SP_BASE_ANGVEL 0   /* base_orientation.angular_velocity (base frame) [3] */
#define UPKIE_SP_BASE_LINVEL 3   /* base_orientation.linear_velocity (world) [3] */
#define UPKIE_SP_PITCH 6         /* base_orientation.pitch */
#define UPKIE_SP_ROT 7           /* base_orientation.rotation_base_to_world, row-major [9] */
#define UPKIE_SP_IMU_QUAT 16     /* imu.orientation (w, x, y, z) in the ARS frame */
#define UPKIE_SP_IMU_ANGVEL 20   /* imu.angular_velocity (IMU frame) [3] */
#define UPKIE_SP_IMU_LINACC 23   /* imu.linear_acceleration (IMU frame) [3] */
#define UPKIE_SP_IMU_RAWACC 26   /* imu.raw_linear_acceleration (IMU frame) [3] */
#define UPKIE_SP_CONTACT 29      /* floor_contact.contact (0/1) */
#define UPKIE_SP_SERVO 30        /* servo[6][5] as in obs */
#define UPKIE_SP_ODOM_POS 60     /* wheel_odometry.position */
#define UPKIE_SP_ODOM_VEL 61     /* wheel_odometry.velocity */
#define UPKIE_SPINE_DIM 62

/* observers_out[N][UPKIE_OBSV_DIM]: outputs of the spine's observer pipeline
 * (spines/common/observers.h:23-44) */
#define UPKIE_OBSV_PITCH 0          /* base_orientation.pitch (upkie/cpp/observers/BaseOrientation.h:73-92) */
#define UPKIE_OBSV_ANGVEL 1         /* base_orientation.angular_velocity [3] (BaseOrientation.h:144-148) */
#define UPKIE_OBSV_ROT 4            /* base_orientation.rotation_base_to_world, row-major [9] */
#define UPKIE_OBSV_CONTACT 13       /* floor_contact.contact (FloorContact.cpp:37-49) */
#define UPKIE_OBSV_WHEEL_CONTACT 14 /* floor_contact.{left,right}_wheel.contact [2] (WheelContact.cpp:19-48) */
#define UPKIE_OBSV_LEG_TORQUE 16    /* floor_contact.upper_leg_torque (FloorContact.cpp:73-91) */
#define UPKIE_OBSV_WHEEL_INERTIA 17 /* floor_contact.{left,right}_wheel.inertia [2] */
#define UPKIE_OBSV_ODOM_POS 19      /* wheel_odometry.position (WheelOdometry.cpp:16-24) */
#define UPKIE_OBSV_ODOM_VEL 20      /* wheel_odometry.velocity */
#define UPKIE_OBSV_DIM 21

/* per-env error flags (sticky until reset) */
#define UPKIE_ERR_NAN_VELOCITY 1u /* NaN target velocity (asserted in pybullet_backend.py:519) */
#define UPKIE_ERR_NAN_STATE 2u    /* non-finite simulator state */
#define UPKIE_ERR_CLAMPED 4u      /* some action entry was clamped (clamp_and_warn, upkie/utils/clamp.py:42-58) */

/* status codes */
#define UPKIE_B200_OK 0
#define UPKIE_B200_EINVAL (-1)
#define UPKIE_B200_ECUDA (-2)
#define UPKIE_B200_ENOMEM (-3)
#define UPKIE_B200_EMODEL (-4)

/* ---- model and configuration (host-side, read once at create) ------------ */

/* Rigid-body model after fixed-joint lumping. Body 0 is the floating base
 * lump; body i (1..6) is attached to parent[i] by revolute joint i-1. Every body
 * frame has its origin at its joint's origin and is aligned with the base frame
 * at the zero configuration. This carries what upkie.model.Model provides
 * (upkie/model/model.py:57-110: wheel radius, wheel base, left-wheeledness,
 * base->IMU rotation, joint limits) plus the masses/inertias that live in the
 * URDF of upkie_description. */
typedef struct UpkieModel {
  int32_t parent[UPKIE_NB];          /* parent[0] = -1 */
  int32_t left_wheeled;              /* upkie/model/model.py:104 */
  double joint_origin[UPKIE_NJ][3];  /* joint origin in the parent body frame */
  double joint_axis[UPKIE_NJ][3];    /* unit rotation axis (same in parent and child frames) */
  double mass[UPKIE_NB];
  double com[UPKIE_NB][3];           /* centre of mass in the body frame */
  double inertia[UPKIE_NB][6];       /* about the CoM, body axes: xx, yy, zz, xy, xz, yz */
  double q_lower[UPKIE_NJ];          /* position limits (-inf/+inf for wheels) */
  double q_upper[UPKIE_NJ];
  double qd_max[UPKIE_NJ];           /* velocity limits */
  double tau_max[UPKIE_NJ];          /* effort limits */
  double wheel_radius;               /* tire collision cylinder radius, model.py:115-144 */
  double wheel_base;                 /* distance between tire frames, model.py:82 */
  double imu_position[3];            /* IMU frame origin in the base frame */
  double rotation_base_to_imu[9];    /* row-major, model.py:106 */
  /* Collision points of the bodies other than the tires (ABI 6): what the <collision> shapes of the URDF links reduce
   * to against the ground plane - a box is its 8 corners, a sphere its centre with a radius, a cylinder / capsule the
   * two end points of its axis with the radius (upkie/model/link.py:53-91 parses the same elements). Point p belongs
   * to moving body collision_body[p] (0 = base lump .. 6) and sits at collision_point[p] in that body's frame.
   * PyBullet collides every link that has a collision shape with plane.urdf (pybullet_backend.py:115,121,306). */
  int32_t n_collision_points;        /* 0 .. UPKIE_MAX_COLLISION_POINTS */
  int32_t collision_body[UPKIE_MAX_COLLISION_POINTS];
  int32_t reserved_collision;
  double collision_point[UPKIE_MAX_COLLISION_POINTS][3];
  double collision_radius[UPKIE_MAX_COLLISION_POINTS];
} UpkieModel;

/* Simulation + environment configuration. Defaults are filled by
 * upkie_b200_default_config(). */
typedef struct UpkieSimConfig {
  /* PyBulletBackend (upkie/envs/backends/pybullet_backend.py:55-112) */
  double dt;                   /* agent period, 1/frequency (0.005) */
  int32_t nb_substeps;         /* int(1000*dt) = 5 */
  int32_t pgs_iterations;      /* Bullet numSolverIterations default (50) */
  double gravity;              /* 9.81, pybullet_backend.py:110 */
  double torque_control_kp;    /* 20.0 */
  double torque_control_kd;    /* 1.0 */
  double joint_friction[UPKIE_NJ]; /* JointProperties.friction, joint_properties.py:24-40 */
  double torque_control_noise[UPKIE_NJ];     /* JointProperties.torque_control_noise: std of the Gaussian noise added to
                                              * every commanded torque before the clip (pybullet_backend.py:545-550) */
  double torque_measurement_noise[UPKIE_NJ]; /* std of the noise on the observed torque (pybullet_backend.py:461-466) */
  double imu_accelerometer_bias[3]; /* ImuUncertainty (upkie/cpp/interfaces/ImuUncertainty.h:29-69): bias and white */
  double imu_accelerometer_noise;   /* noise added to the IMU-frame accelerations (filtered and raw) and angular    */
  double imu_gyroscope_bias[3];     /* velocity of the spine observation (BulletInterface.cpp:252-258)             */
  double imu_gyroscope_noise;
  uint64_t noise_seed;                       /* key of the counter-based generator (the reference draws from an unseeded
                                              * np.random.default_rng(), pybullet_backend.py:160) */
  /* restated Bullet multibody behaviour (third-party; see DESIGN.md) */
  double linear_damping;       /* 0.04 */
  double angular_damping;      /* 0.04 */
  double max_coordinate_velocity; /* 100.0 */
  double contact_stiffness;    /* tire <contact> stiffness */
  double contact_damping;      /* tire <contact> damping */
  double contact_breaking_threshold; /* 0.02 */
  double friction;             /* combined lateral friction (plane 1.0 x tire) */
  /* UpkieServos (upkie/envs/upkie_servos.py:114-170) */
  double max_gain_scale;       /* 5.0 */
  /* UpkieGyropod / UpkiePendulum (upkie/envs/upkie_gyropod.py:105-160) */
  double fall_pitch;           /* 1.0 */
  double leg_gain_scale;       /* 1.0 */
  double max_ground_velocity;  /* 3.0 */
  double max_yaw_velocity;     /* 1.0 */
  /* extension (SURVEY 8d config 3): also terminate UpkieServos envs when
   * |pitch| > fall_pitch or base height < min_base_height; 0 = reference behaviour */
  int32_t servos_fall_termination;
  /* 1 = skip the UpkieServos.get_spine_action clamps (used by the single-env Backend adapter,
   * which receives actions the reference's own UpkieServos already clamped) */
  int32_t skip_action_clamps;
  double min_base_height;
  /* DEPRECATED, ignored since ABI 6 (superseded by solver_residual_threshold, Bullet's own exit rule, at the end of
   * this struct). Was: PGS sweeps stop early once every impulse of a warp changed by less than
   * pgs_tolerance * |impulse| + 1e-9 in one sweep (Bullet: m_leastSquaresResidualThreshold-style
   * exit); 0 = always run pgs_iterations sweeps. Default 1e-5: ~50 ulp of the fp32 impulses, the converged
   * contact impulses then differed from 50 full sweeps by < 1e-6 m/s on velocities */
  double pgs_tolerance;
  /* Bullet's SOLVER_USE_WARMSTARTING: normal contact impulses start each substep at
   * warmstarting_factor x the previous substep's value while the contact persists (Bullet: 0.85), friction rows
   * at 0. Default 0 = cold start: the fixed point is the same and the sweep count did not drop in measurements */
  double warmstarting_factor;
  /* Bullet's joint-limit constraints: PyBullet's URDF importer attaches a btMultiBodyJointLimitConstraint to every
   * revolute joint that declares limits (hips and knees; the wheels are continuous). While a joint sits at or
   * beyond a bound, one unilateral row along that joint joins the contact rows in the PGS solve (solved before the
   * contact normals, in alternating order from sweep to sweep), with Baumgarte factor joint_limit_erp and the
   * impulse capped at joint_limit_max_impulse. 0 = no limit rows (round 1's physics); 2 = rows on, every robot runs
   * the packed ten-row solver (four limit slots + six contact rows); 3 (default) = rows on, the ten-row solver for
   * the warps that hold a robot on a bound and the six-row contact solver for the others; 1 = the scalar reference
   * implementation of the rows, which exists in the HOST build of the kernel arithmetic only (tests): on the device
   * it is an alias of 3 (many times slower than the plain kernel, DESIGN.md section 3).
   * Same results to round-off in all three. */
  int32_t joint_limits;
  int32_t reserved_joint_limits; /* keeps the doubles below 8-byte aligned without implicit padding */
  double joint_limit_erp;         /* btContactSolverInfo::m_erp = 0.2 */
  double joint_limit_max_impulse; /* btMultiBodyConstraint::m_maxAppliedImpulse = 100 */
  /* RobotStateRandomization bounds used by the on-device sampler
   * (upkie/utils/robot_state_randomization.py:135-189) */
  double init_position[3];     /* nominal position_base_in_world (0, 0, 0.6) */
  double init_quat[4];         /* nominal orientation (w, x, y, z) */
  double rand_roll, rand_pitch, rand_x, rand_z;
  double rand_omega_x, rand_omega_y;
  double rand_linear_velocity[3];
  /* nominal joint configuration and base velocities of the initial state (RobotState.joint_configuration,
   * angular_velocity_base_in_base, linear_velocity_base_to_world_in_world; upkie/utils/robot_state.py:175-196):
   * sample_state keeps the joint configuration and ADDS the random velocity parts to the nominal ones, and so does the
   * on-device sampler of the fused auto-reset */
  double init_joint_configuration[6];
  double init_angular_velocity[3];
  double init_linear_velocity[3];
  /* 0 (default): the timing of PyBulletBackend - an env step is nb_substeps physics steps and the observation is
   * taken from the state after the last of them. 1: the timing of the C++ Bullet spine in simulate() mode
   * (spines/bullet_spine.cpp --nb-substeps, upkie/cpp/spine/Spine.cpp:116-140,185-265 and
   * upkie/cpp/interfaces/BulletInterface.cpp:228-352), UpkieServos steps only: every spine cycle reads the joint
   * sensors and the IMU, computes the torques from THOSE readings (tau_max = min(maximum_torque, URDF effort)) and
   * steps Bullet once at 1 / spine_frequency = dt / nb_substeps; the observation an env step returns is the one the
   * spine assembled in its FIRST cycle of that step, i.e. with S physics steps done before it: joint sensors (and the
   * torque commanded with them) of the state after S - 2 steps, IMU of the state after S - 1 steps, IMU acceleration
   * differentiated over one cycle; a reset runs three cycles with the servos stopped (Bullet velocity motors holding
   * 0 rad/s with 100 N m, restated as locked joints) and returns the observation of the third; the base angular
   * velocity of the initial state is rotated to the world frame (BulletInterface.cpp:146-152); servo temperature
   * reads 20.0 (BulletInterface.cpp:70). Needs joint_limits != 0 (the "extras + limits" kernels carry it). */
  int32_t spine_mode;
  int32_t reserved_spine_mode;
  /* Body-ground contacts (ABI 6; Bullet collides every link that has a collision shape with the plane, so a fallen
   * robot rests on its torso instead of passing through the floor). 1: while a collision point of the
   * model (UpkieModel.collision_*) is closer to the ground than contact_breaking_threshold, it holds one normal row
   * and two friction rows in the substep's PGS solve - rigid contact (no <contact> stiffness on those links):
   * cfm 0, Baumgarte factor body_contact_erp, friction coefficient = the env's floor friction x body_friction, friction
   * directions world -y and +x (btPlaneSpace1 of the plane normal); rows are solved after the wheel rows of their kind
   * (normals, then frictions). At most UPKIE_MAX_BODY_CONTACTS points (the deepest) are active per robot. Needs
   * joint_limits != 0. Handles with body_contacts = 1 run their own kernel instantiations (csrc/step_family.h); there a
   * warp that holds no such point runs the packed solvers, one that does solves ALL rows of its 32 robots in a general
   * scalar solver - many times the packed cost for that warp and substep (DESIGN.md section 3), which is
   * why the default is 0 = off (a fallen robot's torso passes through the floor, as in round 1) for batched handles:
   * RL workloads reset fallen robots anyway. B200Backend, the single-env drop-in for PyBulletBackend, turns it on. */
  int32_t body_contacts;
  int32_t reserved_body_contacts;
  double body_contact_erp;   /* btContactSolverInfo::m_erp2 = 0.2 */
  double body_friction;      /* URDF importer default lateral friction of a link without <contact>: 0.5 */
  /* Bullet's solver exit rule (btSequentialImpulseConstraintSolver::solveGroupCacheFriendlyIterations): after every
   * sweep the solver compares the largest squared velocity-level change of a row, (delta_impulse / jacDiagABInv)^2,
   * with btContactSolverInfo::m_leastSquaresResidualThreshold and stops at or below it. Bullet's own default is 0
   * (all numIterations sweeps); PyBullet's physics server sets 1e-7 (setPhysicsEngineParameter solverResidualThreshold,
   * "default 1e-7") and the reference changes neither (it only calls setTimeStep, pybullet_backend.py:112,
   * BulletInterface.cpp:129): a robot's solve ends once no row moved its relative velocity by more than 3.2e-4 m/s in a
   * sweep. Default 1e-7; 0 = always pgs_iterations sweeps. Evaluated per robot after every sweep: a robot that has
   * met the threshold keeps its impulses while the other robots of its warp finish. */
  double solver_residual_threshold;
  /* Episode time limit (ABI 7), per env, with the semantics of Gymnasium's TimeLimit wrapper: 0 (default) = none,
   * truncated is always 0. T > 0: every env counts the agent steps since its last reset (upkie_b200_reset, masked or
   * not, and either fused auto-reset set the count to 0; the next-step auto-reset's own step is not counted) and a
   * step returns truncated = 1 once that count reaches T, independently of terminated (both can be 1). The fused
   * auto-reset fires on terminated | truncated; with auto-reset disabled truncated stays 1 until the env is reset.
   * The counts are kept only while a limit is set: when upkie_b200_set_config turns a limit on or changes it, every
   * env's count is set to 0, so episodes are timed from that call. upkie_b200_get_elapsed / set_elapsed read and
   * restore them. The in-kernel rollout transports (multicast, peers, push) reject a limit. */
  int32_t max_episode_steps;
  int32_t reserved_max_episode_steps;
} UpkieSimConfig;

/* Spine-mode lag record of one env (upkie_b200_get_lag / set_lag, [N][UPKIE_LAG_DIM] floats): the two latest
 * servo replies and the latest IMU reading of the spine's actuation interface. */
#define UPKIE_LAG_REPLY1 0   /* [6][3] position, velocity, torque read / commanded in the latest cycle */
#define UPKIE_LAG_REPLY2 18  /* the cycle before: what the next observation reports */
#define UPKIE_LAG_IMU 36     /* orientation_imu_in_ars wxyz (4), angular velocity (3), linear acceleration (3), raw (3) */
/* the observation the spine assembled last (what the env step / reset returned and get_spine_observation reports) */
#define UPKIE_LAG_OBS_REPLY 49   /* [6][3] */
#define UPKIE_LAG_OBS_IMU 67     /* [13] */
#define UPKIE_LAG_OBS_BASE 80    /* "sim" ground truth at that instant: base quaternion wxyz, linear, angular velocity (world) */
#define UPKIE_LAG_OBS_CONTACT 90
#define UPKIE_LAG_DIM 91

/* Per-env parameter table (upkie_b200_set_env_params / get_env_params, [N][UPKIE_EP_DIM] floats): one row per env
 * that overrides, for that env, the UpkieSimConfig fields of the same meaning, wherever the kernels read them. What N
 * reference envs built with different PyBulletBackend(torque_control_kp=..., torque_control_kd=...,
 * joint_properties={joint: JointProperties(...)}) arguments and different spine ImuUncertainty hold. */
#define UPKIE_EP_KP 0             /* torque_control_kp (pybullet_backend.py:65, used at :528) */
#define UPKIE_EP_KD 1             /* torque_control_kd (pybullet_backend.py:64, used at :529) */
#define UPKIE_EP_FRICTION 2       /* [6] JointProperties.friction (joint_properties.py:24-40, pybullet_backend.py:538-543) */
#define UPKIE_EP_CTRL_NOISE 8     /* [6] JointProperties.torque_control_noise (pybullet_backend.py:545-552) */
#define UPKIE_EP_MEAS_NOISE 14    /* [6] JointProperties.torque_measurement_noise (pybullet_backend.py:461-466) */
#define UPKIE_EP_IMU_ACC_BIAS 20  /* [3] ImuUncertainty accelerometer_bias (ImuUncertainty.h:29-69) */
#define UPKIE_EP_IMU_ACC_NOISE 23 /* ImuUncertainty accelerometer_noise */
#define UPKIE_EP_IMU_GYRO_BIAS 24 /* [3] ImuUncertainty gyroscope_bias */
#define UPKIE_EP_IMU_GYRO_NOISE 27 /* ImuUncertainty gyroscope_noise */
#define UPKIE_EP_DIM 28

/* MPCBalancer parameters (upkie/controllers/mpc_balancer.py:168-181) */
typedef struct UpkieMpcConfig {
  double fall_pitch;              /* 1.0 */
  double leg_length;              /* 0.58 */
  double max_ground_accel;        /* 10.0 */
  double max_ground_velocity;     /* 3.0 */
  int32_t nb_timesteps;           /* 50 */
  int32_t max_iterations;         /* active-set iteration cap */
  double sampling_period;         /* 0.02 */
  double stage_input_cost_weight; /* 1e-3 */
  double stage_state_cost_weight; /* 1e-3 */
  double terminal_cost_weight;    /* 1.0 */
  double gravity;                 /* 9.81 (qpmpc GRAVITY) */
} UpkieMpcConfig;

/* Observer pipeline parameters: spine configuration defaults of
 * upkie/envs/backends/spine_backend.py:77-105,140-165 */
typedef struct UpkieObserverConfig {
  double dt;                          /* 1 / spine_frequency (0.001) */
  double cutoff_period;               /* wheel_contact.cutoff_period (0.2) */
  double liftoff_inertia;             /* 1e-3 */
  double min_touchdown_acceleration;  /* 2.0 */
  double min_touchdown_torque;        /* 0.015 */
  double touchdown_inertia;           /* 4e-3 */
  double upper_leg_torque_threshold;  /* floor_contact.upper_leg_torque_threshold (10.0) */
  double signed_radius[2];            /* wheel_odometry.signed_radius: left, right */
  double rotation_base_to_imu[9];     /* base_orientation.rotation_base_to_imu, row-major */
} UpkieObserverConfig;

/* WheelBalancer::Parameters (upkie/cpp/controllers/WheelBalancer.h:48-91) */
typedef struct UpkieWheelBalancerConfig {
  double contact_radius;       /* 0.1524 */
  double dt;                   /* 1 / spine_frequency (spines/common/controllers.h:34) */
  double fall_pitch;           /* 1.0 */
  double max_ground_velocity;  /* 2.0 */
  double pitch_damping;        /* 1.8 */
  double pitch_stiffness;      /* 20.0 */
  double position_damping;     /* 0.7 */
  double position_stiffness;   /* 1.6 */
  double stiff_yaw_velocity;   /* 0.1 */
  double wheel_radius;         /* 0.06 (spines/common/controllers.h:35) */
} UpkieWheelBalancerConfig;

/* where a controller reads pitch / floor contact / wheel-odometry position */
#define UPKIE_OBS_LAYOUT_SPINE 0     /* spine_obs rows [N][UPKIE_SPINE_DIM] */
#define UPKIE_OBS_LAYOUT_OBSERVERS 1 /* observers_out rows [N][UPKIE_OBSV_DIM] */

/* ---- library ------------------------------------------------------------ */

int upkie_b200_abi_version(void);
const char* upkie_b200_last_error(void);

/* Fill `config` with the reference's defaults. */
int upkie_b200_default_config(UpkieSimConfig* config);
int upkie_b200_default_mpc_config(UpkieMpcConfig* config);

/* ---- simulation handle --------------------------------------------------
 * Replaces PyBulletBackend.__init__ (pybullet_backend.py:55-197). */
int upkie_b200_create(const UpkieModel* model, const UpkieSimConfig* config,
                      int n_envs, int device, void** handle);
void upkie_b200_destroy(void* handle);
int upkie_b200_num_envs(void* handle);

/* Replace the simulation configuration of a live handle (same model): the initial-state bounds and nominal values
 * the on-device reset sampler draws from (UpkieEnv.update_init_rand, upkie/envs/upkie_env.py:244-251), noise levels,
 * gains... Takes effect for launches enqueued after the call; the robot state is untouched. */
int upkie_b200_set_config(void* handle, const UpkieSimConfig* config);

/* Vector-env auto-reset, fused into the step kernels (the reference has no
 * auto-reset: "you are responsible for calling reset()", upkie_env.py:200-201;
 * Gymnasium vector envs do). mode 0 = disabled (reference behaviour, default),
 * 1 = next-step (an env that terminated at step t is re-initialised by the call
 * at t+1, which returns its reset observation and ignores its action),
 * 2 = same-step (re-initialised inside the terminating call, which returns the
 * reset observation together with terminated = 1). Initial states are drawn on
 * the device as in upkie_b200_reset(init_state = NULL). With a time limit
 * (UpkieSimConfig.max_episode_steps) an env resets on terminated | truncated;
 * in same-step mode upkie_b200_step / upkie_b200_step_host can also return the
 * observation the resetting envs reached before their reset (final_obs). */
int upkie_b200_set_autoreset(void* handle, int mode, uint64_t seed, uint64_t env_offset);

/* Per-env actuator and IMU parameters (ABI 8): rows[N][UPKIE_EP_DIM] (device pointer, layout UPKIE_EP_*) replace,
 * env by env, the config's torque_control_kp / kd, joint_friction, torque_control_noise, torque_measurement_noise and
 * imu_* fields, wherever the kernels use them: the torque law of every substep (spine mode: kp and kd only, the C++
 * spine has no joint friction or torque noise, BulletInterface.cpp:329-352), the torque measurement noise of the
 * observations and the ImuUncertainty of upkie_b200_spine_obs. noise_seed still comes from the config; noise is drawn
 * with the same keys as without a table, so an env draws the same numbers whatever its batch holds.
 * Every value must be finite, gains, friction and noise standard deviations >= 0 (biases may be negative); otherwise
 * UPKIE_B200_EINVAL and the previous table stays. NULL drops the table: every env runs the config's values again.
 * upkie_b200_set_config keeps the table. Waits for the device (not a hot-path call); takes effect for launches
 * enqueued after it. The in-kernel rollout transports (multicast, peers, push) reject a handle with a table. */
int upkie_b200_set_env_params(void* handle, const float* rows, void* stream);
/* The parameters in force, rows[N][UPKIE_EP_DIM] (device pointer): the table, or without one the config's values
 * (as floats) in every row. */
int upkie_b200_get_env_params(void* handle, float* rows, void* stream);

/* Per-env domain randomisation; either pointer may be NULL (= nominal).
 * friction[N]: combined floor friction (extension, SURVEY 8d config 3).
 * inertia_eps[N][6]: epsilon of randomize_inertias (pybullet_backend.py:571-601),
 * one per non-base body; mass and inertia scale by (1 + eps). */
int upkie_b200_set_randomization(void* handle, const float* friction,
                                 const float* inertia_eps, void* stream);
/* The randomisation in force: friction[N] and inertia_eps[N][6] (device pointers, either may be NULL). Without a
 * buffer set, the nominal values: the config's friction, epsilon 0. An addition to ABI 8. */
int upkie_b200_get_randomization(void* handle, float* friction, float* inertia_eps, void* stream);

/* Reset randomisation (an addition to ABI 8: no existing layout, constant or signature changed). While a spec is set,
 * every reset of an env - both fused auto-resets, and upkie_b200_reset with device-sampled or host init rows, masked or
 * not - redraws the selected columns of that env on the device, each uniformly from [low, high]:
 *   columns 0 .. UPKIE_EP_DIM - 1    the env's row of the per-env parameter table (UPKIE_EP_*),
 *   UPKIE_RR_INERTIA + b (b < 6)     inertia_eps of body b + 1 (upkie_b200_set_randomization; randomize_inertias),
 *   UPKIE_RR_FRICTION                the floor friction.
 * Bit k of `columns` selects column k; the other columns keep their values bit for bit.
 * Draw law: env i's draws are numbered 1, 2, ... by a per-env counter (upkie_b200_get_draws / set_draws); draw d of
 * the env of global index g = env_offset + i is keyed on (seed, g, d), with the seed and env_offset of
 * upkie_b200_set_autoreset: block b = 0 .. 8 of Philox4x32-10 with counter (g, 2^63 | d << 4 | b) and key seed gives
 * the uniform words of columns 4b .. 4b + 3, u = (word >> 8) * 2^-24, value = min(low + (high - low) * u, high) in
 * fp32, the product rounded on its own (no FMA). All 35 columns are always drawn. The values are in force from the
 * env's reset substep on, as if set with upkie_b200_set_env_params / set_randomization just before the reset; the
 * terminal observations of same-step auto-resets (final_obs, upkie_b200_final_spine_obs) still use the values of the
 * episode that ended.
 * Setting a spec gives the handle a parameter table (the config's values) and randomisation buffers (friction of the
 * config, epsilon 0) if it has none; noise models that some range can turn on are switched on. Needs
 * joint_limits != 0. Rejected with UPKIE_B200_EINVAL, the previous spec kept: a bound that is not finite, low > high,
 * low < 0 on a gain, joint friction or noise standard deviation column, an inertia bound <= -1, a floor friction low < 0.
 * While a spec is set, upkie_b200_set_env_params(NULL) and upkie_b200_set_randomization with a NULL pointer return
 * UPKIE_B200_EINVAL (the draws write into those buffers). NULL turns reset randomisation off; the values then in force
 * stay. The in-kernel rollout transports reject a handle with a parameter table, hence with this. */
#define UPKIE_RR_INERTIA 28 /* [6] inertia_eps of the non-base bodies */
#define UPKIE_RR_FRICTION 34 /* floor friction */
#define UPKIE_RR_DIM 35
typedef struct UpkieResetRandomization {
  uint64_t columns;          /* bit k: column k is redrawn at every reset */
  float low[UPKIE_RR_DIM];
  float high[UPKIE_RR_DIM];
} UpkieResetRandomization;
int upkie_b200_set_reset_randomization(void* handle, const UpkieResetRandomization* spec);
/* Per-env draw counters draws[N] (device pointers), for checkpoints: 0 = never drawn. */
int upkie_b200_get_draws(void* handle, uint32_t* draws, void* stream);
int upkie_b200_set_draws(void* handle, const uint32_t* draws, void* stream);

/* Replaces UpkieEnv.reset -> PyBulletBackend.reset (upkie_env.py:162-194,
 * pybullet_backend.py:220-267): set state, ONE physics substep, observe.
 * mask[N] (u8) selects the envs to reset (NULL = all). init_state[N][25] gives
 * the sampled RobotState per env; NULL = sample on the device from the
 * configuration's RobotStateRandomization bounds with a counter-based generator
 * keyed on (seed, global env index = env_offset + i). */
int upkie_b200_reset(void* handle, const uint8_t* mask, const float* init_state,
                     uint64_t seed, uint64_t env_offset, void* stream);

/* Replaces UpkieServos.step = UpkieEnv.step -> get_spine_action ->
 * PyBulletBackend.step -> get_env_observation (upkie_env.py:196-242,
 * upkie_servos.py:288-344, pybullet_backend.py:269-311). */
int upkie_b200_step_servos(void* handle, const float* action /* [N][6][6] */,
                           float* obs /* [N][6][5] */, float* reward /* [N] */,
                           uint8_t* terminated /* [N] */, uint8_t* truncated /* [N] */,
                           void* stream);

/* Replaces UpkieGyropod.step (act_dim = 2, obs[N][6]) and UpkiePendulum.step
 * (act_dim = 1, obs[N][4]) (upkie_gyropod.py:354-392, upkie_pendulum.py:124-142). */
int upkie_b200_step_gyropod(void* handle, const float* action /* [N][act_dim] */,
                            int act_dim, float* obs, float* reward,
                            uint8_t* terminated, uint8_t* truncated, void* stream);

/* UpkieServos step, device buffers, compact observation rows obs[N][6][3] (position, velocity, torque; see
 * upkie_b200_step_servos_host_compact for what is left out and why). What a rollout buffer gathered across
 * GPUs should carry: 73 B instead of 126 B per env and step over NVLink. */
int upkie_b200_step_servos_compact(void* handle, const float* action, float* obs, uint8_t* terminated, void* stream);

/* Same step, but obs_mc / terminated_mc are NVSwitch MULTICAST addresses (CUmulticastObject mapping of a buffer
 * that exists at the same offset on every GPU of the node, e.g. torch.distributed._symmetric_memory's
 * multicast_ptr + offset): rows leave through multimem.st and land in every GPU's buffer, which is the per-step
 * all-gather of the rollout with no collective kernel. n_envs must be a multiple of 32. The caller synchronises the
 * ranks (a barrier per rollout) before reading (DESIGN.md section 7). */
int upkie_b200_step_servos_multicast(void* handle, const float* action, float* obs_mc, uint8_t* terminated_mc, void* stream);

/* Same kernel without a multicast object: the compact rows and `terminated` words of this step are stored into
 * n_peers buffers (peer-mapped device memory of the GPUs of the node, e.g. torch.distributed._symmetric_memory
 * buffers; list this rank's own buffer too if it should hold the rows). obs_ptrs[p] / terminated_ptrs[p] address
 * this step's slot in buffer p (16-byte / 4-byte aligned). 1 <= n_peers <= UPKIE_MAX_PEERS; n_envs a multiple of 32.
 * Replaces the per-rollout all-gather of SURVEY.md section 8(e) like the multicast variant, over plain NVLink stores. */
#define UPKIE_MAX_PEERS 8
int upkie_b200_step_servos_peers(void* handle, const float* action, float* const* obs_ptrs,
                                 uint8_t* const* terminated_ptrs, int n_peers, void* stream);

/* Deferred form of the two transports above (what bench.py runs): this step's compact rows and `terminated` bytes go
 * to LOCAL buffers (obs / terminated: this rank's slot of the step, plain stores), and the prologue of the same launch
 * sends the rows of an EARLIER step - read from src_obs / src_terminated, this rank's local slot of that step - to
 * every GPU: to the multicast addresses mc_obs / mc_terminated when n_peers == 0, else into the n_peers buffers
 * peer_obs[p] / peer_terminated[p]. The remote stores then drain under the ~0.1 ms of simulation instead of holding up
 * the completion of the launch.
 * src_obs == NULL: nothing to send (first step). upkie_b200_push_rows sends a slot on its own (last step of a
 * rollout, before the ranks' barrier). Alignment as above; n_envs a multiple of 32. */
typedef struct UpkiePush {
  const float* src_obs;
  const uint8_t* src_terminated;
  float* mc_obs;
  uint8_t* mc_terminated;
  float* peer_obs[UPKIE_MAX_PEERS];
  uint8_t* peer_terminated[UPKIE_MAX_PEERS];
  int32_t n_peers;
  int32_t reserved;
} UpkiePush;
int upkie_b200_step_servos_push(void* handle, const float* action, float* obs, uint8_t* terminated,
                                const UpkiePush* push, void* stream);
int upkie_b200_push_rows(void* handle, const UpkiePush* push, void* stream);

/* Same calls with HOST buffers and a stream synchronisation inside the call
 * (the `e2e` path of bench.py). When every buffer is pinned and mapped
 * (cudaHostAlloc / cudaHostRegister(..Mapped), torch pin_memory) the step is
 * ONE kernel launch that reads the action rows from host memory and writes the
 * observation rows back over PCIe itself (coalesced through shared memory);
 * pageable buffers go through pinned staging in pipelined chunks (H2D copy ->
 * kernel -> D2H copy on rotating streams).
 * `reward` and `truncated` may be NULL here and in the device-buffer calls: the
 * reference returns a constant reward (0.0, upkie_env.py:230) and leaves
 * truncation to a TimeLimit wrapper (False, upkie_env.py:197,232). truncated
 * is 0 for every env unless the configuration sets max_episode_steps, so a
 * caller without a limit that knows it saves the bytes. */
int upkie_b200_step_servos_host(void* handle, const float* action, float* obs,
                                float* reward, uint8_t* terminated,
                                uint8_t* truncated);
int upkie_b200_step_gyropod_host(void* handle, const float* action, int act_dim,
                                 float* obs, float* reward, uint8_t* terminated,
                                 uint8_t* truncated);
/* UpkieServos step that transports only what changes: obs[N][6][3] = position,
 * velocity, torque per joint. Temperature (42.0) and voltage (18.0) are
 * constants of the simulator (pybullet_backend.py:471-472), reward a constant
 * of the env (upkie_env.py:230): the caller fills them once. truncated is not
 * returned: it is 0 without a time limit; with max_episode_steps set, use
 * upkie_b200_step_host with compact = 1. 72 + 1 B per env over PCIe instead
 * of 126 B. */
int upkie_b200_step_servos_host_compact(void* handle, const float* action,
                                        float* obs, uint8_t* terminated);

/* General form of the step calls above: outputs in one struct, so that the compact servo rows can come with
 * `truncated`, and any step with the observations of its same-step auto-resets.
 * act_dim: 36 = UpkieServos (obs [N][6][5], or [N][6][3] with compact = 1), 2 = UpkieGyropod (obs [N][6]),
 * 1 = UpkiePendulum (obs [N][4]). reward, truncated and final_obs may be NULL.
 * final_obs (same-step auto-reset only; ignored in the other modes): every env that resets in this step first
 * stores there, at its own row, the observation it would have returned without the reset (layout of `obs`; spine
 * mode: the rows its spine assembled before the reset). The rows of the other envs are left untouched: mask them
 * with terminated | truncated (Gymnasium's info["final_obs"] / info["_final_obs"]).
 * final_state (same-step auto-reset only; ignored in the other modes): 1 = every env that resets in this step also
 * stashes its pre-reset state in the handle, from which upkie_b200_final_spine_obs computes the spine observation of
 * the terminal step. The stash stays in device memory, for host buffers too. The field was a reserved pad (0) before:
 * the struct's layout is unchanged, and so is the ABI version. The in-kernel rollout transports have no such flag. */
typedef struct UpkieStepOutputs {
  float* obs;
  float* reward;
  uint8_t* terminated;
  uint8_t* truncated;
  float* final_obs;
  int32_t compact;      /* UpkieServos: 1 = compact rows [6][3] (position, velocity, torque) */
  int32_t final_state;  /* 1 = stash the pre-reset states of this step's same-step auto-resets */
} UpkieStepOutputs;
/* device buffers, asynchronous on `stream` */
int upkie_b200_step(void* handle, int act_dim, const float* action, const UpkieStepOutputs* out, void* stream);
/* host buffers, synchronous, as upkie_b200_step_servos_host: final_obs, when given, is stored into by the kernel
 * itself (through its mapped alias when it is pinned, else through a pinned copy of the caller's rows) */
int upkie_b200_step_host(void* handle, int act_dim, const float* action, const UpkieStepOutputs* out);

/* Replaces PyBulletBackend.get_spine_observation without side effects: returns
 * the observation assembled by the last reset/step. out[N][UPKIE_SPINE_DIM]. */
int upkie_b200_spine_obs(void* handle, float* out, void* stream);
/* Spine observation of the terminal step of a same-step auto-reset (Gymnasium's info["final_info"]): for every env that
 * reset in the last step, out[i] (device buffer [N][UPKIE_SPINE_DIM]) receives exactly what upkie_b200_spine_obs would
 * have returned after that step had the env not reset: the post-step state's observation with the same torque
 * measurement noise and IMU uncertainty (same noise keys, same row of the per-env parameter table), in spine mode the
 * observation of the pre-reset lag record. The rows of the other envs are left untouched. Needs the last call that
 * advanced or reset the simulator to be an upkie_b200_step / upkie_b200_step_host in same-step mode with
 * final_state = 1; otherwise (a step without the flag, any other step call, upkie_b200_reset, set_state, set_lag,
 * set_counters, set_elapsed, set_config, set_env_params, set_autoreset) it returns UPKIE_B200_EINVAL. The handle knows
 * which envs stashed in that step: each step with the flag has a number, which a resetting env writes to its column of
 * the stash. An addition to ABI 8: no existing layout, constant or signature changed. */
int upkie_b200_final_spine_obs(void* handle, float* out, void* stream);

/* Gyropod observation after a reset (upkie_gyropod.py:216-244): obs[N][obs_dim],
 * obs_dim 6 (gyropod) or 4 (pendulum); servo observation obs[N][6][5] for
 * UpkieServos when obs_dim = 30. */
int upkie_b200_reset_obs(void* handle, int obs_dim, float* obs, void* stream);

int upkie_b200_get_state(void* handle, float* state /* [N][UPKIE_STATE_DIM] */, void* stream);
/* Body-ground contacts of the last substep (what PyBulletBackend.get_contact_points reports for links other than the
 * tires, pybullet_backend.py:660-716): rows [N][UPKIE_BODY_REC_DIM] = bit mask of the model's collision points that
 * held rows (as a float), then for each of the UPKIE_MAX_BODY_CONTACTS slots: collision point index, normal impulse,
 * friction impulses along world -y and +x. Zero rows when the handle has no body contacts. */
#define UPKIE_BODY_REC_DIM (1 + 4 * UPKIE_MAX_BODY_CONTACTS)
int upkie_b200_get_body_contacts(void* handle, float* rows, void* stream);
/* spine mode: the lag records [N][UPKIE_LAG_DIM] (device buffers), for checkpoints and parity tests */
int upkie_b200_get_lag(void* handle, float* lag_rows, void* stream);
int upkie_b200_set_lag(void* handle, const float* lag_rows, void* stream);
int upkie_b200_set_state(void* handle, const float* state, void* stream);
int upkie_b200_error_flags(void* handle, uint32_t* flags /* [N] */, void* stream);

/* Checkpoint / resume of what get_state does not carry: per-env episode counters (keys of the on-device reset
 * sampler), tick counters (keys of the noise generator), pending next-step auto-resets and sticky error flags.
 * Device pointers, any of them may be NULL. Together with get_state / set_state, the randomisation and
 * external-force tensors the caller owns, and the seed / env_offset it passed, this is the complete simulator
 * state: a restored handle continues bit for bit (the reference has no counterpart, SURVEY.md section 5). */
int upkie_b200_get_counters(void* handle, uint32_t* episode /* [N] */, uint32_t* tick /* [N] */,
                            uint8_t* pending_reset /* [N] */, uint32_t* error_flags /* [N] */, void* stream);
int upkie_b200_set_counters(void* handle, const uint32_t* episode, const uint32_t* tick,
                            const uint8_t* pending_reset, const uint32_t* error_flags, void* stream);
/* Checkpoint / resume of the time-limit counts (UpkieSimConfig.max_episode_steps): agent steps since each env's
 * last reset, elapsed[N] (device pointer). The steps count them only while a limit is set. An env whose next-step
 * auto-reset is pending holds 0xffffffff: its reset step adds 1 and is thus not counted. */
int upkie_b200_get_elapsed(void* handle, uint32_t* elapsed, void* stream);
int upkie_b200_set_elapsed(void* handle, const uint32_t* elapsed, void* stream);

/* Replaces PyBulletBackend.set_external_forces (pybullet_backend.py:603-625):
 * force[N][UPKIE_NB][3] (device pointer, newtons) acts at the centre of mass of
 * body b of env i on every substep of every following step, until overwritten;
 * NULL clears. Bit b of `local_mask`: the force on body b is expressed in the
 * body frame (ExternalForce.local, upkie/utils/external_force.py:20-23) instead
 * of the world frame. The substep of a reset runs without them (:227-228).
 * Bodies are the lumps of UpkieModel (a force on a fixed-joint link acts at the
 * centre of mass of its lump). */
int upkie_b200_set_external_forces(void* handle, const float* force, uint32_t local_mask, void* stream);

/* Push randomisation (an addition to ABI 8: no existing layout, constant or signature changed). While a spec is set,
 * every env runs a schedule of random pushes, drawn and applied inside the step kernels. After every reset of the env
 * (both fused auto-resets, and upkie_b200_reset with device-sampled or host init rows, masked or not) it
 *   1. waits `gap` steps without a push,
 *   2. is pushed for `duration` steps by a constant world-frame force F on body `body`, acting at the body's centre
 *      of mass exactly as a force of upkie_b200_set_external_forces, and added to any force that call put there,
 *   3. draws the next (gap, duration, F) and repeats.
 * Steps are counted on the clock of max_episode_steps: the step of a next-step auto-reset is not counted. The reset
 * substep runs without external forces; the terminal step of a same-step auto-reset runs under the push then in
 * force, and the reset starts a new schedule.
 * Draw law: a per-env counter k numbers the draws, +1 at every reset and +1 at the end of every push. Draw k of the env
 * of global index g = env_offset + i (the seed and env_offset of upkie_b200_set_autoreset) is Philox4x32-10 with key
 * seed and counter (g, 2^62 | k << 4 | b) for blocks b = 0, 1, whose words w0 .. w3 of block 0 and w0 of block 1 are
 * numbered words 0 .. 4:
 *   gap      = gap_low + (((word0 >> 8) * (gap_high - gap_low + 1)) >> 24)                (integer arithmetic, exact)
 *   duration = duration_low + (((word1 >> 8) * (duration_high - duration_low + 1)) >> 24)
 *   F[a]     = min(force_low[a] + (force_high[a] - force_low[a]) * u, force_high[a]), u = (word(2 + a) >> 8) * 2^-24,
 *              in fp32 with the product rounded on its own (no FMA), a = x, y, z.
 * The tag bit 62 keeps these counters apart from those of the initial states ((episode << 2) | b) and of the reset
 * randomisation (bit 63). The schedule depends neither on the physics nor on the number of GPUs.
 * Per-env state (upkie_b200_get_push_state / set_push_state, for checkpoints): count[i] = k, the draw in force, and
 * timer[i] = steps taken since draw k was made, 0 .. gap + duration. The steps gap + 1 .. gap + duration of a draw are
 * pushed; a timer at gap + duration means the push has run out, and the next step starts draw k + 1 (a reset then
 * starts draw k + 2). A reset sets the timer to 0. A new spec restarts no counter; while no spec is set, neither steps
 * nor resets change the state.
 * Needs joint_limits != 0 (the pushes run in copies of the table and body-contact kernels). Rejected with UPKIE_B200_EINVAL, the
 * previous spec kept: body outside 0 .. UPKIE_NB - 1, a low above its high, duration_low == 0, gap_high or
 * duration_high above UPKIE_PUSH_MAX_STEPS, a force bound that is not finite, spine_mode (whose cycles take no external
 * forces), a body whose bit is set in the local_mask of upkie_b200_set_external_forces (which rejects that bit while a
 * spec pushes the body). The in-kernel rollout transports (step_servos_multicast / _peers / push rows) reject a
 * handle with a spec. NULL turns pushes off; the state stays. The call waits for the device. */
#define UPKIE_PUSH_MAX_STEPS (1u << 30)
typedef struct UpkiePushRandomization {
  int32_t body;            /* the pushed body: 0 .. UPKIE_NB - 1, the lumps of UpkieModel */
  uint32_t gap_low, gap_high;            /* steps without a push after a reset or a push, >= 0 */
  uint32_t duration_low, duration_high;  /* steps of a push, >= 1 */
  float force_low[3];      /* newtons, world frame */
  float force_high[3];
} UpkiePushRandomization;
int upkie_b200_set_push_randomization(void* handle, const UpkiePushRandomization* spec);
/* The push force applied in each env's last step, force[N][3] (device pointer, world frame); zero where that step was
 * not pushed, after a reset (whose substep runs without it), and while no spec is set. */
int upkie_b200_get_push_forces(void* handle, float* force, void* stream);
/* The per-env push state count[N], timer[N] (device pointers), see above; 0, 0 on a handle that never had one. */
int upkie_b200_get_push_state(void* handle, uint32_t* count, uint32_t* timer, void* stream);
int upkie_b200_set_push_state(void* handle, const uint32_t* count, const uint32_t* timer, void* stream);

/* Action-delay randomisation (an addition to ABI 8: no existing layout, constant or signature changed). While a spec is
 * set, every env applies its servo command d_i substeps into the tick, 0 <= d_i <= nb_substeps. The servo command is
 * the clamped [UPKIE_ACT_DIM] row the torque law reads: the clamped action of step_servos, and of step_gyropod /
 * step_pendulum the row their action front end builds from the action. A tick then runs substeps 0 .. d_i - 1 under the
 * command of the env's previous tick and substeps d_i .. nb_substeps - 1 under its own; d_i = nb_substeps runs the
 * whole tick on the previous command (one tick of latency, the most there is). The gyropod leg filter, the yaw
 * integration and the clamp flags of the error flags stay at the start of the tick; torque-control noise keeps its
 * per-substep keys.
 * At every reset of the env (both fused auto-resets, and upkie_b200_reset with device-sampled or host init rows, masked
 * or not) the previous command becomes the stop row, per joint {position NaN, velocity 0, feedforward 0, kp_scale 0,
 * kd_scale 0, maximum_torque 0}, whose torque is exactly 0 (the torque limit is applied last), and a new d_i is drawn:
 * the first d_i substeps of an episode run with the servos stopped. The reset substep runs as without a spec; the
 * terminal step of a same-step auto-reset runs under the delay in force, and its reset then applies.
 * Draw law: a per-env counter k, +1 at every reset; the reset uses draw k (after the +1). Draw k of the env of global
 * index g = env_offset + i (the seed and env_offset of upkie_b200_set_autoreset) is Philox4x32-10 with key seed and
 * counter (g, 2^61 | k << 4), whose word w0 gives
 *   d = substeps_low + (((w0 >> 8) * (substeps_high - substeps_low + 1)) >> 24)          (integer arithmetic, exact)
 * The tag bit 61 keeps these counters apart from those of the initial states ((episode << 2) | b, below 2^34), the
 * reset randomisation (bit 63) and the push randomisation (bit 62). The draws depend neither on the physics nor on the
 * number of GPUs.
 * Setting a spec draws nothing: each env keeps its delay (0 on a handle that never had a spec) until its next reset,
 * where a changed spec takes effect. NULL turns the delay off; the state stays. Per-env state
 * (upkie_b200_get_action_delay_state / set_action_delay_state, for checkpoints): count[N], delay[N] and the previous
 * command[N][UPKIE_ACT_DIM] (device pointers); 0, 0 and stop rows on a handle that never had a spec. A delay above
 * nb_substeps acts as nb_substeps.
 * Needs joint_limits != 0 (the delay runs in copies of the table and body-contact kernels). Rejected with
 * UPKIE_B200_EINVAL, the previous spec kept: substeps_low > substeps_high, substeps_high > nb_substeps, joint_limits
 * == 0, spine_mode (which models the spine's own lag). upkie_b200_set_config rejects an nb_substeps below a set spec's
 * substeps_high; the in-kernel rollout transports reject a handle with a spec. The set call waits for the device. */
typedef struct UpkieActionDelay {
  uint32_t substeps_low, substeps_high; /* range of the delay, in substeps of dt / nb_substeps */
} UpkieActionDelay;
int upkie_b200_set_action_delay(void* handle, const UpkieActionDelay* spec);
int upkie_b200_get_action_delay_state(void* handle, uint32_t* count, uint32_t* delay, float* command, void* stream);
int upkie_b200_set_action_delay_state(void* handle, const uint32_t* count, const uint32_t* delay, const float* command,
                                      void* stream);

/* Number of step-kernel launches issued through this handle since create
 * (bench.py's `gpu_launches`). */
int upkie_b200_launch_count(void* handle, uint64_t* count);

/* ---- MPC balancer handle -------------------------------------------------
 * Replaces MPCBalancer.__init__/reset/step (mpc_balancer.py:168-312). */
int upkie_b200_mpc_create(const UpkieMpcConfig* config, int n_robots, int device,
                          void** mpc);
void upkie_b200_mpc_destroy(void* mpc);
int upkie_b200_mpc_reset(void* mpc, const uint8_t* mask, void* stream);
/* x0[N][4] = (ground position, pitch, ground velocity, pitch velocity);
 * v_cmd[N] is the commanded velocity, read and updated in place
 * (MPCBalancer.commanded_velocity); first_input[N] (may be NULL) receives the
 * first optimal ground acceleration; found[N] (may be NULL) the solver status. */
int upkie_b200_mpc_step(void* mpc, const float* x0, const float* v_target,
                        const uint8_t* floor_contact, float dt, float* v_cmd,
                        float* first_input, uint8_t* found, void* stream);
/* Full optimal input sequence of the last solve, plan[N][nb_timesteps]. */
int upkie_b200_mpc_plan(void* mpc, float* plan, void* stream);

/* ---- UpkieBaseVelocity epilogue ---------------------------------------------
 * An addition to ABI 8: a new entry point and a new struct, no existing layout or signature changed, so a caller
 * built against an earlier ABI-8 header keeps working with this library.
 * Replaces the end of UpkieBaseVelocity.step (upkie/envs/upkie_base_velocity.py:194-202: dead reckoning of the
 * commanded linear velocity along the post-step yaw, observation [x, y, yaw]) and, for the envs that reset in this
 * tick, UpkieBaseVelocity.reset (upkie_base_velocity.py:137-162: MPCBalancer.reset, x = y = 0, observation
 * [0, 0, 0]). One launch per tick, after the tick's gyropod step (upkie_b200_step_gyropod / upkie_b200_step with
 * act_dim 2) and upkie_b200_spine_obs, on the stream of those calls; `mpc` is the balancer whose upkie_b200_mpc_step
 * produced the ground velocity of that step. Which envs reset is read on the device: every reset the step kernels
 * sample (both fused auto-resets) counts an episode of the sim handle, which keeps a copy of the counters as of its
 * last post step (upkie_b200_reset with init_state = NULL and upkie_b200_set_counters update that copy too). An
 * explicit upkie_b200_reset from host rows cancels a pending next-step reset and is not seen here: the caller resets
 * x, y and the balancer of those envs itself.
 * Per env i, by autoreset_mode (must equal the sim handle's, upkie_b200_set_autoreset):
 *  - no reset in this tick (always in mode 0): xy[i] += v cos(yaw) dt, v sin(yaw) dt with v = action[i][0] and
 *    yaw = gyropod_obs[i][2], each product and sum rounded to nearest fp32 (no FMA) with the IEEE cosf / sinf;
 *    obs[i] = [x, y, yaw];
 *  - reset, mode 2 (same step): final_obs[i] = [x, y, yaw] as above with the pre-reset yaw gyropod_final_obs[i][2];
 *  - reset, modes 1 and 2: xy[i] = 0, obs[i] = [0, 0, 0], commanded_velocity[i] = 0 and the mpc handle's warm start
 *    of env i is dropped (upkie_b200_mpc_reset for that env). Rows of final_obs of the other envs are left untouched.
 * Device buffers; gyropod_final_obs and final_obs are read / written in mode 2 only (may be NULL otherwise). */
typedef struct UpkieBaseVelocityPost {
  const float* action;             /* [N][2] the agent's action: commanded linear velocity, yaw velocity */
  const float* gyropod_obs;        /* [N][6] observation of this tick's gyropod step */
  const float* gyropod_final_obs;  /* [N][6] final-observation rows of that step (mode 2) */
  float* xy;                       /* [N][2] dead-reckoned position, read and updated in place */
  float* commanded_velocity;       /* [N] MPCBalancer.commanded_velocity of `mpc`, zeroed for the envs that reset */
  float* obs;                      /* [N][3] out: [x, y, yaw] */
  float* final_obs;                /* [N][3] out (mode 2): [x, y, yaw] the resetting envs reached */
  float dt;                        /* agent period (the fp32 value the dead reckoning multiplies by) */
  int32_t autoreset_mode;          /* 0 disabled, 1 next step, 2 same step */
} UpkieBaseVelocityPost;
int upkie_b200_base_velocity_post(void* handle, void* mpc, const UpkieBaseVelocityPost* args, void* stream);

/* ---- observer pipeline handle --------------------------------------------
 * Replaces the spine's BaseOrientation -> FloorContact -> WheelOdometry observers
 * (upkie/cpp/observers/, spines/common/observers.h:23-44) for N robots: one call
 * = one spine cycle. spine_obs[N][UPKIE_SPINE_DIM] supplies imu.orientation,
 * imu.angular_velocity and servo.*.{torque, velocity}; out[N][UPKIE_OBSV_DIM]. */
int upkie_b200_default_observer_config(const UpkieModel* model, UpkieObserverConfig* config);
int upkie_b200_observers_create(const UpkieObserverConfig* config, int n_robots, int device, void** observers);
void upkie_b200_observers_destroy(void* observers);
int upkie_b200_observers_reset(void* observers, const uint8_t* mask, void* stream);
int upkie_b200_observers_step(void* observers, const float* spine_obs, float* out, void* stream);

/* ---- controller pipeline handle -------------------------------------------
 * Replaces the spine's "wheel_balancer" controller pipeline
 * (spines/common/controllers.h:24-44): WheelStopper::write (WheelStopper.cpp:15-22)
 * then WheelBalancer::read / write (WheelBalancer.cpp:35-110) for N robots, one
 * call = one controller cycle of period config.dt. `obs` rows in `obs_layout`
 * supply base_orientation.pitch, floor_contact.contact and
 * wheel_odometry.position; target[N][2] = (target_ground_velocity,
 * target_yaw_velocity) of the "bullet" action key; NULL = the key is absent: ground target 0 for this cycle, the yaw
 * target keeps its last value (WheelBalancer.cpp:37-42); action[N][6][6]
 * is updated in place: wheel entries overwritten, leg kp/kd scales set. */
int upkie_b200_default_wheel_balancer_config(UpkieWheelBalancerConfig* config);
int upkie_b200_wheel_balancer_create(const UpkieWheelBalancerConfig* config, int n_robots, int device, void** balancer);
void upkie_b200_wheel_balancer_destroy(void* balancer);
int upkie_b200_wheel_balancer_reset(void* balancer, const uint8_t* mask, void* stream);
int upkie_b200_wheel_balancer_step(void* balancer, const float* obs, int obs_layout, const float* target,
                                   float* action, void* stream);
/* controller state [N][4]: ground_velocity, integral_velocity, target_ground_position, target_yaw_velocity */
int upkie_b200_wheel_balancer_state(void* balancer, float* state, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UPKIE_B200_H_ */
