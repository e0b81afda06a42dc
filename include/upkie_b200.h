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

/* Observation-delay randomisation (an addition to ABI 8: no existing layout, constant or signature changed). While a
 * spec is set, env i holds a delay d_i, 0 <= d_i <= nb_substeps, and everything a step reports about the robot's
 * sensors describes the robot at the end of substep nb_substeps - d_i of the tick, d_i substeps old: the observation of
 * all four env types (servo rows full and compact, gyropod, pendulum rows, and so UpkieBaseVelocity's), the spine
 * observation (upkie_b200_spine_obs), the same-step final_obs and upkie_b200_final_spine_obs, and
 * upkie_b200_reset_obs (whose envs a reset took report their post-reset state, the others their last snapshot). d_i = 0 is the
 * observation without a spec; d_i = nb_substeps is the state at the start of the tick (one tick of latency, the most
 * there is). The sensed fields of a state row are the base pose and twist, the joint positions and velocities, the
 * commanded torques (the measured torques are those of the last substep that ran before the snapshot, with this tick's
 * noise keys), the floor contact and the IMU pair: the IMU acceleration is the finite difference over dt of the IMU
 * velocities of two consecutive snapshots, as the undelayed observation differentiates two consecutive ticks, so the
 * sensed rows carry their own UPKIE_ST_PREV_IMU_VEL.
 * Not delayed: terminated, truncated and the auto-resets (a fall is the simulator's judgement, not a sensor's: under
 * the same actions the physics and the reset schedule do not depend on the draws), upkie_b200_get_state, the
 * contact impulses of the state rows (get_contact_points), body contacts, push forces, error flags, and the gyropod
 * wrapper's own state (yaw, yaw_vel, leg targets), which is software.
 * Every reset has no earlier state to lag behind: the env's sensed row becomes a copy of the post-reset state, so a
 * reset's observation is undelayed (both fused auto-resets, and upkie_b200_reset with device-sampled or host init rows,
 * masked or not), and a new d_i is drawn. upkie_b200_set_state copies the state into the sensed rows while a spec is
 * set. The terminal step of a same-step auto-reset is observed under the delay in force (final_obs, final spine obs).
 * Draw law: a per-env counter k, +1 at every reset; the reset uses draw k (after the +1). Draw k of the env of global
 * index g = env_offset + i (the seed and env_offset of upkie_b200_set_autoreset) is Philox4x32-10 with key seed and
 * counter (g, 2^60 | k << 4), whose word w0 gives
 *   d = substeps_low + (((w0 >> 8) * (substeps_high - substeps_low + 1)) >> 24)          (integer arithmetic, exact)
 * The tag bit 60 keeps these counters apart from those of the initial states ((episode << 2) | b, below 2^34), the
 * reset randomisation (bit 63), the pushes (bit 62) and the action delay (bit 61). The draws depend neither on the
 * physics nor on the number of GPUs.
 * Setting a spec draws nothing: each env keeps its delay (0 on a handle that never had a spec) until its next reset.
 * The first spec (or set_observation_delay_state) allocates the sensed rows and fills them from the current state; a
 * spec set while the delay is off fills them again from the current state (the sensors did not follow the robot while
 * it was off), while replacing a spec in force keeps them. NULL turns the delay off: upkie_b200_spine_obs and
 * upkie_b200_reset_obs read the true state again; the counters and delays stay for a later spec.
 * Per-env state (upkie_b200_get_observation_delay_state / set_observation_delay_state, for checkpoints): count[N],
 * delay[N] and the sensed rows[N][UPKIE_STATE_DIM] (device pointers); 0, 0 and the current state on a handle that never
 * had one. A delay above nb_substeps acts as nb_substeps.
 * Needs joint_limits != 0 (the delay runs in a copy of the table kernels). Rejected with UPKIE_B200_EINVAL, the
 * previous spec kept: substeps_low > substeps_high, substeps_high > nb_substeps, joint_limits == 0, spine_mode (which
 * models the spine's own lag), body_contacts (no body-contact copy of the kernels). upkie_b200_set_config rejects an
 * nb_substeps below a set spec's substeps_high, and turning body_contacts on while a spec is set; the in-kernel rollout
 * transports reject a handle with a spec. The set call waits for the device. */
typedef struct UpkieObservationDelay {
  uint32_t substeps_low, substeps_high; /* range of the delay, in substeps of dt / nb_substeps */
} UpkieObservationDelay;
int upkie_b200_set_observation_delay(void* handle, const UpkieObservationDelay* spec);
int upkie_b200_get_observation_delay_state(void* handle, uint32_t* count, uint32_t* delay, float* rows, void* stream);
int upkie_b200_set_observation_delay_state(void* handle, const uint32_t* count, const uint32_t* delay,
                                           const float* rows, void* stream);

/* Delays of more than one tick (an addition to ABI 8: no existing layout, constant or signature changed). Each delay
 * may keep a history of max_ticks whole ticks, 1 <= max_ticks <= UPKIE_MAX_DELAY_TICKS, and then takes any delay
 * d <= max_ticks * nb_substeps (a delay stored above acts as max_ticks * nb_substeps). upkie_b200_set_action_delay and
 * upkie_b200_set_observation_delay are the max_ticks = 1 calls. Write d = q * nb + r with 0 <= q < max_ticks and
 * 1 <= r <= nb (nb = nb_substeps; q = r = 0 for d = 0): a delay of at most one tick is q = 0, the rule above.
 * - Action delay: in tick t, substeps s < r run the servo command of tick t - q - 1 and substeps s >= r that of tick
 *   t - q. A command from before the env's last reset is the stop row, so the first d substeps of an episode run with
 *   the servos stopped. Everything else is as for one tick (leg filter, yaw, clamps and noise keys at the start of the
 *   tick, an undelayed reset substep, a same-step terminal tick under the delay in force).
 * - Observation delay: after tick t everything the step reports about the sensors (the observations, spine_obs,
 *   final_obs, the final spine observation, reset_obs of the envs a reset does not take) is the snapshot that a delay
 *   of r substeps takes in tick t - q: what a handle with delay r reported q ticks earlier under the same actions, IMU
 *   acceleration included. If tick t - q comes before the env's last reset, the report is the post-reset state.
 *   Terminations, truncations, auto-resets, get_state and the gyropod wrapper's yaw and leg targets are not delayed.
 * The draws keep their laws, counters and tags; only the range widens. A reset (fused or upkie_b200_reset) fills the
 * whole history with stop rows / the post-reset state, and upkie_b200_set_state fills the snapshots with the state.
 * Rejected with UPKIE_B200_EINVAL, the previous spec kept: max_ticks of 0 or above UPKIE_MAX_DELAY_TICKS,
 * substeps_high > max_ticks * nb_substeps, and everything the one-tick calls reject; upkie_b200_set_config rejects an
 * nb_substeps below ceil(substeps_high / max_ticks).
 * The depth may change between calls: the history is kept in age order and truncated or extended, the added commands
 * stop rows and the added snapshots copies of the oldest.
 * History (for checkpoints), in age order, index 0 the newest (device pointers): the commands [max_ticks][N]
 * [UPKIE_ACT_DIM] of the env's last ticks, and the snapshots [max_ticks][N][UPKIE_STATE_DIM] of its last ticks (at
 * depth 1 the sensed rows of get_observation_delay_state; their unsensed columns carry no meaning at depth > 1). The
 * *_delay_state calls keep their meaning: count, delay, the previous tick's command (age 0 of the history) and the
 * sensed rows the last step reported. */
#define UPKIE_MAX_DELAY_TICKS 8
int upkie_b200_set_action_delay_ticks(void* handle, const UpkieActionDelay* spec, uint32_t max_ticks);
int upkie_b200_get_action_delay_history(void* handle, float* commands, void* stream);
int upkie_b200_set_action_delay_history(void* handle, const float* commands, void* stream);
int upkie_b200_set_observation_delay_ticks(void* handle, const UpkieObservationDelay* spec, uint32_t max_ticks);
int upkie_b200_get_observation_delay_history(void* handle, float* rows, void* stream);
int upkie_b200_set_observation_delay_history(void* handle, const float* rows, void* stream);

/* ---- Servo reply dropouts (upkie/cpp/observers/observe_servos.cpp:32-52) ---------------------------------------
 * An addition to ABI 8: no existing layout, constant or signature changed. The spine refreshes a servo's observation
 * only from a reply that arrived intact: a reply that is lost (or reports a NaN torque) writes nothing, and the servo's
 * position, velocity and torque keep the values of its last good reply. While a spec is set:
 * - Draw per reset: at every reset of env i (both fused auto-resets, upkie_b200_reset with or without a mask) its loss
 *   probability p_i ~ U(prob_low, prob_high) is drawn. Draw law: a per-env counter k, +1 at every reset; draw k of the
 *   env of global index g = env_offset + i is Philox4x32-10 with key seed (upkie_b200_set_autoreset) and counter
 *   (g, 2^59 | k << 4), whose word w0 gives p_i = min(low + fl(fl(high - low) * u(w0)), high), u(w) = (w >> 8) / 2^24.
 * - Loss per cycle: every substep is one 1 kHz spine cycle. In substep s of the env's tick t (the per-env tick counter
 *   of upkie_b200_get_counters after the step), the reply of servo j of joint_mask is lost when u(w) < p_i, w word
 *   j % 4 of Philox4x32-10 with key seed and counter (g, 2^59 | 2^58 | t << 20 | s << 1 | j / 4). The tag bits 59 and
 *   58 keep these counters apart from the initial states ((episode << 2) | b, below 2^34), the reset randomisation
 *   (bit 63), the pushes (62), the action delay (61) and the observation delay (60); s < 2^19.
 * - A received reply latches the servo's q_j, qd_j and commanded torque after that substep; a lost one latches
 *   nothing. Every servo-derived output reports the latched triple: the [6][5] and compact [6][3] servo rows, the servo
 *   block of upkie_b200_spine_obs and of the final spine observation and the wheel odometry built from them, the
 *   gyropod and pendulum rows (whose p and pdot are odometry), final_obs, reset_obs, and the servo and odometry columns
 *   of every entry of an observation history. Torque measurement noise is added to the latched torque as it is added
 *   to the true one. Under an observation delay the snapshot takes the values latched at the delayed instant.
 * - Not affected: the physics, terminated, truncated, the auto-resets, the gyropod's leg targets and
 *   upkie_b200_get_state. Every reply of a reset's cycles arrives, so a reset latches the post-reset state.
 * - Off is free: with the spec off, or prob_high = 0, every output equals the same handle's without a spec.
 * Setting a spec draws nothing: each env keeps its probability (0 on a handle that never had a spec) until its next
 * reset. A spec set while the feature is off latches the current state; replacing a spec in force keeps the latched
 * values of the servos both masks hold and latches the current state of the servos it adds; NULL turns it off (the per-env state is freed once the device is idle). upkie_b200_set_state latches the
 * state set. Per-env state (get/set_servo_dropout_state, for checkpoints; device pointers): count[N], prob[N] and
 * held[N][18], the latched [joint][position, velocity, torque] of each env; UPKIE_B200_EINVAL without a spec.
 * Rejected with UPKIE_B200_EINVAL, the previous spec kept: prob_low < 0, prob_low > prob_high, prob_high > 1, a
 * joint_mask of zero or with bits above 5, joint_limits == 0 and body_contacts (it runs in the observation-delay
 * kernels), spine_mode (whose spine reports its own replies). upkie_b200_set_config rejects joint_limits = 0 and
 * body_contacts while a spec is set; the in-kernel rollout transports reject a handle with one. The set call waits for
 * the device. */
typedef struct UpkieServoDropout {
  float prob_low, prob_high; /* range of each env's per-cycle reply loss probability */
  uint32_t joint_mask;       /* bit j: servo j (UPKIE_NJ order) may lose replies */
  uint32_t reserved;         /* 0 */
} UpkieServoDropout;
int upkie_b200_set_servo_dropout(void* handle, const UpkieServoDropout* spec);
int upkie_b200_get_servo_dropout_state(void* handle, uint32_t* count, float* prob, float* held, void* stream);
int upkie_b200_set_servo_dropout_state(void* handle, const uint32_t* count, const float* prob, const float* held,
                                       void* stream);

/* ---- IMU mounting misalignment (upkie/cpp/observers/BaseOrientation.h:29-35,106-112) ---------------------------
 * An addition to ABI 8: no existing layout, constant or signature changed. The spine derives the base orientation, its
 * angular velocity and rotation_base_to_world from the IMU through a fixed rotation_base_to_imu; a board mounted
 * slightly off its nominal pose rotates every one of those readings by the mounting error. While a spec is set:
 * - Draw per reset: at every reset of env i (both fused auto-resets, upkie_b200_reset with or without a mask or host
 *   rows) three angles are drawn. Draw law: a per-env counter k, +1 at every reset; draw k of the env of global index
 *   g = env_offset + i is Philox4x32-10 with key seed (upkie_b200_set_autoreset) and counter (g, 2^57 | k << 4), whose
 *   words w0, w1, w2 give roll, pitch and yaw = min(low + fl(fl(high - low) * u(w)), high), u(w) = (w >> 8) / 2^24 (the
 *   servo dropouts' map). Tag bit 57 keeps these counters apart from the initial states (below 2^34), the reset
 *   randomisation (bit 63), the pushes (62), the action delay (61), the observation delay (60) and the servo dropouts
 *   (59, 59 | 58). The env keeps its misalignment as the unit quaternion e_i (w, x, y, z) of
 *   E_i = Rz(yaw) Ry(pitch) Rx(roll), a rotation in the base frame.
 * - Model: the true IMU frame is the nominal one rotated by E_i, and the pipeline still assumes the nominal mounting.
 *   Every orientation-derived observation is that of a robot whose base orientation is R E_i instead of R, everything
 *   else unchanged: base_orientation.pitch, base_orientation.angular_velocity ((R E)^T omega), rotation_base_to_world,
 *   imu.orientation, imu.angular_velocity, imu.linear_acceleration, imu.raw_linear_acceleration, and the gyropod and
 *   pendulum pitch and pitch rate, in the step's rows, upkie_b200_spine_obs, the final observation and final spine
 *   observation, reset_obs and every entry of an observation history. IMU bias and noise (UPKIE_EP_IMU_*) are then
 *   added in the true IMU frame as without a misalignment. Under an observation delay the misalignment is applied to
 *   the sensed snapshot when the observation is built. A same-step terminal step's final observation and final spine
 *   observation use the terminal episode's e_i, the reset observation the new one.
 * - Not affected: the physics, terminated, truncated and the auto-resets (a fall is the simulator's judgement, as for
 *   the observation delay), base_orientation.linear_velocity (world frame), the world-frame UPKIE_ST_IMU_ACC state
 *   column, the servo rows and the wheel odometry, upkie_b200_get_state, contacts and push forces.
 * Setting a spec draws nothing: each env keeps its e_i (the identity on a handle that never had a spec) until its next
 * reset; NULL turns the feature off (the per-env state is freed once the device is idle). upkie_b200_set_state and
 * explicit resets need nothing else: e_i depends on the draws only. Per-env state (get/set_imu_misalignment_state, for
 * checkpoints and for fixed offsets chosen by the caller; device pointers): count[N] and quat[N][4];
 * UPKIE_B200_EINVAL without a spec, or when a quaternion is not unit within 1e-5.
 * Rejected with UPKIE_B200_EINVAL, the previous spec kept: a bound that is not finite, low > high, |bound| > pi/4 (a
 * misalignment, not a remount), spine_mode (whose spine models its own IMU), joint_limits == 0 and body_contacts (it
 * runs in the observation-delay kernels). upkie_b200_set_config rejects joint_limits = 0 and body_contacts while a spec
 * is set; the in-kernel rollout transports reject a handle with one. The set call waits for the device. */
typedef struct UpkieImuMisalignment {
  float roll_low, roll_high;   /* radians, about the base x axis */
  float pitch_low, pitch_high; /* radians, about the base y axis */
  float yaw_low, yaw_high;     /* radians, about the base z axis */
} UpkieImuMisalignment;
int upkie_b200_set_imu_misalignment(void* handle, const UpkieImuMisalignment* spec);
int upkie_b200_get_imu_misalignment_state(void* handle, uint32_t* count, float* quat, void* stream);
int upkie_b200_set_imu_misalignment_state(void* handle, const uint32_t* count, const float* quat, void* stream);

/* ---- Servo encoder zero offsets (pi3hat_spine.cpp:181-236, moteus/QueryResult.h:33-39) --------------------------
 * An addition to ABI 8: no existing layout, constant or signature changed. The hip and knee servos are zeroed by hand
 * (upkie_tool rezero); each servo then reports its encoder position, and its position loop tracks targets in that same
 * frame. A leg zeroed off by delta reports every position shifted by delta and lands every target shifted by it.
 * While a spec is set:
 * - Draw per reset: at every reset of env i (both fused auto-resets, upkie_b200_reset with or without a mask or host
 *   rows) an offset per joint is drawn. Draw law: a per-env counter k, +1 at every reset; draw k of the env of global
 *   index g = env_offset + i is Philox4x32-10 with key seed (upkie_b200_set_autoreset) and counters
 *   (g, 2^56 | k << 4 | b), b = 0, 1; word j % 4 of block b = j / 4 gives delta_ij = min(low + fl(fl(high - low) *
 *   u(w)), high), u(w) = (w >> 8) / 2^24 (the servo dropouts' map). Every joint's word is drawn whatever the mask, and a
 *   joint outside joint_mask gets exactly 0, so that changing the mask changes no other joint's draw. Tag bit 56 keeps
 *   these counters apart from the initial states (below 2^34), the noise (below bit 42), the reset randomisation (bit
 *   63), the pushes (62), the action delay (61), the observation delay (60), the servo dropouts (59, 59 | 58) and the
 *   IMU misalignment (57).
 * - Model: the servo frame is the joint frame shifted by delta, q_servo = q + delta. Everything the agent and the
 *   wrapper exchange with the servos is in the servo frame:
 *   - reported positions are q_j + delta_ij: the [6][5] and compact [6][3] servo rows, the servo block of
 *     upkie_b200_spine_obs and of the final spine observation, the wheel odometry position (wheels in the mask), the
 *     gyropod and pendulum p, final_obs, reset_obs, and the servo-position and odometry columns of every entry of an
 *     observation history;
 *   - executed position targets are target - delta_ij, after the action clamps (which stay in the servo frame); a NaN
 *     target stays NaN;
 *   - the gyropod, pendulum and base-velocity leg targets (UPKIE_ST_LEG_TARGET) are servo-frame values: a reset sets
 *     them from the reported positions q + delta with the new episode's offsets, and they decay toward the servo zero,
 *     so that the legs settle at the physical angle -delta.
 * - Not affected: velocities and torques (torque measurement noise included), the joint-limit rows (on the true q),
 *   terminated, truncated and the auto-resets, and the q of upkie_b200_get_state, whose leg-target columns hold the
 *   servo-frame targets above.
 * - Episode boundaries: a same-step terminal step's final observation and final spine observation use the terminal
 *   episode's offsets, the reset observation and the history refilled at the reset the new ones.
 * - Composition: the offset is applied last, when an observation is built: under an observation delay to the delayed
 *   snapshot, under servo dropouts to the latched values. The dropouts' held rows, the observation-delay rows and
 *   their get/set state keep true joint values. The action-delay buffers (and get/set_action_delay_history) hold the
 *   commands as the agent sent them; the shift applies to the row the substeps execute.
 * - Off is free: with the spec off, or low = high = 0, every output is bit for bit the same handle's without a spec.
 * Setting a spec draws nothing: each env keeps its offsets (zeros on a handle that never had a spec) until its next
 * reset; a spec that replaces another zeroes the offsets of the joints it drops from the mask; NULL turns the feature
 * off (the per-env state is freed once the device is idle). Per-env state (get/set_encoder_offset_state, for
 * checkpoints and for fixed offsets measured on a robot; device pointers): count[N] and offset[N][6];
 * UPKIE_B200_EINVAL without a spec, for a value that is not finite or |value| > 0.5, and for a nonzero value of a joint
 * outside the mask.
 * Rejected with UPKIE_B200_EINVAL, the previous spec kept: a bound that is not finite, low > high, |bound| > 0.5 rad (a
 * calibration error, not a remount), a joint_mask of zero or with bits above 5, spine_mode (whose spine reports its
 * own servos), joint_limits == 0 and body_contacts (it runs in the observation-delay kernels).
 * upkie_b200_set_config rejects joint_limits = 0 and body_contacts while a spec is set; the in-kernel rollout
 * transports reject a handle with one. The set call waits for the device. */
typedef struct UpkieEncoderOffset {
  float low, high;     /* radians, range of each joint's zero offset */
  uint32_t joint_mask; /* bit j: joint j (UPKIE_NJ order) has an offset */
  uint32_t reserved;   /* 0 */
} UpkieEncoderOffset;
int upkie_b200_set_encoder_offset(void* handle, const UpkieEncoderOffset* spec);
int upkie_b200_get_encoder_offset_state(void* handle, uint32_t* count, float* offset, void* stream);
int upkie_b200_set_encoder_offset_state(void* handle, const uint32_t* count, const float* offset, void* stream);

/* ---- Servo measurement noise (observe_servos.cpp:62-75, pybullet_backend.py:448-466) ------------------------------
 * An addition to ABI 8: no existing layout, constant or signature changed. Each servo reply carries the moteus
 * encoder's estimates of position and velocity, which reach the spine once per cycle; the velocity estimate is visibly
 * noisy. The torque reply keeps its own noise (UPKIE_EP_MEAS_NOISE). While a spec is set:
 * - Draw per reset: at every reset of env i (both fused auto-resets, upkie_b200_reset with or without a mask or host
 *   rows) twelve standard deviations are drawn, columns 0-5 the position noise of joints 0-5 (UPKIE_NJ order), 6-11 the
 *   velocity noise. Draw law: a per-env counter k, +1 at every reset; draw k of the env of global index
 *   g = env_offset + i is Philox4x32-10 with key seed (upkie_b200_set_autoreset) and counters (g, 2^55 | k << 4 | b),
 *   b = 0, 1, 2; word c % 4 of block c / 4 gives sigma_ic = min(low_c + fl(fl(high_c - low_c) * u(w)), high_c),
 *   u(w) = (w >> 8) / 2^24 (the servo dropouts' map). Every column is drawn whatever the ranges, so that changing one
 *   joint's range changes no other joint's draw.
 * - Noise per cycle: every reported position and velocity is the true value plus sigma * n, n a standard normal that
 *   depends only on (seed, g, the cycle reported, joint, quantity). Cycle s (0 .. nb_substeps - 1) of tick t (the
 *   per-env tick counter after the step, as the dropout losses use it) draws counters (g, 2^55 | 2^54 | t << 20 |
 *   s << 2 | b), b = 0, 1, 2; the twelve words pass in pairs through gaussian8's Box-Muller transform (normal c from
 *   words 2p, 2p + 1 of block c / 4, p = (c % 4) / 2, the cosine for even c). A reset's observation is a cycle of its
 *   own, (g, 2^55 | 2^54 | 2^53 | k << 2 | b) with the draw counter k after the reset, which every reset advances
 *   (with host rows too, which do not count an episode): it never coincides with a step cycle, and two resets of an env
 *   report different normals unless a restart of the counters (a set_servo_noise_state with count 0, as
 *   B200VectorEnv.reset(seed=s) does) repeats a draw on purpose. A cycle reported twice reports the same value.
 *   Tag bit 55 keeps these counters apart from the initial states (below 2^34), the noise (below bit 42), the reset
 *   randomisation (bit 63), the pushes (62), the action delay (61), the observation delay (60), the servo dropouts
 *   (59, 59 | 58), the IMU misalignment (57) and the encoder offsets (56).
 * - Where it appears: wherever the encoder offsets appear: the [6][5] and compact [6][3] servo rows, the servo block of
 *   upkie_b200_spine_obs and of the final spine observation and the wheel odometry built from them, the gyropod and
 *   pendulum p and pdot, final_obs, reset_obs, and the servo-position, servo-velocity and odometry columns of every
 *   history entry, each entry with the noise of its own cycle. A ring a reset refills holds the reset observation as
 *   its newest entry and, as each older entry, the post-reset state with the noise of the cycle that entry stands for.
 * - Composition: the reported position is fl(fl(q + fl(sigma_q * n_q)) + delta) with the encoder offset delta, the
 *   velocity fl(qd + fl(sigma_v * n_v)). Under an observation delay the noise is that of the cycle observed, d
 *   substeps before the tick's last cycle (d = min(delay, K * nb_substeps), K the delay's depth in ticks), applied to
 *   the snapshot when the observation is built; a snapshot that a reset refilled is reported with the noise of the
 *   cycle it stands for. Under servo dropouts a lost reply repeats the last received reply as it was received: the
 *   held rows latch the noisy position and velocity (the reset latches the reset observation's). The gyropod,
 *   pendulum and base-velocity leg targets a reset sets from the reported hip and knee positions include the reset
 *   cycle's noise. upkie_b200_spine_obs and upkie_b200_reset_obs report the reset cycle for the envs whose last event
 *   was a reset, the last step's observed cycle for the others: a per-env mark, 1 after a reset and 0 after a step that
 *   does not reset (get/set_servo_noise_mark, mark[N] of 0 or 1, for checkpoints; a spec switched on starts every env
 *   at 0).
 * - Not affected: the physics (the servo's torque law runs on the true q and qd: this models the reply, not the
 *   servo's internal estimate), the joint-limit rows, terminated, truncated and the auto-resets, the torques, the q and
 *   qd of upkie_b200_get_state (whose leg-target columns hold the reset targets above; k_reset does not know the env
 *   type, so UpkieServos handles carry them too, unused), the observation-delay rows and their get/set state, and
 *   UPKIE_EP_DIM.
 * - Off is free: with the spec off, or every high bound 0, every output is bit for bit the same handle's without one.
 * Setting a spec draws nothing: each env keeps its sigmas (zeros on a handle that never had a spec) until its next
 * reset; a spec that replaces another zeroes the columns whose high bound is 0; NULL turns the feature off (the per-env
 * state is freed once the device is idle). Per-env state (get/set_servo_noise_state, for checkpoints; device
 * pointers): count[N] and sigma[N][12]; UPKIE_B200_EINVAL without a spec, for a sigma that is not finite or negative,
 * above the caps of every spec (0.1 rad for a position, 5 rad/s for a velocity: a narrower spec leaves each env's
 * sigmas until its next reset, so the spec in force does not bound them), or nonzero in a column whose high bound is
 * zero in the spec in force.
 * Rejected with UPKIE_B200_EINVAL, the previous spec kept: a bound that is not finite, a negative low bound, low > high,
 * a position high above 0.1 rad or a velocity high above 5 rad/s (a sensor noise, not a broken encoder), spine_mode
 * (whose spine reports its own servos), joint_limits == 0 and body_contacts (it runs in the observation-delay kernels),
 * and an observation delay together with servo dropouts (a delayed snapshot does not record which of its replies were
 * held). upkie_b200_set_config rejects joint_limits = 0 and body_contacts while a spec is set, and
 * upkie_b200_set_observation_delay(_ticks) and upkie_b200_set_servo_dropout reject the third of the three; the in-kernel
 * rollout transports reject a handle with a spec. The set call waits for the device. */
typedef struct UpkieServoNoise {
  float position_low[6], position_high[6]; /* rad, range of each joint's position noise std (UPKIE_NJ order) */
  float velocity_low[6], velocity_high[6]; /* rad/s, range of each joint's velocity noise std */
} UpkieServoNoise;
int upkie_b200_set_servo_noise(void* handle, const UpkieServoNoise* spec);
int upkie_b200_get_servo_noise_state(void* handle, uint32_t* count, float* sigma, void* stream);
int upkie_b200_set_servo_noise_state(void* handle, const uint32_t* count, const float* sigma, void* stream);
int upkie_b200_get_servo_noise_mark(void* handle, uint8_t* mark, void* stream);
int upkie_b200_set_servo_noise_mark(void* handle, const uint8_t* mark, void* stream);

/* ---- Servo velocity limits (tools/configure_servos:99-104, moteus servo.max_velocity) -----------------------------
 * An addition to ABI 8: no existing layout, constant or signature changed. Every Upkie's servos are configured with a
 * velocity limit (servo.max_velocity: 2 rev/s on the hips and knees, 8 rev/s on the wheels); past it the moteus
 * firmware reduces its output, which reaches zero at max_velocity + servo.max_velocity_derate. The model implemented
 * here rests on two assumptions taken from the moteus documentation, not from a source in this project: the derate
 * band's default of 2 rev/s (UPKIE_VELOCITY_DERATE in upkie_b200.envs), and that only motoring torque is limited.
 * While a spec is set:
 * - Draw per reset: at every reset of env i (both fused auto-resets, upkie_b200_reset with or without a mask or host
 *   rows) a limit per joint is drawn. Draw law: a per-env counter k, +1 at every reset; draw k of the env of global
 *   index g = env_offset + i is Philox4x32-10 with key seed (upkie_b200_set_autoreset) and counters
 *   (g, 2^52 | k << 4 | b), b = 0, 1; word j % 4 of block b = j / 4 gives v_ij = min(low_j + fl(fl(high_j - low_j) *
 *   u(w)), high_j), u(w) = (w >> 8) / 2^24 (the servo dropouts' map). Every joint's word is drawn whatever the mask,
 *   and a joint outside joint_mask stores exactly 0, so that changing the mask changes no other joint's draw. Tag bit
 *   52 keeps these counters apart from the initial states (below 2^34), the noise (below bit 42), the reset
 *   randomisation (bit 63), the pushes (62), the action delay (61), the observation delay (60), the servo dropouts (59,
 *   59 | 58, below bit 52 otherwise), the IMU misalignment (57), the encoder offsets (56) and the servo noise (55,
 *   55 | 54 below bit 52, 55 | 54 | 53).
 * - Law: in every substep, t is the torque of the servo law as without a spec (PD law, joint friction and control
 *   noise, clipped to +-maximum_torque). For a joint of the mask with |qd| > v_ij (qd the true joint velocity of the
 *   substep): f = clamp((v_ij + derate_j - |qd|) / derate_j, 0, 1), cap = f * tau_max_j (the model's effort limit),
 *   and t = min(t, cap) for qd > 0, max(t, -cap) for qd < 0. A torque that brakes the joint passes unchanged, and
 *   below the limit t is left bit for bit. The derated torque is what the physics integrates and what the torque
 *   replies report (torque measurement noise added on top of it). External forces and pushes are added after the law,
 *   the action delay's command is derated like any other, and the zero-torque substep of a reset is untouched.
 * - Not affected: the observations but the torque, servo noise, encoder offsets and delays (the law runs on the true
 *   qd), the velocity target clamp (qd_max) and max_coordinate_velocity.
 * Setting a spec draws nothing: each env keeps the limits of the joints that stay in the mask until its next reset;
 * the joints a spec adds to the mask (every joint of the first spec) take max_velocity_high until then, and the joints
 * it drops store 0. NULL turns the feature off (the per-env state is freed once the device is idle). Per-env state
 * (get/set_velocity_derate_state, for checkpoints and fixed limits; device pointers): count[N] and
 * max_velocity[N][6] in rad/s; UPKIE_B200_EINVAL without a spec, for a value of a joint of the mask in force that is
 * not finite or <= 0, and for a nonzero value of a joint outside it.
 * Rejected with UPKIE_B200_EINVAL, the previous spec kept: a bound that is not finite, max_velocity_low <= 0 or
 * low > high or derate <= 0 on a joint of the mask, a joint_mask of zero or with bits above 5, reserved != 0,
 * spine_mode (whose spine applies its own torque law), joint_limits == 0 and body_contacts (it runs in the
 * observation-delay kernels). upkie_b200_set_config rejects joint_limits = 0 and body_contacts while a spec is set;
 * the in-kernel rollout transports reject a handle with one. The set call waits for the device. */
typedef struct UpkieVelocityDerate {
  float max_velocity_low[6], max_velocity_high[6]; /* rad/s, range of each joint's velocity limit (UPKIE_NJ order) */
  float derate[6];     /* rad/s, the band past the limit over which the motoring torque falls to zero */
  uint32_t joint_mask; /* bit j: joint j has a velocity limit */
  uint32_t reserved;   /* 0 */
} UpkieVelocityDerate;
int upkie_b200_set_velocity_derate(void* handle, const UpkieVelocityDerate* spec);
int upkie_b200_get_velocity_derate_state(void* handle, uint32_t* count, float* max_velocity, void* stream);
int upkie_b200_set_velocity_derate_state(void* handle, const uint32_t* count, const float* max_velocity, void* stream);

/* ---- IMU attitude estimation (Pi3HatInterface.cpp:151-169, pi3hat/imu.h:84-95) ----------------------------------
 * An addition to ABI 8: no existing layout, constant or signature changed. On the robot the spine never sees the true
 * tilt: it reads orientation_imu_in_ars from the pi3hat's attitude filter, which has its own gyro-bias estimate. While
 * a spec is set every env runs an attitude filter on its simulated IMU, and every orientation-derived observation
 * reports its estimate instead of the true orientation.
 * Assumption: the pi3hat's filter is an unscented Kalman filter whose source is in neither this project nor its
 * reference. The model implemented here is an explicit complementary filter with gyro-bias estimation (Mahony), chosen
 * because it has the three error classes of such a filter (convergence after a start or a disturbance, a tilt error
 * toward atan(a / g) under sustained horizontal acceleration, drift from a gyro bias not yet estimated) and is cheap
 * enough to run in every spine cycle. It does not reproduce the UKF's gains or transients.
 * - Per-env state (device pointers): count[N], gains[N][2] (kp in 1/s, ki in 1/s^2), quat[N][4] (w, x, y, z: the
 *   estimated IMU-to-world rotation q) and bias[N][3] (b, rad/s, IMU frame).
 * - Law: once per substep (one 1 kHz spine cycle at the default 200 Hz / 5 substeps), after that substep's physics,
 *   with h = dt / nb_substeps. Inputs, in the true IMU frame (the misaligned one under an IMU misalignment):
 *   w_m = R_i^T omega + the env's gyro bias, and a_m = R_i^T ((v_i - v_i') / h + 9.81 e_z) + the env's accelerometer
 *   bias, with R_i the IMU-to-world rotation, v_i the world-frame IMU velocity after the substep and v_i' the one
 *   after the previous substep (the step's observation update's at the first substep of a tick), as the observation
 *   history differentiates it. The biases are the parameter table's columns, or the config's (ImuUncertainty). The
 *   white IMU noise is not an input: it stays a per-step draw on the report (drawing it in every substep would cost
 *   two more Philox blocks per substep). In float, in this order:
 *     v = (2 (x z - y w), 2 (y z + x w), 1 - 2 (x x + y y))      R(q)^T e_z, the predicted "up" in the IMU frame
 *     n = |a_m|; e = n > 1e-3 ? (a_m * (1 / n)) x v : 0
 *     b_k = b_k - (ki * e_k) * h;  w_k = (w_m,k - b_k) + kp * e_k
 *     t = 0.5 * |w| * h; if |w| > 0: c = cos t, s = sin t / |w| (t < 0.25: c = 1 - t^2 (1/2 - t^2 (1/24 - t^2 / 720)),
 *     s = 0.5 h (1 - t^2 (1/6 - t^2 (1/120 - t^2 / 5040)))), r = q (x) (c, s w), q = r * (1 / |r|); q unchanged at |w| = 0.
 * - Draw per reset: at every reset of env i (both fused auto-resets, upkie_b200_reset with or without a mask or host
 *   rows) a per-env counter k goes up by 1, and Philox4x32-10 with key seed (upkie_b200_set_autoreset) and counters
 *   (g, 2^51 | k << 4), g = env_offset + i, gives four words: kp, ki, roll and pitch, each
 *   min(low + fl(fl(high - low) * u(w)), high), u(w) = (w >> 8) / 2^24 (the servo dropouts' map). Tag bit 51 alone
 *   keeps these counters apart from every tag listed in the velocity-limit block above (63 ... 52) and from the cycle
 *   counters below bit 52, which carry bits 59 | 58 or 55 | 54.
 * - Initialisation: after the reset substep, the estimate is that of a base oriented R_b E (the estimate taken back to
 *   the base through the nominal rotation_base_to_imu), R_b the observed (misaligned) base orientation of the
 *   post-reset state and E = Ry(pitch) Rx(roll) the drawn error, a rotation in the base frame; b = 0.
 *   upkie_b200_set_state re-initialises every env the same way with E = I, keeping gains and counts (the sensors see
 *   the state set).
 * - Where it appears: imu.orientation, base_orientation.pitch, base_orientation.rotation_base_to_world (the estimate
 *   taken back to the base) and the gyropod and pendulum pitch: in step rows, upkie_b200_spine_obs, reset_obs, the
 *   final observation and final spine observation, and the UPKIE_SP_IMU_QUAT / PITCH / ROT columns of every history
 *   entry (each the estimate after its own substep). Under an observation delay of one tick the report is the estimate
 *   of the cycle observed. A same-step auto-reset's final observation carries the terminal episode's estimate.
 * - Not affected: every angular velocity (the gyro's true-frame rates), the accelerations, the linear velocity, the
 *   servo rows and odometry, the physics, terminations and auto-resets (a fall stays the simulator's judgement), and
 *   upkie_b200_get_state.
 * Setting a spec draws nothing: an env of a handle that had no filter takes kp_high and ki_high, the true orientation
 * and b = 0 until its next reset; a replacement keeps each env's state. NULL turns the filter off (the per-env state is
 * freed once the device is idle). Either invalidates the last step's stash of terminal states
 * (upkie_b200_final_spine_obs), whose layout follows the spec. get/set_attitude_filter_state: UPKIE_B200_EINVAL without
 * a spec, and for a quaternion that is not unit within 1e-5, a value that is not finite, or gains outside the caps
 * below. get/set_attitude_filter_report: report[N][4], the estimate each env's observation reports under an
 * observation delay (that of the cycle its snapshot observed; a checkpoint carries it, as it carries the snapshot);
 * set_attitude_filter_state leaves it, as setting the estimate leaves the snapshot; UPKIE_B200_EINVAL for a
 * quaternion that is not unit within 1e-5.
 * Rejected with UPKIE_B200_EINVAL, the previous spec kept: a bound that is not finite or low > high; kp_low < 0 or
 * kp_high * h > 0.5 (the discrete correction must not overshoot); ki_low < 0 or ki_high > 10; a roll or pitch bound
 * beyond pi/4 in magnitude; spine_mode, joint_limits == 0 and body_contacts (it runs in the observation-delay kernels);
 * an observation delay of more than one tick (upkie_b200_set_observation_delay_ticks with max_ticks > 1, refused in
 * both orders: the report of a deeper delay would need a ring of estimates). upkie_b200_set_config refuses
 * joint_limits = 0, body_contacts and a dt / nb_substeps for which kp * h > 0.5 for the largest kp an env holds or
 * the spec's kp_high while a spec is set; the in-kernel rollout transports reject a handle with one. The set call waits
 * for the device. */
typedef struct UpkieAttitudeFilter {
  float kp_low, kp_high;       /* 1/s, proportional gain of the accelerometer correction */
  float ki_low, ki_high;       /* 1/s^2, integral gain of the gyro-bias estimate */
  float roll_low, roll_high;   /* rad, initial estimate error about the base x axis */
  float pitch_low, pitch_high; /* rad, initial estimate error about the base y axis */
} UpkieAttitudeFilter;
int upkie_b200_set_attitude_filter(void* handle, const UpkieAttitudeFilter* spec);
int upkie_b200_get_attitude_filter_state(void* handle, uint32_t* count, float* gains, float* quat, float* bias,
                                         void* stream);
int upkie_b200_set_attitude_filter_state(void* handle, const uint32_t* count, const float* gains, const float* quat,
                                         const float* bias, void* stream);
int upkie_b200_get_attitude_filter_report(void* handle, float* quat, void* stream);
int upkie_b200_set_attitude_filter_report(void* handle, const float* quat, void* stream);

/* ---- Servo torque-constant errors (pybullet_backend.py:457-459, moteus current loop) -----------------------------
 * An addition to ABI 8: no existing layout, constant or signature changed. The reference applies every commanded
 * torque exactly and reports it as measured. A moteus servo closes its loop on current and converts it to torque
 * through a nominal torque constant, and it reports that same estimate; the torque its joint receives differs by the
 * constant's error and the gearbox losses, from motor to motor. While a spec is set each joint of each env delivers a
 * scale s_ij of the torque its servo commands and reports ("motor strength" in legged-robot RL, where (0.9, 1.1) is a
 * usual range; no measured tolerance of the Upkie's servos is known to this project).
 * - Draw per reset: at every reset of env i (both fused auto-resets, upkie_b200_reset with or without a mask or host
 *   rows) a per-env counter k goes up by 1, and Philox4x32-10 with key seed (upkie_b200_set_autoreset) and counters
 *   (g, 2^50 | k << 4 | b), b = 0, 1, g = env_offset + i, gives joint j word j % 4 of block b = j / 4:
 *   s_ij = min(low_j + fl(fl(high_j - low_j) * u(w)), high_j), u(w) = (w >> 8) / 2^24 (the servo dropouts' map). Every
 *   joint's word is drawn whatever the mask, and a joint outside joint_mask stores exactly 1, so that changing the mask
 *   changes no other joint's draw. Tag bit 50 alone keeps these counters apart from every tag listed above (63 ... 51)
 *   and from the cycle counters below bit 52, which carry bits 59 | 58 or 55 | 54.
 * - Law: in every substep, t is the torque of the servo law as without a spec (PD law, joint friction and control
 *   noise, clipped to +-maximum_torque, then the velocity limit's derate if one is set). The torque reply is t (what
 *   the servo believes it applies; torque measurement noise added on top of it), and the physics integrates
 *   fl(s_ij * t) (rounded once: never contracted into the substep's next add). External forces and pushes are added
 *   after the scale, unscaled; the action delay's command is scaled like any other; the zero-torque substep of a reset
 *   stays zero. Consequences of keeping the reference's law: the joint friction, folded into the command before the
 *   clip (pybullet_backend.py:537-552), is scaled with it, and the velocity derate acts on the servo's side, so that
 *   its cap is s_ij * f * tau_max in delivered torque.
 * - Not affected: every observation but through the physics (the torque replies of step rows, upkie_b200_spine_obs,
 *   history entries, final and reset observations, and the UPKIE_ST_TORQUE columns of upkie_b200_get_state all report
 *   t), terminations and auto-resets, and the stash of terminal states (whose layout does not change).
 * Setting a spec draws nothing: each env keeps the scales of the joints that stay in the mask until its next reset;
 * the joints a spec adds to the mask (every joint of the first spec) hold 1 until then, and the joints it drops store
 * 1. NULL turns the feature off (the per-env state is freed once the device is idle). Per-env state
 * (get/set_torque_scale_state, for checkpoints and fixed scales; device pointers): count[N] and scale[N][6];
 * UPKIE_B200_EINVAL without a spec, for a value of a joint of the mask in force that is not finite or outside (0, 2],
 * and for a value other than exactly 1 of a joint outside it.
 * Rejected with UPKIE_B200_EINVAL, the previous spec kept: a bound that is not finite, low <= 0, low > high or
 * high > 2 on a joint of the mask, a joint_mask of zero or with bits above 5, reserved != 0, spine_mode (whose spine
 * applies its own torque law), joint_limits == 0 and body_contacts (it runs in the observation-delay kernels).
 * upkie_b200_set_config rejects joint_limits = 0 and body_contacts while a spec is set; the in-kernel rollout
 * transports reject a handle with one. The set call waits for the device. */
typedef struct UpkieTorqueScale {
  float scale_low[6], scale_high[6]; /* dimensionless, range of each joint's delivered-torque scale (UPKIE_NJ order) */
  uint32_t joint_mask;               /* bit j: joint j's delivered torque is scaled */
  uint32_t reserved;                 /* 0 */
} UpkieTorqueScale;
int upkie_b200_set_torque_scale(void* handle, const UpkieTorqueScale* spec);
int upkie_b200_get_torque_scale_state(void* handle, uint32_t* count, float* scale, void* stream);
int upkie_b200_set_torque_scale_state(void* handle, const uint32_t* count, const float* scale, void* stream);

/* ---- Spine-rate observation history (HistoryObserver.h, upkie/cpp/observers/) ----------------------------------
 * An addition to ABI 8: no existing layout, constant or signature changed. The step runs nb_substeps substeps per
 * tick, each one cycle of a 1 kHz spine at the default 200 Hz / 5 substeps. A history makes each env report the last
 * K substeps of chosen columns of its spine observation, as a HistoryObserver in the spine's observer pipeline reports
 * its vector of the last `size` values of a key (HistoryObserver::read_value pushes each cycle's value to the front).
 * At 1 kHz, where a tick is one substep, it is plain per-tick frame stacking.
 * Spec: `count` = C columns of the spine observation row (UPKIE_SP_*, 0 .. UPKIE_SPINE_DIM - 1), 1 <= C <=
 * UPKIE_MAX_HISTORY_CHANNELS, and `size` = K entries, 1 <= K <= UPKIE_MAX_HISTORY.
 * - After a step, entry 0 (the newest) holds each column as it was after the tick's last substep, and entry k as it
 *   was k substeps earlier; entries cross tick boundaries when K > nb_substeps. Newest first, as HistoryObserver.
 * - Every column has the arithmetic of upkie_b200_spine_obs applied to the state after that substep, except two:
 *   the IMU linear and raw accelerations differentiate the IMU velocity over one substep dt / nb_substeps, as a 1 kHz
 *   spine does (the tick's own observation keeps its difference over dt), and the servo torques are those applied in
 *   the substep, without measurement noise. No IMU uncertainty is added.
 * - Under an observation delay of d substeps, entry 0 is the instant the observation reports, d substeps before the
 *   end of the tick, and the window moves back with it: entry 0 then equals the delayed spine observation's columns
 *   (but for the two exceptions above). The ring holds K + max_ticks * nb_substeps entries, max_ticks the observation
 *   delay's depth (1 without upkie_b200_set_observation_delay_ticks).
 * - Every reset of an env (fused next-step or same-step auto-reset, upkie_b200_reset with or without a mask) fills all
 *   of that env's entries with its post-reset observation's columns (IMU acceleration: the reset's); the other envs
 *   keep theirs. The reference's HistoryObserver keeps its vector across a spine reset: here a new episode starts
 *   without the previous episode's samples. A new spec, upkie_b200_set_state, and a change of the ring's size (a new
 *   observation-delay depth, a new nb_substeps) fill every env's entries from the current state in the same way.
 * - The history records only: observations, rewards, terminations, truncations, final_obs, the final spine
 *   observation, the state and every draw are those of the same handle without a history. It runs in the kernels of
 *   the observation delay (FAM_SENSE), so it needs joint_limits != 0 and is rejected with spine_mode (whose spine
 *   reports lagged replies) and with body_contacts; the in-kernel rollout transports reject a handle with a history.
 * upkie_b200_set_history: NULL turns it off (the ring is freed once the device is idle); an invalid spec returns
 * UPKIE_B200_EINVAL and keeps the previous one. upkie_b200_set_config rejects joint_limits = 0 and body_contacts while
 * a history is set. The set call waits for the device. upkie_b200_get_history: out[N][K][C] (device pointer), env i's
 * entries newest first; without a history, UPKIE_B200_EINVAL. Checkpoints: upkie_b200_get_history_state /
 * set_history_state copy the whole ring in age order, rows[ticks][N][C] with ticks = upkie_b200_history_entries (age 0
 * the entry the last substep wrote); the ring's head is implied by the age order. */
#define UPKIE_MAX_HISTORY 64
#define UPKIE_MAX_HISTORY_CHANNELS 16
typedef struct UpkieHistory {
  uint32_t size;                                /* K, entries reported */
  uint32_t count;                               /* C, columns */
  int32_t columns[UPKIE_MAX_HISTORY_CHANNELS];  /* UPKIE_SP_* columns, the first `count` used */
} UpkieHistory;
int upkie_b200_set_history(void* handle, const UpkieHistory* spec);
int upkie_b200_get_history(void* handle, float* out, void* stream);
int upkie_b200_history_entries(void* handle, int* ticks);
int upkie_b200_get_history_state(void* handle, float* rows, void* stream);
int upkie_b200_set_history_state(void* handle, const float* rows, void* stream);

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
