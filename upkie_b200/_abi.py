# SPDX-License-Identifier: Apache-2.0
"""ctypes mirror of ``include/upkie_b200.h`` (struct layouts and constants).

Kept in one place so that the product loader (``upkie_b200._lib``) and the test
infrastructure bind the very same layouts. The constants follow the reference:
action keys ``upkie/envs/upkie_servos.py:98-105``, observation keys
``upkie/envs/upkie_servos.py:221-253``, spine observation dictionary
``upkie/envs/backends/pybullet_backend.py:313-331``.
"""

import ctypes as C
import math

import numpy as np

ABI_VERSION = 8
LAG_REPLY1, LAG_REPLY2, LAG_IMU, LAG_OBS_REPLY, LAG_OBS_IMU, LAG_OBS_BASE, LAG_OBS_CONTACT, LAG_DIM = 0, 18, 36, 49, 67, 80, 90, 91  # spine-mode lag record (include/upkie_b200.h)

NJ = 6
NB = 7
MAX_COLLISION_POINTS = 16  # UPKIE_MAX_COLLISION_POINTS
MAX_BODY_CONTACTS = 4  # UPKIE_MAX_BODY_CONTACTS
BODY_REC_DIM = 1 + 4 * MAX_BODY_CONTACTS  # rows of upkie_b200_get_body_contacts

ACT_KEYS = (
    "position",
    "velocity",
    "feedforward_torque",
    "kp_scale",
    "kd_scale",
    "maximum_torque",
)
OBS_KEYS = ("position", "velocity", "torque", "temperature", "voltage")
JOINT_NAMES = (
    "left_hip",
    "left_knee",
    "left_wheel",
    "right_hip",
    "right_knee",
    "right_wheel",
)
UPPER_LEG_JOINTS = (0, 1, 3, 4)
WHEEL_JOINTS = (2, 5)

ACT_DIM = 36
OBS_DIM = 30
INIT_DIM = 25
STATE_DIM = 50
SPINE_DIM = 62

# init_state offsets
INIT_POS, INIT_QUAT, INIT_LINVEL, INIT_ANGVEL, INIT_Q, INIT_QD = 0, 3, 7, 10, 13, 19
# state offsets
ST_POS, ST_QUAT, ST_LINVEL, ST_ANGVEL, ST_Q, ST_QD = 0, 3, 7, 10, 13, 19
ST_PREV_IMU_VEL, ST_TORQUE, ST_LEG_TARGET, ST_YAW, ST_YAW_VEL, ST_CONTACT = 25, 28, 34, 38, 39, 40
ST_IMU_ACC = 41
ST_CONTACT_IMPULSE = 44
ST_FRICTION_IMPULSE = 46  # rolling / lateral friction impulses of the last substep, left wheel then right wheel
# per-env parameter table (upkie_b200_set_env_params): row offsets, UPKIE_EP_* of include/upkie_b200.h
EP_KP, EP_KD, EP_FRICTION, EP_CTRL_NOISE, EP_MEAS_NOISE = 0, 1, 2, 8, 14
EP_IMU_ACC_BIAS, EP_IMU_ACC_NOISE, EP_IMU_GYRO_BIAS, EP_IMU_GYRO_NOISE = 20, 23, 24, 27
EP_DIM = 28
# reset randomisation (upkie_b200_set_reset_randomization): columns 0 .. EP_DIM - 1 are the table's, then UPKIE_RR_*
RR_INERTIA, RR_FRICTION, RR_DIM = 28, 34, 35
# spine observation offsets
SP_BASE_ANGVEL, SP_BASE_LINVEL, SP_PITCH, SP_ROT = 0, 3, 6, 7
SP_IMU_QUAT, SP_IMU_ANGVEL, SP_IMU_LINACC, SP_IMU_RAWACC = 16, 20, 23, 26
SP_CONTACT, SP_SERVO, SP_ODOM_POS, SP_ODOM_VEL = 29, 30, 60, 61

ERR_NAN_VELOCITY, ERR_NAN_STATE, ERR_CLAMPED = 1, 2, 4


class UpkieModel(C.Structure):
    _fields_ = [
        ("parent", C.c_int32 * NB),
        ("left_wheeled", C.c_int32),
        ("joint_origin", (C.c_double * 3) * NJ),
        ("joint_axis", (C.c_double * 3) * NJ),
        ("mass", C.c_double * NB),
        ("com", (C.c_double * 3) * NB),
        ("inertia", (C.c_double * 6) * NB),
        ("q_lower", C.c_double * NJ),
        ("q_upper", C.c_double * NJ),
        ("qd_max", C.c_double * NJ),
        ("tau_max", C.c_double * NJ),
        ("wheel_radius", C.c_double),
        ("wheel_base", C.c_double),
        ("imu_position", C.c_double * 3),
        ("rotation_base_to_imu", C.c_double * 9),
        ("n_collision_points", C.c_int32),
        ("collision_body", C.c_int32 * MAX_COLLISION_POINTS),
        ("reserved_collision", C.c_int32),
        ("collision_point", (C.c_double * 3) * MAX_COLLISION_POINTS),
        ("collision_radius", C.c_double * MAX_COLLISION_POINTS),
    ]


class UpkieSimConfig(C.Structure):
    _fields_ = [
        ("dt", C.c_double),
        ("nb_substeps", C.c_int32),
        ("pgs_iterations", C.c_int32),
        ("gravity", C.c_double),
        ("torque_control_kp", C.c_double),
        ("torque_control_kd", C.c_double),
        ("joint_friction", C.c_double * NJ),
        ("torque_control_noise", C.c_double * NJ),
        ("torque_measurement_noise", C.c_double * NJ),
        ("imu_accelerometer_bias", C.c_double * 3),
        ("imu_accelerometer_noise", C.c_double),
        ("imu_gyroscope_bias", C.c_double * 3),
        ("imu_gyroscope_noise", C.c_double),
        ("noise_seed", C.c_uint64),
        ("linear_damping", C.c_double),
        ("angular_damping", C.c_double),
        ("max_coordinate_velocity", C.c_double),
        ("contact_stiffness", C.c_double),
        ("contact_damping", C.c_double),
        ("contact_breaking_threshold", C.c_double),
        ("friction", C.c_double),
        ("max_gain_scale", C.c_double),
        ("fall_pitch", C.c_double),
        ("leg_gain_scale", C.c_double),
        ("max_ground_velocity", C.c_double),
        ("max_yaw_velocity", C.c_double),
        ("servos_fall_termination", C.c_int32),
        ("skip_action_clamps", C.c_int32),
        ("min_base_height", C.c_double),
        ("pgs_tolerance", C.c_double),
        ("warmstarting_factor", C.c_double),
        ("joint_limits", C.c_int32),
        ("reserved_joint_limits", C.c_int32),
        ("joint_limit_erp", C.c_double),
        ("joint_limit_max_impulse", C.c_double),
        ("init_position", C.c_double * 3),
        ("init_quat", C.c_double * 4),
        ("rand_roll", C.c_double),
        ("rand_pitch", C.c_double),
        ("rand_x", C.c_double),
        ("rand_z", C.c_double),
        ("rand_omega_x", C.c_double),
        ("rand_omega_y", C.c_double),
        ("rand_linear_velocity", C.c_double * 3),
        ("init_joint_configuration", C.c_double * 6),
        ("init_angular_velocity", C.c_double * 3),
        ("init_linear_velocity", C.c_double * 3),
        ("spine_mode", C.c_int32),
        ("reserved_spine_mode", C.c_int32),
        ("body_contacts", C.c_int32),
        ("reserved_body_contacts", C.c_int32),
        ("body_contact_erp", C.c_double),
        ("body_friction", C.c_double),
        ("solver_residual_threshold", C.c_double),
        ("max_episode_steps", C.c_int32),
        ("reserved_max_episode_steps", C.c_int32),
    ]


class UpkieMpcConfig(C.Structure):
    _fields_ = [
        ("fall_pitch", C.c_double),
        ("leg_length", C.c_double),
        ("max_ground_accel", C.c_double),
        ("max_ground_velocity", C.c_double),
        ("nb_timesteps", C.c_int32),
        ("max_iterations", C.c_int32),
        ("sampling_period", C.c_double),
        ("stage_input_cost_weight", C.c_double),
        ("stage_state_cost_weight", C.c_double),
        ("terminal_cost_weight", C.c_double),
        ("gravity", C.c_double),
    ]


class UpkieObserverConfig(C.Structure):
    _fields_ = [
        ("dt", C.c_double),
        ("cutoff_period", C.c_double),
        ("liftoff_inertia", C.c_double),
        ("min_touchdown_acceleration", C.c_double),
        ("min_touchdown_torque", C.c_double),
        ("touchdown_inertia", C.c_double),
        ("upper_leg_torque_threshold", C.c_double),
        ("signed_radius", C.c_double * 2),
        ("rotation_base_to_imu", C.c_double * 9),
    ]


class UpkieWheelBalancerConfig(C.Structure):
    _fields_ = [
        ("contact_radius", C.c_double),
        ("dt", C.c_double),
        ("fall_pitch", C.c_double),
        ("max_ground_velocity", C.c_double),
        ("pitch_damping", C.c_double),
        ("pitch_stiffness", C.c_double),
        ("position_damping", C.c_double),
        ("position_stiffness", C.c_double),
        ("stiff_yaw_velocity", C.c_double),
        ("wheel_radius", C.c_double),
    ]


def default_wheel_balancer_config(spine_frequency: float = 1000.0) -> UpkieWheelBalancerConfig:
    """``WheelBalancer::Parameters`` defaults (``upkie/cpp/controllers/WheelBalancer.h:60-90``) with the spine's
    overrides ``dt = 1 / spine_frequency``, ``wheel_radius = 0.06`` (``spines/common/controllers.h:33-36``)."""
    c = UpkieWheelBalancerConfig()
    c.contact_radius = 0.1524
    c.dt = 1.0 / spine_frequency
    c.fall_pitch = 1.0
    c.max_ground_velocity = 2.0
    c.pitch_damping = 1.8
    c.pitch_stiffness = 20.0
    c.position_damping = 0.7
    c.position_stiffness = 1.6
    c.stiff_yaw_velocity = 0.1
    c.wheel_radius = 0.06
    return c


OBS_LAYOUT_SPINE, OBS_LAYOUT_OBSERVERS = 0, 1
OBSV_PITCH, OBSV_ANGVEL, OBSV_ROT, OBSV_CONTACT, OBSV_WHEEL_CONTACT = 0, 1, 4, 13, 14
OBSV_LEG_TORQUE, OBSV_WHEEL_INERTIA, OBSV_ODOM_POS, OBSV_ODOM_VEL, OBSV_DIM = 16, 17, 19, 20, 21


def default_observer_config(model, spine_frequency: float = 1000.0) -> UpkieObserverConfig:
    """Spine configuration defaults (``upkie/envs/backends/spine_backend.py:77-105,140-165``)."""
    c = UpkieObserverConfig()
    c.dt = 1.0 / spine_frequency
    c.cutoff_period = 0.2
    c.liftoff_inertia = 1e-3
    c.min_touchdown_acceleration = 2.0
    c.min_touchdown_torque = 0.015
    c.touchdown_inertia = 4e-3
    c.upper_leg_torque_threshold = 10.0
    sign = 1.0 if model.left_wheeled else -1.0
    c.signed_radius[0] = sign * model.wheel_radius
    c.signed_radius[1] = -sign * model.wheel_radius
    for k, x in enumerate(np.asarray(model.rotation_base_to_imu, dtype=float).reshape(9)):
        c.rotation_base_to_imu[k] = float(x)
    return c


def default_sim_config(frequency: float = 200.0) -> UpkieSimConfig:
    """Reference defaults (``pybullet_backend.py:55-112``,
    ``upkie_servos.py:114-124``, ``upkie_gyropod.py:105-112``,
    ``upkie_env.py:87-90``) plus the restated Bullet constants (DESIGN.md).

    Must stay equal to ``upkie_b200_default_config`` in the C library; a test
    checks it.
    """
    c = UpkieSimConfig()
    c.dt = 1.0 / frequency
    c.nb_substeps = int(1000.0 * c.dt)
    c.pgs_iterations = 50
    c.gravity = 9.81
    c.torque_control_kp = 20.0
    c.torque_control_kd = 1.0
    for j in range(NJ):
        c.joint_friction[j] = 0.0
        c.torque_control_noise[j] = 0.0
        c.torque_measurement_noise[j] = 0.0
    for k in range(3):
        c.imu_accelerometer_bias[k] = 0.0
        c.imu_gyroscope_bias[k] = 0.0
    c.imu_accelerometer_noise = 0.0
    c.imu_gyroscope_noise = 0.0
    c.noise_seed = 0
    c.linear_damping = 0.04
    c.angular_damping = 0.04
    c.max_coordinate_velocity = 100.0
    c.contact_stiffness = 30000.0
    c.contact_damping = 1000.0
    c.contact_breaking_threshold = 0.02
    c.friction = 1.0
    c.max_gain_scale = 5.0
    c.fall_pitch = 1.0
    c.leg_gain_scale = 1.0
    c.max_ground_velocity = 3.0
    c.max_yaw_velocity = 1.0
    c.servos_fall_termination = 0
    c.skip_action_clamps = 0
    c.min_base_height = 0.0
    c.pgs_tolerance = 0.0  # deprecated, ignored (see solver_residual_threshold)
    c.warmstarting_factor = 0.0  # measured: no fewer sweeps (friction rows dominate); Bullet's value would be 0.85
    c.joint_limits = 3  # Bullet's hip / knee limit rows on (0 off, 1 scalar reference path [host build], 2 ten-row, 3 ten-row per warp on demand)
    c.joint_limit_erp = 0.2
    c.joint_limit_max_impulse = 100.0
    c.init_position[0], c.init_position[1], c.init_position[2] = 0.0, 0.0, 0.6
    c.init_quat[0], c.init_quat[1], c.init_quat[2], c.init_quat[3] = 1.0, 0.0, 0.0, 0.0
    c.rand_roll = c.rand_pitch = c.rand_x = c.rand_z = 0.0
    c.rand_omega_x = c.rand_omega_y = 0.0
    for k in range(3):
        c.rand_linear_velocity[k] = 0.0
        c.init_angular_velocity[k] = 0.0
        c.init_linear_velocity[k] = 0.0
    for j in range(NJ):
        c.init_joint_configuration[j] = 0.0
    c.spine_mode = 0  # 1: timing of the C++ Bullet spine in simulate() mode (include/upkie_b200.h)
    c.reserved_spine_mode = 0
    c.body_contacts = 0  # 1: collision points of the model (torso box...) hold contact rows against the ground, as every link with a <collision> does in Bullet; B200Backend turns it on, batched envs opt in (include/upkie_b200.h)
    c.reserved_body_contacts = 0
    c.body_contact_erp = 0.2  # btContactSolverInfo::m_erp2
    c.body_friction = 0.5  # URDF importer default lateral friction of a link without <contact>
    c.solver_residual_threshold = 1e-7  # PyBullet's solverResidualThreshold default (Bullet's m_leastSquaresResidualThreshold)
    c.max_episode_steps = 0  # no time limit (include/upkie_b200.h: max_episode_steps)
    c.reserved_max_episode_steps = 0
    return c


class UpkiePush(C.Structure):
    """``UpkiePush`` of include/upkie_b200.h: which earlier slot a launch sends to the other GPUs, and where."""

    _fields_ = [
        ("src_obs", C.c_void_p),
        ("src_terminated", C.c_void_p),
        ("mc_obs", C.c_void_p),
        ("mc_terminated", C.c_void_p),
        ("peer_obs", C.c_void_p * 8),
        ("peer_terminated", C.c_void_p * 8),
        ("n_peers", C.c_int32),
        ("reserved", C.c_int32),
    ]


class UpkieStepOutputs(C.Structure):
    """``UpkieStepOutputs`` of include/upkie_b200.h: the output buffers of ``upkie_b200_step`` / ``_step_host``."""

    _fields_ = [
        ("obs", C.c_void_p),
        ("reward", C.c_void_p),
        ("terminated", C.c_void_p),
        ("truncated", C.c_void_p),
        ("final_obs", C.c_void_p),
        ("compact", C.c_int32),
        ("final_state", C.c_int32),  # 1 = stash the same-step auto-resets' pre-reset states (final_spine_obs)
    ]


class UpkieBaseVelocityPost(C.Structure):
    """``UpkieBaseVelocityPost`` of include/upkie_b200.h: the buffers of ``upkie_b200_base_velocity_post``."""

    _fields_ = [
        ("action", C.c_void_p),
        ("gyropod_obs", C.c_void_p),
        ("gyropod_final_obs", C.c_void_p),
        ("xy", C.c_void_p),
        ("commanded_velocity", C.c_void_p),
        ("obs", C.c_void_p),
        ("final_obs", C.c_void_p),
        ("dt", C.c_float),
        ("autoreset_mode", C.c_int32),
    ]


class UpkieResetRandomization(C.Structure):
    """``UpkieResetRandomization`` of include/upkie_b200.h: which columns every reset redraws, and their ranges."""

    _fields_ = [
        ("columns", C.c_uint64),  # bit k: column k is redrawn
        ("low", C.c_float * RR_DIM),
        ("high", C.c_float * RR_DIM),
    ]


PUSH_MAX_STEPS = 1 << 30  # UPKIE_PUSH_MAX_STEPS


class UpkiePushRandomization(C.Structure):
    """``UpkiePushRandomization`` of include/upkie_b200.h: the pushed body, and the ranges of the gaps, durations (steps)
    and world-frame forces (N) of the pushes."""

    _fields_ = [
        ("body", C.c_int32),
        ("gap_low", C.c_uint32),
        ("gap_high", C.c_uint32),
        ("duration_low", C.c_uint32),
        ("duration_high", C.c_uint32),
        ("force_low", C.c_float * 3),
        ("force_high", C.c_float * 3),
    ]


class UpkieActionDelay(C.Structure):
    """``UpkieActionDelay`` of include/upkie_b200.h: the range of each env's action delay, in substeps."""

    _fields_ = [
        ("substeps_low", C.c_uint32),
        ("substeps_high", C.c_uint32),
    ]


MAX_DELAY_TICKS = 8  # UPKIE_MAX_DELAY_TICKS: the deepest history of an action or observation delay, in ticks


class UpkieObservationDelay(C.Structure):
    """``UpkieObservationDelay`` of include/upkie_b200.h: the range of each env's observation delay, in substeps."""

    _fields_ = [
        ("substeps_low", C.c_uint32),
        ("substeps_high", C.c_uint32),
    ]


class UpkieServoDropout(C.Structure):
    """``UpkieServoDropout`` of include/upkie_b200.h: the range each env's per-cycle servo reply loss probability is
    drawn from at its resets, and the servos (bit j, ``NJ`` order) whose replies may be lost."""

    _fields_ = [
        ("prob_low", C.c_float),
        ("prob_high", C.c_float),
        ("joint_mask", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


SERVO_HELD_DIM = 18  # the held rows of an env under servo dropouts: [joint][position, velocity, torque]


class UpkieImuMisalignment(C.Structure):
    """``UpkieImuMisalignment`` of include/upkie_b200.h: the ranges, in radians, of the roll, pitch and yaw of the IMU
    mounting error each env draws at its resets (E = Rz(yaw) Ry(pitch) Rx(roll), a rotation in the base frame)."""

    _fields_ = [
        ("roll_low", C.c_float),
        ("roll_high", C.c_float),
        ("pitch_low", C.c_float),
        ("pitch_high", C.c_float),
        ("yaw_low", C.c_float),
        ("yaw_high", C.c_float),
    ]


class UpkieServoNoise(C.Structure):
    """``UpkieServoNoise`` of include/upkie_b200.h: the ranges of the standard deviations of each joint's position
    (radians) and velocity (rad/s) measurement noise, drawn per env at every reset (UPKIE_NJ order)."""

    _fields_ = [
        ("position_low", C.c_float * 6),
        ("position_high", C.c_float * 6),
        ("velocity_low", C.c_float * 6),
        ("velocity_high", C.c_float * 6),
    ]


SERVO_NOISE_MAX = {"position": 0.1, "velocity": 5.0}  # the largest high bound of each quantity (rad, rad/s)


class UpkieEncoderOffset(C.Structure):
    """``UpkieEncoderOffset`` of include/upkie_b200.h: the range, in radians, of the encoder zero offset each joint of
    ``joint_mask`` draws at every reset of its env (the servo frame is the joint frame shifted by it)."""

    _fields_ = [
        ("low", C.c_float),
        ("high", C.c_float),
        ("joint_mask", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


ENCODER_OFFSET_DEFAULT_JOINTS = ("left_hip", "left_knee", "right_hip", "right_knee")  # zeroed by hand on the robot


RAD_PER_REV = 2.0 * math.pi  # a speed in rev/s (the moteus unit) times this is in rad/s
# servo.max_velocity_derate, the band past servo.max_velocity over which a moteus servo's output falls to zero: 2 rev/s,
# the default of the moteus reference documentation as remembered (an assumption: no source in this project states it)
MOTEUS_MAX_VELOCITY_DERATE = 2.0 * RAD_PER_REV


class UpkieVelocityDerate(C.Structure):
    """``UpkieVelocityDerate`` of include/upkie_b200.h: the range of each joint's velocity limit, drawn per env at every
    reset, and the band past it over which the servo's motoring torque falls to zero, in rad/s (UPKIE_NJ order;
    rev/s times 2 pi)."""

    _fields_ = [
        ("max_velocity_low", C.c_float * 6),
        ("max_velocity_high", C.c_float * 6),
        ("derate", C.c_float * 6),
        ("joint_mask", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


class UpkieAttitudeFilter(C.Structure):
    """``UpkieAttitudeFilter`` of include/upkie_b200.h: the ranges each reset draws an env's attitude-filter gains
    (kp in 1/s, ki in 1/s^2) and initial estimate error (roll, pitch about the base axes, rad) from."""

    _fields_ = [
        ("kp_low", C.c_float), ("kp_high", C.c_float),
        ("ki_low", C.c_float), ("ki_high", C.c_float),
        ("roll_low", C.c_float), ("roll_high", C.c_float),
        ("pitch_low", C.c_float), ("pitch_high", C.c_float),
    ]


ATTITUDE_FILTER_MAX_KP_H = 0.5  # kp_high * (dt / nb_substeps) at most: the discrete correction must not overshoot
ATTITUDE_FILTER_MAX_KI = 10.0  # 1/s^2, the largest ki_high
ATTITUDE_FILTER_MAX_ERROR = 0.78539816  # rad, the largest |roll| or |pitch| bound of the initial error (pi/4)


class UpkieTorqueScale(C.Structure):
    """``UpkieTorqueScale`` of include/upkie_b200.h: the range of each joint's delivered-torque scale, drawn per env at
    every reset (dimensionless, UPKIE_NJ order): the physics integrates the scale times the torque the servo commands
    and reports."""

    _fields_ = [
        ("scale_low", C.c_float * 6),
        ("scale_high", C.c_float * 6),
        ("joint_mask", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


TORQUE_SCALE_MAX = 2.0  # the largest scale_high (and scale a state may hold)


MAX_HISTORY = 64  # UPKIE_MAX_HISTORY: the most entries an observation history reports
MAX_HISTORY_CHANNELS = 16  # UPKIE_MAX_HISTORY_CHANNELS: the most spine columns it records


class UpkieHistory(C.Structure):
    """``UpkieHistory`` of include/upkie_b200.h: the spine-observation columns an observation history records
    (``SP_*``, the first ``count`` of ``columns``) and the entries it reports (``size``)."""

    _fields_ = [
        ("size", C.c_uint32),
        ("count", C.c_uint32),
        ("columns", C.c_int32 * MAX_HISTORY_CHANNELS),
    ]


def default_mpc_config() -> UpkieMpcConfig:
    """``MPCBalancer.__init__`` defaults (``mpc_balancer.py:168-181``)."""
    c = UpkieMpcConfig()
    c.fall_pitch = 1.0
    c.leg_length = 0.58
    c.max_ground_accel = 10.0
    c.max_ground_velocity = 3.0
    c.nb_timesteps = 50
    c.max_iterations = 30
    c.sampling_period = 0.02
    c.stage_input_cost_weight = 1e-3
    c.stage_state_cost_weight = 1e-3
    c.terminal_cost_weight = 1.0
    c.gravity = 9.81
    return c


def struct_to_dict(s: C.Structure) -> dict:
    """Nested lists/floats view of a ctypes structure (for comparisons)."""
    out = {}
    for name, _ in s._fields_:
        v = getattr(s, name)
        if isinstance(v, C.Array):
            out[name] = [list(x) if isinstance(x, C.Array) else x for x in v]
        else:
            out[name] = v
    return out


def config_env_params(c: "UpkieSimConfig") -> np.ndarray:
    """The row ``[EP_DIM]`` float32 of the per-env parameter table that holds a configuration's own values: what every
    env runs without a table (``upkie_b200_get_env_params``)."""
    r = np.empty(EP_DIM, dtype=np.float64)
    r[EP_KP], r[EP_KD] = c.torque_control_kp, c.torque_control_kd
    r[EP_FRICTION : EP_FRICTION + NJ] = list(c.joint_friction)
    r[EP_CTRL_NOISE : EP_CTRL_NOISE + NJ] = list(c.torque_control_noise)
    r[EP_MEAS_NOISE : EP_MEAS_NOISE + NJ] = list(c.torque_measurement_noise)
    r[EP_IMU_ACC_BIAS : EP_IMU_ACC_BIAS + 3] = list(c.imu_accelerometer_bias)
    r[EP_IMU_ACC_NOISE] = c.imu_accelerometer_noise
    r[EP_IMU_GYRO_BIAS : EP_IMU_GYRO_BIAS + 3] = list(c.imu_gyroscope_bias)
    r[EP_IMU_GYRO_NOISE] = c.imu_gyroscope_noise
    return r.astype(np.float32)  # the kernels' fp32 values of the double fields (round to nearest, as params.h)
