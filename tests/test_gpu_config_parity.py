# SPDX-License-Identifier: Apache-2.0
"""The step kernels against the fp64 oracle away from the default configuration.

At the defaults (50 PGS sweeps, a 1e-7 residual threshold, no warm start, clamps and impulse caps far from binding) the
contact solve reaches its fixed point: sweep order, sweep count and the per-lane exit barely move the result, and a
kernel that ran one sweep too many, kept updating a frozen lane or lost its warm start would still sit inside the
one-tick tolerances. Each row of VARIANTS sets the knobs the kernels read from the configuration to values where that
code decides the result - a truncated or early-exiting solve, a warm start, a binding velocity clamp or limit impulse,
other substep counts, contact constants and gains - and every row proves on the fp64 oracle that it moves the one-tick
state by at least BITE times what fp32 alone costs (its bite check), so that it tests something.

One tick from the same states and actions on every side: the fp64 oracle, the fp32 oracle, the kernels' arithmetic
compiled for the host (tests/hostsim), the library built without --use_fast_math where the family exists there, and the
device on each path the row names. The device's error against the fp64 oracle may be at most RATIO x the worst fp32
side's, plus a floor, at the worst robot and at the 99th percentile (the rule of test_gpu_trajectory_parity.py).
tests/test_kernel_arithmetic_cpu.py runs the same table through the host build without a GPU. Measured errors go to the
JSON file named by UPKIE_PARITY_REPORT."""
import numpy as np
import pytest

from conftest import at_joint_bounds, random_servo_actions
from test_gpu_trajectory_parity import RATIO, _config, _Device, _Exact, _Host, _initial, _Oracle, _report
from upkie_b200 import _abi

pytestmark = pytest.mark.gpu

N = 2083  # neither a whole warp nor a whole block
BITE = 100.0  # a row must move the fp64 one-tick state by BITE x the worst fp32 side's 99th-percentile error
# the compared quantities of a state row; floors in their units (m/s and rad/s, N s). The lateral friction rows of the
# two wheels push along the wheel axle in mirrored directions (sgn2 in sim_pair.cuh), so adding the same impulse to both
# stored values moves nothing: no joint and no net force or moment on the base. The solve leaves that split to its
# sweep history, and only the difference of the two stored values is physics; the rolling rows are compared as stored.
F = _abi.ST_FRICTION_IMPULSE
GROUPS = {"base_twist": lambda st: st[:, _abi.ST_LINVEL:_abi.ST_LINVEL + 6],
          "joint_rates": lambda st: st[:, _abi.ST_QD:_abi.ST_QD + 6],
          "contact_impulse": lambda st: st[:, _abi.ST_CONTACT_IMPULSE:_abi.ST_CONTACT_IMPULSE + 2],
          "friction_impulse": lambda st: np.stack([st[:, F], st[:, F + 2], st[:, F + 1] - st[:, F + 3]], axis=1)}
FLOOR = {"base_twist": 1e-5, "joint_rates": 1e-4, "contact_impulse": 1e-6, "friction_impulse": 1e-6}

# The step paths: (kind, joint_limits, body_contacts, device path of test_gpu_trajectory_parity._Device, the exact
# library has the family). "headline" is the benchmark's compact TILE=1 kernel with next-step auto-reset, "table" the
# FAM_TABLE kernels (a per-env parameter table equal to the config), "spine" the FAM_SPINE kernels, which start from a
# reset (three stopped cycles) instead of a state row.
PATHS = {
    "limits0": ("servos", 0, 0, "servos", True),
    "limits2": ("servos", 2, 0, "servos", True),
    "limits3": ("servos", 3, 0, "servos", True),
    "headline": ("servos", 3, 0, "compact", False),
    "table": ("servos", 3, 0, "table", False),
    "body": ("servos", 3, 1, "servos", False),
    "spine": ("spine", 2, 0, "servos", False),
    "gyropod": ("gyropod", 3, 0, "gyropod", True),
    "pendulum": ("pendulum", 3, 0, "pendulum", True),
}
SOLVE = ("limits0", "limits2", "limits3", "headline", "table")
LIMITS = ("limits2", "limits3", "headline", "table")
TIMING = SOLVE + ("spine", "gyropod", "pendulum")
# name: (config overrides, paths, initial states). "bounds": conftest.at_joint_bounds (half of the robots on or near
# the ground, a third of the hips and knees on a bound); "warm": the same with cached normal impulses in [0, 1.5] N s;
# "dropping": the same moving down 3 m/s faster, so that wheels a few millimetres above the floor reach it within the
# tick; "fallen": robots lying on their torso (the setup of test_body_contacts.py after 1.5 s); "thrown": the same with
# random base and joint velocities, fast enough for a 3 rad/s clamp to bind. The body path starts from "thrown" where
# the row names no body state: its torso contact rows are then active and every robot goes through the general
# body-contact solver. Spine-mode runs start from a reset (inputs()).
VARIANTS = {
    "pgs_1_sweep": ((("pgs_iterations", 1), ("solver_residual_threshold", 0.0)), SOLVE + ("gyropod",), "bounds"),
    "pgs_2_sweeps": ((("pgs_iterations", 2), ("solver_residual_threshold", 0.0)), SOLVE, "bounds"),
    "pgs_3_sweeps": ((("pgs_iterations", 3), ("solver_residual_threshold", 0.0)), SOLVE + ("pendulum", "body"), "bounds"),
    "threshold_1e-4": ((("solver_residual_threshold", 1e-4),), SOLVE, "bounds"),
    "threshold_1e-2": ((("solver_residual_threshold", 1e-2),), SOLVE + ("body",), "bounds"),
    "warm_start_3_sweeps": ((("warmstarting_factor", 0.85), ("pgs_iterations", 3), ("solver_residual_threshold", 0.0)),
                            SOLVE, "warm"),
    "velocity_clamp_3": ((("max_coordinate_velocity", 3.0),), SOLVE + ("body",), "bounds"),
    "no_damping": ((("linear_damping", 0.0), ("angular_damping", 0.0)), SOLVE + ("gyropod",), "bounds"),
    "1000hz_1_substep": ((("dt", 0.001), ("nb_substeps", 1)), TIMING, "bounds"),
    "250hz_4_substeps": ((("dt", 0.004), ("nb_substeps", 4)), TIMING, "bounds"),
    "100hz_10_substeps": ((("dt", 0.01), ("nb_substeps", 10)), TIMING, "bounds"),
    "friction_0.1": ((("friction", 0.1),), SOLVE + ("gyropod",), "bounds"),
    "stiff_tires": ((("contact_stiffness", 3e5), ("contact_damping", 3e3)), SOLVE, "bounds"),
    "soft_tires": ((("contact_stiffness", 3e3), ("contact_damping", 300.0)), SOLVE, "bounds"),
    "breaking_2mm": ((("contact_breaking_threshold", 0.002),), SOLVE, "dropping"),
    "limit_impulse_0.05": ((("joint_limit_max_impulse", 0.05),), LIMITS, "bounds"),
    "limit_erp_0.8": ((("joint_limit_erp", 0.8),), LIMITS, "bounds"),
    "body_erp_0.8": ((("body_contact_erp", 0.8),), ("body",), "fallen"),
    "body_friction_0.1": ((("body_friction", 0.1),), ("body",), "fallen"),
    "gains_kp60_kd0.3": ((("torque_control_kp", 60.0), ("torque_control_kd", 0.3)), SOLVE, "bounds"),
}
CASES = [(row, path) for row, (_, paths, _) in VARIANTS.items() for path in paths]
# The bite of a row that sets several knobs is measured against the row without the one under test (here: the same
# truncated solve without the warm start), so that the check fails if that knob alone stopped mattering.
BITE_BASELINE = {"warm_start_3_sweeps": (("pgs_iterations", 3), ("solver_residual_threshold", 0.0))}


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def path_config(path, overrides=()):
    kind, limits, body, _, _ = PATHS[path]
    if kind == "spine":
        return _config("servos", limits, body, overrides + (("spine_mode", 1),))
    return _config(kind, limits, body, overrides)


# -- inputs ---------------------------------------------------------------------------------------------------------
_INPUTS = {}


def start_states(row, path):
    states = VARIANTS[row][2]
    return "thrown" if PATHS[path][2] and states != "fallen" else states


def inputs(model, states, kind, n=N):
    """(start rows, actions): state rows [n, STATE_DIM], or for spine-mode runs init rows [n, INIT_DIM]; the same on
    every side, seeded. Spine-mode robots start with both wheels on the floor: two thirds stand on nearly straight legs
    with the base 0.57 to 0.59 m high, one third crouch with the knees 0.01 rad inside their bound."""
    key = (states, kind, n)
    if key not in _INPUTS:
        if kind == "spine":
            start = _initial(n, seed=31)[0]
            rng = np.random.default_rng(32)
            start[:, 2] = rng.uniform(0.57, 0.59, n)
            start[:, _abi.INIT_Q:_abi.INIT_Q + 6] = rng.uniform(-0.05, 0.05, (n, 6))
            start[::3] = _initial(n, seed=33, crouch=True)[0][::3]
        elif states == "fallen":
            start = _fallen(model, n)
        elif states == "thrown":
            start = _throw(inputs(model, "fallen", kind, n)[0].astype(np.float64))
        else:
            start = at_joint_bounds(model, n, seed=41)
            if states == "warm":
                start[:, _abi.ST_CONTACT_IMPULSE:_abi.ST_CONTACT_IMPULSE + 2] = np.random.default_rng(42).uniform(
                    0.0, 1.5, (n, 2))
            if states == "dropping":
                start[:, _abi.ST_LINVEL + 2] -= 3.0
        rng = np.random.default_rng(43)
        if kind == "gyropod":
            act = rng.uniform(-1.5, 1.5, (n, 2)).astype(np.float32)
        elif kind == "pendulum":
            act = rng.uniform(-1.5, 1.5, (n, 1)).astype(np.float32)
        else:
            act = random_servo_actions(n, model, seed=44).astype(np.float32)
        _INPUTS[key] = (start.astype(np.float32), act)
    return _INPUTS[key]


def _fallen(model, n):
    """Robots that fell from pitches in +-[0.05, 0.4] rad with their servos damped, after 300 ticks (1.5 s) of the
    host build with body contacts on: most lie on their torso, some still slide or rock."""
    from test_body_contacts import _falling_setup

    init, act = _falling_setup(model, n)
    side = _Host(model, path_config("body"), n)
    side.reset(init.astype(np.float32))
    for _ in range(300):
        side.servos(act)
    st = side.state()
    side.close()
    return st


def _throw(st):
    """Random base velocities (1 m/s towards the floor, +-1 m/s, +-4 rad/s) and joint rates (+-5 rad/s) added."""
    n = st.shape[0]
    rng = np.random.default_rng(34)
    st[:, _abi.ST_LINVEL:_abi.ST_LINVEL + 3] += rng.uniform(-1.0, 1.0, (n, 3)) - [0.0, 0.0, 1.0]
    st[:, _abi.ST_ANGVEL:_abi.ST_ANGVEL + 3] += rng.uniform(-4.0, 4.0, (n, 3))
    st[:, _abi.ST_QD:_abi.ST_QD + 6] += rng.uniform(-5.0, 5.0, (n, 6))
    return st


# -- one tick -------------------------------------------------------------------------------------------------------
class _HostSpine(_Host):
    """The host build in spine mode: a reset runs the three stopped cycles, a step one spine cycle per substep."""

    def reset(self, init):
        self._each(lambda p, i: p.reset_spine(i), init)

    def servos(self, a):
        self._each(lambda p, x: p.step_servos_spine(x), a)


def tick(side, kind, start, act):
    """One tick of ``side`` from ``start``: (state rows fp64, terminated or None)."""
    if kind == "spine":
        side.reset(start)
    else:
        side.set_state(start)
    term = side.gyro(act)[1] if kind in ("gyropod", "pendulum") else side.servos(act)
    return side.state(), (None if term is None else np.asarray(term).astype(np.uint8))


_REFS = {}


def references(model, oracle_lib, row, path, torch=None):
    """The sides that do not depend on the device path, after one tick of ``row`` on ``path``: "oracle" (fp64),
    "oracle32", "host" and, when ``torch`` is given and the family exists there, "exact"; plus "default", the fp64
    oracle under the path's default configuration or the row's BITE_BASELINE (the bite check's baseline), and on the
    body path "flat", the fp64 oracle under the row's configuration without body contacts. Cached per physics: paths
    that share it (limits3, headline, table) share the sides."""
    overrides = VARIANTS[row][0]
    kind, limits, body, _, has_exact = PATHS[path]
    exact = has_exact and torch is not None
    key = (row, kind, limits, body, exact)
    if key not in _REFS:
        start, act = inputs(model, start_states(row, path), kind)
        cfg, cfg0 = path_config(path, overrides), path_config(path, BITE_BASELINE.get(row, ()))
        n = start.shape[0]
        sides = {"oracle": _Oracle(oracle_lib, model, cfg, n, False), "oracle32": _Oracle(oracle_lib, model, cfg, n, True),
                 "host": (_HostSpine if kind == "spine" else _Host)(model, cfg, n),
                 "default": _Oracle(oracle_lib, model, cfg0, n, False)}
        if body:
            flat = path_config(path, overrides)
            flat.body_contacts = 0
            sides["flat"] = _Oracle(oracle_lib, model, flat, n, False)
        if exact:
            sides["exact"] = _Exact(torch, model, cfg, n)
        _REFS[key] = {k: tick(s, kind, start, act) for k, s in sides.items()}
        sides["host"].close()
        if exact:
            sides["exact"].close()
    return _REFS[key]


def errors(run, ref, mask):
    """Per compared group: (worst, 99th percentile) over the masked robots of each robot's largest difference."""
    out = {}
    for g, q in GROUPS.items():
        e = np.abs(q(run[0][mask]) - q(ref[0][mask])).max(axis=1)
        out[g] = (e.max(), np.percentile(e, 99))
    return out


def fp32_sides(refs):
    return [k for k in refs if k not in ("oracle", "default", "flat")]


def contact_mismatch(run, ref):
    return run[0][:, _abi.ST_CONTACT] != ref[0][:, _abi.ST_CONTACT]


def bite(refs):
    """(the row's largest change of base twist or joint rates against its baseline config on the fp64 oracle, the
    worst fp32 side's 99th-percentile error on them)."""
    o, d = refs["oracle"][0], refs["default"][0]
    cols = np.r_[_abi.ST_LINVEL:_abi.ST_LINVEL + 6, _abi.ST_QD:_abi.ST_QD + 6]
    move = np.abs(o[:, cols] - d[:, cols]).max()
    mask = ~np.any([contact_mismatch(refs[k], refs["oracle"]) for k in fp32_sides(refs)], axis=0)
    e = [errors(refs[k], refs["oracle"], mask) for k in fp32_sides(refs)]
    return move, max(max(x["base_twist"][1], x["joint_rates"][1]) for x in e)


def check_inputs_exercise_the_path(refs, path):
    """On the fp64 oracle: the body path's robots are held by their body contact rows (with the rows off, their base
    twist or joint rates come out more than 0.1 different), and spine-mode robots stand on their wheels (nearly all
    hold contact rows, and a quarter or more end the tick with a non-zero normal impulse)."""
    st = refs["oracle"][0]
    cols = np.r_[_abi.ST_LINVEL:_abi.ST_LINVEL + 6, _abi.ST_QD:_abi.ST_QD + 6]
    if "flat" in refs:
        held = np.abs(st[:, cols] - refs["flat"][0][:, cols]).max(axis=1) > 0.1
        assert held.mean() > 0.9, held.mean()
    if PATHS[path][0] == "spine":
        assert st[:, _abi.ST_CONTACT].mean() > 0.9, st[:, _abi.ST_CONTACT].mean()
        assert (st[:, _abi.ST_CONTACT_IMPULSE:_abi.ST_CONTACT_IMPULSE + 2] > 0).any(axis=1).mean() > 0.25


# -- one-tick parity ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row,path", CASES)
def test_one_tick_matches_the_oracle(model, oracle_lib, torch, row, path):
    """One tick of 2 083 robots on ``path`` under ``row``'s configuration: base twist, joint rates, normal and friction
    impulses within RATIO x the worst fp32 side's error plus a floor, at the worst robot and at the 99th percentile;
    `terminated` equal to the oracle's; the floor-contact flag equal except for robots within round-off of the breaking
    threshold (at most as many as an fp32 side flips, plus one)."""
    overrides = VARIANTS[row][0]
    kind, _, _, dev_path, _ = PATHS[path]
    refs = references(model, oracle_lib, row, path, torch)
    start, act = inputs(model, start_states(row, path), kind)
    dev = tick(_Device(torch, model, path_config(path, overrides), start.shape[0], dev_path), kind, start, act)
    ref = refs["oracle"]
    sides = fp32_sides(refs)
    flips = {k: contact_mismatch(r, ref) for k, r in [(k, refs[k]) for k in sides] + [("device", dev)]}
    mask = ~np.any(list(flips.values()), axis=0)
    err = {k: errors(r, ref, mask) for k, r in [(k, refs[k]) for k in sides] + [("device", dev)]}
    move, fp32 = bite(refs)
    _report(f"config_{row}_{path}", bite=move, **{f"{k}_{g}_{q}": v[i] for k, e in err.items() for g, v in e.items()
                                                  for i, q in enumerate(("worst", "p99"))})
    assert move >= BITE * fp32, (row, path, move, fp32)
    check_inputs_exercise_the_path(refs, path)
    assert flips["device"].sum() <= max(flips[k].sum() for k in fp32_sides(refs)) + 1, (row, path)
    if dev[1] is not None:
        assert np.array_equal(dev[1], ref[1]), (row, path, np.flatnonzero(dev[1] != ref[1]))
    for g in GROUPS:
        for i, q in enumerate(("worst", "p99")):
            worst32 = max(err[k][g][i] for k in fp32_sides(refs))
            assert err["device"][g][i] <= RATIO * worst32 + FLOOR[g], (row, path, g, q, err["device"][g][i], worst32)



# -- neighbour independence -----------------------------------------------------------------------------------------
def _classes(model, st):
    """Per robot: airborne (no wheel within the breaking threshold after the tick), on a hip or knee bound."""
    lo = np.array([j.limit.lower for j in model.joints])[[0, 1, 3, 4]]
    hi = np.array([j.limit.upper for j in model.joints])[[0, 1, 3, 4]]
    q = st[:, _abi.ST_Q:_abi.ST_Q + 6][:, [0, 1, 3, 4]]
    return st[:, _abi.ST_CONTACT] == 0, ((q <= lo) | (q >= hi)).any(axis=1)


@pytest.mark.parametrize("limits", [2, 0])
def test_a_robot_does_not_depend_on_its_neighbours(model, oracle_lib, torch, limits):
    """With the residual threshold at 1e-2 lanes freeze after a few sweeps while their warp goes on; with joint_limits
    = 2 every warp runs the ten-row solver, with 0 the six-row one. One tick of a batch, then of the same robots in a
    shuffled order: every robot's state row is bit for bit the same. Every warp of both orders mixes airborne robots,
    robots in contact and robots on a hip or knee bound. Equal as numbers; where the bits differ, both are zeros (a
    signed zero of an impulse can depend on the warp's solver path)."""
    cfg = _config("servos", limits, 0, (("solver_residual_threshold", 1e-2),))
    start, act = inputs(model, "bounds", "servos")
    n = start.shape[0]
    orders = [np.random.default_rng(seed).permutation(n) for seed in (51, 52)]
    out = [tick(_Device(torch, model, cfg, n, "servos"), "servos", start[o], act[o])[0][np.argsort(o)] for o in orders]
    air, bound = _classes(model, out[0])
    for order in orders:
        w = n // 32 * 32
        a, b = air[order][:w].reshape(-1, 32), bound[order][:w].reshape(-1, 32)
        assert a.any(axis=1).all() and (~a).any(axis=1).all() and b.any(axis=1).all()
    _assert_same_but_zero_signs(f"neighbours_limits{limits}", out[0].astype(np.float32), out[1].astype(np.float32))


def _assert_same_but_zero_signs(name, a, b):
    assert np.array_equal(a, b), np.argwhere(a != b)[:8]
    bits = a.view(np.uint32) != b.view(np.uint32)
    assert (a[bits] == 0).all(), np.argwhere(bits)[:8]
    _report(name, robots=bits.any(axis=1).sum(), **{f"column_{c}": k for c, k in enumerate(bits.sum(axis=0)) if k})


# -- spine mode: next-step resets in a launch of one or two substeps ------------------------------------------------
@pytest.mark.parametrize("nb", [1, 2])
def test_spine_lanes_beside_a_reset_run_their_own_substeps(model, oracle_lib, torch, nb):
    """Spine mode at nb_substeps = 1 or 2 with next-step auto-reset: a resetting lane runs its three stopped cycles, so
    the launch loops three times, and the other lanes must still run exactly nb_substeps cycles. A third of the robots
    start tipped past fall_pitch and terminate in the first tick; in the second, every other robot comes out bit for
    bit as on a handle without resetting neighbours started from the same state and lag records, and within the spine
    tolerances of test_spine_mode.py of the fp64 oracle (one cycle more or less moves the joint rates by tens of
    rad/s). Equal as numbers; where the bits differ, both are zeros."""
    from upkie_b200.sim import UpkieSim

    cfg = _config("servos", 2, 0, (("dt", nb / 1000.0), ("nb_substeps", nb), ("spine_mode", 1)))
    n = N
    init = _initial(n, seed=61)[0]
    tipped = np.arange(n) % 3 == 0
    init[tipped, 3], init[tipped, 5] = np.cos(0.65), np.sin(0.65)  # pitch 1.3 rad
    act = random_servo_actions(n, model, seed=62).astype(np.float32)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()  # noqa: E731
    a = UpkieSim(n, model=model, config=cfg)
    a.set_autoreset(1, 2025, 0)
    a.reset(init_state=t(init))
    term = a.step_servos(t(act))[2].cpu().numpy().astype(bool)
    assert np.array_equal(term, tipped)
    keep = ~term
    st1, lag1 = a.get_state().cpu().numpy()[keep], a.get_lag().cpu().numpy()[keep]
    a.step_servos(t(act))
    st2 = a.get_state().cpu().numpy()[keep]
    b = UpkieSim(int(keep.sum()), model=model, config=cfg)
    b.set_state(t(st1))
    b.set_lag(t(lag1))
    b.step_servos(t(act[keep]))
    _assert_same_but_zero_signs(f"spine_twin_{nb}_substeps", st2, b.get_state().cpu().numpy())
    osim = oracle_lib.OracleSim(model, cfg, int(keep.sum()), threads=8)
    osim.set_state(st1.astype(np.float64))
    lag = osim.get_lag()
    lag[:, :49] = lag1[:, :49]
    osim.set_lag(lag)
    osim.step_servos(act[keep].astype(np.float64))
    d = np.abs(st2[:, :25].astype(np.float64) - osim.get_state()[:, :25])
    _report(f"spine_next_step_reset_{nb}_substeps", pose_worst=d[:, :7].max(), joint_rate_p99=np.percentile(
        d[:, 19:25].max(axis=1), 99), joint_rate_worst=d[:, 19:25].max())
    assert d[:, :7].max() < 2e-5 and d[:, 13:19].max() < 2e-4
    assert np.median(d[:, 19:25].max(axis=1)) < 5e-5 and np.percentile(d[:, 19:25].max(axis=1), 99) < 5e-3


# -- set_config -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row", list(VARIANTS))
def test_set_config_steps_like_a_handle_created_with_it(model, oracle_lib, torch, row):
    """A handle created with the path's default configuration and switched to the row's with set_config steps bit for
    bit like one created with the row's: the derived parameters (substep h, 1 / h, the contact rows' cfm and erp, the
    squared residual threshold) are rebuilt by set_config."""
    overrides, paths, _ = VARIANTS[row]
    path = "limits3" if "limits3" in paths else paths[0]
    kind, _, _, dev_path, _ = PATHS[path]
    start, act = inputs(model, start_states(row, path), kind)
    cfg = path_config(path, overrides)
    switched = _Device(torch, model, path_config(path), start.shape[0], dev_path)
    switched.sim.set_config(cfg)
    fresh = _Device(torch, model, cfg, start.shape[0], dev_path)
    (sa, ta), (sb, tb) = tick(switched, kind, start, act), tick(fresh, kind, start, act)
    assert np.array_equal(sa.astype(np.float32).view(np.uint32), sb.astype(np.float32).view(np.uint32)), row
    assert ta is None or np.array_equal(ta, tb)
