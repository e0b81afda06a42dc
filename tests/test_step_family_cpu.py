# SPDX-License-Identifier: Apache-2.0
"""The step kernels' families (upkie_b200/csrc/step_family.h), compiled for the CPU (tests/hostsim/step_family.cpp):
what each family compiles in, the family the host picks for a handle's features and transport, with every rejection
and its message, and the (TILE, family) pairs the library instantiates, against build.py's unit table. The GPU tests
of each feature run the kernels the choice names. No GPU needed."""
import ctypes as C
import itertools
import os
import subprocess
import tempfile

import pytest

from upkie_b200 import build

HERE = os.path.dirname(os.path.abspath(__file__))

MODE_SERVOS, MODE_GYROPOD, MODE_PENDULUM = 0, 1, 2
DEVICE, HOST_TILE, IN_KERNEL = 0, 1, 2  # the TILE of the step kernels
(FAM_PLAIN, FAM_EXTRAS, FAM_LIMITS, FAM_SPINE, FAM_BODY, FAM_TABLE, FAM_PUSH, FAM_BODY_PUSH, FAM_DELAY,
 FAM_BODY_DELAY) = range(10)

TRAITS = ("extras", "limits", "table", "reset_rand", "spine", "body", "push", "delay")
# family: the traits it compiles in
FAMILY_TRAITS = {
    FAM_PLAIN: {"table"},
    FAM_EXTRAS: {"extras", "table"},
    FAM_LIMITS: {"extras", "limits"},
    FAM_SPINE: {"extras", "limits", "table", "reset_rand", "spine", "body"},
    FAM_BODY: {"extras", "limits", "table", "reset_rand", "body"},
    FAM_TABLE: {"extras", "limits", "table", "reset_rand"},
    FAM_PUSH: {"extras", "limits", "table", "reset_rand", "push"},
    FAM_BODY_PUSH: {"extras", "limits", "table", "reset_rand", "body", "push"},
    FAM_DELAY: {"extras", "limits", "table", "reset_rand", "push", "delay"},
    FAM_BODY_DELAY: {"extras", "limits", "table", "reset_rand", "body", "push", "delay"},
}

NO_TABLE = ("the per-env parameter table has no in-kernel rollout transport (use upkie_b200_step with compact rows)")
NO_PUSH = "push randomisation has no in-kernel rollout transport (use upkie_b200_step with compact rows)"
NO_DELAY = "action delay has no in-kernel rollout transport (use upkie_b200_step with compact rows)"
NO_LIMIT = ("max_episode_steps has no in-kernel rollout transport: it does not carry truncated (use upkie_b200_step "
            "with compact rows)")
NO_BODY = "body_contacts has no in-kernel rollout transport (use upkie_b200_step_servos_compact)"
SPINE_SERVOS = "spine_mode supports UpkieServos steps only"
NO_SPINE = "spine_mode has no in-kernel rollout transport"

# the handle features step_family reads, in the argument order of hostsim_step_family
FEATURES = ("joint_limits", "ctrl_noise", "meas_noise", "ext", "table", "body_contacts", "push", "delay", "spine_mode",
            "max_episode_steps")

_LIBS = {}


def _lib(exact=False):
    """the CPU build of step_family.h; `exact`: as the exact-arithmetic library compiles it (UPKIE_EXACT_BUILD)"""
    if exact not in _LIBS:
        src = os.path.join(HERE, "hostsim", "step_family.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_family_"), "libhostsim_family.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split() + (["-DUPKIE_EXACT_BUILD=1"] if exact else [])
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        L.hostsim_family_traits.argtypes = [C.c_int, C.POINTER(C.c_uint8)]
        L.hostsim_step_family.argtypes = [C.c_int] * (len(FEATURES) + 2) + [C.c_char_p, C.c_int]
        L.hostsim_step_family.restype = C.c_int
        L.hostsim_step_instantiated.argtypes = [C.c_int, C.c_int]
        L.hostsim_step_instantiated.restype = C.c_int
        _LIBS[exact] = L
    return _LIBS[exact]


def traits(family):
    out = (C.c_uint8 * len(TRAITS))()
    _lib().hostsim_family_traits(family, out)
    return {name for name, v in zip(TRAITS, out) if v}


def step_family(mode=MODE_SERVOS, transport=DEVICE, **features):
    """(family, rejection message or None) of a handle with `features` (FEATURES, all 0 by default)"""
    assert set(features) <= set(FEATURES)
    why = C.create_string_buffer(256)
    f = _lib().hostsim_step_family(*(features.get(k, 0) for k in FEATURES), mode, transport, why, len(why))
    return f, (why.value.decode() or None)


def instantiated(tile, family, exact=False):
    return bool(_lib(exact).hostsim_step_instantiated(tile, family))


@pytest.mark.parametrize("family", sorted(FAMILY_TRAITS))
def test_trait_table(family):
    assert traits(family) == FAMILY_TRAITS[family]


@pytest.mark.parametrize("transport", [DEVICE, HOST_TILE, IN_KERNEL])
@pytest.mark.parametrize("mode", [MODE_SERVOS, MODE_GYROPOD, MODE_PENDULUM])
def test_base_families(mode, transport):
    assert step_family(mode, transport) == (FAM_PLAIN, None)
    for extra in ({"ctrl_noise": 1}, {"meas_noise": 1}, {"ext": 1}):
        assert step_family(mode, transport, **extra) == (FAM_EXTRAS, None)
    for jl in (1, 2, 3):  # joint limits take the limit family whatever the noise and external forces
        assert step_family(mode, transport, joint_limits=jl) == (FAM_LIMITS, None)
        assert step_family(mode, transport, joint_limits=jl, ctrl_noise=1, ext=1) == (FAM_LIMITS, None)


@pytest.mark.parametrize("transport", [DEVICE, HOST_TILE])
@pytest.mark.parametrize("mode", [MODE_SERVOS, MODE_GYROPOD, MODE_PENDULUM])
def test_feature_families(mode, transport):
    # a table with joint limits: the table family; without limits the plain and extras kernels read it
    assert step_family(mode, transport, joint_limits=2, table=1) == (FAM_TABLE, None)
    assert step_family(mode, transport, table=1) == (FAM_PLAIN, None)
    assert step_family(mode, transport, table=1, meas_noise=1) == (FAM_EXTRAS, None)
    # body contacts, with or without limits or a table
    for kw in ({}, {"joint_limits": 2}, {"joint_limits": 2, "table": 1}, {"ext": 1}):
        assert step_family(mode, transport, body_contacts=1, **kw) == (FAM_BODY, None)
    # pushes: the table family's push copy, or the body-contact family's with body contacts
    assert step_family(mode, transport, joint_limits=2, push=1) == (FAM_PUSH, None)
    assert step_family(mode, transport, joint_limits=2, table=1, push=1) == (FAM_PUSH, None)
    assert step_family(mode, transport, joint_limits=2, body_contacts=1, push=1) == (FAM_BODY_PUSH, None)
    # a time limit does not change the family
    assert step_family(mode, transport, joint_limits=2, max_episode_steps=10) == (FAM_LIMITS, None)


@pytest.mark.parametrize("transport", [DEVICE, HOST_TILE])
def test_spine_family(transport):
    for kw in ({}, {"joint_limits": 2}, {"joint_limits": 2, "table": 1}, {"body_contacts": 1}, {"push": 1},
               {"ctrl_noise": 1, "ext": 1}):
        assert step_family(MODE_SERVOS, transport, spine_mode=1, **kw) == (FAM_SPINE, None)
    for mode in (MODE_GYROPOD, MODE_PENDULUM):
        assert step_family(mode, transport, spine_mode=1) == (-1, SPINE_SERVOS)


def test_in_kernel_transport_rejections():
    def reject(**kw):
        return step_family(MODE_SERVOS, IN_KERNEL, joint_limits=2, **kw)[1]

    assert reject(table=1) == NO_TABLE
    assert reject(push=1) == NO_PUSH
    assert reject(max_episode_steps=1) == NO_LIMIT
    assert reject(body_contacts=1) == NO_BODY
    assert reject(spine_mode=1) == NO_SPINE
    assert step_family(MODE_GYROPOD, IN_KERNEL, spine_mode=1) == (-1, SPINE_SERVOS)
    # with several at once, the first of this order is reported
    assert reject(table=1, push=1, max_episode_steps=1, body_contacts=1, spine_mode=1) == NO_TABLE
    assert reject(push=1, max_episode_steps=1, body_contacts=1, spine_mode=1) == NO_PUSH
    assert reject(max_episode_steps=1, body_contacts=1, spine_mode=1) == NO_LIMIT
    assert reject(body_contacts=1, spine_mode=1) == NO_BODY
    for transport in (DEVICE, HOST_TILE):
        assert step_family(MODE_SERVOS, transport, joint_limits=2, max_episode_steps=1) == (FAM_LIMITS, None)


# ---- the action delay (upkie_b200_set_action_delay needs joint limits) --------------------------------------------------


def test_delay_traits():
    base = {"extras", "limits", "table", "reset_rand", "push"}
    assert traits(FAM_DELAY) == base | {"delay"}
    assert traits(FAM_BODY_DELAY) == base | {"body", "delay"}
    assert traits(FAM_DELAY) - {"delay"} == traits(FAM_PUSH)
    assert traits(FAM_BODY_DELAY) - {"delay"} == traits(FAM_BODY_PUSH)
    for fam in range(8):
        assert "delay" not in traits(fam)


@pytest.mark.parametrize("transport", [DEVICE, HOST_TILE])
@pytest.mark.parametrize("mode", [MODE_SERVOS, MODE_GYROPOD, MODE_PENDULUM])
def test_delay_families(mode, transport):
    def family(**kw):
        return step_family(mode, transport, joint_limits=2, **kw)

    assert family(delay=1) == (FAM_DELAY, None)
    assert family(delay=1, table=1) == (FAM_DELAY, None)
    assert family(delay=1, push=1) == (FAM_DELAY, None)
    assert family(delay=1, table=1, push=1, max_episode_steps=9) == (FAM_DELAY, None)
    assert family(delay=1, body_contacts=1) == (FAM_BODY_DELAY, None)
    assert family(delay=1, body_contacts=1, push=1) == (FAM_BODY_DELAY, None)
    # without a delay the choice is the one before the feature
    assert family(push=1) == (FAM_PUSH, None)
    assert family(table=1) == (FAM_TABLE, None)
    assert family(body_contacts=1) == (FAM_BODY, None)


def test_in_kernel_transport_rejects_a_delay_after_the_push_message():
    def reject(**kw):
        return step_family(MODE_SERVOS, IN_KERNEL, joint_limits=2, **kw)

    assert reject(delay=1) == (-1, NO_DELAY)
    assert reject(delay=1, push=1)[1] == NO_PUSH
    assert reject(delay=1, table=1)[1] == NO_TABLE
    assert reject(delay=1, max_episode_steps=1, body_contacts=1)[1] == NO_DELAY
    assert reject(max_episode_steps=1)[1] == NO_LIMIT


# ---- the instantiated pairs -----------------------------------------------------------------------------------------------


@pytest.mark.parametrize("transport", [DEVICE, HOST_TILE, IN_KERNEL])
@pytest.mark.parametrize("mode", [MODE_SERVOS, MODE_GYROPOD, MODE_PENDULUM])
def test_every_family_choice_is_instantiated(mode, transport):
    # every combination of the features step_family reads: a rejection, or a pair the step dispatch launches
    for values in itertools.product((0, 1), repeat=len(FEATURES)):
        kw = dict(zip(FEATURES, values))
        family, why = step_family(mode, transport, **kw)
        if family < 0:
            assert why, kw
        else:
            assert why is None and instantiated(transport, family), (kw, family)


@pytest.mark.parametrize("exact", [False, True])
def test_unit_table_holds_each_instantiated_pair_once(exact):
    units = [u for u in (build.EXACT_UNITS if exact else build.UNITS) if isinstance(u, build.StepUnit)]
    pairs = [(u.tile, f) for u in units for f in u.families]
    twice = sorted({p for p in pairs if pairs.count(p) > 1})
    assert not twice, f"(TILE, family) pairs in more than one unit of build.py: {twice}"
    named = {(t, f) for t in range(-1, 4) for f in range(-1, 11) if instantiated(t, f, exact)}
    assert not named - set(pairs), f"(TILE, family) pairs step_instantiated names without a unit in build.py: " \
                                   f"{sorted(named - set(pairs))}"
    assert not set(pairs) - named, f"(TILE, family) pairs of build.py's units that step_instantiated does not name: " \
                                   f"{sorted(set(pairs) - named)}"
    for u in units:  # the unit's UPKIE_BODY_CONTACTS_BUILD (launch_step asserts it at compile time too)
        assert {"body" in traits(f) for f in u.families} == {bool(u.body)}, u
