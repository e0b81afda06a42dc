# SPDX-License-Identifier: Apache-2.0
"""The step kernels' families (upkie_b200/csrc/step_family.h), compiled for the CPU (tests/hostsim/step_family.cpp):
what each family compiles in, and the family the host picks for a handle's features and transport, with every
rejection and its message. The GPU tests of each feature run the kernels the choice names. No GPU needed."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))

MODE_SERVOS, MODE_GYROPOD, MODE_PENDULUM = 0, 1, 2
DEVICE, HOST_TILE, IN_KERNEL = 0, 1, 2  # the TILE of the step kernels
FAM_PLAIN, FAM_EXTRAS, FAM_LIMITS, FAM_SPINE, FAM_BODY, FAM_TABLE, FAM_PUSH, FAM_BODY_PUSH = range(8)

TRAITS = ("extras", "limits", "table", "reset_rand", "spine", "body", "push")
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
}

NO_TABLE = ("the per-env parameter table has no in-kernel rollout transport (use upkie_b200_step with compact rows)")
NO_PUSH = "push randomisation has no in-kernel rollout transport (use upkie_b200_step with compact rows)"
NO_LIMIT = ("max_episode_steps has no in-kernel rollout transport: it does not carry truncated (use upkie_b200_step "
            "with compact rows)")
NO_BODY = "body_contacts has no in-kernel rollout transport (use upkie_b200_step_servos_compact)"
SPINE_SERVOS = "spine_mode supports UpkieServos steps only"
NO_SPINE = "spine_mode has no in-kernel rollout transport"

_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "step_family.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_family_"), "libhostsim_family.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        L.hostsim_family_traits.argtypes = [C.c_int, C.POINTER(C.c_uint8)]
        L.hostsim_step_family.argtypes = [C.c_int] * 11 + [C.c_char_p, C.c_int]
        L.hostsim_step_family.restype = C.c_int
        _LIB = L
    return _LIB


def traits(family):
    out = (C.c_uint8 * len(TRAITS))()
    _lib().hostsim_family_traits(family, out)
    return {name for name, v in zip(TRAITS, out) if v}


def step_family(mode=MODE_SERVOS, transport=DEVICE, joint_limits=0, ctrl_noise=0, meas_noise=0, ext=0, table=0,
                body_contacts=0, push=0, spine_mode=0, max_episode_steps=0):
    """(family, rejection message or None)"""
    why = C.create_string_buffer(256)
    f = _lib().hostsim_step_family(joint_limits, ctrl_noise, meas_noise, ext, table, body_contacts, push, spine_mode,
                                   max_episode_steps, mode, transport, why, len(why))
    return f, (why.value.decode() or None)


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
