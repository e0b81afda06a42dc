# SPDX-License-Identifier: Apache-2.0
"""info["final_info"] without a GPU: the ctypes mirror of UpkieStepOutputs with its final_state field, the binding of
upkie_b200_final_spine_obs, and the vector env's lazy terminal spine observations over a stub simulator."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from upkie_b200 import _abi

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "upkie_b200.h")


def test_step_outputs_mirror_keeps_its_layout():
    S = _abi.UpkieStepOutputs
    assert C.sizeof(S) == 48
    offsets = {name: getattr(S, name).offset for name, _ in S._fields_}
    assert offsets == {"obs": 0, "reward": 8, "terminated": 16, "truncated": 24, "final_obs": 32, "compact": 40,
                       "final_state": 44}
    with open(HEADER) as f:
        header = f.read()
    body = re.search(r"typedef struct UpkieStepOutputs \{(.*?)\} UpkieStepOutputs;", header, re.S).group(1)
    fields = re.findall(r"\b(\w+);", body)
    assert fields == [name for name, _ in S._fields_]
    assert "#define UPKIE_B200_ABI_VERSION 8" in header and _abi.ABI_VERSION == 8


def test_final_spine_obs_is_declared_and_bound():
    from upkie_b200 import _lib

    with open(HEADER) as f:
        assert "int upkie_b200_final_spine_obs(void* handle, float* out, void* stream);" in f.read()
    restype, argtypes = _lib.SYMBOLS["upkie_b200_final_spine_obs"]
    assert restype is C.c_int and argtypes == [C.c_void_p] * 3
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libupkie_b200.so is not built")
    lib = _lib.lib()
    assert lib.upkie_b200_final_spine_obs.argtypes == [C.c_void_p] * 3
    assert lib.upkie_b200_final_spine_obs(None, None, None) == -1  # EINVAL before any device call


def same_dict(a, b) -> bool:
    """Nested dictionaries of the reference's spine observation (lists, floats, arrays) are equal."""
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(same_dict(a[k], b[k]) for k in a)
    return np.array_equal(np.asarray(a), np.asarray(b))


class StubSim:
    """What the lazy spine observations read from UpkieSim: the launch count and the two row fetches."""

    def __init__(self, n):
        rng = np.random.default_rng(0)
        self.n = n
        self.launches = 7
        self.rows = torch.from_numpy(rng.normal(size=(n, _abi.SPINE_DIM)).astype(np.float32))
        self.final_rows = torch.from_numpy(rng.normal(size=(n, _abi.SPINE_DIM)).astype(np.float32))
        self.fetches = 0

    def spine_obs(self):
        self.fetches += 1
        return self.rows

    def final_spine_obs(self):
        self.fetches += 1
        return self.final_rows


def test_final_spine_observations_format_rows_like_the_reference():
    from upkie_b200.envs import FinalSpineObservations, SpineObservations, spine_row_to_dict

    sim = StubSim(5)
    fin = FinalSpineObservations(sim)
    assert isinstance(fin, SpineObservations) and len(fin) == 5
    assert sim.fetches == 0  # lazy
    assert fin.tensor is sim.final_rows
    assert np.array_equal(fin.array, sim.final_rows.numpy())
    assert same_dict(fin[3], spine_row_to_dict(sim.final_rows.numpy()[3]))
    assert sim.fetches == 1  # fetched once
    obs = SpineObservations(sim)
    assert obs.tensor is sim.rows and same_dict(obs[1], spine_row_to_dict(sim.rows.numpy()[1]))


def test_lazy_rows_refuse_a_later_tick():
    from upkie_b200.envs import FinalSpineObservations, SpineObservations
    from upkie_b200.exceptions import UpkieRuntimeError

    sim = StubSim(4)
    fin, obs = FinalSpineObservations(sim), SpineObservations(sim)
    read = FinalSpineObservations(sim)
    read.array
    sim.launches += 1
    with pytest.raises(UpkieRuntimeError, match=r"info\['final_info'\]\['spine_observation'\]"):
        fin.array
    with pytest.raises(UpkieRuntimeError, match=r"info\['final_info'\]\['spine_observation'\]"):
        fin.tensor
    with pytest.raises(UpkieRuntimeError, match=r"info\['spine_observation'\]"):
        obs[0]
    assert read[2] is not None  # read before the simulator moved on: kept


@pytest.mark.parametrize("arrays", ["numpy", "torch"])
def test_final_info_keys_and_masks(arrays):
    """Gymnasium 1.x SyncVectorEnv layout in same-step mode: final_info = {key: ..., _key: mask}, _final_info = mask,
    next to final_obs / _final_obs; no key at all on a step without a reset."""
    from upkie_b200.envs import B200VectorEnv, FinalSpineObservations

    n = 6
    env = B200VectorEnv.__new__(B200VectorEnv)
    env.sim = StubSim(n)
    term = np.array([0, 1, 0, 0, 1, 0], np.uint8)
    trunc = np.array([0, 0, 1, 0, 1, 0], np.uint8)
    fin = np.zeros((n, 4), np.float32)
    if arrays == "torch":
        term, trunc, fin = torch.from_numpy(term), torch.from_numpy(trunc), torch.from_numpy(fin)
    info = {}
    env._add_final_obs(info, term * 0, trunc * 0, fin, lambda f: f)
    assert info == {}
    env._add_final_obs(info, term, trunc, fin, lambda f: f)
    assert set(info) == {"final_obs", "_final_obs", "final_info", "_final_info"}
    assert set(info["final_info"]) == {"spine_observation", "_spine_observation"}
    assert isinstance(info["final_info"]["spine_observation"], FinalSpineObservations)
    expect = np.array([0, 1, 1, 0, 1, 0], bool)
    masks = [info["_final_obs"], info["_final_info"], info["final_info"]["_spine_observation"]]
    for m in masks:
        m = m.numpy() if arrays == "torch" else m
        assert m.dtype == np.bool_ and np.array_equal(m, expect)
    # separate mask objects, as Gymnasium's: editing one leaves the others
    masks[1][0] = True
    assert not masks[0][0] and not masks[2][0]
    row = info["final_info"]["spine_observation"][2]
    assert row["base_orientation"]["pitch"] == pytest.approx(float(env.sim.final_rows[2, _abi.SP_PITCH]))
