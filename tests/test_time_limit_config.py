# SPDX-License-Identifier: Apache-2.0
"""Episode time limit (max_episode_steps): configuration plumbing and forwarding, no GPU needed."""
import sys
import types

import pytest

from upkie_b200 import UpkieException, _abi


def test_make_config_carries_the_limit():
    from upkie_b200.envs import make_config

    assert make_config().max_episode_steps == 0  # default: no limit, as the reference
    assert _abi.default_sim_config().max_episode_steps == 0
    assert make_config(max_episode_steps=1000).max_episode_steps == 1000
    assert make_config(200.0, max_episode_steps=1).max_episode_steps == 1


@pytest.mark.parametrize("bad", [-1, -1000, 2.5, 2**31])
def test_invalid_limits_are_rejected(bad):
    from upkie_b200.envs import B200VectorEnv, make_config

    with pytest.raises(UpkieException):
        make_config(max_episode_steps=bad)
    # rejected before any device is touched
    with pytest.raises(UpkieException):
        B200VectorEnv(4, "pendulum", max_episode_steps=bad)


class _Recorder:
    calls = []

    def __init__(self, num_envs, env_type, **kwargs):
        _Recorder.calls.append((num_envs, env_type, kwargs))


def test_make_vec_and_register_forward_the_limit(monkeypatch):
    import upkie_b200
    from upkie_b200 import envs

    _Recorder.calls.clear()
    monkeypatch.setattr(envs, "B200VectorEnv", _Recorder)
    upkie_b200.make_vec("Upkie-B200-Pendulum", 8, max_episode_steps=300)
    assert _Recorder.calls[-1] == (8, "pendulum", {"max_episode_steps": 300})

    registered = {}
    gym = types.ModuleType("gymnasium")
    gym.registry = {}
    gym.register = lambda id, vector_entry_point: registered.__setitem__(id, vector_entry_point)
    monkeypatch.setitem(sys.modules, "gymnasium", gym)
    upkie_b200.register()
    registered["Upkie-B200-Servos"](num_envs=16, max_episode_steps=50)
    assert _Recorder.calls[-1] == (16, "servos", {"max_episode_steps": 50})
