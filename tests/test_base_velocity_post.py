# SPDX-License-Identifier: Apache-2.0
"""UpkieBaseVelocity auto-resets and the fused epilogue (upkie_b200_base_velocity_post), no GPU needed: the CPU
build of the kernel's per-env arithmetic against a NumPy statement of the auto-reset table, the golden runs of the
reference's own class under both Gymnasium modes replayed through base_velocity_tick on the oracle, the ABI mirror,
and the forwarding of autoreset_mode through make_vec / register()."""
import ctypes as C
import json
import os
import re
import subprocess
import sys
import tempfile
import types

import numpy as np
import pytest

from upkie_b200 import _abi

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "base_velocity_autoreset_runs.json")


def test_post_step_struct_mirror_matches_the_header():
    """The entry point is an addition to ABI 8: the version is unchanged and the ctypes mirror of
    UpkieBaseVelocityPost (seven pointers, then dt and the mode) has the header's fields and size."""
    header = open(os.path.join(HERE, "..", "include", "upkie_b200.h")).read()
    defs = dict(re.findall(r"#define (UPKIE_\w+) (\d+)", header))
    assert int(defs["UPKIE_B200_ABI_VERSION"]) == _abi.ABI_VERSION
    fields = re.search(r"typedef struct UpkieBaseVelocityPost \{(.*?)\} UpkieBaseVelocityPost;", header, re.S).group(1)
    names = re.findall(r"\b(\w+);", fields)
    assert names == [f for f, _ in _abi.UpkieBaseVelocityPost._fields_]
    assert C.sizeof(_abi.UpkieBaseVelocityPost) == 7 * 8 + 8


# ---- the kernel's per-env arithmetic on the CPU ----------------------------------------------------------------------

@pytest.fixture(scope="module")
def post_lib():
    src = os.path.join(HERE, "hostsim", "base_velocity_post.cpp")
    out = os.path.join(tempfile.mkdtemp(prefix="upkie_bv_"), "libhostsim_bv_post.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
    L = C.CDLL(out)
    L.hostsim_bv_post.argtypes = [C.c_int, C.c_int, C.c_float] + [C.c_void_p] * 8
    L.hostsim_bv_post.restype = None
    return L


SENTINEL = -12345.0


def _post(L, mode, dt, reset, action, gyro_obs, gyro_fin, xy, v_cmd):
    n = action.shape[0]
    xy, v_cmd = xy.copy(), v_cmd.copy()
    obs = np.full((n, 3), np.nan, np.float32)
    fin = np.full((n, 3), SENTINEL, np.float32)
    L.hostsim_bv_post(n, mode, dt, reset.ctypes.data, action.ctypes.data, gyro_obs.ctypes.data, gyro_fin.ctypes.data,
                      xy.ctypes.data, v_cmd.ctypes.data, obs.ctypes.data, fin.ctypes.data)
    return xy, v_cmd, obs, fin


def _numpy_post(mode, dt, reset, action, gyro_obs, gyro_fin, xy, v_cmd):
    """The auto-reset table in NumPy fp32: base_velocity_tick's dead reckoning (v * cos(yaw)) * dt, then the add,
    and UpkieBaseVelocity.reset for the envs that reset."""
    f32 = np.float32
    v = action[:, 0]

    def reckon(x, y, yaw):
        c = np.cos(yaw.astype(np.float64)).astype(f32)  # correctly rounded cos / sin: the kernel's cosf / sinf are
        s = np.sin(yaw.astype(np.float64)).astype(f32)  # IEEE routines within 1 ulp of them
        return (x + (v * c) * f32(dt)).astype(f32), (y + (v * s) * f32(dt)).astype(f32)

    r = reset.astype(bool) & (mode != 0)
    x, y = reckon(xy[:, 0], xy[:, 1], gyro_obs[:, 2])
    obs = np.stack([x, y, gyro_obs[:, 2]], 1)
    fx, fy = reckon(xy[:, 0], xy[:, 1], gyro_fin[:, 2])
    fin = np.full_like(obs, SENTINEL)
    if mode == 2:
        fin[r] = np.stack([fx, fy, gyro_fin[:, 2]], 1)[r]
    obs[r] = 0.0
    new_xy = np.stack([x, y], 1)
    new_xy[r] = 0.0
    v_new = v_cmd.copy()
    v_new[r] = 0.0
    return new_xy, v_new, obs, fin


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_post_step_matches_the_autoreset_table(post_lib, mode):
    rng = np.random.default_rng(mode)
    n, dt = 4096, 1.0 / 200.0
    f32 = np.float32
    action = rng.uniform(-3, 3, (n, 2)).astype(f32)
    gyro_obs = rng.uniform(-1, 1, (n, 6)).astype(f32)
    gyro_obs[:, 2] = rng.uniform(-40, 40, n).astype(f32)  # yaw is never wrapped (upkie_gyropod.py:383-384)
    gyro_fin = rng.uniform(-1, 1, (n, 6)).astype(f32)
    gyro_fin[:, 2] = rng.uniform(-40, 40, n).astype(f32)
    xy = rng.uniform(-5, 5, (n, 2)).astype(f32)
    v_cmd = rng.uniform(-3, 3, n).astype(f32)
    reset = (rng.random(n) < 0.3).astype(np.uint8)
    got = _post(post_lib, mode, dt, reset, action, gyro_obs, gyro_fin, xy, v_cmd)
    want = _numpy_post(mode, dt, reset, action, gyro_obs, gyro_fin, xy, v_cmd)
    r = reset.astype(bool) & (mode != 0)
    for g, w, name in zip(got, want, ("xy", "v_cmd", "obs", "final_obs")):
        # reset rows, final rows, untouched rows and the yaw column: exact; dead-reckoned values: within the
        # difference of cosf / sinf and the correctly rounded values (one rounding of a product of size v * dt)
        assert np.array_equal(g[r], w[r]), name
        if name == "final_obs":
            assert np.all(g[~r] == SENTINEL)
            ok = r if mode == 2 else np.zeros(n, bool)
            assert np.allclose(g[ok], w[ok], rtol=0, atol=1e-6)
        elif name == "v_cmd":
            assert np.array_equal(g, w)  # untouched where no reset
        else:
            assert np.allclose(g[~r], w[~r], rtol=0, atol=1e-6), name
    obs = got[2]
    assert np.array_equal(obs[~r, 2], gyro_obs[~r, 2])
    assert np.array_equal(obs[~r, :2], got[0][~r])  # the observation is the updated (x, y)
    assert not obs[r].any() and not got[0][r].any()


def test_dead_reckoning_rounds_each_product_and_the_sum(post_lib):
    """At yaw = 0, cos = 1 and sin = 0 exactly: x + v * dt must be round(x + round(v * float32(dt))), not an FMA."""
    f32 = np.float32
    n, dt = 1 << 14, 1.0 / 200.0
    rng = np.random.default_rng(7)
    action = rng.uniform(-3, 3, (n, 2)).astype(f32)
    gyro = np.zeros((n, 6), f32)
    xy = rng.uniform(-100, 100, (n, 2)).astype(f32)
    xy_new, _, obs, _ = _post(post_lib, 0, dt, np.zeros(n, np.uint8), action, gyro, gyro, xy, np.zeros(n, f32))
    want = (xy[:, 0] + (action[:, 0] * f32(1.0)) * f32(dt)).astype(f32)
    assert np.array_equal(xy_new[:, 0], want) and np.array_equal(xy_new[:, 1], xy[:, 1])
    fused = (xy[:, 0].astype(np.float64) + action[:, 0].astype(np.float64) * f32(dt)).astype(f32)
    assert (fused != want).any()  # the check separates the two roundings


# ---- golden runs of the reference's class under both auto-reset modes -----------------------------------------------

@pytest.mark.parametrize("mode", ["next_step", "same_step"])
def test_autoreset_golden_replays_through_base_velocity_tick(model, oracle_lib, mode):
    import torch

    from upkie_b200.base_velocity import base_velocity_tick, mpc_inputs_from_spine

    runs = json.load(open(GOLDEN))
    run, T = runs[mode], runs["time_limit"]
    cfg = _abi.default_sim_config()
    osim = oracle_lib.OracleSim(model, cfg, 1, threads=1)
    om = oracle_lib.OracleMpc(_abi.default_mpc_config())
    init = np.asarray(run["init_row"]).reshape(1, -1)
    state = {"v": np.zeros(1)}

    def mpc_step_spine(target, spine, dt):
        x0, contact = mpc_inputs_from_spine(spine)
        vc, _, found, _ = om.step(x0.numpy().astype(np.float64), target.numpy().astype(np.float64), contact.numpy(), dt,
                                  state["v"])
        assert found.all()
        state["v"] = vc
        return torch.from_numpy(vc.astype(np.float32))

    def step_gyropod(a):
        obs, rew, term, trunc = osim.step_gyropod(a.numpy().astype(np.float64), 2)
        return (torch.from_numpy(obs.astype(np.float32)), torch.from_numpy(rew.astype(np.float32)),
                torch.from_numpy(term), torch.from_numpy(trunc))

    def spine_obs():
        return torch.from_numpy(osim.spine_obs().astype(np.float64))

    def reset():  # UpkieBaseVelocity.reset (upkie_base_velocity.py:137-162): nominal state, MPC reset, x = y = 0
        osim.reset(init)
        state["v"] = np.zeros(1)
        xy.zero_()
        return spine_obs()

    xy = torch.zeros((1, 2), dtype=torch.float64)
    spine = reset()
    elapsed, pending = 0, False
    worst = worst_fin = 0.0
    episodes = 1
    for t, a in enumerate(run["actions"]):
        fin = None
        if mode == "next_step" and pending:
            spine = reset()
            obs, term, trunc, elapsed = np.zeros(3), False, False, 0
            episodes += 1
        else:
            o, rew, te, _, spine = base_velocity_tick(torch.tensor([a], dtype=torch.float32), spine, xy, cfg.dt,
                                                      mpc_step_spine, step_gyropod, spine_obs)
            obs, term = o.numpy()[0], bool(te[0])
            assert float(rew[0]) == 0.0
            elapsed += 1
            trunc = elapsed >= T
            if mode == "same_step" and (term or trunc):
                fin, obs, elapsed = obs, np.zeros(3), 0
                spine = reset()
                episodes += 1
        assert term == run["terminated"][t] and trunc == run["truncated"][t], t
        assert (fin is None) == (run["final_obs"][t] is None), t
        if fin is not None:
            worst_fin = max(worst_fin, float(np.abs(fin - np.asarray(run["final_obs"][t])).max()))
        worst = max(worst, float(np.abs(obs - np.asarray(run["obs"][t])).max()))
        assert abs(float(state["v"][0]) - run["commanded_velocity"][t]) < 1e-6, t
        pending = term or trunc
    assert worst < 5e-6 and worst_fin < 5e-6, (worst, worst_fin)
    assert episodes >= 4 and any(run["truncated"])


# ---- forwarding ------------------------------------------------------------------------------------------------------

class _Recorder:
    calls = []

    def __init__(self, num_envs, env_type, **kwargs):
        _Recorder.calls.append((num_envs, env_type, kwargs))


@pytest.mark.parametrize("mode", ["next_step", "same_step", "disabled"])
def test_make_vec_and_register_forward_autoreset_mode(monkeypatch, mode):
    import upkie_b200
    from upkie_b200 import envs

    _Recorder.calls.clear()
    monkeypatch.setattr(envs, "B200VectorEnv", _Recorder)
    for robot in ("Upkie", "Cookie"):
        upkie_b200.make_vec(f"{robot}-B200-BaseVelocity", 8, autoreset_mode=mode, model=object())
        assert _Recorder.calls[-1][:2] == (8, "base_velocity")
        assert _Recorder.calls[-1][2]["autoreset_mode"] == mode

    registered = {}
    gym = types.ModuleType("gymnasium")
    gym.registry = {}
    gym.register = lambda id, vector_entry_point: registered.__setitem__(id, vector_entry_point)
    monkeypatch.setitem(sys.modules, "gymnasium", gym)
    upkie_b200.register()
    registered["Upkie-B200-BaseVelocity"](num_envs=16, autoreset_mode=mode, max_episode_steps=50)
    assert _Recorder.calls[-1] == (16, "base_velocity", {"autoreset_mode": mode, "max_episode_steps": 50})

