# SPDX-License-Identifier: Apache-2.0
"""The shared-memory-tile step kernels (TILE=1) keep each lane's clamped action row in its warp's tile for the
substeps, and size the tile from the tiles a block walks: one buffer per warp when every block steps one tile (the
device-buffer compact step), two for the persistent host-buffer launch (UPKIE_B200_ZERO_COPY=1: 128-thread blocks,
about four tiles per block, the next tile's rows prefetched into the second buffer). Both launches run the same kernel
and must give the same bits, full and partial last warps alike, in the headline family, in the action-delay family
with the new command switching in inside the tick, and in spine mode. The device-buffer kernel (TILE=0) keeps the row
in registers; it is a separate compilation, so it agrees to round-off (tests/test_gpu_envs.py)."""
import numpy as np
import pytest

from conftest import random_servo_actions, random_states
from upkie_b200 import _abi

pytestmark = pytest.mark.gpu

SEED = 31


def _config(feature):
    cfg = _abi.default_sim_config()
    cfg.servos_fall_termination = 1  # robots fall and reset (next-step auto-reset) during the ticks
    cfg.min_base_height = 0.15
    if feature == "spine":
        cfg.spine_mode = 1
    return cfg


def _sim(model, feature, n, zero_copy, monkeypatch):
    import torch

    from upkie_b200.sim import AUTORESET_NEXT_STEP, UpkieSim

    monkeypatch.setenv("UPKIE_B200_ZERO_COPY", str(zero_copy))  # read when the handle is created
    s = UpkieSim(n, model=model, config=_config(feature))
    monkeypatch.delenv("UPKIE_B200_ZERO_COPY")
    s.set_autoreset(AUTORESET_NEXT_STEP, SEED, 0)
    if feature == "delay":
        s.set_action_delay(1, 4)  # substeps: every env switches to its new command inside the tick
    s.reset(seed=SEED)
    s.set_state(torch.from_numpy(random_states(n, seed=7).astype(np.float32)).cuda())
    torch.cuda.synchronize()  # the host-buffer steps run on the handle's own streams
    return s


@pytest.mark.parametrize("feature", ["limits", "delay", "spine"])
@pytest.mark.parametrize("n", [65536, 65536 - 40])
def test_one_tile_and_persistent_launches_agree(model, monkeypatch, feature, n):
    import torch

    tile = _sim(model, feature, n, 2, monkeypatch)  # step_servos_compact: one tile per block, one buffer
    host = _sim(model, feature, n, 1, monkeypatch)  # zero-copy host step: persistent blocks, two buffers
    dev = _sim(model, feature, n, 2, monkeypatch)   # step_servos: TILE=0, the row in registers
    pinned = host.host_action_buffer(36)
    for k in range(4):
        # torque commands up to the limits: robots on joint bounds, in contact and in flight in the same warps
        a = random_servo_actions(n, model, seed=40 + k, torque_mode=True).astype(np.float32)
        o1, t1 = tile.step_servos_compact(torch.from_numpy(a).cuda())
        pinned[:] = a
        o2, t2 = host.step_servos_host_compact(pinned)
        o3, _, t3, _ = dev.step_servos(torch.from_numpy(a).cuda())
        torch.cuda.synchronize()
        o1, t1 = o1.cpu().numpy(), t1.cpu().numpy()
        assert np.array_equal(o1, o2) and np.array_equal(t1, t2), f"tick {k}"
        if k == 0:
            d = np.abs(o3.cpu().numpy()[:, :, :3] - o1)
            assert np.median(d) < 1e-5 and np.mean(d.max(axis=(1, 2)) > 1e-3) < 1e-3, (np.median(d), d.max())
            assert np.mean(t3.cpu().numpy() != t1) < 1e-3
    assert torch.equal(tile.get_state(), host.get_state())
    assert (tile.error_flags() == host.error_flags()).all()
