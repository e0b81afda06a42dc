# SPDX-License-Identifier: Apache-2.0
"""The shared-memory-tile step kernel at the block size the library picks for a large batch: one 256-thread block per
SM, whose two tile buffers (72 KB) need the opt-in above 48 KB of dynamic shared memory. Its results must not depend on
the block size: the same ticks with 128-thread blocks (36 KB, no opt-in) are bit-identical, full and partial last
warps alike."""
import numpy as np
import pytest

from conftest import random_servo_actions, random_states
from upkie_b200 import _abi

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n", [65536, 65536 - 40])
def test_tile_kernel_results_do_not_depend_on_the_block_size(model, monkeypatch, n):
    import torch

    from upkie_b200.sim import UpkieSim

    st = torch.from_numpy(random_states(n, seed=5).astype(np.float32)).cuda()
    sims = {}
    for block in (None, "128"):
        if block:
            monkeypatch.setenv("UPKIE_B200_BLOCK", block)  # read when the handle is created
        else:
            monkeypatch.delenv("UPKIE_B200_BLOCK", raising=False)
        sims[block] = UpkieSim(n, model=model, config=_abi.default_sim_config())
        sims[block].set_state(st)
    monkeypatch.delenv("UPKIE_B200_BLOCK", raising=False)
    for k in range(3):
        # torque commands up to the limits: robots on joint bounds, in contact and in flight in the same blocks
        a = torch.from_numpy(random_servo_actions(n, model, seed=10 + k, torque_mode=True).astype(np.float32)).cuda()
        (o_new, t_new), (o_ref, t_ref) = (sims[b].step_servos_compact(a) for b in (None, "128"))
        torch.cuda.synchronize()
        assert torch.equal(o_new, o_ref) and torch.equal(t_new, t_ref), f"tick {k}"
    assert torch.equal(sims[None].get_state(), sims["128"].get_state())
