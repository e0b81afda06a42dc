# SPDX-License-Identifier: Apache-2.0
"""Exact-mode parity: the device-buffer kernels compiled WITHOUT --use_fast_math (libupkie_b200_exact.so,
upkie_b200/build.py: build_exact) against the fp64 oracle, next to the product library with its shortcut (fast-math)
on the same inputs; both stop their PGS sweeps by Bullet's residual rule (solver_residual_threshold), like the oracle.
Through the C ABI of include/upkie_b200.h, loaded a second time with ctypes."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import random_servo_actions, random_states
from upkie_b200 import _abi

pytestmark = pytest.mark.gpu


def _load_exact():
    from upkie_b200 import _lib, build

    path = build.EXACT_LIB_PATH
    if not os.path.exists(path):
        pytest.fail(f"{path} missing: __graft_entry__.build() builds it")
    L = C.CDLL(path)
    for name, (restype, argtypes) in _lib.SYMBOLS.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    assert L.upkie_b200_abi_version() == _abi.ABI_VERSION
    return L


def _one_tick(L, model, cfg, st32, act32, torch):
    n = st32.shape[0]
    ms = model.to_struct()
    h = C.c_void_p()
    assert L.upkie_b200_create(C.byref(ms), C.byref(cfg), n, 0, C.byref(h)) == 0, L.upkie_b200_last_error()
    dev = torch.device("cuda", 0)
    state = torch.from_numpy(st32).to(dev)
    act = torch.from_numpy(act32).to(dev)
    obs = torch.empty((n, 6, 5), dtype=torch.float32, device=dev)
    rew = torch.empty(n, dtype=torch.float32, device=dev)
    term = torch.empty(n, dtype=torch.uint8, device=dev)
    trunc = torch.empty(n, dtype=torch.uint8, device=dev)
    out = torch.empty((n, _abi.STATE_DIM), dtype=torch.float32, device=dev)
    s = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    assert L.upkie_b200_set_state(h, p(state), s) == 0
    assert L.upkie_b200_step_servos(h, p(act), p(obs), p(rew), p(term), p(trunc), s) == 0, L.upkie_b200_last_error()
    assert L.upkie_b200_get_state(h, p(out), s) == 0
    torch.cuda.synchronize()
    res = out.cpu().numpy().astype(np.float64), term.cpu().numpy().copy()
    L.upkie_b200_destroy(h)
    return res


def test_exact_mode_one_tick_against_the_oracle(model, oracle_lib):
    import torch

    from upkie_b200 import _lib
    from test_gpu_sim_parity import _report

    n = 2048
    st32 = random_states(n, seed=3).astype(np.float32)
    act32 = random_servo_actions(n, model, seed=4).astype(np.float32)
    cfg_exact = _abi.default_sim_config()
    cfg_fast = _abi.default_sim_config()
    osim = oracle_lib.OracleSim(model, cfg_exact, n, threads=8)
    osim.set_state(st32.astype(np.float64))
    _, _, oterm, _ = osim.step_servos(act32.astype(np.float64))
    ref = osim.get_state()
    exact, eterm = _one_tick(_load_exact(), model, cfg_exact, st32, act32, torch)
    fast, fterm = _one_tick(_lib.lib(), model, cfg_fast, st32, act32, torch)
    err = {}
    for name, g in (("exact", exact), ("fast", fast)):
        d = np.abs(g[:, :25] - ref[:, :25])
        err[name] = {"pose": d[:, :7].max(), "twist": d[:, 7:13].max(), "q": d[:, 13:19].max(),
                     "qd_worst": d[:, 19:25].max(), "qd_p99": np.percentile(d[:, 19:25].max(axis=1), 99),
                     "qd_median": np.median(d[:, 19:25].max(axis=1))}
    _report("exact_mode_one_tick_2048", **{f"{k}_{m}": v for k, e in err.items() for m, v in e.items()})
    e = err["exact"]
    assert e["pose"] < 2e-5 and e["q"] < 2e-4
    assert e["qd_median"] < 5e-5 and e["qd_p99"] < 1e-3 and e["qd_worst"] < 2e-2 and e["twist"] < 1e-3
    # the shortcut of the product library (fast-math) stays in the same error class as plain fp32 (no order-of-magnitude loss)
    f = err["fast"]
    assert f["pose"] < 2e-5 and f["twist"] < 1e-3, (f["pose"], f["twist"])  # the caps of the exact library
    assert f["qd_median"] < 5 * max(e["qd_median"], 2e-6) and f["qd_p99"] < 5 * max(e["qd_p99"], 5e-5)
    assert np.array_equal(eterm, oterm) and np.array_equal(fterm, oterm)
