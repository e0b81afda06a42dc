# SPDX-License-Identifier: Apache-2.0
"""Delays of more than one tick without a GPU: the history helpers the step kernels and the delay kernels inline
(tests/hostsim/delay_ticks.cpp, compiled for the CPU) against a NumPy statement of the rule of include/upkie_b200.h,
for every delay up to the history's depth; and the Python spec functions' rounding, depth bound and messages."""

import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import action_delay_spec, observation_delay_spec

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")

_LIB = None
u32p, fp = C.POINTER(C.c_uint32), C.POINTER(C.c_float)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "delay_ticks.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_delay_ticks_"), "libhostsim_delay_ticks.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        u32 = C.c_uint32
        L.hostsim_delay_split.argtypes = [u32, u32, u32, u32p]
        L.hostsim_delay_ring_row.argtypes = [u32, u32, u32]
        L.hostsim_delay_ring_row.restype = u32
        L.hostsim_action_delay_rows.argtypes = [u32, u32, u32, u32, u32p]
        L.hostsim_obs_delay_rows.argtypes = [u32, u32, u32, u32, u32p]
        L.hostsim_action_delay_reset_ticks.argtypes = [C.POINTER(_abi.UpkieActionDelay), C.c_uint64, C.c_int, u32p,
                                                       u32p, fp, C.c_int, C.c_int]
        L.hostsim_obs_delay_fill_history.argtypes = [fp, C.c_int, C.c_int, C.c_int, fp]
        L.hostsim_delay_ticks_spec_error.argtypes = [C.c_int, u32, u32, C.c_int, u32, C.c_char_p, C.c_int]
        _LIB = L
    return _LIB


def _call3(fn, *args):
    out = (C.c_uint32 * 3)()
    fn(*args, out)
    return tuple(out)


CASES = [(nb, K) for nb in (1, 2, 5) for K in (1, 2, 4, _abi.MAX_DELAY_TICKS)]
TICKS = 20  # ticks after a reset: more than the deepest history, so that the ring wraps


@pytest.mark.parametrize("nb, K", CASES)
def test_action_command_of_each_substep(nb, K):
    """Simulate the ring of one env after a reset with commands named by their tick (-1 the stop row): substep s of
    tick t runs the command of tick t - q - 1 for s < r and t - q for s >= r, d = q * nb + r with 0 <= r < nb, stop
    rows before the reset; a delay above K * nb acts as K * nb"""
    L = _lib()
    for d in range(K * nb + 3):
        dd = min(d, K * nb)
        q, r = divmod(dd, nb)
        ring, head = [-1] * K, 0  # the reset's stop rows
        for t in range(TICKS):
            first_row, second_row, r_k = _call3(L.hostsim_action_delay_rows, d, nb, K, head)
            first = ring[first_row]  # read before the store, as the kernel does
            ring[head] = t
            second = ring[second_row]
            head = (head + 1) % K
            for s in range(nb):
                got = first if s < r_k else second
                want = t - q - 1 if s < r else t - q
                assert got == max(want, -1), (nb, K, d, t, s)
        # the ring in age order: age a is the command of tick TICKS - 1 - a
        ages = [ring[L.hostsim_delay_ring_row(head, K, a)] for a in range(K)]
        assert ages == [TICKS - 1 - a for a in range(K)]


@pytest.mark.parametrize("nb, K", CASES)
def test_observation_instant_of_each_report(nb, K):
    """Simulate the snapshot ring of one env after a reset with snapshots named by their instant (substeps since the
    reset): after tick t the step reports the end of substep nb - r of tick t - q, d = q * nb + r with 0 <= r < nb,
    the post-reset state (instant 0) for instants before the reset; each snapshot differentiates its IMU velocity
    against the previous tick's snapshot"""
    L = _lib()
    for d in range(K * nb + 3):
        dd = min(d, K * nb)
        q, r = divmod(dd, nb)
        ring, head, last = [0] * K, 0, 0
        for t in range(TICKS):
            newest, report, r_k = _call3(L.hostsim_obs_delay_rows, d, nb, K, head)
            assert ring[newest] == last  # the previous snapshot (the post-reset state at t = 0)
            ring[head] = t * nb + (nb - r_k)
            last = ring[head]
            head = (head + 1) % K
            assert ring[report] == max((t - q) * nb + (nb - r), 0), (nb, K, d, t)
        if dd <= nb:  # one tick: the snapshot of this tick, as the one-tick kernels take it
            assert (q, r) in ((0, dd), (1, 0))


@pytest.mark.parametrize("nb, K", CASES)
def test_delay_split(nb, K):
    L = _lib()
    out = (C.c_uint32 * 2)()
    for d in range(K * nb + 3):
        L.hostsim_delay_split(d, nb, K, out)
        dd = min(d, K * nb)
        q, r = out
        assert q * nb + r == dd and q < K and (1 <= r <= nb if dd else r == 0)


def test_ring_rows_are_a_permutation():
    L = _lib()
    for K in range(1, _abi.MAX_DELAY_TICKS + 1):
        for head in range(K):
            rows = [L.hostsim_delay_ring_row(head, K, a) for a in range(K)]
            assert sorted(rows) == list(range(K))
            assert rows[K - 1] == head  # the oldest row is the next write


@pytest.mark.parametrize("K", [1, 3, _abi.MAX_DELAY_TICKS])
def test_reset_fills(K):
    L = _lib()
    n, stride = 5, 8
    cmd = np.full((K, _abi.ACT_DIM, stride), 7.0, dtype=np.float32)
    count = np.zeros(n, dtype=np.uint32)
    delay = np.zeros(n, dtype=np.uint32)
    spec = _abi.UpkieActionDelay(0, 3 * K)
    L.hostsim_action_delay_reset_ticks(C.byref(spec), 11, n, count.ctypes.data_as(u32p), delay.ctypes.data_as(u32p),
                                       cmd.ctypes.data_as(fp), stride, K)
    stop = np.zeros(_abi.ACT_DIM, dtype=np.float32)
    stop[0::len(_abi.ACT_KEYS)] = np.nan
    for s in range(K):
        np.testing.assert_array_equal(cmd[s, :, :n], np.repeat(stop[:, None], n, axis=1))
    assert np.all(cmd[:, :, n:] == 7.0)  # the padding columns are untouched
    assert np.all(count == 1) and np.all(delay <= 3 * K)

    hist = np.full((K, _abi.STATE_DIM, stride), 7.0, dtype=np.float32)
    row = np.arange(_abi.STATE_DIM, dtype=np.float32)
    L.hostsim_obs_delay_fill_history(hist.ctypes.data_as(fp), stride, K, 2, row.ctypes.data_as(fp))
    for s in range(K):
        np.testing.assert_array_equal(hist[s, :, 2], row)
    assert np.all(np.delete(hist, 2, axis=2) == 7.0)


def _c_error(which, low, high, nb, K):
    buf = C.create_string_buffer(256)
    return buf.value.decode() if _lib().hostsim_delay_ticks_spec_error(which, low, high, nb, K, buf, 256) else None


@pytest.mark.parametrize("which, name", [(0, "set_action_delay"), (1, "set_observation_delay")])
def test_c_spec_bound(which, name):
    assert _c_error(which, 0, 5, 5, 1) is None
    assert "at most one tick" in _c_error(which, 0, 6, 5, 1)  # depth 1: the one-tick message
    assert _c_error(which, 0, 20, 5, 4) is None
    assert _c_error(which, 20, 20, 5, 4) is None
    why = _c_error(which, 0, 21, 5, 4)
    assert why.startswith(name) and "max_ticks * nb_substeps" in why
    assert "substeps_low > substeps_high" in _c_error(which, 3, 2, 5, 4)


def test_header_constant():
    with open(HEADER) as f:
        m = re.search(r"#define UPKIE_MAX_DELAY_TICKS (\d+)", f.read())
    assert m and int(m.group(1)) == _abi.MAX_DELAY_TICKS


@pytest.mark.parametrize("spec_fn", [action_delay_spec, observation_delay_spec])
def test_spec_rounding_with_ticks(spec_fn):
    dt = 1.0 / 1000.0  # one substep of 1 ms
    assert spec_fn(0.004, dt, 1, max_ticks=4) == (4, 4)
    assert spec_fn((0.001, 0.004), dt, 1, max_ticks=4) == (1, 4)
    assert spec_fn(0.0035, dt, 1, max_ticks=4) == (4, 4)  # halves up
    assert spec_fn((0.0, 0.0044), dt, 1, max_ticks=4) == (0, 4)
    dt = 1.0 / 200.0  # 5 substeps of 1 ms
    assert spec_fn(0.012, dt, 5, max_ticks=3) == (12, 12)
    assert spec_fn((0.0, 0.015), dt, 5, max_ticks=3) == (0, 15)
    assert spec_fn(0.003, dt, 5) == spec_fn(0.003, dt, 5, max_ticks=1) == (3, 3)
    assert spec_fn(None, dt, 5, max_ticks=8) is None


@pytest.mark.parametrize("spec_fn, name", [(action_delay_spec, "action_delay"),
                                           (observation_delay_spec, "observation_delay")])
def test_spec_rejections_with_ticks(spec_fn, name):
    dt = 1.0 / 1000.0
    with pytest.raises(UpkieException, match=f"{name}: 0.002 s is more than one tick"):
        spec_fn(0.002, dt, 1)
    with pytest.raises(UpkieException, match=f"{name}: 0.002 s is more than one tick"):
        spec_fn(0.002, dt, 1, max_ticks=1)
    with pytest.raises(UpkieException, match=f"{name}: 0.005 s is more than max_ticks = 4 ticks"):
        spec_fn(0.005, dt, 1, max_ticks=4)
    for bad in (0, -1, _abi.MAX_DELAY_TICKS + 1):
        with pytest.raises(UpkieException, match="max_ticks: expected 1 <= max_ticks"):
            spec_fn(0.001, dt, 1, max_ticks=bad)
    for bad in (2.0, True, "2"):
        with pytest.raises(UpkieException, match="max_ticks: expected an integer"):
            spec_fn(0.001, dt, 1, max_ticks=bad)
    with pytest.raises(UpkieException, match="spine_mode"):
        spec_fn(0.001, dt, 1, spine_mode=True, max_ticks=4)
