# SPDX-License-Identifier: Apache-2.0
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def model():
    from upkie_b200.model import Model

    return Model.standard_upkie()


@pytest.fixture(scope="session")
def oracle_lib():
    from oracle import oracle

    oracle.build()
    return oracle


def random_states(n, seed=0, z_range=(0.57, 0.62), vel=1.0, qd=5.0, tilt=0.3):
    """Random simulator states [n, 44] (float64), quaternions normalised."""
    from upkie_b200 import _abi

    rng = np.random.default_rng(seed)
    st = np.zeros((n, _abi.STATE_DIM))
    st[:, 2] = rng.uniform(z_range[0], z_range[1], n)
    quat = rng.normal(size=(n, 4)) * [1, 0.5 * tilt, tilt, 0.5 * tilt]
    quat[:, 0] = 1.0
    quat /= np.linalg.norm(quat, axis=1, keepdims=True)
    st[:, 3:7] = quat
    st[:, 7:13] = rng.uniform(-vel, vel, (n, 6))
    st[:, 13:19] = rng.uniform(-0.8, 0.8, (n, 6))
    st[:, 19:25] = rng.uniform(-qd, qd, (n, 6))
    return st


def random_servo_actions(n, model, seed=1, torque_mode=False):
    """Random UpkieServos actions [n, 6, 6] inside (and slightly outside) the box."""
    rng = np.random.default_rng(seed)
    a = np.zeros((n, 6, 6))
    tau = np.asarray(model.tau_max)
    if torque_mode:
        a[:, :, 0] = np.nan
        a[:, :, 2] = rng.uniform(-1, 1, (n, 6)) * tau
        a[:, :, 5] = tau
        return a
    a[:, :, 0] = rng.uniform(-1.0, 1.0, (n, 6))
    a[:, [2, 5], 0] = np.nan
    nan_mask = rng.uniform(size=(n, 6)) < 0.2
    a[:, :, 0] = np.where(nan_mask, np.nan, a[:, :, 0])
    a[:, :, 1] = rng.uniform(-1, 1, (n, 6)) * np.asarray(model.qd_max) * 0.2
    a[:, :, 2] = rng.uniform(-1.2, 1.2, (n, 6)) * tau * 0.3
    a[:, :, 3] = rng.uniform(-0.5, 6.0, (n, 6))
    a[:, :, 4] = rng.uniform(-0.5, 6.0, (n, 6))
    a[:, :, 5] = rng.uniform(0.2, 1.1, (n, 6)) * tau
    return a


def mpc_kkt_residual(P, q, U, bound):
    """Infinity-norm KKT residual of ``min 1/2 U'PU + q'U  s.t. |U| <= bound`` at ``U`` (the accuracy gate of
    SURVEY.md 8d config 4: <= 1e-3, ProxQP's eps_abs at mpc_balancer.py:76). With g = PU + q the multipliers of
    the box are max(-g, 0) on the upper and max(g, 0) on the lower side: stationarity holds by construction,
    what remains is complementarity (g must vanish, or push outwards, exactly where a bound is active) and
    primal feasibility."""
    U = np.asarray(U, dtype=np.float64)
    g = P @ U + q
    tol_active = 1e-6 * max(1.0, bound)
    upper = U >= bound - tol_active
    lower = U <= -bound + tol_active
    r = np.abs(g)
    r[upper] = np.maximum(g[upper], 0.0)   # at the upper bound the gradient may only point down (g <= 0)
    r[lower] = np.maximum(-g[lower], 0.0)  # at the lower bound only up
    primal = max(0.0, float(np.max(np.abs(U)) - bound))
    return max(float(r.max()), primal)


def at_joint_bounds(model, n, seed):
    """Random states with about a third of the hips and knees at or slightly beyond a bound."""
    rng = np.random.default_rng(seed)
    st = random_states(n, seed=seed + 1).astype(np.float32)
    st[: n // 2, 2] = rng.uniform(0.45, 0.62, n // 2)  # half of them on or near the ground
    for j in (0, 1, 3, 4):
        sel = rng.random(n) < 0.35
        bound = np.where(rng.random(n) < 0.5, model.joints[j].limit.lower, model.joints[j].limit.upper)
        st[sel, 13 + j] = (bound + np.sign(bound) * rng.uniform(-0.01, 0.03, n))[sel]
    return st
