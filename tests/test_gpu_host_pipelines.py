# SPDX-License-Identifier: Apache-2.0
"""Host-buffer steps (upkie_b200_step_host and the *_host calls) at the benchmark's batch size: every pipeline, every
chunking and every kernel family held bit for bit to a device-buffer twin that runs the same kernel, and the rows at
the seams (chunk boundaries, first and last warp, the wrap of a persistent launch's tile walk) held to the fp64 oracle.

step_host cuts the envs into chunks, one step_range launch each with i0 > 0 past the first, or runs one persistent
launch whose blocks walk several tiles. Per-env state is indexed by the env's index on the handle, so an index taken
relative to a launch shows here: in the observations, the flags, the final observations and the checkpoint.

The pipelines (upkie_b200.cu, step_host): 2 (servos default) copies the actions chunk by chunk and each chunk's TILE=1
kernel writes host memory; 1 is one persistent TILE=1 launch (gyropod and pendulum always); 0 stages every chunk through
device buffers on three rotating streams (TILE=1 for compact rows, TILE=0 otherwise)."""
import ctypes as C

import numpy as np
import pytest

from conftest import at_joint_bounds, random_servo_actions, random_states
from test_gpu_sim_parity import TOL_JOINT_RATE_WORST, TOL_POS, TOL_VEL_STEADY, TOL_VEL_WORST, _report
from test_push_randomization_cpu import make_spec
from upkie_b200 import _abi

pytestmark = pytest.mark.gpu

SEED = 23
KNOBS = ("ZERO_COPY", "HOST_CHUNKS", "HOST_SPLIT", "HOST_KERNEL_STREAMS", "HOST_BLOCK", "HOST_BLOCKS_PER_SM")
NEXT_STEP, SAME_STEP = 1, 2


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


# ---- 1. the chunk map ----------------------------------------------------------------------------------------------

def chunk_starts(n, chunks=2, split=(), pipeline=2):
    """The first env of each launch of step_host, then n: a restatement of its chunk boundaries (multiples of 256
    envs). Pipeline 1 is one launch; below 2 x 8192 envs one chunk, below 4 x 8192 two, from there `chunks` equal ones
    or the fractions `split`, the last of which ends at n (a chunk that would end where the previous one did is
    dropped)."""
    if pipeline == 1:
        return [0, n]
    starts = [0]
    if split and n >= 4 * 8192:
        acc = 0.0
        for c, f in enumerate(split):
            if len(starts) - 1 >= 62:
                break
            acc += f
            end = n if c + 1 == len(split) else int(acc * n + 0.5)
            end = min((end + 255) // 256 * 256, n)
            if end > starts[-1]:
                starts.append(end)
        if starts[-1] < n:
            starts.append(n)
        return starts
    want = chunks if n >= 4 * 8192 else (2 if n >= 2 * 8192 else 1)
    per = ((n + want - 1) // want + 255) // 256 * 256
    i0 = 0
    while i0 < n and len(starts) - 1 < 63:
        starts.append(min(i0 + per, n))
        i0 += per
    return starts


def plan(n, knobs, mode="servos"):
    """chunk_starts of a handle created with the developer knobs `knobs` (names without UPKIE_B200_)."""
    pipeline = int(knobs.get("ZERO_COPY", 2))
    if pipeline == 2 and mode != "servos":
        pipeline = 1  # tiny rows: nothing to stream
    split = tuple(v for v in (float(x) for x in str(knobs.get("HOST_SPLIT", "")).split(",") if x) if v > 0)[:8]
    return chunk_starts(n, int(knobs.get("HOST_CHUNKS", 2)), split, pipeline)


def handle(monkeypatch, model, n, cfg, knobs=None):
    """An UpkieSim created with the developer knobs `knobs` set (and every other one unset); they are read when the
    handle is created, and unset again afterwards."""
    from upkie_b200.sim import UpkieSim

    for k in KNOBS:
        monkeypatch.delenv("UPKIE_B200_" + k, raising=False)
    for k, v in (knobs or {}).items():
        monkeypatch.setenv("UPKIE_B200_" + k, str(v))
    try:
        return UpkieSim(n, model=model, config=cfg)
    finally:
        for k in KNOBS:
            monkeypatch.delenv("UPKIE_B200_" + k, raising=False)


def host_step(sim, starts, fn, *args, **kw):
    """One host-buffer step through `fn`; it must have launched one step kernel per chunk of `starts`."""
    l0 = sim.launches
    out = fn(*args, **kw)
    assert sim.launches - l0 == len(starts) - 1, (sim.launches - l0, len(starts) - 1)
    return out


def bits(x):
    """The bits of an array or tensor, as a numpy array (NaN payloads compare too)."""
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    x = np.ascontiguousarray(x)
    return x.view({4: np.uint32, 2: np.uint16, 1: np.uint8, 8: np.uint64}[x.dtype.itemsize])


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def same_checkpoint(a, b):
    """Every entry of two state_dict()s equal, tensors bit for bit: the checkpoint holds every feature's state."""
    sa, sb = a.state_dict(), b.state_dict()
    assert sa.keys() == sb.keys()
    for k in sa:
        if hasattr(sa[k], "detach"):
            assert same_bits(sa[k], sb[k]), k
        else:
            assert sa[k] == sb[k], k
    return sa


def every_chunk(mask, starts):
    """Whether `mask` [n] holds in some env of every chunk."""
    return all(bool(mask[s:e].any()) for s, e in zip(starts[:-1], starts[1:]))


def pinned(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()


# ---- 2. the headline family: every pipeline and chunking -----------------------------------------------------------

def headline(torch, model, n, seed=SEED):
    """The bench's servos workload (bench.py servos_config and bench_env): floor friction U(0.5, 1.2) and inertia
    epsilons U(-0.2, 0.2), four rotating torque-action buffers, next-step auto-reset; the robots start from random
    states, a few percent of them beyond the fall pitch, so that robots fall and reset in every chunk."""
    from bench import servos_config

    rng = np.random.default_rng(seed)
    mu = torch.from_numpy(rng.uniform(0.5, 1.2, n).astype(np.float32)).cuda()
    eps = torch.from_numpy(rng.uniform(-0.2, 0.2, (n, 6)).astype(np.float32)).cuda()
    tau = np.asarray(model.tau_max, np.float32)
    acts = []
    for _ in range(4):
        a = np.zeros((n, 6, 6), np.float32)
        a[:, :, 0] = np.nan
        a[:, :, 5] = tau
        a[:, :, 2] = rng.uniform(-1, 1, (n, 6)) * tau
        acts.append(a)
    state = torch.from_numpy(random_states(n, seed=seed + 1).astype(np.float32)).cuda()

    def setup(s):
        s.set_autoreset(NEXT_STEP, SEED, 0)
        s.reset(seed=SEED)
        s.set_randomization(friction=mu, inertia_eps=eps)
        s.set_state(state)
        torch.cuda.synchronize()  # the host-buffer steps run on the handle's own streams
        return s

    return servos_config(), setup, acts


# (id, n, knobs, chunks of pipelines 0 and 2, pageable action)
CHUNKINGS = [
    ("default", 65536, {}, 2, False),
    ("chunks7_partial_warp", 65496, {"HOST_CHUNKS": 7}, 7, False),
    ("two_chunk_branch", 20000, {}, 2, False),
    ("host_chunks_threshold", 32768, {}, 2, False),
    ("one_chunk", 16383, {}, 1, False),
    ("split_0.9_0.1", 65536, {"HOST_SPLIT": "0.9,0.1"}, 2, False),
    ("split_first_rounds_up", 65536, {"HOST_SPLIT": "0.001,0.999"}, 2, False),
    ("split_above_one", 65536, {"HOST_SPLIT": "0.5,0.6,0.2"}, 2, False),
    ("chunks62", 65536, {"HOST_CHUNKS": 62}, 52, False),
    ("two_kernel_streams", 65536, {"HOST_KERNEL_STREAMS": 2, "HOST_CHUNKS": 4}, 4, False),
    ("chunks5", 65536, {"HOST_CHUNKS": 5}, 5, False),
    ("pageable_action", 65536, {}, 2, True),
]


def test_chunk_map_of_the_cases():
    """The chunk map gives the chunkings the cases are named for."""
    for _, n, knobs, chunks, _ in CHUNKINGS:
        for p in (0, 2):
            assert len(plan(n, dict(knobs, ZERO_COPY=p))) - 1 == chunks
    assert plan(65536, {"HOST_SPLIT": "0.001,0.999"})[:2] == [0, 256]
    assert plan(65536, {"HOST_SPLIT": "0.5,0.6,0.2"}) == [0, 32768, 65536]
    assert plan(65536, {"HOST_SPLIT": "0.9,0.1"}) == [0, 59136, 65536]
    s = plan(65496, {"HOST_CHUNKS": 7})
    assert (s[-1] - s[-2]) % 32 != 0  # the last chunk ends in a partial warp
    assert plan(65536, {"ZERO_COPY": 1}) == [0, 65536] and plan(65536, {}, "gyropod") == [0, 65536]


def _headline_cases():
    for cid, n, knobs, chunks, pageable in CHUNKINGS:
        for p in (2, 0):
            for rows in ("compact", "full"):
                yield pytest.param(n, dict(knobs, ZERO_COPY=p), rows, pageable, id=f"{cid}-p{p}-{rows}")
    for n in (65536, 65496):  # one persistent launch, its blocks walking about four tiles
        for rows in ("compact", "full"):
            yield pytest.param(n, {"ZERO_COPY": 1}, rows, False, id=f"persistent{n}-p1-{rows}")


@pytest.mark.parametrize("n, knobs, rows, pageable", list(_headline_cases()))
def test_headline_host_step_equals_the_device_twin(model, torch, monkeypatch, n, knobs, rows, pageable):
    """The host call against a twin that gets the same inputs on device buffers through the same kernel: compact rows
    (every pipeline) and full rows of pipelines 1 and 2 run TILE=1, as step_servos_compact does; full rows of pipeline 0
    run TILE=0, as step_servos does. Observations and terminated on every tick, then the checkpoint."""
    cfg, setup, acts = headline(torch, model, n)
    starts = plan(n, knobs)
    pipeline = knobs["ZERO_COPY"]
    host = setup(handle(monkeypatch, model, n, cfg, knobs))
    twin = setup(handle(monkeypatch, model, n, cfg))
    src = acts if pageable else [pinned(torch, a) for a in acts]
    dev = [torch.from_numpy(a).cuda() for a in acts]
    fell = np.zeros(n, bool)
    for k in range(30):
        if rows == "compact":
            o, t = host_step(host, starts, host.step_servos_host_compact, src[k % 4])
            ro, rt = twin.step_servos_compact(dev[k % 4])
            assert same_bits(o, ro) and np.array_equal(t, rt.cpu().numpy()), k
        else:
            o, r, t, u = host_step(host, starts, host.step_servos_host, src[k % 4])
            if pipeline == 0:  # TILE=0 on both sides
                ro, _, rt, _ = twin.step_servos(dev[k % 4])
                assert same_bits(o, ro), k
            else:
                ro, rt = twin.step_servos_compact(dev[k % 4])
                assert same_bits(np.ascontiguousarray(o[:, :, :3]), ro), k
                assert (o[:, :, 3] == 42.0).all() and (o[:, :, 4] == 18.0).all(), k
            assert np.array_equal(t, rt.cpu().numpy()) and not r.any() and not u.any(), k
        fell |= t.astype(bool)
    assert every_chunk(fell, starts), "robots fall and reset in every chunk"
    assert torch.equal(host.get_state(), twin.get_state())
    assert torch.equal(host.error_flags(), twin.error_flags())
    same_checkpoint(host, twin)  # episode, tick and pending-reset counters, elapsed counts, randomisation


# ---- 3. every feature family, composed, on chunked launches --------------------------------------------------------

_RR = ([(15.0, 25.0), (0.5, 1.5)] + [(0.0, 0.05)] * 18 + [(-0.1, 0.1)] * 3 + [(0.0, 0.05)] + [(-0.01, 0.01)] * 3
       + [(0.0, 0.01)] + [(-0.2, 0.2)] * 6 + [(0.6, 1.2)])

# what each family's handle turns on (step_family.h): every feature the family carries
FAMILIES = {
    "table": dict(table=1, rr=1),
    "push": dict(table=1, rr=1, push=1),
    "delay": dict(table=1, rr=1, push=1, delay=2),
    "sense": dict(table=1, rr=1, push=1, delay=2, sense=2, history=1, dropout=1),
    "body_delay": dict(body=1, table=1, rr=1, push=1, delay=2),
    "spine": dict(spine=1, body=1, table=1, rr=1),
}


def _reset_randomization():
    s = _abi.UpkieResetRandomization()
    s.columns = (1 << _abi.RR_DIM) - 1
    for k, (lo, hi) in enumerate(_RR):
        s.low[k], s.high[k] = lo, hi
    return s


def family_setup(torch, model, n, family):
    """(config, setup, actions) of the family's handle: same-step auto-reset, robots that fall and reset in every
    chunk, the table, the reset randomisation, pushes, two-tick action and observation delays, the history and the
    servo dropouts as the family carries them."""
    f = FAMILIES[family]
    cfg = _abi.default_sim_config()
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.6
    cfg.max_episode_steps = 12  # time-outs as well as falls: every env resets during the run
    cfg.body_contacts = f.get("body", 0)
    cfg.spine_mode = f.get("spine", 0)
    nb = cfg.nb_substeps
    rng = np.random.default_rng(5)
    table = np.tile(_abi.config_env_params(cfg).astype(np.float32), (n, 1))
    table[:, _abi.EP_MEAS_NOISE:_abi.EP_MEAS_NOISE + 6] = rng.uniform(0.0, 0.5, (n, 6))
    table[:, _abi.EP_IMU_ACC_BIAS:_abi.EP_IMU_ACC_BIAS + 3] = rng.uniform(-0.2, 0.2, (n, 3))
    table[:, _abi.EP_IMU_ACC_NOISE] = rng.uniform(0.0, 0.3, n)
    table = torch.from_numpy(table).cuda()
    state = torch.from_numpy(random_states(n, seed=6).astype(np.float32)).cuda()
    tau = np.asarray(model.tau_max, np.float32)
    acts = []
    for _ in range(4):
        a = np.zeros((n, 6, 6), np.float32)
        a[:, :, 0] = np.nan
        a[:, :, 5] = tau
        a[:, :, 2] = rng.uniform(-1, 1, (n, 6)) * tau
        acts.append(a)

    def setup(s):
        s.set_autoreset(SAME_STEP, SEED, 0)
        if f.get("table"):
            s.set_env_params(table)
        if f.get("rr"):
            s.set_reset_randomization(_reset_randomization())
        if f.get("push"):
            s.set_push_randomization(make_spec(gap=(0, 6), duration=(1, 5),
                                               force=((-30.0, -30.0, -5.0), (30.0, 30.0, 5.0))))
        if f.get("delay"):
            s.set_action_delay(1, f["delay"] * nb, max_ticks=f["delay"])
        if f.get("sense"):
            s.set_observation_delay(0, f["sense"] * nb, max_ticks=f["sense"])
        if f.get("history"):
            s.set_history([_abi.SP_PITCH, _abi.SP_SERVO, _abi.SP_SERVO + 1, _abi.SP_ODOM_POS], 3)
        if f.get("dropout"):
            s.set_servo_dropout(0.2, 0.5)
        s.reset(seed=SEED)
        if not f.get("spine"):
            s.set_state(state)  # a few percent beyond the fall pitch: falls in every chunk from the first tick
        torch.cuda.synchronize()
        return s

    return cfg, setup, acts


FAMILY_CASES = [pytest.param(fam, 65536, {}, id=f"{fam}-default") for fam in FAMILIES] + [
    pytest.param(fam, n, knobs, id=f"{fam}-{kid}")
    for fam in ("sense", "body_delay")
    for kid, n, knobs in (("chunks7", 65496, {"HOST_CHUNKS": 7}), ("kernel_streams2", 65536, {"HOST_KERNEL_STREAMS": 2}))
]
# per-env draw counters of the checkpoint, and the feature that advances each where it acted (a reset drew, a push
# was drawn)
COUNTERS = {"draws": "rr", "push_count": "push", "action_delay_count": "delay", "observation_delay_count": "sense",
            "servo_dropout_count": "dropout"}


@pytest.mark.parametrize("family, n, knobs", FAMILY_CASES)
def test_feature_families_on_chunked_launches(model, torch, monkeypatch, family, n, knobs):
    """step_host(compact=True, final_obs=True, final_state=True) on chunked launches against the same actions through
    upkie_b200_step with compact rows on device buffers (TILE=1, one launch from env 0): observations, terminated,
    truncated, the final-observation rows, final_spine_obs() and the history on every tick, every checkpoint tensor at
    the end. Every feature acts in every chunk during the run."""
    cfg, setup, acts = family_setup(torch, model, n, family)
    starts = plan(n, knobs)
    assert len(starts) - 1 >= 2
    host = setup(handle(monkeypatch, model, n, cfg, knobs))
    twin = setup(handle(monkeypatch, model, n, cfg))
    before = twin.state_dict()
    src = [pinned(torch, a) for a in acts]
    dev = [torch.from_numpy(a).cuda() for a in acts]
    fin = torch.zeros((n, 6, 3), device="cuda")
    reset = np.zeros(n, bool)
    pushed = torch.zeros(n, dtype=torch.bool, device="cuda")
    for k in range(30):
        o, t, r, f = host_step(host, starts, host.step_host, src[k % 4], 36, compact=True, final_obs=True,
                               final_state=True)
        ro, rt, rr = twin.step_servos_compact_truncated(dev[k % 4], final_obs=fin, final_state=True)
        assert same_bits(o, ro) and np.array_equal(t, rt.cpu().numpy()) and np.array_equal(r, rr.cpu().numpy()), k
        assert same_bits(f, fin), k  # the rows of this step's resets and the untouched rows of the earlier ones
        assert same_bits(host.final_spine_obs(), twin.final_spine_obs()), k
        if host.history_spec is not None:
            assert same_bits(host.get_history(), twin.get_history()), k
        if "push" in FAMILIES[family]:
            pushed |= (host.get_push_forces() != 0).any(dim=1)
        reset |= (t | r).astype(bool)
    assert every_chunk(reset, starts)
    if "push" in FAMILIES[family]:
        assert every_chunk(pushed.cpu().numpy(), starts)
    after = same_checkpoint(host, twin)
    for key, feature in COUNTERS.items():
        if feature in FAMILIES[family]:
            moved = (after[key] != before[key].to(after[key].device)).cpu().numpy()
            assert every_chunk(moved, starts), key


# ---- 4. gyropod and pendulum: persistent launches that walk tiles --------------------------------------------------

def fall_and_reset(torch, n, act_dim):
    """The gyropod / pendulum workload of tests/test_gpu_final_info.py: same-step auto-reset, an 80-step limit, full
    ground velocity one way or the other per env, so that robots fall and time out."""
    cfg = _abi.default_sim_config()
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.6
    cfg.max_episode_steps = 80
    rng = np.random.default_rng(5)
    act = (3.0 * np.where(rng.random((n, act_dim)) < 0.5, -1.0, 1.0)).astype(np.float32)

    def setup(s):
        s.set_autoreset(SAME_STEP, 7, 0)
        s.reset(seed=7)
        torch.cuda.synchronize()
        return s

    return cfg, setup, act


def _sync(torch, dst, src):
    """dst takes src's state and counters (episode, tick, pending reset, flags, elapsed): one tick from the same
    start."""
    from upkie_b200._lib import check, lib

    n = src.n
    i32 = dict(dtype=torch.int32, device="cuda")
    ep, tk, fl, el = (torch.empty(n, **i32) for _ in range(4))
    pend = torch.empty(n, dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    check(lib().upkie_b200_get_counters(src._h, p(ep), p(tk), p(pend), p(fl), None))
    check(lib().upkie_b200_get_elapsed(src._h, p(el), None))
    check(lib().upkie_b200_set_counters(dst._h, p(ep), p(tk), p(pend), p(fl), None))
    check(lib().upkie_b200_set_elapsed(dst._h, p(el), None))
    dst.set_state(src.get_state())
    torch.cuda.synchronize()


@pytest.mark.parametrize("act_dim", [2, 1], ids=["gyropod", "pendulum"])
@pytest.mark.parametrize("n", [65536, 65496])
def test_walking_persistent_launches(model, torch, monkeypatch, n, act_dim):
    """step_gyropod_host under pipeline 1 (blocks of 128 envs, one block per SM: about four tiles per block) equals
    the same handle configuration with 8 blocks per SM (one tile each) and with 32-env blocks (about sixteen tiles each)
    bit for bit, and a TILE=0 device step from the same state and counters to the round-off of
    tests/test_gpu_envs.py, with the same flags. Pipeline 0 runs TILE=0 and equals step_gyropod bit for bit."""
    cfg, setup, act = fall_and_reset(torch, n, act_dim)
    mode = "gyropod" if act_dim == 2 else "pendulum"
    walk = setup(handle(monkeypatch, model, n, cfg))
    few = setup(handle(monkeypatch, model, n, cfg, {"HOST_BLOCKS_PER_SM": 8}))
    small = setup(handle(monkeypatch, model, n, cfg, {"HOST_BLOCK": 32}))
    staged = setup(handle(monkeypatch, model, n, cfg, {"ZERO_COPY": 0}))
    dev = setup(handle(monkeypatch, model, n, cfg))
    tol = setup(handle(monkeypatch, model, n, cfg))
    one, chunked = plan(n, {}, mode), plan(n, {"ZERO_COPY": 0}, mode)
    assert len(one) == 2 and len(chunked) - 1 == 2
    host_act = pinned(torch, act)
    dev_act = torch.from_numpy(act).cuda()
    step_dev = tol.step_gyropod if act_dim == 2 else tol.step_pendulum
    pitch = 1 if act_dim == 2 else 0  # column of the observation
    ended = np.zeros(n, bool)
    for k in range(100):
        _sync(torch, tol, walk)
        ro, _, rt, rr = step_dev(dev_act)
        o, _, t, r = [x.copy() for x in host_step(walk, one, walk.step_gyropod_host, host_act)]
        for other in (few, small):
            o2, _, t2, r2 = host_step(other, one, other.step_gyropod_host, host_act)
            assert same_bits(o2, o) and np.array_equal(t2, t) and np.array_equal(r2, r), k
        o3, _, t3, r3 = host_step(staged, chunked, staged.step_gyropod_host, host_act)
        do, _, dt, dr = (dev.step_gyropod if act_dim == 2 else dev.step_pendulum)(dev_act)
        assert same_bits(o3, do) and np.array_equal(t3, dt.cpu().numpy()) and np.array_equal(r3, dr.cpu().numpy()), k
        # TILE=1 against TILE=0, compiled apart: round-off, and the same flags but where the pitch sits within
        # round-off of the fall threshold
        ro, rt, rr = ro.cpu().numpy(), rt.cpu().numpy(), rr.cpu().numpy()
        same = (t == rt) & (r == rr)
        keep = same & ~(t.astype(bool) | r.astype(bool))  # rows of the same episode on both sides
        d = np.abs(ro[keep] - o[keep])
        assert d.max() < 2e-2 and np.median(d) < 1e-5, (k, d.max(), np.median(d))
        if not same.all():
            # the side that did not reset shows the pitch it ended the tick with
            kept = np.where(t[~same].astype(bool), ro[~same, pitch], o[~same, pitch])
            assert (~same).sum() <= 2 and (np.abs(np.abs(kept) - cfg.fall_pitch) < 1e-3).all(), (k, kept)
        ended |= (t | r).astype(bool)
    assert ended.all()
    assert torch.equal(walk.get_state(), few.get_state()) and torch.equal(walk.get_state(), small.get_state())
    assert torch.equal(staged.get_state(), dev.get_state())
    same_checkpoint(walk, few)
    same_checkpoint(staged, dev)


# ---- 5. buffers the Python layer never passes ----------------------------------------------------------------------

def _pinned_view(torch, shape, dtype, offset):
    """A pinned array of `shape` that starts `offset` bytes into its pinned allocation (which is kept alive by the
    returned array's base)."""
    size = int(np.prod(shape)) * np.dtype(dtype).itemsize
    raw = torch.empty(size + 64, dtype=torch.uint8, pin_memory=True).numpy()
    return raw[offset:offset + size].view(dtype).reshape(shape)


def _step_c(sim, act_dim, action, obs, term, trunc, fin, compact):
    from upkie_b200._lib import check, lib

    out = _abi.UpkieStepOutputs(obs.ctypes.data, None, term.ctypes.data, trunc.ctypes.data,
                                None if fin is None else fin.ctypes.data, 1 if compact else 0, 0)
    check(lib().upkie_b200_step_host(sim._h, int(act_dim), action.ctypes.data, C.byref(out)))


OFFSET_CASES = [pytest.param("servos", p, rows, off, id=f"servos-p{p}-{rows}-{off}B")
                for p in (1, 2) for rows in ("compact", "full") for off in (8, 4)] + [
    pytest.param(mode, 1, "full", off, id=f"{mode}-p1-{off}B") for mode in ("gyropod", "pendulum") for off in (8, 4)]


@pytest.mark.parametrize("mode, pipeline, rows, offset", OFFSET_CASES)
def test_pinned_buffers_off_alignment(model, torch, monkeypatch, mode, pipeline, rows, offset):
    """Pinned actions and observation rows that start `offset` bytes into their allocation. 8 bytes: the rows are used
    in place, and the tile kernel stores every warp's rows lane by lane instead of through its tile; 4 bytes: short of
    the kernels' vector accesses, the buffers are staged through the handle's pinned buffers. Both equal the aligned
    pinned call bit for bit."""
    n = 65536
    act_dim = {"servos": 36, "gyropod": 2, "pendulum": 1}[mode]
    obs_dim = {"servos": 18 if rows == "compact" else 30, "gyropod": 6, "pendulum": 4}[mode]
    knobs = {"ZERO_COPY": pipeline}
    starts = plan(n, knobs, mode)
    if mode == "servos":
        cfg, setup, acts = headline(torch, model, n)
    else:
        cfg, setup, act = fall_and_reset(torch, n, act_dim)
        acts = [act] * 4
    ref = setup(handle(monkeypatch, model, n, cfg, knobs))
    odd = setup(handle(monkeypatch, model, n, cfg, knobs))
    action = _pinned_view(torch, (n, act_dim), np.float32, offset)
    obs = _pinned_view(torch, (n, obs_dim), np.float32, offset)
    term = _pinned_view(torch, (n,), np.uint8, 0)
    trunc = _pinned_view(torch, (n,), np.uint8, 0)
    for k in range(6):
        a = acts[k % 4].reshape(n, act_dim)
        ro, rt, rr, _ = host_step(ref, starts, ref.step_host, pinned(torch, a), act_dim, compact=rows == "compact")
        action[:] = a
        host_step(odd, starts, _step_c, odd, act_dim, action, obs, term, trunc, None, rows == "compact")
        assert same_bits(obs, ro.reshape(n, obs_dim)) and np.array_equal(term, rt) and np.array_equal(trunc, rr), k
    same_checkpoint(ref, odd)


@pytest.mark.parametrize("pipeline", [2, 1, 0])
def test_pageable_outputs_and_final_obs(model, torch, monkeypatch, pipeline):
    """Pageable observation rows, flags and final observations (staged through the handle's pinned buffers, the final
    rows through a pinned copy of the caller's) equal the pinned call bit for bit; the final rows of the envs that did
    not reset keep the caller's sentinel."""
    n = 65536
    cfg, setup, acts = family_setup(torch, model, n, "sense")
    knobs = {"ZERO_COPY": pipeline}
    starts = plan(n, knobs)
    ref = setup(handle(monkeypatch, model, n, cfg, knobs))
    pag = setup(handle(monkeypatch, model, n, cfg, knobs))
    obs = np.zeros((n, 6, 3), np.float32)
    term = np.zeros(n, np.uint8)
    trunc = np.zeros(n, np.uint8)
    fin = np.empty((n, 6, 3), np.float32)
    resets = 0
    for k in range(14):
        ro, rt, rr, rf = host_step(ref, starts, ref.step_host, pinned(torch, acts[k % 4]), 36, compact=True,
                                   final_obs=True)
        fin.fill(-12345.0)
        host_step(pag, starts, _step_c, pag, 36, acts[k % 4], obs, term, trunc, fin, True)
        assert same_bits(obs, ro) and np.array_equal(term, rt) and np.array_equal(trunc, rr), k
        ended = (rt | rr).astype(bool)
        assert same_bits(fin[ended], rf[ended]) and (fin[~ended] == -12345.0).all(), k
        resets += int(ended.sum())
    assert resets > 0
    same_checkpoint(ref, pag)


# ---- 6. anchors to the fp64 oracle at the seams --------------------------------------------------------------------

def seam_rows(n, starts):
    """32 envs on each side of every chunk boundary, the first warp and the last (partial) warp."""
    rows = set(range(0, 32)) | set(range((n - 1) // 32 * 32, n))
    for b in starts[1:-1]:
        rows |= set(range(b - 32, b + 32))
    return np.array(sorted(rows))


def _anchor_states(model, n):
    """random_states, every other warp at_joint_bounds (robots on a hip or knee bound: the ten-row solver)."""
    st = random_states(n, seed=3).astype(np.float32)
    jb = at_joint_bounds(model, n, seed=4)
    odd = (np.arange(n) // 32) % 2 == 1
    st[odd] = jb[odd]
    return st


def _hold_to_oracle(name, oracle_lib, model, cfg, gs, rows, st, step):
    """One tick of the oracle on `rows` from `st`; the state rows `gs` of the GPU against it, with the one-tick
    tolerances of tests/test_gpu_sim_parity.py. Returns the oracle's outputs."""
    osim = oracle_lib.OracleSim(model, cfg, len(rows), threads=8)
    osim.set_state(st[rows].astype(np.float64))
    out = step(osim)
    o = osim.get_state()
    g = gs.astype(np.float64)
    dpos, dq = np.abs(g[:, :7] - o[:, :7]).max(), np.abs(g[:, 13:19] - o[:, 13:19]).max()
    dvel, dqd = np.abs(g[:, 7:13] - o[:, 7:13]), np.abs(g[:, 19:25] - o[:, 19:25])
    _report(name, base_twist_worst=dvel.max(), joint_rate_worst=dqd.max(), position_worst=dpos, joint_angle_worst=dq,
            rows=len(rows))
    assert dpos < TOL_POS and dq < 2e-4, (dpos, dq)
    assert np.median(dvel.max(axis=1)) < TOL_VEL_STEADY and np.median(dqd.max(axis=1)) < TOL_VEL_STEADY
    assert dvel.max() < TOL_VEL_WORST and dqd.max() < TOL_JOINT_RATE_WORST, (dvel.max(), dqd.max())
    return out


ANCHOR_CASES = [pytest.param(n, dict(knobs, ZERO_COPY=p), rows, id=f"{cid}-p{p}-{rows}")
                for cid, n, knobs, chunks, pageable in CHUNKINGS if not pageable
                for p, rows in ((2, "compact"), (0, "compact"), (0, "full"))]


@pytest.mark.parametrize("n, knobs, rows", ANCHOR_CASES)
def test_seam_rows_match_the_oracle(model, oracle_lib, torch, monkeypatch, n, knobs, rows):
    """One host step from random states (auto-reset disabled): the rows at the chunk seams against the fp64 oracle."""
    cfg = _abi.default_sim_config()
    starts = plan(n, knobs)
    sim = handle(monkeypatch, model, n, cfg, knobs)
    st = _anchor_states(model, n)
    act = random_servo_actions(n, model, seed=4).astype(np.float32)
    sim.set_state(torch.from_numpy(st).cuda())
    torch.cuda.synchronize()
    if rows == "compact":
        obs, term = host_step(sim, starts, sim.step_servos_host_compact, pinned(torch, act))
    else:
        obs, _, term, _ = host_step(sim, starts, sim.step_servos_host, pinned(torch, act))
    sel = seam_rows(n, starts)
    gs = sim.get_state().cpu().numpy()[sel]
    key = "-".join(f"{k}={v}" for k, v in sorted(knobs.items()))
    oobs, _, oterm, _ = _hold_to_oracle(f"host_seams_{n}_{key}_{rows}", oracle_lib, model, cfg, gs, sel, st,
                                        lambda o: o.step_servos(act[sel].astype(np.float64)))
    g = obs[sel].astype(np.float64)
    assert np.abs(g[:, :, 0] - oobs[:, :, 0]).max() < 2e-4  # the rows the host got are these envs' rows
    assert np.median(np.abs(g[:, :, 2] - oobs[:, :, 2])) < 1e-3
    assert np.array_equal(term[sel], oterm)


@pytest.mark.parametrize("act_dim", [2, 1], ids=["gyropod", "pendulum"])
def test_tile_walk_wrap_matches_the_oracle(model, oracle_lib, torch, monkeypatch, act_dim):
    """The persistent launch's blocks walk tiles with a stride of grid x host_block envs: the envs on each side of
    every wrap, and the last partial warp, after one gyropod / pendulum host step, against the fp64 oracle."""
    n = 65496
    cfg = _abi.default_sim_config()
    mode = "gyropod" if act_dim == 2 else "pendulum"
    sim = handle(monkeypatch, model, n, cfg)
    st = _anchor_states(model, n)
    act = np.random.default_rng(43).uniform(-1.5, 1.5, (n, act_dim)).astype(np.float32)
    sim.set_state(torch.from_numpy(st).cuda())
    torch.cuda.synchronize()
    obs, _, term, _ = host_step(sim, plan(n, {}, mode), sim.step_gyropod_host, pinned(torch, act))
    stride = torch.cuda.get_device_properties(0).multi_processor_count * 128  # grid x host_block
    sel = seam_rows(n, list(range(0, n, stride)) + [n])
    assert len(sel) > 64 * 3
    gs = sim.get_state().cpu().numpy()[sel]
    oobs, _, oterm, _ = _hold_to_oracle(f"host_walk_wrap_{mode}", oracle_lib, model, cfg, gs, sel, st,
                                        lambda o: o.step_gyropod(act[sel].astype(np.float64), act_dim))
    cols = [0, 1, 2, 5] if act_dim == 2 else [0, 1]
    assert np.abs(obs[sel][:, cols].astype(np.float64) - oobs[:, cols]).max() < 2e-4
    assert np.array_equal(term[sel], oterm)


# ---- 7. the benchmark's own call -----------------------------------------------------------------------------------

@pytest.mark.parametrize("autoreset", ["next_step", "same_step"])
def test_bench_vector_env_call(model, torch, autoreset):
    """B200VectorEnv(65536, "servos", copy=False).step(pinned numpy action), bench.py's end-to-end call, against a twin
    whose sim.step_servos_compact (same-step mode: step_servos_compact_truncated with the final rows) gets the same
    actions as tensors."""
    from bench import servos_config
    from upkie_b200.envs import B200VectorEnv

    n = 65536
    limit = 12 if autoreset == "same_step" else 0
    envs = [B200VectorEnv(n, "servos", config=servos_config(), autoreset_mode=autoreset, model=model, copy=False,
                          max_episode_steps=limit) for _ in range(2)]
    gen = torch.Generator(device="cuda")
    gen.manual_seed(2025)
    mu = torch.empty(n, device="cuda").uniform_(0.5, 1.2, generator=gen)
    eps = torch.empty((n, 6), device="cuda").uniform_(-0.2, 0.2, generator=gen)
    tau = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
    acts = []
    for _ in range(4):
        a = torch.zeros((n, 6, 6), device="cuda")
        a[:, :, 0] = float("nan")
        a[:, :, 5] = tau
        a[:, :, 2] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * tau
        acts.append(a.contiguous())
    host_acts = [a.cpu().pin_memory().numpy() for a in acts]
    for e in envs:
        e.sim.set_randomization(friction=mu, inertia_eps=eps)
        e.sim.set_autoreset(NEXT_STEP if autoreset == "next_step" else SAME_STEP, 2025, 0)
        e.sim.reset(seed=2025)
    env, twin = envs
    torch.cuda.synchronize()
    fin = torch.zeros((n, 6, 3), device="cuda")
    finals = 0
    for k in range(30):
        obs, rew, te, tr, info = env.step(host_acts[k % 4])
        if autoreset == "next_step":
            ro, rt = twin.sim.step_servos_compact(acts[k % 4])
            rr = torch.zeros_like(rt)
        else:
            ro, rt, rr = twin.sim.step_servos_compact_truncated(acts[k % 4], final_obs=fin, final_state=True)
        got = np.stack([np.concatenate([obs[j][key] for key in ("position", "velocity", "torque")], axis=1)
                        for j in _abi.JOINT_NAMES], axis=1)
        assert same_bits(got, ro), k
        assert all((obs[j]["temperature"] == 42.0).all() and (obs[j]["voltage"] == 18.0).all() for j in _abi.JOINT_NAMES)
        rt, rr = rt.cpu().numpy().astype(bool), rr.cpu().numpy().astype(bool)
        assert np.array_equal(te, rt) and np.array_equal(tr, rr) and not rew.any(), k
        ended = rt | rr
        assert ("final_obs" in info) == (autoreset == "same_step" and bool(ended.any())), k
        if "final_obs" in info:
            assert np.array_equal(info["_final_obs"], ended) and np.array_equal(info["_final_info"], ended)
            f = np.stack([np.concatenate([info["final_obs"][j][key] for key in ("position", "velocity", "torque")],
                                         axis=1) for j in _abi.JOINT_NAMES], axis=1)
            assert same_bits(f[ended], fin.cpu().numpy()[ended]), k
            finals += 1
    assert autoreset == "next_step" or finals > 0
    assert torch.equal(env.sim.get_state(), twin.sim.get_state())
    for e in envs:
        e.close()
