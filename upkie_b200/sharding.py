# SPDX-License-Identifier: Apache-2.0
"""Env-index sharding across GPUs and the rollout all-gather (SURVEY.md 8e).

Every env is independent, so the path shards by env index with no collective
inside ``step()``: rank ``r`` of ``G`` owns the contiguous block
``shard_range(N, r, G)`` and passes its ``offset`` as ``env_offset`` so that the
device RNG is keyed on the *global* env index (results do not depend on G).
The only exchange is one all-gather of the trajectory buffer per rollout, over
NCCL (NVLink/NVSwitch) on GPUs or gloo in the CPU tests.
"""

from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist


def shard_range(num_envs: int, rank: int, world_size: int) -> Tuple[int, int]:
    """``(offset, count)`` of the contiguous env block owned by ``rank``.
    The first ``num_envs % world_size`` ranks take one extra env."""
    if not (0 <= rank < world_size):
        raise ValueError(f"rank {rank} outside world of size {world_size}")
    base, rem = divmod(int(num_envs), int(world_size))
    count = base + (1 if rank < rem else 0)
    offset = rank * base + min(rank, rem)
    return offset, count


class RolloutBuffer:
    """One rollout of this rank: ``obs[T, n, obs_dim]`` f32, ``reward[T, n]`` f32,
    ``terminated[T, n]`` u8, ``truncated[T, n]`` u8, carved out of ONE byte buffer
    (``4 * obs_dim + 6`` bytes per env and step: 126 B for UpkieServos).

    ``slot(t)`` returns the four views of time step ``t``; handing them to
    ``UpkieSim.step_*`` as output tensors makes the step kernel write the rollout
    in place (no copy kernels). ``gather()`` all-gathers the byte buffer once and
    returns the rollout of ALL envs ordered by global env index, identical on
    every rank.
    """

    def __init__(self, horizon: int, n_local: int, obs_dim: int, device, group: Optional[dist.ProcessGroup] = None,
                 compact: bool = False):
        self.T, self.n, self.obs_dim = int(horizon), int(n_local), int(obs_dim)
        # compact records carry observation rows and `terminated` only: reward (0.0) and truncated (False) are
        # constants of the reference (upkie_env.py:197,230) and stay out of the gather
        self.compact = bool(compact)
        self.rec = 4 * self.obs_dim + (1 if self.compact else 6)
        self.group = group
        self.device = torch.device(device)
        T, n, d = self.T, self.n, self.obs_dim
        self._sizes = [T * n * d * 4, 0 if self.compact else T * n * 4, T * n, 0 if self.compact else T * n]
        total = sum(self._sizes)
        self.nbytes = (total + 15) // 16 * 16
        self.raw = torch.zeros(self.nbytes, dtype=torch.uint8, device=self.device)
        self.obs, self.reward, self.terminated, self.truncated = self._views(self.raw, n)

    def _views(self, raw: torch.Tensor, n: int):
        T, d = self.T, self.obs_dim
        o0 = 0
        o1 = o0 + T * n * d * 4
        o2 = o1 + T * n * 4
        o3 = o2 + T * n
        obs = raw[o0:o1].view(torch.float32).view(T, n, d)
        if self.compact:
            return obs, None, raw[o1:o1 + T * n].view(T, n), None
        rew = raw[o1:o2].view(torch.float32).view(T, n)
        term = raw[o2:o3].view(T, n)
        trunc = raw[o3:o3 + T * n].view(T, n)
        return obs, rew, term, trunc

    def slot(self, t: int):
        """Output tensors of time step ``t`` (modulo the horizon)."""
        k = t % self.T
        if self.compact:
            return self.obs[k], None, self.terminated[k], None
        return self.obs[k], self.reward[k], self.terminated[k], self.truncated[k]

    def record(self, t: int, obs: torch.Tensor, reward: torch.Tensor, terminated: torch.Tensor, truncated: torch.Tensor):
        """Copy-in variant of ``slot`` for producers that own their output tensors."""
        o, r, te, tr = self.slot(t)
        o.copy_(obs.reshape(self.n, self.obs_dim))
        te.copy_(terminated)
        if not self.compact:
            r.copy_(reward)
            tr.copy_(truncated)

    def gather(self) -> Dict[str, torch.Tensor]:
        """``{"obs": [T, N, obs_dim], "reward": [T, N], "terminated": [T, N], "truncated": [T, N]}``
        over all ranks (``N = world_size * n``; equal shards)."""
        if not dist.is_initialized() or dist.get_world_size(self.group) == 1:
            if self.compact:
                return {"obs": self.obs, "terminated": self.terminated}
            return {"obs": self.obs, "reward": self.reward, "terminated": self.terminated, "truncated": self.truncated}
        world = dist.get_world_size(self.group)
        out = torch.empty(world * self.nbytes, dtype=torch.uint8, device=self.device)
        dist.all_gather_into_tensor(out, self.raw, group=self.group)
        parts = [self._views(out[r * self.nbytes:(r + 1) * self.nbytes], self.n) for r in range(world)]
        if self.compact:
            return {"obs": torch.cat([p[0] for p in parts], dim=1), "terminated": torch.cat([p[2] for p in parts], dim=1)}
        return {
            "obs": torch.cat([p[0] for p in parts], dim=1),
            "reward": torch.cat([p[1] for p in parts], dim=1),
            "terminated": torch.cat([p[2] for p in parts], dim=1),
            "truncated": torch.cat([p[3] for p in parts], dim=1),
        }

    def gather_raw(self, async_op: bool = False):
        """The all-gather alone (``[world, nbytes]`` bytes, rank-major), without re-assembly.

        With ``async_op=True`` returns ``(tensor, work)``: the collective runs on the
        communication stream while the next rollout (in another buffer) is simulated;
        call ``work.wait()`` before touching ``tensor`` or re-using this buffer's slots."""
        if not dist.is_initialized() or dist.get_world_size(self.group) == 1:
            out = self.raw.view(1, -1)
            return (out, None) if async_op else out
        world = dist.get_world_size(self.group)
        if getattr(self, "_gathered", None) is None:
            self._gathered = torch.empty(world * self.nbytes, dtype=torch.uint8, device=self.device)
        work = dist.all_gather_into_tensor(self._gathered, self.raw, group=self.group, async_op=async_op)
        out = self._gathered.view(world, self.nbytes)
        return (out, work) if async_op else out


class PeerRolloutBuffer(RolloutBuffer):
    """Rollout buffer in symmetric memory (one node, NVLink / NVSwitch): every rank holds the FULL
    ``[world, nbytes]`` gathered buffer; its step kernels write the rank's own slot in place, and ``push()``
    copies that slot into the same slot of every peer's buffer with the copy engines (peer-to-peer
    ``cudaMemcpyAsync`` over NVLink) on a side stream.

    Why not NCCL's all-gather here: the step kernel occupies every SM (255 registers x 224 threads leave no
    room for another block), so a collective implemented as SM kernels only advances when simulation blocks
    retire and slows the simulation it is meant to overlap. Copy
    engines need no SM.
    """

    def __init__(self, horizon: int, n_local: int, obs_dim: int, device, group: Optional[dist.ProcessGroup] = None,
                 compact: bool = False):
        import torch.distributed._symmetric_memory as symm_mem

        self.T, self.n, self.obs_dim = int(horizon), int(n_local), int(obs_dim)
        self.compact = bool(compact)
        self.rec = 4 * self.obs_dim + (1 if self.compact else 6)
        self.group = group if group is not None else dist.group.WORLD
        self.device = torch.device(device)
        T, n, d = self.T, self.n, self.obs_dim
        self._sizes = [T * n * d * 4, 0 if self.compact else T * n * 4, T * n, 0 if self.compact else T * n]
        self.nbytes = (sum(self._sizes) + 255) // 256 * 256
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self.all = symm_mem.empty(self.world * self.nbytes, dtype=torch.uint8, device=self.device)
        self.all.zero_()
        self._hdl = symm_mem.rendezvous(self.all, self.group)
        self.raw = self.all[self.rank * self.nbytes:(self.rank + 1) * self.nbytes]
        self.obs, self.reward, self.terminated, self.truncated = self._views(self.raw, n)
        self._peers = [
            self._hdl.get_buffer(p, (self.world * self.nbytes,), torch.uint8, 0)[self.rank * self.nbytes:(self.rank + 1) * self.nbytes]
            for p in range(self.world)
        ]
        # several side streams so that the pushes to different peers run on different copy engines at once
        self._copy_streams = [torch.cuda.Stream(device=self.device) for _ in range(min(4, max(1, self.world - 1)))]
        self._done = None

    def push(self) -> "torch.cuda.Event":
        """Start pushing this rank's slot to every peer (asynchronous, side streams). Destinations are visited in
        ring order (rank + 1, rank + 2, ...): at any moment every GPU receives from one sender instead of all
        ranks converging on peer 0, then peer 1, ... The returned event fires when this rank's copies are done AND
        every peer's copies into this rank's buffer are done (cross-rank barrier on a side stream): after it,
        ``gathered()`` is complete and the slot may be rewritten."""
        cur = torch.cuda.current_stream(self.device)
        for s_ in self._copy_streams:
            s_.wait_stream(cur)
        for i in range(1, self.world):
            p = (self.rank + i) % self.world
            with torch.cuda.stream(self._copy_streams[(i - 1) % len(self._copy_streams)]):
                self._peers[p].copy_(self.raw, non_blocking=True)
        main = self._copy_streams[0]
        for s_ in self._copy_streams[1:]:
            main.wait_stream(s_)
        with torch.cuda.stream(main):
            self._hdl.barrier(channel=0)
            ev = torch.cuda.Event()
            ev.record(main)
        self._done = ev
        return ev

    # ---- in-kernel transports: NVSwitch multicast stores, or stores into every peer's buffer ------------------
    @property
    def multicast_supported(self) -> bool:
        return bool(getattr(self._hdl, "has_multicast_support", False)) and int(self._hdl.multicast_ptr) != 0

    def multicast_slot(self, t: int):
        """``(obs_ptr, terminated_ptr)``: multicast addresses of this rank's slot at time step ``t`` (compact
        records only). Stores to them (``UpkieSim.step_servos_multicast``) land in EVERY rank's buffer."""
        if not self.compact:
            raise ValueError("multicast slots carry compact records")
        k = t % self.T
        base = int(self._hdl.multicast_ptr) + self.rank * self.nbytes
        obs_off = k * self.n * self.obs_dim * 4
        term_off = self.T * self.n * self.obs_dim * 4 + k * self.n
        return base + obs_off, base + term_off

    def peer_slots(self, t: int):
        """``(obs_ptrs, terminated_ptrs)``: device addresses of this rank's slot at time step ``t`` in EVERY rank's
        buffer (own buffer included), for ``UpkieSim.step_servos_peers`` (compact records only)."""
        if not self.compact:
            raise ValueError("peer slots carry compact records")
        k = t % self.T
        obs_off = k * self.n * self.obs_dim * 4
        term_off = self.T * self.n * self.obs_dim * 4 + k * self.n
        bases = [p_.data_ptr() for p_ in self._peers]
        return [b + obs_off for b in bases], [b + term_off for b in bases]

    def local_slot(self, t: int):
        """``(obs_ptr, terminated_ptr)``: LOCAL device addresses of this rank's slot at time step ``t`` (the deferred
        transport writes a step's rows there and sends them with a later launch)."""
        if not self.compact:
            raise ValueError("deferred slots carry compact records")
        k = t % self.T
        base = self.raw.data_ptr()
        return base + k * self.n * self.obs_dim * 4, base + self.T * self.n * self.obs_dim * 4 + k * self.n

    def push_descriptor(self, t: int, multicast: bool):
        """``_abi.UpkiePush`` that sends this rank's slot of step ``t`` to every rank: to the multicast address of the
        slot, or (``multicast=False``) into every PEER's buffer (this rank's own copy is already in place)."""
        from . import _abi

        d = _abi.UpkiePush()
        d.src_obs, d.src_terminated = self.local_slot(t)
        if multicast:
            d.mc_obs, d.mc_terminated = self.multicast_slot(t)
            d.n_peers = 0
        else:
            obs_ptrs, term_ptrs = self.peer_slots(t)
            k = 0
            for p in range(self.world):
                if p == self.rank:
                    continue
                d.peer_obs[k], d.peer_terminated[k] = obs_ptrs[p], term_ptrs[p]
                k += 1
            d.n_peers = k
        return d

    def publish(self) -> None:
        """After the last multicast step of a rollout: cross-rank barrier on the current stream; once it has
        passed, ``gathered()`` holds every rank's records on every rank."""
        self._hdl.barrier(channel=1)

    def wait(self) -> None:
        """Make the current stream wait for the last ``push()``."""
        if self._done is not None:
            torch.cuda.current_stream(self.device).wait_event(self._done)
            self._done = None

    def gathered(self) -> torch.Tensor:
        """``[world, nbytes]`` bytes, rank-major (same layout as ``RolloutBuffer.gather_raw``)."""
        return self.all.view(self.world, self.nbytes)
