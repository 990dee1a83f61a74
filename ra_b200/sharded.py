"""Members of a group on different GPUs: the cross-shard RPC router (SURVEY §8e, config 4).

Placement: member (group g, slot s) lives on shard (g + s) mod N, at local group index g div N.
A record from slot s to slot t of the same group therefore always goes to shard
(shard + t - s) mod N and to the same local row index there, so routing needs no table.

Per step and shard:  raft_step kernels  ->  records for other shards land in dense per-destination
buckets in HBM (ra_engine_set_outbox)  ->  ONE all-to-all of the bucket counts and ONE all-to-all
of the buckets (NCCL over NVLink/NVSwitch, `torch.distributed.all_to_all_single`)  ->
ra_engine_deliver scatters the received records into the mailboxes of the next step.
No other collective exists on the data path.  Everything is enqueued on one CUDA stream per
shard (the engine is switched to torch's current stream), nothing synchronises with the host.

`LocalTransport` runs all shards in one process on one device (plain device copies instead of
NCCL): the single-GPU parity tests use it, so the sharded kernels and ABI are covered without
a second GPU.
"""
from __future__ import annotations

from typing import List, Sequence

import torch

from . import abi
from .engine import Engine

import ctypes as C


def shard_of(group: int, slot: int, n_shards: int) -> int:
    return (group + slot) % n_shards


def local_group(group: int, n_shards: int) -> int:
    return group // n_shards


def global_group(local_q: int, slot: int, shard: int, n_shards: int) -> int:
    return n_shards * local_q + ((shard - slot) % n_shards)


def hashed_group(app_group: int, total_groups: int) -> int:
    """SURVEY 8e asks for `gpu = (hash32(group) + slot) mod N`.  The engine's placement is
    `(group + slot) mod N` on the group ids IT is given, so a hash placement is a relabelling on the host: hand the
    engine `hashed_group(g, G)` -- a bijection of [0, G) (multiplicative hash with a multiplier coprime to G) --
    instead of g.  Neighbouring application groups then land on unrelated shards and rows, and routing still
    needs no table (the inverse is `unhashed_group`)."""
    return (app_group * _multiplier(total_groups)) % total_groups


def unhashed_group(engine_group: int, total_groups: int) -> int:
    return (engine_group * pow(_multiplier(total_groups), -1, total_groups)) % total_groups


def _multiplier(total: int) -> int:
    import math
    a = 2654435761 % total or 1                 # Knuth's multiplicative constant, made coprime to `total`
    while math.gcd(a, total) != 1:
        a += 1
    return a


class Shard:
    """One shard = one engine + its exchange buffers (torch tensors on the engine's device)."""

    def __init__(self, groups_local: int, members: int, n_shards: int, shard: int, device: int = 0,
                 cap: int | None = None, buckets: bool = True, **kw):
        self.n_shards, self.shard, self.dev = n_shards, shard, device
        self.eng = Engine(groups_local, members, device=device, route_on_device=True, n_shards=n_shards,
                          shard=shard, **kw)
        rows = groups_local * members
        # per destination and step: a flood emits ~3.2 records per row (2 AppendEntries per follower -- the entry, then
        # the commit_index update -- and 2 replies each), spread over the destination shards; with N > M two slot
        # offsets can share one destination (N = 8, M = 5: +4 and -4), which then takes 0.8 records per row
        self.cap = cap or max(4096, (rows * 6) // n_shards, rows)
        tdev = torch.device("cuda", device)
        with torch.cuda.device(tdev):
            stream = torch.cuda.current_stream(tdev).cuda_stream
        e = self.eng
        e.call("set_stream", C.c_void_p(stream))
        if buckets:                      # bucket + all-to-all transport; not needed for peer stores
            self.outbox = torch.zeros((n_shards, self.cap, 64), dtype=torch.uint8, device=tdev)
            self.inbox = torch.zeros((n_shards, self.cap, 64), dtype=torch.uint8, device=tdev)
            self.out_cnt = torch.zeros(n_shards, dtype=torch.int32, device=tdev)
            self.in_cnt = torch.zeros(n_shards, dtype=torch.int32, device=tdev)
            e.call("set_outbox", self.outbox.data_ptr(), self.out_cnt.data_ptr(), self.cap)

    def peer_ptrs(self) -> abi.RaPeerPtrs:
        p = abi.RaPeerPtrs()
        self.eng.call("peer_get", C.byref(p))
        return p

    def peer_set(self, shard: int, p: abi.RaPeerPtrs) -> None:
        self.eng.call("peer_set", shard, C.byref(p))

    def ipc_export(self) -> bytes:
        h = abi.RaIpcHandles()
        self.eng.call("ipc_export", C.byref(h))
        return bytes(h)

    def ipc_import(self, shard: int, raw: bytes) -> None:
        self.eng.call("ipc_import", shard, C.byref(abi.RaIpcHandles.from_buffer_copy(raw)))

    def peer_barrier(self) -> None:
        self.eng.call("peer_barrier")

    def deliver(self) -> None:
        self.eng.call("deliver", self.inbox.data_ptr(), self.in_cnt.data_ptr(), self.cap)

    def bootstrap_events(self) -> List[abi.RaEvent]:
        """election_timeout for the slot-0 member of every group that lives here."""
        return [abi.ev_simple(self.eng.row_of(q, 0), abi.EV_ELECTION_TIMEOUT) for q in range(self.eng.n_groups)]

    def global_row(self, local_row: int, total_groups: int) -> int:
        slot, q = divmod(local_row, self.eng.n_groups)
        return slot * total_groups + global_group(q, slot, self.shard, self.n_shards)


class LocalTransport:
    """All shards in this process, same device: the exchange is device-to-device copies."""

    def __init__(self, shards: Sequence[Shard]):
        self.shards = list(shards)

    def exchange(self) -> None:
        for b in self.shards:
            for a in self.shards:
                if a is b:
                    b.in_cnt[a.shard] = 0
                    continue
                b.inbox[a.shard].copy_(a.outbox[b.shard])
                b.in_cnt[a.shard] = a.out_cnt[b.shard]
        for s in self.shards:
            s.deliver()

    def exchange_barrier(self) -> None:
        pass


class NcclTransport:
    """One shard per rank: two all_to_all_single calls per step (counts, then equal-size buckets)."""

    def __init__(self, shard: Shard):
        import torch.distributed as dist
        self.dist = dist
        self.shard = shard
        self.shards = [shard]

    def exchange(self) -> None:
        s = self.shard
        self.dist.all_to_all_single(s.in_cnt, s.out_cnt)
        self.dist.all_to_all_single(s.inbox.view(s.n_shards, -1), s.outbox.view(s.n_shards, -1))
        s.deliver()

    def exchange_barrier(self) -> None:
        pass


class LocalPeerTransport:
    """All shards in this process on one device, peer-store mode: every shard knows the others'
    mailbox buffers and writes into them directly; nothing to exchange between steps."""

    def __init__(self, shards: Sequence[Shard]):
        self.shards = list(shards)
        ptrs = {s.shard: s.peer_ptrs() for s in self.shards}
        for s in self.shards:
            for k, p in ptrs.items():
                if k != s.shard:
                    s.peer_set(k, p)

    def exchange(self) -> None:
        pass

    def exchange_barrier(self) -> None:
        pass


class NvlinkPeerTransport:
    """One shard per rank on one NVLink/NVSwitch domain: mailbox buffers are mapped across
    processes with CUDA IPC at start-up, the step kernels store RPC records straight into the
    destination GPU's HBM.  Lock step between steps: a device-side flag barrier over the same IPC mappings
    (default; ra_engine_flood appends it to every step, so a multi-step flood runs without the host), or with
    RA_PEER_BARRIER=nccl a 1-element NCCL all-reduce on the compute stream."""

    def __init__(self, shard: Shard, device_barrier: bool | None = None):
        import os
        import torch.distributed as dist
        self.dist = dist
        self.shard = shard
        self.shards = [shard]
        # step barrier: a kernel on the engine's stream (flag words in the peers' HBM) or a 1-element all-reduce
        self.device_barrier = (os.environ.get("RA_PEER_BARRIER", "device") == "device") if device_barrier is None \
            else device_barrier
        handles = [None] * dist.get_world_size()
        dist.all_gather_object(handles, shard.ipc_export())
        for k, raw in enumerate(handles):
            if k != shard.shard:
                shard.ipc_import(k, raw)
        self._tok = torch.zeros(1, dtype=torch.int32, device=torch.device("cuda", shard.dev))
        # with the device barrier a multi-step flood needs no host between steps: ra_engine_flood appends it
        self.fused = bool(self.device_barrier)
        shard.eng.call("set_flood_barrier", 1 if self.fused else 0)
        dist.barrier()

    def exchange(self) -> None:
        if self.device_barrier:
            self.shard.peer_barrier()            # lock step without a collective
        else:
            self.dist.all_reduce(self._tok)      # lock step: nobody starts step t+1 before all finished t

    def exchange_barrier(self) -> None:
        torch.cuda.synchronize(self.shard.dev)
        self.dist.barrier()


class ShardedFlood:
    """The flood of ra_engine_flood over sharded members: step, exchange, deliver, repeat."""

    def __init__(self, transport):
        self.t = transport

    def bootstrap(self) -> None:
        # every shard must be reset before any shard steps: with peer stores a step writes into
        # the other shards' mailboxes
        for s in self.t.shards:
            s.eng.reset_empty()
        self.t.exchange_barrier()
        for s in self.t.shards:
            s.eng.step(s.bootstrap_events())
        self.t.exchange()

    def run(self, n_steps: int, cmds: int = 1, permille: int = 0, seed: int = 1, faults=None) -> None:
        if getattr(self.t, "fused", False):                  # every step ends with the device-side barrier
            for s in self.t.shards:
                s.eng.flood(n_steps, cmds, permille, seed, sync=False, faults=faults)
            return
        for _ in range(n_steps):
            for s in self.t.shards:
                s.eng.flood(1, cmds, permille, seed, sync=False, faults=faults)
            self.t.exchange()

    def sync(self) -> None:
        for s in self.t.shards:
            torch.cuda.synchronize(s.dev)

    def counters(self) -> dict:
        tot: dict = {}
        for s in self.t.shards:
            for k, v in s.eng.counters().items():
                tot[k] = tot.get(k, 0) + v
        return tot
