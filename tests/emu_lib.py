"""TEST INFRASTRUCTURE: loader for the host emulation of the engine's device logic
(tests/emu/libra_emu.so = ra_b200/csrc/raft_step.cuh + raft_row.cuh compiled by g++ through
tests/emu/cuda_shim.h).  Lets the CPU test tier diff the source the GPU runs against the oracle;
it is never imported by the product package and is not a fallback for it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from ra_b200 import abi

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DIR = os.path.join(_ROOT, "tests", "emu")
_SO = os.path.join(_DIR, "libra_emu.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        srcs = [os.path.join(_DIR, "ra_emu.cpp"), os.path.join(_DIR, "step_row.inc"), os.path.join(_DIR, "cuda_shim.h"),
                *[os.path.join(_ROOT, "ra_b200", "csrc", f) for f in
                  ("raft_step.cuh", "raft_common.cuh", "raft_logic.cuh", "raft_row_logic.cuh", "raft_row.cuh")],
                os.path.join(_ROOT, "include", "ra_engine.h")]
        if (not os.path.exists(_SO)) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["make", "-C", _DIR], stdout=subprocess.DEVNULL)
        _lib = C.CDLL(_SO)
        _lib.ra_emu_flood.restype = C.c_int
        _lib.ra_emu_flood.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64]
        _lib.ra_emu_stall_histogram.restype = C.c_int
        _lib.ra_emu_stall_histogram.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    return _lib


class Emu(abi.Backend):
    name = "emu"

    def __init__(self, n_groups: int, n_members: int, **kw):
        super().__init__(lib(), "ra_emu", n_groups, n_members, **kw)

    def flood(self, n_steps: int, cmds_per_step: int = 1, election_permille: int = 0, seed: int = 1, faults=None,
              **_kw) -> None:
        if faults is None:
            self._check(lib().ra_emu_flood(self._h, n_steps, cmds_per_step, election_permille, seed), "flood")
            return
        f = lib().ra_emu_flood_faults
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.POINTER(abi.RaFloodFaults)]
        ff = abi.RaFloodFaults(*faults)
        self._check(f(self._h, n_steps, cmds_per_step, election_permille, seed, C.byref(ff)), "flood_faults")

    @staticmethod
    def narrow_stats(reset: bool = True) -> dict:
        """Process-wide: rows stepped by the 32-bit pass of the hot kernel's logic, records it refused (a field
        >= 2^30), rows it left to the 64-bit general path because their sticky `wide` byte is set."""
        arr = (C.c_ulonglong * 3)()
        lib().ra_emu_narrow_stats(arr, 1 if reset else 0)
        return dict(rows_narrow=arr[0], records_refused=arr[1], rows_wide=arr[2])

    @staticmethod
    def stall_stats(reset: bool = True) -> dict:
        """Process-wide: stall contexts the hot kernel's logic handed to the general path, and those of them that
        carried per-peer "not short" bits (StallCtx::wk_hi) across the stall."""
        arr = (C.c_ulonglong * 2)()
        lib().ra_emu_stall_stats(arr, 1 if reset else 0)
        return dict(stalls=arr[0], stalls_wk_hi=arr[1])

    @staticmethod
    def underfetched(reset: bool = True) -> int:
        """Process-wide: records the hot kernel's logic decoded although the size flags of their tile did not let the
        kernel fetch all of their chunks (0 while every writer sets its flags)."""
        arr = (C.c_ulonglong * 1)()
        lib().ra_emu_fetch_stats(arr, 1 if reset else 0)
        return int(arr[0])

    @staticmethod
    def set_fetch_poison(pattern: int) -> None:
        """Process-wide: which poison pattern stands for the bytes the hot kernel did not fetch (0 or 1)."""
        lib().ra_emu_set_fetch_poison(pattern)

    def stall_histogram(self) -> dict:
        arr = (C.c_uint64 * 128)()
        self._check(lib().ra_emu_stall_histogram(self._h, arr), "stall_histogram")
        return {(i // 16, i % 16): int(v) for i, v in enumerate(arr) if v}


class EmuHostFlood:
    """ra_hostsim (ra_b200/csrc/host_flood.cu, the host-side ABI caller of the e2e benchmark) compiled
    into the emulation library and driving an Emu through its step() entry point."""

    def __init__(self, emu: Emu):
        self.e = emu
        l = lib()
        l.ra_hostsim_create.restype = C.c_int
        l.ra_hostsim_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        l.ra_hostsim_run.restype = C.c_int
        l.ra_hostsim_run.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_int]
        l.ra_hostsim_stats.restype = C.c_int
        l.ra_hostsim_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                       C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
        l.ra_hostsim_destroy.restype = None
        l.ra_hostsim_destroy.argtypes = [C.c_void_p]
        self._h = C.c_void_p()
        emu._check(l.ra_hostsim_create(emu._h, C.byref(self._h)), "hostsim_create")

    def run(self, n_steps: int, cmds: int = 1, permille: int = 0, seed: int = 1, bootstrap: bool = False) -> dict:
        self.e._check(lib().ra_hostsim_run(self._h, n_steps, cmds, permille, seed, 1 if bootstrap else 0), "hostsim_run")
        h2d, d2h, calls, sec = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_double(0)
        lib().ra_hostsim_stats(self._h, C.byref(h2d), C.byref(d2h), C.byref(sec), C.byref(calls))
        return dict(h2d_bytes=int(h2d.value), d2h_bytes=int(d2h.value), engine_calls=int(calls.value))

    def close(self) -> None:
        if self._h:
            lib().ra_hostsim_destroy(self._h)
            self._h = C.c_void_p()


class PeerPtrs(C.Structure):
    """ra_peer_ptrs (include/ra_engine.h)"""
    _fields_ = [("mbox", C.c_void_p * 2), ("mbox_cnt", C.c_void_p * 2)]


class EmuShards:
    """N emulated shards in this process: the CPU twin of ra_b200.sharded.Shard + LocalTransport + ShardedFlood
    (member (g, s) on shard (g + s) mod N), or with peer=True of Shard + LocalPeerTransport: every shard stores
    into the others' mailboxes (ra_emu_peer_set) and exchange() has nothing to do."""

    def __init__(self, n_shards: int, groups_local: int, members: int, cap: int = 4096, peer: bool = False, **kw):
        l = lib()
        l.ra_emu_set_outbox.restype = C.c_int
        l.ra_emu_set_outbox.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
        l.ra_emu_deliver.restype = C.c_int
        l.ra_emu_deliver.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
        l.ra_emu_peer_get.restype = C.c_int
        l.ra_emu_peer_get.argtypes = [C.c_void_p, C.POINTER(PeerPtrs)]
        l.ra_emu_peer_set.restype = C.c_int
        l.ra_emu_peer_set.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(PeerPtrs)]
        self.n, self.gl, self.m, self.cap, self.peer = n_shards, groups_local, members, cap, peer
        self.shards = [Emu(groups_local, members, route_on_device=True, n_shards=n_shards, shard=k, **kw)
                       for k in range(n_shards)]
        if peer:
            ptrs = []
            for s in self.shards:
                p = PeerPtrs()
                s._check(l.ra_emu_peer_get(s._h, C.byref(p)), "peer_get")
                ptrs.append(p)
            for k, s in enumerate(self.shards):
                for j, p in enumerate(ptrs):
                    if j != k:
                        s._check(l.ra_emu_peer_set(s._h, j, C.byref(p)), "peer_set")
            return
        self.outbox = [(abi.RaEvent * (n_shards * cap))() for _ in range(n_shards)]
        self.inbox = [(abi.RaEvent * (n_shards * cap))() for _ in range(n_shards)]
        self.out_cnt = [(C.c_uint32 * n_shards)() for _ in range(n_shards)]
        self.in_cnt = [(C.c_uint32 * n_shards)() for _ in range(n_shards)]
        for k, s in enumerate(self.shards):
            s._check(l.ra_emu_set_outbox(s._h, self.outbox[k], self.out_cnt[k], cap), "set_outbox")

    def exchange(self) -> None:
        if self.peer:                                  # the stores landed during the step
            return
        sz = C.sizeof(abi.RaEvent)
        for b in range(self.n):
            for a in range(self.n):
                if a == b:
                    self.in_cnt[b][a] = 0
                    continue
                cnt = min(int(self.out_cnt[a][b]), self.cap)
                C.memmove(C.byref(self.inbox[b], a * self.cap * sz), C.byref(self.outbox[a], b * self.cap * sz), cnt * sz)
                self.in_cnt[b][a] = self.out_cnt[a][b]
        for b, s in enumerate(self.shards):
            s._check(lib().ra_emu_deliver(s._h, self.inbox[b], self.in_cnt[b], self.cap), "deliver")

    def bootstrap(self) -> None:
        for s in self.shards:
            s.reset_empty()
        for s in self.shards:
            s.step([abi.ev_simple(s.row_of(q, 0), abi.EV_ELECTION_TIMEOUT) for q in range(self.gl)])
        self.exchange()

    def run(self, n_steps: int, cmds: int = 1, permille: int = 0, seed: int = 1) -> None:
        for _ in range(n_steps):
            for s in self.shards:
                s.flood(1, cmds, permille, seed)
            self.exchange()

    def global_row(self, shard: int, local_row: int) -> int:
        slot, q = divmod(local_row, self.gl)
        return slot * (self.n * self.gl) + self.n * q + ((shard - slot) % self.n)

    def counters(self) -> dict:
        tot: dict = {}
        for s in self.shards:
            for k, v in s.counters().items():
                tot[k] = tot.get(k, 0) + v
        return tot
