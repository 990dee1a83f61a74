"""TEST INFRASTRUCTURE: loader for the host emulation of the engine's device logic
(tests/emu/libra_emu.so = ra_b200/csrc/raft_step.cuh + raft_row.cuh compiled by g++ through
tests/emu/cuda_shim.h).  Lets the CPU test tier diff the source the GPU runs against the oracle;
it is never imported by the product package and is not a fallback for it.
"""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
from collections import namedtuple

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
    return _lib


_stats_lib = None


def stats_lib() -> C.CDLL:
    """tests/emu/plane_stats.cpp: the host emulation built with per-form store counters, compiled on first use into a
    temporary directory (the tree is left as it is).  Emu(..., library=stats_lib()) runs on it."""
    global _stats_lib
    if _stats_lib is None:
        d = tempfile.mkdtemp(prefix="ra_plane_stats_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libra_plane_stats.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-fPIC", "-shared", "-Wl,-Bsymbolic",
                               "-Wl,--no-undefined", "-o", so, os.path.join(_DIR, "plane_stats.cpp")])
        _stats_lib = C.CDLL(so)
    return _stats_lib


_ull_p = C.POINTER(C.c_ulonglong)
_int_p = C.POINTER(C.c_int)
EXTRAS = {                                     # ra_emu_<name>: the emulation's own calls, process-wide per library
    "narrow_stats": (None, [_ull_p, C.c_int]),
    "stall_stats": (None, [_ull_p, C.c_int]),
    "fetch_stats": (None, [_ull_p, C.c_int]),
    "set_fetch_poison": (None, [C.c_int]),
    "codec_roundtrip": (C.c_int, [C.POINTER(abi.RaEvent), C.POINTER(abi.RaEvent), C.POINTER(C.c_int)]),
    # the plane-stats build only
    "codec_roundtrip2": (C.c_int, [C.POINTER(abi.RaEvent), C.c_int, C.POINTER(abi.RaEvent), _int_p,
                                   C.POINTER(abi.RaEvent), _int_p, _int_p]),
    "plane_forms": (None, [_ull_p, C.c_int]),
}


def extras(library: C.CDLL | None = None) -> abi.Binding:
    """EXTRAS of an emulation library (default: tests/emu/libra_emu.so)"""
    return abi.bind(library or lib(), "ra_emu", EXTRAS)


SHORT, HEAD, LONG = 0, 1, 3          # what st_rec_plane reports: nothing but chunk 0 / chunks 0-1 / chunks 0-3
Forms = namedtuple("Forms", "short head long")


def plane_forms() -> dict:
    """Records the plane-stats build stored into a record plane since the last call, by type: {type: Forms}."""
    arr = (C.c_ulonglong * 64)()
    extras(stats_lib()).plane_forms(arr, 1)
    return {t: Forms(arr[4 * t + SHORT], arr[4 * t + HEAD], arr[4 * t + LONG]) for t in range(16)}


class Emu(abi.Backend):
    """The emulation in `library` (default: tests/emu/libra_emu.so; stats_lib() builds a plane-stats one).  The stats
    calls are process-wide: they read the counters of `library`, by default of libra_emu.so."""
    name = "emu"

    def __init__(self, n_groups: int, n_members: int, library: C.CDLL | None = None, **kw):
        super().__init__(library or lib(), "ra_engine", n_groups, n_members, **kw)

    @staticmethod
    def narrow_stats(reset: bool = True, library: C.CDLL | None = None) -> dict:
        """Rows stepped by the 32-bit pass of the hot kernel's logic, records it refused (a field >= 2^30), rows it
        left to the 64-bit general path because their sticky `wide` byte is set."""
        arr = (C.c_ulonglong * 3)()
        extras(library).narrow_stats(arr, 1 if reset else 0)
        return dict(rows_narrow=arr[0], records_refused=arr[1], rows_wide=arr[2])

    @staticmethod
    def stall_stats(reset: bool = True, library: C.CDLL | None = None) -> dict:
        """Stall contexts the hot kernel's logic handed to the general path, and those of them that carried per-peer
        "not short" bits (StallCtx::wk_hi) across the stall."""
        arr = (C.c_ulonglong * 2)()
        extras(library).stall_stats(arr, 1 if reset else 0)
        return dict(stalls=arr[0], stalls_wk_hi=arr[1])

    @staticmethod
    def underfetched(reset: bool = True, library: C.CDLL | None = None) -> int:
        """Records the hot kernel's logic decoded although the size flags of their tile did not let the kernel fetch
        all of their chunks (0 while every writer sets its flags)."""
        arr = (C.c_ulonglong * 1)()
        extras(library).fetch_stats(arr, 1 if reset else 0)
        return int(arr[0])

    @staticmethod
    def set_fetch_poison(pattern: int, library: C.CDLL | None = None) -> None:
        """Which poison pattern stands for the bytes the hot kernel did not fetch (0 or 1)."""
        extras(library).set_fetch_poison(pattern)


class EmuShards:
    """N emulated shards in this process: the CPU twin of ra_b200.sharded.Shard + LocalTransport + ShardedFlood
    (member (g, s) on shard (g + s) mod N), or with peer=True of Shard + LocalPeerTransport: every shard stores
    into the others' mailboxes (ra_engine_peer_set) and exchange() has nothing to do."""

    def __init__(self, n_shards: int, groups_local: int, members: int, cap: int = 4096, peer: bool = False, **kw):
        self.n, self.gl, self.m, self.cap, self.peer = n_shards, groups_local, members, cap, peer
        self.shards = [Emu(groups_local, members, route_on_device=True, n_shards=n_shards, shard=k, **kw)
                       for k in range(n_shards)]
        if peer:
            ptrs = []
            for s in self.shards:
                p = abi.RaPeerPtrs()
                s.call("peer_get", C.byref(p))
                ptrs.append(p)
            for k, s in enumerate(self.shards):
                for j, p in enumerate(ptrs):
                    if j != k:
                        s.call("peer_set", j, C.byref(p))
            return
        self.outbox = [(abi.RaEvent * (n_shards * cap))() for _ in range(n_shards)]
        self.inbox = [(abi.RaEvent * (n_shards * cap))() for _ in range(n_shards)]
        self.out_cnt = [(C.c_uint32 * n_shards)() for _ in range(n_shards)]
        self.in_cnt = [(C.c_uint32 * n_shards)() for _ in range(n_shards)]
        for k, s in enumerate(self.shards):
            s.call("set_outbox", self.outbox[k], self.out_cnt[k], cap)
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
            s.call("deliver", self.inbox[b], self.in_cnt[b], self.cap)

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
