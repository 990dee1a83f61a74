"""TEST INFRASTRUCTURE: loader for the CPU oracle (oracle/libra_oracle.so).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may use this; the product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from ra_b200 import abi

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO = os.path.join(_ROOT, "oracle", "libra_oracle.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        src = os.path.join(_ROOT, "oracle", "ra_oracle.c")
        if (not os.path.exists(_SO)) or os.path.getmtime(_SO) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", os.path.join(_ROOT, "oracle")], stdout=subprocess.DEVNULL)
        _lib = C.CDLL(_SO)
    return _lib


_u32 = C.c_uint32
_FLOOD = [C.c_void_p, _u32, _u32, _u32, C.c_uint64, _u32]          # ..., seed, threads
EXTRAS = {                                                          # ra_oracle_<name> beyond include/ra_engine.h
    "flood": (C.c_int, _FLOOD),
    "flood_faults": (C.c_int, [*_FLOOD, C.POINTER(abi.RaFloodFaults)]),
    "set_sample": (C.c_int, [C.c_void_p, _u32, _u32, _u32]),
    "agreed_commit": (C.c_uint64, [C.POINTER(C.c_uint64), C.c_size_t]),
}


class Oracle(abi.Backend):
    name = "oracle"
    SIGNATURES = {**abi.SIGNATURES, **EXTRAS}

    def __init__(self, n_groups: int, n_members: int, **kw):
        super().__init__(lib(), "ra_oracle", n_groups, n_members, **kw)

    def flood(self, n_steps: int, cmds_per_step: int = 1, election_permille: int = 0, seed: int = 1,
              threads: int = 1, faults=None) -> None:
        """threads > 1: groups are sharded statically over that many pthreads"""
        self.call("flood_faults", n_steps, cmds_per_step, election_permille, seed, threads, abi.faults_arg(faults))

    def set_sample(self, stride: int, offset: int, total_groups: int) -> None:
        """group g of this oracle plays global group offset + g * stride of a flood over total_groups groups"""
        self.call("set_sample", stride, offset, total_groups)


def agreed_commit(indexes):
    arr = (C.c_uint64 * len(indexes))(*indexes)
    return int(abi.bind(lib(), "ra_oracle", Oracle.SIGNATURES).agreed_commit(arr, len(indexes)))
