"""Host binding of the CUDA engine (ra_b200/csrc/libra_engine.so) through its C ABI.

There is deliberately no fallback: if the shared library is missing, or no CUDA device is
present, construction raises -- the product path never routes through a CPU implementation.
"""
from __future__ import annotations

import ctypes as C
import os

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.environ.get("RA_ENGINE_SO") or os.path.join(_HERE, "csrc", "libra_engine.so")
_lib = None


class EngineUnavailable(RuntimeError):
    pass


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            raise EngineUnavailable(
                "%s is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). The engine has no CPU fallback." % _SO)
        _lib = C.CDLL(_SO)
        _lib.ra_engine_flood.restype = C.c_int
        _lib.ra_engine_flood.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64]
        _lib.ra_engine_sync.restype = C.c_int
        _lib.ra_engine_sync.argtypes = [C.c_void_p]
        _lib.ra_engine_last_kernel_ms.restype = C.c_int
        _lib.ra_engine_last_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_uint32)]
        _lib.ra_engine_strerror.restype = C.c_char_p
        _lib.ra_engine_strerror.argtypes = [C.c_int]
        _lib.ra_engine_last_cuda_error.restype = C.c_char_p
        _lib.ra_engine_last_cuda_error.argtypes = [C.c_void_p]
        _lib.ra_hostsim_create.restype = C.c_int
        _lib.ra_hostsim_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        _lib.ra_hostsim_destroy.restype = None
        _lib.ra_hostsim_destroy.argtypes = [C.c_void_p]
        _lib.ra_hostsim_run.restype = C.c_int
        _lib.ra_hostsim_run.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_int]
        _lib.ra_hostsim_stats.restype = C.c_int
        _lib.ra_hostsim_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                          C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
    return _lib


EXPORTS = ["ra_engine_create", "ra_engine_destroy", "ra_engine_load_rows", "ra_engine_reset_empty",
           "ra_engine_read_rows", "ra_engine_step", "ra_engine_flood", "ra_engine_sync",
           "ra_engine_counters", "ra_engine_last_kernel_ms", "ra_engine_strerror",
           "ra_engine_last_cuda_error", "ra_engine_get_cfg", "ra_engine_alloc_host",
           "ra_engine_free_host", "ra_engine_stall_histogram", "ra_engine_set_stream",
           "ra_engine_set_outbox", "ra_engine_deliver", "ra_engine_peer_get", "ra_engine_peer_set",
           "ra_engine_ipc_export", "ra_engine_ipc_import", "ra_engine_peer_barrier",
           "ra_engine_load_query_state", "ra_engine_read_query_state", "ra_engine_step_host",
           "ra_engine_submit", "ra_engine_submit_host", "ra_engine_collect", "ra_engine_pending_output",
           "ra_engine_fetch_output", "ra_engine_register_host", "ra_engine_unregister_host",
           "ra_engine_set_flood_barrier", "ra_engine_flood_faults", "ra_engine_set_note_format",
           "ra_engine_last_ext_count", "ra_engine_submit_host_segs"]
HOST_EXPORTS = ["ra_wal_batch_to_events", "ra_notes16_expand"]            # host-only helpers of the same library
HOSTSIM_EXPORTS = ["ra_hostsim_create", "ra_hostsim_create_multi", "ra_hostsim_destroy", "ra_hostsim_run",
                   "ra_hostsim_stats", "ra_hostsim_breakdown"]


class Engine(abi.Backend):
    """One engine = the Raft members resident on one GPU."""
    name = "engine"

    def __init__(self, n_groups: int, n_members: int, **kw):
        try:
            super().__init__(lib(), "ra_engine", n_groups, n_members, **kw)
        except abi.RaError as e:
            if e.status == abi.RA_E_NODEVICE:
                raise EngineUnavailable("no CUDA device: the engine has no CPU fallback") from e
            raise

    def _check(self, st: int, what: str) -> None:
        if st != abi.RA_OK:
            msg = lib().ra_engine_strerror(st).decode()
            if st == abi.RA_E_CUDA and self._h:
                msg += ": " + lib().ra_engine_last_cuda_error(self._h).decode()
            err = abi.RaError(st, "ra_engine_%s" % what)
            err.args = ("%s (%s)" % (err.args[0], msg),)
            raise err

    def flood(self, n_steps: int, cmds_per_step: int = 1, election_permille: int = 0, seed: int = 1,
              sync: bool = True, faults=None) -> None:
        """faults: None or (drop_permille, withhold_permille, partition_permille, partition_steps)"""
        if faults is None:
            self._check(lib().ra_engine_flood(self._h, n_steps, cmds_per_step, election_permille, seed), "flood")
        else:
            f = lib().ra_engine_flood_faults
            f.restype = C.c_int
            f.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.POINTER(abi.RaFloodFaults)]
            ff = abi.RaFloodFaults(*faults)
            self._check(f(self._h, n_steps, cmds_per_step, election_permille, seed, C.byref(ff)), "flood_faults")
        if sync:
            self.sync()

    def sync(self) -> None:
        self._check(lib().ra_engine_sync(self._h), "sync")

    # -- compact note stream (16-byte units; include/ra_engine.h ra_note16) ------------------------------------
    def set_note_format(self, compact: bool) -> None:
        f = lib().ra_engine_set_note_format
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.c_int]
        self._check(f(self._h, 1 if compact else 0), "set_note_format")
        self._last_c = (C.c_uint64 * self.n_rows)() if compact else None

    def step_compact(self, events, msgs_cap: int = 4096, units_cap: int | None = None):
        """ra_engine_step in compact mode -> (msgs, notes as expanded by ra_notes16_expand, raw units, n_ext)"""
        l = lib()
        sz = C.c_size_t
        n = len(events)
        ev = (abi.RaEvent * max(n, 1))(*events)
        units_cap = units_cap or max(256, self.n_rows * abi.RA_NOTE_CAP)
        msgs = (abi.RaEvent * msgs_cap)()
        units = (abi.RaNote16 * units_cap)()
        nm, nn = sz(0), sz(0)
        f = l.ra_engine_step
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_void_p, sz, C.POINTER(sz), C.c_void_p, sz, C.POINTER(sz)]
        self._check(f(self._h, ev, n, msgs, msgs_cap, C.byref(nm), units, units_cap, C.byref(nn)), "step")
        l.ra_engine_last_ext_count.restype = sz
        l.ra_engine_last_ext_count.argtypes = [C.c_void_p]
        n_ext = l.ra_engine_last_ext_count(self._h)
        out = (abi.RaNote * max(nn.value, 1))()
        x = l.ra_notes16_expand
        x.restype = sz
        x.argtypes = [C.c_void_p, sz, sz, C.c_void_p, C.c_void_p, sz]
        got = x(units, nn.value, n_ext, self._last_c, out, max(nn.value, 1))
        assert got == nn.value
        return list(msgs[: nm.value]), list(out[: nn.value]), list(units[: nn.value + 2 * n_ext]), n_ext

    def stall_histogram(self) -> dict:
        """{(role, event_type): count} of events that took the general kernel."""
        arr = (C.c_uint64 * 128)()
        f = lib().ra_engine_stall_histogram
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        self._check(f(self._h, arr), "stall_histogram")
        return {(i // 16, i % 16): int(arr[i]) for i in range(128) if arr[i]}

    def last_kernel_ms(self):
        ms = C.c_float(0)
        n = C.c_uint32(0)
        self._check(lib().ra_engine_last_kernel_ms(self._h, C.byref(ms), C.byref(n)), "last_kernel_ms")
        return float(ms.value), int(n.value)


class HostFlood:
    """The flood driven from the host through ra_engine_step (host buffers every step)."""

    def __init__(self, engine):
        """engine: one Engine, or a list of Engines holding disjoint sets of groups (one host thread keeps all of
        them busy through ra_engine_submit_host / ra_engine_collect: ra_hostsim_create_multi)."""
        engines = list(engine) if isinstance(engine, (list, tuple)) else [engine]
        self.e = engines[0]
        self.engines = engines
        self._h = C.c_void_p()
        f = lib().ra_hostsim_create_multi
        f.restype = C.c_int
        f.argtypes = [C.POINTER(C.c_void_p), C.c_uint32, C.POINTER(C.c_void_p)]
        arr = (C.c_void_p * len(engines))(*[e_._h for e_ in engines])
        self.e._check(f(arr, len(engines), C.byref(self._h)), "hostsim_create_multi")

    def run(self, n_steps: int, cmds_per_step: int = 1, election_permille: int = 0, seed: int = 1,
            bootstrap: bool = False) -> dict:
        self.e._check(lib().ra_hostsim_run(self._h, n_steps, cmds_per_step, election_permille, seed,
                                           1 if bootstrap else 0), "hostsim_run")
        h2d, d2h, calls = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        sec = C.c_double(0)
        lib().ra_hostsim_stats(self._h, C.byref(h2d), C.byref(d2h), C.byref(sec), C.byref(calls))
        ts, tm = C.c_double(0), C.c_double(0)
        f = lib().ra_hostsim_breakdown
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        f(self._h, C.byref(ts), C.byref(tm))
        return dict(h2d_bytes=int(h2d.value), d2h_bytes=int(d2h.value), seconds=float(sec.value),
                    engine_calls=int(calls.value), step_seconds=float(ts.value), model_seconds=float(tm.value))

    def close(self) -> None:
        if self._h:
            lib().ra_hostsim_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass
