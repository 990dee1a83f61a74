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
    return _lib


EXPORTS = ["ra_engine_" + n for n in abi.SIGNATURES]
HOSTSIM_EXPORTS = ["ra_" + n for n in abi.HOST_SIGNATURES if n.startswith("hostsim_")]
HOST_EXPORTS = ["ra_" + n for n in abi.HOST_SIGNATURES if not n.startswith("hostsim_")]   # host-only helpers

# entry points beyond include/ra_engine.h, of a build variant only (the probe build of tools/warp_timeline.py)
EXTRAS = {"warp_timeline": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t])}


def host(library: C.CDLL | None = None) -> abi.Binding:
    """ra_hostsim_*, ra_notes16_expand and ra_wal_batch_to_events of `library` (default: the engine library), host
    code that needs no device"""
    return abi.bind(library or lib(), "ra", abi.HOST_SIGNATURES)


def notes16_expand(units, n_notes: int, n_ext: int, last_c) -> list:
    """ra_notes16_expand: compact units + their extension area (an array or bytes) -> the ra_note records"""
    out = (abi.RaNote * max(n_notes, 1))()
    got = host().notes16_expand(units, n_notes, n_ext, last_c, out, max(n_notes, 1))
    assert got == n_notes
    return list(out[:n_notes])


class Engine(abi.Backend):
    """One engine = the Raft members resident on one GPU."""
    name = "engine"
    SIGNATURES = {**abi.SIGNATURES, **EXTRAS}

    def __init__(self, n_groups: int, n_members: int, **kw):
        try:
            super().__init__(lib(), "ra_engine", n_groups, n_members, **kw)
        except abi.RaError as e:
            if e.status == abi.RA_E_NODEVICE:
                raise EngineUnavailable("no CUDA device: the engine has no CPU fallback") from e
            raise

    def _check(self, st: int, what: str) -> None:
        if st != abi.RA_OK:
            msg = self._api.strerror(st).decode()
            if st == abi.RA_E_CUDA and self._h:
                msg += ": " + self._api.last_cuda_error(self._h).decode()
            err = abi.RaError(st, "ra_engine_%s" % what)
            err.args = ("%s (%s)" % (err.args[0], msg),)
            raise err

    def flood(self, n_steps: int, cmds_per_step: int = 1, election_permille: int = 0, seed: int = 1,
              sync: bool = True, faults=None) -> None:
        """faults: None or (drop_permille, withhold_permille, partition_permille, partition_steps)"""
        super().flood(n_steps, cmds_per_step, election_permille, seed, faults)
        if sync:
            self.sync()

    def sync(self) -> None:
        self.call("sync")

    # -- compact note stream (16-byte units; include/ra_engine.h ra_note16) ------------------------------------
    def set_note_format(self, compact: bool) -> None:
        self.call("set_note_format", 1 if compact else 0)
        self._last_c = (C.c_uint64 * self.n_rows)() if compact else None

    def last_ext_count(self) -> int:
        return self._api.last_ext_count(self._h)

    def step_compact(self, events, msgs_cap: int = 4096, units_cap: int | None = None):
        """ra_engine_step in compact mode -> (msgs, notes as expanded by ra_notes16_expand, raw units, n_ext)"""
        n = len(events)
        ev = (abi.RaEvent * max(n, 1))(*events)
        units_cap = units_cap or max(256, self.n_rows * abi.RA_NOTE_CAP)
        msgs = (abi.RaEvent * msgs_cap)()
        units = (abi.RaNote16 * units_cap)()
        nm, nn = C.c_size_t(0), C.c_size_t(0)
        self.call("step", ev, n, msgs, msgs_cap, C.byref(nm), units, units_cap, C.byref(nn))
        n_ext = self.last_ext_count()
        out = notes16_expand(units, nn.value, n_ext, self._last_c)
        return list(msgs[: nm.value]), out, list(units[: nn.value + 2 * n_ext]), n_ext

    def last_kernel_ms(self):
        ms = C.c_float(0)
        n = C.c_uint32(0)
        self.call("last_kernel_ms", C.byref(ms), C.byref(n))
        return float(ms.value), int(n.value)


class HostFlood:
    """The flood driven from the host through the step calls of the C ABI (host buffers every step): ra_hostsim, on
    the library of the backends it is given (the engine, or the host emulation in tests/emu)."""

    def __init__(self, engine):
        """engine: one backend, or a list of backends holding disjoint sets of groups (one host thread keeps all of
        them busy through ra_engine_submit_host / ra_engine_collect: ra_hostsim_create_multi)."""
        engines = list(engine) if isinstance(engine, (list, tuple)) else [engine]
        self.e = engines[0]
        self.engines = engines
        self._api = host(self.e._lib)
        self._h = C.c_void_p()
        arr = (C.c_void_p * len(engines))(*[e_._h for e_ in engines])
        self.e._check(self._api.hostsim_create_multi(arr, len(engines), C.byref(self._h)), "hostsim_create_multi")

    def run(self, n_steps: int, cmds_per_step: int = 1, election_permille: int = 0, seed: int = 1,
            bootstrap: bool = False) -> dict:
        self.e._check(self._api.hostsim_run(self._h, n_steps, cmds_per_step, election_permille, seed,
                                            1 if bootstrap else 0), "hostsim_run")
        h2d, d2h, calls = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        sec = C.c_double(0)
        self._api.hostsim_stats(self._h, C.byref(h2d), C.byref(d2h), C.byref(sec), C.byref(calls))
        ts, tm = C.c_double(0), C.c_double(0)
        self._api.hostsim_breakdown(self._h, C.byref(ts), C.byref(tm))
        return dict(h2d_bytes=int(h2d.value), d2h_bytes=int(d2h.value), seconds=float(sec.value),
                    engine_calls=int(calls.value), step_seconds=float(ts.value), model_seconds=float(tm.value))

    def close(self) -> None:
        if self._h:
            self._api.hostsim_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass
