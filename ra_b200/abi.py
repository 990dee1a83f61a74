"""ctypes mirror of include/ra_engine.h (the C ABI of the batched multi-Raft engine).

Everything here is layout only: constants, POD structs, the signature of every entry point
(SIGNATURES, HOST_SIGNATURES) and a thin call wrapper that works for any shared library
exporting the ``<prefix>_create/_step/...`` entry points declared in include/ra_engine.h.
The product binds it to ``libra_engine.so`` (CUDA); the tests bind the same wrapper to the
CPU oracle and to the host emulation to diff the backends.

Reference records mirrored: src/ra.hrl:122-169 (RPC records), src/ra.hrl:63-75
(ra_peer_state()), src/ra_server.erl:73-112 (ra_server_state()).
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List, Sequence, Tuple

RA_MAX_MEMBERS = 8
RA_MAX_RUNS = 8
RA_NO_SLOT = 0xFF
RA_UNDEF_TERM = 0xFFFFFFFFFFFFFFFF
RA_MBOX_DEPTH = 4
RA_LOCAL_CAP = 4
RA_MSG_CAP = 16
RA_NOTE_CAP = 16
RA_NOTE_RESERVE = 4

# enum ra_role
FOLLOWER, CANDIDATE, PRE_VOTE, LEADER, AWAIT_CONDITION = 0, 1, 2, 3, 4
ROLE_NAMES = {FOLLOWER: "follower", CANDIDATE: "candidate", PRE_VOTE: "pre_vote",
              LEADER: "leader", AWAIT_CONDITION: "await_condition"}
# enum ra_membership
VOTER, PROMOTABLE, NON_VOTER, UNKNOWN = 0, 1, 2, 3
# enum ra_peer_status
PEER_NORMAL, PEER_SENDING_SNAPSHOT, PEER_SNAPSHOT_BACKOFF, PEER_SUSPENDED, PEER_DISCONNECTED = range(5)

# enum ra_event_type
(EV_NONE, EV_AER, EV_AER_REPLY, EV_REQUEST_VOTE, EV_REQUEST_VOTE_RES, EV_PRE_VOTE,
 EV_PRE_VOTE_RES, EV_WRITTEN, EV_COMMAND, EV_ELECTION_TIMEOUT, EV_AWAIT_COND_TIMEOUT,
 EV_PIPELINE_RPCS, EV_TICK, EV_HEARTBEAT_RPC, EV_HEARTBEAT_REPLY, EV_CONSISTENT_QUERY) = range(16)

EVF_NOOP = 0x01
EVF_NEXT_EVENT = 0x02
EVF_INFO = 0x08

# enum ra_note_type
(NOTE_NONE, NOTE_WAL_APPEND, NOTE_TRUNCATE, NOTE_COMMIT, NOTE_APPLY, NOTE_STATUS,
 NOTE_SEND_SNAPSHOT, NOTE_NOT_LEADER, NOTE_QUERY_INDEX, NOTE_QUERY_AGREED, NOTE_QUERY_APPLY,
 NOTE_CANCEL_SNAPSHOT_RETRY) = range(12)

ST_TERM_VOTE_CHANGED = 0x0001
ST_ROLE_CHANGED = 0x0002
ST_LEADER_MSG = 0x0004
ST_START_ELECTION_TMO = 0x0008
ST_MSG_DROPPED = 0x0010
ST_PIPELINE_PENDING = 0x0020
ST_FATAL = 0x0040
ST_CMD_POSTPONED = 0x0080
ST_BECAME_LEADER = 0x0100
ST_NOTE_OVERFLOW = 0x0200

FATAL_LEADER_SAW_AER_SAME_TERM = 1
FATAL_WRITE_INTEGRITY = 2
FATAL_SET_LAST_INDEX_NOT_FOUND = 3
FATAL_ASSERT = 4
FATAL_NO_SNAPSHOT = 5
FATAL_LEADER_SAW_HEARTBEAT_SAME_TERM = 6
FATAL_NOTE_OVERFLOW = 7

RA_OK, RA_E_INVAL, RA_E_NOMEM, RA_E_CUDA, RA_E_UNGROUPED, RA_E_CAPACITY, RA_E_NODEVICE = 0, -1, -2, -3, -4, -5, -6
RA_E_BUSY = -7
RA_E_PENDING = -8


class RaEvent(C.Structure):
    _fields_ = [("row", C.c_uint32), ("type", C.c_uint8), ("from_slot", C.c_uint8),
                ("flags", C.c_uint8), ("_pad", C.c_uint8), ("n", C.c_uint16), ("n1", C.c_uint16),
                ("seq", C.c_uint32),
                ("term", C.c_uint64), ("a", C.c_uint64), ("b", C.c_uint64), ("c", C.c_uint64),
                ("d", C.c_uint64), ("e", C.c_uint64)]

    def key(self) -> Tuple:
        return (self.row, self.type, self.from_slot, self.flags, self.n, self.n1, self.seq, self.term,
                self.a, self.b, self.c, self.d, self.e)

    def __repr__(self) -> str:  # pragma: no cover - debugging aid
        return ("RaEvent(row=%d type=%d from=%d flags=%d n=%d n1=%d seq=%d term=%d a=%d b=%d c=%d d=%d e=%d)"
                % self.key())


class RaNote(C.Structure):
    _fields_ = [("row", C.c_uint32), ("type", C.c_uint8), ("slot", C.c_uint8), ("aux", C.c_uint16),
                ("a", C.c_uint64), ("b", C.c_uint64), ("c", C.c_uint64)]

    def key(self) -> Tuple:
        return (self.row, self.type, self.slot, self.aux, self.a, self.b, self.c)

    def __repr__(self) -> str:  # pragma: no cover
        return "RaNote(row=%d type=%d slot=%d aux=0x%x a=%d b=%d c=%d)" % self.key()


class RaPeerInit(C.Structure):
    _fields_ = [("next_index", C.c_uint64), ("match_index", C.c_uint64),
                ("commit_index_sent", C.c_uint64), ("status", C.c_uint8), ("voter", C.c_uint8),
                ("_pad", C.c_uint8 * 6)]


class RaRowState(C.Structure):
    _fields_ = [("row", C.c_uint32), ("role", C.c_uint8), ("self_slot", C.c_uint8),
                ("n_members", C.c_uint8), ("leader_slot", C.c_uint8), ("voted_for", C.c_uint8),
                ("membership", C.c_uint8), ("condition", C.c_uint8), ("has_snapshot", C.c_uint8),
                ("votes", C.c_uint32), ("machine_version", C.c_uint32),
                ("effective_machine_version", C.c_uint32), ("n_runs", C.c_uint32),
                ("flags", C.c_uint32),
                ("current_term", C.c_uint64), ("commit_index", C.c_uint64),
                ("last_applied", C.c_uint64), ("pre_vote_token", C.c_uint64),
                ("token_counter", C.c_uint64),
                ("first_index", C.c_uint64), ("last_index", C.c_uint64), ("last_term", C.c_uint64),
                ("last_written_index", C.c_uint64), ("last_written_term", C.c_uint64),
                ("snapshot_index", C.c_uint64), ("snapshot_term", C.c_uint64),
                ("run_start", C.c_uint64 * RA_MAX_RUNS), ("run_term", C.c_uint64 * RA_MAX_RUNS),
                ("cond_reply_term", C.c_uint64), ("cond_reply_next_index", C.c_uint64),
                ("cond_reply_last_index", C.c_uint64), ("cond_reply_last_term", C.c_uint64),
                ("peers", RaPeerInit * RA_MAX_MEMBERS)]

    def key(self) -> Tuple:
        """Every field the parity diff compares, as one tuple."""
        nr = self.n_runs
        return (self.row, self.role, self.self_slot, self.n_members, self.leader_slot, self.voted_for,
                self.membership, self.condition, self.has_snapshot, self.votes, self.n_runs, self.flags,
                self.current_term, self.commit_index, self.last_applied, self.pre_vote_token,
                self.token_counter, self.first_index, self.last_index, self.last_term,
                self.last_written_index, self.last_written_term, self.snapshot_index, self.snapshot_term,
                tuple(self.run_start[i] for i in range(nr)), tuple(self.run_term[i] for i in range(nr)),
                (self.cond_reply_term, self.cond_reply_next_index, self.cond_reply_last_index,
                 self.cond_reply_last_term) if (self.flags & 2) else None,
                tuple((p.next_index, p.match_index, p.commit_index_sent, p.status, p.voter)
                      for p in list(self.peers)[: self.n_members]))


class RaNote16(C.Structure):
    """ra_note16: one 16-byte unit of the compact note stream (include/ra_engine.h)"""
    _fields_ = [("row", C.c_uint32), ("type", C.c_uint8), ("n", C.c_uint8), ("aux", C.c_uint16), ("a", C.c_uint64)]


N16_EXT, N16_SAME_TERM = 0x80, 0x40


class RaHostEvent(C.Structure):
    """ra_host_event: 32-byte record for batches of host-origin events (ra_engine_step_host)."""
    _fields_ = [("row", C.c_uint32), ("type", C.c_uint8), ("flags", C.c_uint8), ("n", C.c_uint16),
                ("term", C.c_uint64), ("a", C.c_uint64), ("b", C.c_uint64)]

    @classmethod
    def of(cls, e: "RaEvent") -> "RaHostEvent":
        return cls(row=e.row, type=e.type, flags=e.flags, n=e.n, term=e.term, a=e.a, b=e.b)


class RaQueryState(C.Structure):
    _fields_ = [("row", C.c_uint32), ("_pad", C.c_uint32), ("query_index", C.c_uint64),
                ("agreed_index", C.c_uint64), ("peer_query_index", C.c_uint64 * RA_MAX_MEMBERS)]

    def key(self, n_members: int = RA_MAX_MEMBERS) -> Tuple:
        return (self.row, self.query_index, self.agreed_index, tuple(self.peer_query_index[:n_members]))


class RaFloodFaults(C.Structure):
    """ra_flood_faults: (drop_permille, withhold_permille, partition_permille, partition_steps)"""
    _fields_ = [("drop_permille", C.c_uint32), ("withhold_permille", C.c_uint32),
                ("partition_permille", C.c_uint32), ("partition_steps", C.c_uint32)]


class RaEngineCfg(C.Structure):
    _fields_ = [("n_groups", C.c_uint32), ("n_members", C.c_uint32),
                ("max_pipeline_count", C.c_uint32), ("max_aer_batch", C.c_uint32),
                ("device", C.c_int32), ("route_on_device", C.c_uint32), ("pure", C.c_uint32),
                ("n_shards", C.c_uint32), ("shard", C.c_uint32), ("note_cap", C.c_uint32)]


class RaCounters(C.Structure):
    _fields_ = [("events", C.c_uint64), ("commits", C.c_uint64), ("applied", C.c_uint64),
                ("msgs_out", C.c_uint64), ("msgs_dropped", C.c_uint64),
                ("elections_won", C.c_uint64), ("fatal_rows", C.c_uint64), ("steps", C.c_uint64),
                ("aer_received_follower", C.c_uint64), ("aer_received_follower_empty", C.c_uint64),
                ("aer_replies_success", C.c_uint64), ("aer_replies_failed", C.c_uint64),
                ("elections", C.c_uint64), ("pre_vote_elections", C.c_uint64),
                ("term_and_voted_for_updates", C.c_uint64)]

    def as_dict(self) -> dict:
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class RaHostEventSeg(C.Structure):
    """ra_host_event_seg: one piece of a batch handed to ra_engine_submit_host_segs"""
    _fields_ = [("ev", C.POINTER(RaHostEvent)), ("n", C.c_size_t)]


class RaPeerPtrs(C.Structure):
    """ra_peer_ptrs: a shard's mailbox buffers (device pointers)"""
    _fields_ = [("mbox", C.c_void_p * 2), ("mbox_cnt", C.c_void_p * 2)]


class RaIpcHandles(C.Structure):
    """ra_ipc_handles: the same buffers as CUDA IPC handles"""
    _fields_ = [("h", (C.c_ubyte * 64) * 4)]


class RaWalWriter(C.Structure):
    """ra_wal_writer: one writer of a WAL batch, n_ranges x {from, to}"""
    _fields_ = [("row", C.c_uint32), ("n_ranges", C.c_uint32), ("term", C.c_uint64),
                ("ranges", C.POINTER(C.c_uint64))]


class RaWalResume(C.Structure):
    """ra_wal_resume: the first range ra_wal_batch_to_events has not emitted"""
    _fields_ = [("writer", C.c_uint32), ("range", C.c_uint32)]


assert C.sizeof(RaEvent) == 64
assert C.sizeof(RaHostEvent) == 32
assert C.sizeof(RaNote) == 32
assert C.sizeof(RaPeerInit) == 32


# ---- the entry points of include/ra_engine.h: name -> (restype, argtypes) ----------------------------------------
_vp, _sz, _u32, _u64, _P = C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint64, C.POINTER
# A notes buffer holds ra_note records or, in the compact format (ra_engine_set_note_format), ra_note16 units: it is
# declared void* so that arrays of either pass.  Device buffers (outbox, inbox, their counts) are addresses too.
_OUT = [_P(RaEvent), _sz, _P(_sz), _vp, _sz, _P(_sz)]            # msgs, msgs_cap, n_msgs, notes, notes_cap, n_notes
_SUBMIT_OUT = [_P(RaEvent), _sz, _vp, _sz]                       # msgs, msgs_cap, notes, notes_cap
_FLOOD = [_vp, _u32, _u32, _u32, _u64]                           # e, n_steps, cmds_per_step, election_permille, seed

SIGNATURES = {                                                   # ra_engine_<name>
    "create": (C.c_int, [_P(RaEngineCfg), _P(_vp)]),
    "destroy": (None, [_vp]),
    "get_cfg": (C.c_int, [_vp, _P(RaEngineCfg)]),
    "load_rows": (C.c_int, [_vp, _P(RaRowState), _sz]),
    "reset_empty": (C.c_int, [_vp]),
    "read_rows": (C.c_int, [_vp, _P(RaRowState), _sz]),
    "load_query_state": (C.c_int, [_vp, _P(RaQueryState), _sz]),
    "read_query_state": (C.c_int, [_vp, _P(RaQueryState), _sz]),
    "step": (C.c_int, [_vp, _P(RaEvent), _sz, *_OUT]),
    "pending_output": (C.c_int, [_vp, _P(_sz), _P(_sz)]),
    "fetch_output": (C.c_int, [_vp, *_OUT]),
    "flood": (C.c_int, _FLOOD),
    "flood_faults": (C.c_int, [*_FLOOD, _P(RaFloodFaults)]),
    "sync": (C.c_int, [_vp]),
    "counters": (C.c_int, [_vp, _P(RaCounters)]),
    "stall_histogram": (C.c_int, [_vp, _P(_u64)]),
    "last_kernel_ms": (C.c_int, [_vp, _P(C.c_float), _P(_u32)]),
    "set_stream": (C.c_int, [_vp, _vp]),
    "set_outbox": (C.c_int, [_vp, _vp, _vp, _u32]),
    "deliver": (C.c_int, [_vp, _vp, _vp, _u32]),
    "peer_get": (C.c_int, [_vp, _P(RaPeerPtrs)]),
    "peer_set": (C.c_int, [_vp, _u32, _P(RaPeerPtrs)]),
    "ipc_export": (C.c_int, [_vp, _P(RaIpcHandles)]),
    "ipc_import": (C.c_int, [_vp, _u32, _P(RaIpcHandles)]),
    "peer_barrier": (C.c_int, [_vp]),
    "set_flood_barrier": (C.c_int, [_vp, C.c_int]),
    "step_host": (C.c_int, [_vp, _P(RaHostEvent), _sz, *_OUT]),
    "submit": (C.c_int, [_vp, _P(RaEvent), _sz, *_SUBMIT_OUT]),
    "submit_host": (C.c_int, [_vp, _P(RaHostEvent), _sz, *_SUBMIT_OUT]),
    "submit_host_segs": (C.c_int, [_vp, _P(RaHostEventSeg), _sz, *_SUBMIT_OUT]),
    "collect": (C.c_int, [_vp, _P(_sz), _P(_sz)]),
    "set_note_format": (C.c_int, [_vp, C.c_int]),
    "last_ext_count": (_sz, [_vp]),
    "register_host": (C.c_int, [_vp, _sz]),
    "unregister_host": (C.c_int, [_vp]),
    "alloc_host": (_vp, [_sz]),
    "free_host": (None, [_vp]),
    "strerror": (C.c_char_p, [C.c_int]),
    "last_cuda_error": (C.c_char_p, [_vp]),
}

HOST_SIGNATURES = {                                              # ra_<name>: host code of the same library
    "hostsim_create": (C.c_int, [_vp, _P(_vp)]),
    "hostsim_create_multi": (C.c_int, [_P(_vp), _u32, _P(_vp)]),
    "hostsim_destroy": (None, [_vp]),
    "hostsim_run": (C.c_int, [_vp, _u32, _u32, _u32, _u64, C.c_int]),
    "hostsim_stats": (C.c_int, [_vp, _P(_u64), _P(_u64), _P(C.c_double), _P(_u64)]),
    "hostsim_breakdown": (C.c_int, [_vp, _P(C.c_double), _P(C.c_double)]),
    "notes16_expand": (_sz, [_vp, _sz, _sz, _P(_u64), _P(RaNote), _sz]),
    "wal_batch_to_events": (_sz, [_P(RaWalWriter), _sz, _u32, _P(RaEvent), _sz, _P(RaWalResume)]),
}


class Binding:
    """The entry points `<prefix>_<name>` of one library, as private ctypes function objects made from a signature
    table on first use: a library that lacks a symbol fails only when that call is made.  Nothing is declared on the
    CDLL's shared attributes, so what another caller assigns to `lib.<symbol>.argtypes` does not change these."""

    def __init__(self, lib: C.CDLL, prefix: str, table: dict):
        self._lib, self._prefix, self._table, self._fns = lib, prefix, table, {}

    def __getattr__(self, name: str):
        if name.startswith("_") or name not in self._table:
            raise AttributeError(name)
        f = self._fns.get(name)
        if f is None:
            f = self._fns[name] = self.make(name)
        return f

    def make(self, name: str):
        """A new function object for `name`, with the table's signature and not shared with this binding."""
        restype, argtypes = self._table[name]
        return C.CFUNCTYPE(restype, *argtypes)(("%s_%s" % (self._prefix, name), self._lib))


_bindings: dict = {}


def bind(lib: C.CDLL, prefix: str, table: dict = SIGNATURES) -> Binding:
    """The Binding of `lib` for `prefix` and `table`, made once per library."""
    key = (lib, prefix, id(table))
    if key not in _bindings:
        _bindings[key] = Binding(lib, prefix, table)
    return _bindings[key]


class RaError(RuntimeError):
    def __init__(self, status: int, what: str):
        super().__init__("%s failed: status %d" % (what, status))
        self.status = status


def empty_row(row: int, n_groups: int, n_members: int) -> RaRowState:
    """ra_server_SUITE:empty_state/2 (test/ra_server_SUITE.erl:4022-4032) for one row."""
    s = RaRowState()
    s.row = row
    s.role = FOLLOWER
    s.self_slot = row // n_groups
    s.n_members = n_members
    s.leader_slot = RA_NO_SLOT
    s.voted_for = RA_NO_SLOT
    s.membership = VOTER
    s.n_runs = 1
    s.run_start[0] = 0
    s.run_term[0] = 0
    for p in range(n_members):
        s.peers[p].next_index = 1
        s.peers[p].voter = 1
    return s


def set_log(s: RaRowState, entries: Sequence[Tuple[int, int]], last_written: Tuple[int, int] | None = None,
            snapshot: Tuple[int, int] | None = None) -> None:
    """Fill the log view of ``s`` from ``[(index, term), ...]`` (contiguous, ascending)."""
    runs: List[Tuple[int, int]] = []
    for idx, term in entries:
        if not runs or runs[-1][1] != term:
            runs.append((idx, term))
    if len(runs) > RA_MAX_RUNS:
        raise ValueError("more than RA_MAX_RUNS term runs")
    s.n_runs = len(runs)
    for i, (st, t) in enumerate(runs):
        s.run_start[i] = st
        s.run_term[i] = t
    if entries:
        s.first_index = entries[0][0]
        s.last_index, s.last_term = entries[-1]
    else:
        assert snapshot is not None
        s.first_index = snapshot[0] + 1
        s.last_index, s.last_term = snapshot
    if snapshot is not None:
        s.has_snapshot = 1
        s.snapshot_index, s.snapshot_term = snapshot
    if last_written is not None:
        s.last_written_index, s.last_written_term = last_written


def faults_arg(faults):
    """None, or (drop_permille, withhold_permille, partition_permille, partition_steps) -> ra_flood_faults*"""
    return None if faults is None else C.byref(RaFloodFaults(*faults))


class Backend:
    """One implementation of the include/ra_engine.h entry points (the CUDA engine, the CPU oracle, the host
    emulation), called through its Binding of SIGNATURES.  A subclass names the table its library follows."""
    SIGNATURES = SIGNATURES

    def __init__(self, lib: C.CDLL, prefix: str, n_groups: int, n_members: int, *, device: int = 0,
                 route_on_device: bool = False, pure: bool = False, max_pipeline_count: int = 4096,
                 max_aer_batch: int = 128, n_shards: int = 1, shard: int = 0, note_cap: int = 0):
        self._lib = lib
        self._p = prefix
        self._api = bind(lib, prefix, self.SIGNATURES)
        self.n_groups = n_groups
        self.n_members = n_members
        self.n_rows = n_groups * n_members
        self.cfg = RaEngineCfg(n_groups, n_members, max_pipeline_count, max_aer_batch, device,
                               1 if route_on_device else 0, 1 if pure else 0, n_shards, shard, note_cap)
        self._h = C.c_void_p()
        self._check(self._api.create(C.byref(self.cfg), C.byref(self._h)), "create")

    # -- plumbing -----------------------------------------------------
    def _check(self, st: int, what: str) -> None:
        if st != RA_OK:
            raise RaError(st, "%s_%s" % (self._p, what))

    def _fn(self, name: str):
        """The entry point `name` as a function object of its own, for a caller that passes the handle itself or
        declares on it: nothing it does changes this backend's binding."""
        return self._api.make(name)

    def call(self, name: str, *args) -> None:
        """The entry point `name` on this backend's handle; a status other than RA_OK raises RaError."""
        self._check(getattr(self._api, name)(self._h, *args), name)

    def close(self) -> None:
        if self._h:
            self._api.destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    # -- rows and query state -----------------------------------------
    def row_of(self, group: int, slot: int) -> int:
        return slot * self.n_groups + group

    def reset_empty(self) -> None:
        self.call("reset_empty")

    def load_rows(self, rows: Sequence[RaRowState]) -> None:
        self.call("load_rows", (RaRowState * len(rows))(*rows), len(rows))

    def _read_rows(self, ids: Sequence[int]):
        arr = (RaRowState * len(ids))()
        for i, r in enumerate(ids):
            arr[i].row = r
        self.call("read_rows", arr, len(ids))
        return arr

    def read_rows(self, row_ids: Iterable[int]) -> List[RaRowState]:
        return list(self._read_rows(list(row_ids)))

    def rows_bytes(self, chunk: int = 65536) -> bytes:
        """Every row as raw ra_row_state bytes, `chunk` rows per call."""
        return b"".join(bytes(self._read_rows(range(lo, min(self.n_rows, lo + chunk))))
                        for lo in range(0, self.n_rows, chunk))

    def load_query_state(self, qs: Sequence[RaQueryState]) -> None:
        self.call("load_query_state", (RaQueryState * max(len(qs), 1))(*qs), len(qs))

    def read_query_state(self, row_ids: Iterable[int]) -> List[RaQueryState]:
        ids = list(row_ids)
        arr = (RaQueryState * max(len(ids), 1))()
        for i, r in enumerate(ids):
            arr[i].row = r
        self.call("read_query_state", arr, len(ids))
        return list(arr)[: len(ids)]

    # -- one call: step and step_host ---------------------------------
    def _default_caps(self, n: int) -> Tuple[int, int]:
        """Output buffers for a batch of n events when the caller names none."""
        if self.cfg.route_on_device and not self.cfg.pure:   # routed: RPC records never reach the host
            return 1024, max(64, self.n_rows * RA_NOTE_CAP)
        msgs = max(64, n * RA_MSG_CAP, min(max(n, 1) * RA_MSG_CAP + RA_MSG_CAP * 64, self.n_rows * RA_MSG_CAP))
        touched = self.n_rows if self.cfg.route_on_device else min(self.n_rows, max(n, 1) + 64)
        return msgs, max(64 + n * RA_NOTE_CAP, touched * RA_NOTE_CAP)

    def step(self, events: Sequence[RaEvent], msgs_cap: int | None = None,
             notes_cap: int | None = None) -> Tuple[List[RaEvent], List[RaNote]]:
        return self._step("step", (RaEvent * max(len(events), 1))(*events), len(events), msgs_cap, notes_cap)

    def step_host(self, events: Sequence[RaEvent], msgs_cap: int | None = None,
                  notes_cap: int | None = None) -> Tuple[List[RaEvent], List[RaNote]]:
        """step() for a batch of host-origin events, handed over as 32-byte records."""
        return self._step("step_host", _host_events(events), len(events), msgs_cap, notes_cap)

    def _step(self, name, ev, n, msgs_cap, notes_cap):
        dm, dn = self._default_caps(n)
        msgs_cap = dm if msgs_cap is None else msgs_cap
        notes_cap = dn if notes_cap is None else notes_cap
        msgs, notes = (RaEvent * msgs_cap)(), (RaNote * notes_cap)()
        nm, nn = C.c_size_t(0), C.c_size_t(0)
        self.call(name, ev, n, msgs, msgs_cap, C.byref(nm), notes, notes_cap, C.byref(nn))
        return list(msgs[: nm.value]), list(notes[: nn.value])

    # -- output capacity: a step whose outputs did not fit lost nothing (include/ra_engine.h "Capacity") --------
    def pending_output(self) -> Tuple[int, int]:
        nm, nn = C.c_size_t(0), C.c_size_t(0)
        self.call("pending_output", C.byref(nm), C.byref(nn))
        return nm.value, nn.value

    def fetch_output(self, msgs_cap: int, notes_cap: int, out=None):
        """-> (status, n_msgs, n_notes, msgs, notes): RA_OK, or RA_E_CAPACITY with the sizes needed.
        out: the caller's (msgs, notes) buffers, else new ones of those capacities."""
        msgs, notes = out or _buffers(msgs_cap, notes_cap)
        nm, nn = C.c_size_t(0), C.c_size_t(0)
        st = self._api.fetch_output(self._h, msgs, msgs_cap, C.byref(nm), notes, notes_cap, C.byref(nn))
        if st not in (RA_OK, RA_E_CAPACITY):
            self._check(st, "fetch_output")
        return _outputs(st, nm.value, nn.value, msgs, notes)

    # -- split-phase calls: submit returns the status and a ticket holding the buffers until collect() ----------
    def submit(self, events: Sequence[RaEvent], msgs_cap: int, notes_cap: int, out=None):
        return self._submit("submit", (RaEvent * max(len(events), 1))(*events), len(events), msgs_cap, notes_cap, out)

    def submit_host(self, events: Sequence[RaEvent], msgs_cap: int, notes_cap: int, out=None):
        return self._submit("submit_host", _host_events(events), len(events), msgs_cap, notes_cap, out)

    def submit_host_segs(self, parts: Sequence[Sequence[RaEvent]], msgs_cap: int, notes_cap: int, out=None):
        """The batch handed over in pieces, one buffer per piece (the segments keep the pieces alive)."""
        segs = (RaHostEventSeg * max(len(parts), 1))(*[RaHostEventSeg(_host_events(p), len(p)) for p in parts])
        return self._submit("submit_host_segs", segs, len(parts), msgs_cap, notes_cap, out)

    def _submit(self, name, ev, n, msgs_cap, notes_cap, out):
        msgs, notes = out or _buffers(msgs_cap, notes_cap)
        return getattr(self._api, name)(self._h, ev, n, msgs, msgs_cap, notes, notes_cap), (ev, msgs, notes)

    def collect(self, ticket):
        """-> (status, n_msgs, n_notes, msgs, notes) of the oldest call submitted"""
        nm, nn = C.c_size_t(0), C.c_size_t(0)
        st = self._api.collect(self._h, C.byref(nm), C.byref(nn))
        _ev, msgs, notes = ticket
        return _outputs(st, nm.value, nn.value, msgs, notes)

    # -- the device-side flood and what it counts ---------------------
    def flood(self, n_steps: int, cmds_per_step: int = 1, election_permille: int = 0, seed: int = 1,
              faults=None) -> None:
        """faults: None or (drop_permille, withhold_permille, partition_permille, partition_steps)"""
        self.call("flood_faults", n_steps, cmds_per_step, election_permille, seed, faults_arg(faults))

    def counters(self) -> dict:
        c = RaCounters()
        self.call("counters", C.byref(c))
        return c.as_dict()

    def get_cfg(self) -> RaEngineCfg:
        cfg = RaEngineCfg()
        self.call("get_cfg", C.byref(cfg))
        return cfg

    def stall_histogram(self) -> dict:
        """{(role, event_type): count} of events that took the general kernel."""
        arr = (C.c_uint64 * 128)()
        self.call("stall_histogram", arr)
        return {(i // 16, i % 16): int(v) for i, v in enumerate(arr) if v}


def _host_events(events: Sequence[RaEvent]):
    return (RaHostEvent * max(len(events), 1))(*[RaHostEvent.of(e) for e in events])


def _buffers(msgs_cap: int, notes_cap: int):
    return (RaEvent * max(msgs_cap, 1))(), (RaNote * max(notes_cap, 1))()


def _outputs(st, nm, nn, msgs, notes):
    ok = st == RA_OK
    return st, nm, nn, (list(msgs[:nm]) if ok else []), (list(notes[:nn]) if ok else [])


# ---- constructors for the wire records (ra.hrl record -> 64-byte record) -----------

def ev_aer(row, leader, term, prev_idx, prev_term, leader_commit, entry_terms: Sequence[int] = ()):
    """#append_entries_rpc{} (src/ra.hrl:122-128); entry_terms = terms of prev+1..prev+n."""
    e = RaEvent(row=row, type=EV_AER, from_slot=leader, n=len(entry_terms), term=term, a=prev_idx,
                b=prev_term, c=leader_commit)
    if entry_terms:
        e.d = entry_terms[0]
        for k, t in enumerate(entry_terms):
            if t != e.d:
                e.n1 = k
                e.e = t
                if any(x != t for x in entry_terms[k:]):
                    raise ValueError("an AER record spans at most two term runs")
                break
    return e


def ev_aer_reply(row, peer, term, success, next_index, last_index, last_term):
    """{PeerId, #append_entries_reply{}} (src/ra.hrl:130-141)."""
    return RaEvent(row=row, type=EV_AER_REPLY, from_slot=peer, term=term, a=next_index, b=last_index,
                   c=last_term, d=1 if success else 0)


def ev_request_vote(row, candidate, term, last_log_index, last_log_term):
    return RaEvent(row=row, type=EV_REQUEST_VOTE, from_slot=candidate, term=term, a=last_log_index,
                   b=last_log_term)


def ev_request_vote_result(row, term, granted, voter=RA_NO_SLOT):
    return RaEvent(row=row, type=EV_REQUEST_VOTE_RES, from_slot=voter, term=term, d=1 if granted else 0)


def ev_pre_vote(row, candidate, term, token, last_log_index, last_log_term, version=1, machine_version=0):
    return RaEvent(row=row, type=EV_PRE_VOTE, from_slot=candidate, term=term, a=last_log_index,
                   b=last_log_term, c=token, d=version | (machine_version << 32))


def ev_pre_vote_result(row, term, token, granted, voter=RA_NO_SLOT):
    return RaEvent(row=row, type=EV_PRE_VOTE_RES, from_slot=voter, term=term, c=token,
                   d=1 if granted else 0)


def ev_written(row, term, first, last):
    """{ra_log_event, {written, Term, [{First, Last}]}}."""
    return RaEvent(row=row, type=EV_WRITTEN, from_slot=RA_NO_SLOT, term=term, a=first, b=last)


def ev_heartbeat_rpc(row, leader, term, query_index):
    return RaEvent(row=row, type=EV_HEARTBEAT_RPC, from_slot=leader, term=term, a=query_index)


def ev_heartbeat_reply(row, peer, term, query_index):
    return RaEvent(row=row, type=EV_HEARTBEAT_REPLY, from_slot=peer, term=term, a=query_index)


def ev_consistent_query(row):
    return RaEvent(row=row, type=EV_CONSISTENT_QUERY, from_slot=RA_NO_SLOT)


def ev_command(row, n=1, noop=False):
    return RaEvent(row=row, type=EV_COMMAND, from_slot=RA_NO_SLOT, n=n, flags=EVF_NOOP if noop else 0)


def ev_simple(row, type_):
    return RaEvent(row=row, type=type_, from_slot=RA_NO_SLOT)
