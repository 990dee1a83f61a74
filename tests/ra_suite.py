"""Fixtures of test/ra_server_SUITE.erl restated for the include/ra_engine.h ABI.

One group, `pure` mode: a call evaluates exactly one ra_server:handle_<state>/2 clause and
returns {next_event,_} effects as records instead of chasing them -- the shape the
reference suite asserts on.  Works against any backend (oracle on CPU, engine on GPU).
"""
from __future__ import annotations

import copy
import ctypes as C
from typing import List, Sequence, Tuple

from ra_b200 import abi
from ra_b200.abi import *  # noqa: F401,F403  (constants + record constructors)

N1, N2, N3, N4, N5 = 0, 1, 2, 3, 4


def make_backend(name: str, n_groups: int, n_members: int, **kw):
    if name == "oracle":
        from oracle_lib import Oracle
        return Oracle(n_groups, n_members, **kw)
    if name == "engine":
        from ra_b200.engine import Engine
        return Engine(n_groups, n_members, **kw)
    if name == "emu":                                   # the engine's device logic compiled for the host (tests/emu/)
        from emu_lib import Emu
        return Emu(n_groups, n_members, **kw)
    raise ValueError(name)


def clone(x):
    """a copy of any ctypes record (row state, event, note, query state)"""
    d = type(x)()
    C.memmove(C.byref(d), C.byref(x), C.sizeof(x))
    return d


def closed_loop(b, steps: int, step_fn) -> List[Tuple[list, list]]:
    """A host-routed closed loop from an election timeout on every group's slot-0 member: every RPC record goes back
    in as an event of the next step, WAL_APPEND notes as written events, leaders get a command every third step.
    step_fn(events) -> (msgs, notes) steps b; returns the keys of every step's outputs."""
    evs = [abi.ev_simple(b.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(b.n_groups)]
    out = []
    for t in range(steps):
        evs.sort(key=lambda e: e.row)
        # at most RA_LOCAL_CAP per row
        take, rest, cnt = [], [], {}
        for e in evs:
            c = cnt.get(e.row, 0)
            (take if c < 4 else rest).append(e)
            cnt[e.row] = c + 1
        msgs, notes = step_fn(take)
        out.append(([m.key() for m in msgs], [n.key() for n in notes]))
        evs = rest
        for m in msgs:
            evs.append(clone(m))
            evs[-1].seq = 0
        for n in notes:
            if n.type == abi.NOTE_WAL_APPEND:
                evs.append(abi.ev_written(n.row, n.c, n.a, n.b))
        if t % 3 == 0:
            rows = b.read_rows(range(b.n_rows))
            evs += [abi.ev_command(r.row, 1) for r in rows if r.role == abi.LEADER]
    return out


def empty_state(n_servers: int, me: int) -> abi.RaRowState:
    """empty_state/2 (ra_server_SUITE.erl:4022-4032): ra_server:init/1 on a fresh log."""
    return abi.empty_row(me, 1, n_servers)


def base_state(n_servers: int) -> abi.RaRowState:
    """base_state/2 (ra_server_SUITE.erl:4034-4075): n1, term 5, log {1,1},{2,3},{3,5},
    last_written {3,5}, commit_index = last_applied = 3, every peer next=4 match=3."""
    s = abi.empty_row(N1, 1, n_servers)
    s.leader_slot = N1
    s.current_term = 5
    s.commit_index = 3
    s.last_applied = 3
    abi.set_log(s, [(0, 0), (1, 1), (2, 3), (3, 5)], last_written=(3, 5))
    for p in range(n_servers):
        s.peers[p].next_index = 4
        s.peers[p].match_index = 3
    return s


def install_snapshot(s: abi.RaRowState, idx: int, term: int) -> None:
    """ra_log_memory:install_snapshot/4 (test/ra_log_memory.erl:240-250)."""
    abi.set_log(s, [], last_written=(idx, term), snapshot=(idx, term))
    s.n_runs = 0


class Node:
    """One member under test."""

    def __init__(self, backend: str, n_servers: int, **kw):
        self.b = make_backend(backend, 1, n_servers, pure=kw.pop("pure", True), **kw)
        self.n = n_servers

    def handle(self, role: int, ev: abi.RaEvent, state: abi.RaRowState
               ) -> Tuple[int, abi.RaRowState, List[abi.RaEvent], List[abi.RaNote]]:
        st = clone(state)
        st.role = role
        ev.row = st.row
        self.b.load_rows([st])
        msgs, notes = self.b.step([ev])
        out = self.b.read_rows([st.row])[0]
        return out.role, out, msgs, notes

    def handle_follower(self, ev, state):
        return self.handle(abi.FOLLOWER, ev, state)

    def handle_leader(self, ev, state):
        return self.handle(abi.LEADER, ev, state)

    def handle_candidate(self, ev, state):
        return self.handle(abi.CANDIDATE, ev, state)

    def handle_pre_vote(self, ev, state):
        return self.handle(abi.PRE_VOTE, ev, state)

    def handle_await_condition(self, ev, state):
        return self.handle(abi.AWAIT_CONDITION, ev, state)


# ---- effect helpers ----------------------------------------------------------------

def of_type(msgs: Sequence[abi.RaEvent], t: int, next_event: bool = False) -> List[abi.RaEvent]:
    return [m for m in msgs if m.type == t and bool(m.flags & abi.EVF_NEXT_EVENT) == next_event]


def next_events(msgs: Sequence[abi.RaEvent]) -> List[abi.RaEvent]:
    return [m for m in msgs if m.flags & abi.EVF_NEXT_EVENT]


def sent(msgs: Sequence[abi.RaEvent]) -> List[abi.RaEvent]:
    return [m for m in msgs if not (m.flags & abi.EVF_NEXT_EVENT)]


def status(notes: Sequence[abi.RaNote]) -> int:
    for n in notes:
        if n.type == abi.NOTE_STATUS:
            return n.aux
    return notes[-1].aux if notes else 0       # record_leader_msg alone rides in the last note's aux


def notes_of(notes: Sequence[abi.RaNote], t: int) -> List[abi.RaNote]:
    return [n for n in notes if n.type == t]


def reply_fields(m: abi.RaEvent) -> dict:
    """#append_entries_reply{} view of an AER_REPLY record."""
    assert m.type == abi.EV_AER_REPLY
    return dict(to=m.row, from_=m.from_slot, term=m.term, success=bool(m.d), next_index=m.a,
                last_index=m.b, last_term=m.c)


def aer_fields(m: abi.RaEvent) -> dict:
    assert m.type == abi.EV_AER
    terms = [m.d if (m.n1 == 0 or k < m.n1) else m.e for k in range(m.n)]
    return dict(to=m.row, leader=m.from_slot, term=m.term, prev_log_index=m.a, prev_log_term=m.b,
                leader_commit=m.c, entries=[(m.a + 1 + k, t) for k, t in enumerate(terms)])


def log_entries(s: abi.RaRowState) -> List[Tuple[int, int]]:
    out = []
    for r in range(s.n_runs):
        end = s.run_start[r + 1] - 1 if r + 1 < s.n_runs else s.last_index
        out += [(i, s.run_term[r]) for i in range(s.run_start[r], end + 1)]
    return out


def peer(s: abi.RaRowState, slot: int) -> Tuple[int, int, int]:
    p = s.peers[slot]
    return p.next_index, p.match_index, p.commit_index_sent
