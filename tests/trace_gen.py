"""TEST INFRASTRUCTURE: closed-loop RPC trace generator.

Drives the CPU oracle as a cluster simulator: RPC records it emits are queued for their
destination rows (with seeded loss, delay and duplication), WAL_APPEND notes come back as
written events after a random fsync delay, clients send commands, election timers fire,
and now and then an adversarial AppendEntries is injected.  The per-step event batches are
recorded so that the identical trace can be replayed through any backend.
"""
from __future__ import annotations

import random
from collections import defaultdict, deque
from typing import Dict, List, Sequence, Tuple

from ra_b200 import abi
from ra_suite import clone


class Cluster:
    """Network + WAL + clients around one backend (non-routed engine or oracle)."""

    def __init__(self, backend, seed: int, *, p_drop=0.02, p_dup=0.01, p_delay=0.15, p_cmd=0.5,
                 p_timeout=0.01, p_adversarial=0.01, p_withhold_written=0.05, max_cmd=3, p_query=0.0):
        self.b = backend
        self.rng = random.Random(seed)
        self.p_drop, self.p_dup, self.p_delay = p_drop, p_dup, p_delay
        self.p_cmd, self.p_timeout, self.p_adv = p_cmd, p_timeout, p_adversarial
        self.p_withhold = p_withhold_written
        self.max_cmd = max_cmd
        self.p_query = p_query                                  # consistent queries handed to leaders
        self.queues: Dict[int, deque] = defaultdict(deque)      # row -> events ready now
        self.delayed: List[Tuple[int, abi.RaEvent]] = []        # (due_step, event)
        self.step_no = 0
        self.roles: Dict[int, int] = {}
        self.idle: Dict[int, int] = defaultdict(int)

    def on_wal_append(self, note: abi.RaNote, written: abi.RaEvent) -> None:
        """Called with every WAL_APPEND note and the written event made from it, before that event is queued
        (a subclass that models the WAL's durability hooks in here; the default draws nothing)."""

    def restarted(self, row: int) -> None:
        """The member on `row` was restarted: a new process has an empty mailbox and is a follower.  Records it
        sent before, still in flight to other rows, stay in flight."""
        self.queues.pop(row, None)
        self.delayed = [x for x in self.delayed if x[1].row != row]
        self.roles[row] = abi.FOLLOWER
        self.idle[row] = 0

    def _post(self, e: abi.RaEvent, min_delay: int = 0, duplicate: bool = False) -> None:
        """queue e for a later step; duplicate: e is the network's second copy of a record already posted"""
        d = min_delay
        while self.rng.random() < self.p_delay:
            d += 1
        self.delayed.append((self.step_no + 1 + d, e))

    def next_batch(self) -> List[abi.RaEvent]:
        rng = self.rng
        b = self.b
        self.step_no += 1
        due = [x for x in self.delayed if x[0] <= self.step_no]
        self.delayed = [x for x in self.delayed if x[0] > self.step_no]
        for _, e in due:
            self.queues[e.row].append(e)
        # clients, timers
        for row in range(b.n_rows):
            role = self.roles.get(row, abi.FOLLOWER)
            if role == abi.LEADER and rng.random() < self.p_cmd:
                self.queues[row].append(abi.ev_command(row, rng.randint(1, self.max_cmd)))
            elif rng.random() < self.p_cmd * 0.02:
                self.queues[row].append(abi.ev_command(row, 1))           # misdirected command
            if self.p_query and rng.random() < (self.p_query if role == abi.LEADER else self.p_query * 0.05):
                self.queues[row].append(abi.ev_consistent_query(row))
            if rng.random() < self.p_timeout or self.idle[row] > 12 + (row % 7):
                self.queues[row].append(abi.ev_simple(row, abi.EV_ELECTION_TIMEOUT))
                self.idle[row] = 0
            if role == abi.LEADER and rng.random() < 0.05:
                self.queues[row].append(abi.ev_simple(row, abi.EV_TICK))
            if role == abi.AWAIT_CONDITION and rng.random() < 0.2:
                self.queues[row].append(abi.ev_simple(row, abi.EV_AWAIT_COND_TIMEOUT))
            if rng.random() < self.p_adv:
                self.queues[row].append(self._adversarial(row))
        batch: List[abi.RaEvent] = []
        for row in sorted(self.queues):
            q = self.queues[row]
            for _ in range(min(len(q), abi.RA_LOCAL_CAP)):
                batch.append(q.popleft())
        return batch

    def _adversarial(self, row: int) -> abi.RaEvent:
        rng = self.rng
        M = self.b.n_members
        kind = rng.randint(0, 5)
        frm = rng.randrange(M)
        term = rng.randint(0, 6)
        if kind == 0:      # AER with a guessed prev entry and one or two term runs
            n = rng.randint(0, 5)
            t1 = rng.randint(0, 5)
            terms = [t1] * n
            if n > 1 and rng.random() < 0.5:
                cut = rng.randint(1, n - 1)
                terms = [t1] * cut + [t1 + rng.randint(0, 2)] * (n - cut)
            return abi.ev_aer(row, frm, term, rng.randint(0, 12), rng.randint(0, 5), rng.randint(0, 12), terms)
        if kind == 1:
            return abi.ev_aer_reply(row, frm, term, rng.random() < 0.5, rng.randint(0, 14), rng.randint(0, 12),
                                    rng.randint(0, 5))
        if kind == 2:
            return abi.ev_request_vote(row, frm, term, rng.randint(0, 12), rng.randint(0, 5))
        if kind == 3:
            return abi.ev_pre_vote(row, frm, term, rng.randint(0, 5), rng.randint(0, 12), rng.randint(0, 5))
        if kind == 4:
            return abi.ev_written(row, rng.randint(0, 5), rng.randint(0, 8), rng.randint(0, 12))
        return abi.ev_request_vote_result(row, term, rng.random() < 0.5, frm)

    def absorb(self, msgs: Sequence[abi.RaEvent], notes: Sequence[abi.RaNote]) -> None:
        rng = self.rng
        for m in msgs:
            if rng.random() < self.p_drop:
                continue
            self._post(clone(m))
            if rng.random() < self.p_dup:
                self._post(clone(m), 1, duplicate=True)
        saw_leader = set()
        for i, n in enumerate(notes):
            last_of_row = i + 1 == len(notes) or notes[i + 1].row != n.row
            if last_of_row and n.type != abi.NOTE_STATUS and (n.aux & abi.ST_LEADER_MSG):
                saw_leader.add(n.row)                      # flags riding in the row's last note
            if n.type == abi.NOTE_WAL_APPEND:
                w = abi.ev_written(n.row, n.c, n.a, n.b)
                self.on_wal_append(n, w)
                if rng.random() < self.p_withhold:
                    self._post(w, rng.randint(3, 12))   # lagging fsync
                else:
                    self._post(w)
            elif n.type == abi.NOTE_STATUS:
                self.roles[n.row] = (n.b >> 24) & 0xff
                if n.aux & abi.ST_LEADER_MSG:
                    saw_leader.add(n.row)
        for row in range(self.b.n_rows):
            if self.roles.get(row, abi.FOLLOWER) == abi.LEADER or row in saw_leader:
                self.idle[row] = 0
            else:
                self.idle[row] += 1


def generate(make_backend, n_groups: int, n_members: int, n_steps: int, seed: int, **kw
             ) -> List[List[abi.RaEvent]]:
    """Run the simulator on a fresh oracle; return the per-step event batches."""
    b = make_backend(n_groups, n_members)
    cl = Cluster(b, seed, **kw)
    batches = []
    for _ in range(n_steps):
        batch = cl.next_batch()
        msgs, notes = b.step(batch)
        cl.absorb(msgs, notes)
        batches.append([clone(e) for e in batch])
    b.close()
    return batches


def replay(backend, batches: Sequence[Sequence[abi.RaEvent]]):
    """Feed a recorded trace to a backend; return per-step (msgs, notes) keys and final rows."""
    out = []
    for batch in batches:
        msgs, notes = backend.step([clone(e) for e in batch])
        out.append(([m.key() for m in msgs], [n.key() for n in notes]))
    rows = [r.key() for r in backend.read_rows(range(backend.n_rows))]
    return out, rows, backend.counters()
