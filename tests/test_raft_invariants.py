"""Raft's safety properties and the host-note contract, checked without the oracle.

Every other parity test asks whether a backend does what oracle/ra_oracle.c does.  A mistake made in the oracle and in
the device logic alike passes all of them.  Here the oracle is one more backend under test (`oracle`, `emu` and, on a
GPU, `engine` with RA_STEP_WIDE=0 and =1), and nothing asks it for expected values.  Four kinds of check:

1. A host shadow built only from the notes (include/ra_engine.h, DESIGN §2 item 6), checked after every step against
   one read of every row:
     N1  the shadow log equals the row's log view on [first_index, last_index] (term runs, last_index, last_term);
     N2  current_term / voted_for equal the last STATUS note with RA_ST_TERM_VOTE_CHANGED (term = a, voted_for = b & 0xff);
     N3  last_applied equals the end of the APPLY chain (each APPLY{a,b} starts at the previous b + 1);
     N4  a leader's commit index changes exactly as its COMMIT{old,new} notes say (old = the commit index before);
     N5  the role changes exactly when RA_ST_ROLE_CHANGED says so, from role_old to role_new.
   Rules the header leaves to the implementation, as the oracle fixes them:
     - WAL_APPEND{a,b,c} drops every entry at a and above, then a..b have term c.  A write that starts at or below
       last_index overwrites without a TRUNCATE note (ra_log:write/2 replaces the tail; in ra_oracle.c only
       log_set_last_index, the empty-AppendEntries reset of ra_server.erl:1294-1303, emits TRUNCATE).
     - TRUNCATE{a,b} drops the entries above a, and the entry at a has term b.
     - A view that holds more than RA_MAX_RUNS term runs forgets the oldest run (DESIGN §2 item 3).
     - Adjacent view runs of one term are one run (the oracle counts a run per term change: log_push).
     - A leader's commit index may drop without a note in exactly one case: in a step in which it lowered a peer's
       match index.  A failure reply whose last index lies below the match index resets it (ra_server.erl:611-622);
       a restarted follower's mismatch reply carries its last_applied, and so does a reply to a duplicated stale
       AppendEntries.  increment_commit_index then takes the lower agreed index (:3621-3630).  In such a step a
       COMMIT note may start below the commit index before it; in every other step N4 and the leader's commit
       monotonicity are exact.
2. A closed loop (trace_gen.Cluster: loss, duplicates, delays, lagging fsync) with member restarts.  A restarted member
   is rebuilt only from what its host persisted, as ra_server:init/1 does (src/ra_server.erl:380-457): the term and
   vote of the last RA_ST_TERM_VOTE_CHANGED, the log the acknowledged WAL operations leave (the WAL is FIFO, so a
   written event acknowledges its operation and every one before it; TRUNCATE is not a WAL record, so an old tail
   may come back), at most RA_MAX_RUNS runs of it, and commit_index = last_applied = the applied index, but no
   further than the durable log holds the entries that were applied.  A follower applies entries that are not yet
   fsynced (ra_server.erl:2236-2240), so the durable log may end below them or still hold an overwritten version;
   a host persists last_applied no further than its log is durable.  Raft's properties are checked on
   every group after every step: Election Safety, one granted vote per (voter, term) across restarts, Log Matching,
   Leader Completeness, State Machine Safety, and no term / commit index / last_applied going back within a life.
3. Device-routed floods, with and without fault injection, in chunks of 1-8 steps, with the state-only properties.
4. Scripts: Figure 8 of the Raft paper (the §5.4.2 commit gate), and AppendEntries over runs longer than 65535 entries.
"""
from __future__ import annotations

import bisect
import random

import numpy as np
import pytest

import trace_gen
from emu_lib import Emu
from ra_b200 import abi
from ra_suite import clone, make_backend

LIM = 1 << 30
BIG = 1 << 62
ROW_DT = np.dtype(abi.RaRowState)
CPU_BACKENDS = ["oracle", "emu"]
WIDTHS = ["0", "1"]                         # RA_STEP_WIDE: the 32-bit hot kernel / the 64-bit one


def _backend(name, g, m, monkeypatch, width=None, **kw):
    if width is not None:
        monkeypatch.setenv("RA_STEP_WIDE", width)           # read when the backend is created
    else:
        monkeypatch.delenv("RA_STEP_WIDE", raising=False)
    return make_backend(name, g, m, **kw)


def read_all(b) -> np.ndarray:
    return np.frombuffer(b.rows_bytes(), dtype=ROW_DT).copy()


def step(b, batch):
    """One ra_engine_step with room for every row's outputs -> (RPC records, notes)."""
    return b.step(batch, 1024 if b.cfg.route_on_device else b.n_rows * abi.RA_MSG_CAP, b.n_rows * abi.RA_NOTE_CAP)


# ---- logs as term runs ------------------------------------------------------------------------------------------
class RunLog:
    """Entries (base, last]: run k covers starts[k] .. starts[k+1]-1 (or last) with terms[k]; the entry at `base`
    (a snapshot, or nothing known) has base_term (None = unknown)."""
    __slots__ = ("base", "base_term", "starts", "terms", "last")

    def __init__(self, base, base_term, starts, terms, last):
        self.base, self.base_term, self.starts, self.terms, self.last = base, base_term, list(starts), list(terms), last

    @classmethod
    def of_row(cls, r) -> "RunLog":
        n = int(r["n_runs"])
        starts, terms = _merged([int(x) for x in r["run_start"][:n]], [int(x) for x in r["run_term"][:n]])
        if n == 0:
            return cls(int(r["last_index"]), int(r["last_term"]), [], [], int(r["last_index"]))
        return cls(starts[0] - 1, None, starts, terms, int(r["last_index"]))

    def copy(self) -> "RunLog":
        return RunLog(self.base, self.base_term, self.starts, self.terms, self.last)

    def term_at(self, i):
        if i == self.base and not (self.starts and self.starts[0] == i):
            return self.base_term
        if not self.starts or i < self.starts[0] or i > self.last:
            return None
        return self.terms[bisect.bisect_right(self.starts, i) - 1]

    def write(self, a, b, c, what):
        assert self.base < a <= self.last + 1, "%s: WAL_APPEND{%d,%d,%d} leaves a gap after %d" % (what, a, b, c, self.last)
        assert b >= a, what
        k = bisect.bisect_left(self.starts, a)
        del self.starts[k:], self.terms[k:]
        if not self.terms or self.terms[-1] != c:
            self.starts.append(a)
            self.terms.append(c)
        self.last = b

    def truncate(self, a, t, what):
        have = self.term_at(a)
        assert have is None or have == t, "%s: TRUNCATE{%d,%d} but the entry there has term %s" % (what, a, t, have)
        assert a <= self.last, "%s: TRUNCATE{%d,%d} above last index %d" % (what, a, t, self.last)
        k = bisect.bisect_right(self.starts, a)
        del self.starts[k:], self.terms[k:]
        self.last = a
        if not self.starts:
            self.base, self.base_term = a, t

    def view(self, first):
        """(start, term) runs clipped to [first, last]"""
        if not self.starts or first > self.last:
            return ()
        k = max(bisect.bisect_right(self.starts, first) - 1, 0)
        return ((max(first, self.starts[k]), self.terms[k]),) + tuple(zip(self.starts[k + 1:], self.terms[k + 1:]))

    def agree_upto(self, other):
        """the last index up to which both logs hold the same entries (from the first index both know)"""
        hi = min(self.last, other.last)
        lo = max(self.starts[0] if self.starts else self.last + 1, other.starts[0] if other.starts else other.last + 1)
        for p in sorted({lo, *(x for x in self.starts + other.starts if lo < x <= hi)}):
            if p <= hi and self.term_at(p) != other.term_at(p):
                return p - 1
        return hi

    def horizon(self):
        """the last RA_MAX_RUNS runs, as a load_rows view"""
        return self.starts[-abi.RA_MAX_RUNS:], self.terms[-abi.RA_MAX_RUNS:]


def _merged(starts, terms):
    s, t = [], []
    for a, b in zip(starts, terms):
        if not t or t[-1] != b:
            s.append(a)
            t.append(b)
    return s, t


# ---- the state-only properties, vectorised over all groups --------------------------------------------------
class Views:
    """log views of N rows as arrays: S/T (N, 8) run starts / terms (padding BIG / -1), F/L first / last index"""

    def __init__(self, S, T, F, L):
        self.S, self.T, self.F, self.L = S, T, F, L

    @classmethod
    def of(cls, rows):
        n = rows["n_runs"].astype(np.int64)
        pad = np.arange(abi.RA_MAX_RUNS)[None, :] >= n[:, None]
        S = np.where(pad, BIG, rows["run_start"].astype(np.int64))
        T = np.where(pad, -1, rows["run_term"].astype(np.int64))
        F = rows["first_index"].astype(np.int64)
        L = rows["last_index"].astype(np.int64)
        F = np.where(n == 0, L + 1, F)
        return cls(S, T, F, L)

    def take(self, idx):
        return Views(self.S[idx], self.T[idx], self.F[idx], self.L[idx])

    def term_at(self, P, missing):
        k = (self.S[:, None, :] <= P[:, :, None]).sum(2) - 1
        t = np.take_along_axis(self.T, np.clip(k, 0, None), 1)
        ok = (k >= 0) & (P >= self.F[:, None]) & (P <= self.L[:, None])
        return np.where(ok, t, missing)


def _segments(A: Views, B: Views, lo, hi):
    """the pieces of [lo, hi] on which both logs are constant: (start, valid, terms agree)"""
    P = np.concatenate([A.S, B.S], 1)
    P = np.where((P > lo[:, None]) & (P <= hi[:, None]), P, BIG)
    P = np.sort(np.concatenate([lo[:, None], P], 1), 1)
    nxt = np.concatenate([P[:, 1:], np.full((len(lo), 1), BIG)], 1)
    end = np.minimum(nxt - 1, hi[:, None])
    valid = (P <= end) & (P < BIG) & (lo <= hi)[:, None]
    agree = A.term_at(P, -2) == B.term_at(P, -3)
    return P, valid, agree


def log_matching_violations(A, B, lo, hi):
    """rows where some index holds the same term in both logs but a lower one (inside lo..hi) differs"""
    P, valid, agree = _segments(A, B, lo, hi)
    top_agree = np.where(valid & agree, P, -1).max(1)
    low_disagree = np.where(valid & ~agree, P, BIG).min(1)
    return np.nonzero(low_disagree < top_agree)[0]


def differ_on(A, B, lo, hi):
    """rows where the two logs differ somewhere on lo..hi (an index missing from one of them counts)"""
    _, valid, agree = _segments(A, B, lo, hi)
    return np.nonzero((valid & ~agree).any(1))[0]


class Checker:
    """Election Safety, Log Matching, Leader Completeness, State Machine Safety and monotonicity over all groups."""

    def __init__(self, g, m):
        self.g, self.m = g, m
        self.leaders = {}                                   # (group, term) -> slot
        self.C = Views(np.full((g, abi.RA_MAX_RUNS), BIG), np.full((g, abi.RA_MAX_RUNS), -1),
                       np.zeros(g, np.int64), np.full(g, -1, np.int64))  # committed entries as first seen on a leader
        self.c_term = np.zeros(g, np.int64)                 # the term of the leader that showed them
        self.prev = None
        self.n_leader_obs = self.n_commit_adv = 0

    def restarted(self, row, state):
        if self.prev is not None:
            for k in ("current_term", "commit_index", "last_applied", "role"):
                self.prev[k][row] = int(getattr(state, k))
            self.prev["match"][row] = [p.match_index for p in state.peers]

    def check(self, rows, what):
        g, m = self.g, self.m
        V = Views.of(rows)
        grp = np.arange(len(rows)) % g
        slot = np.arange(len(rows)) // g
        term = rows["current_term"].astype(np.int64)
        commit = rows["commit_index"].astype(np.int64)
        applied = rows["last_applied"].astype(np.int64)
        lead = np.nonzero(rows["role"] == abi.LEADER)[0]
        # Election Safety
        for r, t in zip(lead.tolist(), term[lead].tolist()):
            s = self.leaders.setdefault((r % g, t), r // g)
            assert s == r // g, "%s: group %d has two leaders in term %d: slots %d and %d" % (what, r % g, t, s, r // g)
        self.n_leader_obs += len(lead)
        # Log Matching, every pair of members of every group, inside both horizons
        for a in range(m):
            for c in range(a + 1, m):
                A, B = V.take(slice(a * g, (a + 1) * g)), V.take(slice(c * g, (c + 1) * g))
                bad = log_matching_violations(A, B, np.maximum(A.F, B.F), np.minimum(A.L, B.L))
                assert not len(bad), "%s: Log Matching fails in group %d between slots %d and %d:\n%s\n%s" % (
                    what, bad[0], a, c, _fmt(rows[a * g + bad[0]]), _fmt(rows[c * g + bad[0]]))
        # Leader Completeness: a leader of the committing term or later holds every committed entry it could see
        Cg = self.C.take(grp[lead])
        Vl = V.take(lead)
        chk = term[lead] >= self.c_term[grp[lead]]
        lo = np.maximum(Vl.F, Cg.F)
        bad = differ_on(Vl, Cg, lo, np.where(chk, Cg.L, -1))
        assert not len(bad), "%s: leader row %d (term %d) lacks committed entries up to %d:\n%s" % (
            what, lead[bad[0]], term[lead[bad[0]]], Cg.L[bad[0]], _fmt(rows[lead[bad[0]]]))
        # record what leaders newly show committed
        for r in lead[np.argsort(term[lead], kind="stable")].tolist():
            q = r % g
            if commit[r] > self.C.L[q] and commit[r] >= V.F[r]:
                self.n_commit_adv += 1
                keep = V.S[r] <= commit[r]
                self.C.S[q], self.C.T[q] = np.where(keep, V.S[r], BIG), np.where(keep, V.T[r], -1)
                self.C.F[q], self.C.L[q], self.c_term[q] = V.F[r], commit[r], term[r]
        # State Machine Safety: what a member applied holds the committed term
        Ca = self.C.take(grp)
        hi = np.minimum(np.minimum(applied, V.L), Ca.L)
        bad = differ_on(V, Ca, np.maximum(V.F, Ca.F), hi)
        assert not len(bad), "%s: row %d applied up to %d, against committed entries:\n%s" % (
            what, bad[0], applied[bad[0]], _fmt(rows[bad[0]]))
        # within one life: term, a leader's commit index (a follower takes its leader's verbatim, ra_server.erl:1315)
        # and last_applied never go back
        role = rows["role"]
        if self.prev is not None:
            same_leader = (role == abi.LEADER) & (self.prev["role"] == abi.LEADER) & (term == self.prev["current_term"])
            same_leader &= ~match_reset(self.prev["match"], rows)
            for k, now in (("current_term", term), ("commit_index", np.where(same_leader, commit, BIG)),
                           ("last_applied", applied)):
                back = np.nonzero(now < self.prev[k])[0]
                assert not len(back), "%s: row %d %s went back from %d to %d" % (what, back[0], k, self.prev[k][back[0]],
                                                                                now[back[0]])
        self.prev = dict(current_term=term, commit_index=commit, last_applied=applied, role=role.copy(),
                         match=rows["peers"]["match_index"].copy())
        return V

    def check_applied(self, applies, what):
        """State Machine Safety on what was applied: every (row, first, last, runs) -- runs = the (start, term) of
        the entries as the row held them when it applied them -- must carry the committed terms.  Returns the
        ranges not yet covered by what leaders have shown committed."""
        keep, cache = [], {}
        for r, a, b, runs in applies:
            q = r % self.g
            if q not in cache:
                cache[q] = RunLog(int(self.C.F[q]) - 1, None, [x for x in self.C.S[q].tolist() if x < BIG],
                                  [x for x in self.C.T[q].tolist() if x >= 0], int(self.C.L[q]))
            c = cache[q]
            mine = RunLog(a - 1, None, [x for x, _ in runs], [t for _, t in runs], b)
            lo, hi = max(a, c.starts[0] if c.starts else c.last + 1), min(b, c.last)
            for p in sorted({lo, *(x for x in mine.starts + c.starts if lo < x <= hi)}):
                if p <= hi:
                    assert mine.term_at(p) == c.term_at(p), "%s: row %d applied index %d of term %s, committed term %s" % (
                        what, r, p, mine.term_at(p), c.term_at(p))
            if b > c.last:
                keep.append((r, max(a, c.last + 1), b, runs))
        return keep


def match_reset(match_before, rows):
    """Rows that lowered a peer's match index in this step.  A failure reply whose last index lies below the peer's
    match index resets it (ra_server.erl:611-622): a restarted follower's mismatch reply carries its last_applied,
    and so does a follower's reply to a duplicated, stale AppendEntries.  increment_commit_index then takes the
    lower agreed index (:3621-3630), so only in such a step may a leader's commit index drop, without a note."""
    return (rows["peers"]["match_index"] < match_before).any(1)


def _fmt(r):
    n = int(r["n_runs"])
    return ("row %d role %d term %d first %d last %d (term %d) commit %d applied %d runs %s"
            % (r["row"], r["role"], r["current_term"], r["first_index"], r["last_index"], r["last_term"],
               r["commit_index"], r["last_applied"], list(zip(r["run_start"][:n].tolist(), r["run_term"][:n].tolist()))))


# ---- the host: shadow from the notes, WAL durability, restarts ---------------------------------------------
class Host:
    """What ra_server_proc learns from the output stream, per row, and what it persisted."""

    def __init__(self, b, rows):
        self.b = b
        self.template = [abi.RaRowState.from_buffer_copy(rows[i].tobytes()) for i in range(len(rows))]
        self.log = [RunLog.of_row(r) for r in rows]
        self.durable = [l.copy() for l in self.log]
        self.meta = [(int(r["current_term"]), int(r["voted_for"])) for r in rows]
        self.applied = [int(r["last_applied"]) for r in rows]
        self.before = None
        self.ops = [[] for _ in rows]                       # WAL operations not yet acknowledged: (number, a, b, c)
        self.op_no = [0] * len(rows)
        self.pending_written = {}                           # id(written event) -> (event, row, operation number)
        self.votes = {}                                     # (voter row, term) -> candidate slot
        self.fatal = {}                                     # row -> reason
        self.applies = []                                   # APPLY ranges to check against committed terms
        self.n_became_leader = self.n_commit_notes = self.n_restart_cut = 0
        self.set_before(rows)

    def set_before(self, rows):
        self.before = dict(role=rows["role"].tolist(), commit=rows["commit_index"].tolist(),
                           match=rows["peers"]["match_index"].copy())

    # WAL
    def on_wal_append(self, note, written):
        r = note.row
        self.op_no[r] += 1
        self.ops[r].append((self.op_no[r], note.a, note.b, note.c))
        self.pending_written[id(written)] = (written, r, self.op_no[r])

    def delivered(self, batch):
        """the batch goes to the members: each written event in it acknowledges its WAL operation and those before"""
        for e in batch:
            if e.type == abi.EV_WRITTEN:
                hit = self.pending_written.pop(id(e), None)
                if hit is None:
                    continue
                _, r, no = hit
                ops = self.ops[r]
                while ops and ops[0][0] <= no:
                    _, a, b_, c = ops.pop(0)
                    self.durable[r].write(a, b_, c, "durable log of row %d" % r)

    # notes
    def absorb(self, msgs, notes, rows, what):
        g = self.b.n_groups
        for m_ in msgs:                                     # vote uniqueness on the RPC stream
            if m_.type == abi.EV_REQUEST_VOTE_RES and m_.d == 1:
                voter = (m_.from_slot * g) + (m_.row % g)
                cand = self.votes.setdefault((voter, m_.term), m_.row // g)
                assert cand == m_.row // g, "%s: row %d granted votes in term %d to slots %d and %d" % (
                    what, voter, m_.term, cand, m_.row // g)
        role0, commit0 = self.before["role"], self.before["commit"]
        role1, commit1 = rows["role"].tolist(), rows["commit_index"].tolist()
        may_drop = match_reset(self.before["match"], rows)
        touched = {}
        for n in notes:
            r, t = n.row, n.type
            w = "%s row %d" % (what, r)
            st = touched.setdefault(r, [role0[r], commit0[r], False])
            if t == abi.NOTE_WAL_APPEND:
                self.log[r].write(n.a, n.b, n.c, w)
            elif t == abi.NOTE_TRUNCATE:
                self.log[r].truncate(n.a, n.b, w)
            elif t == abi.NOTE_APPLY:
                assert n.a == self.applied[r] + 1 and n.b >= n.a, "%s: APPLY{%d,%d} after %d" % (w, n.a, n.b, self.applied[r])
                self.applied[r] = n.b
                runs = self.log[r].view(n.a)
                self.applies.append((r, n.a, n.b, [x for x in runs if x[0] <= n.b]))
            elif t == abi.NOTE_COMMIT:
                self.n_commit_notes += 1
                if role0[r] == abi.LEADER or st[2]:
                    ok = n.a == st[1] or (n.a < st[1] and may_drop[r])
                    assert ok, "%s: COMMIT{%d,%d} but the commit index was %d" % (w, n.a, n.b, st[1])
                assert n.b > n.a, w
                st[1], st[2] = n.b, True
            elif t == abi.NOTE_STATUS:
                if n.aux & abi.ST_TERM_VOTE_CHANGED:
                    self.meta[r] = (n.a, n.b & 0xff)
                if n.aux & abi.ST_ROLE_CHANGED:
                    old, new = (n.b >> 16) & 0xff, (n.b >> 24) & 0xff
                    assert old == st[0], "%s: role_old %d, but the role was %d" % (w, old, st[0])
                    st[0] = new
                if n.aux & abi.ST_BECAME_LEADER:
                    self.n_became_leader += 1
                if n.aux & abi.ST_FATAL:
                    self.fatal[r] = n.c
        for r, (role, cm, saw) in touched.items():          # N4, N5 for rows with notes
            assert role1[r] == role, "%s row %d: role %d after the step, notes say %d" % (what, r, role1[r], role)
            if role1[r] == abi.LEADER and (saw or role0[r] == abi.LEADER):
                ok = commit1[r] == cm or (commit1[r] < cm and may_drop[r])
                assert ok, "%s row %d: leader commit index %d, notes say %d" % (what, r, commit1[r], cm)
        r0, c0 = np.asarray(role0), np.asarray(commit0, dtype=np.uint64)
        moved = np.where(may_drop, rows["commit_index"] > c0, rows["commit_index"] != c0)
        for r in np.nonzero((rows["role"] != r0) | ((rows["role"] == abi.LEADER) & (r0 == abi.LEADER) & moved))[0].tolist():
            assert r in touched, "%s row %d: role / leader commit index changed without a note" % (what, r)
        self.compare(rows, what)
        self.set_before(rows)

    def check_applied(self, chk, what):
        """after the Checker saw this step's rows: what was applied carries the committed terms"""
        self.applies = chk.check_applied(self.applies, what)[-4 * self.b.n_rows:]

    def compare(self, rows, what):
        """N1-N3 for every row"""
        F, L, LT = rows["first_index"].tolist(), rows["last_index"].tolist(), rows["last_term"].tolist()
        n, RS, RT = rows["n_runs"].tolist(), rows["run_start"].tolist(), rows["run_term"].tolist()
        term, voted, applied = rows["current_term"].tolist(), rows["voted_for"].tolist(), rows["last_applied"].tolist()
        for r in range(len(F)):
            lg = self.log[r]
            s, t = _merged(RS[r][: n[r]], RT[r][: n[r]])
            view = tuple(zip(s, t))
            assert lg.last == L[r] and lg.view(F[r]) == view and (lg.term_at(L[r]) in (None, LT[r])), (
                "%s row %d: N1 the notes describe the log %s (last %d), the row holds %s (first %d last %d/%d)"
                % (what, r, lg.view(F[r]), lg.last, view, F[r], L[r], LT[r]))
            assert (term[r], voted[r]) == self.meta[r], "%s row %d: N2 term/voted_for %s, persisted %s" % (
                what, r, (term[r], voted[r]), self.meta[r])
            assert applied[r] == self.applied[r], "%s row %d: N3 last_applied %d, APPLY notes end at %d" % (
                what, r, applied[r], self.applied[r])

    # restart
    def restart_state(self, r):
        """ra_server:init/1 from what the host persisted"""
        s = abi.RaRowState.from_buffer_copy(bytes(self.template[r]))
        d = self.durable[r]
        starts, terms = d.horizon()
        if len(d.starts) > abi.RA_MAX_RUNS:
            self.n_restart_cut += 1
        s.role, s.leader_slot, s.votes, s.flags, s.condition = abi.FOLLOWER, abi.RA_NO_SLOT, 0, 0, 0
        s.current_term, s.voted_for = self.meta[r]
        s.n_runs = len(starts)
        for k in range(abi.RA_MAX_RUNS):
            s.run_start[k] = starts[k] if k < len(starts) else 0
            s.run_term[k] = terms[k] if k < len(terms) else 0
        s.first_index = starts[0] if starts else d.last + 1
        s.last_index = d.last
        s.last_term = terms[-1] if starts else d.base_term
        s.last_written_index, s.last_written_term = s.last_index, s.last_term
        s.commit_index = s.last_applied = max(min(self.applied[r], d.agree_upto(self.log[r])), self.template[r].last_applied)
        s.pre_vote_token = s.token_counter = 0
        return s

    def restart(self, r, s):
        d = self.durable[r]
        starts, terms = d.horizon()
        self.log[r] = RunLog(starts[0] - 1 if starts else d.base, None if starts else d.base_term, starts, terms, d.last)
        self.applied[r] = s.last_applied
        self.ops[r] = []
        self.fatal.pop(r, None)
        self.before["role"][r], self.before["commit"][r] = abi.FOLLOWER, s.commit_index


class HostCluster(trace_gen.Cluster):
    """The Cluster with the host's WAL model, over channels that delay and duplicate but keep their order, like the
    Erlang distribution ra runs on: ra_server asserts on a re-ordered stale empty AppendEntries (ra_server.erl:
    1294-1303).  The WAL answers in order too (ra_log_wal is one process): a written event that overtook an earlier
    one would move last_written, and with it a leader's commit index, back (ra_log.erl:849-896 takes any matching
    written index).  Vote results are never duplicated: ra counts granted votes (`Votes + 1`, ra_server.erl:1028-1034,
    1215-1222), so a duplicated grant would elect a second leader, and Erlang distribution never duplicates."""

    def __init__(self, backend, seed, host=None, **kw):
        super().__init__(backend, seed, **kw)
        self.host = host
        self.last_due = {}
        self.n_dup = 0

    def on_wal_append(self, note, written):
        self.host.on_wal_append(note, written)

    def _post(self, e, min_delay=0, duplicate=False):
        if duplicate:
            if e.type in (abi.EV_REQUEST_VOTE_RES, abi.EV_PRE_VOTE_RES):
                return
            self.n_dup += 1
        d = min_delay
        while self.rng.random() < self.p_delay:
            d += 1
        key = (e.row, e.from_slot if e.type != abi.EV_WRITTEN else -1)
        due = max(self.step_no + 1 + d, self.last_due.get(key, 0))
        self.last_due[key] = due
        self.delayed.append((due, e))


def _restarted_cluster(b, base, term):
    """Every member restarts from a snapshot at (base, term): empty log, everything written / applied up to it
    (as tests/test_narrow_pass.py starts its runs across the 32-bit limit)."""
    rows = []
    for r in range(b.n_rows):
        s = abi.empty_row(r, b.n_groups, b.n_members)
        abi.set_log(s, [], last_written=(base, term), snapshot=(base, term))
        s.current_term = term
        s.commit_index = s.last_applied = base
        for p in range(b.n_members):
            s.peers[p].next_index = base + 1
        rows.append(s)
    b.load_rows(rows)


# ---- 2. the closed loop with restarts -------------------------------------------------------------------------
def run_closed_loop(b, steps, seed, pure=False, p_restart=0.03, min_restarts=3, base=None, **knobs):
    """Routed (route_on_device): the members' records travel through the device mailboxes and never reach the host,
    so loss, duplicates, delays and the vote check on the RPC stream apply only to the unrouted loop; the notes,
    the WAL, restarts and every state check are the same."""
    g, m = b.n_groups, b.n_members
    routed = bool(b.cfg.route_on_device)
    if base is None:
        b.reset_empty()
    else:
        _restarted_cluster(b, *base)
    rows = read_all(b)
    chk = Checker(g, m)
    host = Host(b, rows)
    kw = dict(p_drop=0.05, p_dup=0.02, p_delay=0.15, p_timeout=0.02, p_withhold_written=0.1, p_adversarial=0.0)
    kw.update(knobs)
    cl = HostCluster(b, seed, host, **kw)
    rng = random.Random(seed * 7 + 1)
    restarts = {"leader": 0, "other": 0}
    won_after_restart = 0
    became0 = None
    for t in range(steps):
        batch = cl.next_batch()
        host.delivered(batch)
        msgs, notes = step(b, batch)
        rows = read_all(b)
        what = "step %d" % t
        host.absorb(msgs, notes, rows, what)
        chk.check(rows, what)
        host.check_applied(chk, what)
        if pure:                                            # {next_event, _}: to the member itself, first
            nxt = [x for x in msgs if x.flags & abi.EVF_NEXT_EVENT]
            for x in reversed(nxt):
                e = clone(x)
                e.flags &= ~abi.EVF_NEXT_EVENT
                cl.queues[e.row].appendleft(e)
            msgs = [x for x in msgs if not x.flags & abi.EVF_NEXT_EVENT]
        cl.absorb(msgs, notes)
        # restarts between steps: a leader or any other member of a random group
        if t > 20 and rng.random() < p_restart * g ** 0.5:
            q = rng.randrange(g)
            roles = [int(rows["role"][s * g + q]) for s in range(m)]
            s = roles.index(abi.LEADER) if abi.LEADER in roles and rng.random() < 0.5 else rng.randrange(m)
            kind = "leader" if roles[s] == abi.LEADER else "other"
            r = s * g + q
            st = host.restart_state(r)
            b.load_rows([st])
            cl.restarted(r)
            host.restart(r, st)
            chk.restarted(r, st)
            restarts[kind] += 1
            if became0 is None:
                became0 = host.n_became_leader
            rows = read_all(b)
            host.compare(rows, what + " after restarting row %d" % r)
            host.set_before(rows)
    if became0 is not None:
        won_after_restart = host.n_became_leader - became0
    # a leader whose view forgot the entries a lagging or restarted follower needs -- the horizon of DESIGN §2 item 3,
    # or a restart that kept only RA_MAX_RUNS runs -- stops like ra_server without a snapshot (:2378); nothing else may
    bad = {r: c for r, c in host.fatal.items() if c != abi.FATAL_NO_SNAPSHOT}
    assert not bad, "fatal rows other than RA_FATAL_NO_SNAPSHOT: %s" % bad
    assert len(host.fatal) <= max(2, g * m // 50), (host.fatal, host.n_restart_cut)
    assert restarts["leader"] >= min_restarts and restarts["other"] >= min_restarts, restarts
    assert won_after_restart >= restarts["leader"] // 2, "too few elections after restarts"
    assert chk.n_commit_adv > g and host.n_commit_notes > g, "the run committed too little"
    assert kw["p_withhold_written"] > 0 and (routed or (kw["p_delay"] > 0 and cl.n_dup > 0))
    return dict(restarts=restarts, fatal=len(host.fatal), commits=chk.n_commit_adv, won=won_after_restart)


CLOSED_CPU = [(m, g, steps, mode) for m, g, steps in ((3, 16, 400), (4, 12, 350), (5, 12, 400), (7, 8, 300), (8, 8, 300))
              for mode in ("chased", "pure")]


@pytest.mark.parametrize("backend", CPU_BACKENDS)
@pytest.mark.parametrize("m,g,steps,mode", CLOSED_CPU)
def test_closed_loop_with_restarts(backend, m, g, steps, mode, monkeypatch):
    b = _backend(backend, g, m, monkeypatch, pure=(mode == "pure"))
    run_closed_loop(b, steps, 100 * m + g + (mode == "pure"), pure=(mode == "pure"))


NARROW_STARTS = [(LIM - 150, 3), ((1 << 32) - 150, (1 << 32) - 4)]


@pytest.mark.parametrize("backend", CPU_BACKENDS)
@pytest.mark.parametrize("base,term", NARROW_STARTS)
def test_closed_loop_with_restarts_across_the_narrow_limit(backend, base, term, monkeypatch):
    b = _backend(backend, 12, 5, monkeypatch)
    if backend == "emu":
        Emu.narrow_stats()
    run_closed_loop(b, 350, 31 + base % 7, base=(base, term), p_cmd=0.9, max_cmd=3)
    if backend == "emu":
        st = Emu.narrow_stats()
        if base < LIM:
            assert st["rows_narrow"] > 0 and st["rows_wide"] > 0, st     # rows on both sides of 2^30
        else:
            assert st["rows_narrow"] == 0, st                            # a bulk load this wide: the 64-bit hot pass
    assert int(read_all(b)["last_index"].max()) > (LIM if base < LIM else 1 << 32)


@pytest.mark.parametrize("backend", CPU_BACKENDS)
@pytest.mark.parametrize("m", [1, 2, 3, 5, 6, 7])
def test_closed_loop_with_restarts_routed(backend, m, monkeypatch):
    b = _backend(backend, 12, m, monkeypatch, route_on_device=True)
    run_closed_loop(b, 300, 500 + m)


# The kernel each engine case launches (ra_b200/csrc/engine.cu, table k_step_kernels): routed, M = 3, 5 and 7
# have their own hot kernel in both passes; unrouted, only M = 5 has one (TR_HOST); every other M runs the runtime-M
# kernel, which has no 32-bit pass -- so RA_STEP_WIDE only matters for the first two.
CLOSED_GPU = ([(m, g, True, w) for m, g in ((3, 512), (5, 384), (7, 256)) for w in WIDTHS]
              + [(5, 384, False, w) for w in WIDTHS] + [(4, 384, False, None), (8, 256, False, None)]
              + [(2, 512, True, None), (6, 256, True, None)])


@pytest.mark.gpu
@pytest.mark.parametrize("m,g,routed,width", CLOSED_GPU)
def test_closed_loop_with_restarts_engine(m, g, routed, width, monkeypatch):
    b = _backend("engine", g, m, monkeypatch, width, route_on_device=routed)
    run_closed_loop(b, 200, 900 + m, p_restart=0.01)


@pytest.mark.gpu
@pytest.mark.parametrize("width", WIDTHS)
def test_closed_loop_with_restarts_across_the_narrow_limit_engine(width, monkeypatch):
    b = _backend("engine", 256, 5, monkeypatch, width, route_on_device=True)
    run_closed_loop(b, 200, 77, base=(LIM - 120, LIM - 3), p_restart=0.01, p_cmd=0.9, max_cmd=3, p_timeout=0.03)
    top = read_all(b)
    assert int(max(top["last_index"].max(), top["current_term"].max())) > LIM, "the run did not cross 2^30"


# ---- 3. floods in chunks ------------------------------------------------------------------------------------
def run_flood(b, steps, cmds, permille, seed, faults=None, base=None):
    g = b.n_groups
    if base is None:
        b.reset_empty()
        b.step([abi.ev_simple(b.row_of(i, 0), abi.EV_ELECTION_TIMEOUT) for i in range(g)])
    else:
        _restarted_cluster(b, *base)
        b.step([abi.ev_simple(b.row_of(i, 0), abi.EV_ELECTION_TIMEOUT) for i in range(g)])
    chk = Checker(g, b.n_members)
    rng = random.Random(seed)
    kw = dict(threads=4) if b.name == "oracle" else {}
    done = rejoined = 0
    prev = None
    while done < steps:
        k = min(rng.randint(1, 8), steps - done)
        b.flood(k, cmds, permille, seed=seed + done, faults=faults, **kw)
        done += k
        rows = read_all(b)
        V = chk.check(rows, "flood step %d" % done)
        if prev is not None:                                # a tail cut or rewritten below the old last index
            pL, pT = prev
            now = V.term_at(pL[:, None], -2)[:, 0]
            rejoined += int(((V.L < pL) | ((now >= 0) & (now != pT))).sum())
        prev = (V.L.copy(), rows["last_term"].astype(np.int64))
    c = b.counters()
    assert c["fatal_rows"] == 0 and c["commits"] > g * steps // 8
    return c, chk, rejoined


FLOODS_CPU = [("oracle", 300, 5, 120, 2, 10, None), ("emu", 300, 5, 120, 2, 10, None),
              ("oracle", 200, 7, 200, 1, 10, (20, 50, 100, 16)), ("emu", 200, 7, 200, 1, 10, (20, 50, 100, 16)),
              ("emu", 150, 3, 200, 1, 10, (0, 0, 100, 24))]


@pytest.mark.parametrize("be,g,m,steps,cmds,permille,faults", FLOODS_CPU)
def test_flood_in_chunks(be, g, m, steps, cmds, permille, faults, monkeypatch):
    b = _backend(be, g, m, monkeypatch, route_on_device=True)
    c, chk, rejoined = run_flood(b, steps, cmds, permille, 5 + g, faults)
    if faults and faults[2]:
        assert c["elections_won"] > g and rejoined > 0, (c["elections_won"], rejoined)


@pytest.mark.parametrize("be", CPU_BACKENDS)
def test_flood_in_chunks_across_the_narrow_limit(be, monkeypatch):
    b = _backend(be, 120, 5, monkeypatch, route_on_device=True)
    run_flood(b, 120, 1, 20, 9, base=(LIM - 40, 7))
    assert int(read_all(b)["last_index"].max()) > LIM


# fault floods launch the fault kernels (5 and 7 routed, runtime-M for the rest), which have no 32-bit pass
FLOODS_GPU = [(2000, 5, 150, 64, 10, None, "0"), (2000, 5, 150, 64, 10, None, "1"),
              (2000, 5, 200, 1, 10, (20, 50, 100, 16), None), (2000, 4, 200, 1, 10, (20, 50, 100, 16), None),
              (10_000, 7, 400, 1, 0, (5, 20, 10, 32), None)]                 # configs[4] at its stated size


@pytest.mark.gpu
@pytest.mark.parametrize("g,m,steps,cmds,permille,faults,width", FLOODS_GPU)
def test_flood_in_chunks_engine(g, m, steps, cmds, permille, faults, width, monkeypatch):
    b = _backend("engine", g, m, monkeypatch, width, route_on_device=True)
    c, chk, rejoined = run_flood(b, steps, cmds, permille, 11, faults)
    if faults and faults[2]:
        assert c["elections_won"] > g and rejoined > 0, (c["elections_won"], rejoined)


@pytest.mark.gpu
def test_flood_in_chunks_across_the_narrow_limit_engine(monkeypatch):
    b = _backend("engine", 4000, 5, monkeypatch, route_on_device=True)
    run_flood(b, 120, 1, 20, 9, base=(LIM - 40, 7))
    assert int(read_all(b)["last_index"].max()) > LIM


# ---- 4a. Figure 8 of the Raft paper -----------------------------------------------------------------------------
class Script:
    """One group, records delivered by hand: `link(src, dst, record)` decides what arrives.  WAL writes are
    acknowledged at once for members that are up, except on slots in `hold` (a lagging fsync)."""

    def __init__(self, backend, m, monkeypatch, **kw):
        self.b = _backend(backend, 1, m, monkeypatch, **kw)
        self.b.reset_empty()
        rows = read_all(self.b)
        self.chk = Checker(1, m)
        self.host = Host(self.b, rows)
        self.up = set(range(m))
        self.mail = []                                      # records and written events not yet delivered
        self.hold = set()
        self.t = 0

    def run(self, extra=(), link=lambda s, d, r: True, max_steps=60):
        """deliver what `link` lets through until nothing is left to deliver (or max_steps) -> the rows"""
        self.mail += list(extra)
        for _ in range(max_steps):
            batch, keep, per = [], [], {}
            for e in self.mail:
                if e.row in self.up and per.get(e.row, 0) < abi.RA_LOCAL_CAP:
                    per[e.row] = per.get(e.row, 0) + 1
                    batch.append(e)
                elif e.row in self.up:
                    keep.append(e)
            self.mail = keep
            batch.sort(key=lambda e: e.row)
            self.host.delivered(batch)
            msgs, notes = step(self.b, batch)
            rows = read_all(self.b)
            self.t += 1
            self.host.absorb(msgs, notes, rows, "script step %d" % self.t)
            self.chk.check(rows, "script step %d" % self.t)
            self.host.check_applied(self.chk, "script step %d" % self.t)
            for x in msgs:
                if x.row in self.up and link(x.from_slot, x.row, x):
                    self.mail.append(clone(x))
            for n in notes:
                if n.type == abi.NOTE_WAL_APPEND and n.row in self.up:
                    w = abi.ev_written(n.row, n.c, n.a, n.b)
                    self.host.on_wal_append(n, w)
                    if n.row not in self.hold:
                        self.mail.append(w)
            if not self.mail:
                break
        return rows

    def crash(self, s):
        self.up.discard(s)
        self.mail = [e for e in self.mail if e.row != s]

    def restart(self, s):
        st = self.host.restart_state(s)
        self.b.load_rows([st])
        self.host.restart(s, st)
        self.chk.restarted(s, st)
        self.up.add(s)
        rows = read_all(self.b)
        self.host.compare(rows, "restart of slot %d" % s)
        self.host.set_before(rows)

    def elect(self, s, link, term_min):
        """election timeouts on slot s until it leads in a term >= term_min, then let the records settle"""
        for _ in range(8):
            self.mail.append(abi.ev_simple(s, abi.EV_ELECTION_TIMEOUT))
            for _ in range(12):
                rows = self.run((), link, max_steps=1)
                if rows["role"][s] == abi.LEADER and rows["current_term"][s] >= term_min:
                    return self.run((), link)
        raise AssertionError("slot %d did not win an election of term >= %d" % (s, term_min))


def _among(*slots):
    ss = set(slots)
    return lambda s, d, r: s in ss and d in ss


@pytest.mark.parametrize("backend", CPU_BACKENDS + [pytest.param("engine", marks=pytest.mark.gpu)])
def test_figure_8(backend, monkeypatch):
    S1, S2, S3, S4, S5 = range(5)
    sc = Script(backend, 5, monkeypatch, max_aer_batch=1)
    def entries_to(dst):
        return lambda s, d, r: r.type == abi.EV_AER and r.n > 0 and d in dst
    # S1 leads a term t1 and the noop at idx that opens it reaches S2 only
    among = _among(S1, S2, S3)
    rows = sc.elect(S1, lambda s, d, r: among(s, d, r) and not entries_to((S3,))(s, d, r), 1)
    t1, idx = int(rows["current_term"][S1]), int(rows["last_index"][S1])
    rows = sc.run((), lambda s, d, r: (s, d) in ((S1, S2), (S2, S1)))
    assert sc.host.log[S2].term_at(idx) == t1 and sc.host.log[S3].last < idx
    sc.crash(S1)
    # S5 wins a later term t5 with S3, S4 and itself, appends at idx in t5 (durably), and crashes
    among = _among(S3, S4, S5)
    rows = sc.elect(S5, lambda s, d, r: among(s, d, r) and not entries_to((S3, S4))(s, d, r), t1 + 1)
    t5 = int(rows["current_term"][S5])
    assert sc.host.durable[S5].term_at(idx) == t5 and sc.host.log[S3].last < idx
    sc.crash(S5)
    # S1 restarts and wins a later term; of its AppendEntries only those that carry nothing above idx travel, so
    # S3 and S4 take idx of term t1 and idx is on a majority -- but its term is not the leader's
    sc.restart(S1)
    live = (S1, S2, S3, S4)
    old_only = lambda s, d, r: s in live and d in live and (r.type != abi.EV_AER or r.n == 0 or r.a + r.n <= idx)
    sc.elect(S1, old_only, t5 + 1)
    rows = sc.run((), old_only)
    assert all(sc.host.log[s].term_at(idx) == t1 for s in (S1, S3, S4)), "idx did not reach a majority"
    assert int(rows["commit_index"][S1]) < idx, "S1 committed an entry of an older term by counting replicas (§5.4.2)"
    # S1 crashes, S5 restarts and is elected, and overwrites idx: nothing was committed there
    sc.crash(S1)
    sc.restart(S5)
    live5 = lambda s, d, r: S1 not in (s, d)
    sc.elect(S5, live5, int(rows["current_term"][S1]) + 1)
    rows = sc.run([abi.ev_command(S5, 1)], live5)
    for s in (S2, S3, S4, S5):
        assert sc.host.log[s].term_at(idx) == t5, "slot %d holds term %s at %d" % (s, sc.host.log[s].term_at(idx), idx)
    assert int(rows["commit_index"][S5]) > idx


@pytest.mark.parametrize("backend", CPU_BACKENDS + [pytest.param("engine", marks=pytest.mark.gpu)])
def test_no_reply_before_written(backend, monkeypatch):
    """A follower acknowledges entries only once they are written (ra_server.erl:1348-1371 writes and replies on
    the written event, :2236-2240).  S2 holds a new entry whose fsync lags, S3 is cut off: the leader must not
    commit it.  If it did, S2 could restart without it and S2 and S3 elect a leader that lacks a committed entry."""
    S1, S2, S3 = range(3)
    sc = Script(backend, 3, monkeypatch)
    rows = sc.elect(S1, lambda s, d, r: True, 1)
    t1, idx = int(rows["current_term"][S1]), int(rows["last_index"][S1]) + 1
    assert int(rows["commit_index"][S1]) == idx - 1, "the leader's first entry is not committed"
    sc.hold.add(S2)
    rows = sc.run([abi.ev_command(S1, 1)], lambda s, d, r: S3 not in (s, d))
    assert sc.host.log[S2].term_at(idx) == t1 and sc.host.durable[S2].last < idx, "S2 did not take the entry unwritten"
    assert int(rows["commit_index"][S1]) < idx, "S1 committed %d on a reply sent before S2 had written it" % idx
    # the leader crashes, S2 restarts from its durable log, S2 and S3 elect a leader: nothing committed is lost
    sc.crash(S1)
    sc.crash(S2)
    sc.hold.clear()
    sc.restart(S2)
    sc.elect(S3, lambda s, d, r: S1 not in (s, d), t1 + 1)
    rows = sc.run([abi.ev_command(S3, 1)], lambda s, d, r: S1 not in (s, d))
    assert int(rows["commit_index"][S3]) >= idx and sc.host.log[S2].term_at(idx) == int(rows["current_term"][S3])


# ---- 4b. AppendEntries over runs longer than 65535 entries ----------------------------------------------------
def _long_leader(b, runs, last):
    rows = []
    for r in range(b.n_rows):
        s = abi.empty_row(r, b.n_groups, b.n_members)
        s.current_term = runs[-1][1]
        if r // b.n_groups == 0:
            s.role, s.leader_slot = abi.LEADER, 0
            s.n_runs = len(runs) + 1
            for k, (a, t) in enumerate([(0, 0)] + list(runs)):
                s.run_start[k], s.run_term[k] = a, t
            s.last_index, s.last_term = last, runs[-1][1]
            s.last_written_index, s.last_written_term = last, runs[-1][1]
            for p in range(b.n_members):
                s.peers[p].next_index = 1
        else:
            s.leader_slot = 0
        rows.append(s)
    b.load_rows(rows)


LONG_LOGS = [([(1, 1)], 70_001), ([(1, 1), (70_001, 2)], 70_100)]


@pytest.mark.parametrize("routed", [False, True])
@pytest.mark.parametrize("runs,last", LONG_LOGS)
@pytest.mark.parametrize("backend", CPU_BACKENDS + [pytest.param("engine", marks=pytest.mark.gpu)])
def test_append_entries_longer_than_65535(backend, runs, last, routed, monkeypatch):
    g, m = 2, 3
    b = _backend(backend, g, m, monkeypatch, max_aer_batch=0xFFFFFFFF, max_pipeline_count=0xFFFFFFFF,
                 route_on_device=routed)
    _long_leader(b, runs, last)
    chk = Checker(g, m)
    host = Host(b, read_all(b))
    mail = [abi.ev_simple(b.row_of(q, 0), abi.EV_PIPELINE_RPCS) for q in range(g)]
    for t in range(12):
        batch = sorted(mail, key=lambda e: e.row)
        mail = []
        host.delivered(batch)
        msgs, notes = step(b, batch)
        rows = read_all(b)
        host.absorb(msgs, notes, rows, "step %d" % t)
        chk.check(rows, "step %d" % t)
        for x in msgs:
            if x.type == abi.EV_AER:
                assert x.n >= x.n1 and x.a + x.n <= last, "step %d: AppendEntries prev %d n %d n1 %d, leader last %d" % (
                    t, x.a, x.n, x.n1, last)
            mail.append(clone(x))
        for n in notes:
            if n.type == abi.NOTE_WAL_APPEND:
                w = abi.ev_written(n.row, n.c, n.a, n.b)
                host.on_wal_append(n, w)
                mail.append(w)
        if (rows["last_index"] == last).all() and (rows["commit_index"] == last).all():
            break
    rows = read_all(b)
    assert (rows["last_index"] == last).all(), "followers did not reach the leader's last index %d: %s" % (
        last, rows["last_index"].tolist())
