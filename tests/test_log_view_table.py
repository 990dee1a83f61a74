"""Every step kernel's log view against the rule restated over a literal per-index log, one crafted member per case.

The kernels keep a member's log as at most RA_MAX_RUNS (start, term) runs, a cached start of the last run (lrs) and a
cold first_index; the oracle keeps a literal term per index.  Every clause that reads or changes the log walks the runs
(raft_logic.cuh: run_find, log_fetch_term, log_append and its horizon, log_truncate, log_set_last_index,
log_handle_written, drop_existing in handle_follower, make_aer and its two-run cut).  Here the rule is restated once
more, over a plain {index: term} map, and for every M from 1 to 8 the table holds

- views of 0 runs plus a snapshot and of 1 to 8 runs of 1, 2 or several entries, with a snapshot just below
  first_index, further below, or none, and applied / commit / last_written at, below and above run boundaries;
- followers' AppendEntries with prev_idx at every run's start - 1, start, start + 1 and end, last_index and
  last_index + 1, first_index - 1 and the snapshot index (right and wrong term), carrying 0, 1 or several entries of
  one run or two-run batches whose first piece matches up to the first entry, the middle of a local run, a run
  boundary or throughout; conflicts 1..7 runs deep, truncations onto the snapshot that empty the view, appends that
  start a 9th run and two-run batches on 7 and 8 runs (one AppendEntries, two evictions);
- written events ending in the last run, in an earlier run, above last_index and at or below the snapshot, with terms
  that match at `to`, only lower down, or nowhere;
- up to 4 events in one row's step (lrs cached, invalidated and rebuilt), and a second step with the host's own written
  event for each WAL_APPEND note of the first, read by a fresh launch;
- leaders of 1 to 8 runs whose peers' next_index sit at the same positions, stepped with a pipeline pass, a successful
  reply or a command (a command on 8 runs whose last run is an earlier term evicts in the hot kernel, and pushes peers
  below first_index: a snapshot send or RA_FATAL_NO_SNAPSHOT).

What every backend reads back, its WAL_APPEND / TRUNCATE / SEND_SNAPSHOT notes and (where records come back: host and
pure) its append_entries_reply and append_entries_rpc records must equal the restated rule; the emulation's and the
engine's records, notes, raw rows, counters and query state must equal the oracle's.  The stall histogram must show
that same-term appends at last_index, written events ending in the last run and leaders' commands stayed in the hot
kernel and that everything else reached the general kernel: a change that only moves work between the kernels changes
no result, so only this can catch it.

Two restated branches cannot be reached from a valid row: set_last_index's {not_found, _} (the empty AppendEntries that
calls it has already found its prev entry in the log or at the snapshot), and the 65535-entry cut (no batch here is
that large; tests/test_raft_invariants.py sends one).
"""
import copy
import functools
import random
from collections import Counter

import pytest

from emu_lib import Emu
from fuzz_lib import TABLE_SETTINGS, compare, observe, shift_event, shift_state
from oracle_lib import Oracle
from ra_b200 import abi
from ra_suite import clone, make_backend

UNDEF = abi.RA_UNDEF_TERM
NO = abi.RA_NO_SLOT
MEMBERS = list(range(1, abi.RA_MAX_MEMBERS + 1))
# two more settings: AppendEntries cut at 3 entries (inside runs) and a small pipeline
SETTINGS = dict(TABLE_SETTINGS)
SETTINGS["batch3-routed"] = (dict(route_on_device=True, max_aer_batch=3, max_pipeline_count=5), "0", None, True)
SETTINGS["batch3-host"] = (dict(route_on_device=False, max_aer_batch=3, max_pipeline_count=5), "1", None, True)
DEFAULT_BATCH, DEFAULT_PIPE = 128, 4096          # abi.Backend's defaults


# ---- the rule, restated over a literal log ---------------------------------------------------------------------------
class Log:
    """A member as the reference keeps it: {index: term} over [first, last], an optional snapshot (idx, term),
    last_written, applied, commit; the role, its peers and what one step emitted.  No runs: runs() derives them."""

    def __init__(self, m, me, role, term, entries, snap, lw, applied, commit, leader, first=None):
        self.m, self.me, self.role, self.term, self.leader = m, me, role, term, leader
        self.t = dict(entries)
        self.first = entries[0][0] if entries else (first or snap[0] + 1)
        self.last = entries[-1][0] if entries else self.first - 1
        self.last_term = entries[-1][1] if entries else snap[1]
        self.snap = snap
        self.lw = (lw, srv_fetch_term(self, lw) if srv_fetch_term(self, lw) is not None else 0)
        self.applied, self.commit = applied, commit
        self.peers = [[1, 0, 0] for _ in range(m)]              # next_index, match_index, commit_index_sent
        self.fatal = 0
        self.notes, self.msgs, self.tags = [], [], set()

    def __deepcopy__(self, memo):
        x = copy.copy(self)
        x.t, x.peers = dict(self.t), [list(p) for p in self.peers]
        x.notes, x.msgs, x.tags = list(self.notes), list(self.msgs), set(self.tags)
        return x

    def runs(self):
        out = []
        for i in range(self.first, self.last + 1):
            if not out or out[-1][1] != self.t[i]:
                out.append((i, self.t[i]))
        return out

    def spans(self):
        """(start, end, term) of every run"""
        r = self.runs()
        return [(s, (r[k + 1][0] - 1 if k + 1 < len(r) else self.last), t) for k, (s, t) in enumerate(r)]

    def row(self, row):
        s = abi.empty_row(row, 1, self.m)
        s.row, s.self_slot = row, self.me
        abi.set_log(s, [(i, self.t[i]) for i in range(self.first, self.last + 1)], last_written=self.lw,
                    snapshot=self.snap)
        s.first_index, s.last_index, s.last_term = self.first, self.last, self.last_term   # (gaps above a snapshot)
        s.role, s.current_term, s.leader_slot, s.voted_for = self.role, self.term, self.leader, self.leader
        s.commit_index, s.last_applied = self.commit, self.applied
        for p in range(self.m):
            s.peers[p].next_index, s.peers[p].match_index, s.peers[p].commit_index_sent = self.peers[p]
            s.peers[p].voter = 1
        return s


def fetch_term(L, i):
    """ra_log:fetch_term/2 (ra_log.erl:1140-1152): only inside [first_index, last_index]"""
    return L.t[i] if L.first <= i <= L.last and i >= 0 else None


def srv_fetch_term(L, i):
    """ra_server:fetch_term/2 (ra_server.erl:3158-3169): falls back on the snapshot"""
    t = fetch_term(L, i)
    if t is None and L.snap is not None and L.snap[0] == i:
        return L.snap[1]
    return t


def has_entry(L, idx, term):
    """has_log_entry_or_snapshot/3 (:3141-3156)"""
    t = fetch_term(L, idx)
    if t is None:
        if L.snap is not None and L.snap[0] == idx:
            return "ok" if L.snap[1] == term else "term_mismatch"
        return "missing"
    return "ok" if t == term else "term_mismatch"


def horizon(L):
    """contract (DESIGN §2 item 3): while the log holds more than RA_MAX_RUNS term runs, the oldest is forgotten and
    first_index moves past it"""
    n = 0
    while len(L.runs()) > abi.RA_MAX_RUNS:
        nxt = L.runs()[1][0]
        for i in range(L.first, nxt):
            del L.t[i]
        L.first = nxt
        n += 1
    return n


def append(L, n, term):
    """ra_log:append/2, the tail of write/2: n entries of one term at last_index + 1; returns the runs forgotten"""
    ev = 0
    for _ in range(n):
        idx = L.last + 1
        if L.first > L.last:
            L.first = idx
        L.t[idx] = term
        L.last, L.last_term = idx, term
        ev += horizon(L)
    return ev


def truncate(L, idx, fallback):
    """drop everything above idx (ra_range:limit); an emptied view keeps `fallback` as last_term"""
    cut = [(s, e) for s, e, _ in L.spans() if e > idx]
    if cut:
        L.tags.add("conflict %d runs deep" % len(cut))
    for i in [i for i in L.t if i > idx]:
        del L.t[i]
    if idx < L.first:
        L.first, L.last_term = idx + 1, fallback
        L.tags.add("truncation empties the view")
    else:
        L.last_term = L.t[idx]
    L.last = idx


def set_last_index(L, idx):
    """ra_log:set_last_index/2 (ra_log.erl:800-845); False = {not_found, _}"""
    t = fetch_term(L, idx)
    at_snap = L.snap is not None and L.snap[0] == idx
    if t is None and not at_snap:
        return False
    if at_snap:
        truncate(L, idx, L.snap[1])
        L.last_term, L.lw = L.snap[1], L.snap
        L.tags.add("set_last_index at the snapshot")
        return True
    lwidx = min(idx, L.lw[0])
    lwterm = L.snap[1] if L.snap is not None and L.snap[0] == lwidx else fetch_term(L, lwidx)
    truncate(L, idx, t)
    L.lw = (lwidx, UNDEF if lwterm is None else lwterm)
    return True


def written(L, term, frm, to):
    """ra_log:handle_event({written, Term, [{From, To}]}) (ra_log.erl:849-896), index by index: the highest index of
    [from, to] whose term is Term becomes last_written; undefined above the log is a mismatch; at or below the
    snapshot the walk ends.  (A truncating write leaves last_written alone, ra_log.erl:543-557.)"""
    i = to
    while True:
        t = fetch_term(L, i)
        if t is not None and t == term:
            L.lw = (i, term)
            L.tags.add("written matches at to" if i == to else "written matches lower down")
            return
        if t is None and L.snap is not None and i <= L.snap[0]:
            L.tags.add("written at or below the snapshot")
            return
        if i == 0 or i - 1 < frm:
            L.tags.add("written matches nowhere")
            return
        i -= 1


def reply(L, to, term, a, b, c, d):
    L.msgs.append((abi.EV_AER_REPLY, to, term, a, b, c, d))


def aer_reply(L, term, ok):
    """append_entries_reply/3 (:3597-3604): next_index, last written index and term"""
    reply(L, L.leader, term, L.last + 1, L.lw[0], L.lw[1], 1 if ok else 0)


def note(L, kind, *args):
    L.notes.append((kind,) + args)


def set_fatal(L, code):
    L.fatal = L.fatal or code


def apply_to(L, idx):
    """apply_to/3 (:3217-3255): last_applied up to min(idx, last_index)"""
    to = min(L.last, idx)
    if idx > L.applied and to > L.applied:
        L.applied = to


def drop_existing(L, prev, terms):
    """drop_existing/3 (:3673-3681): how many leading entries the log already holds"""
    k = 0
    while k < len(terms) and fetch_term(L, prev + 1 + k) == terms[k]:
        k += 1
    if terms:
        fst = prev + 1 + k
        L.tags.add("drop_existing never stops" if k == len(terms) else
                   "drop_existing stops at the first entry" if k == 0 else
                   "drop_existing stops at a run boundary" if fetch_term(L, fst) is None or
                   fetch_term(L, fst) != fetch_term(L, fst - 1) else
                   "drop_existing stops inside a local run")
    return k


def follower_aer(L, e):
    """handle_follower(#append_entries_rpc{}) (:1266-1424), the rpc's term at least the current term"""
    prev, pt, terms, leader, lc = e["prev"], e["pt"], e["terms"], e["from"], e["commit"]
    L.leader = leader
    r = has_entry(L, prev, pt)
    L.tags.add("prev entry " + r)
    if r == "ok":
        k = drop_existing(L, prev, terms)
        if k == len(terms):                                             # Entries == [] :1288
            if not terms and L.last > prev:                             # :1294-1303
                if prev < L.applied:
                    L.tags.add("fatal: set_last_index below applied")
                    return set_fatal(L, abi.FATAL_ASSERT)
                if not set_last_index(L, prev):
                    L.tags.add("fatal: set_last_index not_found")
                    return set_fatal(L, abi.FATAL_SET_LAST_INDEX_NOT_FOUND)
                note(L, abi.NOTE_TRUNCATE, L.last, L.last_term)
                ok = True
            else:
                ok = L.last <= prev + k
            if ok:                                                      # :1313-1326
                L.tags.add("validated reply")
                L.commit = lc
                apply_to(L, L.commit)
                aer_reply(L, e["term"], True)
            else:                                                       # :1327-1346
                L.tags.add("reply with last_validated_index")
                lvi = max(L.applied, prev + k)
                reply(L, leader, L.term, lvi + 1, lvi, UNDEF if srv_fetch_term(L, lvi) is None else
                      srv_fetch_term(L, lvi), 1)
            return
        fst = prev + 1 + k                                              # [{FstIdx, _, _} | _] :1348-1371
        if fst < L.applied:
            L.tags.add("fatal: write below applied")
            return set_fatal(L, abi.FATAL_ASSERT)
        if fst > L.last + 1 or (L.first > L.last and fst != L.last + 1):
            L.tags.add("fatal: write integrity")
            return set_fatal(L, abi.FATAL_WRITE_INTEGRITY)
        L.commit = lc
        if fst <= L.last:
            t = fetch_term(L, fst - 1)
            truncate(L, fst - 1, t if t is not None else (L.snap[1] if L.snap else 0))
        ev, i = 0, fst
        while i <= prev + len(terms):                                   # at most two term pieces
            t, j = terms[i - prev - 1], i
            while j + 1 <= prev + len(terms) and terms[j + 1 - prev - 1] == t:
                j += 1
            ev += append(L, j - i + 1, t)
            note(L, abi.NOTE_WAL_APPEND, i, j, t)
            i = j + 1
        if ev:
            L.tags.add("AppendEntries evicts %s" % ("twice" if ev > 1 else "once"))
        apply_to(L, L.commit)
        return
    if r == "missing":                                                  # :1373-1387
        aer_reply(L, e["term"], False)
        L.role = abi.AWAIT_CONDITION
        return
    la = L.applied                                                      # term_mismatch :1388-1413, :3587-3595
    lat = srv_fetch_term(L, la)
    if lat is None:
        L.tags.add("fatal: mismatch with applied unknown")
        return set_fatal(L, abi.FATAL_ASSERT)
    reply(L, leader, e["term"], la + 1, la, lat, 0)
    L.role = abi.AWAIT_CONDITION


def agreed_commit(indexes):
    return sorted(indexes, reverse=True)[len(indexes) // 2]


def evaluate_quorum(L):
    """evaluate_quorum/2 (:3606-3630) with the §5.4.2 gate"""
    cand = agreed_commit([L.lw[0]] + [L.peers[p][1] for p in range(L.m) if p != L.me])
    if srv_fetch_term(L, cand) == L.term:
        L.commit = cand


def make_aer(L, s, prev, pt, num):
    """make_append_entries_rpc/6 (:2401-2418): the batch ends at min(last, prev + num), is cut after 65535 entries and
    after the end of its second term run (contract, DESIGN §2 item 2); returns the peer's new next_index"""
    frm, to = prev + 1, min(L.last, prev + num)
    if to >= frm and to - frm >= 0xFFFF:
        to = frm + 0xFFFE
    n = n1 = d = e = 0
    if to >= frm and fetch_term(L, frm) is not None:
        d = fetch_term(L, frm)
        i = frm
        while i <= to and fetch_term(L, i) == d:
            i += 1
        if i <= to:
            e, j = fetch_term(L, i), i
            while j <= to and fetch_term(L, j) == e:
                j += 1
            n1 = i - frm
            if j - 1 < to:
                L.tags.add("AppendEntries cut after its second run")
            to = j - 1
        n = to - frm + 1
        if n < L.last - prev and (not n1 and fetch_term(L, to + 1) == d or n1 and fetch_term(L, to + 1) == e):
            L.tags.add("AppendEntries cut by the batch size inside a run")
        L.tags.add("AppendEntries of two runs" if n1 else "AppendEntries of one run")
    else:
        to = min(frm - 1, L.last)
        L.tags.add("AppendEntries without entries")
    L.msgs.append((abi.EV_AER, s, L.term, prev, pt, L.commit, n, n1, d, e))
    return to + 1


def make_rpc_effect(L, s, nxt, num):
    """make_rpc_effect/5 (:2365-2399): -> (new next_index, snapshot sent)"""
    prev = nxt - 1
    pt = fetch_term(L, prev)
    if pt is not None:
        return make_aer(L, s, prev, pt, num), False
    if L.snap is None:
        L.tags.add("fatal: no snapshot")
        set_fatal(L, abi.FATAL_NO_SNAPSHOT)
        return nxt, False
    if prev == L.snap[0]:
        L.tags.add("AppendEntries from the snapshot")
        return make_aer(L, s, prev, L.snap[1], num), False
    if not prev < L.snap[0]:
        L.tags.add("fatal: next_index between snapshot and first_index")
        set_fatal(L, abi.FATAL_ASSERT)
        return nxt, False
    L.tags.add("snapshot sent")
    note(L, abi.NOTE_SEND_SNAPSHOT, s, L.snap[0])
    return L.snap[0], True


def pipeline_pass(L, max_pipe, max_batch):
    """make_pipelined_rpc_effects/3 (:2268-2329), every peer normal"""
    for s in range(L.m):
        if s == L.me:
            continue
        nx, mt, cs = L.peers[s]
        if not (nx < L.last + 1 or cs < L.commit):
            continue
        inflight = nx - mt - 1
        if not inflight < max_pipe:
            L.tags.add("peer at the pipeline limit")
            continue
        nn, _snap = make_rpc_effect(L, s, nx, max(1, min(max_pipe - inflight, max_batch)))
        if L.fatal:
            return
        if not nn >= nx:
            return set_fatal(L, abi.FATAL_ASSERT)
        L.peers[s][0], L.peers[s][2] = nn, L.commit


def step_event(L, e, cfg):
    """one event through the member; cfg: (pure, max_pipeline_count, max_aer_batch)"""
    pure, max_pipe, max_batch = cfg
    if L.fatal:
        return
    if e["type"] == abi.EV_AER:
        return follower_aer(L, e)
    if e["type"] == abi.EV_WRITTEN:
        before = L.lw
        written(L, e["term"], e["a"], e["b"])
        if L.role == abi.FOLLOWER and L.lw != before and L.leader != NO:   # :1441-1458
            aer_reply(L, L.term, True)
        elif L.role == abi.LEADER:                                      # :730-735
            evaluate_quorum(L)
            if not pure:
                pipeline_pass(L, max_pipe, max_batch)
        return
    if e["type"] == abi.EV_COMMAND:                                     # :644-729
        frm = L.last + 1
        ev = append(L, e["n"], L.term)
        if ev:
            L.tags.add("command evicts")
        note(L, abi.NOTE_WAL_APPEND, frm, frm + e["n"] - 1, L.term)
        return pipeline_pass(L, max_pipe, max_batch)
    if e["type"] == abi.EV_PIPELINE_RPCS:                               # :784-792
        return pipeline_pass(L, max_pipe, max_batch)
    if e["type"] == abi.EV_AER_REPLY:                                   # :522-561, then the chased pass
        p = L.peers[e["from"]]
        p[0], p[1] = max(p[0], e["a"]), max(p[1], e["b"])
        evaluate_quorum(L)
        if not pure:
            pipeline_pass(L, max_pipe, max_batch)
        return
    raise AssertionError(e)


def hot_event(L, e):
    """The hot kernel's fast paths (raft_logic.cuh, the end of the file) take: a follower's same-term append or
    empty AppendEntries at last_index, a written event ending inside the last run, a leader's command and its
    successful replies; anything else stalls the row to the general kernel."""
    nonempty = L.first <= L.last
    if L.fatal:
        return True
    lrs = L.runs()[-1][0] if nonempty else None
    if e["type"] == abi.EV_AER:
        if L.role != abi.FOLLOWER or not nonempty or e["term"] != L.term or e["n1"]:
            return False
        if e["prev"] != L.last or e["pt"] != L.last_term:
            return False
        return not e["terms"] or (e["terms"][0] == L.last_term and L.last + 1 >= L.applied)
    if e["type"] == abi.EV_WRITTEN:
        return nonempty and e["term"] == L.last_term and lrs <= e["b"] <= L.last
    if e["type"] == abi.EV_COMMAND:
        return L.role == abi.LEADER and nonempty and e["n"] > 0
    if e["type"] == abi.EV_AER_REPLY:
        return L.role == abi.LEADER and e["term"] == L.term and e["from"] < L.m
    return False


# ---- the cases ------------------------------------------------------------------------------------------------------
def ev_dict(type_, **kw):
    d = dict(type=type_, prev=0, pt=0, terms=[], n1=0, term=0, a=0, b=0, n=0, commit=0)
    d.update(kw)
    if type_ == abi.EV_AER:
        t = d["terms"]
        d["n1"] = next((k for k in range(len(t)) if t[k] != t[0]), 0)
    return d


def to_event(row, e, m):
    t = e["type"]
    if t == abi.EV_AER:
        return abi.ev_aer(row, e["from"], e["term"], e["prev"], e["pt"], e["commit"], e["terms"])
    if t == abi.EV_WRITTEN:
        return abi.ev_written(row, e["term"], e["a"], e["b"])
    if t == abi.EV_COMMAND:
        return abi.ev_command(row, e["n"])
    if t == abi.EV_AER_REPLY:
        return abi.ev_aer_reply(row, e["from"], e["term"], True, e["a"], e["b"], 0)
    x = abi.ev_simple(row, abi.EV_PIPELINE_RPCS)
    x.flags = abi.EVF_INFO
    return x


class Case:
    def __init__(self, log, events, desc):
        self.log, self.events, self.desc = log, events, desc


def view(rng, m, me, role, nr, snap_mode, leader_ahead=None):
    """A member of nr term runs of 1, 2 or several entries; snap_mode: None, "adjacent" (just below first_index) or
    "gap" (further below, as after an eviction)."""
    if nr == 0:
        snap_mode = snap_mode or "adjacent"
    t = rng.choice([1, 2])
    si = rng.choice([3, 6]) if snap_mode else None
    first = (si + 1 + (2 if snap_mode == "gap" else 0)) if snap_mode else rng.choice([1, 2, 5])
    entries, i = [], first
    for k in range(nr):
        t += rng.choice([1, 1, 2]) if k else 0
        for _ in range(rng.choice([1, 1, 2, 2, 3, 5])):
            entries.append((i, t))
            i += 1
    snap = (si, max(0, t - nr - rng.choice([0, 1]))) if snap_mode else None
    last_t = entries[-1][1] if entries else snap[1]
    term = last_t + (2 if role != abi.LEADER else (leader_ahead if leader_ahead is not None else rng.choice([0, 1])))
    lo = si if snap_mode else 0
    last = entries[-1][0] if entries else first - 1
    marks = sorted({x for s in ([lo, last] + [j for j, _ in entries[:1]] +
                                [j for k, (j, tt) in enumerate(entries) if k and entries[k - 1][1] != tt])
                    for x in (s - 1, s, s + 1) if lo <= x <= last})
    lw = rng.choice(marks)
    applied = rng.choice([x for x in marks if x <= last])
    commit = rng.choice([x for x in marks if applied <= x <= last])
    leader = me if role == abi.LEADER else rng.choice([p for p in range(m) if p != me])
    L = Log(m, me, role, term, entries, snap, lw, applied, commit, leader, first)
    if role == abi.LEADER:                      # every peer caught up; leader_cases move them
        L.peers = [[last + 1, last, commit] for _ in range(m)]
    return L


def positions(L):
    """prev_idx positions: every run's start - 1, start, start + 1 and end; last_index and last_index + 1;
    first_index - 1; the snapshot index"""
    out = set()
    for s, e, _ in L.spans():
        out |= {s - 1, s, min(s + 1, e), e}
    out |= {L.last, L.last + 1, L.first - 1}
    if L.snap:
        out.add(L.snap[0])
    return sorted(x for x in out if x >= 0)


def entries_for(rng, L, p, kind):
    """entry terms after prev p: kind "empty", "one" (one run) or a two-run batch whose first piece matches up to
    "first" (no entry), "middle" (inside a local run), "boundary" (a local run's end) or "never" (throughout)"""
    local = fetch_term(L, p + 1)
    span = next(((s, e) for s, e, _ in L.spans() if s <= p + 1 <= e), None)
    base = srv_fetch_term(L, p)
    base = base if base is not None else L.last_term
    if kind == "empty":
        return []
    if kind == "one":
        t = rng.choice([x for x in (local, L.last_term, L.term) if x is not None and x >= base] or [L.term])
        return [t] * rng.choice([1, 2, 4])
    if kind == "middle" and span and span[1] > p + 1:
        n1 = rng.randint(1, span[1] - p - 1)
        return [local] * n1 + [local + 1] * rng.choice([1, 2])
    if kind in ("boundary", "never") and span:
        n1 = span[1] - p
        nxt = fetch_term(L, span[1] + 1)
        if kind == "never" and nxt is not None:
            ln = next(e - s + 1 for s, e, _ in L.spans() if s == span[1] + 1)
            return [local] * n1 + [nxt] * rng.randint(1, min(3, ln))
        return [local] * n1 + [(nxt + 1) if nxt is not None else L.term] * rng.choice([1, 3])
    d = max(base, local if local is not None else 0) + 1
    return [d] * rng.choice([1, 2]) + [d + 1] * rng.choice([1, 2])


def aer_event(L, p, pt, terms):
    return ev_dict(abi.EV_AER, prev=p, pt=pt, terms=terms, term=L.term, commit=min(L.commit + 1, p + len(terms)),
                   **{"from": L.leader})


def follower_cases(rng, m):
    out = []
    me = lambda: rng.randrange(m)
    for nr in range(0, abi.RA_MAX_RUNS + 1):
        for snap_mode in ([None, "adjacent", "gap"] if nr else ["adjacent", "gap"]):
            L = view(rng, m, me(), abi.FOLLOWER, nr, snap_mode)
            for p in positions(L):
                right = srv_fetch_term(L, p)
                for kind in rng.sample(["empty", "one", "first", "middle", "boundary", "never"], 2):
                    x = copy.deepcopy(L)
                    x.me = me()
                    x.leader = rng.choice([q for q in range(m) if q != x.me])
                    wrong = right is None or rng.random() < 0.2 or (L.snap and p == L.snap[0] and kind == "empty")
                    pt = (right + 1 if right is not None else L.last_term) if wrong else right
                    out.append(Case(x, [aer_event(x, p, pt, entries_for(rng, x, p, kind))],
                                    "follower %d runs snapshot %s: AppendEntries prev %d term %d, %s" %
                                    (nr, L.snap, p, pt, kind)))
        # conflicts k runs deep, the 9th run, two evictions, truncations onto the snapshot
        L = view(rng, m, me(), abi.FOLLOWER, nr, rng.choice([None, "adjacent"]) if nr else "adjacent")
        sp = L.spans()
        if nr == abi.RA_MAX_RUNS:
            for k in range(1, nr):
                s, e, t = sp[nr - 1 - k]
                terms = [L.term] * rng.choice([1, 2]) if k % 2 else [t + 1, L.term]
                out.append(Case(copy.deepcopy(L), [aer_event(L, e, t, terms)], "conflict %d runs deep" % k))
        if nr >= abi.RA_MAX_RUNS - 1:
            out.append(Case(copy.deepcopy(L), [aer_event(L, L.last, L.last_term, [L.term] * 2)], "9th run"))
            out.append(Case(copy.deepcopy(L), [aer_event(L, L.last, L.last_term, [L.term - 1, L.term])],
                            "two new runs on %d" % nr))
        if nr == 0:                             # an empty view whose last_index is above the snapshot
            x = view(rng, m, me(), abi.FOLLOWER, 0, "gap")
            x.applied = x.commit = x.snap[0]
            out.append(Case(x, [aer_event(x, x.snap[0], x.snap[1], [x.term])], "write above an empty view"))
        if L.snap:
            L.applied = L.commit = L.snap[0]
            for terms in ([], [L.term] * 2, [L.term - 1, L.term]):
                out.append(Case(copy.deepcopy(L), [aer_event(L, L.snap[0], L.snap[1], terms)],
                                "onto the snapshot with %d entries" % len(terms)))
    return out


def written_cases(rng, m, roles):
    out = []
    for nr in range(0, abi.RA_MAX_RUNS + 1):
        for role in roles:
            L = view(rng, m, rng.randrange(m), role, nr, rng.choice([None, "adjacent", "gap"]) if nr else "gap")
            sp = L.spans()
            ranges = []
            if sp:
                s, e, t = sp[-1]
                to = rng.randint(s, e)
                ranges += [(t, max(0, to - rng.randint(0, 3)), to), (t, e, e)]            # ends in the last run
                k = rng.randrange(len(sp))
                s, e, t = sp[k]
                to = rng.randint(s, e)
                ranges.append((t, max(0, s - 2), to))                                     # an earlier run: at to
                if k:
                    ranges.append((sp[k - 1][2], max(0, sp[k - 1][1] - rng.randint(0, 2)), to))   # lower down
                ranges.append((L.term + 1, max(0, to - 4), to))                           # nowhere
                ranges.append((L.last_term, L.last - 1, L.last + rng.choice([1, 2])))     # above last_index
            if L.snap:
                ranges.append((L.snap[1], max(0, L.snap[0] - 1), L.snap[0] + rng.choice([0, 1, 2])))
                ranges.append((L.last_term, L.snap[0] - 2, L.snap[0] - 1))
            for term, a, b in ranges:
                if a <= b:
                    x = copy.deepcopy(L)
                    out.append(Case(x, [ev_dict(abi.EV_WRITTEN, term=term, a=a, b=b)],
                                    "%s %d runs snapshot %s: written %d %d..%d" %
                                    (abi.ROLE_NAMES[role], nr, L.snap, term, a, b)))
    return out


def sequence_cases(rng, m):
    """up to 4 events in one row's step"""
    out = []
    for nr in range(1, abi.RA_MAX_RUNS + 1):
        L = view(rng, m, rng.randrange(m), abi.FOLLOWER, nr, rng.choice([None, "adjacent"]))
        L.applied = min(L.applied, L.first)
        sp = L.spans()
        # all in the hot kernel: same-term appends at last_index and written events ending in the last run
        x = copy.deepcopy(L)
        a = rng.choice([1, 2])
        evs = [aer_event(x, x.last, x.last_term, [x.last_term] * a),
               ev_dict(abi.EV_WRITTEN, term=x.last_term, a=x.last + 1, b=x.last + a),
               aer_event(x, x.last + a, x.last_term, [x.last_term]),
               ev_dict(abi.EV_WRITTEN, term=x.last_term, a=x.last + 1, b=x.last + a + 1)]
        for k, e in enumerate(evs):
            if e["type"] == abi.EV_AER:
                e["commit"] = x.commit
        out.append(Case(x, evs, "%d runs: same-term appends and written events" % nr))
        # a truncating AppendEntries, a written event for the old term, a same-term append at the new last index,
        # a written event for the new range
        if nr >= 2:
            k = rng.randrange(max(0, nr - 3), nr - 1)
            s, e, t = sp[k]
            p = rng.randint(max(s, L.applied), e) if max(s, L.applied) <= e else e
            x = copy.deepcopy(L)
            new = x.term
            evs = [aer_event(x, p, fetch_term(x, p), [new] * 2),
                   ev_dict(abi.EV_WRITTEN, term=x.last_term, a=p + 1, b=x.last),
                   ev_dict(abi.EV_AER, prev=p + 2, pt=new, terms=[new], term=x.term, commit=x.commit,
                           **{"from": x.leader}),
                   ev_dict(abi.EV_WRITTEN, term=new, a=p + 1, b=p + 3)]
            out.append(Case(x, evs, "%d runs: truncate at %d, written old, append, written new" % (nr, p)))
    return out


def leader_cases(rng, m):
    out = []
    for nr in range(1, abi.RA_MAX_RUNS + 1):
        for kind in ("pipeline", "reply", "command", "snapshot"):
            L = view(rng, m, rng.randrange(m), abi.LEADER, nr, rng.choice([None, "adjacent", "gap"]))
            pos = [p for p in positions(L) + ([L.snap[0] - 1, 0] if L.snap else []) if 0 <= p <= L.last]
            safe = [p for p in pos if fetch_term(L, p) is not None or (L.snap and p <= L.snap[0])]
            for s in range(m):
                nx = (rng.choice(safe if rng.random() < 0.9 else pos) + 1) if s != L.me else L.last + 1
                L.peers[s] = [nx, max(0, nx - 1 - rng.choice([0, 0, 1, 3, 6])), L.commit]
            if kind == "snapshot" and L.snap:                   # peers at, just below and far below the snapshot
                for k, s in enumerate(p for p in range(m) if p != L.me):
                    nx = [L.snap[0] + 1, L.snap[0], 1][k % 3]
                    L.peers[s] = [nx, nx - 1, L.commit]
            L.lw = (L.last, L.last_term) if rng.random() < 0.5 else L.lw
            others = [p for p in range(m) if p != L.me]
            if kind == "command":
                e = ev_dict(abi.EV_COMMAND, n=rng.choice([1, 2, 3]))
            elif kind == "reply" and others:
                f = rng.choice(others)
                e = ev_dict(abi.EV_AER_REPLY, term=L.term, a=L.peers[f][0], b=L.peers[f][0] - 1, **{"from": f})
            else:
                e = ev_dict(abi.EV_PIPELINE_RPCS)
            out.append(Case(L, [e], "leader %d runs snapshot %s next %s: %s" %
                            (nr, L.snap, [p[0] for p in L.peers], kind)))
    # a command on 8 runs whose last run is an earlier term: the new run evicts the oldest in the hot kernel, and
    # peers whose next_index sat in it fall below first_index
    for k, snap_mode in enumerate((None, None, "adjacent", "adjacent")):
        L = view(rng, m, rng.randrange(m), abi.LEADER, abi.RA_MAX_RUNS, snap_mode, leader_ahead=1)
        s0, e0, _ = L.spans()[0]
        for s in range(m):
            nx = [s0 + 1, e0 + 1, L.last + 1][(s + k) % 3] if s != L.me else L.last + 1
            L.peers[s] = [nx, nx - 1, L.commit]
        out.append(Case(L, [ev_dict(abi.EV_COMMAND, n=rng.choice([1, 2]))],
                        "leader 8 runs snapshot %s, command evicts" % (L.snap,)))
    return out


@functools.lru_cache(maxsize=None)
def table(m):
    """Every case of M members: case i is group i, its member at the case's slot is row slot * G + i."""
    rng = random.Random(3000 + m)
    cases = (follower_cases(rng, m) + written_cases(rng, m, [abi.FOLLOWER, abi.LEADER]) + sequence_cases(rng, m)
             if m >= 2 else written_cases(rng, m, [abi.LEADER])) + leader_cases(rng, m)
    return len(cases), cases


# ---- one run --------------------------------------------------------------------------------------------------------
def expect(cases, cfg):
    """the model after step 1 of every case, and the (role, event type) each case stalls on (None: stays hot)"""
    out, stalls = [], []
    for c in cases:
        L = copy.deepcopy(c.log)
        stall = None
        for e in c.events:
            if stall is None and not hot_event(L, e):
                stall = (L.role, e["type"])
            step_event(L, e, cfg)
        out.append(L)
        stalls.append(stall)
    return out, stalls


def wal_notes(notes):
    """WAL_APPEND ranges with contiguous same-term neighbours merged (the engine merges a note only into the one
    just before it)"""
    out = []
    for n in notes:
        if n[0] == abi.NOTE_WAL_APPEND and out and out[-1][0] == n[0] and out[-1][3] == n[3] and out[-1][2] + 1 == n[1]:
            out[-1] = (n[0], out[-1][1], n[2], n[3])
        else:
            out.append(tuple(n))
    return out


def _un(v, d):
    return v if v == UNDEF else v - d


def row_view(s, di, dt, leader):
    """what the rule fixes in a read-back row, moved back by (di, dt)"""
    runs = [(s.run_start[k] - di, s.run_term[k] - dt) for k in range(s.n_runs)]
    v = dict(first_index=s.first_index - di, last_index=s.last_index - di, last_term=_un(s.last_term, dt), runs=runs,
             last_written=(s.last_written_index - di, _un(s.last_written_term, dt)), role=s.role,
             fatal=bool(s.flags & 4), commit_index=s.commit_index - di)
    if leader:
        v["peers"] = [(s.peers[p].next_index - di, s.peers[p].commit_index_sent - di) for p in range(s.n_members)]
    return v


def model_view(L, leader):
    v = dict(first_index=L.first, last_index=L.last, last_term=L.last_term, runs=L.runs(), last_written=L.lw,
             role=L.role, fatal=bool(L.fatal), commit_index=L.commit)
    if leader:
        v["peers"] = [(p[0], p[2]) for p in L.peers]
    return v


def by_row(xs):
    out = {}
    for x in xs:
        out.setdefault(x.row, []).append(x)
    return out


def note_view(notes, di, dt):
    out, code = [], 0
    for n in notes:
        if n.type == abi.NOTE_WAL_APPEND:
            out.append((n.type, n.a - di, n.b - di, n.c - dt))
        elif n.type == abi.NOTE_TRUNCATE:
            out.append((n.type, n.a - di, _un(n.b, dt)))
        elif n.type == abi.NOTE_SEND_SNAPSHOT:
            out.append((n.type, n.a, n.b - di))
        elif n.type == abi.NOTE_STATUS and n.aux & abi.ST_FATAL:
            code = n.c & 0xff
    return wal_notes(out), code


def msg_view(msgs, G, di, dt):
    out = []
    for x in msgs:
        if x.type == abi.EV_AER_REPLY:
            out.append((x.type, x.row // G, x.term - dt, x.a - di, x.b - di, _un(x.c, dt), x.d))
        elif x.type == abi.EV_AER:
            out.append((x.type, x.row // G, x.term - dt, x.a - di, x.b - dt, x.c - di, x.n, x.n1,
                        x.d - dt if x.n else x.d, x.e - dt if x.n1 else x.e))
    return out


def _check_rule(b, m, setting, G, cases, want, outs, records, di, dt):
    rows = b.read_rows([c.log.me * G + g for g, c in enumerate(cases)])
    msgs, notes = outs
    notes, sent = by_row(notes), {}
    for x in msgs:
        if not x.flags & abi.EVF_NEXT_EVENT:
            sent.setdefault((x.row % G, x.from_slot), []).append(x)
    bad = []
    for g, (c, L, s) in enumerate(zip(cases, want, rows)):
        leader = c.log.role == abi.LEADER
        got, exp = row_view(s, di, dt, leader and not L.fatal), model_view(L, leader and not L.fatal)
        if not L.fatal:
            got["notes"], code = note_view(notes.get(s.row, []), di, dt)
            exp["notes"] = wal_notes(L.notes)
            if records:
                got["msgs"] = msg_view(sent.get((g, c.log.me), []), G, di, dt)
                exp["msgs"] = list(L.msgs)
        else:
            _, code = note_view(notes.get(s.row, []), di, dt)
            got["fatal code"], exp["fatal code"] = code, L.fatal
        if got != exp:
            diff = {k: (exp[k], got.get(k)) for k in exp if exp[k] != got.get(k)}
            bad.append("case %d %s: %s (rule, got)" % (g, c.desc, diff))
    assert not bad, "M=%d %s %s: %d of %d cases differ from the rule, e.g.\n  %s" % (
        m, setting, b.name, len(bad), len(cases), "\n  ".join(bad[:6]))


def _check_written(b, m, setting, G, cases, want, di, dt):
    """after the second step: the log view of every row, read by a fresh launch"""
    rows = b.read_rows([c.log.me * G + g for g, c in enumerate(cases)])
    bad = []
    for g, (c, L, s) in enumerate(zip(cases, want, rows)):
        got, exp = row_view(s, di, dt, False), model_view(L, False)
        got = {k: got[k] for k in ("first_index", "last_index", "last_term", "runs", "last_written")}
        exp = {k: exp[k] for k in got}
        if got != exp:
            bad.append("case %d %s: %s (rule, got)" % (g, c.desc, {k: (exp[k], got[k]) for k in exp
                                                                     if exp[k] != got[k]}))
    assert not bad, "M=%d %s %s, step 2: %d of %d cases differ from the rule, e.g.\n  %s" % (
        m, setting, b.name, len(bad), len(cases), "\n  ".join(bad[:6]))


REACHED = {
    "all": ["view of %d runs" % k for k in range(abi.RA_MAX_RUNS + 1)] + [
        "written matches at to", "written matches lower down", "written matches nowhere",
        "written at or below the snapshot", "command evicts"],
    "peers": ["AppendEntries of one run", "AppendEntries of two runs", "AppendEntries cut after its second run",
              "AppendEntries without entries", "AppendEntries from the snapshot", "snapshot sent",
              "fatal: no snapshot"],
    "follower": ["prev entry ok", "prev entry missing", "prev entry term_mismatch", "validated reply",
                 "reply with last_validated_index", "set_last_index at the snapshot",
                 "fatal: write below applied", "fatal: write integrity", "truncation empties the view",
                 "drop_existing stops at the first entry", "drop_existing stops inside a local run",
                 "drop_existing stops at a run boundary", "drop_existing never stops",
                 "AppendEntries evicts once", "AppendEntries evicts twice"] +
                ["conflict %d runs deep" % k for k in range(1, abi.RA_MAX_RUNS)] +
                ["prev at %s" % w for w in ("a run's start - 1", "a run's start", "a run's start + 1", "a run's end",
                                            "last_index", "last_index + 1", "first_index - 1 on the snapshot",
                                            "first_index - 1 without a snapshot there")],
    "batch": ["AppendEntries cut by the batch size inside a run", "peer at the pipeline limit"],
}


def _coverage(m, cases, want, cfg):
    """the table reaches what it is for (every tag is set by the restated rule, which the backends matched)"""
    seen = set()
    for c, L in zip(cases, want):
        seen |= L.tags
        seen.add("view of %d runs" % len(c.log.runs()))
        for e in c.events:
            if e["type"] == abi.EV_AER and e is c.events[0]:
                p, x = e["prev"], c.log
                for s, end, _ in x.spans():
                    for off, w in ((-1, "a run's start - 1"), (0, "a run's start"), (1, "a run's start + 1")):
                        if p == s + off:
                            seen.add("prev at " + w)
                    if p == end:
                        seen.add("prev at a run's end")
                seen |= {"prev at last_index"} if p == x.last else set()
                seen |= {"prev at last_index + 1"} if p == x.last + 1 else set()
                if p == x.first - 1:
                    seen.add("prev at first_index - 1 " + ("on the snapshot" if x.snap and x.snap[0] == p else
                                                           "without a snapshot there"))
    want_tags = set(REACHED["all"])
    if m >= 2:
        want_tags |= set(REACHED["follower"]) | set(REACHED["peers"])
    if cfg[1] < DEFAULT_PIPE:
        want_tags |= set(REACHED["batch"]) if m >= 2 else set()
        want_tags.discard("AppendEntries cut after its second run")     # (three entries seldom span three runs)
    assert want_tags <= seen, "M=%d: the table does not reach %s" % (m, sorted(want_tags - seen))
    return seen


def run_table(backend, setting, m, monkeypatch):
    kw, wide, shift, _ = SETTINGS[setting]
    pure = kw.get("pure", False)
    cfg = (pure, kw.get("max_pipeline_count", DEFAULT_PIPE), kw.get("max_aer_batch", DEFAULT_BATCH))
    records = not kw.get("route_on_device", False) or pure          # host and pure: the records come back
    monkeypatch.setenv("RA_STEP_WIDE", wide)
    G, cases = table(m)
    di, dt = shift or (0, 0)
    rows, events = [], []
    for g, c in enumerate(cases):
        r = c.log.row(c.log.me * G + g)
        if shift:
            shift_state(r, di, dt, m)
        rows.append(r)
        for e in c.events:
            x = to_event(r.row, e, m)
            if shift:
                shift_event(x, di, dt)
            events.append(x)
    want, stalls = expect(cases, cfg)
    o = Oracle(G, m, **kw)
    bs = [o] if backend == "oracle" else [o, make_backend(backend, G, m, **kw)]
    Emu.narrow_stats()
    outs = []
    for b in bs:
        b.load_rows(rows)
        b.load_query_state([])
        outs.append(b.step([clone(e) for e in events]))
    ns = Emu.narrow_stats()
    b = bs[-1]
    _check_rule(b, m, setting, G, cases, want, outs[-1], records, di, dt)
    if backend != "oracle":
        compare(observe(o, m, outs[0]), observe(b, m, outs[1]), "M=%d %s %s" % (m, setting, backend), events, o)
        if not pure and not shift:              # which kernel took each case
            hist = b.stall_histogram()
            exp = Counter(s for s in stalls if s is not None)
            assert hist == dict(exp), "M=%d %s: general-kernel events by (role, type): expected %s, got %s" % (
                m, setting, dict(exp), hist)
        if backend == "emu" and m == 5 and not pure and wide == "0":    # the emulation's 32-bit pass: M = 5
            assert Emu.underfetched() == 0
            if shift:                                                   # every row refused to the general kernel
                assert ns["rows_narrow"] == 0 and ns["rows_wide"] >= len(cases), ns
            else:
                assert ns["rows_narrow"] >= len(cases) and ns["rows_wide"] == 0, ns
    # step 2: the host's own written event for each WAL_APPEND note of step 1
    w2, ev2, notes1 = [], [], by_row(outs[0][1])
    for g, (c, L) in enumerate(zip(cases, want)):
        L = copy.deepcopy(L)
        row = c.log.me * G + g
        if not L.fatal:
            for n in notes1.get(row, []):
                if n.type == abi.NOTE_WAL_APPEND:
                    ev2.append(abi.ev_written(row, n.c, n.a, n.b))
                    step_event(L, ev_dict(abi.EV_WRITTEN, term=n.c - dt, a=n.a - di, b=n.b - di), cfg)
        w2.append(L)
    outs2 = [x.step([clone(e) for e in ev2]) for x in bs]
    _check_written(b, m, setting, G, cases, w2, di, dt)
    if backend == "oracle":
        if not shift:
            _coverage(m, cases, want, cfg)
        return
    compare(observe(o, m, outs2[0]), observe(b, m, outs2[1]), "M=%d %s %s step 2" % (m, setting, backend), ev2, o)


@pytest.mark.parametrize("m", MEMBERS)
@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("backend", ["oracle", "emu"])
def test_log_view_table(backend, setting, m, monkeypatch):
    run_table(backend, setting, m, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("m", MEMBERS)
@pytest.mark.parametrize("setting", list(SETTINGS))
def test_log_view_table_engine(setting, m, monkeypatch):
    run_table("engine", setting, m, monkeypatch)
