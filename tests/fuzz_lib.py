"""TEST INFRASTRUCTURE: the differential fuzz of the step logic, shared by the fuzz tests.

Generators of random but well-formed member states and events, the rounds of the kernel fuzz (fresh states loaded
into most rows, an event batch drawn from the oracle's state of the others) and `fuzz_rounds`, which steps the oracle
and any number of backends on copies of each batch and compares them after every step: RPC records and notes in order,
every row as raw ra_row_state bytes, counters and query state.
"""
import ctypes as C
import random
import socket

from emu_lib import Emu
from oracle_lib import Oracle
from ra_b200 import abi
from ra_suite import clone

ROLES = [abi.FOLLOWER, abi.CANDIDATE, abi.PRE_VOTE, abi.LEADER, abi.AWAIT_CONDITION]

MEMBERS = [1, 2, 3, 4, 5, 6, 7, 8]
MODES = ["pure", "chased", "routed", "flood"]
WIDTHS = ["0", "1"]                          # RA_STEP_WIDE: the 32-bit hot kernel / the 64-bit one
FAULTS = (20, 50, 30, 16)                    # drop, withhold, partition permille, partition steps
FLOOD_CMDS, PERMILLE = 300, 15
RELOAD, WIDE_ROWS = 0.7, 0.05               # per round and row: fresh state / moved to the narrow limit

# small note budgets (cfg.note_cap, RA_NOTE_RESERVE + 2 ..) per M, in the order of MODES: every budget meets several
# modes; the larger ones go where more peers make more notes, so that each case still runs into its budget
NOTE_CAPS = {1: [6, 6, 6, 6], 2: [6, 7, 6, 7], 3: [6, 7, 6, 7], 4: [7, 6, 7, 6], 5: [9, 6, 9, 7], 6: [9, 6, 8, 7],
             7: [12, 6, 7, 9], 8: [9, 12, 6, 9]}


def kw(mode, note_cap=0):
    return dict(pure=(mode == "pure"), route_on_device=mode in ("routed", "flood"), max_aer_batch=512, note_cap=note_cap)


# ---- generators -----------------------------------------------------------------------------------------------------
def random_state(rng: random.Random, row: int, n_groups: int, m: int, role: int, rich: bool = False) -> abi.RaRowState:
    """rich = False draws exactly what the (state, event) pair fuzz always drew (its seeds stay meaningful); rich =
    True adds up to 8 term runs, the pending-pipeline flag, machine versions, promotable / non-voter / unknown
    membership and all five peer statuses."""
    s = abi.empty_row(row, n_groups, m)
    me = s.self_slot
    term = rng.randint(1, 12 if rich else 6)
    # log: maybe a snapshot, then 0..4 (rich: 0..8) runs of non-decreasing terms <= term
    has_snap = rng.random() < 0.3
    snap_idx = rng.randint(1, 6) if has_snap else 0
    snap_term = rng.randint(1, term) if has_snap else 0
    entries = []
    idx = snap_idx + 1 if has_snap else 0
    t = snap_term if has_snap else 0
    n_runs = rng.randint(0 if has_snap else 1, abi.RA_MAX_RUNS if rich else 4)
    for _ in range(n_runs):
        t = rng.randint(t, term) if entries or has_snap else (0 if rng.random() < 0.6 else rng.randint(0, term))
        for _ in range(rng.randint(1, 4)):
            entries.append((idx, t))
            idx += 1
        if t >= term:
            break
    abi.set_log(s, entries, snapshot=(snap_idx, snap_term) if has_snap else None)
    last = s.last_index
    lo = snap_idx if has_snap else 0

    def term_at(i):
        for (j, tt) in entries:
            if j == i:
                return tt
        return snap_term if (has_snap and i == snap_idx) else None

    lw = rng.randint(lo, last)
    s.last_written_index, s.last_written_term = lw, term_at(lw) or 0
    s.commit_index = rng.randint(lo, last + (2 if role != abi.LEADER and rng.random() < 0.2 else 0))
    s.last_applied = rng.randint(lo, min(s.commit_index, last))
    s.current_term = max(term, s.last_term)
    s.role = role
    s.voted_for = rng.choice([abi.RA_NO_SLOT] + list(range(m)))
    s.leader_slot = me if role == abi.LEADER else rng.choice([abi.RA_NO_SLOT] + [p for p in range(m) if p != me])
    s.votes = rng.randint(0, m // 2) if role in (abi.CANDIDATE, abi.PRE_VOTE) else 0
    s.membership = abi.VOTER if rng.random() < 0.9 else (
        rng.choice([abi.PROMOTABLE, abi.NON_VOTER, abi.UNKNOWN]) if rich else abi.PROMOTABLE)
    s.pre_vote_token = rng.randint(1, 3)
    s.token_counter = s.pre_vote_token + rng.randint(0, 2)
    for p in range(m):
        pe = s.peers[p]
        pe.voter = 1 if (p == me and s.membership == abi.VOTER) or (p != me and rng.random() < 0.9) else 0
        pe.next_index = rng.randint(max(1, lo), last + 1)
        pe.match_index = rng.randint(0, pe.next_index - 1)
        pe.commit_index_sent = rng.randint(0, s.commit_index)
        pe.status = abi.PEER_NORMAL if rng.random() < 0.9 else rng.choice(
            [abi.PEER_SENDING_SNAPSHOT, abi.PEER_SNAPSHOT_BACKOFF, abi.PEER_SUSPENDED, abi.PEER_DISCONNECTED] if rich else
            [abi.PEER_SENDING_SNAPSHOT, abi.PEER_SUSPENDED, abi.PEER_DISCONNECTED])
    if role == abi.AWAIT_CONDITION:
        s.condition = 1                                  # follower catch-up (the condition on this path)
        s.flags |= 2
        s.cond_reply_term = s.current_term
        s.cond_reply_next_index = last + 1
        s.cond_reply_last_index = lw
        s.cond_reply_last_term = s.last_written_term
    if rich:
        if rng.random() < 0.15:
            s.flags |= 1                                 # a pipeline pass deferred from the step before
        if rng.random() < 0.3:
            s.machine_version, s.effective_machine_version = rng.randint(0, 3), rng.randint(0, 3)
    return s


def random_event(rng: random.Random, s: abi.RaRowState, m: int, rich: bool = False) -> abi.RaEvent:
    """rich = True adds AppendEntries of 255, 256 and 300 entries (one or two term runs), replies from unknown slots
    (9, 14, m) and commands of 256 and 1000 entries: records stored as 32-byte heads or 64-byte long records."""
    row, me, term, last = s.row, s.self_slot, s.current_term, s.last_index
    other = rng.choice([p for p in range(m) if p != me] or [me])
    t = max(0, term + rng.choice([-1, 0, 0, 0, 1]))
    near = lambda x: max(0, x + rng.choice([-2, -1, 0, 0, 0, 1, 2]))
    kinds = ["aer", "aer", "reply", "reply", "rv", "rvres", "pv", "pvres", "written", "cmd",
             "etmo", "ctmo", "tick", "pipe", "hb", "hbr", "cq"]
    kind = rng.choice(kinds + ["aer_long", "reply_unknown", "cmd_long"] if rich else kinds)
    if kind == "aer_long":
        prev = near(last)
        pt = rng.randint(0, t)
        n = rng.choice([255, 256, 300])
        t2 = rng.randint(pt, max(pt, t))
        k = rng.choice([n, rng.randint(1, n - 1)])          # one term run, or two split at k
        terms = [pt] * k + [t2] * (n - k)
        return abi.ev_aer(row, other, t, prev, pt, near(s.commit_index), terms)
    if kind == "reply_unknown":
        return abi.ev_aer_reply(row, rng.choice([9, 14, m]), t, rng.random() < 0.7, near(last + 1), near(last),
                                rng.randint(0, t))
    if kind == "cmd_long":
        return abi.ev_command(row, rng.choice([256, 1000]))
    if kind == "hb":
        return abi.ev_heartbeat_rpc(row, other, t, rng.randint(0, 4))
    if kind == "hbr":
        return abi.ev_heartbeat_reply(row, rng.choice([other, other, 7]), t, rng.randint(0, 4))
    if kind == "cq":
        return abi.ev_consistent_query(row)
    if kind == "aer":
        prev = near(last)
        pt = rng.randint(0, t)
        n = rng.choice([0, 0, 1, 2, 3])
        terms = sorted(rng.randint(pt, max(pt, t)) for _ in range(n))
        if len(set(terms)) > 2:
            terms = [terms[0]] * (n - 1) + [terms[-1]]
        return abi.ev_aer(row, other, t, prev, pt, near(s.commit_index), terms)
    if kind == "reply":
        li = near(last)
        return abi.ev_aer_reply(row, other, t, rng.random() < 0.7, near(last + 1), li, rng.randint(0, t))
    if kind == "rv":
        return abi.ev_request_vote(row, other, t, near(last), rng.randint(0, t))
    if kind == "rvres":
        return abi.ev_request_vote_result(row, t, rng.random() < 0.7, voter=other)
    if kind == "pv":
        return abi.ev_pre_vote(row, other, t, rng.randint(1, 5), near(last), rng.randint(0, t),
                               machine_version=rng.choice([0, 0, 1]))
    if kind == "pvres":
        return abi.ev_pre_vote_result(row, t, rng.choice([s.pre_vote_token, s.pre_vote_token + 1]),
                                      rng.random() < 0.7, voter=other)
    if kind == "written":
        a = near(s.last_written_index + 1)
        return abi.ev_written(row, rng.randint(max(0, term - 1), term), a, a + rng.randint(0, 3))
    if kind == "cmd":
        return abi.ev_command(row, rng.randint(1, 4))
    if kind == "etmo":
        return abi.ev_simple(row, abi.EV_ELECTION_TIMEOUT)
    if kind == "ctmo":
        return abi.ev_simple(row, abi.EV_AWAIT_COND_TIMEOUT)
    if kind == "tick":
        return abi.ev_simple(row, abi.EV_TICK)
    e = abi.ev_simple(row, abi.EV_PIPELINE_RPCS)
    e.flags = abi.EVF_INFO
    return e


def rich_event(rng, st, m):
    return random_event(rng, st, m, rich=True)


HOST_TYPES = {abi.EV_WRITTEN, abi.EV_COMMAND, abi.EV_ELECTION_TIMEOUT, abi.EV_AWAIT_COND_TIMEOUT, abi.EV_PIPELINE_RPCS,
              abi.EV_TICK, abi.EV_CONSISTENT_QUERY}


def host_event(rng, st, m):
    """The rich generator, redrawn until it gives a host-origin kind (written, cmd, cmd_long, etmo, ctmo, tick,
    pipe with EVF_INFO, cq)."""
    while True:
        e = rich_event(rng, st, m)
        if e.type in HOST_TYPES:
            return e


def random_query(rng, row, m):
    """consistent-query indexes of the row and its peers"""
    q = abi.RaQueryState(row=row, query_index=rng.randint(0, 4), agreed_index=rng.randint(0, 2))
    for p in range(m):
        q.peer_query_index[p] = rng.randint(0, 4)
    return q


def batch(rng, o, draw, density):
    """a batch drawn from the oracle's current state (no reload: calls may be in flight)"""
    evs = []
    for st in o.read_rows(range(o.n_rows)):
        if rng.random() < density:
            evs += [draw(rng, st, o.n_members) for _ in range(rng.randint(1, abi.RA_LOCAL_CAP))]
    return evs


# ---- the same corners, moved to where the hot kernel's 32-bit pass ends (tests/test_narrow_pass.py) ----------------
LIM = 1 << 30
OFFSETS = [(0, 0), (LIM - 9, 0), (0, LIM - 4), (LIM - 9, LIM - 4), (LIM + 5, 3), ((1 << 31) - 9, (1 << 31) - 4),
           ((1 << 32) - 9, (1 << 32) - 4), ((1 << 40) + 1, 1 << 35)]


# the settings of the crafted-case tables (tests/test_quorum_table.py, tests/test_log_view_table.py), by name:
# (engine config, RA_STEP_WIDE, (index shift, term shift) or None, leaders' replies stay in the hot kernel)
TABLE_SETTINGS = {
    "routed-32bit": (dict(route_on_device=True), "0", None, True),
    "routed-64bit": (dict(route_on_device=True), "1", None, True),
    "host": (dict(route_on_device=False), "0", None, True),
    "pure": (dict(pure=True), "0", None, False),
    "past2^30-32bit": (dict(route_on_device=True), "0", (LIM + 5, LIM + 3), False),
    "past2^30-64bit": (dict(route_on_device=True), "1", (LIM + 5, LIM + 3), True),
    "past2^32-32bit": (dict(route_on_device=True), "0", ((1 << 32) + 5, (1 << 32) + 3), False),
    "past2^32-64bit": (dict(route_on_device=True), "1", ((1 << 32) + 5, (1 << 32) + 3), True),
}


def shift_state(s: abi.RaRowState, di: int, dt: int, m: int) -> None:
    for f in ("commit_index", "last_applied", "first_index", "last_index", "last_written_index", "snapshot_index",
              "cond_reply_next_index", "cond_reply_last_index"):
        setattr(s, f, getattr(s, f) + di)
    for f in ("current_term", "last_term", "last_written_term", "snapshot_term", "cond_reply_term", "cond_reply_last_term"):
        setattr(s, f, getattr(s, f) + dt)
    for k in range(s.n_runs):
        s.run_start[k] += di
        s.run_term[k] += dt
    for p in range(m):
        s.peers[p].next_index += di
        s.peers[p].match_index += di
        s.peers[p].commit_index_sent += di


def shift_event(e: abi.RaEvent, di: int, dt: int) -> None:
    t = e.type
    if t == abi.EV_AER:
        e.term += dt; e.a += di; e.b += dt; e.c += di; e.d += dt; e.e += dt
    elif t == abi.EV_AER_REPLY:
        e.term += dt; e.a += di; e.b += di; e.c += dt
    elif t == abi.EV_REQUEST_VOTE or t == abi.EV_PRE_VOTE:
        e.term += dt; e.a += di; e.b += dt
    elif t in (abi.EV_REQUEST_VOTE_RES, abi.EV_PRE_VOTE_RES, abi.EV_HEARTBEAT_RPC, abi.EV_HEARTBEAT_REPLY):
        e.term += dt
    elif t == abi.EV_WRITTEN:
        e.term += dt; e.a += di; e.b += di


# ---- observation and comparison -------------------------------------------------------------------------------------
def observe(b, m, out=None):
    msgs, notes = out if out is not None else ([], [])
    q = b.read_query_state(range(b.n_rows))
    return dict(msgs=[x.key() for x in msgs], notes=[x.key() for x in notes], rows=b.rows_bytes(),
                counters=b.counters(), query=[x.key(m) for x in q])


def first_row(a, b):
    """the first row whose ra_row_state bytes differ between two rows_bytes() images, -1 if none"""
    sz = C.sizeof(abi.RaRowState)
    return next((i // sz for i in range(0, len(a), sz) if a[i:i + sz] != b[i:i + sz]), -1)


def same_keys(want, got, what, k):
    """Lists of record, note or query-state keys (each starting with its row) must be equal; the message names the
    first entry that differs and its row."""
    if got != want:
        i = next((i for i, (x, y) in enumerate(zip(want, got)) if x != y), min(len(want), len(got)))
        row = (want[i:i + 1] or got[i:i + 1])[0][0]
        raise AssertionError("%s: %s differ from #%d on (row %d): oracle %r, got %r (%d / %d)"
                             % (what, k, i, row, want[i:i + 1], got[i:i + 1], len(want), len(got)))


def compare(want, got, what, events, oracle):
    """First difference between the oracle's and a backend's observation, with the row's role and its events."""
    if got["rows"] != want["rows"]:
        r = first_row(want["rows"], got["rows"])
        role = oracle.read_rows([r])[0].role
        evs = [(e.type, e.from_slot, e.flags, e.n, e.n1, e.term, e.a, e.b, e.c, e.d, e.e) for e in events if e.row == r]
        raise AssertionError("%s: first differing row %d (oracle role %d), its events %r" % (what, r, role, evs))
    same_keys(want["msgs"], got["msgs"], what, "msgs")
    same_keys(want["notes"], got["notes"], what, "notes")
    if got["counters"] != want["counters"]:
        raise AssertionError("%s: counters differ: oracle %r, got %r" % (what, want["counters"], got["counters"]))
    same_keys(want["query"], got["query"], what, "query")


# ---- rounds ---------------------------------------------------------------------------------------------------------
def fuzz_round(rng, o, rnd, draw=rich_event):
    """States to load, their query states and the event batch of one round (events drawn by draw(rng, state, m) from
    the oracle's state of rows not reloaded)."""
    m, G = o.n_members, o.n_groups
    cur = o.read_rows(range(o.n_rows))
    loads, events, qs = [], [], []
    for r in range(o.n_rows):
        st = cur[r]
        shift = None
        if rnd == 0 or rng.random() < RELOAD:
            st = random_state(rng, r, G, m, rng.choice(ROLES), rich=True)
            if rng.random() < WIDE_ROWS:
                shift = rng.choice(OFFSETS[1:])
                shift_state(st, shift[0], shift[1], m)
            loads.append(st)
            qs.append(random_query(rng, r, m))
        for _ in range(rng.randint(0, abi.RA_LOCAL_CAP)):
            e = draw(rng, st, m)
            if shift:
                shift_event(e, shift[0], shift[1])
            events.append(e)
    return loads, qs, events


def unconsumed(notes, events):
    """The host events a note budget left unconsumed (include/ra_engine.h RA_ST_NOTE_OVERFLOW): STATUS.c bits 8..15 =
    how many of the LAST events of the row's run in the batch; the caller submits them again."""
    left = []
    for n in notes:
        k = (n.c >> 8) & 0xff if n.type == abi.NOTE_STATUS and n.aux & abi.ST_NOTE_OVERFLOW else 0
        if k:
            left += [e for e in events if e.row == n.row][-k:]
    return left


def snapshot_bursts(rng, loads, m):
    """Half the loaded leaders with a snapshot need it sent to every peer: their next pipeline pass or tick emits one
    SEND_SNAPSHOT per peer, a burst of notes that a small budget cannot hold (RA_FATAL_NOTE_OVERFLOW)."""
    for st in loads:
        if st.role == abi.LEADER and st.has_snapshot and rng.random() < 0.5:
            for p in range(m):
                pe = st.peers[p]
                pe.next_index = max(1, st.snapshot_index)
                pe.match_index = min(pe.match_index, pe.next_index - 1)


def fuzz_rounds(o, bs, mode, rounds, seed, draw=rich_event, note_cap=0, flood_chunk=4):
    """Rounds of fuzz_round through the oracle `o` and the (label, backend) pairs `bs`, every backend compared with the
    oracle after every step.  A backend needs load_rows, load_query_state, step, flood, rows_bytes, counters and
    read_query_state.

    mode (MODES): "routed" follows the fuzzed step with two empty steps; "flood" follows it with a 4-step flood, plain
    in even rounds and with FAULTS in odd ones, run as floods of flood_chunk steps with a comparison after each, then
    one empty step.  The host events a note budget left unconsumed are submitted again in a step of their own (or in
    the empty step that follows); note_cap != 0 also gives loaded leaders snapshot bursts.  Returns the coverage:
    events refused, rows stopped by RA_FATAL_NOTE_OVERFLOW and records the faulted floods dropped."""
    m = o.n_members
    xs = [o] + [b for _, b in bs]
    rng = random.Random(seed)
    cov = dict(refused=0, fatal_overflow=0, fault_drops=0)
    for rnd in range(rounds):
        loads, qs, events = fuzz_round(rng, o, rnd, draw)
        if note_cap:
            snapshot_bursts(rng, loads, m)
        for x in xs:
            x.load_rows(loads)
            x.load_query_state(qs)

        def check(what, outs, evs):
            want = observe(o, m, outs[0])
            for (label, b), out in zip(bs, outs[1:]):
                compare(want, observe(b, m, out), "M=%d %s round %d %s: %s" % (m, mode, rnd, label, what), evs, o)

        steps = [events] + ([[], []] if mode == "routed" else [])
        k = 0
        while k < len(steps):
            evs = steps[k]
            outs = [x.step([clone(e) for e in evs]) for x in xs]
            check("step %d" % k, outs, evs)
            left = unconsumed(outs[0][1], evs)
            cov["refused"] += len(left)
            cov["fatal_overflow"] += sum(1 for n in outs[0][1] if n.type == abi.NOTE_STATUS and n.aux & abi.ST_FATAL
                                         and n.c & 0xff == abi.FATAL_NOTE_OVERFLOW)
            if left:
                if k + 1 < len(steps):
                    steps[k + 1] = left + steps[k + 1]
                else:
                    steps.append(left)
            k += 1
        if mode == "flood":
            faults = FAULTS if rnd % 2 else None
            for t in range(0, 4, flood_chunk):                   # the flood's step count carries over between calls
                dropped = o.counters()["msgs_dropped"]
                o.flood(flood_chunk, FLOOD_CMDS, PERMILLE, seed=seed + rnd, threads=4, faults=faults)
                for _, b in bs:
                    b.flood(flood_chunk, FLOOD_CMDS, PERMILLE, seed=seed + rnd, faults=faults)
                check("flood%s from step %d" % (" with faults" if faults else "", t), [([], [])] * len(xs), [])
                if faults:
                    cov["fault_drops"] += o.counters()["msgs_dropped"] - dropped
            check("the step after the flood", [x.step([]) for x in xs], [])
    return cov


def budget_coverage(o, m, mode, cov):
    assert cov["refused"] > 0, "no host event was left unconsumed by the budget"
    if m >= 7 and mode != "flood":                  # a burst of 6-7 SEND_SNAPSHOT notes (the flood case has one
        assert cov["fatal_overflow"] > 0, "no row stopped with RA_FATAL_NOTE_OVERFLOW"       # fuzzed step only)
    if mode in ("routed", "flood") and m > 1:       # a group of one member sends no records, so none is dropped
        assert o.counters()["msgs_dropped"] > 0


def widths(monkeypatch):
    """Each RA_STEP_WIDE of WIDTHS in turn, set while the caller creates a backend (it is read at creation)."""
    for w in WIDTHS:
        monkeypatch.setenv("RA_STEP_WIDE", w)
        yield w


# ---- the (state, event) pair fuzz around the narrow limit -----------------------------------------------------------
def fuzz_around_the_narrow_limit(pure, backend=None, G=64):
    """Every row of a batch sits at its own distance from 2^30 / 2^31 / 2^32 (state and events moved together, and --
    one time in five -- the events moved but not the state, or the other way round: records that do not fit handed to
    rows that do).  M = 5: the emulated step kernel takes the 32-bit pass wherever it may.  backend(G, m, pure=..):
    the emulation (None), or the engine with G groups."""
    m = 5
    rng = random.Random(777 + (1 if pure else 0))
    o, e = Oracle(G, m, pure=pure), (backend or Emu)(G, m, pure=pure)
    Emu.narrow_stats()
    for rnd in range(40):
        states, events = [], []
        for g in range(G):
            slot = rng.randrange(m)
            st = random_state(rng, slot * G + g, G, m, rng.choice(ROLES))
            evs = [random_event(rng, st, m) for _ in range(rng.choice([1, 1, 2]))]
            di, dt = rng.choice(OFFSETS)
            mode = rng.random()
            if mode < 0.9:
                shift_state(st, di, dt, m)
            if mode > 0.1:
                for ev in evs:
                    shift_event(ev, di, dt)
            states.append(st)
            events.extend(evs)
        outs = []
        for b in (o, e):
            b.load_rows(states)
            outs.append(observe(b, m, b.step([clone(x) for x in events])))
        compare(outs[0], outs[1], "round %d" % rnd, events, o)
    if backend is None:
        st = Emu.narrow_stats()
        assert st["rows_narrow"] > 0 and st["rows_wide"] > 0 and st["records_refused"] > 0


# ---- small helpers --------------------------------------------------------------------------------------------------
def bootstrap(b, settle=0):
    """Every group's slot-0 member gets an election timeout, then `settle` empty steps (4: pre-vote and vote done,
    slot 0 leads every group)."""
    b.reset_empty()
    b.step([abi.ev_simple(b.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(b.n_groups)])
    for _ in range(settle):
        b.step([])


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p
