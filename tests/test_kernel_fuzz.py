"""Differential fuzz of the step kernels: random member states and random event batches, oracle against the host
emulation (CPU tier) and against the engine (GPU tier, the 32-bit and the 64-bit hot kernel), every step.

The states and events come from the generator of tests/test_emu_fuzz.py with rich = True: up to 8 term runs, pending
pipeline passes, machine versions, odd memberships and peer statuses; AppendEntries of 255-300 entries over one or
two term runs, replies from unknown slots, commands of 256 and 1000 entries.  Every row of every slot gets 0..4
events, so warps are full of mixed roles and records of every form share tiles.  One row in twenty sits at 2^30 /
2^32 / 2^40, so the 32-bit pass both runs and refuses.  Rounds follow each other on the same backends: each round
loads fresh states into most rows (mail still in flight to them is dropped, include/ra_engine.h) and leaves the
others as the round before left them.

Modes: not routed, pure and chased; routed, where the fuzzed step is followed by two empty steps that evaluate the
records sent from fuzzed states and the deferred pipeline passes; routed with a 4-step flood from the fuzzed states,
plain and with faults in turn, then an empty step.  Every step compares RPC records and notes in order, every row
as raw ra_row_state bytes, counters and query state.
"""
import ctypes as C
import random

import pytest

import test_emu_fuzz as fz
from emu_lib import Emu
from oracle_lib import Oracle
from ra_b200 import abi
from ra_suite import make_backend
from test_record_forms import HEAD, LONG
from test_short_records import plane_forms, stats_lib

MEMBERS = [3, 4, 5, 7, 8]
MODES = ["pure", "chased", "routed", "flood"]
WIDTHS = ["0", "1"]                          # RA_STEP_WIDE: the 32-bit hot kernel / the 64-bit one
FAULTS = (20, 50, 30, 16)                    # drop, withhold, partition permille, partition steps
FLOOD_CMDS, PERMILLE = 300, 15
RELOAD, WIDE_ROWS = 0.7, 0.05               # per round and row: fresh state / moved to the narrow limit


# small note budgets (cfg.note_cap, RA_NOTE_RESERVE + 2 ..) per M, in the order of MODES: every budget meets several
# modes; the larger ones go where more peers make more notes, so that each case still runs into its budget
NOTE_CAPS = {3: [6, 7, 6, 7], 4: [7, 6, 7, 6], 5: [9, 6, 9, 7], 7: [12, 6, 7, 9], 8: [9, 12, 6, 9]}


def _kw(mode, note_cap=0):
    return dict(pure=(mode == "pure"), route_on_device=mode in ("routed", "flood"), max_aer_batch=512, note_cap=note_cap)


def _observe(b, m, out=None):
    msgs, notes = out if out is not None else ([], [])
    q = b.read_query_state(range(b.n_rows))
    return dict(msgs=[x.key() for x in msgs], notes=[x.key() for x in notes], rows=b.rows_bytes(),
                counters=b.counters(), query=[x.key(m) for x in q])


def _first_row(a, b):
    sz = C.sizeof(abi.RaRowState)
    return next((i // sz for i in range(0, len(a), sz) if a[i:i + sz] != b[i:i + sz]), -1)


def _compare(want, got, what, events, oracle):
    """First difference between the oracle's and a backend's observation, with the row's role and its events."""
    if got["rows"] != want["rows"]:
        r = _first_row(want["rows"], got["rows"])
        role = oracle.read_rows([r])[0].role
        evs = [(e.type, e.from_slot, e.flags, e.n, e.n1, e.term, e.a, e.b, e.c, e.d, e.e) for e in events if e.row == r]
        raise AssertionError("%s: first differing row %d (oracle role %d), its events %r" % (what, r, role, evs))
    for k in ("msgs", "notes", "counters", "query"):
        if got[k] != want[k]:
            if isinstance(want[k], list):
                i = next((i for i, (x, y) in enumerate(zip(want[k], got[k])) if x != y), min(len(want[k]), len(got[k])))
                row = (want[k][i:i + 1] or got[k][i:i + 1])[0][0]
                raise AssertionError("%s: %s differ from #%d on (row %d): oracle %r, got %r (%d / %d)"
                                     % (what, k, i, row, want[k][i:i + 1], got[k][i:i + 1], len(want[k]), len(got[k])))
            raise AssertionError("%s: %s differ: oracle %r, got %r" % (what, k, want[k], got[k]))


def _fuzz_round(rng, o, m, G, rnd, draw=None):
    """States to load and the event batch of one round (events drawn from the oracle's state of rows not reloaded).
    draw(rng, state, m) -> event replaces the rich generator (tests/test_call_paths_fuzz.py: host events only)."""
    n_rows = G * m
    cur = o.read_rows(range(n_rows))
    loads, events, qs = [], [], []
    for r in range(n_rows):
        st = cur[r]
        shift = None
        if rnd == 0 or rng.random() < RELOAD:
            st = fz.random_state(rng, r, G, m, rng.choice(fz.ROLES), rich=True)
            if rng.random() < WIDE_ROWS:
                shift = rng.choice(fz.OFFSETS[1:])
                fz._shift_state(st, shift[0], shift[1], m)
            loads.append(st)
            q = abi.RaQueryState(row=r, query_index=rng.randint(0, 4), agreed_index=rng.randint(0, 2))
            for p in range(m):
                q.peer_query_index[p] = rng.randint(0, 4)
            qs.append(q)
        for _ in range(rng.randint(0, abi.RA_LOCAL_CAP)):
            e = draw(rng, st, m) if draw else fz.random_event(rng, st, m, rich=True)
            if shift:
                fz._shift_event(e, shift[0], shift[1])
            events.append(e)
    return loads, qs, events


def _unconsumed(notes, events):
    """The host events a note budget left unconsumed (include/ra_engine.h RA_ST_NOTE_OVERFLOW): STATUS.c bits 8..15 =
    how many of the LAST events of the row's run in the batch; the caller submits them again."""
    left = []
    for n in notes:
        k = (n.c >> 8) & 0xff if n.type == abi.NOTE_STATUS and n.aux & abi.ST_NOTE_OVERFLOW else 0
        if k:
            left += [e for e in events if e.row == n.row][-k:]
    return left


def _snapshot_bursts(rng, loads, m):
    """Half the loaded leaders with a snapshot need it sent to every peer: their next pipeline pass or tick emits one
    SEND_SNAPSHOT per peer, a burst of notes that a small budget cannot hold (RA_FATAL_NOTE_OVERFLOW)."""
    for st in loads:
        if st.role == abi.LEADER and st.has_snapshot and rng.random() < 0.5:
            for p in range(m):
                pe = st.peers[p]
                pe.next_index = max(1, st.snapshot_index)
                pe.match_index = min(pe.match_index, pe.next_index - 1)


def _fuzz(make, mode, m, G, rounds, seed, note_cap=0):
    """make(width) -> a backend built with RA_STEP_WIDE = width; returns the oracle, the backends for the coverage
    checks and what the note budget did.  note_cap != 0: every backend runs with that budget, and after each step the
    host events it left unconsumed are submitted again in a step of their own (or in the empty step that follows)."""
    rng = random.Random(seed)
    o = Oracle(G, m, **_kw(mode, note_cap))
    bs = [(w, make(w, G, m, **_kw(mode, note_cap))) for w in WIDTHS]
    cov = dict(refused=0, fatal_overflow=0)
    for rnd in range(rounds):
        loads, qs, events = _fuzz_round(rng, o, m, G, rnd)
        if note_cap:
            _snapshot_bursts(rng, loads, m)
        steps = [events] + ([[], []] if mode == "routed" else [])
        for x in [o] + [b for _, b in bs]:
            x.load_rows(loads)
            x.load_query_state(qs)

        def check(what, outs, evs):
            want = _observe(o, m, out=outs[0])
            for (w, b), out in zip(bs, outs[1:]):
                _compare(want, _observe(b, m, out=out), "M=%d %s round %d RA_STEP_WIDE=%s: %s" % (m, mode, rnd, w, what),
                         evs, o)

        k = 0
        while k < len(steps):
            evs = steps[k]
            outs = [x.step([fz._copy(e) for e in evs]) for x in [o] + [b for _, b in bs]]
            check("step %d" % k, outs, evs)
            left = _unconsumed(outs[0][1], evs)
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
            o.flood(4, FLOOD_CMDS, PERMILLE, seed=seed + rnd, threads=4, faults=faults)
            for _, b in bs:
                b.flood(4, FLOOD_CMDS, PERMILLE, seed=seed + rnd, faults=faults)
            check("flood%s" % (" with faults" if faults else ""), [([], [])] * (1 + len(bs)), [])
            outs = [x.step([]) for x in [o] + [b for _, b in bs]]
            check("the step after the flood", outs, [])
    return o, bs, cov


def _maker(name, monkeypatch):
    def make(width, G, m, **kw):
        monkeypatch.setenv("RA_STEP_WIDE", width)               # read when the backend is created
        return make_backend(name, G, m, **kw)
    return make


# ---- CPU tier: the host emulation -----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("m", MEMBERS)
def test_kernel_fuzz_emu(m, mode, monkeypatch):
    Emu.narrow_stats(); Emu.stall_stats(); Emu.underfetched()
    o, bs, _ = _fuzz(_maker("emu", monkeypatch), mode, m, 64, 12, 4000 + 10 * m + MODES.index(mode))
    assert Emu.underfetched() == 0, "the hot path decoded a record from bytes its tile's fetch did not cover"
    assert Emu.stall_stats()["stalls"] > 0
    assert o.counters()["fatal_rows"] > 0
    ns = Emu.narrow_stats()
    if m == 5:                                                 # the emulation's 32-bit pass runs at M = 5
        assert ns["rows_narrow"] > 0 and ns["rows_wide"] > 0 and ns["records_refused"] > 0, ns


def test_kernel_fuzz_routed_twin():
    """The routed fuzz on the plane-stats build: the two empty steps after a fuzzed step store head and long records
    in the mailbox planes (no host event is ingested in them)."""
    G, m = 48, 5
    rng = random.Random(4321)
    o, e = Oracle(G, m, **_kw("routed")), Emu(G, m, library=stats_lib(), **_kw("routed"))
    heads = longs = cmds = 0
    for rnd in range(4):
        loads, qs, events = _fuzz_round(rng, o, m, G, rnd)
        for x in (o, e):
            x.load_rows(loads)
            x.step([fz._copy(v) for v in events])
        plane_forms()
        for x in (o, e):
            x.step([])
            x.step([])
        forms = plane_forms()
        heads += forms[abi.EV_AER][HEAD]
        longs += forms[abi.EV_AER][LONG]
        cmds += forms[abi.EV_COMMAND][HEAD] + forms[abi.EV_COMMAND][LONG]
        assert e.rows_bytes() == o.rows_bytes()
    assert heads > 0 and longs > 0, (heads, longs)
    assert cmds == 0                                           # (commands only come from the host)


# ---- GPU tier: the engine, the 32-bit and the 64-bit hot kernel -----------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("m", MEMBERS)
def test_kernel_fuzz_engine(m, mode, monkeypatch):
    o, bs, _ = _fuzz(_maker("engine", monkeypatch), mode, m, 1200 if m <= 5 else 1024, 3, 7000 + 10 * m + MODES.index(mode))
    for w, b in bs:
        assert b.stall_histogram(), "RA_STEP_WIDE=%s: no row took the general kernel" % w


# ---- small note budgets: events refused and submitted again, rows stopped by a burst of notes -----------------------
def _note_cap_of(m, mode):
    return NOTE_CAPS[m][MODES.index(mode)]


def _budget_coverage(o, m, mode, cov):
    assert cov["refused"] > 0, "no host event was left unconsumed by the budget"
    if m >= 7 and mode != "flood":                  # a burst of 6-7 SEND_SNAPSHOT notes (the flood case has one
        assert cov["fatal_overflow"] > 0, "no row stopped with RA_FATAL_NOTE_OVERFLOW"       # fuzzed step only)
    if mode in ("routed", "flood"):
        assert o.counters()["msgs_dropped"] > 0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("m", MEMBERS)
def test_kernel_fuzz_note_cap_emu(m, mode, monkeypatch):
    o, _, cov = _fuzz(_maker("emu", monkeypatch), mode, m, 64, 8, 4500 + 10 * m + MODES.index(mode), _note_cap_of(m, mode))
    _budget_coverage(o, m, mode, cov)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("m", [3, 5, 8])
def test_kernel_fuzz_note_cap_engine(m, mode, monkeypatch):
    o, _, cov = _fuzz(_maker("engine", monkeypatch), mode, m, 1024, 2, 7500 + 10 * m + MODES.index(mode),
                      _note_cap_of(m, mode))
    _budget_coverage(o, m, mode, cov)


@pytest.mark.gpu
@pytest.mark.parametrize("wide", WIDTHS)
@pytest.mark.parametrize("pure", [True, False])
def test_fuzz_around_the_narrow_limit_engine(pure, wide, monkeypatch):
    monkeypatch.setenv("RA_STEP_WIDE", wide)
    fz._fuzz_around_the_narrow_limit(pure, backend=lambda G, m, **kw: make_backend("engine", G, m, **kw), G=1200)


# ---- two regressions, against the emulation and the engine ----------------------------------------------------------
BACKENDS = ["emu", pytest.param("engine", marks=pytest.mark.gpu)]


def _bootstrap(b):
    b.reset_empty()
    b.step([abi.ev_simple(b.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(b.n_groups)])
    for _ in range(4):                                         # pre-vote, vote: slot 0 leads every group
        b.step([])


def _fatal_then_reload(b, G, m=3):
    """Slot-0 leaders replicate; in the step their followers acknowledge the write (and reply), each leader is made
    fatal by an AppendEntries from another member at its own term, so the replies wait in its mailbox.  Two steps of
    ticks later -- its followers run, and send it nothing -- the leader is reloaded as it was before, not fatal, and
    stepped.  It must not evaluate the replies addressed to its earlier life."""
    _bootstrap(b)
    leaders = [b.row_of(g, 0) for g in range(G)]
    st = b.read_rows(leaders)
    assert all(s.role == abi.LEADER for s in st)
    out = [b.step([abi.ev_command(r, 2) for r in leaders])]
    written = [abi.ev_written(n.row, n.c, n.a, n.b) for n in out[0][1] if n.type == abi.NOTE_WAL_APPEND and n.row >= G]
    assert written
    fatal = [abi.ev_aer(r, 1, s.current_term, s.last_index, s.last_term, 0, [s.current_term]) for r, s in zip(leaders, st)]
    out.append(b.step(sorted(written + fatal, key=lambda e: e.row)))
    ticks = [abi.ev_simple(b.row_of(g, s), abi.EV_TICK) for s in range(1, m) for g in range(G)]
    for _ in range(2):
        out.append(b.step([fz._copy(e) for e in ticks]))
    assert all(s.flags & 4 for s in b.read_rows(leaders))     # fatal
    b.load_rows(st)
    out.append(b.step([abi.ev_simple(r, abi.EV_TICK) for r in leaders]))
    out.append(b.step([]))
    return [([x.key() for x in msgs], [n.key() for n in notes]) for msgs, notes in out]


@pytest.mark.parametrize("backend", BACKENDS)
def test_reloaded_fatal_row_gets_no_stale_mail(backend):
    G = 40 if backend == "emu" else 1200
    b = make_backend(backend, G, 3, route_on_device=True)
    o = Oracle(G, 3, route_on_device=True)
    want, got = _fatal_then_reload(o, G), _fatal_then_reload(b, G)
    for k, (w, x) in enumerate(zip(want, got)):
        assert x == w, "step %d differs" % k
    assert b.counters() == o.counters()
    assert b.rows_bytes() == o.rows_bytes()


def _flood_then_step(b):
    _bootstrap(b)
    b.flood(3, 1, PERMILLE, seed=11)
    leader = next(r.row for r in b.read_rows(range(b.n_rows)) if r.role == abi.LEADER)
    msgs, notes = b.step([abi.ev_command(leader, 1)])
    return [n.key() for n in notes], leader


@pytest.mark.parametrize("backend", BACKENDS)
def test_step_after_flood_returns_only_its_own_notes(backend):
    G = 40 if backend == "emu" else 1200
    b = make_backend(backend, G, 5, route_on_device=True)
    o = Oracle(G, 5, route_on_device=True)
    want, got = _flood_then_step(o), _flood_then_step(b)
    assert got == want
    assert b.counters() == o.counters()
