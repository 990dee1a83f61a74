"""Differential fuzz of the step kernels: random member states and random event batches, oracle against the host
emulation (CPU tier) and against the engine (GPU tier, the 32-bit and the 64-bit hot kernel), every step.

The states and events come from the generator of tests/fuzz_lib.py with rich = True: up to 8 term runs, pending
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
import random

import pytest

from emu_lib import Emu, plane_forms, stats_lib
from fuzz_lib import (MEMBERS, MODES, NOTE_CAPS, PERMILLE, WIDTHS, bootstrap, budget_coverage,
                      fuzz_around_the_narrow_limit, fuzz_round, fuzz_rounds, kw, widths)
from oracle_lib import Oracle
from ra_b200 import abi
from ra_suite import clone, make_backend


def _fuzz(name, monkeypatch, mode, m, G, rounds, seed, note_cap=0):
    """The oracle and a backend `name` for each RA_STEP_WIDE through fuzz_rounds -> (oracle, backends, coverage).
    note_cap != 0: every backend runs with that budget."""
    o = Oracle(G, m, **kw(mode, note_cap))
    bs = [("RA_STEP_WIDE=" + w, make_backend(name, G, m, **kw(mode, note_cap))) for w in widths(monkeypatch)]
    return o, bs, fuzz_rounds(o, bs, mode, rounds, seed, note_cap=note_cap)


# ---- CPU tier: the host emulation -----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("m", MEMBERS)
def test_kernel_fuzz_emu(m, mode, monkeypatch):
    Emu.narrow_stats(); Emu.stall_stats(); Emu.underfetched()
    o, _, _ = _fuzz("emu", monkeypatch, mode, m, 64, 12, 4000 + 10 * m + MODES.index(mode))
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
    o, e = Oracle(G, m, **kw("routed")), Emu(G, m, library=stats_lib(), **kw("routed"))
    heads = longs = cmds = 0
    for rnd in range(4):
        loads, qs, events = fuzz_round(rng, o, rnd)
        for x in (o, e):
            x.load_rows(loads)
            x.step([clone(v) for v in events])
        plane_forms()
        for x in (o, e):
            x.step([])
            x.step([])
        forms = plane_forms()
        heads += forms[abi.EV_AER].head
        longs += forms[abi.EV_AER].long
        cmds += forms[abi.EV_COMMAND].head + forms[abi.EV_COMMAND].long
        assert e.rows_bytes() == o.rows_bytes()
    assert heads > 0 and longs > 0, (heads, longs)
    assert cmds == 0                                           # (commands only come from the host)


# ---- GPU tier: the engine, the 32-bit and the 64-bit hot kernel -----------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("m", MEMBERS)
def test_kernel_fuzz_engine(m, mode, monkeypatch):
    _, bs, _ = _fuzz("engine", monkeypatch, mode, m, 1200 if m <= 5 else 1024, 3, 7000 + 10 * m + MODES.index(mode))
    for label, b in bs:
        assert b.stall_histogram(), "%s: no row took the general kernel" % label


# ---- small note budgets: events refused and submitted again, rows stopped by a burst of notes -----------------------
def _note_cap_of(m, mode):
    return NOTE_CAPS[m][MODES.index(mode)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("m", MEMBERS)
def test_kernel_fuzz_note_cap_emu(m, mode, monkeypatch):
    o, _, cov = _fuzz("emu", monkeypatch, mode, m, 64, 8, 4500 + 10 * m + MODES.index(mode), _note_cap_of(m, mode))
    budget_coverage(o, m, mode, cov)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("m", [3, 5, 8])
def test_kernel_fuzz_note_cap_engine(m, mode, monkeypatch):
    o, _, cov = _fuzz("engine", monkeypatch, mode, m, 1024, 2, 7500 + 10 * m + MODES.index(mode), _note_cap_of(m, mode))
    budget_coverage(o, m, mode, cov)


@pytest.mark.gpu
@pytest.mark.parametrize("wide", WIDTHS)
@pytest.mark.parametrize("pure", [True, False])
def test_fuzz_around_the_narrow_limit_engine(pure, wide, monkeypatch):
    monkeypatch.setenv("RA_STEP_WIDE", wide)
    fuzz_around_the_narrow_limit(pure, backend=lambda G, m, **cfg: make_backend("engine", G, m, **cfg), G=1200)


# ---- two regressions, against the emulation and the engine ----------------------------------------------------------
BACKENDS = ["emu", pytest.param("engine", marks=pytest.mark.gpu)]


def _fatal_then_reload(b, G, m=3):
    """Slot-0 leaders replicate; in the step their followers acknowledge the write (and reply), each leader is made
    fatal by an AppendEntries from another member at its own term, so the replies wait in its mailbox.  Two steps of
    ticks later -- its followers run, and send it nothing -- the leader is reloaded as it was before, not fatal, and
    stepped.  It must not evaluate the replies addressed to its earlier life."""
    bootstrap(b, settle=4)                                     # pre-vote, vote: slot 0 leads every group
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
        out.append(b.step([clone(e) for e in ticks]))
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
    bootstrap(b, settle=4)
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
