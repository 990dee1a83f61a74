"""Differential fuzz of the engine's host call paths: the ways a real caller (INTEGRATION.md, ra_engine_nif.c,
ra_hostsim) hands batches over and takes outputs back, each against the oracle with ample buffers in the plain
format.  States and events come from the generator of tests/fuzz_lib.py (rich = True) through the rounds of the
kernel fuzz: RPC records and notes in order, every row as raw ra_row_state bytes, counters and query
state are compared.

- host-event batches, each sent three ways: ra_engine_step_host (32-byte records), ra_engine_submit_host_segs split
  at random row boundaries, ra_engine_step (64-byte records);
- two calls in flight: batch t+1 drawn from the oracle's state after step t and submitted before t is collected,
  with pageable and with pinned output buffers, and output sizes that swing from step to step (the predicted-size
  copy and its top-up);
- tight output buffers: RA_E_CAPACITY, ra_engine_pending_output and a fetch of exactly the reported size, in the
  plain and the compact note format, one and two calls deep;
- the compact note stream, unit for unit against a reference encoder of the rule in include/ra_engine.h, and the
  decoder (ra_notes16_expand) on every note form the fuzz produces.
"""
import ctypes as C
import random
import struct

import pytest

from fuzz_lib import (HOST_TYPES, MEMBERS, MODES, batch, fuzz_round, fuzz_rounds, host_event, kw, rich_event,
                      same_keys, widths)
from oracle_lib import Oracle
from ra_b200 import abi
from ra_b200.engine import Engine, notes16_expand
from ra_suite import clone, make_backend


def _segments(rng, evs):
    """1..256 pieces cut at row boundaries (a row's events never straddle two), some of them empty"""
    bounds = [0] + [i for i in range(1, len(evs)) if evs[i].row != evs[i - 1].row] + [len(evs)]
    cuts = sorted(rng.choice(bounds) for _ in range(rng.randint(1, 256) - 1))
    edges = [0] + cuts + [len(evs)]
    return [evs[a:b] for a, b in zip(edges, edges[1:])]


class _Path:
    """A backend whose step() hands the batch over through one call path with ample buffers: ra_engine_step_host,
    ra_engine_submit_host_segs with pieces cut by rng, or ra_engine_step."""

    def __init__(self, b, path, rng):
        self.b, self.path, self.rng = b, path, rng

    def __getattr__(self, name):
        return getattr(self.b, name)

    def step(self, evs):
        b = self.b
        mc, nc = b.n_rows * abi.RA_MSG_CAP, b.n_rows * abi.RA_NOTE_CAP
        if self.path == "step":
            return b.step(evs, mc, nc)
        if self.path == "step_host":
            return b.step_host(evs, mc, nc)
        st, ticket = b.submit_host_segs(_segments(self.rng, evs), mc, nc)
        assert st == abi.RA_OK
        st, _, _, msgs, notes = b.collect(ticket)
        assert st == abi.RA_OK, "%s: status %d" % (self.path, st)
        return msgs, notes


# ---- 1. host-event batches, three ways ------------------------------------------------------------------------------
PATHS = ["step_host", "segs", "step"]
HOST_MODES = ["routed", "flood"]


def _host_fuzz(backend, mode, m, G, rounds, seed, monkeypatch):
    srng = random.Random(seed + 1)
    o = Oracle(G, m, **kw(mode))
    bs = []
    for w in widths(monkeypatch):
        bs += [("RA_STEP_WIDE=%s %s" % (w, p), _Path(make_backend(backend, G, m, **kw(mode)), p, srng)) for p in PATHS]
    drawn = []

    def draw(rng, st, members):
        drawn.append(host_event(rng, st, members))
        return drawn[-1]
    fuzz_rounds(o, bs, mode, rounds, seed, draw=draw)
    assert all(e.type in HOST_TYPES for e in drawn)
    assert any(e.type == abi.EV_COMMAND and e.n >= 256 for e in drawn)   # commands of 256 and 1000 entries: n > 8 bits


@pytest.mark.parametrize("mode", HOST_MODES)
@pytest.mark.parametrize("m", MEMBERS)
def test_host_batches_three_ways_emu(m, mode, monkeypatch):
    _host_fuzz("emu", mode, m, 48, 4, 8000 + 10 * m + HOST_MODES.index(mode), monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", HOST_MODES)
@pytest.mark.parametrize("m", MEMBERS)
def test_host_batches_three_ways_engine(m, mode, monkeypatch):
    _host_fuzz("engine", mode, m, 1200 if m <= 5 else 1024, 2, 8500 + 10 * m + HOST_MODES.index(mode), monkeypatch)


# ---- compact note stream: the reference encoder (include/ra_engine.h, "Compact note stream") ------------------------
def encode16(notes, wal_c):
    """notes (ordered by row, seq) -> (the bytes of units + extension area, n_ext).  wal_c: row -> c of the row's
    previous WAL_APPEND note (absent = 0), updated by every WAL_APPEND."""
    units, ext = [], []
    for n in notes:
        small = n.slot == 0 and n.a <= n.b and n.b - n.a < 256
        if n.type == abi.NOTE_WAL_APPEND:
            same = n.c == wal_c.get(n.row, 0)
            wal_c[n.row] = n.c
            one = small and same
        else:
            one = small and n.c == 0
        if one:
            t = n.type | (abi.N16_SAME_TERM if n.type == abi.NOTE_WAL_APPEND else 0)
            units.append(struct.pack("<IBBHQ", n.row, t, n.b - n.a, n.aux, n.a))
        else:
            units.append(struct.pack("<IBBHQ", n.row, n.type | abi.N16_EXT, n.slot, n.aux, len(ext) // 2))
            ext += [struct.pack("<QQ", n.a, n.b), struct.pack("<QQ", n.c, 0)]
    return b"".join(units + ext), len(ext) // 2


FORMS = ("ext_slot", "range_256", "status_c", "above_2_32", "truncate", "query", "same_term")


def _forms(notes, seen):
    for n in notes:
        seen["ext_slot"] += n.slot != 0
        seen["range_256"] += n.b >= n.a + 256
        seen["status_c"] += n.type == abi.NOTE_STATUS and n.c != 0
        seen["above_2_32"] += max(n.a, n.b, n.c) >= 1 << 32
        seen["truncate"] += n.type == abi.NOTE_TRUNCATE
        seen["query"] += n.type in (abi.NOTE_QUERY_INDEX, abi.NOTE_QUERY_AGREED)


class _RoundTrip(Oracle):
    """CPU tier: the oracle whose notes go through the reference encoder and ra_notes16_expand on their way out."""

    def __init__(self, G, m, **kw):
        super().__init__(G, m, **kw)
        self.wal_c, self.last_c = {}, (C.c_uint64 * (G * m))()
        self.seen = dict.fromkeys(FORMS, 0)

    def load_rows(self, rows):
        super().load_rows(rows)
        for s in rows:
            self.wal_c.pop(s.row, None)
            self.last_c[s.row] = 0

    def step(self, events, msgs_cap=None, notes_cap=None):
        msgs, notes = super().step(events, msgs_cap, notes_cap)
        _forms(notes, self.seen)
        units, n_ext = encode16(notes, self.wal_c)
        self.seen["same_term"] += sum(1 for k in range(len(notes)) if units[16 * k + 4] & abi.N16_SAME_TERM)
        return msgs, notes16_expand(units, len(notes), n_ext, self.last_c)


@pytest.mark.parametrize("mode", MODES)
def test_notes16_expand_on_fuzz_notes(mode):
    """every note the fuzz produces, through the reference encoder and the host decoder, comes back unchanged"""
    seen = dict.fromkeys(FORMS, 0)
    for m in (3, 5, 8):
        b = _RoundTrip(48, m, **kw(mode))
        fuzz_rounds(Oracle(48, m, **kw(mode)), [("notes16 round trip", b)], mode, 4, 9000 + 10 * m)
        for k, v in b.seen.items():
            seen[k] += v
    missing = [k for k in FORMS if not seen[k] and not (k == "query" and mode == "flood")]
    assert not missing, (missing, seen)


class _CompactEngine(Engine):
    """GPU tier: an Engine in the compact note format whose step() returns the notes ra_notes16_expand rebuilt, after
    checking its raw units and extension area against the reference encoder on those notes.  Since the fuzz compares
    the notes with the oracle's, the units equal the encoder's output on the oracle's notes."""

    def __init__(self, G, m, **kw):
        super().__init__(G, m, **kw)
        self.set_note_format(True)
        self.wal_c, self.ext = {}, 0

    def load_rows(self, rows):
        super().load_rows(rows)
        for s in rows:                                           # the engine and the decoder forget the row's c
            self.wal_c.pop(s.row, None)
            self._last_c[s.row] = 0

    def step(self, events, msgs_cap=None, notes_cap=None):
        msgs, notes, units, n_ext = self.step_compact(events, msgs_cap=self.n_rows * abi.RA_MSG_CAP)
        want, want_ext = encode16(notes, self.wal_c)
        got = b"".join(bytes(u) for u in units)
        assert (got, n_ext) == (want, want_ext), "compact units differ from the reference encoder"
        self.ext += n_ext
        return msgs, notes


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_compact_stream_unit_for_unit_engine(mode, monkeypatch):
    bs = [("RA_STEP_WIDE=" + w, _CompactEngine(1200, 5, **kw(mode))) for w in widths(monkeypatch)]
    fuzz_rounds(Oracle(1200, 5, **kw(mode)), bs, mode, 3, 9500 + MODES.index(mode))
    assert all(b.ext > 0 for _, b in bs)


# ---- raw calls with counts on RA_E_CAPACITY -------------------------------------------------------------------------
class _Out:
    """output buffers of one call: pageable ctypes arrays or pinned ra_engine_alloc_host memory; notes_cap counts
    32-byte notes or (compact) 16-byte units"""

    def __init__(self, b, msgs_cap, notes_cap, compact=False, pinned=False):
        self.mc, self.nc, self.compact, self.pinned = msgs_cap, notes_cap, compact, pinned
        nt = abi.RaNote16 if compact else abi.RaNote
        if pinned:
            self._api = b._api
            self._p = [self._api.alloc_host(max(msgs_cap, 1) * 64), self._api.alloc_host(max(notes_cap, 1) * 32)]
            assert all(self._p)
            self.msgs = (abi.RaEvent * max(msgs_cap, 1)).from_address(self._p[0])
            self.notes = (nt * max(notes_cap, 1)).from_address(self._p[1])
        else:
            self.msgs, self.notes = (abi.RaEvent * max(msgs_cap, 1))(), (nt * max(notes_cap, 1))()

    def free(self):
        if self.pinned:
            for p in self._p:
                self._api.free_host(p)
            self.pinned = False

    def result(self, nm, nn, n_ext=0, last_c=None):
        msgs = [clone(x) for x in self.msgs[:nm]]
        if not self.compact:
            return msgs, [abi.RaNote.from_buffer_copy(x) for x in self.notes[:nn]]
        return msgs, notes16_expand(bytes(self.notes)[: 16 * (nn + 2 * n_ext)], nn, n_ext, last_c)

    def units(self, nn, n_ext):
        return bytes(self.notes)[: 16 * (nn + 2 * n_ext)]


def _submit(b, api, evs, out):
    st, ticket = getattr(b, api)(evs, out.mc, out.nc, out=(out.msgs, out.notes))
    assert st == abi.RA_OK, "%s: status %d" % (api, st)
    return ticket                                                # (holds the batch until it is collected)


# ---- 2 + 3. two calls in flight; tight output buffers, one and two calls deep ---------------------------------------
def _chain(b, o, m, G, mode, api, rng, rounds, steps, depth, tight=False, compact=False, pinned=False):
    """rounds of `steps` batches; every batch goes in while `depth - 1` calls are still in flight.  tight: each call's
    buffers hold 0 .. all of what it needs; a call answered RA_E_CAPACITY is fetched with exactly the reported size,
    and a call submitted behind it must come back RA_E_PENDING and is submitted again."""
    draw = host_event if api == "submit_host" else rich_event
    wal_c, last_c = {}, ((C.c_uint64 * (G * m))() if compact else None)
    cov = dict(capacity=0, pending=0, calls=0)
    for rnd in range(rounds):
        loads, qs, _ = fuzz_round(rng, o, rnd, draw)
        for x in (o, b):
            x.load_rows(loads)
            x.load_query_state(qs)
        for s in loads:
            wal_c.pop(s.row, None)
            if compact:
                last_c[s.row] = 0
        wants, fly = [], []                                      # oracle outputs of every batch; calls in flight

        def new_out(k):
            msgs, notes = wants[k][1]
            n_units = len(notes)
            if compact:
                wants[k][2], wants[k][3] = encode16(notes, dict(wal_c_at[k]))
                n_units += 2 * wants[k][3]
            if tight:
                return _Out(b, rng.randint(0, len(msgs)), rng.randint(0, n_units), compact, pinned)
            return _Out(b, G * m * abi.RA_MSG_CAP, G * m * abi.RA_NOTE_CAP * (2 if compact else 1), compact, pinned)

        wal_c_at = []

        def submit(k):
            out = new_out(k)
            fly.append((k, out, _submit(b, api, wants[k][0], out)))

        def finish(k, out, nm, nn):
            msgs, notes = wants[k][1]
            what = "M=%d %s round %d batch %d" % (m, mode, rnd, k)
            n_ext = 0
            if compact:
                n_ext = b.last_ext_count()
                assert n_ext == wants[k][3], "%s: ra_engine_last_ext_count %d, the encoder %d" % (what, n_ext, wants[k][3])
                assert out.units(nn, n_ext) == wants[k][2], "%s: compact units differ" % what
            got_msgs, got_notes = out.result(nm, nn, n_ext, last_c)
            same_keys([x.key() for x in msgs], [x.key() for x in got_msgs], what, "msgs")
            same_keys([x.key() for x in notes], [x.key() for x in got_notes], what, "notes")
            out.free()

        def collect_oldest():
            k, out, ticket = fly.pop(0)
            st, nm, nn, _, _ = b.collect(ticket)
            cov["calls"] += 1
            msgs, notes = wants[k][1]
            what = "M=%d %s round %d batch %d" % (m, mode, rnd, k)
            if st == abi.RA_E_CAPACITY:
                cov["capacity"] += 1
                assert (nm, nn) == (len(msgs), len(notes)), "%s: RA_E_CAPACITY reports %r, needed %r" % (
                    what, (nm, nn), (len(msgs), len(notes)))
                assert b.pending_output() == (len(msgs), len(notes)), "%s: pending_output %r" % (what, b.pending_output())
                behind = []
                while fly:                                       # calls submitted behind it: not evaluated
                    k2, out2, ticket2 = fly.pop(0)
                    st2 = b.collect(ticket2)[0]
                    assert st2 == abi.RA_E_PENDING, "%s: the call submitted behind it returned %d, not " \
                        "RA_E_PENDING" % (what, st2)
                    cov["pending"] += 1
                    out2.free()
                    behind.append(k2)
                units = nn + 2 * b.last_ext_count() if compact else nn
                out.free()
                out = _Out(b, nm, units, compact, pinned)
                st, nm2, nn2, _, _ = b.fetch_output(out.mc, out.nc, out=(out.msgs, out.notes))
                assert st == abi.RA_OK and (nm2, nn2) == (nm, nn), "%s: fetch of the reported size: %d %r" % (
                    what, st, (nm2, nn2))
                finish(k, out, nm, nn)
                for k2 in behind:
                    submit(k2)
            else:
                assert st == abi.RA_OK, "%s: collect status %d" % (what, st)
                finish(k, out, nm, nn)

        for t in range(steps):
            evs = batch(rng, o, draw, rng.choice([0.02, 0.3, 1.0]))
            wal_c_at.append(dict(wal_c))
            want = o.step([clone(e) for e in evs], G * m * abi.RA_MSG_CAP, G * m * abi.RA_NOTE_CAP)
            encode16(want[1], wal_c)                             # the per-row memory the engine keeps
            wants.append([evs, want, None, 0])
            submit(t)
            while len(fly) >= depth:
                collect_oldest()
        while fly:
            collect_oldest()
        assert b.rows_bytes() == o.rows_bytes(), "M=%d %s round %d: rows differ" % (m, mode, rnd)
        assert b.counters() == o.counters()
    return cov


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("api", ["submit", "submit_host"])
def test_two_calls_in_flight_engine(api, pinned):
    G, m = 1200, 5
    rng = random.Random(9700 + 2 * (api == "submit_host") + pinned)
    o, b = Oracle(G, m, **kw("chased")), Engine(G, m, **kw("chased"))
    cov = _chain(b, o, m, G, "chased", api, rng, rounds=2, steps=8, depth=2, pinned=pinned)
    assert cov["calls"] == 16


TIGHT = [("emu", "plain", 1), ("emu", "plain", 2), pytest.param("engine", "plain", 1, marks=pytest.mark.gpu),
         pytest.param("engine", "compact", 1, marks=pytest.mark.gpu),
         pytest.param("engine", "plain", 2, marks=pytest.mark.gpu),
         pytest.param("engine", "compact", 2, marks=pytest.mark.gpu)]


@pytest.mark.parametrize("backend,fmt,depth", TIGHT)
@pytest.mark.parametrize("mode", ["chased", "routed"])
def test_tight_output_buffers(backend, fmt, depth, mode):
    """every call gets 0 .. all of the buffer space it needs; what RA_E_CAPACITY reports must be exactly what a
    fetch needs, and a call in flight behind it must change nothing"""
    G, m = (48, 5) if backend == "emu" else (1200, 5)
    rng = random.Random(9800 + 10 * depth + (fmt == "compact") + 100 * (mode == "routed"))
    o, b = Oracle(G, m, **kw(mode)), make_backend(backend, G, m, **kw(mode))
    if fmt == "compact":
        b.set_note_format(True)
    api = "submit" if backend == "engine" else "submit_host"      # (tests/test_nif_shim.py takes the emulation's submit)
    cov = _chain(b, o, m, G, mode, api, rng, rounds=2, steps=6, depth=depth, tight=True, compact=fmt == "compact")
    assert cov["capacity"] > 0
    if depth == 2:
        assert cov["pending"] > 0
