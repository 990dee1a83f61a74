"""SURVEY 8f-2: the written-event source.  ra_wal_batch_to_events (host code of the product library,
callable without a GPU) turns one WAL batch -- {written, Term, Seq} per writer, ra_log_wal.erl:784-808 --
into the grouped event array of step(); applied through the oracle and through the host build of the
device logic it must leave what ra_log:handle_event/2 (ra_log.erl:849-896) leaves for the whole seq."""
import ctypes as C

import pytest

from emu_lib import Emu
from oracle_lib import Oracle
from ra_b200 import abi
from ra_b200.engine import host
from ra_suite import base_state, make_backend


def batch_events(writers, max_per_row=abi.RA_LOCAL_CAP, cap=1024):
    """writers: [(row, term, [(from, to), ...])] -> list of per-step event lists"""
    keep = []
    arr = (abi.RaWalWriter * len(writers))()
    for i, (row, term, ranges) in enumerate(writers):
        flat = (C.c_uint64 * (2 * len(ranges)))(*[x for r in ranges for x in r])
        keep.append(flat)
        arr[i] = abi.RaWalWriter(row, len(ranges), term, flat)
    res = abi.RaWalResume(0, 0)
    out = (abi.RaEvent * cap)()
    steps = []
    while res.writer < len(writers):
        n = host().wal_batch_to_events(arr, len(writers), max_per_row, out, cap, C.byref(res))   # no device needed
        assert n > 0
        steps.append([abi.RaEvent.from_buffer_copy(bytes(out[i])) for i in range(n)])
    return steps


def test_conversion_groups_rows_and_respects_caps():
    steps = batch_events([(3, 5, [(1, 3), (7, 9)]), (1, 5, [(4, 4)]), (2, 6, [(1, 1), (3, 3), (5, 5), (7, 7), (9, 9)])])
    assert len(steps) == 2
    s0 = [(e.row, e.type, e.term, e.a, e.b) for e in steps[0]]
    assert s0 == [(3, abi.EV_WRITTEN, 5, 1, 3), (3, abi.EV_WRITTEN, 5, 7, 9), (1, abi.EV_WRITTEN, 5, 4, 4),
                  (2, abi.EV_WRITTEN, 6, 1, 1), (2, abi.EV_WRITTEN, 6, 3, 3), (2, abi.EV_WRITTEN, 6, 5, 5),
                  (2, abi.EV_WRITTEN, 6, 7, 7)]
    assert [(e.row, e.a, e.b) for e in steps[1]] == [(2, 9, 9)]
    # a writer that changed term mid-batch: two notifications, one run of its row, one cap
    steps = batch_events([(4, 5, [(1, 2), (3, 3), (4, 4)]), (4, 6, [(5, 5), (6, 6)])])
    assert [len(s) for s in steps] == [4, 1] and all(e.row == 4 for s in steps for e in s)


@pytest.mark.parametrize("be", ["oracle", "emu"])
def test_seq_with_gap_ends_at_the_highest_matching_index(be):
    """{written, 5, [{4,5},{7,8}]} on a follower whose entries 4..8 are of term 5: last_written = {8,5};
    the same seq for term 4 matches nothing (ra_log:handle_event walks the whole seq down, :884-895)."""
    b = make_backend(be, 1, 3, pure=True)
    st = base_state(3)
    abi.set_log(st, [(0, 0), (1, 1), (2, 3), (3, 5), (4, 5), (5, 5), (6, 5), (7, 5), (8, 5)], last_written=(3, 5))
    st.role = abi.FOLLOWER
    st.leader_slot = 1
    for term, want in ((5, (8, 5)), (4, (3, 5))):
        b.load_rows([st])
        for evs in batch_events([(st.row, term, [(4, 5), (7, 8)])]):
            b.step(evs)
        r = b.read_rows([st.row])[0]
        assert (r.last_written_index, r.last_written_term) == want


def test_flood_driven_by_wal_batches_equals_per_note_written_events():
    """One WAL batch per step built from the step's WAL_APPEND notes (what ra_log_wal does with the
    appends of all its writers) drives the same cluster to the same state as the per-note events."""
    g, m, steps = 40, 3, 40
    a, b = Oracle(g, m, route_on_device=True), Emu(g, m, route_on_device=True)
    for be in (a, b):
        be.reset_empty()
        msgs, notes = be.step([abi.ev_simple(be.row_of(i, 0), abi.EV_ELECTION_TIMEOUT) for i in range(g)])
        for _ in range(steps):
            writers, roles = {}, {}
            for n in notes:
                if n.type == abi.NOTE_WAL_APPEND:
                    writers.setdefault((n.row, n.c), []).append((n.a, n.b))
            evs = []
            for batch in batch_events([(row, term, rs) for (row, term), rs in sorted(writers.items())]) or [[]]:
                evs += batch
            # leaders get one client command per step, after their written events (row-adjacent)
            by_row = {}
            for e in evs:
                by_row.setdefault(e.row, []).append(e)
            for r in be.read_rows(range(be.n_rows)):
                if r.role == abi.LEADER:
                    by_row.setdefault(r.row, []).append(abi.ev_command(r.row, 1))
            flat = [e for row in sorted(by_row) for e in by_row[row][:abi.RA_LOCAL_CAP]]
            msgs, notes = be.step(flat)
    ra, rb = [r.key() for r in a.read_rows(range(a.n_rows))], [r.key() for r in b.read_rows(range(b.n_rows))]
    assert ra == rb and a.counters() == b.counters()
    assert a.counters()["commits"] > 0


@pytest.mark.parametrize("be", ["oracle", "emu", pytest.param("engine", marks=pytest.mark.gpu)])
def test_step_host_equals_step(be):
    """ra_engine_step_host: the same batch as 32-byte host events leaves the same records, notes and rows."""
    g, m = 24, 3
    outs = []
    for use_host in (False, True):
        b = make_backend(be, g, m, route_on_device=True)
        b.reset_empty()
        res = []
        evs = [abi.ev_simple(b.row_of(i, 0), abi.EV_ELECTION_TIMEOUT) for i in range(g)]
        for _ in range(25):
            msgs, notes = (b.step_host if use_host else b.step)(evs)
            res.append(([x.key() for x in msgs], [x.key() for x in notes]))
            evs = []
            by_row = {}
            for n in notes:
                if n.type == abi.NOTE_WAL_APPEND:
                    by_row.setdefault(n.row, []).append(abi.ev_written(n.row, n.c, n.a, n.b))
            for r in b.read_rows(range(b.n_rows)):
                if r.role == abi.LEADER:
                    by_row.setdefault(r.row, []).append(abi.ev_command(r.row, 2))
            for row in sorted(by_row):
                evs += by_row[row][:abi.RA_LOCAL_CAP]
        outs.append((res, [r.key() for r in b.read_rows(range(b.n_rows))], b.counters()))
    assert outs[0] == outs[1]
    assert outs[0][2]["commits"] > 0
    b = make_backend(be, g, m)
    with pytest.raises(abi.RaError) as ei:                      # an RPC is not a host event
        b.step_host([abi.ev_aer(0, 1, 1, 0, 0, 0, [])])
    assert ei.value.status == abi.RA_E_INVAL
