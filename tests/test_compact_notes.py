"""Compact note stream (include/ra_engine.h: ra_note16, ra_engine_set_note_format, ra_notes16_expand): 16-byte units
instead of 32-byte notes on the device->host path.  The decoder must rebuild exactly the notes the plain format
carries; in the steady-state flood every note is one unit."""
import ctypes as C

import pytest

from ra_b200 import abi
from ra_b200.engine import notes16_expand
from ra_suite import *  # noqa: F401,F403


def test_expand_hand_made_units():
    """host code only (no GPU): units + extension area -> notes, including the per-row WAL_APPEND term memory"""
    U = abi.RaNote16
    units = (U * 8)()
    # row 3: WAL_APPEND 10..12 with an explicit term (extension 0), then WAL_APPEND 13..13 "same term", APPLY 9..12
    units[0] = U(3, NOTE_WAL_APPEND | abi.N16_EXT, 0, 0, 0)
    units[1] = U(3, NOTE_WAL_APPEND | abi.N16_SAME_TERM, 0, 0, 13)
    units[2] = U(3, NOTE_APPLY, 3, 0x0004, 9)
    # row 5: a STATUS note (slot 2, c != 0): extension 1
    units[3] = U(5, NOTE_STATUS | abi.N16_EXT, 2, 0x0003, 1)
    ext = (C.c_uint64 * 8).from_buffer(units, 4 * C.sizeof(U))
    ext[0], ext[1], ext[2], ext[3] = 10, 12, 7, 0            # {a, b}, {c, 0}
    ext[4], ext[5], ext[6], ext[7] = 99, 0x03000102, 6, 0
    last_c = (C.c_uint64 * 8)()
    got = [(n.row, n.type, n.slot, n.aux, n.a, n.b, n.c) for n in notes16_expand(units, 4, 2, last_c)]
    assert got == [(3, NOTE_WAL_APPEND, 0, 0, 10, 12, 7), (3, NOTE_WAL_APPEND, 0, 0, 13, 13, 7),
                   (3, NOTE_APPLY, 0, 4, 9, 12, 0), (5, NOTE_STATUS, 2, 3, 99, 0x03000102, 6)]
    assert last_c[3] == 7


def _cluster(groups=48, members=3):
    from ra_b200.engine import Engine
    b = Engine(groups, members)
    b.reset_empty()
    return b


@pytest.mark.gpu
def test_compact_stream_carries_the_same_notes():
    ref = _cluster()
    cp = _cluster()
    cp.set_note_format(True)
    stats = dict(units=0, ext=0, notes=0)

    def compact_step(evs):
        msgs, notes, units, n_ext = cp.step_compact(evs)
        stats["notes"] += len(notes); stats["ext"] += n_ext; stats["units"] += len(units)
        return msgs, notes
    want = closed_loop(ref, 30, lambda evs: ref.step(evs))
    got = closed_loop(cp, 30, compact_step)
    assert got == want
    assert [r.key() for r in cp.read_rows(range(cp.n_rows))] == [r.key() for r in ref.read_rows(range(ref.n_rows))]
    assert stats["notes"] > 500 and stats["ext"] < stats["notes"] // 3     # most notes are one unit


@pytest.mark.gpu
def test_host_driven_flood_compact_equals_plain(monkeypatch):
    """ra_hostsim_run with notes as 16-byte units leaves the rows the plain format leaves, at ~half the D2H bytes"""
    from ra_b200.engine import Engine, HostFlood
    res = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("RA_HOSTSIM_COMPACT", mode)
        e = Engine(3000, 5, route_on_device=True)
        e.reset_empty()
        hf = HostFlood(e)
        st = hf.run(60, 1, 10, seed=5, bootstrap=True)
        res[mode] = ([r.key() for r in e.read_rows(range(0, e.n_rows, 7))], e.counters(), st["d2h_bytes"])
        hf.close(); e.close()
    assert res["0"][0] == res["1"][0]
    for k in ("events", "commits", "applied", "msgs_out", "elections_won"):
        assert res["0"][1][k] == res["1"][1][k]
    assert res["1"][2] < 0.62 * res["0"][2]
