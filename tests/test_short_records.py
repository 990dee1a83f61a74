"""CPU tier: the 16-byte short form of the record planes (ra_b200/csrc/raft_logic.cuh, "record planes").

A record whose fields fit is stored in chunk 0 of its tile alone; everything else keeps the 32-byte head or the
64-byte long form.  Checked here through the host emulation of the device logic: round trips through both index
widths at every limit of the short form, stale bytes in chunks 1..3 of the tile, and -- at the shapes of the
benchmark's configurations -- that every record the steady state writes into a plane is short."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest

from ra_b200 import abi

SHORT, HEAD, LONG = 0, 1, 3          # what st_rec_plane reports: nothing but chunk 0 / chunks 0-1 / chunks 0-3
NARROW_LIMIT = 1 << 30
_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu", "plane_stats.cpp")
_lib_cache = []


def _lib():
    """tests/emu/plane_stats.cpp: the host emulation built with per-form store counters, compiled on first use into a
    temporary directory (the tree is left as it is)."""
    if _lib_cache:
        return _lib_cache[0]
    d = tempfile.mkdtemp(prefix="ra_plane_stats_")
    atexit.register(shutil.rmtree, d, True)
    so = os.path.join(d, "libra_plane_stats.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-fPIC", "-shared", "-Wl,-Bsymbolic",
                           "-Wl,--no-undefined", "-o", so, _SRC])
    l = C.CDLL(so)
    f = l.ra_emu_codec_roundtrip2
    f.restype = C.c_int
    f.argtypes = [C.POINTER(abi.RaEvent), C.c_int, C.POINTER(abi.RaEvent), C.POINTER(C.c_int),
                  C.POINTER(abi.RaEvent), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    l.ra_emu_plane_forms.restype = None
    l.ra_emu_plane_forms.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    l.ra_emu_flood_faults.restype = C.c_int
    l.ra_emu_flood_faults.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64,
                                      C.POINTER(abi.RaFloodFaults)]
    _lib_cache.append(l)
    return l


class StatsEmu(abi.Backend):
    """The emulation of the plane-stats build (same entry points as tests/emu_lib.Emu)."""
    name = "emu_stats"

    def __init__(self, n_groups: int, n_members: int, **kw):
        super().__init__(_lib(), "ra_emu", n_groups, n_members, **kw)

    def flood(self, n_steps, cmds, permille, seed, faults=None):
        ff = C.byref(abi.RaFloodFaults(*faults)) if faults else None
        self._check(_lib().ra_emu_flood_faults(self._h, n_steps, cmds, permille, seed, ff), "flood_faults")


def _fields(e):
    return (e.type, e.from_slot, e.flags, e.n, e.n1, e.term, e.a, e.b, e.c, e.d, e.e)


def roundtrip(e, want_form):
    """Store e through both passes over tiles full of stale bytes; every field the logic reads comes back."""
    l = _lib()
    fits_narrow = max(e.term, e.a, e.b, e.c, e.d, e.e) < NARROW_LIMIT
    for fill in (0x00, 0xA5, 0xFF):
        ow, on = abi.RaEvent(), abi.RaEvent()
        form, fits, form_n = C.c_int(-1), C.c_int(-1), C.c_int(-1)
        assert l.ra_emu_codec_roundtrip2(C.byref(e), fill, C.byref(ow), C.byref(form), C.byref(on), C.byref(fits),
                                         C.byref(form_n)) == 0
        assert form.value == want_form, (fill, _fields(e))
        assert _fields(ow) == _fields(e) and ow._pad == 0, (fill, _fields(ow), _fields(e))
        # the narrow pass refuses every record with a field >= 2^30, in any form
        assert fits.value == (1 if fits_narrow else 0), (fill, _fields(e))
        if fits_narrow:
            assert form_n.value == want_form
            assert _fields(on) == _fields(e) and on._pad == 0, (fill, _fields(on), _fields(e))


@pytest.mark.parametrize("v,form", [(2**30 - 1, SHORT), (2**30, SHORT), (2**32 - 1, SHORT), (2**32, HEAD)])
def test_value_limits(v, form):
    roundtrip(abi.ev_written(3, v, 5, 6), form)                               # term
    roundtrip(abi.ev_written(3, 5, v, 6), form)                               # x
    roundtrip(abi.ev_written(3, 5, 6, v), form)                               # y
    roundtrip(abi.ev_aer(3, 1, v, 100, v, 98, [v, v]), form)                   # RS_AER: b, d rebuilt from term
    roundtrip(abi.ev_aer(3, 1, 9, 100, 9, v, [9]), form)                       # RS_AER: leader_commit in y
    roundtrip(abi.ev_aer_reply(3, 2, v, True, 104, 103, v), form)              # RS_REPLY: c rebuilt from term
    roundtrip(abi.ev_aer_reply(3, 2, 9, False, v, 103, 9), form)


@pytest.mark.parametrize("field", ["n", "n1"])
@pytest.mark.parametrize("v,form", [(255, SHORT), (256, HEAD), (65535, HEAD)])
def test_count_limits(field, v, form):
    e = abi.RaEvent(row=7, type=abi.EV_COMMAND, from_slot=abi.RA_NO_SLOT)
    setattr(e, field, v)
    roundtrip(e, form)
    roundtrip(abi.ev_aer(7, 2, 9, 100, 9, 98, [9] * 255), SHORT)
    roundtrip(abi.ev_aer(7, 2, 9, 100, 9, 98, [9] * 256), HEAD)


@pytest.mark.parametrize("frm,form", [(0, SHORT), (7, SHORT), (8, HEAD), (14, HEAD), (15, HEAD), (254, HEAD),
                                      (255, SHORT)])
def test_from_limits(frm, form):
    roundtrip(abi.ev_aer_reply(3, frm, 9, True, 104, 103, 9), form)
    roundtrip(abi.RaEvent(row=3, type=abi.EV_REQUEST_VOTE, from_slot=frm, term=9, a=100, b=9), form)


@pytest.mark.parametrize("bit", range(8))
def test_flag_bits(bit):
    e = abi.ev_command(5, 3)
    e.flags = 1 << bit
    roundtrip(e, SHORT if bit < 4 else HEAD)


def test_type_limits_and_long_form():
    for t in range(16):
        roundtrip(abi.RaEvent(row=1, type=t, from_slot=3, term=4, a=5, b=6), SHORT)
    roundtrip(abi.RaEvent(row=1, type=16, from_slot=3, term=4, a=5, b=6), HEAD)
    roundtrip(abi.RaEvent(row=1, type=200, from_slot=3, term=4, a=5, b=6), HEAD)
    # anything with a tail keeps the long form, whatever its magnitudes
    roundtrip(abi.ev_aer(3, 1, 9, 100, 8, 98, [9]), LONG)
    roundtrip(abi.ev_pre_vote(3, 1, 9, 77, 100, 9), LONG)
    roundtrip(abi.ev_aer(3, 1, 2**40, 100, 8, 98, [9]), LONG)


def test_random_records_roundtrip():
    import random
    rng = random.Random(11)
    vals = [0, 1, 2**30 - 1, 2**30, 2**32 - 1, 2**32, 2**64 - 1]
    l = _lib()
    for _ in range(5000):
        t = rng.choice(vals + [rng.getrandbits(rng.choice([8, 31, 33]))])
        e = abi.RaEvent(row=rng.randrange(1 << 20), type=rng.randrange(20), from_slot=rng.choice([0, 5, 7, 8, 15, 255]),
                        flags=rng.choice([0, 1, 2, 8, 15, 16, 0x80]), n=rng.choice([0, 1, 255, 256]),
                        n1=rng.choice([0, 255, 256]), term=t, a=rng.choice(vals), b=rng.choice([t, 0, rng.choice(vals)]),
                        c=rng.choice([t, 0, rng.choice(vals)]), d=rng.choice([0, 1, t]), e=rng.choice([0, 0, 5]))
        ow, on = abi.RaEvent(), abi.RaEvent()
        form, fits, form_n = C.c_int(-1), C.c_int(-1), C.c_int(-1)
        assert l.ra_emu_codec_roundtrip2(C.byref(e), rng.randrange(256), C.byref(ow), C.byref(form), C.byref(on),
                                         C.byref(fits), C.byref(form_n)) == 0
        assert _fields(ow) == _fields(e)
        if fits.value:
            assert _fields(on) == _fields(e) and form_n.value == form.value
        if form.value == SHORT:
            assert max(e.term, e.a, e.b, e.c, e.d, e.e) < 2**32 and e.n < 256 and e.n1 < 256 and e.flags < 16


def plane_forms():
    arr = (C.c_ulonglong * 64)()
    _lib().ra_emu_plane_forms(arr, 1)
    return {t: (arr[4 * t + SHORT], arr[4 * t + HEAD], arr[4 * t + LONG]) for t in range(16)}


# the benchmark's configurations 3, 4 and 5 at a size the emulation runs in seconds
SHAPES = [
    dict(groups=300, members=5, cmds=1, permille=10, faults=None),           # AppendEntries + 1 % election timeouts
    dict(groups=300, members=5, cmds=64, permille=10, faults=None),          # 64-entry pipelined AppendEntries
    dict(groups=150, members=7, cmds=1, permille=0, faults=(5, 20, 10, 32)), # losses, lagging fsync, partitions
]


@pytest.mark.parametrize("shape", SHAPES, ids=["config3", "config4", "config5"])
def test_steady_state_records_are_written_short(shape):
    e = StatsEmu(shape["groups"], shape["members"], route_on_device=True)
    e.reset_empty()
    e.step([abi.ev_simple(e.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(shape["groups"])])
    e.flood(20, shape["cmds"], shape["permille"], seed=0xA03, faults=shape["faults"])
    plane_forms()                                                              # reset
    e.flood(60, shape["cmds"], shape["permille"], seed=0xA03, faults=shape["faults"])
    forms = plane_forms()
    # no record without a tail needed more than chunk 0: every AppendEntries of the leader's term, every reply,
    # written and command event (and every vote record without a tail) was written short
    assert all(h == 0 for _, h, _ in forms.values()), forms
    for t in (abi.EV_AER, abi.EV_AER_REPLY, abi.EV_WRITTEN, abi.EV_COMMAND):
        short, _, long_ = forms[t]
        assert short > 0, (t, forms[t])
    aer_short, _, aer_long = forms[abi.EV_AER]
    assert aer_long < 0.05 * aer_short, forms[abi.EV_AER]                    # the long ones follow leader changes
    assert e.counters()["commits"] > 0
