"""CPU tier: the engine's DEVICE LOGIC (ra_b200/csrc/raft_step.cuh + raft_row.cuh, compiled for the
host by tests/emu/) against the oracle, with the inputs of the `-m gpu` parity tests.

What this covers: every handler / fast path / codec / end-of-step line the GPU executes, driven
with the control flow of the two step kernels.  What it does not: the kernels' own frame (TMA
ring, warp reductions, launches) -- tests/test_parity_gpu.py does that on an H100.
"""
import ctypes as C

import pytest

import trace_gen
from emu_lib import Emu
from fuzz_lib import bootstrap, first_row
from oracle_lib import Oracle
from ra_b200 import abi

TRACES = [
    (8, 3, 150, 11, {}),
    (16, 5, 300, 7, {}),
    (12, 7, 250, 3, dict(p_drop=0.05, p_withhold_written=0.1)),
    (32, 5, 200, 5, dict(p_timeout=0.04, p_adversarial=0.05)),
    (4, 1, 60, 2, {}),
    (10, 8, 120, 13, dict(p_drop=0.0, p_dup=0.0, p_delay=0.0, p_adversarial=0.0)),
    (6, 5, 200, 17, dict(max_cmd=200, p_cmd=0.9)),
    (300, 7, 60, 29, dict(p_drop=0.005, p_withhold_written=0.02, p_timeout=0.003, p_dup=0.0, p_adversarial=0.0)),
    (24, 5, 250, 41, dict(p_query=0.3, p_timeout=0.02)),          # consistent queries: heartbeat rounds in the loop
]


@pytest.mark.parametrize("g,m,steps,seed,knobs", TRACES)
def test_trace_parity_emu(g, m, steps, seed, knobs):
    batches = trace_gen.generate(lambda gg, mm: Oracle(gg, mm), g, m, steps, seed, **knobs)
    want, want_rows, want_cnt = trace_gen.replay(Oracle(g, m), batches)
    got, got_rows, got_cnt = trace_gen.replay(Emu(g, m), batches)
    for t, (w, x) in enumerate(zip(want, got)):
        assert x[0] == w[0], "RPC records differ at step %d" % t
        assert x[1] == w[1], "host notes differ at step %d" % t
    assert got_rows == want_rows
    assert got_cnt == want_cnt


def test_trace_parity_emu_small_pipeline_window():
    kw = dict(max_pipeline_count=8, max_aer_batch=3)
    batches = trace_gen.generate(lambda gg, mm: Oracle(gg, mm, **kw), 8, 5, 250, 23, max_cmd=9, p_cmd=0.9)
    want = trace_gen.replay(Oracle(8, 5, **kw), batches)
    got = trace_gen.replay(Emu(8, 5, **kw), batches)
    assert got == want


FLOODS = [
    (64, 3, 60, 1, 0),
    (1000, 5, 80, 1, 0),
    (1000, 5, 120, 2, 10),
    (500, 7, 100, 1, 20),
    (333, 1, 20, 3, 0),
    (200, 5, 150, 64, 30),     # 64-entry commands (config 4 shape), frequent elections
]


@pytest.mark.parametrize("g,m,steps,cmds,permille", FLOODS)
def test_flood_parity_emu(g, m, steps, cmds, permille):
    o = Oracle(g, m, route_on_device=True)
    e = Emu(g, m, route_on_device=True)
    for b in (o, e):
        bootstrap(b)
    for part in (steps // 3, steps - steps // 3):
        o.flood(part, cmds, permille, seed=42, threads=2)
        e.flood(part, cmds, permille, seed=42)
    assert e.counters() == o.counters()
    assert o.counters()["commits"] > 0
    ro, re_ = o.rows_bytes(), e.rows_bytes()
    assert re_ == ro, "first differing row: %d" % first_row(ro, re_)


def test_emu_fast_paths_carry_the_steady_state():
    """The stall histogram of the emulated step kernel: in a clean flood well under 1 % of the events
    leave the fast paths once leaders are elected (what keeps raft_general_kernel at ~3 % of a step)."""
    e = Emu(500, 5, route_on_device=True)
    bootstrap(e)
    e.flood(30, 1, 0, seed=3)
    h0, ev0 = sum(e.stall_histogram().values()), e.counters()["events"]
    e.flood(50, 1, 0, seed=3)
    h1, ev1 = sum(e.stall_histogram().values()), e.counters()["events"]
    assert ev1 - ev0 > 50 * 500 * 5
    assert (h1 - h0) <= 0.01 * (ev1 - ev0)


def test_emu_step_input_validation():
    e = Emu(4, 3)
    r0, r1 = e.row_of(0, 0), e.row_of(1, 0)
    with pytest.raises(abi.RaError) as ei:
        e.step([abi.ev_command(r0), abi.ev_command(r1), abi.ev_command(r0)])
    assert ei.value.status == abi.RA_E_UNGROUPED
    with pytest.raises(abi.RaError) as ei:
        e.step([abi.ev_command(r0) for _ in range(abi.RA_LOCAL_CAP + 1)])
    assert ei.value.status == abi.RA_E_CAPACITY
    with pytest.raises(abi.RaError) as ei:
        e.step([abi.ev_command(10_000)])
    assert ei.value.status == abi.RA_E_INVAL
    # a sender slot a row cannot hold (15..254), through step and through submit / collect
    bad = [abi.ev_command(r0), abi.ev_request_vote(r1, 17, 1, 0, 0)]
    with pytest.raises(abi.RaError) as ei:
        e.step(bad)
    assert ei.value.status == abi.RA_E_INVAL
    st, ticket = e.submit(bad, 64, 64)
    assert st == abi.RA_OK and e.collect(ticket)[0] == abi.RA_E_INVAL
    msgs, notes = e.step([])
    assert msgs == [] and notes == []
    assert e.counters()["events"] == 0
    # a batch in more than 256 pieces
    st, _ = e.submit_host_segs([[] for _ in range(257)], 64, 64)
    assert st == abi.RA_E_INVAL
    # reset_empty drops outputs that did not fit
    with pytest.raises(abi.RaError) as ei:
        e.step([abi.ev_simple(r0, abi.EV_ELECTION_TIMEOUT)], msgs_cap=0, notes_cap=0)
    assert ei.value.status == abi.RA_E_CAPACITY
    e.reset_empty()
    assert e.step([]) == ([], [])
    # note budgets outside RA_NOTE_RESERVE + 2 .. RA_NOTE_CAP
    for cap in (abi.RA_NOTE_RESERVE + 1, abi.RA_NOTE_CAP + 1):
        with pytest.raises(abi.RaError) as ei:
            Emu(4, 3, note_cap=cap)
        assert ei.value.status == abi.RA_E_INVAL


@pytest.mark.parametrize("threads", ["1", "4"])
def test_host_driven_flood_equals_device_flood_emu(threads, monkeypatch):
    """ra_hostsim_run (the product's host-side caller, every step through step() with host buffers)
    leaves exactly the rows the device-side flood leaves, and both equal the oracle -- the CPU twin
    of tests/test_parity_gpu.py::test_host_driven_flood_equals_device_flood."""
    from ra_b200.engine import HostFlood
    monkeypatch.setenv("RA_HOSTSIM_THREADS", threads)
    g, m, steps = 1200, 5, 70
    a = Emu(g, m, route_on_device=True)
    b = Emu(g, m, route_on_device=True)
    o = Oracle(g, m, route_on_device=True)
    bootstrap(a)
    a.flood(steps, 1, 10, seed=5)
    bootstrap(o)
    o.flood(steps, 1, 10, seed=5, threads=2)
    b.reset_empty()
    hf = HostFlood(b)
    st = hf.run(steps, 1, 10, seed=5, bootstrap=True)
    assert st["h2d_bytes"] > 0 and st["d2h_bytes"] > 0 and st["engine_calls"] == steps + 1
    ca, cb, co = a.counters(), b.counters(), o.counters()
    assert ca == co
    for k in ("events", "commits", "applied", "msgs_out", "elections_won"):
        assert cb[k] == ca[k]
    assert b.rows_bytes() == a.rows_bytes()
    hf.close()


SHARDED = [
    # shards, members, local groups per slot, steps, election permille, commands per leader and step
    (2, 5, 96, 60, 10, 1),
    (4, 3, 64, 50, 0, 1),
    (8, 5, 32, 60, 20, 1),
    (3, 7, 40, 50, 10, 1),
    (8, 5, 64, 60, 10, 64),   # the config-4-shaped case of tests/test_sharded_gpu.py
]


@pytest.mark.parametrize("n,m,gl,steps,permille,cmds", SHARDED)
def test_sharded_emu_equals_unsharded_oracle(n, m, gl, steps, permille, cmds):
    """Members of a group on different shards (bucket transport: emit into per-destination buckets,
    exchange, deliver) must leave every member identical to the UNSHARDED oracle run -- the CPU twin
    of tests/test_sharded_gpu.py, same device logic."""
    from emu_lib import EmuShards
    fl = EmuShards(n, gl, m)
    fl.bootstrap()
    fl.run(steps, cmds, permille, seed=77)
    g = n * gl
    o = Oracle(g, m, route_on_device=True)
    bootstrap(o)
    o.flood(steps, cmds, permille, seed=77, threads=2)
    want = {r.row: r.key()[1:] for r in o.read_rows(range(o.n_rows))}
    seen = 0
    for k, s in enumerate(fl.shards):
        for r in s.read_rows(range(s.n_rows)):
            assert r.key()[1:] == want[fl.global_row(k, r.row)], (k, r.row)
            seen += 1
    assert seen == g * m
    co, ce = o.counters(), fl.counters()
    for key in ("events", "commits", "applied", "msgs_out", "msgs_dropped", "elections_won", "fatal_rows"):
        assert ce[key] == co[key], key
    assert co["commits"] > 0 and co["msgs_dropped"] == 0


def test_record_plane_codec_is_lossless():
    """The 32-byte head / optional tail re-encoding of the record planes (raft_step.cuh: st_rec_plane,
    rec_decode): every field the logic reads comes back bit-identical for arbitrary records, the shapes
    the steady state relies on really are heads only, and stale bytes of the tile never leak."""
    import random
    from emu_lib import extras
    roundtrip = extras().codec_roundtrip
    rng = random.Random(7)
    big = [0, 1, 2, 5, 2**32 - 1, 2**32, 2**63, 2**64 - 1]

    def val():
        return rng.choice(big) if rng.random() < 0.5 else rng.getrandbits(rng.choice([3, 16, 40, 64]))

    def check(e, want_tail=None):
        out, tail = abi.RaEvent(), C.c_int(-1)
        assert roundtrip(C.byref(e), C.byref(out), C.byref(tail)) == 0
        # row and seq are positional inside a plane (the reader knows them), _pad is scratch
        got = (out.type, out.from_slot, out.flags, out.n, out.n1, out.term, out.a, out.b, out.c, out.d, out.e)
        exp = (e.type, e.from_slot, e.flags, e.n, e.n1, e.term, e.a, e.b, e.c, e.d, e.e)
        assert got == exp and out._pad == 0
        if want_tail is not None:
            assert bool(tail.value) == want_tail
    for _ in range(20000):
        t = val()
        e = abi.RaEvent(row=rng.randrange(1 << 20), type=rng.randrange(16), from_slot=rng.choice([0, 3, 7, 255]),
                        flags=rng.choice([0, 1, 2, 8, 11]), n=rng.randrange(1 << 16), n1=rng.randrange(1 << 16),
                        term=t, a=val(), b=rng.choice([t, val()]), c=rng.choice([t, 0, val()]),
                        d=rng.choice([0, 1, t, val()]), e=rng.choice([0, 0, val()]))
        check(e)
    # the steady-state shapes are heads only; anything else carries a tail
    check(abi.ev_aer(3, 1, 9, 100, 9, 98, [9, 9, 9]), want_tail=False)          # entries of the leader's term
    check(abi.ev_aer(3, 1, 9, 100, 9, 98, []), want_tail=False)                  # empty AER (commit update)
    check(abi.ev_aer_reply(3, 2, 9, True, 104, 103, 9), want_tail=False)
    check(abi.ev_written(3, 9, 101, 103), want_tail=False)
    check(abi.ev_command(3, 64), want_tail=False)
    check(abi.ev_aer(3, 1, 9, 100, 8, 98, [9]), want_tail=True)                  # prev entry of an older term
    check(abi.ev_aer(3, 1, 9, 100, 9, 98, [8, 9]), want_tail=True)               # two term runs
    check(abi.ev_pre_vote(3, 1, 9, 77, 100, 9), want_tail=True)
