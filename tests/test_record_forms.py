"""Head and long records in every specialisation of the hot kernel (ra_b200/csrc/raft_step_kernel.cuh).

The hot kernel fetches 512 B of a record tile when the size flags that travel with the record counts say that every
record of it is short, 1 KB when none has a tail, and 2 KB otherwise; past that, its staging slot holds an earlier
tile's bytes.  The flags are set by emit_msg (local and peer stores), row_end_of_step (also after a stall, from
StallCtx::wk_hi), deliver_record, both forms of ingest_kernel and the flood host model.  Every case here makes
records of 256 or more entries (stored as 32-byte heads) and records with a tail (64-byte long form) share tiles with
short ones, and compares the result with the oracle bit for bit: counters and raw row state, for traces and scripted
steps also every record and note.

CPU tier: the host emulation (tests/emu) reads the bytes the kernel would not have fetched as poison and counts every
record it decoded from them (Emu.underfetched), so a lost flag shows there.  Each case has a twin at reduced size on
the plane-stats build (emu_lib.stats_lib()) that asserts the precondition: the targeted records really were
stored as heads (or long).  GPU tier: the same cases on the engine, with the 32-bit (RA_STEP_WIDE=0) and the 64-bit
(RA_STEP_WIDE=1) hot kernel.
"""
import functools
from collections import defaultdict

import pytest

import trace_gen
from emu_lib import Emu, EmuShards, plane_forms, stats_lib
from fuzz_lib import WIDTHS, bootstrap, first_row
from oracle_lib import Oracle
from ra_b200 import abi
from ra_suite import make_backend

BACKENDS = ["emu", pytest.param("engine", marks=pytest.mark.gpu)]
PERMILLE, SEED = 15, 0x5EC


@pytest.fixture(autouse=True)
def _poison_and_underfetch():
    """The emulation's cases alternate the two poison patterns (by pass, see _make) and must end without a record
    decoded from bytes the kernel did not fetch; every test starts with both libraries' counts at zero."""
    Emu.underfetched()
    Emu.underfetched(library=stats_lib())
    yield
    Emu.set_fetch_poison(0)


def _make(name, wide, monkeypatch, groups, members, **kw):
    monkeypatch.setenv("RA_STEP_WIDE", wide)
    if name == "emu":
        Emu.set_fetch_poison(int(wide))
    return make_backend(name, groups, members, **kw)


def _check_fetch(name):
    if name == "emu":
        assert Emu.underfetched() == 0, "the hot path decoded a record from bytes its tile's fetch did not cover"


def _same_rows(got, want):
    a, b = got.rows_bytes(), want.rows_bytes()
    assert a == b, "first differing row: %d" % first_row(a, b)


def _keys(out):
    msgs, notes = out
    return [m.key() for m in msgs], [n.key() for n in notes]


# ---- floods: mailbox planes (emit_msg, row_end_of_step) and host planes (the flood host model) ----------------------
FLOODS = [
    # members, commands per step, max_aer_batch, faults
    (5, 255, 512, None),                  # control: every record short
    (5, 256, 512, None),                  # a head COMMAND, head AppendEntries of 256 entries
    (5, 300, 128, None),                  # a head COMMAND, AppendEntries of 128 + 128 + 44 entries: mailbox depth 3
    (3, 300, 1024, None),                 # the narrow M = 3 kernel
    (7, 300, 1024, None),                 # the narrow M = 7 kernel
    (4, 300, 512, None),                  # the runtime-M kernel
    (8, 300, 512, None),
    (7, 300, 512, (5, 20, 10, 32)),       # the fault kernels: catch-up AppendEntries spanning two term runs
    (5, 300, 512, (20, 50, 30, 16)),
]
FLOOD_IDS = ["m%d-c%d-b%d%s" % (m, c, b, "-faults" if f else "") for m, c, b, f in FLOODS]


def _flood(b, o, steps, cmds, faults):
    for x in (o, b):
        bootstrap(x)
    o.flood(steps, cmds, PERMILLE, seed=SEED, threads=4, faults=faults)
    b.flood(steps, cmds, PERMILLE, seed=SEED, faults=faults)


@pytest.mark.parametrize("wide", WIDTHS)
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("members,cmds,batch,faults", FLOODS, ids=FLOOD_IDS)
def test_flood_with_head_and_long_records(members, cmds, batch, faults, backend, wide, monkeypatch):
    groups, steps = (1500, 60) if backend == "engine" else (64, 40)
    b = _make(backend, wide, monkeypatch, groups, members, route_on_device=True, max_aer_batch=batch)
    o = Oracle(groups, members, route_on_device=True, max_aer_batch=batch)
    _flood(b, o, steps, cmds, faults)
    assert b.counters() == o.counters()
    assert o.counters()["commits"] > 0
    _same_rows(b, o)
    _check_fetch(backend)


@pytest.mark.parametrize("members,cmds,batch,faults", FLOODS, ids=FLOOD_IDS)
def test_flood_with_head_and_long_records_twin(members, cmds, batch, faults):
    e = Emu(48, members, library=stats_lib(), route_on_device=True, max_aer_batch=batch)
    bootstrap(e)
    plane_forms()
    e.flood(40, cmds, PERMILLE, SEED, faults)
    forms = plane_forms()
    assert Emu.underfetched(library=stats_lib()) == 0
    assert e.counters()["commits"] > 0
    if cmds < 256:
        assert all(f.head == 0 for f in forms.values()), forms
        return
    assert forms[abi.EV_COMMAND].head > 0, forms[abi.EV_COMMAND]
    if batch >= 256:
        assert forms[abi.EV_AER].head > 0, forms[abi.EV_AER]
    else:                                  # 300 entries as three records per follower and step, all short
        assert forms[abi.EV_AER].head == 0
        assert forms[abi.EV_AER].short >= 2 * (members - 1) * forms[abi.EV_COMMAND].head, forms
    if faults:
        assert forms[abi.EV_AER].long > 0, forms[abi.EV_AER]


# ---- closed-loop traces, not routed: RPC records return as host events (ingest_kernel) ------------------------------
@functools.lru_cache(maxsize=None)
def _trace(members):
    return trace_gen.generate(lambda gg, mm: Oracle(gg, mm, max_aer_batch=512), 10, members, 150, 40 + members,
                              max_cmd=400, p_cmd=0.9)


def _replay_equal(got_backend, members):
    batches = _trace(members)
    want, want_rows, want_cnt = trace_gen.replay(Oracle(10, members, max_aer_batch=512), batches)
    got, got_rows, got_cnt = trace_gen.replay(got_backend, batches)
    for t, (w, x) in enumerate(zip(want, got)):
        assert x[0] == w[0], "RPC records differ at step %d" % t
        assert x[1] == w[1], "host notes differ at step %d" % t
    assert got_rows == want_rows
    assert got_cnt == want_cnt


@pytest.mark.parametrize("wide", WIDTHS)
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("members", [3, 5, 7])
def test_trace_with_long_batches(members, backend, wide, monkeypatch):
    _replay_equal(_make(backend, wide, monkeypatch, 10, members, max_aer_batch=512), members)
    _check_fetch(backend)


@pytest.mark.parametrize("members", [3, 5, 7])
def test_trace_with_long_batches_twin(members):
    plane_forms()
    _replay_equal(Emu(10, members, library=stats_lib(), max_aer_batch=512), members)
    forms = plane_forms()
    assert Emu.underfetched(library=stats_lib()) == 0
    assert forms[abi.EV_COMMAND].head > 0 and forms[abi.EV_AER].head > 0, forms


# ---- one scripted step batch: every form in the same host slot of every tile ----------------------------------------
def _scripted_kinds(row):
    return [
        abi.ev_command(row, 1),                                               # short
        abi.ev_command(row, 256),                                             # head
        abi.ev_command(row, 1000),
        abi.ev_command(row, 65535),
        abi.ev_aer(row, 0, 3, 40, 3, 30, [3] * 300),                          # one term run, 300 entries: head
        abi.ev_aer(row, 0, 3, 40, 2, 30, [2, 2, 3, 3]),                       # two term runs: long
        abi.ev_aer_reply(row, 9, 3, False, 2, 1, 3),                          # from slot 9 (unknown): head
        abi.ev_pre_vote(row, 1, 4, 77, 40, 2),                                # long
    ]


def _scripted(b):
    bootstrap(b)
    out = []
    for shift in (0, 3, 5):
        batch = []
        for r in range(b.n_rows):
            kinds = _scripted_kinds(r)
            batch += [kinds[(r + 2 * k + shift) % len(kinds)] for k in range(abi.RA_LOCAL_CAP)]
        out.append(_keys(b.step(batch)))
    return out


@pytest.mark.parametrize("wide", WIDTHS)
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("members", [3, 5])
def test_scripted_step_mixes_every_form_in_a_tile(members, backend, wide, monkeypatch):
    groups = 400 if backend == "engine" else 40
    b = _make(backend, wide, monkeypatch, groups, members)
    o = Oracle(groups, members)
    assert _scripted(b) == _scripted(o)
    assert b.counters() == o.counters()
    _same_rows(b, o)
    _check_fetch(backend)


def test_scripted_step_mixes_every_form_in_a_tile_twin():
    e = Emu(40, 5, library=stats_lib())
    plane_forms()
    _scripted(e)
    forms = plane_forms()
    assert Emu.underfetched(library=stats_lib()) == 0
    assert forms[abi.EV_COMMAND].short > 0 and forms[abi.EV_COMMAND].head > 0, forms[abi.EV_COMMAND]
    assert forms[abi.EV_AER].head > 0 and forms[abi.EV_AER].long > 0, forms[abi.EV_AER]
    assert forms[abi.EV_AER_REPLY].head > 0 and forms[abi.EV_PRE_VOTE].long > 0, forms


# ---- step_host: 32-byte host events through ingest_kernel<ra_host_event>, closed loop over a routed engine ---------
def _host_loop(b, wide_values, steps=12):
    base, term = ((1 << 32) + 100, (1 << 32) + 5) if wide_values else (100, 5)
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
    roles, out = {}, []
    msgs, notes = b.step_host([abi.ev_simple(b.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(b.n_groups)])
    for t in range(steps):
        per_row = defaultdict(list)
        for n in notes:
            if n.type == abi.NOTE_STATUS:
                roles[n.row] = (n.b >> 24) & 0xff
            elif n.type == abi.NOTE_WAL_APPEND:
                per_row[n.row].append(abi.ev_written(n.row, n.c, n.a, n.b))
        for r, role in roles.items():
            if role == abi.LEADER:
                per_row[r].append(abi.ev_command(r, 256 + 37 * t))
        batch = [e for r in sorted(per_row) for e in per_row[r][:abi.RA_LOCAL_CAP]]
        msgs, notes = b.step_host(batch)
        out.append(_keys((msgs, notes)))
    return out


@pytest.mark.parametrize("wide", WIDTHS)
@pytest.mark.parametrize("backend", BACKENDS)
def test_step_host_long_commands_and_wide_written(backend, wide, monkeypatch):
    """n >= 256 commands; in the 64-bit run, written events whose term and indexes are at or above 2^32 (heads)."""
    groups = 1200 if backend == "engine" else 40
    b = _make(backend, wide, monkeypatch, groups, 5, route_on_device=True, max_aer_batch=512)
    o = Oracle(groups, 5, route_on_device=True, max_aer_batch=512)
    assert _host_loop(b, wide == "1") == _host_loop(o, wide == "1")
    assert b.counters() == o.counters()
    assert o.counters()["commits"] > 0
    _same_rows(b, o)
    _check_fetch(backend)


@pytest.mark.parametrize("wide_values", [False, True])
def test_step_host_long_commands_and_wide_written_twin(wide_values):
    e = Emu(40, 5, library=stats_lib(), route_on_device=True, max_aer_batch=512)
    plane_forms()
    _host_loop(e, wide_values)
    forms = plane_forms()
    assert Emu.underfetched(library=stats_lib()) == 0
    assert forms[abi.EV_COMMAND].head > 0 and forms[abi.EV_AER].head > 0, forms
    if wide_values:
        assert forms[abi.EV_WRITTEN].head > 0 and forms[abi.EV_WRITTEN].short == 0, forms[abi.EV_WRITTEN]


# ---- sharded: bucket transport (deliver_record's CAS) and peer stores against the unsharded oracle ------------------
SHARDED = [(2, 5, 300), (8, 5, 64)]          # shards, members, local groups per slot


def _sharded_oracle(n, m, gl, steps):
    g = n * gl
    o = Oracle(g, m, route_on_device=True, max_aer_batch=512)
    bootstrap(o)
    o.flood(steps, 300, PERMILLE, seed=SEED, threads=8)
    return o, {r.row: r.key()[1:] for r in o.read_rows(range(o.n_rows))}


def _check_sharded(o, want, counters, shard_rows):
    seen = 0
    for shard, rows, global_row in shard_rows:
        for r in rows:
            assert r.key()[1:] == want[global_row(r.row)], (shard, r.row)
            seen += 1
    assert seen == o.n_rows
    co = o.counters()
    for k in ("events", "commits", "applied", "msgs_out", "msgs_dropped", "elections_won", "fatal_rows"):
        assert counters[k] == co[k], k
    assert co["commits"] > 0 and co["msgs_dropped"] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("wide", WIDTHS)
@pytest.mark.parametrize("transport", ["buckets", "peer"])
@pytest.mark.parametrize("n,m,gl", SHARDED)
def test_sharded_flood_with_head_records(n, m, gl, transport, wide, monkeypatch):
    from ra_b200.sharded import LocalPeerTransport, LocalTransport, Shard, ShardedFlood
    monkeypatch.setenv("RA_STEP_WIDE", wide)
    steps = 40
    shards = [Shard(gl, m, n, k, buckets=(transport == "buckets"), max_aer_batch=512) for k in range(n)]
    fl = ShardedFlood(LocalTransport(shards) if transport == "buckets" else LocalPeerTransport(shards))
    fl.bootstrap()
    fl.run(steps, 300, PERMILLE, seed=SEED)
    fl.sync()
    o, want = _sharded_oracle(n, m, gl, steps)
    g = n * gl
    _check_sharded(o, want, fl.counters(),
                   [(s.shard, s.eng.read_rows(range(s.eng.n_rows)), functools.partial(s.global_row, total_groups=g)) for s in shards])


@pytest.mark.parametrize("n,m,gl", [(2, 5, 24), (3, 5, 16)])
def test_sharded_buckets_with_head_records_emu(n, m, gl):
    """The bucket transport on the CPU: every record crossing shards goes through deliver_record."""
    steps = 30
    es = EmuShards(n, gl, m, max_aer_batch=512)
    es.bootstrap()
    es.run(steps, 300, PERMILLE, seed=SEED)
    o, want = _sharded_oracle(n, m, gl, steps)
    _check_sharded(o, want, es.counters(),
                   [(k, s.read_rows(range(s.n_rows)), functools.partial(es.global_row, k)) for k, s in enumerate(es.shards)])
    _check_fetch("emu")


# ---- a stall after a head record: row_end_of_step runs in the general kernel and publishes bit 4 from wk_hi ---------
def _stall_crossing(b):
    """Leaders take a 300-entry command in the hot kernel (head AppendEntries to every follower), then stall on a reply
    from an unknown slot; the step after, the followers read those heads in the hot kernel."""
    bootstrap(b)
    out = []
    for _ in range(4):                                       # elections complete; the leaders' noop entries replicate
        out.append(_keys(b.step([])))
    leaders = [r.row for r in b.read_rows(range(b.n_rows)) if r.role == abi.LEADER]
    assert leaders
    out.append(_keys(b.step([e for r in leaders for e in
                             (abi.ev_command(r, 300), abi.ev_aer_reply(r, 9, 1, False, 2, 1, 1))])))
    for _ in range(3):
        out.append(_keys(b.step([])))
    return out


@pytest.mark.parametrize("wide", WIDTHS)
@pytest.mark.parametrize("backend", BACKENDS)
def test_head_record_sent_before_a_stall(backend, wide, monkeypatch):
    groups = 1500 if backend == "engine" else 64
    b = _make(backend, wide, monkeypatch, groups, 5, route_on_device=True, max_aer_batch=512)
    o = Oracle(groups, 5, route_on_device=True, max_aer_batch=512)
    assert _stall_crossing(b) == _stall_crossing(o)
    assert b.counters() == o.counters()
    _same_rows(b, o)
    assert b.stall_histogram().get((abi.LEADER, abi.EV_AER_REPLY), 0) >= groups
    _check_fetch(backend)


def test_head_record_sent_before_a_stall_twin():
    e = Emu(64, 5, library=stats_lib(), route_on_device=True, max_aer_batch=512)
    Emu.stall_stats(library=stats_lib())
    plane_forms()
    _stall_crossing(e)
    forms = plane_forms()
    assert Emu.underfetched(library=stats_lib()) == 0
    assert forms[abi.EV_AER].head >= 4 * 64, forms[abi.EV_AER]
    assert Emu.stall_stats(library=stats_lib())["stalls_wk_hi"] >= 64
