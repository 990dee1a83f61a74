"""The hot kernel's 32-bit pass (ra_b200/csrc/raft_logic.cuh "narrow pass", raft_step_kernel.cuh): rows whose every
index / term is below 2^30 are evaluated on 32-bit arithmetic, everything else -- a row whose sticky `wide` byte is
set, a record with a larger field -- by the 64-bit kernels.  Which pass evaluates an event must never show in the
results: every case here is compared with the oracle (64-bit C) bit for bit, around and across the 2^30 boundary.

CPU tier: the device logic through tests/emu (where a value leaving or entering the 32-bit pass out of range
aborts the process: ra_emu_narrow_violation).  GPU tier: the kernels themselves, through the C ABI.
"""
import ctypes as C

import pytest

from emu_lib import Emu
from oracle_lib import Oracle
from ra_b200 import abi

LIM = 1 << 30


@pytest.fixture(autouse=True)
def _auto_mode(monkeypatch):
    """These tests assert which pass ran: start from the default (RA_STEP_WIDE unset), whatever the ambient environment."""
    monkeypatch.delenv("RA_STEP_WIDE", raising=False)


def _keys(out):
    msgs, notes = out
    return [m.key() for m in msgs], [n.key() for n in notes]


def _restarted_cluster(b, base, term):
    """Every member restarts from a snapshot at (base, term): empty log, everything written / applied up to it."""
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
    b.step([abi.ev_simple(b.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(b.n_groups)])


def _flood_pair(o, e, base, term, steps, cmds, permille):
    for b in (o, e):
        _restarted_cluster(b, base, term)
    for part in (steps // 2, steps - steps // 2):
        o.flood(part, cmds, permille, seed=77, threads=2)
        e.flood(part, cmds, permille, seed=77)
    assert e.counters() == o.counters()
    assert o.counters()["commits"] > 0
    ro, re_ = o.rows_bytes(), e.rows_bytes()
    sz = C.sizeof(abi.RaRowState)
    first = next((i // sz for i in range(0, len(ro), sz) if ro[i:i + sz] != re_[i:i + sz]), -1)
    assert re_ == ro, "first differing row: %d" % first
    return o.read_rows(range(o.n_rows))


CROSSINGS = [
    # base index, term, steps, commands per step, election permille
    (1000, 3, 60, 1, 20),                      # far below: the 32-bit pass carries everything
    (LIM - 40, 7, 120, 1, 20),                 # indexes cross 2^30 in the middle of the run
    (5000, LIM - 2, 150, 1, 60),               # terms cross 2^30, election by election
    (LIM - 300, LIM - 1, 100, 16, 30),         # both, 16-entry commands
    ((1 << 31) - 50, 9, 100, 1, 20),           # between 2^30 and 2^31 and across 2^31: wide from the first step
    ((1 << 32) - 30, (1 << 32) - 3, 100, 1, 40),   # across 2^32: what 32-bit arithmetic would wrap
    ((1 << 40) + 5, 1 << 33, 60, 1, 20),       # far above
]


@pytest.mark.parametrize("force_narrow", [False, True])
@pytest.mark.parametrize("base,term,steps,cmds,permille", CROSSINGS)
def test_flood_across_the_narrow_limit_emu(base, term, steps, cmds, permille, force_narrow, monkeypatch):
    """force_narrow: RA_STEP_WIDE=0, the 32-bit hot kernel whatever was loaded (every wide row goes through the general
    path); otherwise the engine picks the 64-bit hot kernel for a bulk load most of whose rows are wide."""
    if force_narrow:
        monkeypatch.setenv("RA_STEP_WIDE", "0")
    else:
        monkeypatch.delenv("RA_STEP_WIDE", raising=False)
    Emu.narrow_stats()
    rows = _flood_pair(Oracle(120, 5, route_on_device=True), Emu(120, 5, route_on_device=True), base, term, steps, cmds, permille)
    st = Emu.narrow_stats()
    top = max(max(r.last_index, r.current_term) for r in rows)
    if base < LIM - 1000 and term < LIM - 1000:
        assert st["rows_narrow"] > 0 and st["rows_wide"] == 0 and top < LIM
    elif base >= LIM or term >= LIM:
        assert st["rows_narrow"] == 0 and (st["rows_wide"] > 0) == force_narrow     # auto: the 64-bit hot kernel
    else:
        assert st["rows_narrow"] > 0 and st["rows_wide"] > 0 and top >= LIM      # the run did cross


def test_narrow_and_wide_pass_agree_emu(monkeypatch):
    """RA_STEP_WIDE=1 (64-bit hot kernel only) and the default produce the same rows, records and notes."""
    outs = []
    for wide in ("0", "1"):                                 # always the 32-bit hot kernel / never
        monkeypatch.setenv("RA_STEP_WIDE", wide)
        Emu.narrow_stats()
        e = Emu(40, 5)
        e.reset_empty()
        log = []
        log.append(_keys(e.step([abi.ev_simple(e.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(40)])))
        # a leaderless cluster answering pre-votes by hand is enough to run followers' fast paths
        log.append(_keys(e.step([abi.ev_pre_vote(e.row_of(g, 1), 0, 0, 1, 0, 0) for g in range(40)])))
        log.append(_keys(e.step([abi.ev_aer(e.row_of(g, 2), 0, 1, 0, 0, 0, [1, 1]) for g in range(40)])))
        outs.append((log, e.rows_bytes(), Emu.narrow_stats()))
    assert outs[0][0] == outs[1][0] and outs[0][1] == outs[1][1]
    assert outs[0][2]["rows_narrow"] > 0 and outs[1][2]["rows_narrow"] == 0


def _wide_record_script(b, groups):
    big = (1 << 35) + 7
    b.reset_empty()
    t = []
    t.append(_keys(b.step([ev for g in range(groups) for ev in
                           (abi.ev_aer(b.row_of(g, 1), 0, 1, 0, 0, 0, [1]), abi.ev_written(b.row_of(g, 1), 1, 1, 1))])))
    t.append(_keys(b.step([ev for g in range(groups) for ev in
                           (abi.ev_aer(b.row_of(g, 1), 0, big if g % 2 else 1, 1, 1, 0, [big if g % 2 else 1]),
                            abi.ev_written(b.row_of(g, 1), big if g % 2 else 1, 2, 2),
                            abi.ev_aer(b.row_of(g, 1), 0, big if g % 2 else 1, 2, big if g % 2 else 1, 1, []))])))
    t.append(_keys(b.step([abi.ev_aer(b.row_of(g, 1), 0, big if g % 2 else 1, 2, big if g % 2 else 1, 2, []) for g in range(groups)])))
    return t, b.rows_bytes()


def test_record_with_a_wide_field_goes_to_the_general_path_emu():
    """A narrow row handed ONE record with a field >= 2^30: the 32-bit pass refuses the record, the general path
    evaluates it (and what follows in the step), the row is wide from then on -- same outputs as the oracle."""
    o, e = Oracle(6, 5), Emu(6, 5)
    Emu.narrow_stats()
    outs = [_wide_record_script(b, 6) for b in (o, e)]
    assert outs[0] == outs[1]
    st = Emu.narrow_stats()
    # step 1 stalls on the term change (general path, rows stay narrow); step 2: three rows are handed the wide
    # record first; step 3 finds those three rows wide
    assert st["records_refused"] == 3 and st["rows_wide"] == 3 and st["rows_narrow"] == 6 + 6 + 3


# ---- the kernels themselves ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("base,term,steps,cmds,permille", CROSSINGS)
def test_flood_across_the_narrow_limit_gpu(base, term, steps, cmds, permille):
    from ra_b200.engine import Engine
    _flood_pair(Oracle(4000, 5, route_on_device=True), Engine(4000, 5, route_on_device=True), base, term, steps, cmds, permille)


@pytest.mark.gpu
@pytest.mark.parametrize("members", [3, 7])
def test_flood_across_the_narrow_limit_gpu_m3_m7(members):
    from ra_b200.engine import Engine
    _flood_pair(Oracle(3000, members, route_on_device=True), Engine(3000, members, route_on_device=True), LIM - 60, LIM - 2, 140, 1, 40)


@pytest.mark.gpu
def test_record_with_a_wide_field_goes_to_the_general_path_gpu():
    from ra_b200.engine import Engine
    outs = [_wide_record_script(b, 600) for b in (Oracle(600, 5), Engine(600, 5))]
    assert outs[0] == outs[1]


# ---- closed-loop traces (loss, delay, duplicates, lagging fsync, elections, adversarial records) across the limit ----
def _restarted(b, base, term):
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
    return b


TRACE_CROSSINGS = [
    # groups, members, steps, seed, base index, term, knobs
    (10, 5, 260, 5, LIM - 60, 3, dict(p_cmd=0.9, max_cmd=3)),                         # indexes cross in mid-run
    (10, 5, 260, 9, 40, LIM - 3, dict(p_timeout=0.06)),                               # terms cross, many elections
    (8, 5, 220, 13, LIM - 400, LIM - 2, dict(p_cmd=0.9, max_cmd=60, p_timeout=0.04, p_adversarial=0.05)),
    (8, 5, 200, 21, (1 << 32) - 200, (1 << 32) - 2, dict(p_cmd=0.9, max_cmd=40, p_timeout=0.04)),   # 32-bit wrap territory
    (6, 3, 200, 31, LIM - 50, LIM - 2, dict(p_drop=0.05, p_withhold_written=0.1)),    # runtime-M specialisation (64-bit pass)
]


@pytest.mark.parametrize("g,m,steps,seed,base,term,knobs", TRACE_CROSSINGS)
def test_trace_parity_across_the_narrow_limit_emu(g, m, steps, seed, base, term, knobs):
    import trace_gen
    batches = trace_gen.generate(lambda gg, mm: _restarted(Oracle(gg, mm), base, term), g, m, steps, seed, **knobs)
    Emu.narrow_stats()
    want, want_rows, want_cnt = trace_gen.replay(_restarted(Oracle(g, m), base, term), batches)
    got, got_rows, got_cnt = trace_gen.replay(_restarted(Emu(g, m), base, term), batches)
    for t, (w, x) in enumerate(zip(want, got)):
        assert x[0] == w[0], "RPC records differ at step %d" % t
        assert x[1] == w[1], "host notes differ at step %d" % t
    assert got_rows == want_rows
    assert got_cnt == want_cnt
    st = Emu.narrow_stats()
    if m == 5 and base < LIM and term < LIM:
        assert st["rows_narrow"] > 0 and st["rows_wide"] > 0      # the run started narrow and crossed


LIMITS = [dict(max_pipeline_count=0xFFFFFFFF), dict(max_pipeline_count=0x80000000, max_aer_batch=0xFFFFFFFF),
          dict(max_aer_batch=0x90000000), dict(max_pipeline_count=3, max_aer_batch=2)]


@pytest.mark.parametrize("kw", LIMITS)
def test_pipeline_limits_beyond_31_bits_emu(kw):
    """max_pipeline_count / max_aer_batch are 32-bit unsigned configuration values; the 32-bit pass compares them with
    signed differences of indexes (found by review: 'unlimited' = 0xFFFFFFFF read as -1 stopped every pipeline pass)."""
    import trace_gen
    o, e = Oracle(50, 5, route_on_device=True, **kw), Emu(50, 5, route_on_device=True, **kw)
    for b in (o, e):
        b.reset_empty()
        b.step([abi.ev_simple(b.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(50)])
    o.flood(60, 3, 20, seed=5, threads=1)
    e.flood(60, 3, 20, seed=5)
    assert e.counters() == o.counters() and e.rows_bytes() == o.rows_bytes() and o.counters()["commits"] > 0
    # and a lossy closed-loop trace (failure replies move next_index below match_index + 1: in_flight < 0)
    batches = trace_gen.generate(lambda gg, mm: Oracle(gg, mm, **kw), 8, 5, 200, 3, p_drop=0.08, p_cmd=0.9, max_cmd=9)
    assert trace_gen.replay(Emu(8, 5, **kw), batches) == trace_gen.replay(Oracle(8, 5, **kw), batches)
