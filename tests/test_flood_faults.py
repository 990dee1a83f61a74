"""Floods with fault injection (include/ra_engine.h: ra_flood_faults) = BASELINE.json configs[4]: 7-member groups,
lagging fsync (withheld WRITTEN), lost AppendEntries (missing -> await_condition -> failure reply -> next_index
back-off) and partitioned members (leader changes whose old leader rejoins with an unreplicated tail: the
term-conflict / truncate path).  Every row and counter must equal the CPU oracle's; on the CPU tier the host
build of the device logic is checked, on a GPU the CUDA engine, up to the stated size 10,000 x 7."""
import pytest

from oracle_lib import Oracle
from ra_b200 import abi
from ra_suite import make_backend

FAULTS = (5, 20, 10, 32)          # 0.5 % AERs lost, 2 % fsync lag, 1 % of groups partitioned per 32-step window


def _run(be, g, m, steps, cmds, permille, faults, seed=0xA05):
    b = make_backend(be, g, m, route_on_device=True)
    b.reset_empty()
    b.step([abi.ev_simple(b.row_of(i, 0), abi.EV_ELECTION_TIMEOUT) for i in range(g)])
    kw = dict(threads=8) if be == "oracle" else {}
    for part in (steps // 3, steps - steps // 3):
        b.flood(part, cmds, permille, seed=seed, faults=faults, **kw)
    return b


CASES = [
    ("emu", 200, 7, 300, 1, 0, FAULTS),
    ("emu", 300, 5, 200, 2, 10, (20, 50, 30, 16)),
    ("emu", 150, 3, 250, 1, 5, (0, 0, 50, 24)),
    pytest.param("engine", 500, 7, 300, 1, 0, FAULTS, marks=pytest.mark.gpu),
    pytest.param("engine", 2000, 5, 200, 64, 10, (20, 50, 30, 16), marks=pytest.mark.gpu),
    pytest.param("engine", 10_000, 7, 400, 1, 0, FAULTS, marks=pytest.mark.gpu),           # configs[4] at its stated size
    ("emu", 200, 2, 250, 1, 5, (20, 50, 30, 16)),            # M = 2 and 6: the runtime-M fault kernel
    ("emu", 150, 6, 250, 1, 5, (20, 50, 30, 16)),
    pytest.param("engine", 2000, 2, 250, 1, 5, (20, 50, 30, 16), marks=pytest.mark.gpu),
    pytest.param("engine", 1500, 6, 250, 1, 5, (20, 50, 30, 16), marks=pytest.mark.gpu),
]


@pytest.mark.parametrize("be,g,m,steps,cmds,permille,faults", CASES)
def test_fault_flood_equals_oracle(be, g, m, steps, cmds, permille, faults):
    o = _run("oracle", g, m, steps, cmds, permille, faults)
    e = _run(be, g, m, steps, cmds, permille, faults)
    co, ce = o.counters(), e.counters()
    assert ce == co
    # the injected faults really exercise the paths config 5 is about
    assert co["msgs_dropped"] > 0 and co["commits"] > g * steps // 4 and co["fatal_rows"] == 0
    if faults[0]:
        assert co["aer_replies_failed"] > 0                    # missing -> failure reply -> back-off
    # leaders changed (from M = 3: a partitioned group of 2 has no quorum on either side, so its leader stays)
    if faults[2] and steps * g >= 30_000 and m >= 3:
        assert co["elections_won"] > g
    assert e.rows_bytes() == o.rows_bytes()
