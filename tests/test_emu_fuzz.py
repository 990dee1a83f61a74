"""CPU tier: differential fuzz of single (state, event) pairs -- random but well-formed member states
of every role against random events of every type, oracle (per-index term array, clause by clause)
against the engine's device logic compiled for the host (run-length log view, fast paths, record
codec).  Closed-loop traces (tests/trace_gen.py) visit the states a cluster really reaches; this
visits the corners around them: term +-1, indices just outside the log, stale tokens, snapshots at
the log edge, non-voters, peers in odd states, with and without next-event chasing."""
import random

import pytest

from emu_lib import Emu
from fuzz_lib import (ROLES, compare, fuzz_around_the_narrow_limit, observe, random_event, random_query,
                      random_state)
from oracle_lib import Oracle
from ra_suite import clone


@pytest.mark.parametrize("m", [3, 5, 7])
@pytest.mark.parametrize("pure", [True, False])
def test_fuzz_state_event_pairs(m, pure):
    rng = random.Random(1000 * m + (1 if pure else 0))
    G = 64
    o, e = Oracle(G, m, pure=pure), Emu(G, m, pure=pure)
    for rnd in range(40):
        states, events = [], []
        for g in range(G):
            slot = rng.randrange(m)
            role = rng.choice(ROLES)
            st = random_state(rng, slot * G + g, G, m, role)
            states.append(st)
            # up to two events for the row, adjacent in the batch (contract item 1)
            for _ in range(rng.choice([1, 1, 2])):
                events.append(random_event(rng, st, m))
        qs = [random_query(rng, st.row, m) for st in states]
        outs = []
        for b in (o, e):
            b.load_rows(states)
            b.load_query_state(qs)
            outs.append(observe(b, m, b.step([clone(x) for x in events])))
        compare(outs[0], outs[1], "round %d" % rnd, events, o)


# ---- the same corners, moved to where the hot kernel's 32-bit pass ends (tests/test_narrow_pass.py) ----------------
@pytest.mark.parametrize("pure", [True, False])
def test_fuzz_state_event_pairs_around_the_narrow_limit(pure, monkeypatch):
    monkeypatch.delenv("RA_STEP_WIDE", raising=False)        # (the test asserts which pass ran)
    fuzz_around_the_narrow_limit(pure)
