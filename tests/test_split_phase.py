"""ra_engine_submit / ra_engine_collect, output capacity and ra_engine_fetch_output (include/ra_engine.h).

The split-phase pair must give exactly what ra_engine_step gives; a call whose outputs do not fit the
caller's buffers must lose nothing; a rejected batch must leave every row untouched, also when another batch
was already submitted behind it.  GPU tests (the emulator covers fetch_output on the CPU tier)."""
import pytest

from ra_suite import *  # noqa: F401,F403


def _cluster(be, groups=64, members=3, **kw):
    b = make_backend(be, groups, members, **kw)
    b.reset_empty()
    return b


@pytest.mark.parametrize("be", ["emu", pytest.param("engine", marks=pytest.mark.gpu)])
def test_output_capacity_loses_nothing(be):
    ref = _cluster(be)
    tiny = _cluster(be)
    want = closed_loop(ref, 12, lambda evs: ref.step(evs))

    def tiny_step(evs):
        try:
            return tiny.step(evs, msgs_cap=1, notes_cap=1)
        except abi.RaError as err:
            assert err.status == RA_E_CAPACITY
        st, nm, nn, _, _ = tiny.fetch_output(1, 1)              # still too small: sizes reported, nothing lost
        assert st == RA_E_CAPACITY and (nm > 1 or nn > 1)
        with pytest.raises(abi.RaError):                        # no other step is accepted before the fetch
            tiny.step([], msgs_cap=4096, notes_cap=4096)
        st, nm2, nn2, msgs, notes = tiny.fetch_output(nm, nn)
        assert st == RA_OK and (nm2, nn2) == (nm, nn)
        return msgs, notes
    got = closed_loop(tiny, 12, tiny_step)
    assert got == want
    assert [r.key() for r in tiny.read_rows(range(tiny.n_rows))] == [r.key() for r in ref.read_rows(range(ref.n_rows))]


@pytest.mark.gpu
def test_submit_collect_equals_step():
    ref = _cluster("engine")
    sp = _cluster("engine")
    want = closed_loop(ref, 15, lambda evs: ref.step(evs))

    def split_step(evs):
        st, tk = sp.submit(evs, 4096, 4096)
        assert st == RA_OK
        st, nm, nn, msgs, notes = sp.collect(tk)
        assert st == RA_OK
        return msgs, notes
    assert closed_loop(sp, 15, split_step) == want


@pytest.mark.gpu
def test_two_batches_in_flight_and_busy():
    a = _cluster("engine", 32, 3)
    b = _cluster("engine", 32, 3)
    e1 = [ev_simple(a.row_of(g, 0), EV_ELECTION_TIMEOUT) for g in range(0, 16)]
    e2 = [ev_simple(a.row_of(g, 0), EV_ELECTION_TIMEOUT) for g in range(16, 32)]
    m1, n1 = b.step(e1)
    m2, n2 = b.step(e2)
    st, t1 = a.submit(e1, 4096, 4096)
    assert st == RA_OK
    st, t2 = a.submit(e2, 4096, 4096)
    assert st == RA_OK
    st, _ = a.submit([], 16, 16)
    assert st == abi.RA_E_BUSY                                  # two slots
    st, _, _, am1, an1 = a.collect(t1)
    assert st == RA_OK
    st, _, _, am2, an2 = a.collect(t2)
    assert st == RA_OK
    assert [m.key() for m in am1] == [m.key() for m in m1] and [n.key() for n in an1] == [n.key() for n in n1]
    assert [m.key() for m in am2] == [m.key() for m in m2] and [n.key() for n in an2] == [n.key() for n in n2]
    assert [r.key() for r in a.read_rows(range(a.n_rows))] == [r.key() for r in b.read_rows(range(b.n_rows))]


@pytest.mark.gpu
def test_rejected_batch_takes_the_one_behind_it_along():
    a = _cluster("engine", 16, 3)
    ref = _cluster("engine", 16, 3)
    good = [ev_simple(a.row_of(g, 0), EV_ELECTION_TIMEOUT) for g in range(16)]
    r0 = a.row_of(0, 0)
    bad = [ev_command(r0), ev_command(a.row_of(1, 0)), ev_command(r0)]          # ungrouped
    before = [r.key() for r in a.read_rows(range(a.n_rows))]
    st, t1 = a.submit(bad, 256, 256)
    assert st == RA_OK
    st, t2 = a.submit(good, 4096, 4096)
    assert st == RA_OK
    st, *_ = a.collect(t1)
    assert st == abi.RA_E_UNGROUPED
    st, *_ = a.collect(t2)
    assert st == abi.RA_E_UNGROUPED                             # submitted behind a rejected batch
    assert [r.key() for r in a.read_rows(range(a.n_rows))] == before
    assert a.counters()["events"] == 0
    # and the engine carries on
    m, n = a.step(good)
    m2, n2 = ref.step(good)
    assert [x.key() for x in m] == [x.key() for x in m2] and [x.key() for x in n] == [x.key() for x in n2]


@pytest.mark.gpu
def test_submit_host_segs_equals_one_batch():
    """a batch of host events handed over in pieces (one per producer thread) = the same batch in one array"""
    a = _cluster("engine", 64, 3, route_on_device=True)
    b = _cluster("engine", 64, 3, route_on_device=True)
    evs = [ev_simple(a.row_of(g, 0), EV_ELECTION_TIMEOUT) for g in range(64)]
    want = a.step_host(evs)
    st, ticket = b.submit_host_segs([evs[0:10], [], evs[10:40], evs[40:64]], 1024, 4096)
    assert st == RA_OK
    st, nm, nn, gm, gn = b.collect(ticket)
    assert st == RA_OK
    assert [x.key() for x in gm] == [x.key() for x in want[0]] and [x.key() for x in gn] == [x.key() for x in want[1]]
    assert [r.key() for r in a.read_rows(range(a.n_rows))] == [r.key() for r in b.read_rows(range(b.n_rows))]
