"""The host-driven flood (ra_hostsim, ra_b200/csrc/host_flood.cu) against the oracle, in the shapes the end-to-end leg
of bench.py runs it: K engines holding disjoint groups of uneven sizes, one ra_hostsim over all of them, the host model
split over threads and drivers, both note formats, and note buffers that start too small for a step's notes.

Partition p of G_p groups is checked against an oracle of its own: Oracle(G_p, M, route_on_device=True), bootstrapped
with the single step of election timeouts to slot 0 that ra_hostsim_run(..., bootstrap=1) submits, then flooded with
seed + p for every run() of the hostsim.  After every run() each partition's rows and counters must equal its oracle's.
Several hostsims, each made under its own RA_HOSTSIM_* settings over its own engines, run side by side against the same
oracles; their byte and call counts must agree where the settings cannot change them.
"""
import pytest

from emu_lib import Emu
from fuzz_lib import bootstrap, first_row
from oracle_lib import Oracle

SEED = 0xA00                                  # bench.py --seed
BENCH_CALLS = [40, 10, 20, 20, 20]            # after run(0, bootstrap=True): settle, warm-up, three (short) timed blocks
SETTLE = BENCH_CALLS[0]
KNOBS = ("RA_HOSTSIM_THREADS", "RA_HOSTSIM_DRIVERS", "RA_HOSTSIM_COMPACT", "RA_HOSTSIM_NOTE_SLOTS")


def split(groups, k):
    """bench.py's partitioning of `groups` over k engines"""
    return [groups // k + (1 if i < groups % k else 0) for i in range(k)]


class Flight:
    """One ra_hostsim over engines of its own (one per partition), made under RA_HOSTSIM_THREADS / _DRIVERS / _COMPACT /
    _NOTE_SLOTS = threads, drivers, compact, slots (None: unset, 6 slots per row).  Every run()'s statistics are kept in
    `stats`.  The host emulation has the plain format only: a flight over it has compact = 0."""

    def __init__(self, make, sizes, m, monkeypatch, threads, drivers, compact=0, slots=None):
        from ra_b200.engine import HostFlood
        self.compact, self.slots = compact, slots
        self.label = "threads=%d drivers=%d %s%s" % (threads, drivers, "compact" if compact else "plain",
                                                     " note_slots=%d" % slots if slots else "")
        for k in KNOBS:                          # read when the hostsim is created
            monkeypatch.delenv(k, raising=False)
        monkeypatch.setenv("RA_HOSTSIM_THREADS", str(threads))
        monkeypatch.setenv("RA_HOSTSIM_DRIVERS", str(drivers))
        monkeypatch.setenv("RA_HOSTSIM_COMPACT", str(compact))
        if slots is not None:
            monkeypatch.setenv("RA_HOSTSIM_NOTE_SLOTS", str(slots))
        self.engines = [make(g, m) for g in sizes]
        for e in self.engines:
            e.reset_empty()
        self.hf = HostFlood(self.engines)
        self.stats = []

    def close(self):
        self.hf.close()
        for e in self.engines:
            e.close()


class Lockstep:
    """The oracles of the partitions and the flights, run() by run(): the first run() bootstraps."""

    def __init__(self, make, sizes, m, variants, monkeypatch, cmds=1, permille=10, oracle_threads=2):
        self.sizes, self.m, self.cmds, self.permille, self.oracle_threads = sizes, m, cmds, permille, oracle_threads
        self.oracles = [Oracle(g, m, route_on_device=True) for g in sizes]
        for o in self.oracles:
            bootstrap(o)
        self.flights = [Flight(make, sizes, m, monkeypatch, *v) for v in variants]
        self.calls = []

    @property
    def rows(self):
        return sum(self.sizes) * self.m

    def run(self, n):
        first = not self.calls
        self.calls.append(n)
        what = "run #%d (%s)" % (len(self.calls) - 1, "bootstrap" if first else "%d steps" % n)
        if n:
            for p, o in enumerate(self.oracles):
                o.flood(n, self.cmds, self.permille, seed=SEED + p, threads=self.oracle_threads)
        want = [(o.rows_bytes(), o.counters()) for o in self.oracles]
        K = len(self.sizes)
        for f in self.flights:
            st = f.hf.run(n, self.cmds, self.permille, seed=SEED, bootstrap=first)
            f.stats.append(st)
            for p, (e, (rows, cnt)) in enumerate(zip(f.engines, want)):
                where = "%s: partition %d (%d groups x %d) after %s" % (f.label, p, self.sizes[p], self.m, what)
                got = e.rows_bytes()
                if got != rows:
                    pytest.fail("%s: first differing row %d" % (where, first_row(rows, got)))
                c = e.counters()
                if c != cnt:
                    diff = {k: (cnt[k], c[k]) for k in cnt if cnt[k] != c.get(k)}
                    pytest.fail("%s: counters differ (oracle, engine): %r" % (where, diff))
            if st["engine_calls"] != K * (int(first) + n):
                pytest.fail("%s: %d engine calls in %s, want %d" % (f.label, st["engine_calls"], what, K * (int(first) + n)))

    def run_calls(self, calls=BENCH_CALLS):
        """bench.py's sequence: run(0, bootstrap=True), then the runs of `calls`"""
        self.run(0)
        for n in calls:
            self.run(n)

    def check_accounting(self):
        """For every run(): h2d_bytes and engine_calls do not depend on threads, drivers, note slots or format; the plain
        d2h_bytes not on threads, drivers or note slots; a compact run of more than one step moves at least half and
        less than all of the plain run's d2h_bytes."""
        fl = self.flights
        plain = [f for f in fl if not f.compact]
        assert fl[0].stats[0]["h2d_bytes"] == 32 * sum(self.sizes)          # one election timeout per group
        for i, n in enumerate(self.calls):
            for f in fl[1:]:
                for k in ("h2d_bytes", "engine_calls"):
                    assert f.stats[i][k] == fl[0].stats[i][k], (k, i, n, f.label, fl[0].label)
            for f in plain[1:]:
                assert f.stats[i]["d2h_bytes"] == plain[0].stats[i]["d2h_bytes"], (i, n, f.label, plain[0].label)
            if plain and n > 1:
                d2h = plain[0].stats[i]["d2h_bytes"]
                for f in fl:
                    if f.compact:
                        assert d2h // 2 <= f.stats[i]["d2h_bytes"] < d2h, (i, n, f.label, f.stats[i]["d2h_bytes"], d2h)
        # the flood did what it is for: commands committed in every partition
        assert all(o.counters()["commits"] > 0 for o in self.oracles)

    def settle_until_regrown(self):
        """1-step runs after the bootstrap until every flight that starts with one note slot per row has had a step
        whose notes took more than rows x 32 bytes: they could not fit the buffer the hostsim started with, so it grew
        the buffer and fetched them again, and run() checked the rows straight after that step.  It must happen within
        the settle period.  Returns the steps taken."""
        waiting = [f for f in self.flights if f.slots == 1]
        assert waiting
        for t in range(SETTLE):
            self.run(1)
            waiting = [f for f in waiting if f.stats[-1]["d2h_bytes"] <= 32 * self.rows]
            if not waiting:
                return t + 1
        pytest.fail("no step of the settle period outgrew the first note buffer of %s" % [f.label for f in waiting])

    def close(self):
        for f in self.flights:
            f.close()


# partitions of uneven sizes (each case has one partition of >= 4096 rows, which the model splits over its threads, and
# one under, which it runs on one), M, election permille, and the flights: (threads, drivers, note slots).  Drivers
# beyond K are clamped to K; 3 threads divide none of the row counts.
CASES = [
    pytest.param([1500], 3, 10, [(1, 1, None), (3, 2, None), (16, 1, 1)], id="K1-M3"),
    pytest.param([1400, 333], 5, 200, [(3, 1, None), (16, 2, None), (1, 3, 1)], id="K2-M5"),
    pytest.param([1000, 997, 300], 7, 0, [(16, 1, None), (3, 4, None), (3, 2, 1)], id="K3-M7"),
    pytest.param([900, 20, 611, 1, 257], 5, 10, [(3, 2, None), (1, 6, None), (16, 1, 1)], id="K5-M5"),
]


def _engine(g, m):
    from ra_b200.engine import Engine
    return Engine(g, m, route_on_device=True)


def _emu(g, m):
    return Emu(g, m, route_on_device=True)


# ---- CPU tier: the hostsim over the host emulation of the engine (plain notes only) ---------------------------------
@pytest.mark.parametrize("sizes,m,permille,flights", CASES)
def test_host_flood_partitions_emu(sizes, m, permille, flights, monkeypatch):
    ls = Lockstep(_emu, sizes, m, [(t, d, 0, s) for (t, d, s) in flights], monkeypatch, permille=permille)
    ls.run_calls()
    ls.check_accounting()
    ls.close()


def test_note_buffer_regrows_emu(monkeypatch):
    """One note slot per row: the steady flood's notes do not fit, the hostsim grows the buffer and fetches them again
    (ra_engine_fetch_output), and every step still equals the oracle."""
    ls = Lockstep(_emu, [1100, 240], 5, [(3, 2, 0, 1), (1, 1, 0, 1), (16, 1, 0, None)], monkeypatch)
    ls.run(0)
    ls.settle_until_regrown()
    ls.run(10)
    ls.check_accounting()
    ls.close()


# ---- GPU tier: the same over CUDA engines sharing one device, in both note formats ----------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("sizes,m,permille,flights", CASES)
def test_host_flood_partitions(sizes, m, permille, flights, monkeypatch):
    ls = Lockstep(_engine, sizes, m, [(t, d, c, s) for (t, d, s) in flights for c in (0, 1)], monkeypatch,
                  permille=permille, oracle_threads=8)
    ls.run_calls()
    ls.check_accounting()
    ls.close()


@pytest.mark.gpu
@pytest.mark.parametrize("groups,flights", [
    pytest.param(100_000, [(16, 1, 1, None), (16, 1, 0, None), (16, 2, 0, None)], id="100000x5"),
    pytest.param(100_003, [(16, 2, 1, None), (16, 1, 1, 1), (16, 2, 0, 1)], id="100003x5"),
])
def test_host_flood_bench_shape(groups, flights, monkeypatch):
    """bench.py's e2e leg: the groups over 4 engines on one GPU, 1 command per leader and step, 1 % election timeouts,
    16 model threads, its call sequence with short timed blocks."""
    ls = Lockstep(_engine, split(groups, 4), 5, flights, monkeypatch, oracle_threads=8)
    ls.run_calls()
    ls.check_accounting()
    ls.close()


@pytest.mark.gpu
@pytest.mark.parametrize("m", [3, 7])
def test_note_buffer_regrows(m, monkeypatch):
    """test_note_buffer_regrows_emu on CUDA engines, both formats: a compact step outgrows the rows x 32-byte buffer when
    its notes and extension entries take more than two 16-byte units per row."""
    ls = Lockstep(_engine, [1100, 240], m, [(3, 2, 0, 1), (16, 1, 1, 1), (16, 1, 0, None)], monkeypatch,
                  oracle_threads=8)
    ls.run(0)
    ls.settle_until_regrown()
    ls.run(10)
    ls.check_accounting()
    ls.close()
