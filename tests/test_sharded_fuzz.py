"""Differential fuzz of the sharded engine: a group's members on N shards, stepped against the UNSHARDED oracle of the
same groups, every step.

The states, event batches and floods are those of tests/test_kernel_fuzz.py (random member states, reloads, fatal
rows, stalls, query state, small note budgets, fault floods); here they run through the code that places a group's
members on different shards: the TR_BUCKET and TR_PEER specialisations of the hot kernel, the sharded branches of
emit_msg and row_end_of_step, deliver_record / deliver_kernel, the peer count-byte stores, and the fault model keyed
by global ids (flood_ids), which must make a sharded run equal the unsharded one.

`Sharded` presents N shards in the oracle's global numbering: row slot * G + g lives on shard (g + slot) mod N at
local row slot * (G / N) + g div N (ra_b200/sharded.py).  Every step compares RPC records and notes in order, every
row as raw ra_row_state bytes, counters and query state; a flood is compared after each of its steps.

Transports: the bucket transport (records for other shards go through per-destination buckets, an exchange and
deliver_record) and peer stores (the step stores into the other shards' mailbox planes and count bytes).  CPU tier:
the host emulation (tests/emu) with both.  GPU tier: ra_b200.sharded.Shard with LocalTransport and with
LocalPeerTransport, all shards on one device and stepped from the host, RA_STEP_WIDE = 0 and 1.

The buckets are sized so that they cannot overflow (local rows x (M - 1) x RA_MBOX_DEPTH records per destination):
which record an overflowing bucket loses depends on the order of the kernel's atomics, so it has no exact oracle
(tests/test_sharded_gpu.py checks that an overflow is counted).
"""
import ctypes as C

import pytest

from emu_lib import Emu, EmuShards
from fuzz_lib import MODES, NOTE_CAPS, budget_coverage, fuzz_rounds, kw, widths
from oracle_lib import Oracle
from ra_b200 import abi
from ra_b200.sharded import global_group, local_group, shard_of
from ra_suite import clone

TRANSPORTS = ["buckets", "peer"]
SHARD_MODES = ["routed", "flood"]                # sharding routes on the device


def _bucket_cap(groups_local, m):
    """Records one destination shard can receive in a step: every local row sends at most RA_MBOX_DEPTH records
    to each of its M - 1 peers."""
    return groups_local * m * (m - 1) * abi.RA_MBOX_DEPTH


class Sharded:
    """N shards (backends in their local numbering) presented in the oracle's global numbering."""

    def __init__(self, shards, exchange, n_groups, n_members, label, keep=None):
        self.shards, self.exchange, self.label, self._keep = shards, exchange, label, keep
        self.n, self.n_groups, self.n_members = len(shards), n_groups, n_members
        self.n_rows = n_groups * n_members
        self.gl = n_groups // self.n
        assert self.gl * self.n == n_groups and all(s.n_groups == self.gl for s in shards)
        self.where = []                                        # global row -> (shard, local row)
        self.glob = [[0] * (self.gl * n_members) for _ in shards]   # [shard][local row] -> global row
        for r in range(self.n_rows):
            slot, g = divmod(r, n_groups)
            k, lr = shard_of(g, slot, self.n), slot * self.gl + local_group(g, self.n)
            assert global_group(local_group(g, self.n), slot, k, self.n) == g
            self.where.append((k, lr))
            self.glob[k][lr] = r

    def _split(self, items):
        """Copies of the items by shard, `row` rewritten to the local row, in their order."""
        per = [[] for _ in self.shards]
        for x in items:
            k, lr = self.where[x.row]
            y = clone(x)
            y.row = lr
            per[k].append(y)
        return per

    def _msg_sender(self, k, x):
        """Global row of the member that sent record x out of shard k (`row` is its local destination row)."""
        to, q = divmod(x.row, self.gl)
        src = x.from_slot if x.from_slot < self.n_members else to
        g = global_group(q, src, k, self.n)
        return src * self.n_groups + g, to * self.n_groups + g

    def load_rows(self, rows):
        for s, part in zip(self.shards, self._split(rows)):
            if part:
                s.load_rows(part)

    def load_query_state(self, qs):
        for s, part in zip(self.shards, self._split(qs)):
            if part:
                s.load_query_state(part)

    def step(self, events):
        outs = [s.step(part) for s, part in zip(self.shards, self._split(events))]
        self.exchange()
        msgs, notes = [], []
        for k, (ms, ns) in enumerate(outs):
            for x in ms:
                sender, x.row = self._msg_sender(k, x)
                msgs.append((sender, x))
            for x in ns:
                x.row = self.glob[k][x.row]
                notes.append((x.row, x))
        # (stable: within a row, the shard's order is the oracle's)
        return ([x for _, x in sorted(msgs, key=lambda t: t[0])], [x for _, x in sorted(notes, key=lambda t: t[0])])

    def flood(self, n_steps, cmds, permille, seed, faults=None):
        for _ in range(n_steps):
            for s in self.shards:
                abi.Backend.flood(s, 1, cmds, permille, seed, faults)     # (an engine's flood without its sync)
            self.exchange()

    def rows_bytes(self):
        sz = C.sizeof(abi.RaRowState)
        out = bytearray(self.n_rows * sz)
        for k, s in enumerate(self.shards):
            for lr, st in enumerate(s.read_rows(range(s.n_rows))):
                g = self.glob[k][lr]
                st.row = g
                out[g * sz:(g + 1) * sz] = bytes(st)
        return bytes(out)

    def read_query_state(self, row_ids):
        q = [None] * self.n_rows
        for k, s in enumerate(self.shards):
            for lr, x in enumerate(s.read_query_state(range(s.n_rows))):
                x.row = self.glob[k][lr]
                q[x.row] = x
        return [q[r] for r in row_ids]

    def counters(self):
        per = [s.counters() for s in self.shards]
        steps = {c["steps"] for c in per}
        assert len(steps) == 1, "%s: the shards disagree on the step count: %r" % (self.label, steps)
        tot = {k: sum(c[k] for c in per) for k in per[0]}
        tot["steps"] = steps.pop()
        return tot

    def stall_histogram(self):
        tot = {}
        for s in self.shards:
            for k, v in s.stall_histogram().items():
                tot[k] = tot.get(k, 0) + v
        return tot


def _fuzz_sharded(bs, mode, m, G, rounds, seed, note_cap=0):
    """bs: Sharded backends over G groups, each stepped with the unsharded oracle and compared with it after every step
    and after each step of a flood -> (oracle, coverage)."""
    o = Oracle(G, m, **kw(mode, note_cap))
    cov = fuzz_rounds(o, [(b.label, b) for b in bs], mode, rounds, seed, note_cap=note_cap, flood_chunk=1)
    assert o.counters()["fatal_rows"] > 0
    if mode == "flood" and rounds > 1:
        assert cov["fault_drops"] > 0, "the faulted floods dropped no record"
    return o, cov


# ---- CPU tier: shards of the host emulation ---------------------------------------------------------------------
def _emu_sharded(transport, n, G, m, monkeypatch, **cfg):
    cfg.pop("route_on_device")
    gl = G // n
    out = []
    for w in widths(monkeypatch):
        es = EmuShards(n, gl, m, cap=_bucket_cap(gl, m), peer=(transport == "peer"), **cfg)
        out.append(Sharded(es.shards, es.exchange, G, m, "N=%d emu %s RA_STEP_WIDE=%s" % (n, transport, w), keep=es))
    return out


def _emu_coverage(transport, m):
    assert Emu.underfetched() == 0, "the hot path decoded a record from bytes its tile's fetch did not cover"
    assert Emu.stall_stats()["stalls"] > 0
    ns = Emu.narrow_stats()
    if transport == "peer" and m == 5:                        # the 32-bit pass runs the peer stores at M = 5
        assert ns["rows_narrow"] > 0 and ns["rows_wide"] > 0 and ns["records_refused"] > 0, ns


# (shards, members); (3, 2): fewer members than shards
EMU_SHAPES = [(2, 5), (3, 5), (2, 3), (3, 7), (8, 5), (4, 4), (5, 8), (8, 3), (3, 2), (2, 6)]


@pytest.mark.parametrize("transport", TRANSPORTS)
@pytest.mark.parametrize("mode", SHARD_MODES)
@pytest.mark.parametrize("n,m", EMU_SHAPES)
def test_sharded_fuzz_emu(n, m, mode, transport, monkeypatch):
    G = 40 if n == 5 else 48
    Emu.narrow_stats(); Emu.stall_stats(); Emu.underfetched()
    bs = _emu_sharded(transport, n, G, m, monkeypatch, **kw(mode))
    _fuzz_sharded(bs, mode, m, G, 6, 9000 + 100 * n + 10 * m + SHARD_MODES.index(mode))
    _emu_coverage(transport, m)


# small note budgets: events refused and submitted again, rows stopped by a burst of notes
BUDGET_CASES = [(3, 7, "routed"), (2, 5, "flood")]


@pytest.mark.parametrize("transport", TRANSPORTS)
@pytest.mark.parametrize("n,m,mode", BUDGET_CASES)
def test_sharded_fuzz_note_cap_emu(n, m, mode, transport, monkeypatch):
    G = 48
    cap = NOTE_CAPS[m][MODES.index(mode)]
    Emu.narrow_stats(); Emu.stall_stats(); Emu.underfetched()
    bs = _emu_sharded(transport, n, G, m, monkeypatch, **kw(mode, cap))
    o, cov = _fuzz_sharded(bs, mode, m, G, 6, 9500 + 100 * n + 10 * m, cap)
    budget_coverage(o, m, mode, cov)
    assert Emu.underfetched() == 0


# ---- GPU tier: ra_b200.sharded.Shard, bucket and peer transports, the 32-bit and the 64-bit hot kernel --------------
def _engine_sharded(transports, n, G, m, monkeypatch, **cfg):
    """Never a device-side barrier here: all shards share one stream, a barrier kernel would wait for shards that
    cannot run.  The host steps the shards in turn instead."""
    from ra_b200.sharded import LocalPeerTransport, LocalTransport, Shard
    cfg.pop("route_on_device")
    gl = G // n
    out = []
    for transport in transports:
        for w in widths(monkeypatch):
            shards = [Shard(gl, m, n, k, cap=_bucket_cap(gl, m), buckets=(transport == "buckets"), **cfg)
                      for k in range(n)]
            t = LocalTransport(shards) if transport == "buckets" else LocalPeerTransport(shards)
            out.append(Sharded([s.eng for s in shards], t.exchange, G, m,
                               "N=%d engine %s RA_STEP_WIDE=%s" % (n, transport, w), keep=(shards, t)))
    return out


GPU_SHAPES = [(2, 5), (8, 5), (5, 5), (3, 7), (4, 3), (8, 8), (3, 2), (2, 6)]   # (5, 5): every member on its own shard


@pytest.mark.gpu
@pytest.mark.parametrize("mode", SHARD_MODES)
@pytest.mark.parametrize("n,m", GPU_SHAPES)
def test_sharded_fuzz_engine(n, m, mode, monkeypatch):
    G = 1200
    bs = _engine_sharded(TRANSPORTS, n, G, m, monkeypatch, **kw(mode))
    _fuzz_sharded(bs, mode, m, G, 3, 9700 + 100 * n + 10 * m + SHARD_MODES.index(mode))
    for b in bs:
        assert b.stall_histogram(), "%s: no row took the general kernel" % b.label


GPU_BUDGET_CASES = [("buckets", 3, 7, "routed"), ("peer", 2, 5, "flood")]


@pytest.mark.gpu
@pytest.mark.parametrize("transport,n,m,mode", GPU_BUDGET_CASES)
def test_sharded_fuzz_note_cap_engine(transport, n, m, mode, monkeypatch):
    G = 1200
    cap = NOTE_CAPS[m][MODES.index(mode)]
    bs = _engine_sharded([transport], n, G, m, monkeypatch, **kw(mode, cap))
    o, cov = _fuzz_sharded(bs, mode, m, G, 2, 9900 + 100 * n + 10 * m, cap)
    budget_coverage(o, m, mode, cov)
