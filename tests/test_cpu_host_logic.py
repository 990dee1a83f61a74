"""`-m "not gpu"`: host logic that needs no GPU -- trace generator determinism, the oracle's
transport contract, and the N>1 sharding / reduction path of bench.py over gloo (world_size 2)."""
import os
import subprocess
import sys
import textwrap

import trace_gen
from fuzz_lib import bootstrap, free_port
from oracle_lib import Oracle
from ra_b200 import abi
from ra_suite import clone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_trace_generator_is_deterministic_and_rich():
    a = trace_gen.generate(lambda g, m: Oracle(g, m), 8, 5, 200, seed=3)
    b = trace_gen.generate(lambda g, m: Oracle(g, m), 8, 5, 200, seed=3)
    assert [[e.key() for e in x] for x in a] == [[e.key() for e in x] for x in b]
    o = Oracle(8, 5)
    out, rows, cnt = trace_gen.replay(o, a)
    assert cnt["commits"] > 100 and cnt["elections_won"] >= 8
    kinds = {n[1] for _, ns in out for n in ns}
    assert {abi.NOTE_WAL_APPEND, abi.NOTE_COMMIT, abi.NOTE_APPLY, abi.NOTE_STATUS, abi.NOTE_TRUNCATE} <= kinds
    # every batch honours the engine contract: rows grouped, <= RA_LOCAL_CAP per row
    for batch in a:
        seen, last, run = set(), None, 0
        for e in batch:
            if e.row != last:
                assert e.row not in seen
                seen.add(e.row)
                last, run = e.row, 0
            run += 1
            assert run <= abi.RA_LOCAL_CAP


def test_oracle_flood_thread_count_does_not_change_results():
    res = []
    for threads in (1, 3, 8):
        o = Oracle(300, 5, route_on_device=True)
        bootstrap(o)
        o.flood(60, 1, 20, seed=4, threads=threads)
        res.append((o.counters(), [r.key() for r in o.read_rows(range(o.n_rows))]))
    assert res[0] == res[1] == res[2]
    assert res[0][0]["commits"] > 0


def test_flood_commits_every_step_in_steady_state():
    o = Oracle(50, 5, route_on_device=True)
    bootstrap(o)
    o.flood(40, 1, 0, seed=1)
    c0 = o.counters()["commits"]
    o.flood(100, 1, 0, seed=1)
    assert o.counters()["commits"] - c0 == 50 * 100          # one commit per group per step
    assert o.counters()["msgs_dropped"] == 0 and o.counters()["fatal_rows"] == 0


def test_unrouted_and_routed_steps_agree_when_the_host_routes():
    """Routing RPC records by hand (non-routed engine) == the mailbox transport."""
    g, m = 6, 3
    a = Oracle(g, m)                       # host routes
    b = Oracle(g, m, route_on_device=True)
    boot = [abi.ev_simple(a.row_of(i, 0), abi.EV_ELECTION_TIMEOUT) for i in range(g)]
    msgs, _ = a.step(boot)
    b.step(boot)
    for _ in range(12):
        # deliver: order by destination row, then sender slot, then send order (contract item 7)
        nxt = sorted((clone(x) for x in msgs), key=lambda e: (e.row, e.from_slot, e.seq))
        msgs, _ = a.step(nxt)
        b.step([])
    assert [r.key() for r in a.read_rows(range(a.n_rows))] == [r.key() for r in b.read_rows(range(b.n_rows))]
    assert any(r.role == abi.LEADER for r in a.read_rows(range(a.n_rows)))


def test_group_sharding_over_gloo_world_size_2(tmp_path):
    """bench.py's N>1 path: groups sharded by rank, SUM of commits, MAX of time -- over gloo."""
    script = tmp_path / "w.py"
    script.write_text(textwrap.dedent("""
        import os, sys, json
        sys.path.insert(0, %r); sys.path.insert(0, os.path.join(%r, "tests"))
        import torch, torch.distributed as dist
        import bench
        from oracle_lib import Oracle
        from ra_b200 import abi
        dist.init_process_group("gloo")
        rank, world = dist.get_rank(), dist.get_world_size()
        G = 200
        o = Oracle(G, 5, route_on_device=True)
        o.reset_empty()
        o.step([abi.ev_simple(o.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(G)])
        o.flood(50, 1, 10, seed=100 + rank)
        c = o.counters()
        ms = 10.0 * (rank + 1)
        ms_max, commits, events = bench.reduce_max_sum(world, None, ms, c["commits"], c["events"])
        if rank == 0:
            print(json.dumps({"ms": ms_max, "commits": commits, "events": events, "mine": c["commits"]}))
        dist.destroy_process_group()
    """ % (ROOT, ROOT)))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", str(free_port()), str(script)],
                         capture_output=True, text=True, env=env, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    import json
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1]
    r = json.loads(line)
    assert r["ms"] == 20.0
    # the other rank's shard, recomputed here
    o = Oracle(200, 5, route_on_device=True)
    bootstrap(o)
    o.flood(50, 1, 10, seed=101)
    assert r["commits"] == r["mine"] + o.counters()["commits"]


def test_hashed_group_is_a_bijection():
    """hash placement (SURVEY 8e) = a host-side relabelling of group ids (ra_b200/sharded.py)"""
    from ra_b200.sharded import hashed_group, shard_of, unhashed_group
    for total in (1, 7, 64, 1000, 100_000):
        seen = {hashed_group(g, total) for g in range(min(total, 5000))}
        assert len(seen) == min(total, 5000)
        for g in {0, 1 % total, total // 2, total - 1}:
            assert unhashed_group(hashed_group(g, total), total) == g
    # neighbours spread over the shards
    shards = [shard_of(hashed_group(g, 100_000), 0, 8) for g in range(64)]
    assert len(set(shards)) == 8
