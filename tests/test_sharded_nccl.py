"""`-m gpu`, needs >= 2 GPUs (run with `gpurun --gpus 2`): one shard per rank, the cross-shard RPC
buckets travel by NCCL all_to_all_single; every rank checks its members against the unsharded
oracle run.  Skipped on a single-GPU box (the same kernels/ABI are covered there by
tests/test_sharded_gpu.py with the in-process transport)."""
import os
import subprocess
import sys
import textwrap

import pytest

from fuzz_lib import free_port

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("transport", ["a2a", "peer", "peer-devbar"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_nccl_sharded_flood_equals_oracle(world, transport, tmp_path):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    # at world 8 > M = 5 two slot offsets share one destination shard: the bucket capacity of
    # sharded.Shard must cover that, or records are dropped and the rows differ -- see DESIGN.md §8
    script = tmp_path / "w.py"
    script.write_text(textwrap.dedent("""
        import os, sys
        sys.path.insert(0, %r); sys.path.insert(0, os.path.join(%r, "tests"))
        import torch, torch.distributed as dist
        from ra_b200 import abi
        from ra_b200.sharded import Shard, NcclTransport, NvlinkPeerTransport, ShardedFlood
        from oracle_lib import Oracle
        rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        gl, m, steps = 256, 5, 70
        peer = %r.startswith("peer")
        os.environ["RA_PEER_BARRIER"] = "device" if %r.endswith("devbar") else "nccl"
        sh = Shard(gl, m, world, rank, device=local, buckets=not peer)
        fl = ShardedFlood(NvlinkPeerTransport(sh) if peer else NcclTransport(sh))
        fl.bootstrap()
        fl.run(steps, 1, 10, seed=31)
        fl.sync()
        g = gl * world
        o = Oracle(g, m, route_on_device=True)
        o.reset_empty()
        o.step([abi.ev_simple(o.row_of(i, 0), abi.EV_ELECTION_TIMEOUT) for i in range(g)])
        o.flood(steps, 1, 10, seed=31, threads=4)
        want = {r.row: r.key()[1:] for r in o.read_rows(range(o.n_rows))}
        bad = 0
        for r in sh.eng.read_rows(range(sh.eng.n_rows)):
            if r.key()[1:] != want[sh.global_row(r.row, g)]:
                bad += 1
        c = sh.eng.counters()
        t = torch.tensor([bad, c["commits"], c["msgs_dropped"]], dtype=torch.int64, device="cuda")
        dist.all_reduce(t)
        if rank == 0:
            print("RESULT", int(t[0]), int(t[1]), int(t[2]), o.counters()["commits"])
        dist.destroy_process_group()
    """ % (ROOT, ROOT, transport, transport)))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                          "--master-addr", "127.0.0.1", "--master-port", str(free_port()), str(script)],
                         capture_output=True, text=True, env=env, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("RESULT")][-1].split()
    bad, commits, dropped, want_commits = map(int, line[1:])
    assert bad == 0 and dropped == 0 and commits == want_commits > 0
