"""Generates the committed golden fixtures of tests/golden/ (run from the repo root:
`python tests/golden/make_golden.py`).

A fixture is a recorded closed-loop trace (tests/trace_gen.py: network with loss / delay /
duplication, lagging fsync, clients, election timers, a few adversarial RPCs) produced and answered
by the CPU oracle -- the restatement of ra_server.erl that the reference's own ra_server_SUITE
vectors pin (tests/test_golden_ra_server_suite.py).  Stored per trace:

  <name>.events.z   zlib of every step's input batch (64-byte ra_event records, u32 count per step)
  <name>.json       sha256 of every step's outputs (RPC records ++ host notes, ABI bytes), sha256 of
                    the final ra_row_state of every row, the final counters

tests/test_golden_fixtures.py replays the inputs against the oracle and the host build of the
device logic (CPU) and against the CUDA engine (`-m gpu`) and compares digests, so the expected
outputs do not depend on running the oracle at test time.
"""
import ctypes as C
import hashlib
import json
import os
import struct
import sys
import zlib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import trace_gen                      # noqa: E402
from oracle_lib import Oracle          # noqa: E402
from ra_b200 import abi                # noqa: E402
from ra_suite import clone             # noqa: E402

TRACES = {
    # name: (groups, members, steps, seed, simulator knobs, engine config)
    "t3_clean":   (8, 3, 150, 11, {}, {}),
    "t5_mixed":   (16, 5, 200, 7, {}, {}),
    "t7_lossy":   (12, 7, 120, 3, dict(p_drop=0.05, p_withhold_written=0.1), {}),
    "t5_window":  (8, 5, 150, 23, dict(max_cmd=9, p_cmd=0.9), dict(max_pipeline_count=8, max_aer_batch=3)),
}


def digest_outputs(msgs, notes) -> str:
    h = hashlib.sha256()
    for m in msgs:
        h.update(bytes(m))
    h.update(b"|")
    for n in notes:
        h.update(bytes(n))
    return h.hexdigest()


def rows_digest(backend) -> str:
    h = hashlib.sha256()
    for r in backend.read_rows(range(backend.n_rows)):
        h.update(repr(r.key()).encode())
    return h.hexdigest()


def replay_digests(backend, batches):
    out = []
    for batch in batches:
        msgs, notes = backend.step([clone(e) for e in batch])
        out.append(digest_outputs(msgs, notes))
    return out, rows_digest(backend), backend.counters()


def pack_batches(batches) -> bytes:
    raw = bytearray()
    for b in batches:
        raw += struct.pack("<I", len(b))
        for e in b:
            raw += bytes(e)
    return zlib.compress(bytes(raw), 9)


def unpack_batches(blob: bytes):
    raw = zlib.decompress(blob)
    sz = C.sizeof(abi.RaEvent)
    out, off = [], 0
    while off < len(raw):
        (n,) = struct.unpack_from("<I", raw, off)
        off += 4
        batch = []
        for _ in range(n):
            batch.append(abi.RaEvent.from_buffer_copy(raw[off:off + sz]))
            off += sz
        out.append(batch)
    return out


FLOODS = [
    # groups, members, steps, commands per leader and step, election permille, seed  (device-routed flood)
    (64, 3, 60, 1, 0, 42),
    (1000, 5, 120, 2, 10, 42),
    (500, 7, 100, 1, 20, 42),
    (200, 5, 150, 64, 30, 42),
    (10000, 5, 60, 1, 10, 42),       # BASELINE.json configs[1] size
    (100000, 5, 40, 1, 10, 9),       # configs[2] size
]


def rows_bytes_digest(b, chunk=65536) -> str:
    h = hashlib.sha256()
    for lo in range(0, b.n_rows, chunk):
        h.update(b"".join(bytes(r) for r in b.read_rows(range(lo, min(b.n_rows, lo + chunk)))))
    return h.hexdigest()


def flood_digest(b, g, m, steps, cmds, permille, seed, **kw):
    b.reset_empty()
    b.step([abi.ev_simple(b.row_of(i, 0), abi.EV_ELECTION_TIMEOUT) for i in range(g)])
    for part in (steps // 3, steps - steps // 3):          # two calls: the step counter carries over
        b.flood(part, cmds, permille, seed=seed, **kw)
    return rows_bytes_digest(b), b.counters()


def main():
    floods = []
    for (g, m, steps, cmds, permille, seed) in FLOODS:
        o = Oracle(g, m, route_on_device=True)
        rows, counters = flood_digest(o, g, m, steps, cmds, permille, seed, threads=8)
        floods.append(dict(groups=g, members=m, steps=steps, cmds=cmds, permille=permille, seed=seed,
                           rows_sha256=rows, counters=counters))
        print("flood", g, m, steps, cmds, permille, counters["commits"])
        o.close()
    with open(os.path.join(HERE, "floods.json"), "w") as f:
        json.dump(floods, f, indent=0)
    for name, (g, m, steps, seed, knobs, cfg) in TRACES.items():
        batches = trace_gen.generate(lambda gg, mm: Oracle(gg, mm, **cfg), g, m, steps, seed, **knobs)
        per_step, rows, counters = replay_digests(Oracle(g, m, **cfg), batches)
        blob = pack_batches(batches)
        with open(os.path.join(HERE, name + ".events.z"), "wb") as f:
            f.write(blob)
        with open(os.path.join(HERE, name + ".json"), "w") as f:
            json.dump(dict(groups=g, members=m, steps=steps, seed=seed, knobs=knobs, cfg=cfg,
                           events=sum(len(b) for b in batches), step_sha256=per_step, rows_sha256=rows,
                           counters=counters), f, indent=0)
        print(name, "events", sum(len(b) for b in batches), "compressed", len(blob), "bytes")


if __name__ == "__main__":
    main()
