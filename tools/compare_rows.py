"""Diff the rows written by erlang/b1/ra_b1_oracle.erl (true reference, BEAM) against the C oracle's replay of
the same recorded trace: python tools/compare_rows.py rows.bin t5_mixed"""
import ctypes as C, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from ra_b200 import abi
from oracle_lib import Oracle
import make_golden
from ra_suite import clone
rows_file, name = sys.argv[1], sys.argv[2]
g, m, steps, seed, knobs, cfg = make_golden.TRACES[name]
batches = make_golden.unpack_batches(open(os.path.join(ROOT, "tests", "golden", name + ".events.z"), "rb").read())
o = Oracle(g, m, **cfg)
for b in batches:
    o.step([clone(e) for e in b])
want = o.read_rows(range(o.n_rows))
raw = open(rows_file, "rb").read()
sz = C.sizeof(abi.RaRowState)
assert len(raw) == sz * len(want), (len(raw), sz * len(want))
bad = 0
for i, w in enumerate(want):
    got = abi.RaRowState.from_buffer_copy(raw[i * sz:(i + 1) * sz])
    if got.key() != w.key():
        bad += 1
        if bad <= 10:
            print("row", i, "differs:\n  beam  ", got.key(), "\n  oracle", w.key())
print("%d of %d rows differ" % (bad, len(want)))
sys.exit(1 if bad else 0)
