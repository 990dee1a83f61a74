"""Where the hot step kernel's time goes, warp by warp and by role.

Builds the engine with the compile-time probe (-DRA_WARP_TIMELINE, see engine.cu: every warp of raft_step_kernel
records its SM, tile, leader lanes, %globaltimer / clock64 at four points and lane 0's cycles per part of the event
loop), settles the 100k x 5 flood, runs single flood steps and prints, per step and over all of them:
  - median and p99 warp duration of leader warps and of follower warps;
  - when the last leader warp starts and ends, against the kernel's end;
  - cycles per leader event by type, and the frame (TMA issue, mbarrier wait, decode) against the handler;
  - the kernel split into the phase while leader warps are resident and the followers-only phase.
The raw per-warp records go to OUT/timeline_<step>.npy and the summary to OUT/timeline.json.

    python tools/warp_timeline.py [--so PATH] [--out DIR] [--groups N] [--members M] [--steps K]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TL_WORDS = 64
EV_NAMES = {1: "AER", 2: "AER_REPLY", 3: "REQ_VOTE", 4: "REQ_VOTE_RES", 5: "PRE_VOTE", 6: "PRE_VOTE_RES",
            7: "WRITTEN", 8: "COMMAND", 9: "ELECTION_TMO", 10: "AWAIT_TMO", 11: "PIPELINE", 12: "TICK", 15: "none"}

ap = argparse.ArgumentParser()
ap.add_argument("--so", default=os.path.join(ROOT, "ra_b200", "csrc", "libra_engine_tl.so"),
                help="probe build of the engine (built with tools/build_variant.sh when missing)")
ap.add_argument("--out", default=None, help="output directory (default: a new temporary directory)")
ap.add_argument("--groups", type=int, default=100_000)
ap.add_argument("--members", type=int, default=5)
ap.add_argument("--settle", type=int, default=40)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--permille", type=int, default=10)
ap.add_argument("--cmds", type=int, default=1)
a = ap.parse_args()

if not os.path.exists(a.so):
    name = os.path.basename(a.so)[len("libra_engine_"):-len(".so")]
    subprocess.check_call([os.path.join(ROOT, "tools", "build_variant.sh"), name, "-DRA_WARP_TIMELINE"])
os.environ["RA_ENGINE_SO"] = a.so
sys.path.insert(0, ROOT)
from ra_b200 import abi                      # noqa: E402
from ra_b200.engine import Engine, lib       # noqa: E402

f = lib().ra_engine_warp_timeline
f.restype = C.c_int
f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]

e = Engine(a.groups, a.members, route_on_device=True)
e.reset_empty()
e.step([abi.ev_simple(e.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(a.groups)])
e.flood(a.settle, a.cmds, a.permille, seed=0xA00)
n_warps = (e.n_rows + 31) // 32
a.out = a.out or tempfile.mkdtemp(prefix="warp_timeline_")
os.makedirs(a.out, exist_ok=True)


def pct(x, q):
    return float(np.percentile(x, q)) if len(x) else float("nan")


def summarise(t):
    ok = (t[:, 0] >> 63) == 1
    t = t[ok]
    lead = ((t[:, 0] >> 32) & 0x7FFFFFFF) > 0
    g = t[:, 2:6].astype(np.int64)
    k0 = g[:, 0].min()
    g = g - k0                                           # ns from the first warp's start
    k_end = int(g[:, 3].max())
    dur = g[:, 3] - g[:, 0]
    cyc = t[:, 6:10].astype(np.int64)
    s = {"warps": int(ok.sum()), "leader_warps": int(lead.sum()), "kernel_span_us": k_end / 1e3}
    for name, sel in (("leader", lead), ("follower", ~lead)):
        d = dur[sel]
        s[name] = {"median_us": pct(d, 50) / 1e3, "p99_us": pct(d, 99) / 1e3, "max_us": float(d.max()) / 1e3 if len(d) else 0,
                   "median_cycles": pct(cyc[sel, 3] - cyc[sel, 0], 50),
                   "median_inputs_us": pct(g[sel, 1] - g[sel, 0], 50) / 1e3,
                   "median_loop_us": pct(g[sel, 2] - g[sel, 1], 50) / 1e3,
                   "median_tail_us": pct(g[sel, 3] - g[sel, 2], 50) / 1e3}
    if lead.any():
        ls = g[lead, 0]
        le = g[lead, 3]
        s["last_leader_start_us"] = float(ls.max()) / 1e3
        s["last_leader_end_us"] = float(le.max()) / 1e3
        s["leaders_resident_us"] = float(le.max()) / 1e3
        s["followers_only_us"] = (k_end - float(le.max())) / 1e3
        L = t[lead]
        planes = L[:, 13].sum()
        frame = {"issue": L[:, 10].sum() / planes, "wait": L[:, 11].sum() / planes, "decode": L[:, 12].sum() / planes}
        ev = {}
        hsum = 0
        for ty in range(16):
            n = L[:, 19 + 2 * ty].sum()
            if n:
                c = L[:, 18 + 2 * ty].sum()
                hsum += c
                ev[EV_NAMES.get(ty, str(ty))] = {"per_warp": n / len(L), "cycles_per_event": c / n}
        frame["handler"] = hsum / planes
        s["leader_planes_per_warp"] = planes / len(L)
        s["leader_cycles_per_plane"] = frame
        s["leader_events"] = ev
        s["leader_tail_cycles"] = {"peers_writeback": float(np.median(L[:, 14])), "row_end_of_step": float(np.median(L[:, 15])),
                                   "member_writeback": float(np.median(L[:, 16])), "stall_and_counters": float(np.median(L[:, 17]))}
    F = t[~lead]
    if len(F):
        planes = max(1, F[:, 13].sum())
        s["follower_cycles_per_plane"] = {"issue": F[:, 10].sum() / planes, "wait": F[:, 11].sum() / planes,
                                          "decode": F[:, 12].sum() / planes,
                                          "handler": sum(F[:, 18 + 2 * ty].sum() for ty in range(16)) / planes}
        s["follower_planes_per_warp"] = planes / len(F)
        s["follower_tail_cycles"] = {"row_end_of_step": float(np.median(F[:, 15])), "member_writeback": float(np.median(F[:, 16]))}
    return s


steps = []
for k in range(a.steps):
    f(e._h, None, 0)
    e.flood(1, a.cmds, a.permille, seed=0xA00)
    buf = np.zeros(n_warps * TL_WORDS, dtype=np.uint64)
    rc = f(e._h, buf.ctypes.data, buf.size)
    if rc != 0:
        raise SystemExit("ra_engine_warp_timeline failed: %d" % rc)
    t = buf.reshape(n_warps, TL_WORDS)
    np.save(os.path.join(a.out, "timeline_%d.npy" % k), t)
    steps.append(summarise(t))
keys = ("kernel_span_us", "last_leader_start_us", "last_leader_end_us", "followers_only_us")
out = {"groups": a.groups, "members": a.members, "steps": steps,
       "median": {k: float(np.median([s[k] for s in steps if k in s])) for k in keys}}
with open(os.path.join(a.out, "timeline.json"), "w") as fh:
    json.dump(out, fh, indent=1)
last = steps[-1]
print(json.dumps(out["median"]))
print(json.dumps(last, indent=1))
print("raw records and summary under", a.out)
