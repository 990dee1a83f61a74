"""Settle a flood, then run a few steps and report where they went.

Without --trace: the counters of those steps and the events that left the fast kernel (stall histogram).
With --trace DIR: the steps run under torch.profiler (CUDA activities); prints the device time per step of
raft_step_kernel, raft_general_kernel, the other kernels and the gaps between kernels, and writes the Chrome
trace under DIR."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ra_b200 import abi
from ra_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--groups", type=int, default=100_000)
ap.add_argument("--members", type=int, default=5)
ap.add_argument("--settle", type=int, default=40)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--permille", type=int, default=10)
ap.add_argument("--cmds", type=int, default=1)
ap.add_argument("--trace", metavar="DIR", default=None,
                help="profile the steps with torch.profiler, print the per-step split, write the trace under DIR")
a = ap.parse_args()


def kernel_split(trace_path: str, steps: int) -> dict:
    """Per-step device time (ms) of the step's kernels and of the gaps between them, from a Chrome trace."""
    with open(trace_path) as f:
        evs = json.load(f)["traceEvents"]
    ks = sorted((e for e in evs if e.get("ph") == "X" and e.get("cat") == "kernel"), key=lambda e: e["ts"])
    if not ks:
        raise RuntimeError("the trace holds no kernel: torch.profiler saw no CUDA activity")
    out = {"raft_step_kernel": 0.0, "raft_general_kernel": 0.0, "other_kernels": 0.0}
    busy = 0.0
    for e in ks:
        name = e["name"]
        key = ("raft_step_kernel" if "raft_step_kernel" in name else
               "raft_general_kernel" if "raft_general_kernel" in name else "other_kernels")
        out[key] += e["dur"]
        busy += e["dur"]
    span = ks[-1]["ts"] + ks[-1]["dur"] - ks[0]["ts"]
    out["gaps"] = span - busy
    out["span"] = span
    res = {k: v / 1e3 / steps for k, v in out.items()}          # us -> ms per step
    res["kernels_per_step"] = len(ks) / steps
    return res


e = Engine(a.groups, a.members, route_on_device=True)
e.reset_empty()
e.step([abi.ev_simple(e.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(a.groups)])
e.flood(a.settle, a.cmds, a.permille, seed=0xA00)
c0 = e.counters()
if a.trace:
    import torch
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(a.trace, exist_ok=True)
    e.sync()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        e.flood(a.steps, a.cmds, a.permille, seed=0xA00)
        e.sync()
    path = os.path.join(a.trace, "flood_%dx%d.json" % (a.groups, a.members))
    prof.export_chrome_trace(path)
    c1 = e.counters()
    split = kernel_split(path, a.steps)
    split["events_per_step"] = (c1["events"] - c0["events"]) / a.steps
    split["msgs_out_per_step"] = (c1["msgs_out"] - c0["msgs_out"]) / a.steps
    split["trace"] = path
    print(json.dumps(split))
    sys.exit(0)
e.flood(a.steps, a.cmds, a.permille, seed=0xA00)
print(e.counters(), e.last_kernel_ms())
names = ["none", "AER", "AER_REPLY", "REQ_VOTE", "REQ_VOTE_RES", "PRE_VOTE", "PRE_VOTE_RES", "WRITTEN", "COMMAND",
         "ELECTION_TMO", "AWAIT_TMO", "PIPELINE", "TICK"]
roles = ["follower", "candidate", "pre_vote", "leader", "await_condition"]
h = e.stall_histogram()
tot = sum(h.values())
print("events that left the fast kernel: %d of %d (%.2f%%)" % (tot, e.counters()["events"], 100.0 * tot / max(1, e.counters()["events"])))
for (ro, ty), v in sorted(h.items(), key=lambda kv: -kv[1]):
    print("  %-16s %-14s %10d" % (roles[ro] if ro < 5 else ro, names[ty] if ty < 13 else ty, v))
