"""The dirty-NIF shim (ra_b200/csrc/ra_engine_nif.c) run through a working erl_nif stub (tests/nif_stub/), against the
oracle.  The shim is compiled with gcc together with the stub and linked against the host emulation of the engine
(tests/emu/libra_emu.so) for the CPU tier and against libra_engine.so for the GPU tier.  A thin Python face mirrors
erlang/src/ra_engine_nif.erl; records travel as binaries of the ABI structs, as the Erlang side sends them.

The shim creates its engines with a zeroed ra_engine_cfg (not routed, not pure, default AER batch, pipeline count and
note budget), so the oracle is built with that configuration too.  What is checked:

- the fuzz rounds of tests/fuzz_lib.py (rich generator, host events for the host paths) through step,
  step_host, submit / submit_host + collect one and two calls deep: records and notes in order, every row as raw
  ra_row_state bytes read back through read_rows, the counters map;
- outputs beyond the shim's first guess of their size, through step and through two calls in flight (the re-fetch and
  the re-submission of the call behind);
- rejected batches, badarg, a third call in flight, step while calls are in flight, collect with nothing pending;
- the engine term dropped with calls in flight: the destructor runs and no binary or resource outlives it;
- engines driven from several threads at once;
- the NIF table against the -export list of the Erlang module.
"""
import ctypes as C
import json
import os
import random
import re
import struct
import subprocess
import sys
import threading

import pytest

from fuzz_lib import ROLES, batch, first_row, fuzz_round, host_event, random_state, rich_event, same_keys
from oracle_lib import Oracle
from ra_b200 import abi
from ra_suite import clone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB = os.path.join(ROOT, "tests", "nif_stub")
SHIM = os.path.join(ROOT, "ra_b200", "csrc", "ra_engine_nif.c")
T = C.c_size_t                            # ERL_NIF_TERM (uintptr_t)
K_INT, K_ATOM, K_BIN, K_TUPLE, K_MAP, K_RES, K_BADARG = range(1, 8)
EV, HEV, NOTE, ROW = 64, 32, 32, C.sizeof(abi.RaRowState)
FIRST_GUESS = 64                          # the shim's output buffers for an empty batch: 0 * CAP + 64 records


# ---- build ----------------------------------------------------------------------------------------------------------
def build_shim(backend: str, out_dir: str) -> str:
    """ra_engine_nif.c + erl_nif_stub.c -> a shared library linked against the emulation or the engine"""
    if backend == "emu":
        import emu_lib
        emu_lib.lib()                                            # (re)builds tests/emu/libra_emu.so if stale
        lib_dir, lib = os.path.join(ROOT, "tests", "emu"), "libra_emu.so"
    else:
        lib_dir, lib = os.path.join(ROOT, "ra_b200", "csrc"), "libra_engine.so"
    assert os.path.exists(os.path.join(lib_dir, lib)), "build first: python -c 'import __graft_entry__ as g; g.build()'"
    so = os.path.join(out_dir, "libra_nif_%s.so" % backend)
    cmd = ["gcc", "-std=c11", "-O1", "-g", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared", "-DRA_HAVE_ERL_NIF",
           "-I" + STUB, "-o", so, SHIM, os.path.join(STUB, "erl_nif_stub.c"),
           "-L" + lib_dir, "-l:" + lib, "-Wl,-rpath," + lib_dir, "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return so


@pytest.fixture(scope="module")
def nif_emu(tmp_path_factory):
    return Nif(build_shim("emu", str(tmp_path_factory.mktemp("nif_emu"))))


@pytest.fixture(scope="module")
def nif_gpu(tmp_path_factory):
    return Nif(build_shim("engine", str(tmp_path_factory.mktemp("nif_gpu"))))


# ---- the runtime side: terms in, terms out --------------------------------------------------------------------------
class Badarg(Exception):
    pass


class Ref:
    """an engine term held by a process: a reference to the resource until drop() (what the garbage collector does
    once no process holds the term any more)"""

    def __init__(self, nif, obj):
        self.nif, self.obj = nif, obj

    def drop(self):
        if self.obj:
            self.nif.l.ra_stub_drop(self.obj)
            self.obj = None


class Nif:
    def __init__(self, path: str):
        l = self.l = C.CDLL(path)
        vp = C.c_void_p
        for name, res, args in (
                ("ra_stub_env_new", vp, []), ("ra_stub_env_free", None, [vp]),
                ("ra_stub_make_binary", T, [vp, C.c_char_p, C.c_size_t]), ("ra_stub_make_int", T, [vp, C.c_longlong]),
                ("ra_stub_make_atom", T, [vp, C.c_char_p]), ("ra_stub_make_resource", T, [vp, vp]),
                ("ra_stub_load", C.c_int, []), ("ra_stub_call", T, [vp, C.c_char_p, C.c_uint, C.POINTER(T)]),
                ("ra_stub_nif_count", C.c_int, []), ("ra_stub_nif_name", C.c_char_p, [C.c_int]),
                ("ra_stub_nif_arity", C.c_uint, [C.c_int]), ("ra_stub_nif_flags", C.c_uint, [C.c_int]),
                ("ra_stub_module", C.c_char_p, []),
                ("ra_stub_kind", C.c_int, [vp, T]), ("ra_stub_element", T, [vp, T, C.c_int]),
                ("ra_stub_atom_text", C.c_int, [vp, T, C.c_char_p, C.c_size_t]),
                ("ra_stub_integer", C.c_int, [vp, T, C.POINTER(C.c_longlong), C.POINTER(C.c_ulonglong)]),
                ("ra_stub_binary", C.c_int, [vp, T, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]),
                ("ra_stub_map_size", C.c_longlong, [vp, T]), ("ra_stub_map_key", T, [vp, T, C.c_size_t]),
                ("ra_stub_map_value", T, [vp, T, C.c_size_t]),
                ("ra_stub_keep", vp, [vp, T]), ("ra_stub_drop", None, [vp]),
                ("ra_stub_live_binaries", C.c_long, []), ("ra_stub_live_resources", C.c_long, []),
                ("ra_stub_bad_releases", C.c_long, []), ("ra_stub_dtor_runs", C.c_long, [])):
            f = getattr(l, name)
            f.restype, f.argtypes = res, args
        assert l.ra_stub_load() == 0

    def counts(self):
        l = self.l
        return dict(binaries=l.ra_stub_live_binaries(), resources=l.ra_stub_live_resources(),
                    bad_releases=l.ra_stub_bad_releases(), dtors=l.ra_stub_dtor_runs())

    def table(self):
        l = self.l
        return [(l.ra_stub_nif_name(k).decode(), l.ra_stub_nif_arity(k), l.ra_stub_nif_flags(k))
                for k in range(l.ra_stub_nif_count())]

    def _term(self, env, x):
        l = self.l
        if isinstance(x, Ref):
            return l.ra_stub_make_resource(env, x.obj)
        if isinstance(x, (bytes, bytearray)):
            return l.ra_stub_make_binary(env, bytes(x), len(x))
        if isinstance(x, str):
            return l.ra_stub_make_atom(env, x.encode())
        if isinstance(x, int):
            return l.ra_stub_make_int(env, x)
        raise TypeError(x)

    def _value(self, env, t):
        l = self.l
        k = l.ra_stub_kind(env, t)
        if k == K_INT:
            i, u = C.c_longlong(), C.c_ulonglong()
            return u.value if l.ra_stub_integer(env, t, C.byref(i), C.byref(u)) == 2 else i.value
        if k == K_ATOM:
            buf = C.create_string_buffer(256)
            l.ra_stub_atom_text(env, t, buf, 256)
            return buf.value.decode()
        if k == K_BIN:
            p, n = C.c_void_p(), C.c_size_t()
            assert l.ra_stub_binary(env, t, C.byref(p), C.byref(n))
            return C.string_at(p, n.value) if n.value else b""
        if k == K_TUPLE:
            return tuple(self._value(env, l.ra_stub_element(env, t, i)) for i in range(2))
        if k == K_MAP:
            return {self._value(env, l.ra_stub_map_key(env, t, i)): self._value(env, l.ra_stub_map_value(env, t, i))
                    for i in range(l.ra_stub_map_size(env, t))}
        if k == K_RES:
            return Ref(self, l.ra_stub_keep(env, t))
        if k == K_BADARG:
            raise Badarg()
        raise AssertionError("term kind %d" % k)

    def call(self, name: str, *args):
        """NAME/len(args) in a fresh env (the calling process); the result is read out and the env freed"""
        l = self.l
        env = l.ra_stub_env_new()
        try:
            argv = (T * max(1, len(args)))(*[self._term(env, a) for a in args])
            t = l.ra_stub_call(env, name.encode(), len(args), argv)
            assert t, "no NIF %s/%d" % (name, len(args))
            return self._value(env, t)
        finally:
            l.ra_stub_env_free(env)


# ---- the Erlang face (erlang/src/ra_engine_nif.erl) ----------------------------------------------------------------
def ev_bin(evs):
    return b"".join(bytes(e) for e in evs)


def hev_bin(evs):
    return b"".join(bytes(abi.RaHostEvent.of(e)) for e in evs)


def outputs(res):
    """{MsgsBin, NotesBin} -> (message keys, note keys); anything else is returned as it is"""
    if not (isinstance(res, tuple) and isinstance(res[0], bytes)):
        return res
    msgs, notes = res
    assert len(msgs) % EV == 0 and len(notes) % NOTE == 0
    return ([abi.RaEvent.from_buffer_copy(msgs, i).key() for i in range(0, len(msgs), EV)],
            [abi.RaNote.from_buffer_copy(notes, i).key() for i in range(0, len(notes), NOTE)])


class NifEngine:
    def __init__(self, nif: Nif, groups: int, members: int, device: int = 0):
        self.nif, self.n_rows = nif, groups * members
        st, self.ref = nif.call("new", groups, members, device)
        assert st == "ok"

    def load_rows(self, rows):
        return self.nif.call("load_rows", self.ref, b"".join(bytes(s) for s in rows))

    def read_rows(self, ids):
        return self.nif.call("read_rows", self.ref, struct.pack("<%dI" % len(ids), *ids))

    def rows_bytes(self):
        return self.read_rows(list(range(self.n_rows)))

    def reset_empty(self):
        return self.nif.call("reset_empty", self.ref)

    def step(self, evs):
        return self.nif.call("step", self.ref, ev_bin(evs))

    def step_host(self, evs):
        return self.nif.call("step_host", self.ref, hev_bin(evs))

    def submit(self, evs):
        return self.nif.call("submit", self.ref, ev_bin(evs))

    def submit_host(self, evs):
        return self.nif.call("submit_host", self.ref, hev_bin(evs))

    def collect(self):
        return self.nif.call("collect", self.ref)

    def counters(self):
        return self.nif.call("counters", self.ref)

    def drop(self):
        self.ref.drop()


def oracle(G, m):
    return Oracle(G, m)                       # = the shim's zeroed ra_engine_cfg


def o_step(o, evs):
    msgs, notes = o.step([clone(e) for e in evs], o.n_rows * abi.RA_MSG_CAP, o.n_rows * abi.RA_NOTE_CAP)
    return [x.key() for x in msgs], [x.key() for x in notes]


def same_state(eng, o, what):
    got, want = eng.rows_bytes(), o.rows_bytes()
    assert isinstance(got, bytes), "%s: read_rows returned %r" % (what, got)
    if got != want:
        raise AssertionError("%s: rows differ from row %d" % (what, first_row(want, got)))
    assert eng.counters() == o.counters(), "%s: counters" % what


def same_out(got, want, what):
    got = outputs(got)
    assert isinstance(got, tuple) and isinstance(got[0], list), "%s: %r" % (what, got)
    for k, g, w in zip(("msgs", "notes"), got, want):
        same_keys(w, g, what, k)


# ---- a. the fuzz through the NIF ------------------------------------------------------------------------------------
LANES = [("step", 1), ("step_host", 1), ("submit", 1), ("submit_host", 1), ("submit", 2), ("submit_host", 2)]


def _lane(nif, path, depth, m, G, rounds, seed):
    rng = random.Random(seed)
    host = path.endswith("host")
    draw = host_event if host else rich_event
    o, eng = oracle(G, m), NifEngine(nif, G, m)
    cov = dict(calls=0, beyond_guess=0)
    for rnd in range(rounds):
        # (the shim has no load_query_state: a loaded member starts with a zero query state on both sides)
        loads, _, events = fuzz_round(rng, o, rnd, draw)
        if rnd % 2:
            # every slot-0 member a leader with a deferred pipeline pass, and an empty first batch: the outputs overrun
            # the shim's first guess (its re-fetch, and the re-submission of the call behind)
            byrow = {s.row: s for s in loads}
            for r in range(G):
                byrow[r] = random_state(rng, r, G, m, abi.LEADER, rich=True)
                byrow[r].flags |= 1
            loads, events = [byrow[r] for r in sorted(byrow)], []
        o.load_rows(loads)
        assert eng.load_rows(loads) == "ok"
        fly = []
        for t in range(3):
            evs = events if t == 0 else batch(rng, o, draw, rng.choice([0.0, 0.01, 0.3, 1.0]))
            want = o_step(o, evs)
            what = "M=%d %s depth %d round %d batch %d" % (m, path, depth, rnd, t)
            cov["calls"] += 1
            cov["beyond_guess"] += len(want[0]) > len(evs) * abi.RA_MSG_CAP + FIRST_GUESS or \
                len(want[1]) > len(evs) * abi.RA_NOTE_CAP + FIRST_GUESS
            if path.startswith("step"):
                same_out(getattr(eng, path)(evs), want, what)
                same_state(eng, o, what)
                continue
            assert getattr(eng, path)(evs) == "ok", what
            fly.append((want, what))
            while len(fly) >= depth:
                w, wh = fly.pop(0)
                same_out(eng.collect(), w, wh)
            if not fly:
                same_state(eng, o, what)
        while fly:
            w, wh = fly.pop(0)
            same_out(eng.collect(), w, wh)
        same_state(eng, o, "M=%d %s depth %d round %d" % (m, path, depth, rnd))
    assert eng.collect() == ("error", abi.RA_E_INVAL)
    eng.drop()
    return cov


def _fuzz_nif(nif, m, G, rounds, seed):
    for k, (path, depth) in enumerate(LANES):
        cov = _lane(nif, path, depth, m, G, rounds, seed + 10 * k)
        assert cov["beyond_guess"] > 0, "%s depth %d: no call overran the shim's first guess" % (path, depth)


@pytest.mark.parametrize("m", [3, 5, 7])
def test_fuzz_through_nif_emu(nif_emu, m):
    _fuzz_nif(nif_emu, m, 64, 4, 12000 + 100 * m)


GPU_FUZZ = [(5, "0"), (5, "1"), (3, None), (7, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("m,wide", GPU_FUZZ)
def test_fuzz_through_nif_engine(nif_gpu, m, wide, monkeypatch):
    """M = 5 runs both passes of the host-transport kernel (the shim never routes on the device), M = 3 and 7 the
    runtime-M kernel; the general kernel runs behind all of them"""
    if wide is None:
        monkeypatch.delenv("RA_STEP_WIDE", raising=False)
    else:
        monkeypatch.setenv("RA_STEP_WIDE", wide)                # read when the engine is created
    _fuzz_nif(nif_gpu, m, 1200, 2, 13000 + 100 * m + (wide == "1"))


# ---- b. outputs beyond the shim's first guess -----------------------------------------------------------------------
def _pipelined_leaders(rng, G, m):
    """every slot-0 member a leader with a deferred pipeline pass (flags bit 0, as the fuzz generator sets it), the
    others fuzzed states"""
    rows = []
    for r in range(G * m):
        role = abi.LEADER if r < G else rng.choice([abi.FOLLOWER, abi.CANDIDATE, abi.PRE_VOTE, abi.AWAIT_CONDITION])
        s = random_state(rng, r, G, m, role, rich=True)
        if role == abi.LEADER:
            s.flags |= 1
        rows.append(s)
    return rows


def _capacity(nif, G, m, seed):
    rng = random.Random(seed)
    rows = _pipelined_leaders(rng, G, m)
    tick = [abi.ev_simple(G + 1, abi.EV_TICK)]                   # one event, for a follower
    # through step
    o, eng = oracle(G, m), NifEngine(nif, G, m)
    o.load_rows(rows)
    assert eng.load_rows(rows) == "ok"
    for k, evs in enumerate([[], tick]):
        want = o_step(o, evs)
        assert len(want[0]) > len(evs) * abi.RA_MSG_CAP + FIRST_GUESS, "precondition: %d records" % len(want[0])
        got = eng.step(evs)
        assert got != ("error", abi.RA_E_CAPACITY)
        same_out(got, want, "step %d" % k)
        same_state(eng, o, "step %d" % k)
        o.load_rows(rows)
        assert eng.load_rows(rows) == "ok"
    eng.drop()
    # through submit, submit, collect, collect: the second call is re-submitted by the shim
    for api in ("submit", "submit_host"):
        o, eng = oracle(G, m), NifEngine(nif, G, m)
        o.load_rows(rows)
        assert eng.load_rows(rows) == "ok"
        w1, w2 = o_step(o, []), o_step(o, tick)
        assert len(w1[0]) > FIRST_GUESS, "precondition: %d records" % len(w1[0])
        assert getattr(eng, api)([]) == "ok" and getattr(eng, api)(tick) == "ok"
        same_out(eng.collect(), w1, "%s: first collect" % api)
        same_out(eng.collect(), w2, "%s: second collect (the call re-submitted behind the first)" % api)
        same_state(eng, o, api)
        assert eng.collect() == ("error", abi.RA_E_INVAL)
        eng.drop()


def test_output_capacity_inside_the_shim_emu(nif_emu):
    _capacity(nif_emu, 64, 5, 14000)


@pytest.mark.gpu
def test_output_capacity_inside_the_shim_engine(nif_gpu):
    _capacity(nif_gpu, 1200, 5, 14100)


# ---- c. rejected batches; d. busy and empty; e. the counters map -----------------------------------------------------
def _bad_batches(G, m):
    n = G * m
    return [("ungrouped", abi.RA_E_UNGROUPED, [abi.ev_simple(0, abi.EV_TICK), abi.ev_simple(1, abi.EV_TICK),
                                               abi.ev_simple(0, abi.EV_TICK)]),
            ("above RA_LOCAL_CAP", abi.RA_E_CAPACITY, [abi.ev_command(G, 1) for _ in range(abi.RA_LOCAL_CAP + 1)]),
            ("bad row", abi.RA_E_INVAL, [abi.ev_simple(1, abi.EV_TICK), abi.ev_simple(n, abi.EV_TICK)]),
            ("bad type", abi.RA_E_INVAL, [abi.ev_simple(2, 16)]),
            ("sender slot 17", abi.RA_E_INVAL, [abi.ev_simple(1, abi.EV_TICK), abi.ev_request_vote(2, 17, 99, 0, 0)])]


HOSTLESS = ("bad type", "sender slot 17")    # a 32-byte host record carries neither an RPC type nor a sender


def _rejected(nif, G, m, seed):
    rng = random.Random(seed)
    rows = [random_state(rng, r, G, m, rng.choice(ROLES), rich=True) for r in range(G * m)]
    o, eng = oracle(G, m), NifEngine(nif, G, m)
    o.load_rows(rows)
    assert eng.load_rows(rows) == "ok"
    good = lambda: [host_event(rng, s, m) for s in o.read_rows(range(0, G * m, 3))]
    for what, code, bad in _bad_batches(G, m):
        before = eng.rows_bytes()
        assert eng.step(bad) == ("error", code), what
        if what not in HOSTLESS:
            assert eng.step_host(bad) == ("error", code), what
        assert eng.step_host([abi.ev_aer(0, 1, 1, 0, 0, 0)]) == ("error", abi.RA_E_INVAL)   # an RPC type
        for api in ("submit", "submit_host"):
            if api == "submit_host" and what in HOSTLESS:
                continue
            evs = good()
            assert getattr(eng, api)(bad) == "ok" and getattr(eng, api)(evs) == "ok", what
            assert eng.collect() == ("error", code), "%s %s" % (what, api)
            assert eng.collect() == ("error", code), "%s %s: the call behind it" % (what, api)
        assert eng.rows_bytes() == before, what
        same_state(eng, o, what)
        evs = good()                                             # the engine carries on
        same_out(eng.step(evs), o_step(o, evs), "after %s" % what)
        same_state(eng, o, "after %s" % what)
    # badarg: a binary that is not a whole number of records, a term that is not an engine
    for name, rec in (("step", EV), ("step_host", HEV), ("submit", EV), ("submit_host", HEV), ("load_rows", ROW),
                      ("read_rows", 4)):
        with pytest.raises(Badarg):
            nif.call(name, eng.ref, b"\0" * (rec + 1))
        for not_engine in (7, "engine", b"\0" * 8):
            with pytest.raises(Badarg):
                nif.call(name, not_engine, b"")
    for name in ("collect", "counters", "reset_empty"):
        with pytest.raises(Badarg):
            nif.call(name, 7)
    with pytest.raises(Badarg):
        nif.call("new", -1, m, 0)
    assert nif.call("new", 0, m, 0) == ("error", abi.RA_E_INVAL)
    assert eng.read_rows([G * m]) == ("error", abi.RA_E_INVAL)
    same_state(eng, o, "after badarg")
    # d. busy and empty
    assert eng.collect() == ("error", abi.RA_E_INVAL)
    e1, e2 = good(), good()
    w1 = o_step(o, e1)
    assert eng.submit_host(e1) == "ok"
    assert eng.step(e2) == ("error", abi.RA_E_BUSY)             # refused: the oracle never sees these two
    assert eng.step_host(e2) == ("error", abi.RA_E_BUSY)
    w2 = o_step(o, e2)
    assert eng.submit(e2) == "ok"
    assert eng.submit(good()) == ("error", abi.RA_E_BUSY)
    assert eng.submit_host(good()) == ("error", abi.RA_E_BUSY)
    same_out(eng.collect(), w1, "busy: first call")
    same_out(eng.collect(), w2, "busy: second call")
    assert eng.collect() == ("error", abi.RA_E_INVAL)
    same_state(eng, o, "busy")
    # e. the counters map: the 15 fields of ra_counters, the oracle's values
    cnt = eng.counters()
    assert sorted(cnt) == sorted(n for n, _ in abi.RaCounters._fields_)
    assert cnt == o.counters() and cnt["events"] > 0 and cnt["steps"] > 0
    eng.drop()


def test_rejected_busy_empty_counters_emu(nif_emu):
    _rejected(nif_emu, 48, 5, 15000)


@pytest.mark.gpu
def test_rejected_busy_empty_counters_engine(nif_gpu):
    _rejected(nif_gpu, 1200, 5, 15100)


# ---- f. the engine term dropped with calls in flight ----------------------------------------------------------------
STATES = ["idle", "one_in_flight", "two_in_flight", "capacity"]


def _lifetime(nif, G, m, state, seed):
    rng = random.Random(seed)
    base = nif.counts()
    rows = _pipelined_leaders(rng, G, m)
    eng = NifEngine(nif, G, m)
    assert eng.load_rows(rows) == "ok"
    evs = [host_event(rng, s, m) for s in rows[::2]]
    if state == "capacity":
        o = oracle(G, m)
        o.load_rows(rows)
        assert len(o_step(o, [])[0]) > FIRST_GUESS, "precondition"
        assert eng.submit([]) == "ok"
    for _ in range({"idle": 0, "one_in_flight": 1, "two_in_flight": 2, "capacity": 0}[state]):
        assert eng.submit_host(evs) == "ok"
        evs = [host_event(rng, s, m) for s in rows[1::2]]
    assert nif.counts()["resources"] == base["resources"] + 1
    eng.drop()
    now = nif.counts()
    assert now["dtors"] == base["dtors"] + 1, "%s: the destructor did not run" % state
    assert now["resources"] == base["resources"], state
    assert now["binaries"] == base["binaries"], "%s: %d binaries outlived the engine" % (
        state, now["binaries"] - base["binaries"])
    assert now["bad_releases"] == base["bad_releases"], state
    # the engine created next has nothing pending and steps like the oracle
    eng, o = NifEngine(nif, G, m), oracle(G, m)
    assert eng.collect() == ("error", abi.RA_E_INVAL), state
    for x in (eng, o):
        x.load_rows(rows)
    for t in range(3):
        evs = [host_event(rng, s, m) for s in o.read_rows(range(t, G * m, 2))]
        assert eng.submit_host(evs) == "ok"
        same_out(eng.collect(), o_step(o, evs), "%s: next engine, step %d" % (state, t))
    same_state(eng, o, state)
    assert eng.collect() == ("error", abi.RA_E_INVAL)
    eng.drop()
    assert nif.counts() == dict(base, dtors=base["dtors"] + 2)


@pytest.mark.parametrize("state", STATES)
def test_engine_dropped_with_calls_in_flight_emu(nif_emu, state):
    _lifetime(nif_emu, 48, 5, state, 16000 + STATES.index(state))


@pytest.mark.gpu
def test_engine_dropped_with_calls_in_flight_engine(nif_gpu):
    _lifetime(nif_gpu, 1200, 5, "two_in_flight", 16100)


# ---- g. engines on threads ------------------------------------------------------------------------------------------
def _thread_plan(k, G, m, rounds):
    """thread k's engine: its rows and 2 * rounds host-event batches"""
    rng = random.Random(17000 + k)
    rows = [random_state(rng, r, G, m, rng.choice(ROLES), rich=True) for r in range(G * m)]
    batches = []
    for _ in range(2 * rounds):
        batches.append([host_event(rng, s, m) for s in rows if rng.random() < 0.3])
    return rows, batches


def _drive(nif, G, m, plan):
    """submit, submit, collect, collect per round -> (every collect's outputs, the final rows)"""
    rows, batches = plan
    eng = NifEngine(nif, G, m)
    assert eng.load_rows(rows) == "ok"
    out = []
    for i in range(0, len(batches), 2):
        out.append(eng.submit_host(batches[i]))
        out.append(eng.submit_host(batches[i + 1]))
        out.append(eng.collect())
        out.append(eng.collect())
    res = (out, eng.rows_bytes())
    eng.drop()
    return res


def _threads(nif, G, m, n_threads, rounds):
    """-> a list of what differs between the threaded run and the single-threaded one (empty: nothing)"""
    plans = [_thread_plan(k, G, m, rounds) for k in range(n_threads)]
    want = [_drive(nif, G, m, p) for p in plans]
    got = [None] * n_threads
    errors = []

    def run(k):
        try:
            got[k] = _drive(nif, G, m, plans[k])
        except Exception as exc:                                # noqa: BLE001 - reported below
            errors.append("thread %d: %r" % (k, exc))
    ts = [threading.Thread(target=run, args=(k,)) for k in range(n_threads)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    bad = list(errors)
    for k in range(n_threads):
        if got[k] is None:
            continue
        (wo, wr), (go, gr) = want[k], got[k]
        i = next((i for i, (x, y) in enumerate(zip(wo, go)) if x != y), None)
        if i is not None:
            bad.append("thread %d: call %d differs: %.200r, single-threaded %.200r" % (k, i, go[i], wo[i]))
        if gr != wr:
            bad.append("thread %d: final rows differ" % k)
    c = nif.counts()
    if c["bad_releases"]:
        bad.append("%d binaries released twice" % c["bad_releases"])
    return bad


def _threads_child(so, G, m, n_threads, rounds):
    """the child process of the CPU-tier case: prints what differs as JSON"""
    nif = Nif(so)
    base = nif.counts()
    bad = _threads(nif, G, m, n_threads, rounds)
    c = nif.counts()
    if c["binaries"] != base["binaries"] or c["resources"] != base["resources"]:
        bad.append("leaked: %d binaries, %d resources" % (c["binaries"] - base["binaries"],
                                                         c["resources"] - base["resources"]))
    print("RESULT " + json.dumps(bad))


def test_engines_on_threads_emu(nif_emu):
    """8 threads, each with its own engine (ctypes releases the GIL for every foreign call).  In a child process, so
    that memory corruption shows as a failed test rather than the end of the test run."""
    so = nif_emu.l._name
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_nif_shim as t; t._threads_child(%r, 16, 3, 8, 300)"
            % (ROOT, os.path.join(ROOT, "tests"), so))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    line = next((x for x in r.stdout.splitlines() if x.startswith("RESULT ")), None)
    assert r.returncode == 0 and line, "child exited %d: %s" % (r.returncode, (r.stderr or r.stdout)[-2000:])
    assert json.loads(line[7:]) == []


@pytest.mark.gpu
def test_engines_on_threads_engine(nif_gpu):
    """two engines on device 0 driven from two threads at once"""
    base = nif_gpu.counts()
    assert _threads(nif_gpu, 1200, 5, 2, 20) == []
    c = nif_gpu.counts()
    assert (c["binaries"], c["resources"]) == (base["binaries"], base["resources"])


# ---- h. the NIF table is the Erlang module's face -------------------------------------------------------------------
def test_nif_table_matches_erlang_exports(nif_emu):
    src = open(os.path.join(ROOT, "erlang", "src", "ra_engine_nif.erl")).read()
    exports = re.search(r"-export\(\[(.*?)\]\)", src, re.S).group(1)
    want = sorted((n, int(a)) for n, a in re.findall(r"(\w+)/(\d+)", exports))
    table = nif_emu.table()
    assert sorted((n, a) for n, a, _ in table) == want
    assert len(table) == len(want)
    assert all(f == 1 for *_, f in table)                         # ERL_NIF_DIRTY_JOB_CPU_BOUND
    assert nif_emu.l.ra_stub_module().decode() == "ra_engine_nif"
