"""`-m "not gpu"`: the C-ABI library loads and exports every symbol include/ra_engine.h declares
(no compute calls: there is no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _prototypes():
    """{name: (returns void, number of parameters)} of every function include/ra_engine.h declares"""
    src = open(os.path.join(ROOT, "include", "ra_engine.h")).read()
    out = {}
    for ret, name, params in re.findall(r"^([A-Za-z_][\w \t*]*?)\s*\b(ra_\w+)\s*\(([^;{]*?)\)\s*;", src, re.M | re.S):
        params = params.strip()
        out[name] = (ret.strip() == "void", 0 if params in ("", "void") else params.count(",") + 1)
    return out


def _table():
    from ra_b200 import abi
    return {**{"ra_engine_" + k: v for k, v in abi.SIGNATURES.items()},
            **{"ra_" + k: v for k, v in abi.HOST_SIGNATURES.items()}}


def test_header_symbols_exported():
    so = os.path.join(ROOT, "ra_b200", "csrc", "libra_engine.so")
    assert os.path.exists(so), "build the engine first: python -c 'import __graft_entry__ as g; g.build()'"
    lib = ctypes.CDLL(so)
    names = sorted(_prototypes())
    assert len(names) >= 10
    for n in names:
        assert hasattr(lib, n), n
    assert sorted(_table()) == names


def test_signature_table_matches_header():
    """Every entry of the signature table has the header prototype's parameter count, and agrees on void."""
    protos = _prototypes()
    for name, (restype, argtypes) in _table().items():
        assert protos[name] == (restype is None, len(argtypes)), (name, protos[name])


def test_binding_ignores_declarations_on_the_shared_library():
    """Backend calls go through private function objects: what another caller declares on the library's own
    attribute for a symbol does not change them."""
    import emu_lib
    from ra_b200 import abi

    def run():
        e = emu_lib.Emu(8, 3, route_on_device=True)
        e.reset_empty()
        msgs, notes = e.step_host([abi.ev_simple(e.row_of(g, 0), abi.EV_ELECTION_TIMEOUT) for g in range(8)])
        return [m.key() for m in msgs], [n.key() for n in notes]
    want = run()
    assert want[1]
    shared = emu_lib.lib().ra_engine_step_host
    shared.argtypes = [ctypes.c_int]
    try:
        assert run() == want
    finally:
        shared.argtypes = None


def test_record_sizes_match_header():
    from ra_b200 import abi
    assert ctypes.sizeof(abi.RaEvent) == 64 and ctypes.sizeof(abi.RaNote) == 32


def test_no_device_fails_loudly():
    """Without a GPU the product refuses to run instead of falling back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from ra_b200.engine import Engine, EngineUnavailable
    with pytest.raises(EngineUnavailable):
        Engine(1, 3)


def test_nif_shim_compiles():
    """ra_b200/csrc/ra_engine_nif.c (the dirty-NIF shim of INTEGRATION.md) against the stub of erl_nif.h with every
    warning an error (tests/test_nif_shim.py builds it with the stub's implementation and runs it)."""
    import subprocess
    r = subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-DRA_HAVE_ERL_NIF",
                        "-I" + os.path.join(ROOT, "tests", "nif_stub"),
                        os.path.join(ROOT, "ra_b200", "csrc", "ra_engine_nif.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
