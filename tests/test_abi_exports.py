"""`-m "not gpu"`: the C-ABI library loads and exports every symbol include/ra_engine.h declares
(no compute calls: there is no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "ra_engine.h")).read()
    return sorted(set(re.findall(r"\b(ra_engine_[a-z_]+)\s*\(", src)))


def test_header_symbols_exported():
    so = os.path.join(ROOT, "ra_b200", "csrc", "libra_engine.so")
    assert os.path.exists(so), "build the engine first: python -c 'import __graft_entry__ as g; g.build()'"
    lib = ctypes.CDLL(so)
    names = _declared()
    assert len(names) >= 10
    for n in names:
        assert hasattr(lib, n), n
    from ra_b200 import engine
    assert sorted(engine.EXPORTS) == names
    src = open(os.path.join(ROOT, "include", "ra_engine.h")).read()
    sim = sorted(set(re.findall(r"\b(ra_hostsim_[a-z_]+)\s*\(", src)))
    assert sim == sorted(engine.HOSTSIM_EXPORTS)
    for n in sim + engine.HOST_EXPORTS:
        assert hasattr(lib, n), n
    assert sorted(set(re.findall(r"\b(ra_wal_[a-z_]+|ra_notes16_[a-z_]+)\s*\(", src))) == sorted(engine.HOST_EXPORTS)


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
