"""The shared object must export every symbol include/dreammat_b200.h declares (no GPU needed)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    names = set()
    for fn in os.listdir(os.path.join(ROOT, "include")):
        if fn.endswith(".h"):
            txt = open(os.path.join(ROOT, "include", fn)).read()
            txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
            names |= set(re.findall(r"\b(dm_[a-z0-9_]+)\s*\(", txt))
    return sorted(names)


def test_library_builds_loads_and_exports_every_declared_symbol():
    import __graft_entry__ as g
    g.build()
    from dreammat_b200 import _cabi
    lib = ctypes.CDLL(_cabi.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/ but not exported"
        assert s in _cabi.SIGNATURES, f"{s} has no ctypes signature in _cabi.SIGNATURES"
    assert _cabi.lib().dm_version() >= 100


def test_missing_library_fails_loudly(monkeypatch):
    from dreammat_b200 import _cabi
    monkeypatch.setattr(_cabi, "_lib", None)
    monkeypatch.setattr(_cabi, "LIB_PATH", "/nonexistent/libdreammat_b200.so")
    with pytest.raises(_cabi.DmError):
        _cabi.lib()


def test_dm_tune_accepts_only_its_switches():
    from dreammat_b200._cabi import lib
    assert lib().dm_tune(b"mc_frontier", 2) == -1
    for key in (b"mc_skip_horizon", b"bvh_leaf", b"no_such_key"):
        assert lib().dm_tune(key, 1) == -1, key
    assert lib().dm_tune(b"mc_frontier", 1) == 0 and lib().dm_tune(b"pdl", 1) == 0   # the defaults


def test_host_side_layout_queries():
    from dreammat_b200 import render_ops as ops
    cfg = ops.default_hashgrid_cfg()
    n, offs = ops.hashgrid_num_params(cfg)
    assert n == 12599920 and offs[1] == 4096 and len(offs) == 17
