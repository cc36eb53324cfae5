"""The C-ABI library loads and exports every symbol include/pase_b200.h declares
(no compute calls: runs without a GPU)."""
import ctypes
import os

import pytest

from pase_b200 import _lib


def test_header_parses():
    assert len(_lib.PROTOS) >= 40
    for name, (ret, params) in _lib.PROTOS.items():
        assert name.startswith("pase_")
        for (t, is_ptr, pname) in params:
            assert t in ("int", "long", "float", "double", "void"), (name, t)


def test_library_exports_every_declared_symbol():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    missing = [n for n in _lib.PROTOS if not hasattr(L, n)]
    assert not missing, "declared in include/pase_b200.h but not exported: %s" % missing
    assert L.pase_version() >= 100
    _lib.lib()


def test_no_cpu_fallback():
    import torch
    with pytest.raises(RuntimeError, match="CUDA device"):
        _lib.call("pase_axpy", torch.zeros(4), torch.zeros(4), 4, 1.0)
    with pytest.raises(TypeError):
        _lib.call("pase_axpy", torch.zeros(4))


def test_product_never_imports_oracle():
    import re
    root = os.path.dirname(os.path.abspath(_lib.__file__))
    for dirpath, _, files in os.walk(root):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(import|from)\s+(pase_oracle|ref_harness|oracle|emul)",
                                     src, re.M), f
