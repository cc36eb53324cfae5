"""The torch emulation of the kernels (tests/emul/) against the C ABI: every emulated name is
declared in include/pase_b200.h with the arguments the emulation takes, every entry point the
product launches is emulated, and ``emul.call`` refuses what ``pase_b200._lib.call`` refuses."""
import inspect
import os
import re
import types

import pytest
import torch

import emul
from pase_b200 import _lib

# declared entry points without an emulation, and why
NOT_EMULATED = {
    "pase_adam_flat_dp": "reads the other ranks' gradients through CUDA peer memory",
    "pase_bn_bwd_plan": "reports the device's launch geometry of a BatchNorm backward; no launch",
    "pase_tc_gemm_nt_plan": "reports the device's tile plan of the NT GEMM; no launch",
    "pase_tc_gemm_tn_plan": "reports the device's split plan of the TN GEMM; no launch",
    "pase_qrnn_scan_plan": "reports the QRNN scan's segmentation; no launch",
    "pase_dp_alloc": "allocates CUDA peer memory",
    "pase_dp_free": "frees CUDA peer memory",
    "pase_dp_open": "maps another process's CUDA peer memory",
    "pase_dp_close": "unmaps another process's CUDA peer memory",
    "pase_device_info": "queries the device",
    "pase_version": "queries the library",
    "pase_last_error": "queries the library",
}


def _launched_names():
    """Entry points named by a string literal as the first argument of call(...) under
    pase_b200/; "pase_x" + suffix counts once for each string literal assigned to suffix in the
    same file."""
    root = os.path.dirname(os.path.abspath(_lib.__file__))
    names = {}
    for dirpath, _, files in os.walk(root):
        for f in files:
            if not f.endswith(".py"):
                continue
            path = os.path.join(dirpath, f)
            src = open(path).read()
            for m in re.finditer(r"\bcall\(\s*\"(pase_\w+)\"(\s*\+\s*(\w+))?", src):
                suffixes = [""]
                if m.group(3):
                    rhs = re.findall(r"^\s*%s\s*=\s*(.*)$" % m.group(3), src, re.M)
                    suffixes = [s for r in rhs for s in re.findall(r"\"(\w*)\"", r)]
                    assert suffixes, "%s: no string assigned to %s" % (path, m.group(3))
                for s in suffixes:
                    names.setdefault(m.group(1) + s, path)
    return names


def test_every_emulation_is_declared():
    undeclared = sorted(set(emul.REGISTRY) - set(_lib.PROTOS))
    assert not undeclared, "emulated but not declared in include/pase_b200.h: %s" % undeclared


def test_emulations_take_the_declared_arguments():
    bad = []
    for name, mod in sorted(emul.REGISTRY.items()):
        params = list(inspect.signature(getattr(mod, name)).parameters.values())
        plain = all(p.kind == p.POSITIONAL_OR_KEYWORD and p.default is p.empty for p in params)
        if not plain or len(params) != emul.user_arity(name):
            bad.append("%s.%s%s (header: %d arguments)" % (
                mod.__name__, name, inspect.signature(getattr(mod, name)), emul.user_arity(name)))
    assert not bad, "emulations whose parameters differ from the header:\n" + "\n".join(bad)


def test_every_launch_is_emulated():
    launched = _launched_names()
    # the GEMM entry points the packed train path names by suffix
    assert {"pase_gemm_nt_var_stats", "pase_tc_gemm_nt_var_stats"} <= set(launched)
    missing = sorted("%s (%s)" % (n, os.path.relpath(p, _lib.ROOT)) for n, p in launched.items()
                     if n not in emul.REGISTRY and n not in NOT_EMULATED)
    assert not missing, "launched but not emulated: %s" % missing
    assert set(NOT_EMULATED) <= set(_lib.PROTOS), "not declared: %s" % (
        sorted(set(NOT_EMULATED) - set(_lib.PROTOS)))
    assert not set(NOT_EMULATED) & set(emul.REGISTRY)
    unaccounted = sorted(set(_lib.PROTOS) - set(emul.REGISTRY) - set(NOT_EMULATED))
    assert not unaccounted, "declared, neither emulated nor excepted: %s" % unaccounted


def test_call_refuses_what_the_library_refuses():
    x, y = torch.ones(4), torch.zeros(4)
    with pytest.raises(TypeError, match="pase_axpy expects 4 arguments, got 3"):
        emul.call("pase_axpy", x, y, 4)
    with pytest.raises(TypeError, match="pase_axpy expects 4 arguments, got 5"):
        emul.call("pase_axpy", x, y, 4, 2.0, None)
    # the trailing stream is the library's to fill, never the caller's
    with pytest.raises(TypeError, match="pase_scatter_copy expects 3 arguments, got 4"):
        emul.call("pase_scatter_copy", torch.zeros(6, dtype=torch.int64), 1, 0, None)
    assert torch.equal(y, torch.zeros(4))
    assert emul.call("pase_axpy", x, y, 4, 2.0) == 0 and torch.equal(y, 2 * x)
    for name in ("pase_adam_flat_dp", "pase_no_such_kernel"):
        with pytest.raises(LookupError, match="no emulation for %s" % name):
            emul.call(name)


def test_registry_refuses_an_entry_point_defined_twice():
    a = types.ModuleType("fam_a")
    b = types.ModuleType("fam_b")
    a.pase_axpy = b.pase_axpy = lambda *args: None
    with pytest.raises(ImportError, match="pase_axpy is emulated in both fam_a and fam_b"):
        emul._registry((a, b))
