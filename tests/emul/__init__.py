"""TEST-ONLY torch emulation of the C-ABI kernels (include/pase_b200.h).

Purpose: (1) on a GPU-less box, check the HOST-side orchestration of pase_b200 (geometry,
buffer plan, padding/folding index math, gradient routing) against the golden vectors by
monkeypatching ``pase_b200.ops.call`` with ``call``; (2) on the GPU, serve as the per-kernel
semantic spec each CUDA kernel is compared with.  It is never imported by the product package.

All buffer arguments are flat 1-D tensor views (base-pointer semantics); the emulation
interprets them with explicit strides exactly like the kernels do and writes results in place.
Each entry point is the function of its name in exactly one family module.
"""
import torch

from pase_b200 import _lib

from . import core, data, heads, input_grad, optim, packed, windowed


def _registry(families):
    reg = {}
    for mod in families:
        for name in vars(mod):
            if name.startswith("pase_"):
                if name in reg:
                    raise ImportError("%s is emulated in both %s and %s"
                                      % (name, reg[name].__name__, mod.__name__))
                reg[name] = mod
    return reg


# entry-point name -> the module that emulates it
REGISTRY = _registry((core, packed, windowed, input_grad, heads, data, optim))


def user_arity(name):
    """Arguments a caller passes to `name`: its header parameters but the trailing stream."""
    params = _lib.PROTOS[name][1]
    return len(params) - (1 if params and params[-1][2] == "stream" else 0)


def call(name, *args):
    """Run the emulation of entry point `name` in place, as ``pase_b200._lib.call`` runs the
    kernel.  The function is looked up on its module at every call, so a module attribute
    swapped in place reaches every path that launches it."""
    mod = REGISTRY.get(name)
    if mod is None:
        raise LookupError("no emulation for %s" % name)
    n_user = user_arity(name)
    if len(args) != n_user:
        raise TypeError("%s expects %d arguments, got %d" % (name, n_user, len(args)))
    with torch.set_grad_enabled(name == "pase_sinc_grad"):     # sinc_grad runs autograd
        getattr(mod, name)(*args)
    return 0
