"""ctypes binding of the C-ABI library (include/pase_b200.h).

The prototypes are parsed from the header, so the binding cannot drift from the
declared ABI.  There is NO fallback: if the shared library is missing or a call
fails, a RuntimeError is raised (the product path must never silently run
anywhere but in the CUDA kernels).
"""
import ctypes
import os
import re
import subprocess
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
HEADER = os.path.join(ROOT, "include", "pase_b200.h")
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(CSRC, "libpase_b200.so")

_CTYPES = {
    "int": ctypes.c_int, "long": ctypes.c_long, "float": ctypes.c_float,
    "double": ctypes.c_double,
}
_PTR_DTYPES = {"float": torch.float32, "double": torch.float64, "int": torch.int32,
               "long": torch.int64, "void": None}


def parse_header(path=HEADER):
    """-> {name: (restype, [(ctype_name, is_pointer, param_name), ...])}"""
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"(const\s+char\s*\*|int)\s+(pase_\w+)\s*\(([^)]*)\)\s*;", src):
        ret, name, args = m.group(1), m.group(2), m.group(3).strip()
        params = []
        if args and args != "void":
            for a in args.split(","):
                a = a.strip()
                is_ptr = "*" in a
                toks = a.replace("*", " ").replace("const", " ").split()
                params.append((toks[0], is_ptr, toks[-1]))
        protos[name] = ("str" if "char" in ret else "int", params)
    return protos


PROTOS = parse_header()
_lib = None


def build(verbose=False):
    """Compile every CUDA source for sm_90a into csrc/libpase_b200.so."""
    cmd = ["make", "-C", CSRC, "-j8"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose:
        print(res.stdout[-4000:])
    if res.returncode != 0:
        raise RuntimeError("building libpase_b200.so failed:\n" + res.stdout[-4000:]
                           + res.stderr[-4000:])
    return LIB_PATH


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "pase_b200: %s not found -- run `python -c 'import __graft_entry__ as g; "
            "g.build()'` (or `make -C pase_b200/csrc`).  There is no CPU fallback."
            % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    for name, (ret, params) in PROTOS.items():
        fn = getattr(L, name)          # AttributeError if the .so lacks a declared symbol
        fn.restype = ctypes.c_char_p if ret == "str" else ctypes.c_int
        fn.argtypes = [ctypes.c_void_p if p else _CTYPES[t] for (t, p, _) in params]
    _lib = L
    return L


def last_error():
    return lib().pase_last_error().decode()


def _ptr(arg, base_type, fname, pname):
    if arg is None:
        return None
    if isinstance(arg, int):
        return arg
    if not isinstance(arg, torch.Tensor):
        raise TypeError("%s(%s): expected tensor/None, got %r" % (fname, pname, type(arg)))
    if not arg.is_cuda:
        raise RuntimeError("%s(%s): tensor must live on a CUDA device (no CPU path)"
                           % (fname, pname))
    want = _PTR_DTYPES[base_type]
    if want is not None and arg.dtype != want:
        raise TypeError("%s(%s): expected %s, got %s" % (fname, pname, want, arg.dtype))
    return arg.data_ptr()


def call(name, *args):
    """Invoke `name` with torch tensors (-> device pointers) and scalars.  The
    trailing `stream` parameter is filled with torch's current stream."""
    L = lib()
    ret, params = PROTOS[name]
    has_stream = bool(params) and params[-1][2] == "stream"
    n_user = len(params) - (1 if has_stream else 0)
    if len(args) != n_user:
        raise TypeError("%s expects %d arguments, got %d" % (name, n_user, len(args)))
    cargs = []
    for (t, is_ptr, pname), a in zip(params, args):
        cargs.append(_ptr(a, t, name, pname) if is_ptr else a)
    if has_stream:
        cargs.append(torch.cuda.current_stream().cuda_stream)
    rc = getattr(L, name)(*cargs)
    if ret == "int" and rc != 0:
        raise RuntimeError("%s failed (code %d): %s" % (name, rc, last_error()))
    return rc


def device_info():
    out = (ctypes.c_int * 4)()
    L = lib()
    rc = L.pase_device_info(ctypes.cast(out, ctypes.c_void_p))
    if rc != 0:
        raise RuntimeError("pase_device_info failed: " + last_error())
    return {"sms": out[0], "cc": (out[1], out[2]), "smem_optin": out[3]}


def tc_gemm_nt_plan(M, N, sms):
    """How pase_tc_gemm_nt covers an M x N output on `sms` SMs: dict(bn, bulk_m, tail_bn,
    tail_pieces); tail_bn 0 = one launch."""
    out = (ctypes.c_int * 4)()
    rc = lib().pase_tc_gemm_nt_plan(M, N, sms, ctypes.cast(out, ctypes.c_void_p))
    if rc != 0:
        raise RuntimeError("pase_tc_gemm_nt_plan failed: " + last_error())
    return {"bn": out[0], "bulk_m": out[1], "tail_bn": out[2], "tail_pieces": out[3]}


def tc_gemm_tn_plan(I, J, groups, rows_per_group, mode):
    """(splits, chunks_per_split) of pase_tc_gemm_tn for this shape on the current device."""
    out = (ctypes.c_int * 2)()
    L = lib()
    rc = L.pase_tc_gemm_tn_plan(I, J, groups, rows_per_group, mode,
                                ctypes.cast(out, ctypes.c_void_p))
    if rc != 0:
        raise RuntimeError("pase_tc_gemm_tn_plan failed: " + last_error())
    return out[0], out[1]


def qrnn_scan_plan(T):
    """Segments per block of the time-segmented QRNN scans for T time steps (16, 24, 32), or 0
    when the sequential kernels run."""
    out = (ctypes.c_int * 1)()
    rc = lib().pase_qrnn_scan_plan(T, ctypes.cast(out, ctypes.c_void_p))
    if rc != 0:
        raise RuntimeError("pase_qrnn_scan_plan failed: " + last_error())
    return out[0]


def bn_bwd_plan(pass_, *args):
    """How a BatchNorm/PReLU backward pass runs on the current device: `args` as the
    pase_bn_bwd_plan arguments after `pass` up to dst_sample_stride (tensors or device
    pointers).  -> dict(path=0 register / 1 staged, rows, items, grid)."""
    out = (ctypes.c_long * 4)()
    call("pase_bn_bwd_plan", pass_, *args, ctypes.addressof(out))
    return {"path": out[0], "rows": out[1], "items": out[2], "grid": out[3]}
