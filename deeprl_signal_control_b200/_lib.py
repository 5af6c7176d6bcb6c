"""Loader of the native library (csrc/libtsc.so, C ABI of include/tsc.h and include/tsc_learn.h).

There is deliberately NO fallback: if the CUDA library is missing or does not load, importing
the simulator fails loudly (the product path never routes through a CPU implementation).

The headers are the one statement of the ABI: every function they declare gets its ctypes `argtypes` / `restype` from
its prototype when the library loads, so callers pass plain values (Python ints / floats / bools, `ptr(t)`, None,
`ctypes.byref(...)`) and a call with too few arguments or a value of the wrong kind raises in Python before any launch.
"""
from __future__ import annotations

import ctypes as C
import os
import re
import subprocess

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")
HEADERS = ("tsc.h", "tsc_learn.h")
LIB_PATH = os.environ.get("TSC_LIB", os.path.join(CSRC, "libtsc.so"))   # TSC_LIB: tuning variants only
_lib = None

# C parameter types of the headers; every pointer (T*, const T*, T**, handles, structs) is a c_void_p
SCALAR_TYPES = {"int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64, "float": C.c_float}
RESULT_TYPES = {"int": C.c_int, "const char*": C.c_char_p}


def _param_type(fn: str, decl: str):
    if "*" in decl:
        return C.c_void_p
    words = decl.split()
    if words[0] == "const":
        words = words[1:]
    if len(words) != 2 or words[0] not in SCALAR_TYPES:
        raise ImportError("%s: no ctypes mapping for parameter `%s` (add its type to _lib.SCALAR_TYPES)" % (fn, decl))
    return SCALAR_TYPES[words[0]]


def _prototypes() -> dict:
    """{name: (restype, [argtypes])} of every function the headers declare, in declaration order."""
    protos = {}
    for header in HEADERS:
        path = os.path.join(INCLUDE, header)
        if not os.path.exists(path):
            raise ImportError("C header %s is missing: the loader takes the library's prototypes from it" % path)
        src = re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)
        for ret, fn, params in re.findall(r"^\s*(int|const char\*)\s+(tscl?_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src,
                                          flags=re.M):
            params = " ".join(params.split())
            protos[fn] = (RESULT_TYPES[ret],
                          [] if params in ("", "void") else [_param_type(fn, p.strip()) for p in params.split(",")])
    return protos


PROTOTYPES = _prototypes()
SYMBOLS = list(PROTOTYPES)


def build_native(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu for sm_90a (H100) with nvcc (cross-compiles without a GPU)."""
    cmd = ["make", "-C", CSRC] + (["-B"] if force else [])
    out = subprocess.run(cmd, capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("nvcc build of libtsc.so failed:\n" + out.stdout + out.stderr)
    if verbose:
        print(out.stdout + out.stderr)
    return LIB_PATH


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "native library %s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)" % LIB_PATH)
        so = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in PROTOTYPES.items():
            fn = getattr(so, name)  # AttributeError here = ABI drift
            fn.restype, fn.argtypes = restype, argtypes
        _lib = so
    return _lib


def ptr(t):
    """Address of tensor `t` as a pointer argument (None: NULL)."""
    return None if t is None else t.data_ptr()


def stream(device=None):
    """Handle of torch's current CUDA stream on `device`, the `void* stream` argument of the entry points."""
    return torch.cuda.current_stream(device).cuda_stream


def check(rc: int):
    if rc != 0:
        raise RuntimeError("libtsc: " + lib().tsc_last_error().decode())
