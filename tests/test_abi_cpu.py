"""CPU: the C-ABI shared library builds for sm_90a without a GPU, loads, and exports every function that
include/tsc.h and include/tsc_learn.h declare; the Python loader's symbol list is exactly that set; and the product
path fails loudly without a CUDA device (there is no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    names = set()
    for h in ("tsc.h", "tsc_learn.h"):
        src = open(os.path.join(ROOT, "include", h)).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        names |= set(re.findall(r"^\s*(?:int|const char\*)\s+(tscl?_[a-z0-9_]+)\s*\(", src, flags=re.M))
    return names


def test_library_exports_every_declared_symbol():
    from deeprl_signal_control_b200 import _lib
    so = _lib.LIB_PATH
    if not os.path.exists(so):
        _lib.build_native()
    lib = C.CDLL(so)
    declared = _declared()
    assert len(declared) >= 37 and "tsc_step" in declared and "tscl_wgrad_tc" in declared
    missing = [n for n in sorted(declared) if not hasattr(lib, n)]
    assert not missing, missing
    assert set(_lib.SYMBOLS) == declared          # the loader checks exactly the declared ABI


def test_product_path_fails_loudly_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("needs a machine without a CUDA device")
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    net, par = build_large_grid(agent="greedy"), EnvParams(agent="greedy")
    with pytest.raises(RuntimeError):
        BatchedSim(net, par, 2)
    # the raw ABI reports the failure instead of computing on the host
    lib = _lib.lib()
    cnet, ccfg, h = net.as_c(), par.as_c(), C.c_void_p()
    rc = lib.tsc_create(C.byref(cnet), C.byref(ccfg), C.c_int32(2), C.c_int32(0), C.byref(h))
    assert rc != 0 and len(lib.tsc_last_error()) > 0
    # and nothing in the product package imports the oracle
    pkg = os.path.join(ROOT, "deeprl_signal_control_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), os.path.join(dp, f)
