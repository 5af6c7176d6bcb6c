"""The CPU oracle with its fixed-time mode (tests/fixedtime_ref.c): `FixedRefSim` is oracle.sim_ref.RefSim on a build of
the oracle source that also exports `ref_step_fixed`.  The library is compiled with the oracle's own flags into a
temporary directory, once per process, so the tree is not written."""
import ctypes as C
import importlib.util
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_MOD = None


def _module():
    """A private copy of oracle/sim_ref.py whose library is the fixed-mode build."""
    global _MOD
    if _MOD is None:
        so = os.path.join(tempfile.mkdtemp(prefix="fixedtime_ref_"), "libtsc_fixed_ref.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                               "-o", so, os.path.join(ROOT, "tests", "fixedtime_ref.c"), "-lm", "-lpthread"])
        spec = importlib.util.spec_from_file_location("fixedtime_sim_ref", os.path.join(ROOT, "oracle", "sim_ref.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod._LIB = C.CDLL(so)
        mod._LIB.ref_create.restype = C.c_void_p
        _MOD = mod
    return _MOD


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def FixedRefSim(net, params, n_replicas):
    """oracle.sim_ref.RefSim (every method as there) with `step_fixed(program, fp=None, record=False)`."""
    mod = _module()

    class _Sim(mod.RefSim):
        def step_fixed(self, program, fp=None, record=False):
            """One control step on `program` (envs.fixedtime.SignalProgram): (obs, reward, greward, done, phase) and,
            with record=True, the per-second traffic statistics [R, control_interval_sec, 8] last."""
            n, R = self.net, self.R
            a = [np.ascontiguousarray(x, t) for x, t in ((program.n_phases, np.int32), (program.dur, np.int32),
                                                        (program.open, np.uint32), (program.major, np.uint32),
                                                        (program.yellow, np.uint32), (program.offset, np.int32))]
            fp = None if fp is None else np.ascontiguousarray(fp, np.float32)
            obs = np.zeros((R, n.n_obs), np.float32)
            reward = np.zeros((R, n.n_nodes), np.float32)
            greward = np.zeros(R, np.float32)
            done = np.zeros(R, np.uint8)
            phase = np.zeros((R, n.n_nodes), np.int32)
            stats = np.zeros((R, self.params.control_interval_sec, 8), np.float32) if record else None
            mod.lib().ref_step_fixed(self.h, C.c_int32(program.max_phases), _p(a[0], C.c_int32), _p(a[1], C.c_int32),
                                     _p(a[2], C.c_uint32), _p(a[3], C.c_uint32), _p(a[4], C.c_uint32),
                                     _p(a[5], C.c_int32), _p(fp, C.c_float), _p(obs, C.c_float),
                                     _p(reward, C.c_float), _p(greward, C.c_float), _p(done, C.c_uint8),
                                     _p(stats, C.c_float), _p(phase, C.c_int32))
            out = (obs, reward, greward, done, phase)
            return out + (stats,) if record else out

    return _Sim(net, params, n_replicas)
