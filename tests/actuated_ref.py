"""The CPU oracle with its actuated mode (tests/actuated_ref.c): `ActuatedRefSim` is oracle.sim_ref.RefSim on a build of
the oracle source that also exports `ref_step_actuated`.  The library is compiled with the oracle's own flags into a
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
    """A private copy of oracle/sim_ref.py whose library is the actuated-mode build."""
    global _MOD
    if _MOD is None:
        so = os.path.join(tempfile.mkdtemp(prefix="actuated_ref_"), "libtsc_actuated_ref.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                               "-o", so, os.path.join(ROOT, "tests", "actuated_ref.c"), "-lm", "-lpthread"])
        spec = importlib.util.spec_from_file_location("actuated_sim_ref", os.path.join(ROOT, "oracle", "sim_ref.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod._LIB = C.CDLL(so)
        mod._LIB.ref_create.restype = C.c_void_p
        _MOD = mod
    return _MOD


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def ActuatedRefSim(net, params, n_replicas, program, max_gap=None):
    """oracle.sim_ref.RefSim (every method as there) running `program` (envs.actuated.ActuatedProgram) with
    `step_actuated(fp=None, record=False)`.  `max_gap` (int32 [n_nodes]) replaces the program's, e.g. 0 (never extend)
    or 256 (always run to max_dur).  `reset` also puts every replica into the program's initial state; `state`
    ([R][n_nodes][2] phase, elapsed) and `gap` ([R][n_lanes]) are the actuated state."""
    mod = _module()

    class _Sim(mod.RefSim):
        def __init__(self):
            super().__init__(net, params, n_replicas)
            self.program = program
            self.max_gap = np.ascontiguousarray(program.max_gap if max_gap is None else max_gap, np.int32)
            self._init_state()

        def _init_state(self):
            self.state = np.ascontiguousarray(np.repeat(program.init[None], self.R, axis=0), np.int32)
            self.gap = np.full((self.R, self.net.n_lanes), 255, np.uint8)

        def reset(self, seeds):
            super().reset(seeds)
            self._init_state()

        def put_vehicle(self, r, lane, xq, route, hop=0, sfq=128):
            """Test set-up: one vehicle at rest on `lane` of replica r, front at xq / 64 m, on hop `hop` of `route`,
            speedFactor 0.5 + sfq / 256 (128: 1.0)."""
            m0 = (int(route) << 16) | (int(hop) << 10) | (int(sfq) << 24)
            if mod.lib().ref_put_vehicle(self.h, C.c_int32(r), C.c_int32(lane), C.c_uint32(int(xq)),
                                         C.c_uint32(m0)) != 0:
                raise ValueError("put_vehicle: lane %d is full" % lane)

        def step_actuated(self, fp=None, record=False):
            """One control step: (obs, reward, greward, done, phase) and, with record=True, the per-second traffic
            statistics [R, control_interval_sec, 8] last."""
            n, R, pg = self.net, self.R, self.program
            a = [np.ascontiguousarray(x, t) for x, t in (
                (pg.n_phases, np.int32), (pg.min_dur, np.int32), (pg.max_dur, np.int32), (pg.open, np.uint32),
                (pg.major, np.uint32), (pg.yellow, np.uint32), (self.max_gap, np.int32), (pg.loop_pos, np.int32))]
            fp = None if fp is None else np.ascontiguousarray(fp, np.float32)
            obs = np.zeros((R, n.n_obs), np.float32)
            reward = np.zeros((R, n.n_nodes), np.float32)
            greward = np.zeros(R, np.float32)
            done = np.zeros(R, np.uint8)
            phase = np.zeros((R, n.n_nodes), np.int32)
            stats = np.zeros((R, self.params.control_interval_sec, 8), np.float32) if record else None
            mod.lib().ref_step_actuated(
                self.h, C.c_int32(pg.max_phases), _p(a[0], C.c_int32), _p(a[1], C.c_int32), _p(a[2], C.c_int32),
                _p(a[3], C.c_uint32), _p(a[4], C.c_uint32), _p(a[5], C.c_uint32), _p(a[6], C.c_int32),
                _p(a[7], C.c_int32), _p(self.state, C.c_int32), _p(self.gap, C.c_uint8), _p(fp, C.c_float),
                _p(obs, C.c_float), _p(reward, C.c_float), _p(greward, C.c_float), _p(done, C.c_uint8),
                _p(stats, C.c_float), _p(phase, C.c_int32))
            out = (obs, reward, greward, done, phase)
            return out + (stats,) if record else out

    return _Sim()
