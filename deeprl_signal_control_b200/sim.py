"""`BatchedSim`: R lock-stepped road-network replicas on one GPU (thin ctypes shim over libtsc).

PyTorch is used only as the owner of device buffers and streams; all simulation work happens in
the hand-written kernel `tsc_step_kernel` (csrc/tsc_sim.cu).  Replaces, for R replicas at once,
what reference envs/env.py does against one SUMO process: `reset` (:544-561), `step` (:566-631),
`update_fingerprint` (:633-635) and the detector reads (:325-407).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .net.tables import EnvParams, NetTables


class BatchedSim:
    def __init__(self, net: NetTables, params: EnvParams, n_replicas: int, device: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("BatchedSim needs a CUDA device (no CPU fallback exists)")
        self.net, self.params, self.R = net, params, int(n_replicas)
        self.device = torch.device("cuda", device)
        self._cnet, self._ccfg = net.as_c(), params.as_c()
        h = C.c_void_p()
        _lib.check(_lib.lib().tsc_create(C.byref(self._cnet), C.byref(self._ccfg), self.R, device, C.byref(h)))
        self._h = h
        N = net.n_nodes
        with torch.cuda.device(self.device):
            self.obs = torch.zeros(self.R, net.n_obs, dtype=torch.float32, device=self.device)
            self.reward = torch.zeros(self.R, N, dtype=torch.float32, device=self.device)
            self.greward = torch.zeros(self.R, dtype=torch.float32, device=self.device)
            self.done = torch.zeros(self.R, dtype=torch.uint8, device=self.device)

    def close(self):
        if getattr(self, "_h", None) is not None:
            _lib.lib().tsc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return _lib.stream(self.device)

    # ---- control -------------------------------------------------------------------------
    def reset(self, seeds) -> None:
        seeds = np.ascontiguousarray(seeds, dtype=np.uint64)
        assert seeds.shape == (self.R,)
        _lib.check(_lib.lib().tsc_reset(self._h, seeds.ctypes.data, self._stream()))

    def set_train_mode(self, train: bool) -> None:
        _lib.check(_lib.lib().tsc_set_train_mode(self._h, int(train)))

    def set_replica_coop_gamma(self, values=None) -> None:
        """MA2C spatial discount per replica (`tsc_set_replica_coop_gamma`): `values` [R] floats, replica r then steps as
        a simulator built with coop_gamma = values[r]; None returns to the configured coop_gamma.  The scaled observation
        entries are the ones the network was built to scale, so a network built with coop_gamma = 1 (none scaled) takes
        only values of 1."""
        if values is None:
            _lib.check(_lib.lib().tsc_set_replica_coop_gamma(self._h, None))
            return
        cg = np.ascontiguousarray(values, dtype=np.float32)
        if cg.shape != (self.R,):
            raise ValueError("set_replica_coop_gamma takes %d values (got shape %s)" % (self.R, cg.shape))
        if not (np.asarray(self.net.obs_scale) != 1.0).any() and (cg != 1.0).any() and self.params.agent == "ma2c":
            raise ValueError("the network was built with coop_gamma = 1, so no observation entry is scaled; build it "
                             "with a coop_gamma other than 1")
        _lib.check(_lib.lib().tsc_set_replica_coop_gamma(self._h, cg.ctypes.data))

    def set_replica_demand(self, levels=None, level_of=None) -> None:
        """Traffic demand per replica (`tsc_set_replica_demand`): `levels` a list of NetTables that differ from the
        built net at most in their demand tables (net.tables.DEMAND_FIELDS; anything else is refused, naming the
        field; under ma2c the observation scale too, which set_replica_coop_gamma sets per replica), `level_of` [R]
        ints, the level of each replica.  Replica r then steps as a simulator built with levels[level_of[r]].
        Identical levels are uploaded once.  None returns to the built tables."""
        from .net.tables import DEMAND_FIELDS, demand_mismatch
        lib = _lib.lib()
        if levels is None:
            _lib.check(lib.tsc_set_replica_demand(self._h, 0, None, None, None, None))
            return
        level_of = np.ascontiguousarray(level_of, dtype=np.int64)
        if level_of.shape != (self.R,):
            raise ValueError("set_replica_demand takes %d levels of replicas (got shape %s)" % (self.R, level_of.shape))
        if len(levels) == 0 or level_of.min() < 0 or level_of.max() >= len(levels):
            raise ValueError("set_replica_demand: every replica's level must index the %d levels" % len(levels))
        n, stoch = self.net, self.net.n_pint > 0
        uniq, index = [], []
        for k, t in enumerate(levels):
            f = demand_mismatch(n, t, ignore=("obs_scale",) if self.params.agent == "ma2c" else ())
            if f is not None:
                raise ValueError("demand level %d differs from the built net in %r, not only in its demand" % (k, f))
            key = tuple(np.asarray(getattr(t, name)).tobytes() for name in DEMAND_FIELDS)
            if key not in [u[0] for u in uniq]:
                uniq.append((key, t))
            index.append([u[0] for u in uniq].index(key))
        due = np.ascontiguousarray(np.stack([np.asarray(t.src_due, np.uint8).reshape(n.horizon, n.n_src)
                                             for _, t in uniq]))
        plo = phi = None
        if stoch:
            plo = np.ascontiguousarray(np.stack([np.asarray(t.src_plo, np.float32) for _, t in uniq]))
            phi = np.ascontiguousarray(np.stack([np.asarray(t.src_phi, np.float32) for _, t in uniq]))
        lv = np.ascontiguousarray(np.asarray(index, np.int32)[level_of])
        _lib.check(lib.tsc_set_replica_demand(self._h, len(uniq), due.ctypes.data, None if plo is None else plo.ctypes.data,
                                              None if phi is None else phi.ctypes.data, lv.ctypes.data))

    def observe(self, fp: Optional[torch.Tensor] = None, obs_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        obs = self.obs if obs_out is None else obs_out
        _lib.check(_lib.lib().tsc_observe(self._h, ptr(fp), ptr(obs), self._stream()))
        return obs

    def step(self, action: torch.Tensor, fp: Optional[torch.Tensor] = None,
             obs_out: Optional[torch.Tensor] = None):
        """action int32 [R, n_nodes] on the device; fp float32 [R, n_nodes, max_na] or None.
        `obs_out` (contiguous [R, n_obs] device tensor) lets the caller receive the observation in
        its own buffer (the learner's rollout slot) without a copy.
        Returns the output tensors (obs, reward, global_reward, done)."""
        assert action.dtype == torch.int32 and action.is_cuda and action.is_contiguous()
        assert action.numel() == self.R * self.net.n_nodes
        if fp is not None:
            assert fp.dtype == torch.float32 and fp.is_contiguous()
            assert fp.numel() == self.R * self.net.n_nodes * self.net.max_na
        obs = self.obs if obs_out is None else obs_out
        assert obs.is_contiguous() and obs.numel() == self.R * self.net.n_obs
        _lib.check(_lib.lib().tsc_step(self._h, ptr(action), ptr(fp), ptr(obs), ptr(self.reward), ptr(self.greward),
                                       ptr(self.done), self._stream()))
        return obs, self.reward, self.greward, self.done

    def step_host(self, action: np.ndarray, fp: Optional[np.ndarray] = None):
        """Host-buffer entry point (`tsc_step_host`): numpy in, numpy out, copies included."""
        n = self.net
        action = np.ascontiguousarray(action, np.int32).reshape(self.R, n.n_nodes)
        fp = None if fp is None else np.ascontiguousarray(fp, np.float32)
        if not hasattr(self, "_h_out"):     # page-locked output buffers: D2H copies run at full PCIe/C2C speed
            self._h_out_t = (torch.zeros(self.R, n.n_obs, dtype=torch.float32).pin_memory(),
                             torch.zeros(self.R, n.n_nodes, dtype=torch.float32).pin_memory(),
                             torch.zeros(self.R, dtype=torch.float32).pin_memory(),
                             torch.zeros(self.R, dtype=torch.uint8).pin_memory())
            self._h_out = tuple(t.numpy() for t in self._h_out_t)
        obs, reward, greward, done = self._h_out
        _lib.check(_lib.lib().tsc_step_host(self._h, action.ctypes.data, None if fp is None else fp.ctypes.data,
                                            obs.ctypes.data, reward.ctypes.data, greward.ctypes.data, done.ctypes.data,
                                            self._stream()))
        return obs, reward, greward, done

    def step_host_range(self, r0: int, n: int, action: np.ndarray, fp: Optional[np.ndarray], obs: np.ndarray,
                        reward: np.ndarray, greward: np.ndarray, done: np.ndarray, sync: bool = True):
        """`tsc_step_host_range`: the host-buffer step for replicas [r0, r0 + n) on the current stream; all arrays are
        the slices of that range (page-locked for full PCIe speed); `action` may be None while a signal program is set.  Blocks until the slice's results are on the host;
        with sync=False (`tsc_step_host_range_async`) the work is only enqueued and the caller synchronises the stream."""
        fn = _lib.lib().tsc_step_host_range if sync else _lib.lib().tsc_step_host_range_async
        _lib.check(fn(self._h, r0, n, None if action is None else action.ctypes.data,
                      None if fp is None else fp.ctypes.data, obs.ctypes.data,
                      reward.ctypes.data, greward.ctypes.data, done.ctypes.data, self._stream()))

    # ---- evaluation / recording path (envs/env.py:409-437, 498-542) ------------------------
    def set_record(self, on: bool = True) -> None:
        """Record mode: per-vehicle trip words + arrival log (call right after reset())."""
        _lib.check(_lib.lib().tsc_set_record(self._h, 1 if on else 0))
        self.record = bool(on)

    def step_record(self, action: torch.Tensor, fp: Optional[torch.Tensor] = None):
        """step() one simulated second per launch; also returns the per-second traffic statistics
        [R, control_interval_sec, 8] (fields of traffic_stats())."""
        n = self.net
        action = action.to(self.device, torch.int32).contiguous()
        obs = torch.empty(self.R, n.n_obs, dtype=torch.float32, device=self.device)
        reward = torch.empty(self.R, n.n_nodes, dtype=torch.float32, device=self.device)
        greward = torch.empty(self.R, dtype=torch.float32, device=self.device)
        done = torch.empty(self.R, dtype=torch.uint8, device=self.device)
        stats = torch.zeros(self.R, self.params.control_interval_sec, 8, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib().tsc_step_record(self._h, ptr(action), ptr(fp), ptr(obs), ptr(reward), ptr(greward),
                                              ptr(done), ptr(stats), self._stream()))
        return obs, reward, greward, done, stats

    def trips(self, replica: int = 0) -> np.ndarray:
        """tripinfo rows of one replica: int array [n, 5] = depart_sec, arrival_sec, route, wait_sec, wait_count."""
        rows = np.zeros((8192, 2), np.uint32)
        nr = C.c_int32(0)
        _lib.check(_lib.lib().tsc_get_trips(self._h, replica, rows.ctypes.data, len(rows), C.byref(nr)))
        w0, w1 = rows[:nr.value, 0].astype(np.int64), rows[:nr.value, 1].astype(np.int64)
        return np.stack([w0 & 4095, (w0 >> 12) & 4095, w0 >> 24, w1 & 65535, w1 >> 16], axis=1)

    def pressure_actions(self, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Max-pressure phases of every replica (`tsc_pressure_actions`) from the state the last step / observe left:
        int32 [R, n_nodes] on the device, into `out` when given."""
        act = torch.empty(self.R, self.net.n_nodes, dtype=torch.int32, device=self.device) if out is None else out
        assert act.dtype == torch.int32 and act.is_contiguous() and act.numel() == self.R * self.net.n_nodes
        _lib.check(_lib.lib().tsc_pressure_actions(self._h, ptr(act), self._stream()))
        return act

    def set_signal_program(self, program=None) -> None:
        """Fixed-time control (`tsc_set_signal_program`): every replica runs `program` (an envs.fixedtime.SignalProgram
        in the net's node order) second by second, and step / step_record / the host steps read no action; their
        phase tap holds the program phase of each interval's first second.  None returns to action-driven stepping."""
        lib = _lib.lib()
        if program is None:
            _lib.check(lib.tsc_set_signal_program(self._h, 0, None, None, None, None, None, None))
            return
        if len(program.n_phases) != self.net.n_nodes:
            raise ValueError("set_signal_program: %d node programs for %d nodes" % (len(program.n_phases), self.net.n_nodes))
        a = [np.ascontiguousarray(x, t) for x, t in ((program.n_phases, np.int32), (program.dur, np.int32),
                                                    (program.open, np.uint32), (program.major, np.uint32),
                                                    (program.yellow, np.uint32), (program.offset, np.int32))]
        _lib.check(lib.tsc_set_signal_program(self._h, program.max_phases, *(x.ctypes.data for x in a)))

    def set_replica_signal_programs(self, programs=None, plan_of=None) -> None:
        """Fixed-time control per replica (`tsc_set_replica_signal_programs`): `programs` a list of
        envs.fixedtime.SignalProgram in the net's node order, `plan_of` [R] ints; replica r then runs programs[plan_of[r]]
        as a simulator under set_signal_program(programs[plan_of[r]]) would.  The programs are padded to the largest
        max_phases, and identical programs are uploaded once.  None returns to action-driven stepping."""
        lib = _lib.lib()
        if programs is None:
            _lib.check(lib.tsc_set_replica_signal_programs(self._h, 0, 0, *([None] * 7)))
            return
        plan_of = np.ascontiguousarray(plan_of, dtype=np.int64)
        if plan_of.shape != (self.R,):
            raise ValueError("set_replica_signal_programs takes %d plans of replicas (got shape %s)"
                             % (self.R, plan_of.shape))
        if len(programs) == 0 or plan_of.min() < 0 or plan_of.max() >= len(programs):
            raise ValueError("set_replica_signal_programs: every replica's plan must index the %d programs" % len(programs))
        N = self.net.n_nodes
        for k, p in enumerate(programs):
            if len(p.n_phases) != N:
                raise ValueError("set_replica_signal_programs: program %d has %d node programs for %d nodes"
                                 % (k, len(p.n_phases), N))
        P = max(p.max_phases for p in programs)
        uniq, index = {}, []                  # tables -> (plan index, tables)
        for p in programs:
            rows = tuple(np.pad(np.asarray(x, t), ((0, 0), (0, P - p.max_phases))) for x, t in
                         ((p.dur, np.int32), (p.open, np.uint32), (p.major, np.uint32), (p.yellow, np.uint32)))
            plan = (np.asarray(p.n_phases, np.int32), np.asarray(p.offset, np.int32)) + rows
            key = tuple(x.tobytes() for x in plan)
            if key not in uniq:
                uniq[key] = (len(uniq), plan)
            index.append(uniq[key][0])
        n_phases, offset, dur, opn, major, yellow = (
            np.ascontiguousarray(np.stack([u[1][f] for u in uniq.values()])) for f in range(6))
        plan = np.ascontiguousarray(np.asarray(index, np.int32)[plan_of])
        _lib.check(lib.tsc_set_replica_signal_programs(self._h, len(uniq), P, n_phases.ctypes.data, dur.ctypes.data,
                                                       opn.ctypes.data, major.ctypes.data, yellow.ctypes.data,
                                                       offset.ctypes.data, plan.ctypes.data))

    def set_actuated_program(self, program=None, max_gap=None) -> None:
        """Actuated control (`tsc_set_actuated_program`): every replica runs `program` (an envs.actuated.ActuatedProgram
        in the net's node order) second by second from its initial state, which reset() restores; the steps read no
        action, as under set_signal_program.  `max_gap` (int32 [n_nodes], whole seconds) replaces the program's.
        None returns to action-driven stepping."""
        lib = _lib.lib()
        if program is None:
            _lib.check(lib.tsc_set_actuated_program(self._h, 0, *([None] * 9)))
            return
        if len(program.n_phases) != self.net.n_nodes or len(program.loop_pos) != self.net.n_lanes:
            raise ValueError("set_actuated_program: %d node programs and %d loop positions for %d nodes and %d lanes"
                             % (len(program.n_phases), len(program.loop_pos), self.net.n_nodes, self.net.n_lanes))
        mg = program.max_gap if max_gap is None else max_gap
        a = [np.ascontiguousarray(x, t) for x, t in (
            (program.n_phases, np.int32), (program.min_dur, np.int32), (program.max_dur, np.int32),
            (program.open, np.uint32), (program.major, np.uint32), (program.yellow, np.uint32), (program.init, np.int32),
            (mg, np.int32), (program.loop_pos, np.int32))]
        _lib.check(lib.tsc_set_actuated_program(self._h, program.max_phases, *(x.ctypes.data for x in a)))

    def program_phase(self, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`tsc_get_program_phase`: int32 [R, n_nodes] on the device, the phase every node's signal program (each
        replica's own under set_replica_signal_programs) shows in the next simulated second (into `out` when given)."""
        ph = torch.empty(self.R, self.net.n_nodes, dtype=torch.int32, device=self.device) if out is None else out
        assert ph.dtype == torch.int32 and ph.is_contiguous() and ph.numel() == self.R * self.net.n_nodes
        _lib.check(_lib.lib().tsc_get_program_phase(self._h, ptr(ph), self._stream()))
        return ph

    # ---- parity taps ---------------------------------------------------------------------
    def counts(self):
        n = self.net
        veh = torch.zeros(self.R, n.n_det, dtype=torch.int32, device=self.device)
        halt, wait = torch.zeros_like(veh), torch.zeros_like(veh)
        phase = torch.zeros(self.R, n.n_nodes, dtype=torch.int32, device=self.device)
        _lib.check(_lib.lib().tsc_get_counts(self._h, ptr(veh), ptr(halt), ptr(wait), ptr(phase), self._stream()))
        return veh, halt, wait, phase

    def dump_state(self, replica: int = 0):
        n = self.net
        cnt = np.zeros(n.n_lanes, np.int32)
        veh = np.zeros((n.n_slots, 3), np.uint32)
        nv = C.c_int32(0)
        _lib.check(_lib.lib().tsc_dump_state(self._h, replica, cnt.ctypes.data, veh.ctypes.data, C.byref(nv)))
        return cnt, veh[:nv.value].copy()

    def traffic_stats(self) -> torch.Tensor:
        """[R, 8] = n_live, departed, arrived, avg_wait, avg_speed, avg_queue, std_queue, backlog
        (the fields of reference _measure_traffic_step, envs/env.py:409-437)."""
        out = torch.zeros(self.R, 8, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib().tsc_get_traffic_stats(self._h, ptr(out), self._stream()))
        return out

    def mean_live(self) -> float:
        v = C.c_double(0)
        _lib.check(_lib.lib().tsc_mean_live(self._h, C.byref(v)))
        return v.value

    def info(self):
        sb, tpb, sm = C.c_int64(0), C.c_int32(0), C.c_int32(0)
        _lib.check(_lib.lib().tsc_info(self._h, C.byref(sb), C.byref(tpb), C.byref(sm)))
        return dict(state_bytes_per_replica=sb.value, threads_per_block=tpb.value, smem_bytes=sm.value)
