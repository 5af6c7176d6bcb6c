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
from .net.tables import EnvParams, NetTables


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _np(a, ct):
    return None if a is None else a.ctypes.data_as(C.POINTER(ct))


class BatchedSim:
    def __init__(self, net: NetTables, params: EnvParams, n_replicas: int, device: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("BatchedSim needs a CUDA device (no CPU fallback exists)")
        self.net, self.params, self.R = net, params, int(n_replicas)
        self.device = torch.device("cuda", device)
        self._cnet, self._ccfg = net.as_c(), params.as_c()
        h = C.c_void_p()
        _lib.check(_lib.lib().tsc_create(C.byref(self._cnet), C.byref(self._ccfg), C.c_int32(self.R),
                                         C.c_int32(device), C.byref(h)))
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
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # ---- control -------------------------------------------------------------------------
    def reset(self, seeds) -> None:
        seeds = np.ascontiguousarray(seeds, dtype=np.uint64)
        assert seeds.shape == (self.R,)
        _lib.check(_lib.lib().tsc_reset(self._h, _np(seeds, C.c_uint64), self._stream()))

    def set_train_mode(self, train: bool) -> None:
        _lib.check(_lib.lib().tsc_set_train_mode(self._h, C.c_int32(int(train))))

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
        _lib.check(_lib.lib().tsc_set_replica_coop_gamma(self._h, _np(cg, C.c_float)))

    def observe(self, fp: Optional[torch.Tensor] = None, obs_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        obs = self.obs if obs_out is None else obs_out
        _lib.check(_lib.lib().tsc_observe(self._h, _ptr(fp), _ptr(obs), self._stream()))
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
        _lib.check(_lib.lib().tsc_step(self._h, _ptr(action), _ptr(fp), _ptr(obs), _ptr(self.reward),
                                       _ptr(self.greward), _ptr(self.done), self._stream()))
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
        _lib.check(_lib.lib().tsc_step_host(self._h, _np(action, C.c_int32), _np(fp, C.c_float),
                                            _np(obs, C.c_float), _np(reward, C.c_float),
                                            _np(greward, C.c_float), _np(done, C.c_uint8), self._stream()))
        return obs, reward, greward, done

    def step_host_range(self, r0: int, n: int, action: np.ndarray, fp: Optional[np.ndarray], obs: np.ndarray,
                        reward: np.ndarray, greward: np.ndarray, done: np.ndarray, sync: bool = True):
        """`tsc_step_host_range`: the host-buffer step for replicas [r0, r0 + n) on the current stream; all arrays are
        the slices of that range (page-locked for full PCIe speed).  Blocks until the slice's results are on the host;
        with sync=False (`tsc_step_host_range_async`) the work is only enqueued and the caller synchronises the stream."""
        fn = _lib.lib().tsc_step_host_range if sync else _lib.lib().tsc_step_host_range_async
        _lib.check(fn(self._h, C.c_int32(r0), C.c_int32(n), _np(action, C.c_int32),
                      _np(fp, C.c_float), _np(obs, C.c_float), _np(reward, C.c_float),
                      _np(greward, C.c_float), _np(done, C.c_uint8), self._stream()))

    # ---- evaluation / recording path (envs/env.py:409-437, 498-542) ------------------------
    def set_record(self, on: bool = True) -> None:
        """Record mode: per-vehicle trip words + arrival log (call right after reset())."""
        _lib.check(_lib.lib().tsc_set_record(self._h, C.c_int32(1 if on else 0)))
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
        _lib.check(_lib.lib().tsc_step_record(self._h, _ptr(action), _ptr(fp), _ptr(obs), _ptr(reward), _ptr(greward),
                                              _ptr(done), _ptr(stats), self._stream()))
        return obs, reward, greward, done, stats

    def trips(self, replica: int = 0) -> np.ndarray:
        """tripinfo rows of one replica: int array [n, 5] = depart_sec, arrival_sec, route, wait_sec, wait_count."""
        rows = np.zeros((8192, 2), np.uint32)
        nr = C.c_int32(0)
        _lib.check(_lib.lib().tsc_get_trips(self._h, C.c_int32(replica), _np(rows, C.c_uint32), C.c_int32(len(rows)),
                                            C.byref(nr)))
        w0, w1 = rows[:nr.value, 0].astype(np.int64), rows[:nr.value, 1].astype(np.int64)
        return np.stack([w0 & 4095, (w0 >> 12) & 4095, w0 >> 24, w1 & 65535, w1 >> 16], axis=1)

    # ---- parity taps ---------------------------------------------------------------------
    def counts(self):
        n = self.net
        veh = torch.zeros(self.R, n.n_det, dtype=torch.int32, device=self.device)
        halt, wait = torch.zeros_like(veh), torch.zeros_like(veh)
        phase = torch.zeros(self.R, n.n_nodes, dtype=torch.int32, device=self.device)
        _lib.check(_lib.lib().tsc_get_counts(self._h, _ptr(veh), _ptr(halt), _ptr(wait), _ptr(phase),
                                             self._stream()))
        return veh, halt, wait, phase

    def dump_state(self, replica: int = 0):
        n = self.net
        cnt = np.zeros(n.n_lanes, np.int32)
        veh = np.zeros((n.n_slots, 3), np.uint32)
        nv = C.c_int32(0)
        _lib.check(_lib.lib().tsc_dump_state(self._h, C.c_int32(replica), _np(cnt, C.c_int32),
                                             _np(veh, C.c_uint32), C.byref(nv)))
        return cnt, veh[:nv.value].copy()

    def traffic_stats(self) -> torch.Tensor:
        """[R, 8] = n_live, departed, arrived, avg_wait, avg_speed, avg_queue, std_queue, backlog
        (the fields of reference _measure_traffic_step, envs/env.py:409-437)."""
        out = torch.zeros(self.R, 8, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib().tsc_get_traffic_stats(self._h, _ptr(out), self._stream()))
        return out

    def mean_live(self) -> float:
        v = C.c_double(0)
        _lib.check(_lib.lib().tsc_mean_live(self._h, C.byref(v)))
        return v.value

    def info(self):
        sb, tpb, sm = C.c_int64(0), C.c_int32(0), C.c_int32(0)
        _lib.check(_lib.lib().tsc_info(self._h, C.byref(sb), C.byref(tpb), C.byref(sm)))
        return dict(state_bytes_per_replica=sb.value, threads_per_block=tpb.value, smem_bytes=sm.value)
