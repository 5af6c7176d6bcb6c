"""Flat road-network / demand tables shared by the CUDA simulator and the CPU oracle.

`NetTables` is the Python image of `tsc_net` (include/tsc.h).  Scenario builders
(`large_grid.py`, later `real_net.py`) fill it from the reference's scenario definitions:

* nodes / neighbours / phases     reference envs/large_grid_env.py:38-42,73-101
* lanes, connections, detectors   reference large_grid/data/build_file.py:27-124,360-391
* demand                          reference large_grid/data/build_file.py:268-326
* observation layout              reference envs/env.py:163-205,303-323

Nothing here touches CUDA; `as_c()` only packs numpy arrays into the ctypes struct.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Sequence

import numpy as np

# --------------------------------------------------------------------------------------
# ctypes mirrors of include/tsc.h
# --------------------------------------------------------------------------------------
_P = C.POINTER


class CNet(C.Structure):
    _fields_ = [
        ("n_lanes", C.c_int32), ("n_links", C.c_int32), ("n_nodes", C.c_int32),
        ("n_routes", C.c_int32), ("max_hops", C.c_int32), ("n_src", C.c_int32),
        ("horizon", C.c_int32), ("n_det", C.c_int32), ("n_obs", C.c_int32),
        ("max_phases", C.c_int32), ("max_na", C.c_int32), ("n_slots", C.c_int32),
        ("lane_len", _P(C.c_float)), ("lane_vmax", _P(C.c_float)),
        ("lane_cap", _P(C.c_int32)), ("lane_slot0", _P(C.c_int32)),
        ("lane_inl_off", _P(C.c_int32)), ("lane_inl", _P(C.c_int32)),
        ("link_from", _P(C.c_int32)), ("link_to", _P(C.c_int32)),
        ("link_node", _P(C.c_int32)), ("link_tlidx", _P(C.c_int32)),
        ("link_vmax", _P(C.c_float)), ("link_cross", _P(C.c_uint32)),
        ("link_merge", _P(C.c_uint32)),
        ("route_len", _P(C.c_int32)), ("route_lane", _P(C.c_int16)),
        ("route_link", _P(C.c_int16)),
        ("node_n_phases", _P(C.c_int32)), ("node_green", _P(C.c_uint32)),
        ("node_major", _P(C.c_uint32)),
        ("node_det_off", _P(C.c_int32)), ("det_lane", _P(C.c_int32)),
        ("node_nbr_off", _P(C.c_int32)), ("node_nbr", _P(C.c_int32)),
        ("node_obs_off", _P(C.c_int32)), ("obs_kind", _P(C.c_int32)),
        ("obs_idx", _P(C.c_int32)), ("obs_scale", _P(C.c_float)),
        ("src_lane", _P(C.c_int32)), ("src_route", _P(C.c_int32)),
        ("src_due", _P(C.c_uint8)),
        ("src_group", _P(C.c_int32)), ("src_plo", _P(C.c_float)), ("src_phi", _P(C.c_float)),
        ("n_pint", C.c_int32), ("pint_sec", C.c_int32),
    ]


class CCfg(C.Structure):
    _fields_ = [
        ("veh_len", C.c_float), ("min_gap", C.c_float), ("accel", C.c_float),
        ("decel", C.c_float), ("tau", C.c_float), ("sigma", C.c_float),
        ("speed_dev", C.c_float),
        ("det_len", C.c_float), ("halt_speed", C.c_float), ("queue_cap", C.c_int32),
        ("control_interval_sec", C.c_int32), ("yellow_interval_sec", C.c_int32),
        ("episode_length_sec", C.c_int32), ("teleport_sec", C.c_int32),
        ("norm_wave", C.c_float), ("norm_wait", C.c_float), ("clip_wave", C.c_float),
        ("clip_wait", C.c_float), ("coef_wait", C.c_float), ("coop_gamma", C.c_float),
        ("objective", C.c_int32), ("agent_mode", C.c_int32),
        ("real_net_norm", C.c_int32), ("use_wait", C.c_int32),
    ]


_CT = {np.dtype(np.float32): C.c_float, np.dtype(np.int32): C.c_int32,
       np.dtype(np.uint32): C.c_uint32, np.dtype(np.int16): C.c_int16,
       np.dtype(np.uint8): C.c_uint8}

OBJECTIVES = {"queue": 0, "wait": 1, "hybrid": 2}
# reward shaping families of reference envs/env.py:591-631
# maxpressure (envs.maxpressure_controller), fixedtime (envs.fixedtime_controller) and actuated
# (envs.actuated_controller) are non-learning controllers like greedy and observe what greedy does
AGENT_MODES = {"greedy": 0, "maxpressure": 0, "fixedtime": 0, "actuated": 0, "a2c": 0, "ia2c": 1, "iqll": 1, "iqld": 1,
               "ma2c": 2}


@dataclass
class EnvParams:
    """Scalar part of [ENV_CONFIG] + vType; becomes `tsc_cfg`."""
    veh_len: float = 5.0      # large_grid/data/build_file.py:279
    min_gap: float = 2.5      # SUMO passenger default (SURVEY App. A)
    accel: float = 5.0        # build_file.py:279
    decel: float = 10.0       # build_file.py:279
    tau: float = 1.0          # SUMO default (README.md:63 removed tau=0.5)
    sigma: float = 0.5        # SUMO Krauss default
    speed_dev: float = 0.1    # SUMO >= 1.0 passenger default
    det_len: float = 50.0     # build_file.py:445 pos=-50 endPos=-1
    halt_speed: float = 1.39  # E2 halting threshold (SURVEY App. A)
    queue_cap: int = 1 << 20
    control_interval_sec: int = 5
    yellow_interval_sec: int = 2
    episode_length_sec: int = 3600
    teleport_sec: int = 600   # envs/env.py:281-284
    norm_wave: float = 5.0
    norm_wait: float = 100.0
    clip_wave: float = 2.0
    clip_wait: float = 2.0
    coef_wait: float = 0.2
    coop_gamma: float = 0.9
    objective: str = "hybrid"
    agent: str = "ma2c"
    real_net_norm: bool = False
    use_wait: bool = True

    def as_c(self) -> CCfg:
        c = CCfg()
        for name, _ in CCfg._fields_:
            if name == "objective":
                c.objective = OBJECTIVES[self.objective]
            elif name == "agent_mode":
                c.agent_mode = AGENT_MODES[self.agent]
            elif name in ("real_net_norm", "use_wait"):
                setattr(c, name, int(getattr(self, name)))
            else:
                setattr(c, name, getattr(self, name))
        return c


@dataclass
class NetTables:
    """Python image of `tsc_net`.  All arrays are C-contiguous numpy arrays."""
    # names (host side only; agents are nodes in sorted-name order, envs/env.py:232)
    node_names: List[str]
    lane_names: List[str]
    neighbor_map: Dict[str, List[str]]
    phases: Dict[str, List[str]]          # node name -> phase strings
    lanes_in: Dict[str, List[str]]        # node name -> controlled lanes in link order
    ilds_in: Dict[str, List[str]]         # node name -> de-duplicated incoming lanes
    # dims
    max_hops: int = 0
    horizon: int = 0
    max_phases: int = 0
    max_na: int = 0
    # arrays (see include/tsc.h for meaning)
    lane_len: np.ndarray = None
    lane_vmax: np.ndarray = None
    lane_cap: np.ndarray = None
    lane_slot0: np.ndarray = None
    lane_inl_off: np.ndarray = None
    lane_inl: np.ndarray = None
    link_from: np.ndarray = None
    link_to: np.ndarray = None
    link_node: np.ndarray = None
    link_tlidx: np.ndarray = None
    link_vmax: np.ndarray = None
    link_cross: np.ndarray = None
    link_merge: np.ndarray = None
    route_len: np.ndarray = None
    route_lane: np.ndarray = None
    route_link: np.ndarray = None
    node_n_phases: np.ndarray = None
    node_green: np.ndarray = None
    node_major: np.ndarray = None
    node_det_off: np.ndarray = None
    det_lane: np.ndarray = None
    node_nbr_off: np.ndarray = None
    node_nbr: np.ndarray = None
    node_obs_off: np.ndarray = None
    obs_kind: np.ndarray = None
    obs_idx: np.ndarray = None
    obs_scale: np.ndarray = None
    src_lane: np.ndarray = None
    src_route: np.ndarray = None
    src_due: np.ndarray = None
    # stochastic demand (small_grid): see include/tsc.h; defaults = off
    src_group: np.ndarray = None
    src_plo: np.ndarray = None
    src_phi: np.ndarray = None
    pint_sec: int = 1
    # derived per-agent dims, reference envs/env.py:303-323
    n_s_ls: List[int] = field(default_factory=list)
    n_a_ls: List[int] = field(default_factory=list)
    n_w_ls: List[int] = field(default_factory=list)
    n_f_ls: List[int] = field(default_factory=list)
    route_names: List[str] = field(default_factory=list)

    # ------------------------------------------------------------------
    @property
    def n_lanes(self): return len(self.lane_len)
    @property
    def n_links(self): return len(self.link_from)
    @property
    def n_nodes(self): return len(self.node_names)
    @property
    def n_routes(self): return len(self.route_len)
    @property
    def n_src(self): return len(self.src_lane)
    @property
    def n_det(self): return len(self.det_lane)
    @property
    def n_obs(self): return len(self.obs_kind)
    @property
    def n_slots(self): return int(self.lane_cap.sum())
    @property
    def n_pint(self): return 0 if self.src_plo is None else int(np.asarray(self.src_plo).reshape(-1, max(self.n_src, 1)).shape[0])

    _ARRAYS = [f for f, _ in CNet._fields_ if f not in (
        "n_lanes", "n_links", "n_nodes", "n_routes", "max_hops", "n_src", "horizon",
        "n_det", "n_obs", "max_phases", "max_na", "n_slots", "n_pint", "pint_sec")]

    def finalize(self) -> "NetTables":
        """Coerce dtypes / contiguity so `as_c` can hand out raw pointers."""
        if self.src_group is None:                      # deterministic demand only
            self.src_group = np.full(self.n_src, -1, np.int32)
            self.src_plo = np.zeros((0, self.n_src), np.float32)
            self.src_phi = np.zeros((0, self.n_src), np.float32)
        want = dict(CNet._fields_)
        for name in self._ARRAYS:
            ct = want[name]._type_
            dt = {v: k for k, v in _CT.items()}[ct]
            arr = np.ascontiguousarray(getattr(self, name), dtype=dt)
            setattr(self, name, arr)
        assert self.link_tlidx.max(initial=0) < 32
        assert self.n_lanes < 32767 and self.n_links < 32767
        # vehicle positions are 16-bit fixed point in 1/64 m (include/tsc.h "vehicle record"): lane ends must lie on that
        # grid, so that "crossed the end of the lane" means the same for the computed and for the stored position
        self.lane_len = (np.round(self.lane_len.astype(np.float64) * 64.0) / 64.0).astype(np.float32)
        return self

    def as_c(self) -> CNet:
        """ctypes struct whose pointers alias this object's arrays (keep `self` alive)."""
        c = CNet()
        for name in ("n_lanes", "n_links", "n_nodes", "n_routes", "max_hops", "n_src",
                     "horizon", "n_det", "n_obs", "max_phases", "max_na", "n_slots", "n_pint", "pint_sec"):
            setattr(c, name, int(getattr(self, name)))
        want = dict(CNet._fields_)
        for name in self._ARRAYS:
            arr = getattr(self, name)
            setattr(c, name, arr.ctypes.data_as(want[name]))
        c._keepalive = self
        return c


# the tables that carry a scenario's traffic demand: two nets that differ only in these are one simulator with
# per-replica demand levels (tsc_set_replica_demand, BatchedSim.set_replica_demand)
DEMAND_FIELDS = ('src_due', 'src_plo', 'src_phi')


def _same_value(a, b) -> bool:
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)
    return a == b


def demand_mismatch(a: NetTables, b: NetTables, ignore=()):
    """The name of the first NetTables field, other than DEMAND_FIELDS and `ignore`, in which `a` and `b` differ, or
    None when they differ at most in their demand."""
    import dataclasses
    for f in dataclasses.fields(NetTables):
        if f.name in DEMAND_FIELDS or f.name in ignore:
            continue
        if not _same_value(getattr(a, f.name), getattr(b, f.name)):
            return f.name
    return None


# --------------------------------------------------------------------------------------
# builders shared by all scenarios
# --------------------------------------------------------------------------------------
def phase_masks(phase_strings: Sequence[str]):
    """'GGgrrr...' -> (green bitmask, major bitmask); bit i <-> link index i.

    Alphabet of the reference phase tables is {G, g, r} (envs/large_grid_env.py:40-41,
    envs/real_net_env.py:49-68)."""
    greens, majors = [], []
    for s in phase_strings:
        g = m = 0
        for i, ch in enumerate(s):
            if ch not in "Ggr":
                raise ValueError("unsupported signal char %r" % ch)
            if ch in "Gg":
                g |= 1 << i
            if ch == "G":
                m |= 1 << i
        greens.append(g)
        majors.append(m)
    return greens, majors


def flow_due_table(flows, horizon: int, n_src: int) -> np.ndarray:
    """flows: iterable of (src index, begin, end, vehsPerHour:int).

    A SUMO `<flow vehsPerHour=q begin=b end=e>` departs vehicle j at b + j*3600/q while that is
    < e; a vehicle becomes due in the first whole second >= its depart time.  Integer
    arithmetic only, so CPU oracle and GPU agree exactly."""
    due = np.zeros((horizon, n_src), dtype=np.int64)
    for s, b, e, q in flows:
        q = int(q)
        if q <= 0:
            continue
        j = 0
        while j * 3600 < (e - b) * q:
            t = b + (j * 3600 + q - 1) // q
            if t < horizon:
                due[t, s] += 1
            j += 1
    assert due.max(initial=0) < 256
    return due.astype(np.uint8)


def build_obs_program(net: NetTables, agent: str, coop_gamma: float, use_wait: bool):
    """Observation layout of reference envs/env.py:163-205 and dims of :303-323.

    per agent: [own wave | neighbour waves (x coop_gamma iff ma2c) | own wait | neighbour
    fingerprints (ma2c)]; greedy, maxpressure, fixedtime and actuated: own wave only."""
    names = net.node_names
    idx = {n: i for i, n in enumerate(names)}
    det_off = net.node_det_off
    kinds, idxs, scales, obs_off = [], [], [], [0]
    n_s_ls, n_w_ls, n_f_ls = [], [], []
    own_only = agent in ("greedy", "maxpressure", "fixedtime", "actuated")
    marl = agent != "a2c" and not own_only
    for i, name in enumerate(names):
        own = list(range(det_off[i], det_off[i + 1]))
        k0 = len(kinds)
        for d in own:
            kinds.append(0); idxs.append(d); scales.append(1.0)
        if marl:
            for nb in net.neighbor_map.get(name, []):
                j = idx[nb]
                sc = coop_gamma if agent == "ma2c" else 1.0
                for d in range(det_off[j], det_off[j + 1]):
                    kinds.append(0); idxs.append(d); scales.append(sc)
        n_w = 0
        if use_wait and not own_only:
            for d in own:
                kinds.append(1); idxs.append(d); scales.append(1.0)
            n_w = len(own)
        n_f = 0
        if agent == "ma2c":
            for nb in net.neighbor_map.get(name, []):
                j = idx[nb]
                for a in range(int(net.node_n_phases[j]) - 1):   # fingerprint = pi[:-1]
                    kinds.append(2); idxs.append(j * net.max_na + a); scales.append(1.0)
                    n_f += 1
        obs_off.append(len(kinds))
        # declared dims follow envs/env.py:303-323 literally: the wait block is counted whenever
        # 'wait' is a state name, even for the greedy agent whose state omits it (:171-172)
        n_w_decl = len(own) if use_wait else 0
        n_s_ls.append(len(kinds) - k0 + (n_w_decl - n_w))
        n_w_ls.append(n_w_decl)
        n_f_ls.append(n_f)
    net.obs_kind = np.array(kinds, dtype=np.int32)
    net.obs_idx = np.array(idxs, dtype=np.int32)
    net.obs_scale = np.array(scales, dtype=np.float32)
    net.node_obs_off = np.array(obs_off, dtype=np.int32)
    net.n_s_ls, net.n_w_ls, net.n_f_ls = n_s_ls, n_w_ls, n_f_ls
    net.n_a_ls = [int(x) for x in net.node_n_phases]
    return net
