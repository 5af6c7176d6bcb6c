"""6-intersection `small_grid` scenario (Ye et al. 2016 benchmark network): geometry, connections, signal programs,
detectors and the stochastic demand.

Everything is derived from constants of the reference generator `small_grid/data/build_file.py` (cited inline) and
`envs/small_grid_env.py`.  The generated `exp.net.xml` / `exp.rou.xml` are not in the reference repo (they need
netconvert / jtrrouter, build_file.py:316-335,436-447), so:

* lane lengths are the Euclidean node distances (zero-length junctions, DESIGN.md §3);
* TLS link order = incoming edges clockwise from north, links of an edge from right to left (SUMO's convention; it
  makes `STATE_PHASE_MAP` of envs/small_grid_env.py:29-31 consistent with alphabetical detector order);
* JTRRouter's per-vehicle route sampling is restated as a per-second draw over the enumerated routes of an origin
  (turn ratios of build_file.py:217-282, time-varying at `npc`; edges without a `<fromEdge>` entry use jtrrouter's
  --turn-defaults 30,50,20 restricted to the existing connections), and `probability=` flows (build_file.py:170-214)
  as one Bernoulli draw per second — `tsc_net.src_group / src_plo / src_phi` (include/tsc.h).
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import numpy as np

from .tables import NetTables, build_obs_program, flow_due_table, phase_masks

SPEED_LIMIT = 20.0                                    # build_file.py:19
L0, L1, L0_END = 200.0, 400.0, 75.0                   # build_file.py:20-21
INF = 1.0e9
# envs/small_grid_env.py:20-25
SMALL_GRID_NEIGHBOR_MAP = {'nt1': ['npc', 'nt2', 'nt6'], 'nt2': ['nt1', 'nt3'], 'nt3': ['npc', 'nt2', 'nt4'],
                           'nt4': ['nt3', 'nt5'], 'nt5': ['npc', 'nt4', 'nt6'], 'nt6': ['nt1', 'nt5']}
# envs/small_grid_env.py:34-38
TWO_PHASE = ['GGrr', 'rrGG']
THREE_PHASE = ['GGGrrrrrr', 'rrrGGGrrr', 'rrrrrrGGG']
# the fixed-time programs the reference generator writes (small_grid/data/build_file.py:output_tls, exp.tll.xml): 30-s
# greens, each followed by a 3-s yellow, offset 0; three greens at nt1, two at every other node
TLS_THREE_PHASE = [(30, 'GGGrrrrrr'), (3, 'yyyrrrrrr'), (30, 'rrrGGGrrr'), (3, 'rrryyyrrr'), (30, 'rrrrrrGGG'),
                   (3, 'rrrrrryyy')]
TLS_TWO_PHASE = [(30, 'GGrr'), (3, 'yyrr'), (30, 'rrGG'), (3, 'rryy')]


def node_xy() -> Dict[str, Tuple[float, float]]:
    """build_file.py:28-55."""
    l2, l2e = L0 / math.sqrt(2), L0_END / math.sqrt(2)
    return {'nt1': (0, 0), 'nt2': (L1, 0), 'nt3': (L1, L0), 'nt4': (L1, L1), 'nt5': (L0, L1), 'nt6': (0, L1),
            'np1': (0, -L0_END), 'np2': (-l2e, -l2e), 'np3': (-L0_END, 0), 'np4': (L0_END + L1, 0),
            'np5': (L1, -L0_END), 'np6': (L0_END + L1, L0), 'np8': (L0_END + L1, L1), 'np9': (L1, L0_END + L1),
            'np11': (L0, L0_END + L1), 'np12': (-L0_END, L1), 'np13': (0, L0_END + L1), 'npc': (l2, l2)}


def small_edges() -> List[Tuple[str, str]]:
    """build_file.py:71-105 (output_edges order)."""
    e = [('np%d' % i, 'nt1') for i in (1, 2, 3)] + [('np%d' % i, 'nt4') for i in (8, 9)]
    e += [('nt1', 'nt2'), ('nt1', 'npc'), ('nt1', 'nt6'), ('npc', 'nt3'), ('npc', 'nt5'), ('nt5', 'nt6'),
          ('nt4', 'nt3'), ('nt4', 'nt5'), ('nt3', 'nt2')]
    e += [('nt6', 'np12'), ('nt6', 'np13'), ('nt2', 'np4'), ('nt2', 'np5'), ('nt5', 'np11'), ('nt3', 'np6')]
    return e


def small_connections() -> List[Tuple[str, str, str]]:
    """(from node, via node, to node): build_file.py:114-157."""
    c = []
    for i in (1, 2, 3):
        c += [('np%d' % i, 'nt1', 'nt2'), ('np%d' % i, 'nt1', 'nt6'), ('np%d' % i, 'nt1', 'npc')]
    for i in (8, 9):
        c += [('np%d' % i, 'nt4', 'nt3'), ('np%d' % i, 'nt4', 'nt5')]
    c += [('nt1', 'npc', 'nt3'), ('nt1', 'npc', 'nt5')]
    for i in (1, 3):
        c += [('nt%d' % i, 'nt2', 'np4'), ('nt%d' % i, 'nt2', 'np5')]
    for i in (1, 5):
        c += [('nt%d' % i, 'nt6', 'np12'), ('nt%d' % i, 'nt6', 'np13')]
    for f in ('npc', 'nt4'):
        c += [(f, 'nt3', 'np6'), (f, 'nt3', 'nt2')]
    for f in ('npc', 'nt4'):
        c += [(f, 'nt5', 'np11'), (f, 'nt5', 'nt6')]
    return c


def _heading(a, b, xy):
    return math.atan2(xy[b][1] - xy[a][1], xy[b][0] - xy[a][0])


def _turn_angle(f, v, t, xy):
    """signed turn at `v` when coming from f and leaving to t: > 0 left, < 0 right (radians)."""
    d = _heading(v, t, xy) - _heading(f, v, xy)
    while d <= -math.pi:
        d += 2 * math.pi
    while d > math.pi:
        d -= 2 * math.pi
    return d


# turn ratios, build_file.py:217-262
TURNS = {('np1', 'nt1'): {'nt2': 0.2, 'nt6': 0.5, 'npc': 0.3}, ('np2', 'nt1'): {'nt2': 0.15, 'nt6': 0.15, 'npc': 0.7},
         ('np3', 'nt1'): {'nt2': 0.5, 'nt6': 0.15, 'npc': 0.35}, ('np8', 'nt4'): {'nt3': 0.4, 'nt5': 0.6},
         ('np9', 'nt4'): {'nt3': 0.6, 'nt5': 0.4}, ('nt3', 'nt2'): {'np5': 1.0}, ('nt1', 'nt2'): {'np4': 1.0},
         ('nt5', 'nt6'): {'np12': 1.0}, ('nt1', 'nt6'): {'np13': 1.0}, ('npc', 'nt3'): {'nt2': 0.3, 'np6': 0.7},
         ('npc', 'nt5'): {'nt6': 0.3, 'np11': 0.7}}
# 10-minute source volumes (veh/h) of x1, x2, x3, x8, x9: build_file.py:190-194
FLOWS = [[500, 100, 700, 800, 550, 550, 100, 200, 250, 250, 400, 800],
         [600, 700, 100, 200, 50, 100, 1000, 500, 450, 150, 400, 200],
         [100, 400, 400, 200, 600, 550, 100, 500, 500, 800, 400, 200],
         [100, 200, 300, 300, 300, 400, 600, 600, 800, 500, 400, 300],
         [600, 400, 400, 600, 800, 400, 300, 300, 300, 200, 250, 250]]
# extra `probability=` flows: build_file.py:173-183
MF_ROUTES = ['nt1_npc npc_nt5 nt5_np11', 'nt1_npc npc_nt5 nt5_nt6 nt6_np12', 'nt4_nt5 nt5_np11',
             'nt4_nt5 nt5_nt6 nt6_np12', 'nt1_nt2 nt2_np4', 'nt1_nt6 nt6_np13', 'nt1_npc npc_nt3 nt3_np6',
             'nt1_npc npc_nt3 nt3_nt2 nt2_np5', 'nt4_nt3 nt3_np6', 'nt4_nt3 nt3_nt2 nt2_np5']
MF_CASES = [(3, 4, 5), (0, 3, 4), (1, 2, 5), (4, 5, 9), (5, 6, 9), (4, 7, 8)]


def build_small_grid(num_car_hourly: int = 1000, agent: str = "greedy", coop_gamma: float = 0.75,
                     use_wait: bool = True, episode_length_sec: int = 3600, veh_len: float = 5.0,
                     min_gap: float = 2.5) -> NetTables:
    xy = node_xy()
    edges = small_edges()
    edge_id = {e: k for k, e in enumerate(edges)}
    lane_names = ['%s_%s_0' % e for e in edges]
    lane_len = [math.hypot(xy[b][0] - xy[a][0], xy[b][1] - xy[a][1]) for a, b in edges]
    lane_vmax = [SPEED_LIMIT] * len(edges)
    n_lanes = len(edges)
    lane_cap = np.array([int(np.ceil(L / (veh_len + min_gap))) + 1 for L in lane_len], np.int32)
    lane_slot0 = np.concatenate([[0], np.cumsum(lane_cap)[:-1]]).astype(np.int32)

    node_names = sorted('nt%d' % i for i in range(1, 7))        # envs/env.py:232
    node_idx = {n: i for i, n in enumerate(node_names)}
    cons = small_connections()
    # ---- links in TLS order: incoming edges clockwise from north, links of an edge right -> left -------------
    link_from, link_to, link_node, link_tlidx, link_vmax = [], [], [], [], []
    lanes_in: Dict[str, List[str]] = {}
    link_of = {}
    for via in node_names + ['npc']:
        inc = sorted({f for f, v, t in cons if v == via},
                     key=lambda f: (math.pi / 2 - _heading(via, f, xy)) % (2 * math.pi))     # clockwise from north
        ctl, tl = [], 0
        for f in inc:
            outs = sorted((t for ff, v, t in cons if v == via and ff == f), key=lambda t: _turn_angle(f, via, t, xy))
            for t in outs:
                ang = math.degrees(_turn_angle(f, via, t, xy))
                if abs(ang) < 30:
                    vm = INF
                elif ang < 0:
                    vm = 5.2 if ang <= -60 else 8.0          # right turns (large_grid.py TURN_VMAX for 90 deg)
                else:
                    vm = 8.1 if ang >= 60 else 10.0
                lid = len(link_from)
                link_from.append(edge_id[(f, via)]); link_to.append(edge_id[(via, t)])
                link_node.append(node_idx.get(via, -1)); link_tlidx.append(tl if via in node_idx else 0)
                link_vmax.append(vm)
                link_of[(f, via, t)] = lid
                ctl.append(lane_names[edge_id[(f, via)]])
                tl += 1
        if via in node_idx:
            lanes_in[via] = ctl
    n_links = len(link_from)
    # every phase serves exactly one incoming lane ('G' only): no crossing or merging foes
    link_cross = np.zeros(n_links, np.uint32)
    link_merge = np.zeros(n_links, np.uint32)
    inl = [[l for l in range(n_links) if link_to[l] == ln] for ln in range(n_lanes)]
    lane_inl_off = np.concatenate([[0], np.cumsum([len(x) for x in inl])]).astype(np.int32)
    lane_inl = np.array([l for x in inl for l in x], np.int32)

    # ---- detectors (E2 over the last 50 m of the 14 non-sink lanes, build_file.py:356-385; ilds = lanes_in order) --
    ilds_in, det_lane, node_det_off = {}, [], [0]
    lane_idx = {n: k for k, n in enumerate(lane_names)}
    for name in node_names:
        seen = []
        for ln in lanes_in[name]:
            if ln not in seen:
                seen.append(ln)
        ilds_in[name] = seen
        det_lane += [lane_idx[s] for s in seen]
        node_det_off.append(len(det_lane))
    # neighbours: `npc` is not an agent (the reference raises KeyError for MARL agents here; we drop it)
    neighbor_map = {k: [n for n in v if n in node_idx] for k, v in SMALL_GRID_NEIGHBOR_MAP.items()}
    node_nbr, node_nbr_off = [], [0]
    for name in node_names:
        node_nbr += [node_idx[n] for n in neighbor_map[name]]
        node_nbr_off.append(len(node_nbr))

    # ---- signal programs (envs/small_grid_env.py:34-38,62-65) --------------------------------------------------
    phases = {n: (THREE_PHASE if n == 'nt1' else TWO_PHASE) for n in node_names}
    max_phases = 3
    node_green = np.zeros((len(node_names), max_phases), np.uint32)
    node_major = np.zeros((len(node_names), max_phases), np.uint32)
    for i, n in enumerate(node_names):
        g, m = phase_masks(phases[n])
        node_green[i, :len(g)] = g; node_major[i, :len(m)] = m
        assert len(phases[n][0]) == len(lanes_in[n])
    node_n_phases = np.array([len(phases[n]) for n in node_names], np.int32)

    # ---- routes: enumerate every path an origin can take, with its probability per 10-minute interval ----------
    n_pint, pint_sec = max(1, episode_length_sec // 600), 600
    fl = np.array(FLOWS, np.float64)
    base = np.array([[0.15, 0.15], [0.35, 0.35], [0.15, 0.2]])              # build_file.py:270-281
    npc_prob = []
    for i in range(12):
        p = fl[:3, i] @ base
        npc_prob.append(p / p.sum())
    out_of: Dict[str, List[str]] = {}
    for f, v, t in cons:
        out_of.setdefault((f, v), []).append(t)

    def turn_probs(f, v, iv):
        if (f, v) == ('nt1', 'npc'):
            return {'nt3': float(npc_prob[iv][0]), 'nt5': float(npc_prob[iv][1])}
        if (f, v) in TURNS:
            return TURNS[(f, v)]
        # jtrrouter --turn-defaults 30,50,20 (right, straight, left) restricted to the existing connections
        w = {}
        for t in out_of[(f, v)]:
            ang = math.degrees(_turn_angle(f, v, t, xy))
            w[t] = 50.0 if abs(ang) < 30 else (30.0 if ang < 0 else 20.0)
        s = sum(w.values())
        return {t: x / s for t, x in w.items()}

    def paths_from(f, v):
        """all node paths continuing from edge (f, v) to a sink edge."""
        if (f, v) not in out_of:
            return [[f, v]]
        res = []
        for t in out_of[(f, v)]:
            for tail in paths_from(v, t):
                res.append([f] + tail)
        return res

    def path_prob(path, iv):
        p = 1.0
        for k in range(len(path) - 2):
            p *= turn_probs(path[k], path[k + 1], iv).get(path[k + 2], 0.0)
        return p

    routes_lane, routes_link, route_names = [], [], []

    def add_route(nodes):
        es = [edge_id[(nodes[k], nodes[k + 1])] for k in range(len(nodes) - 1)]
        links = [link_of[(nodes[k], nodes[k + 1], nodes[k + 2])] for k in range(len(nodes) - 2)] + [-1]
        routes_lane.append(es); routes_link.append(links)
        route_names.append(' '.join('%s_%s' % (nodes[k], nodes[k + 1]) for k in range(len(nodes) - 1)))
        return len(routes_lane) - 1

    origins = [('np1', 'nt1'), ('np2', 'nt1'), ('np3', 'nt1'), ('np8', 'nt4'), ('np9', 'nt4')]   # build_file.py:195-196
    src_lane, src_route, src_group, flow_list = [], [], [], []
    plo, phi = [], []                                   # per source: [n_pint] bounds
    for j, (f, v) in enumerate(origins):
        paths = [pth for pth in paths_from(f, v) if max(path_prob(pth, iv) for iv in range(n_pint)) > 0.0]
        cum = np.zeros(n_pint)
        for k, path in enumerate(paths):
            q = len(src_lane)
            src_lane.append(edge_id[(f, v)]); src_route.append(add_route(path)); src_group.append(j)
            pr = np.array([path_prob(path, iv) for iv in range(n_pint)])
            lo = cum.copy(); cum = cum + pr
            hi = cum.copy() if k + 1 < len(paths) else np.ones(n_pint)
            plo.append(lo); phi.append(hi)
            for i0 in range(n_pint):                                   # build_file.py:208-212: 10-minute volumes
                flow_list.append((q, i0 * 600, (i0 + 1) * 600, int(FLOWS[j][i0])))
    # `probability=` flows: one Bernoulli(p) draw per second while active, build_file.py:170-207
    p_mf = float('%.2f' % (num_car_hourly / 3600.0))
    for c, rt in enumerate(MF_ROUTES):
        es = rt.split(' ')
        nodes = [es[0].split('_')[0]] + [e.split('_')[1] for e in es]
        q = len(src_lane)
        src_lane.append(edge_id[(nodes[0], nodes[1])]); src_route.append(add_route(nodes)); src_group.append(len(origins) + c)
        plo.append(np.zeros(n_pint)); phi.append(np.full(n_pint, p_mf))
        for i, case in enumerate(MF_CASES):
            if c in case and i * 1200 < episode_length_sec:
                flow_list.append((q, i * 1200, min((i + 1) * 1200, episode_length_sec), 3600))   # due every second
    n_src = len(src_lane)
    src_due = flow_due_table(flow_list, episode_length_sec, n_src)
    max_hops = max(len(r) for r in routes_lane)
    route_lane = np.full((len(routes_lane), max_hops), -1, np.int16)
    route_link = np.full((len(routes_lane), max_hops), -1, np.int16)
    for r, (ls, ks) in enumerate(zip(routes_lane, routes_link)):
        route_lane[r, :len(ls)] = ls
        route_link[r, :len(ks)] = ks

    net = NetTables(
        node_names=node_names, lane_names=lane_names, neighbor_map=neighbor_map, phases=phases, lanes_in=lanes_in,
        ilds_in=ilds_in, max_hops=max_hops, horizon=episode_length_sec, max_phases=max_phases, max_na=max_phases,
        lane_len=np.array(lane_len, np.float32), lane_vmax=np.array(lane_vmax, np.float32), lane_cap=lane_cap,
        lane_slot0=lane_slot0, lane_inl_off=lane_inl_off, lane_inl=lane_inl,
        link_from=np.array(link_from, np.int32), link_to=np.array(link_to, np.int32),
        link_node=np.array(link_node, np.int32), link_tlidx=np.array(link_tlidx, np.int32),
        link_vmax=np.array(link_vmax, np.float32), link_cross=link_cross, link_merge=link_merge,
        route_len=np.array([len(r) for r in routes_lane], np.int32), route_lane=route_lane, route_link=route_link,
        node_n_phases=node_n_phases, node_green=node_green, node_major=node_major,
        node_det_off=np.array(node_det_off, np.int32), det_lane=np.array(det_lane, np.int32),
        node_nbr_off=np.array(node_nbr_off, np.int32), node_nbr=np.array(node_nbr, np.int32),
        src_lane=np.array(src_lane, np.int32), src_route=np.array(src_route, np.int32), src_due=src_due,
        src_group=np.array(src_group, np.int32), src_plo=np.stack(plo, 1).astype(np.float32),
        src_phi=np.stack(phi, 1).astype(np.float32), pint_sec=pint_sec, route_names=route_names,
    )
    net.flow_list, net.edges = flow_list, edges
    build_obs_program(net, agent, coop_gamma, use_wait)
    return net.finalize()


def tls_programs():
    """{tlLogic id: program} of the small grid (TLS_THREE_PHASE at nt1, TLS_TWO_PHASE at nt2..nt6), in the form of
    net.sumo_ingest.read_signal_programs."""
    return {'nt%d' % i: {'type': 'static', 'offset': 0,
                         'phases': [[d, st] for d, st in (TLS_THREE_PHASE if i == 1 else TLS_TWO_PHASE)]}
            for i in range(1, 7)}
