"""5x5 `large_grid` scenario: geometry, connections, signal programs, detectors, demand.

Everything is derived from constants of the reference generator
`large_grid/data/build_file.py` (cited inline) and `envs/large_grid_env.py`; the generated
`exp.net.xml` is not in the reference repo (needs netconvert, build_file.py:436), so lane
lengths are the node pitch (junction interiors have zero length in our model, DESIGN.md §3).
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from .tables import NetTables, build_obs_program, flow_due_table, phase_masks

# large_grid/data/build_file.py:14-19
SPEED_LIMIT_ST = 20.0
SPEED_LIMIT_AV = 11.0
L0 = 200.0
L0_END = 75.0
N = 5
# envs/large_grid_env.py:40-41
PHASES = ['GGgrrrGGgrrr', 'rrrGrGrrrGrG', 'rrrGGrrrrGGr', 'rrrGGGrrrrrr', 'rrrrrrrrrGGG']
# the fixed-time program the reference generator writes for every node (large_grid/data/build_file.py:output_tls,
# exp.tll.xml): three greens of 30 s, each followed by a 3-s yellow, offset 0 (envs.fixedtime runs it)
TLS_PROGRAM = [(30, 'GGgrrrGGgrrr'), (3, 'yyyrrryyyrrr'), (30, 'rrrGrGrrrGrG'), (3, 'rrrGryrrrGry'),
               (30, 'rrrGGrrrrGGr'), (3, 'rrryyrrrryyr')]
# turning-speed limits of the junction-internal lanes (netconvert computes them from the
# turning radius with --junctions.limit-turn-speed 5.5: v = sqrt(5.5 r); r ~ 5 m / 12 m)
TURN_VMAX = {"r": 5.2, "s": 1.0e9, "l": 8.1}
INF = 1.0e9


def _nt(i: int) -> str:
    return "nt%d" % i


def _np(i: int) -> str:
    return "np%d" % i


def grid_edges() -> List[Tuple[str, str, str]]:
    """(from, to, type) in the order of build_file.py:66-98 (output_edges)."""
    edges = []
    for in_i, out_i in zip([5, 10, 15, 20, 25, 21, 16, 11, 6, 1],
                           [6, 7, 8, 9, 10, 16, 17, 18, 19, 20]):          # :69-75
        edges.append((_nt(in_i), _np(out_i), "a"))
        edges.append((_np(out_i), _nt(in_i), "a"))
    for in_i, out_i in zip([1, 2, 3, 4, 5, 25, 24, 23, 22, 21],
                           [1, 2, 3, 4, 5, 11, 12, 13, 14, 15]):          # :77-83
        edges.append((_nt(in_i), _np(out_i), "b"))
        edges.append((_np(out_i), _nt(in_i), "b"))
    for i in range(1, 25, 5):                                              # :85-90 streets
        for j in range(4):
            edges.append((_nt(i + j), _nt(i + j + 1), "a"))
            edges.append((_nt(i + j + 1), _nt(i + j), "a"))
    for i in range(1, 6):                                                  # :91-96 avenues
        for j in range(0, 20, 5):
            edges.append((_nt(i + j), _nt(i + j + 5), "b"))
            edges.append((_nt(i + j + 5), _nt(i + j), "b"))
    return edges


def node_neighbours_nswe(i: int) -> Dict[str, str]:
    """n/s/w/e neighbour node names of nt<i> (boundary -> np*), build_file.py:127-184."""
    col, row = (i - 1) % N, (i - 1) // N
    out = {}
    out["n"] = _nt(i + N) if row < N - 1 else _np(15 - col)     # np11..np15 run x = 800..0  (:42-44)
    out["s"] = _nt(i - N) if row > 0 else _np(1 + col)          # np1..np5  run x = 0..800   (:36-38)
    out["e"] = _nt(i + 1) if col < N - 1 else _np(6 + row)      # np6..np10 run y = 0..800   (:39-41)
    out["w"] = _nt(i - 1) if col > 0 else _np(20 - row)         # np16..np20 run y = 800..0  (:45-47)
    return out


def large_neighbor_map() -> Dict[str, List[str]]:
    """envs/large_grid_env.py:73-101 restated as a rule: interior nodes list [n, e, s, w];
    border nodes keep the hand-written orders of the reference."""
    m = {
        'nt1': ['nt6', 'nt2'], 'nt5': ['nt10', 'nt4'], 'nt21': ['nt22', 'nt16'],
        'nt25': ['nt20', 'nt24'],
        'nt2': ['nt7', 'nt3', 'nt1'], 'nt3': ['nt8', 'nt4', 'nt2'], 'nt4': ['nt9', 'nt5', 'nt3'],
        'nt22': ['nt23', 'nt17', 'nt21'], 'nt23': ['nt24', 'nt18', 'nt22'],
        'nt24': ['nt25', 'nt19', 'nt23'],
        'nt10': ['nt15', 'nt5', 'nt9'], 'nt15': ['nt20', 'nt10', 'nt14'],
        'nt20': ['nt25', 'nt15', 'nt19'],
        'nt6': ['nt11', 'nt7', 'nt1'], 'nt11': ['nt16', 'nt12', 'nt6'],
        'nt16': ['nt21', 'nt17', 'nt11'],
    }
    for i in [7, 8, 9, 12, 13, 14, 17, 18, 19]:
        m[_nt(i)] = [_nt(i + 5), _nt(i + 1), _nt(i - 5), _nt(i - 1)]
    return m


def _od_pairs():
    """12 OD edge pairs of build_file.py:282-295 (srcs/sinks zipped per group)."""
    edge_maps = [0, 1, 2, 3, 4, 5, 5, 10, 15, 20, 25, 25, 24, 23, 22, 21, 21, 16, 11, 6, 1]  # :199-200

    def ext(out_edges, dest):
        res = []
        for o in out_edges:
            a, b = _nt(edge_maps[o]), _np(o)
            res.append((a, b) if dest else (b, a))
        return res
    srcs = [ext([12, 13, 14], False), ext([16, 18, 20], False),
            ext([2, 3, 4], False), ext([6, 8, 10], False)]
    sinks = [ext([2, 3, 4], True), ext([6, 8, 10], True),
             ext([14, 13, 12], True), ext([20, 18, 16], True)]
    return [list(zip(s, d)) for s, d in zip(srcs, sinks)]


def _route_nodes(src_edge, dst_edge, turn: str) -> List[str]:
    """Node sequence of the (unique up to ties) fastest route.  All Manhattan paths between
    an OD pair have equal free-flow time (same street/avenue lengths); SUMO's tie-break is
    internal, ours is explicit: 'early' turns at the first junction, 'late' at the last."""
    def pos(nt):  # nt name -> (col,row)
        i = int(nt[2:])
        return (i - 1) % N, (i - 1) // N

    def name(c, r):
        return _nt(r * N + c + 1)
    (o_np, o_nt), (d_nt, d_np) = src_edge, dst_edge
    c0, r0 = pos(o_nt)
    c1, r1 = pos(d_nt)
    seq = [o_np, o_nt]
    # heading of the entry stub: vertical if it enters from top/bottom row boundary
    nb = node_neighbours_nswe(int(o_nt[2:]))
    vertical = o_np in (nb["n"], nb["s"])
    c, r = c0, r0

    def walk_c(target):
        nonlocal c
        while c != target:
            c += 1 if target > c else -1
            seq.append(name(c, r))

    def walk_r(target):
        nonlocal r
        while r != target:
            r += 1 if target > r else -1
            seq.append(name(c, r))
    if vertical:
        if c0 == c1:
            walk_r(r1)
        elif turn == "early":
            walk_c(c1); walk_r(r1)
        else:
            # go down to the exit row first, then across, then exit
            walk_r(r1); walk_c(c1)
    else:
        if r0 == r1:
            walk_c(c1)
        elif turn == "early":
            walk_r(r1); walk_c(c1)
        else:
            walk_c(c1); walk_r(r1)
    seq.append(d_np)
    return seq


MAX_CAR_NUM = 30            # large_grid/data/build_file.py:19


def init_fleet_specs(density: float, seed):
    """The initial fleet of `init_routes` (large_grid/data/build_file.py:223-266): on every lane of every internal edge
    `int(MAX_CAR_NUM * density)` vehicles at t = 0, each group bound for one boundary sink edge drawn with
    `np.random.choice` from numpy's GLOBAL generator right after `np.random.seed(seed)` (build_file.py:275-282) — the
    legacy `RandomState(seed).choice` reproduces those draws.  Returns [(from node, to node, lane, sink edge (nt, np), n)]."""
    in_nodes = [5, 10, 15, 20, 25, 21, 16, 11, 6, 1, 1, 2, 3, 4, 5, 25, 24, 23, 22, 21]
    out_nodes = [6, 7, 8, 9, 10, 16, 17, 18, 19, 20, 1, 2, 3, 4, 5, 11, 12, 13, 14, 15]
    sinks = [(_nt(i), _np(j)) for i, j in zip(in_nodes, out_nodes)]
    rs = np.random.RandomState(seed)
    n = int(MAX_CAR_NUM * density)
    out = []

    def get(a, b, lane):
        out.append((a, b, lane, sinks[int(rs.choice(len(sinks)))], n))
    for i in range(1, 25, 5):                                   # streets: both directions, both lanes
        for j in range(4):
            a, b = _nt(i + j), _nt(i + j + 1)
            get(a, b, 0); get(b, a, 0); get(a, b, 1); get(b, a, 1)
    for i in range(1, 6):                                       # avenues
        for j in range(0, 20, 5):
            a, b = _nt(i + j), _nt(i + j + 5)
            get(a, b, 0); get(b, a, 0)
    return out


def build_large_grid(peak_flow1: int = 1100, peak_flow2: int = 925, agent: str = "ma2c",
                     coop_gamma: float = 0.9, use_wait: bool = True,
                     episode_length_sec: int = 3600, veh_len: float = 5.0,
                     min_gap: float = 2.5, route_turn: str = "early",
                     init_density: float = 0.0, seed=None) -> NetTables:
    edges = grid_edges()
    edge_id = {(a, b): k for k, (a, b, _) in enumerate(edges)}
    # ---- lanes -------------------------------------------------------------------------
    lane_names, lane_len, lane_vmax, lane_edge = [], [], [], []
    edge_lane0 = []
    for k, (a, b, typ) in enumerate(edges):
        nl = 2 if typ == "a" else 1                          # build_file.py:55-56
        length = L0 if (a.startswith("nt") and b.startswith("nt")) else L0_END
        edge_lane0.append(len(lane_names))
        for li in range(nl):
            lane_names.append("%s_%s_%d" % (a, b, li))
            lane_len.append(length)
            lane_vmax.append(SPEED_LIMIT_ST if typ == "a" else SPEED_LIMIT_AV)
            lane_edge.append(k)
    n_lanes = len(lane_names)
    lane_cap = np.array([int(np.ceil(L / (veh_len + min_gap))) + 1 for L in lane_len], np.int32)
    lane_slot0 = np.concatenate([[0], np.cumsum(lane_cap)[:-1]]).astype(np.int32)

    def lane_of(a, b, li):
        return edge_lane0[edge_id[(a, b)]] + li

    # ---- nodes in sorted-name order (envs/env.py:232) ------------------------------------
    node_names = sorted(_nt(i) for i in range(1, N * N + 1))
    node_idx = {n: i for i, n in enumerate(node_names)}
    neighbor_map = large_neighbor_map()

    # ---- links: 12 per junction, clockwise from the north approach, right/straight/left --
    link_from, link_to, link_node, link_tlidx, link_vmax = [], [], [], [], []
    link_to_edge, link_turn = [], []
    lanes_in: Dict[str, List[str]] = {}
    link_of = {}   # (from_lane, to_edge) -> link id
    for i in range(1, N * N + 1):
        cur = _nt(i)
        nb = node_neighbours_nswe(i)
        # (approach neighbour, [(turn, target neighbour, fromLane, toLane)])  build_file.py:107-124
        plan = [
            ("n", [("r", "w", 0, 0), ("s", "s", 0, 0), ("l", "e", 0, 1)]),
            ("e", [("r", "n", 0, 0), ("s", "w", 0, 0), ("l", "s", 1, 0)]),
            ("s", [("r", "e", 0, 0), ("s", "n", 0, 0), ("l", "w", 0, 1)]),
            ("w", [("r", "s", 0, 0), ("s", "e", 0, 0), ("l", "n", 1, 0)]),
        ]
        ctl = []
        tl = 0
        for appr, moves in plan:
            for turn, tgt, fl, tl_lane in moves:
                f = lane_of(nb[appr], cur, fl)
                t = lane_of(cur, nb[tgt], tl_lane)
                lid = len(link_from)
                link_from.append(f); link_to.append(t)
                link_node.append(node_idx[cur]); link_tlidx.append(tl)
                link_vmax.append(TURN_VMAX[turn])
                link_to_edge.append(edge_id[(cur, nb[tgt])]); link_turn.append(turn)
                link_of[(f, edge_id[(cur, nb[tgt])])] = lid
                ctl.append(lane_names[f])
                tl += 1
        lanes_in[cur] = ctl
    n_links = len(link_from)
    # foes: cross = opposing straight for a left turn; merge = higher-priority links into the
    # same outgoing edge (straight > right > left)
    prio = {"s": 0, "r": 1, "l": 2}
    link_cross = np.zeros(n_links, np.uint32)
    link_merge = np.zeros(n_links, np.uint32)
    by_node: Dict[int, List[int]] = {}
    for l in range(n_links):
        by_node.setdefault(link_node[l], []).append(l)
    for node, ls in by_node.items():
        for l in ls:
            if link_turn[l] == "l":
                opp = (link_tlidx[l] // 3 + 2) % 4          # opposite approach
                link_cross[l] |= np.uint32(1 << (opp * 3 + 1))
            for m in ls:
                if m != l and link_to_edge[m] == link_to_edge[l] and prio[link_turn[m]] < prio[link_turn[l]]:
                    link_merge[l] |= np.uint32(1 << link_tlidx[m])
    # links entering each lane (all links into the lane's edge), in merge-priority order
    inl = [[] for _ in range(n_lanes)]
    for l in range(n_links):
        for ln in range(n_lanes):
            if lane_edge[ln] == link_to_edge[l]:
                inl[ln].append(l)
    for ln in range(n_lanes):
        inl[ln].sort(key=lambda l: (prio[link_turn[l]], l))
    lane_inl_off = np.concatenate([[0], np.cumsum([len(x) for x in inl])]).astype(np.int32)
    lane_inl = np.array([l for x in inl for l in x], np.int32)

    # ---- detectors: ilds_in = de-duplicated controlled lanes (envs/env.py:225-230) --------
    ilds_in = {}
    det_lane, node_det_off = [], [0]
    lane_idx = {n: k for k, n in enumerate(lane_names)}
    for name in node_names:
        seen = []
        for ln in lanes_in[name]:
            if ln not in seen:
                seen.append(ln)
        ilds_in[name] = seen
        det_lane += [lane_idx[s] for s in seen]
        node_det_off.append(len(det_lane))
    # neighbours
    node_nbr, node_nbr_off = [], [0]
    for name in node_names:
        node_nbr += [node_idx[n] for n in neighbor_map[name]]
        node_nbr_off.append(len(node_nbr))

    # ---- signal programs ------------------------------------------------------------------
    g, m = phase_masks(PHASES)
    n_nodes = len(node_names)
    node_green = np.tile(np.array(g, np.uint32), (n_nodes, 1))
    node_major = np.tile(np.array(m, np.uint32), (n_nodes, 1))
    node_n_phases = np.full(n_nodes, len(PHASES), np.int32)

    # ---- routes (lane choice at edge entry: lane 1 iff the vehicle turns left at its end) --
    ods = _od_pairs()
    routes_lane, routes_link, route_names = [], [], []
    src_lane, src_route = [], []
    group_src = []      # per group, list of src indices
    for gi, group in enumerate(ods):
        gs = []
        for (se, de) in group:
            seq = _route_nodes(se, de, route_turn)
            hops_e = [edge_id[(seq[k], seq[k + 1])] for k in range(len(seq) - 1)]
            lanes_r, links_r = [], []
            for h, e in enumerate(hops_e):
                if h + 1 < len(hops_e):
                    # find turn type at the end of edge e towards hops_e[h+1]
                    cand = [l for l in range(n_links)
                            if lane_edge[link_from[l]] == e and link_to_edge[l] == hops_e[h + 1]]
                    assert len(cand) == 1, (seq, h)
                    l = cand[0]
                    lanes_r.append(link_from[l])
                    links_r.append(l)
                else:
                    lanes_r.append(edge_lane0[e])
                    links_r.append(-1)
            rid = len(routes_lane)
            routes_lane.append(lanes_r); routes_link.append(links_r)
            route_names.append("%s_%s->%s_%s" % (se[0], se[1], de[0], de[1]))
            gs.append(len(src_lane))
            src_lane.append(lanes_r[0]); src_route.append(rid)
        group_src.append(gs)
    # ---- initial fleet (init_density > 0): fastest route from an internal edge to a drawn boundary sink -------------
    init_flows = []
    if init_density > 0 and int(MAX_CAR_NUM * init_density) > 0:
        import heapq
        n_edges = len(edges)
        cost = [(L0 if (a.startswith("nt") and b.startswith("nt")) else L0_END) /
                (SPEED_LIMIT_ST if typ == "a" else SPEED_LIMIT_AV) for a, b, typ in edges]
        succ = {}
        for l in range(n_links):
            succ.setdefault(lane_edge[link_from[l]], set()).add(link_to_edge[l])

        def fastest(e0, e1):                                    # Dijkstra over edges, ties -> lower edge id
            dist, prev, pq = {e0: 0.0}, {}, [(0.0, e0)]
            while pq:
                dcur, u = heapq.heappop(pq)
                if u == e1:
                    break
                if dcur > dist[u]:
                    continue
                for v in sorted(succ.get(u, ())):
                    nd = dcur + cost[v]
                    if nd < dist.get(v, 1e30) - 1e-9:
                        dist[v], prev[v] = nd, u
                        heapq.heappush(pq, (nd, v))
            path = [e1]
            while path[-1] != e0:
                path.append(prev[path[-1]])
            return path[::-1]
        for (a, b, lane, sink, n_veh) in init_fleet_specs(init_density, seed):
            hops_e = fastest(edge_id[(a, b)], edge_id[sink])
            lanes_r, links_r = [], []
            for h, e in enumerate(hops_e):
                if h + 1 < len(hops_e):
                    cand = [l for l in range(n_links)
                            if lane_edge[link_from[l]] == e and link_to_edge[l] == hops_e[h + 1]]
                    assert len(cand) == 1
                    lanes_r.append(link_from[cand[0]]); links_r.append(cand[0])
                else:
                    lanes_r.append(edge_lane0[e]); links_r.append(-1)
            # lanes are FIFO here (no mid-edge lane change, DESIGN.md section 3): the group starts on the lane its first
            # movement needs, which is `departLane` whenever that lane connects to the route
            rid = len(routes_lane)
            routes_lane.append(lanes_r); routes_link.append(links_r)
            route_names.append("init %s_%s_%d->%s_%s" % (a, b, lane, sink[0], sink[1]))
            init_flows.append((len(src_lane), n_veh))
            src_lane.append(lanes_r[0]); src_route.append(rid)
    max_hops = max(len(r) for r in routes_lane)
    route_lane = np.full((len(routes_lane), max_hops), -1, np.int16)
    route_link = np.full((len(routes_lane), max_hops), -1, np.int16)
    for r, (ls, ks) in enumerate(zip(routes_lane, routes_link)):
        route_lane[r, :len(ls)] = ls
        route_link[r, :len(ks)] = ks
    route_len = np.array([len(r) for r in routes_lane], np.int32)

    # ---- demand: build_file.py:297-324 ---------------------------------------------------
    ratios1 = np.array([0.4, 0.7, 0.9, 1.0, 0.75, 0.5, 0.25])
    ratios2 = np.array([0.3, 0.8, 0.9, 1.0, 0.8, 0.6, 0.2])
    flows = [peak_flow1 * 0.6 * ratios1, peak_flow1 * ratios1,
             peak_flow2 * 0.6 * ratios2, peak_flow2 * ratios2]
    times = np.arange(0, 3001, 300)
    id1 = len(flows[0])
    id2 = len(times) - 1 - id1
    flow_list = []
    for i in range(len(times) - 1):
        tb, te = int(times[i]), int(times[i + 1])
        if i < id1:
            for j in (0, 1):
                for s in group_src[j]:
                    flow_list.append((s, tb, te, int(flows[j][i])))      # '%d' truncation, :277
        if i >= id2:
            for j in (2, 3):
                for s in group_src[j]:
                    flow_list.append((s, tb, te, int(flows[j][i - id2])))
    src_due = flow_due_table(flow_list, episode_length_sec, len(src_lane))
    for q, n_veh in init_flows:         # `begin="0" end="1" number=n`: all due in the first second (inserted one per lane
        src_due[0, q] = n_veh           # and second on the free tail segment, like every other vehicle)

    net = NetTables(
        node_names=node_names, lane_names=lane_names, neighbor_map=neighbor_map,
        phases={n: PHASES for n in node_names}, lanes_in=lanes_in, ilds_in=ilds_in,
        max_hops=max_hops, horizon=episode_length_sec, max_phases=len(PHASES), max_na=len(PHASES),
        lane_len=np.array(lane_len, np.float32), lane_vmax=np.array(lane_vmax, np.float32),
        lane_cap=lane_cap, lane_slot0=lane_slot0, lane_inl_off=lane_inl_off, lane_inl=lane_inl,
        link_from=np.array(link_from, np.int32), link_to=np.array(link_to, np.int32),
        link_node=np.array(link_node, np.int32), link_tlidx=np.array(link_tlidx, np.int32),
        link_vmax=np.array(link_vmax, np.float32), link_cross=link_cross, link_merge=link_merge,
        route_len=route_len, route_lane=route_lane, route_link=route_link,
        node_n_phases=node_n_phases, node_green=node_green, node_major=node_major,
        node_det_off=np.array(node_det_off, np.int32), det_lane=np.array(det_lane, np.int32),
        node_nbr_off=np.array(node_nbr_off, np.int32), node_nbr=np.array(node_nbr, np.int32),
        src_lane=np.array(src_lane, np.int32), src_route=np.array(src_route, np.int32),
        src_due=src_due, route_names=route_names,
    )
    net.flow_list = flow_list
    net.edges = edges
    build_obs_program(net, agent, coop_gamma, use_wait)
    return net.finalize()


def tls_programs():
    """{tlLogic id: program} of the grid (TLS_PROGRAM on nodes nt1..nt25), in the form of
    net.sumo_ingest.read_signal_programs."""
    return {_nt(i): {'type': 'static', 'offset': 0, 'phases': [[d, st] for d, st in TLS_PROGRAM]}
            for i in range(1, N * N + 1)}
