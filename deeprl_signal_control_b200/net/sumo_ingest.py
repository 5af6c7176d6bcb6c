"""General SUMO scenario ingest (SURVEY 8f.2): everything the reference hard-wires per scenario in Python
(envs/real_net_env.py:20-68 NODES / PHASES, real_net/data/build_file.py:27-105 flows) is read from the scenario's
FILES instead, so that an arbitrary netconvert net with a route file loads into `NetTables`:

  * signal programs   <tlLogic id=...><phase state=.../></tlLogic> of the .net.xml (or of an additional .tll.xml):
                      an agent's action set = the program's distinct phases without a yellow ('y'/'Y') link
                      (the reference inserts the yellow transition itself, envs/env.py:128-152), all-red excluded;
  * neighbour map     signalised junction -> the signalised junctions reachable along edges without crossing another
                      signalised junction (what the hand-written lists encode), nearest first, capped at `max_neighbors`;
  * demand            <flow from= to= via= begin= end= vehsPerHour|period|number= .../> and
                      <flow route= ...> / <route id= edges=> of a .rou.xml.

`load_sumo_scenario` hands these to `real_net.build_from_sumo`, which does lanes / links / foes / routing.
"""
from __future__ import annotations

import heapq
import xml.etree.ElementTree as ET
from typing import Dict, List, Optional, Tuple

from .real_net import build_from_sumo
from .tables import NetTables


def read_tls_programs(*files: str) -> Dict[str, List[str]]:
    """{tlLogic id: green phase strings in program order} from net / additional files (later files override)."""
    out: Dict[str, List[str]] = {}
    for f in files:
        if not f:
            continue
        for tl in ET.parse(f).getroot().iter('tlLogic'):
            phases = []
            for ph in tl.findall('phase'):
                st = ph.get('state')
                if 'y' in st or 'Y' in st or 'u' in st:        # transition phases: the env generates yellow itself
                    continue
                if not any(ch in 'Gg' for ch in st):           # all-red clearance
                    continue
                if st not in phases:
                    phases.append(st)
            if phases:
                out[tl.get('id')] = phases
    return out


def read_signal_programs(*files: str) -> Dict[str, dict]:
    """{tlLogic id: {'type', 'offset', 'phases': [[duration, state], ...]}} of the whole static programs in net /
    additional files (later files override; a '.gz' file is read through gzip), the attribute values as the file writes
    them.  envs.fixedtime checks and runs them.  Two keys appear only where the file has them: 'phase_attrs', one
    {attribute: value} per phase of its attributes other than duration and state (minDur, maxDur, next, ...), and
    'params', {key: value} of the tlLogic's <param>s; envs.actuated reads them."""
    import gzip
    out: Dict[str, dict] = {}
    for f in files:
        if not f:
            continue
        with (gzip.open(f) if f.endswith('.gz') else open(f, 'rb')) as fh:
            root = ET.parse(fh).getroot()
        for tl in root.iter('tlLogic'):
            phases = tl.findall('phase')
            prog = {'type': tl.get('type', 'static'), 'offset': tl.get('offset', '0'),
                    'phases': [[ph.get('duration'), ph.get('state')] for ph in phases]}
            attrs = [{k: v for k, v in ph.attrib.items() if k not in ('duration', 'state')} for ph in phases]
            if any(attrs):
                prog['phase_attrs'] = attrs
            params = {p.get('key'): p.get('value') for p in tl.findall('param')}
            if params:
                prog['params'] = params
            out[tl.get('id')] = prog
    return out


def derive_neighbor_map(net_file: str, tls_ids, max_neighbors: int = 5) -> Dict[str, List[str]]:
    """Signalised junction -> neighbouring signalised junctions (by driving distance along normal edges, not passing
    through another signalised junction).  A tlLogic id is matched to the junctions whose connections carry `tl=id`."""
    root = ET.parse(net_file).getroot()
    tls_ids = set(tls_ids)
    edge_from, edge_to, edge_len = {}, {}, {}
    for e in root.findall('edge'):
        if e.get('function') == 'internal':
            continue
        edge_from[e.get('id')], edge_to[e.get('id')] = e.get('from'), e.get('to')
        edge_len[e.get('id')] = float(e.find('lane').get('length'))
    junction_tl: Dict[str, str] = {}
    for c in root.findall('connection'):
        if c.get('tl') in tls_ids and c.get('from') in edge_to:
            junction_tl[edge_to[c.get('from')]] = c.get('tl')
    out_edges: Dict[str, List[str]] = {}
    for eid, j in edge_from.items():
        out_edges.setdefault(j, []).append(eid)
    nbr: Dict[str, List[str]] = {}
    for tl in sorted(tls_ids):
        starts = [j for j, t in junction_tl.items() if t == tl]
        dist: Dict[str, float] = {j: 0.0 for j in starts}
        found: Dict[str, float] = {}
        pq = [(0.0, j) for j in starts]
        while pq:
            d, j = heapq.heappop(pq)
            if d > dist.get(j, 1e30):
                continue
            t = junction_tl.get(j)
            if t is not None and t != tl:
                found[t] = min(found.get(t, 1e30), d)
                continue                                        # do not look past another signalised junction
            for eid in out_edges.get(j, ()):
                nj, nd = edge_to[eid], d + edge_len[eid]
                if nd < dist.get(nj, 1e30):
                    dist[nj] = nd
                    heapq.heappush(pq, (nd, nj))
        nbr[tl] = [t for t, _ in sorted(found.items(), key=lambda kv: (kv[1], kv[0]))][:max_neighbors]
    return nbr


def read_flows(rou_file: str, horizon: int = 3600):
    """-> (flow_defs [(from, to, via)], flow_list [(route index, begin, end, vehsPerHour)])."""
    root = ET.parse(rou_file).getroot()
    routes = {r.get('id'): r.get('edges').split() for r in root.findall('route')}
    defs: List[Tuple[str, str, str]] = []
    index: Dict[Tuple[str, str, str], int] = {}
    flow_list = []
    for fl in root.findall('flow'):
        if fl.get('route') is not None:
            ed = routes[fl.get('route')]
            key = (ed[0], ed[-1], ' '.join(ed[1:-1]))
        elif fl.find('route') is not None:
            ed = fl.find('route').get('edges').split()
            key = (ed[0], ed[-1], ' '.join(ed[1:-1]))
        else:
            key = (fl.get('from'), fl.get('to'), fl.get('via') or '')
        if key not in index:
            index[key] = len(defs)
            defs.append(key)
        tb, te = int(float(fl.get('begin', 0))), int(float(fl.get('end', horizon)))
        if fl.get('vehsPerHour') is not None:
            rate = float(fl.get('vehsPerHour'))
        elif fl.get('period') is not None:
            rate = 3600.0 / float(fl.get('period'))
        elif fl.get('number') is not None:
            rate = float(fl.get('number')) * 3600.0 / max(te - tb, 1)
        else:
            raise ValueError('flow %s: need vehsPerHour, period or number' % fl.get('id'))
        flow_list.append((index[key], tb, min(te, horizon), rate))
    return defs, flow_list


def load_sumo_scenario(net_file: str, rou_file: str, tll_file: Optional[str] = None,
                       tls_phases: Optional[Dict[str, List[str]]] = None,
                       neighbor_map: Optional[Dict[str, List[str]]] = None, agent: str = 'ma2c',
                       coop_gamma: float = 0.9, episode_length_sec: int = 3600, use_wait: bool = False,
                       max_neighbors: int = 5) -> NetTables:
    """One call from SUMO files to simulator tables; explicit `tls_phases` / `neighbor_map` override the derived ones
    (that is how the reference's hand-written Monaco definition is reproduced exactly)."""
    phases = dict(read_tls_programs(net_file, tll_file))
    if tls_phases:
        phases = dict(tls_phases)
    if not phases:
        raise ValueError('no <tlLogic> with a green phase found in %s' % net_file)
    nbr = neighbor_map if neighbor_map is not None else derive_neighbor_map(net_file, phases.keys(), max_neighbors)
    defs, flow_list = read_flows(rou_file, episode_length_sec)
    return build_from_sumo(net_file, phases, nbr, defs, flow_list, agent=agent, coop_gamma=coop_gamma,
                           episode_length_sec=episode_length_sec, use_wait=use_wait)
