"""Monaco `real_net` scenario classes with the reference's names (envs/real_net_env.py)."""
from __future__ import annotations

import os

import numpy as np

from ..net import real_net as _rn
from .env import PhaseMap, PhaseSet, TrafficSimulator

STATE_NAMES = ['wave']                      # envs/real_net_env.py:18
NODES, PHASES = _rn.NODES, _rn.PHASES


class RealNetPhase(PhaseMap):               # envs/real_net_env.py:71-75
    def __init__(self):
        self.phases = {key: PhaseSet(val) for key, val in PHASES.items()}


class RealNetController:
    """Greedy policy of the reference (envs/real_net_env.py:78-111): per node, the phase whose 'G'
    links carry the largest summed wave, every controlled lane counted once."""

    def __init__(self, node_names, nodes):
        self.name = 'greedy'
        self.node_names = node_names
        self.nodes = nodes

    def forward(self, obs):
        return [self.greedy(ob, name) for ob, name in zip(obs, self.node_names)]

    def greedy(self, ob, node_name):
        phases = PHASES[NODES[node_name][0]]
        node = self.nodes[node_name]
        flows = []
        for phase in phases:
            wave, seen = 0, set()
            for i, signal in enumerate(phase):
                if signal == 'G':
                    ild = node.lanes_in[i]
                    if ild not in seen:
                        wave += ob[node.ilds_in.index(ild)]
                        seen.add(ild)
            flows.append(wave)
        return int(np.argmax(np.array(flows)))

    def greedy_program(self, node_obs_off):
        """greedy() as a table for tsc_greedy_actions (envs.env.greedy_table): per phase, the observation entries of its
        'G' lanes, each lane once, in the order greedy() adds them."""
        from .env import greedy_table, green_lane_entries
        return greedy_table([green_lane_entries(self.nodes[name], PHASES[NODES[name][0]], 'G', node_obs_off[i])
                             for i, name in enumerate(self.node_names)])


class RealNetEnv(TrafficSimulator):
    """Drop-in for reference envs/real_net_env.py:114-136.  The net is parsed from
    `<data_path>/in/most.net.xml` when that file exists (a reference checkout), otherwise the
    derived tables shipped with the package are used."""

    def __init__(self, config, port=0, output_path='', is_record=False, record_stat=False,
                 n_replicas=1, device=0):
        self.flow_rate = config.getint('flow_rate')
        super().__init__(config, output_path, is_record, record_stat, port=port,
                         n_replicas=n_replicas, device=device)

    def _get_node_phase_id(self, node_name):
        return self.phase_node_map[node_name]

    def _init_map(self):                    # envs/real_net_env.py:124-128
        self.neighbor_map = dict([(key, val[1]) for key, val in NODES.items()])
        self.phase_map = RealNetPhase()
        self.phase_node_map = dict([(key, val[0]) for key, val in NODES.items()])
        self.state_names = STATE_NAMES

    def _build_tables(self):
        net_file = os.path.join(self.data_path or '', 'in', 'most.net.xml')
        return _rn.real_net_tables(self.agent, net_file if os.path.exists(net_file) else None,
                                   flow_rate=self.flow_rate, coop_gamma=self.coop_gamma)
