"""Environment for an ARBITRARY SUMO scenario given by files (SURVEY 8f.2) — same protocol as the reference's scenario
classes (envs/real_net_env.py:114-136), with the per-scenario Python constants replaced by what the files say.

[ENV_CONFIG] keys on top of the reference's: `net_file`, `route_file`, optional `tll_file`; `scenario` may be any name
(real_net-style normalisation applies iff it is 'real_net')."""
from __future__ import annotations

import numpy as np

from ..net import sumo_ingest as _ing
from .env import PhaseMap, PhaseSet, TrafficSimulator


class SumoFilePhase(PhaseMap):
    def __init__(self, phases):
        self.phases = {key: PhaseSet(val) for key, val in phases.items()}


class SumoNetEnv(TrafficSimulator):
    def __init__(self, config, port=0, output_path='', is_record=False, record_stat=False, n_replicas=1, device=0):
        self.net_file, self.route_file = config.get('net_file'), config.get('route_file')
        self.tll_file = config.get('tll_file', fallback=None)
        self._phases = _ing.read_tls_programs(self.net_file, self.tll_file)
        self._nbr = _ing.derive_neighbor_map(self.net_file, self._phases.keys())
        super().__init__(config, output_path, is_record, record_stat, port=port, n_replicas=n_replicas, device=device)

    def _get_node_phase_id(self, node_name):
        return node_name

    def _init_map(self):
        self.neighbor_map = self._nbr
        self.phase_map = SumoFilePhase(self._phases)
        self.state_names = ['wave', 'wait'] if self.norms['wait'] > 0 and self.coef_wait > 0 else ['wave']

    def _build_tables(self):
        return _ing.load_sumo_scenario(self.net_file, self.route_file, self.tll_file, tls_phases=self._phases,
                                       neighbor_map=self._nbr, agent=self.agent, coop_gamma=self.coop_gamma,
                                       episode_length_sec=self.episode_length_sec,
                                       use_wait='wait' in self.state_names)


class SumoNetController:
    """Greedy controller for file-defined scenarios: the phase whose green links carry the largest summed wave
    (the rule of envs/real_net_env.py:90-111)."""

    def __init__(self, node_names, nodes, phases):
        self.name, self.node_names, self.nodes, self.phases = 'greedy', node_names, nodes, phases

    def forward(self, obs):
        acts = []
        for ob, name in zip(obs, self.node_names):
            node, flows = self.nodes[name], []
            for phase in self.phases[name]:
                wave, seen = 0.0, set()
                for i, sgn in enumerate(phase):
                    if sgn in 'Gg' and node.lanes_in[i] not in seen:
                        wave += ob[node.ilds_in.index(node.lanes_in[i])]
                        seen.add(node.lanes_in[i])
                flows.append(wave)
            acts.append(int(np.argmax(flows)))
        return acts

    def greedy_program(self, node_obs_off):
        """forward() as a table for tsc_greedy_actions (envs.env.greedy_table): the 'G' / 'g' lanes of each phase."""
        from .env import greedy_table, green_lane_entries
        return greedy_table([green_lane_entries(self.nodes[name], self.phases[name], 'Gg', node_obs_off[i])
                             for i, name in enumerate(self.node_names)])
