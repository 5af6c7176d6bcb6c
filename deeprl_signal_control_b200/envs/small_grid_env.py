"""`small_grid` scenario classes with the reference's names and protocol (envs/small_grid_env.py):
`SmallGridEnv`, `SmallGridController`, `SmallGridPhase`.

The reference runs this 6-intersection benchmark with the `greedy` (and centralised `a2c`) agent only: its neighbour map
names the priority junction `npc`, which is not a TLS node, so the MARL state code of envs/env.py:303-323 raises KeyError
there.  Here `npc` is dropped from the neighbour lists (net/small_grid.py), so ia2c / ma2c run as well.
"""
from __future__ import annotations

import numpy as np

from .env import PhaseMap, PhaseSet, TrafficSimulator
from ..net import small_grid as _small

STATE_NAMES = ['wave', 'wait']                                   # envs/small_grid_env.py:27
# map from ild order to signal order (envs/small_grid_env.py:28-31)
STATE_PHASE_MAP = {'nt1': [0, 1, 2], 'nt2': [1, 0], 'nt3': [1, 0], 'nt4': [1, 0], 'nt5': [1, 0], 'nt6': [1, 0]}


class SmallGridPhase(PhaseMap):                                  # envs/small_grid_env.py:34-38
    def __init__(self):
        self.phases = {2: PhaseSet(list(_small.TWO_PHASE)), 3: PhaseSet(list(_small.THREE_PHASE))}


class SmallGridController:
    """Greedy policy of the reference (envs/small_grid_env.py:41-57): the phase mapped to the detector with the
    largest wave.  Accepts the reference's list of per-node arrays or a batched [R, sum n_s] observation array."""

    def __init__(self, node_names):
        self.name = 'greedy'
        self.node_names = node_names

    def forward(self, obs):
        return [self.greedy(ob, name) for ob, name in zip(obs, self.node_names)]

    def greedy(self, ob, node_name):
        phases = STATE_PHASE_MAP[node_name]
        flows = np.asarray(ob)[..., :len(phases)]
        return np.asarray(phases)[np.argmax(flows, axis=-1)]

    def greedy_program(self, node_obs_off):
        """greedy() as a table for tsc_greedy_actions (envs.env.greedy_table): candidate c = wave entry c, mapped to
        STATE_PHASE_MAP's phase."""
        from .env import greedy_table
        return greedy_table([[((node_obs_off[i] + c,), a) for c, a in enumerate(STATE_PHASE_MAP[name])]
                             for i, name in enumerate(self.node_names)])


class SmallGridEnv(TrafficSimulator):
    """Drop-in for reference envs/small_grid_env.py:60-84: `SmallGridEnv(config['ENV_CONFIG'], port=0, output_path='',
    is_record=False, record_stat=False)`; `n_replicas` / `device` are extensions."""

    def __init__(self, config, port=0, output_path='', is_record=False, record_stat=False, n_replicas=1, device=0):
        self.num_car_hourly = config.getint('num_extra_car_per_hour')
        super().__init__(config, output_path, is_record, record_stat, port=port, n_replicas=n_replicas, device=device)

    def _get_node_phase_id(self, node_name):                     # envs/small_grid_env.py:65-68
        return 3 if node_name == 'nt1' else 2

    def _init_map(self):                                          # envs/small_grid_env.py:70-73
        self.neighbor_map = {k: [n for n in v if n != 'npc'] for k, v in _small.SMALL_GRID_NEIGHBOR_MAP.items()}
        self.phase_map = SmallGridPhase()
        self.state_names = STATE_NAMES

    def _build_tables(self):
        return _small.build_small_grid(self.num_car_hourly, agent=self.agent, coop_gamma=self.coop_gamma,
                                       use_wait='wait' in self.state_names,
                                       episode_length_sec=self.episode_length_sec)
