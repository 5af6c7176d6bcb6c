"""large_grid scenario classes with the reference's names (envs/large_grid_env.py)."""
from __future__ import annotations

import numpy as np

STATE_NAMES = ['wave', 'wait']      # envs/large_grid_env.py:19
PHASE_NUM = 5                       # envs/large_grid_env.py:20


class LargeGridController:
    """Greedy policy of the reference (envs/large_grid_env.py:45-60): per node, pick the phase
    whose green lanes carry the largest summed wave.  Accepts [A][>=6] observations (list of
    arrays, as the reference) or a batched [R, A, >=6] array."""

    def __init__(self, node_names):
        self.name = 'greedy'
        self.node_names = node_names

    def forward(self, obs):
        ob = np.asarray(obs) if not isinstance(obs, list) else np.stack([np.asarray(o)[:6] for o in obs])
        flows = np.stack([ob[..., 0] + ob[..., 3], ob[..., 2] + ob[..., 5], ob[..., 1] + ob[..., 4],
                          ob[..., 1] + ob[..., 2], ob[..., 4] + ob[..., 5]], axis=-1)
        return np.argmax(flows, axis=-1)

    def greedy(self, ob, node_name):
        return int(self.forward([ob])[0])

    # the five candidate phases of forward() as pairs of wave entries, candidate index = action
    GREEDY_PAIRS = ((0, 3), (2, 5), (1, 4), (1, 2), (4, 5))

    def greedy_program(self, node_obs_off):
        """forward() as a table for tsc_greedy_actions (envs.env.greedy_table)."""
        from .env import greedy_table
        return greedy_table([[((node_obs_off[i] + a, node_obs_off[i] + b), c) for c, (a, b) in enumerate(self.GREEDY_PAIRS)]
                             for i in range(len(self.node_names))])


from .env import PhaseMap, PhaseSet, TrafficSimulator        # noqa: E402
from ..net import large_grid as _grid                         # noqa: E402


class LargeGridPhase(PhaseMap):                               # envs/large_grid_env.py:38-42
    def __init__(self):
        self.phases = {PHASE_NUM: PhaseSet(list(_grid.PHASES))}


class LargeGridEnv(TrafficSimulator):
    """Drop-in for reference envs/large_grid_env.py:63-223: same constructor
    `LargeGridEnv(config['ENV_CONFIG'], port=0, output_path='', is_record=False, record_stat=False)`;
    `n_replicas`/`device` are extensions (default 1 replica = the reference's behaviour)."""

    def __init__(self, config, port=0, output_path='', is_record=False, record_stat=False,
                 n_replicas=1, device=0):
        self.peak_flow1 = config.getint('peak_flow1')
        self.peak_flow2 = config.getint('peak_flow2')
        self.init_density = config.getfloat('init_density')
        super().__init__(config, output_path, is_record, record_stat, port=port,
                         n_replicas=n_replicas, device=device)

    def _get_node_phase_id(self, node_name):
        return PHASE_NUM

    def _init_map(self):                                       # envs/large_grid_env.py:209-215
        self.neighbor_map = _grid.large_neighbor_map()
        self.phase_map = LargeGridPhase()
        self.state_names = STATE_NAMES

    def _build_tables(self):
        return _grid.build_large_grid(self.peak_flow1, self.peak_flow2, agent=self.agent,
                                      coop_gamma=self.coop_gamma, use_wait='wait' in self.state_names,
                                      episode_length_sec=self.episode_length_sec,
                                      init_density=self.init_density, seed=self.seed)
        # init_density > 0 (large_grid/data/build_file.py:223-266): the destinations of the initial fleet are drawn once per
        # environment from the config seed (the reference redraws them with every episode's seed)
