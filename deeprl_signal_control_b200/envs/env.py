"""`TrafficSimulator`: the reference's environment protocol (envs/env.py:82-635) over libtsc.

Same constructor arguments, attributes and method names as the reference so that its callers
(`utils.py:Trainer/Tester/Evaluator`, `main.py`) work unchanged:

    reset(gui=False, test_ind=0) -> list[np.ndarray]                    envs/env.py:544-561
    step(action) -> (list[np.ndarray], np.ndarray[A], bool, float)      envs/env.py:566-631
    terminate(), update_fingerprint(policy), init_test_seeds, init_data, output_data,
    collect_tripinfo; attributes agent, name, T, n_s, n_a, n_s_ls, n_a_ls, n_w_ls, n_f_ls,
    node_names, nodes, train_mode, test_num, cur_episode, seed.

With `n_replicas == 1` (default) returns exactly the reference's Python types, through the
host-buffer entry point `tsc_step_host`.  With `n_replicas > 1` the batched methods
(`reset_batch/step_batch`) return device tensors [R, ...] for the device-resident learner.
There is no SUMO process: `gui` is accepted and ignored, `terminate()` is a no-op.
"""
from __future__ import annotations

import logging
from typing import List, Optional

import numpy as np

from ..net.tables import EnvParams, NetTables

DEFAULT_PORT = 8000
REALNET_REWARD_NORM = 20     # envs/env.py:18


def greedy_table(cands):
    """CSR form of a greedy controller (tsc_set_greedy_program): cands[i] = list of (observation offsets, action) of node
    i's candidate phases, in the controller's order.  Returns (max_cand, off, idx, act) int32 arrays; padding candidates
    carry action -1."""
    max_cand = max(len(c) for c in cands)
    off, idx, act = [0], [], []
    for node in cands:
        for c in range(max_cand):
            entries, a = node[c] if c < len(node) else ([], -1)
            idx.extend(int(e) for e in entries)
            off.append(len(idx))
            act.append(int(a))
    return (max_cand, np.asarray(off, np.int32), np.asarray(idx, np.int32), np.asarray(act, np.int32))


def green_lane_entries(node, phases, green, base):
    """[(observation offsets, action)] of a node's phases: the detector entry of every lane whose signal is in `green`,
    each lane counted once (envs/real_net_env.py:90-111)."""
    out = []
    for a, phase in enumerate(phases):
        entries, seen = [], set()
        for i, signal in enumerate(phase):
            if signal in green:
                ild = node.lanes_in[i]
                if ild not in seen:
                    entries.append(base + node.ilds_in.index(ild))
                    seen.add(ild)
        out.append((entries, a))
    return out


class PhaseSet:              # envs/env.py:20-39
    def __init__(self, phases):
        self.num_phase = len(phases)
        self.num_lane = len(phases[0])
        self.phases = phases


class PhaseMap:              # envs/env.py:42-59
    def __init__(self):
        self.phases = {}

    def get_phase(self, phase_id, action):
        return self.phases[phase_id].phases[int(action)]

    def get_phase_num(self, phase_id):
        return self.phases[phase_id].num_phase

    def get_lane_num(self, phase_id):
        return self.phases[phase_id].num_lane


class Node:                  # envs/env.py:62-79
    def __init__(self, name, neighbor=(), control=False):
        self.control = control
        self.lanes_in = []
        self.ilds_in = []
        self.fingerprint = []
        self.name = name
        self.neighbor = list(neighbor)
        self.num_state = 0
        self.num_fingerprint = 0
        self.wave_state = []
        self.wait_state = []
        self.phase_id = -1
        self.n_a = 0
        self.prev_action = -1


class TrafficSimulator:
    def __init__(self, config, output_path, is_record, record_stats, port=0, n_replicas=1, device=0):
        self.name = config.get('scenario')
        self.seed = config.getint('seed')
        self.control_interval_sec = config.getint('control_interval_sec')
        self.yellow_interval_sec = config.getint('yellow_interval_sec')
        self.episode_length_sec = config.getint('episode_length_sec')
        self.T = np.ceil(self.episode_length_sec / self.control_interval_sec)
        self.port = DEFAULT_PORT + port
        self.sim_thread = port
        self.obj = config.get('objective')
        self.data_path = config.get('data_path')
        self.agent = config.get('agent')
        self.coop_gamma = config.getfloat('coop_gamma')
        self.cur_episode = 0
        self.norms = {'wave': config.getfloat('norm_wave'), 'wait': config.getfloat('norm_wait')}
        self.clips = {'wave': config.getfloat('clip_wave'), 'wait': config.getfloat('clip_wait')}
        self.coef_wait = config.getfloat('coef_wait')
        # optional key (not in the reference's configs): the driver reaction time of the vType.  1.0 = SUMO's default, which
        # the current reference uses; the paper-era runs used tau="0.5" (reference README.md:63, DESIGN.md §2)
        self.tau = config.getfloat('tau', fallback=1.0)
        self.train_mode = True
        test_seeds = [int(s) for s in config.get('test_seeds').split(',')]
        self.n_replicas = int(n_replicas)
        self.device = device
        self._init_map()
        self.init_data(is_record, record_stats, output_path)
        self.init_test_seeds(test_seeds)
        self._tables: NetTables = self._build_tables()
        self._params: EnvParams = self._build_params()
        self._init_nodes()
        self._sim = None
        self._fp = None
        self.cur_sec = 0

    # ---- to be provided by the scenario subclass --------------------------------------------
    def _init_map(self):
        raise NotImplementedError()

    def _build_tables(self) -> NetTables:
        raise NotImplementedError()

    def _get_node_phase_id(self, node_name):
        raise NotImplementedError()

    # ---- construction -------------------------------------------------------------------------
    def _build_params(self) -> EnvParams:
        real = self.name == 'real_net'
        return EnvParams(
            control_interval_sec=self.control_interval_sec, yellow_interval_sec=self.yellow_interval_sec,
            episode_length_sec=self.episode_length_sec,
            teleport_sec=300 if real else 600,                         # envs/env.py:281-284
            norm_wave=self.norms['wave'], norm_wait=self.norms['wait'],
            clip_wave=self.clips['wave'], clip_wait=self.clips['wait'],
            coef_wait=self.coef_wait, coop_gamma=self.coop_gamma, objective=self.obj, agent=self.agent,
            real_net_norm=real, use_wait='wait' in self.state_names,
            det_len=-1.0 if real else 50.0,                            # envs/env.py:333,376-377
            halt_speed=0.1 if real else 1.39, queue_cap=10 if real else (1 << 20), tau=self.tau)

    def _init_nodes(self):                                            # envs/env.py:207-242
        t = self._tables
        nodes = {}
        for name in t.node_names:
            if name in self.neighbor_map:
                neighbor = self.neighbor_map[name]
            else:
                logging.info('node %s can not be found!' % name)
                neighbor = []
            node = Node(name, neighbor=neighbor, control=True)
            node.lanes_in = list(t.lanes_in[name])
            node.ilds_in = list(t.ilds_in[name])
            nodes[name] = node
        self.nodes = nodes
        self.node_names = sorted(list(nodes.keys()))
        assert self.node_names == t.node_names
        self._init_action_space()
        self._init_state_space()

    def _init_action_space(self):                                     # envs/env.py:244-254
        self.n_a_ls = []
        for name in self.node_names:
            node = self.nodes[name]
            node.phase_id = self._get_node_phase_id(name)
            node.n_a = self.phase_map.get_phase_num(node.phase_id)
            self.n_a_ls.append(node.n_a)
        self.n_a = np.prod(np.array(self.n_a_ls))

    def _init_state_space(self):                                      # envs/env.py:303-323
        self._reset_state()
        t = self._tables
        self.n_s_ls, self.n_w_ls, self.n_f_ls = list(t.n_s_ls), list(t.n_w_ls), list(t.n_f_ls)
        self.n_s = np.sum(np.array(self.n_s_ls))

    def _reset_state(self):                                           # envs/env.py:444-453
        for name in self.node_names:
            node = self.nodes[name]
            node.prev_action = 0
            node.num_fingerprint = node.n_a - 1
            node.num_state = len(node.ilds_in)

    def _init_policy(self):                                           # envs/env.py:263-269
        return [np.array([1. / self.nodes[n].n_a] * self.nodes[n].n_a) for n in self.node_names]

    # ---- data recording (evaluation runs): envs/env.py:409-437, 498-542 ---------------------------
    def init_data(self, is_record, record_stats, output_path):
        self.is_record = is_record
        self.record_stats = record_stats
        self.output_path = output_path
        if self.is_record:
            self.traffic_data, self.control_data, self.trip_data = [], [], []
        if self.record_stats:
            self.state_stat = {name: [] for name in self.state_names}

    def init_test_seeds(self, test_seeds):
        self.test_num = len(test_seeds)
        self.test_seeds = test_seeds

    def _record_traffic(self, stats, sec0):
        """`_measure_traffic_step` rows (envs/env.py:409-437) of replica 0 from the per-second statistics of one
        control step; departed / arrived are per second there, cumulative in the library."""
        for k, st in enumerate(stats):
            dep, arr = int(st[1]), int(st[2])
            self.traffic_data.append({'episode': self.cur_episode, 'time_sec': sec0 + k + 1,
                                      'number_total_car': int(st[0]),
                                      'number_departed_car': dep - self._n_dep_prev,
                                      'number_arrived_car': arr - self._n_arr_prev,
                                      'avg_wait_sec': float(st[3]), 'avg_speed_mps': float(st[4]),
                                      'std_queue': float(st[6]), 'avg_queue': float(st[5])})
            self._n_dep_prev, self._n_arr_prev = dep, arr

    def _record_control(self, action, greward):
        self.control_data.append({'episode': self.cur_episode, 'time_sec': self.cur_sec,
                                  'step': self.cur_sec / self.control_interval_sec,
                                  'action': ','.join(['%d' % a for a in action]),
                                  'reward': float(greward)})

    def collect_tripinfo(self):
        """Trip rows of the episode that just finished (the reference parses SUMO's --tripinfo-output,
        envs/env.py:498-515; here: the arrival log of replica 0, `tsc_get_trips`)."""
        if not self.is_record or self._sim is None:
            return
        for dep, arr, route, wsec, wcnt in self._sim.trips(0):
            self.trip_data.append({'episode': self.cur_episode, 'id': 'r%d.%d' % (route, dep),
                                   'depart_sec': float(dep), 'arrival_sec': float(arr),
                                   'duration_sec': float(arr - dep), 'wait_step': int(wcnt), 'wait_sec': float(wsec)})

    def output_data(self):
        if not self.is_record:
            logging.error('Env: no record to output!')
            return
        import pandas as pd
        base = self.output_path + ('%s_%s_' % (self.name, self.agent))
        pd.DataFrame(self.control_data).to_csv(base + 'control.csv')
        pd.DataFrame(self.traffic_data).to_csv(base + 'traffic.csv')
        pd.DataFrame(self.trip_data).to_csv(base + 'trip.csv')

    # ---- simulator lifecycle --------------------------------------------------------------------
    def _ensure_sim(self):
        if self._sim is None:
            from ..sim import BatchedSim      # fails loudly without CUDA / libtsc.so
            self._sim = BatchedSim(self._tables, self._params, self.n_replicas, device=self.device)
        return self._sim

    def _episode_seeds(self, seed):
        # replica r plays the episode the reference would play r episodes later (seed += 1 per reset)
        return (np.arange(self.n_replicas, dtype=np.uint64) + np.uint64(seed))

    def _fp_array(self) -> Optional[np.ndarray]:
        if self.agent != 'ma2c':
            return None
        return self._fp

    def reset(self, gui=False, test_ind=0):
        self._reset_state()
        seed = self.seed if self.train_mode else self.test_seeds[test_ind]
        sim = self._ensure_sim()
        sim.reset(self._episode_seeds(seed))
        sim.set_train_mode(self.train_mode)
        if self.is_record:
            sim.set_record(True)                                      # trip words + arrival log from second 0
            self._n_dep_prev = self._n_arr_prev = 0
        self.cur_sec = 0
        self.cur_episode += 1
        if self.agent == 'ma2c':
            self.update_fingerprint(self._init_policy())
        self.seed += self.n_replicas if self.n_replicas > 1 else 1
        return self._get_state()

    def terminate(self):
        return

    def update_fingerprint(self, policy):                             # envs/env.py:633-635
        t = self._tables
        if self._fp is None:
            self._fp = np.zeros((self.n_replicas, t.n_nodes, t.max_na), np.float32)
        for i, (name, pi) in enumerate(zip(self.node_names, policy)):
            pi = np.asarray(pi, dtype=np.float32)
            self.nodes[name].fingerprint = np.array(pi)[..., :-1]
            self._fp[:, i, :pi.shape[-1]] = pi

    def _split_obs(self, row: np.ndarray) -> List[np.ndarray]:
        off = self._tables.node_obs_off
        return [row[off[i]:off[i + 1]].astype(np.float64) for i in range(len(self.node_names))]

    def _get_state(self):
        import torch
        sim = self._ensure_sim()
        fp = self._fp_array()
        fp_dev = None if fp is None else torch.from_numpy(fp).to(sim.device)
        obs = sim.observe(fp_dev).cpu().numpy()
        return self._split_obs(obs[0]) if self.n_replicas == 1 else obs

    def step(self, action):
        sim = self._ensure_sim()
        sim.set_train_mode(self.train_mode)
        act = np.asarray(action, dtype=np.int32).reshape(self.n_replicas, -1)
        if self.is_record:
            import torch
            fp = self._fp_array()
            o, r, g, d, st = sim.step_record(torch.from_numpy(act), None if fp is None else torch.from_numpy(fp).to(sim.device))
            obs, reward, greward, done = o.cpu().numpy(), r.cpu().numpy(), g.cpu().numpy(), d.cpu().numpy()
            self._record_traffic(st[0].cpu().numpy(), self.cur_sec)
        else:
            obs, reward, greward, done = sim.step_host(act, self._fp_array())
        self.cur_sec += self.control_interval_sec
        for name, a in zip(self.node_names, act[0]):
            self.nodes[name].prev_action = int(a)
        if self.is_record:
            self._record_control(act[0], greward[0])
        if self.n_replicas > 1:
            return obs.copy(), reward.copy(), bool(done[0]), greward.copy()
        reward0 = reward[0].astype(np.float64)
        if self.train_mode and self.agent in ('a2c', 'greedy'):
            reward0 = float(greward[0])                              # envs/env.py:593-594
        return self._split_obs(obs[0]), reward0, bool(done[0]), float(greward[0])
