"""Test-mode evaluation on the device, every test seed at once — the batched counterpart of reference
utils.py:Tester.perform / Evaluator.run (utils.py:195-234, 311-388).

    Evaluator(env, model, output_path, demo=False, policy_type='default', seed=None).run()
    GroupEvaluator(entries, seeds, policy_type='default', policy='lstm').run()

`Evaluator` evaluates one model on its env's own simulator.  `env` is a scenario env (LargeGridEnv, RealNetEnv, ...)
built with `n_replicas == env.test_num`: replica k plays the episode the one-replica env plays after
`reset(test_ind=k)` (seed `test_seeds[k]`, test-mode rewards), and in record mode `output_data()` writes the control /
traffic / trip CSVs with the rows, in the order, that the one-replica env writes when it runs the seeds one after
another.  `GroupEvaluator` evaluates several agent directories on the same seeds in one process (the reference's
`main.py evaluate --agents`): entries whose simulators would be built identically share one.  Both run `_Group`, one
simulator and the forwards of its members; an `Evaluator` is a group of one member.

A member's model is an IA2C / MA2C wrapper (agents/models.py; only its parameters `batched.P` and the packed image
`batched.Wp` are read), an IQL (`model.name == 'iql'`, LR or DQN; only its `nets` are read), a greedy controller
(`model.name == 'greedy'`), the max-pressure controller (`model.name == 'maxpressure'`, envs.maxpressure_controller;
nothing of it is read), the fixed-time controller (`model.name == 'fixedtime'`, envs.fixedtime_controller) or the
vehicle-actuated controller (`model.name == 'actuated'`, envs.actuated_controller); the last two have their `program`
set on the simulator, which runs it with no action launch and action = NULL.  Fixed-time members read their `program`
at the start of every episode: one program for all is set as it is, different ones as one plan per member on its
replicas (tsc_set_replica_signal_programs).  The parameters are copied into the
group's own buffers at the start of every episode, so a live learner evaluated mid-training is read at its current
weights, and its parameters, optimiser slot, recurrent states, rollout and counters are left as they were.

Per control step, with no host synchronisation inside the episode, one launch per forward family (forward_family): the
grouped pi-only forward tscl_policy_step_pi_g for the A2C members of one fused tensor-core layout (a member on the v1
forward or the fc-policy kernels has its own launches, then tscl_argmax_actions), the grouped fp32 Q forward
tscl_q_step_g per IQL layout (argmax of q, or the normalised-q sample of IQL.forward(stochastic=True)),
tsc_greedy_actions or tsc_pressure_actions; for MA2C the fingerprint is the pi just computed; tsc_step (tsc_step_record
in record mode, the recorded actions copied from the simulator's phase tap: the action applied, or the program phase of
the interval's first second); the global reward goes into a [T][R] float32 trace.
"""
from __future__ import annotations

import ctypes as C
import itertools
import logging

import numpy as np
import torch

from .. import _lib


_p = _lib.ptr


def replica_seeds(env):
    """Replica k plays test episode k: the seed the one-replica env takes after reset(test_ind=k) in test mode (not the
    `seed + r` mapping env.reset uses for n_replicas > 1)."""
    return np.asarray(env.test_seeds, dtype=np.uint64)


def control_frame(actions, greward, ci):
    """Control rows of envs/env.py (the reference's `control_data`): actions [R][T][N] int, greward [R][T] float32;
    replica k is episode k + 1."""
    import pandas as pd
    R, T = greward.shape
    return pd.DataFrame({'episode': np.repeat(np.arange(1, R + 1), T),
                         'time_sec': np.tile(np.arange(1, T + 1) * ci, R),
                         'step': np.tile(np.arange(1, T + 1) * ci / ci, R),
                         'action': [','.join(['%d' % a for a in row]) for row in actions.reshape(R * T, -1)],
                         'reward': greward.reshape(-1).astype(np.float64)})


def traffic_frame(stats):
    """Traffic rows of envs/env.py `_record_traffic`: stats [R][S][8] float32 per simulated second (tsc_step_record
    fields); departed / arrived are per-second differences of the cumulative counters."""
    import pandas as pd
    R, S, _ = stats.shape
    dep, arr = stats[..., 1].astype(np.int64), stats[..., 2].astype(np.int64)
    zero = np.zeros((R, 1), np.int64)
    return pd.DataFrame({'episode': np.repeat(np.arange(1, R + 1), S), 'time_sec': np.tile(np.arange(1, S + 1), R),
                         'number_total_car': stats[..., 0].astype(np.int64).reshape(-1),
                         'number_departed_car': np.diff(dep, axis=1, prepend=zero).reshape(-1),
                         'number_arrived_car': np.diff(arr, axis=1, prepend=zero).reshape(-1),
                         'avg_wait_sec': stats[..., 3].astype(np.float64).reshape(-1),
                         'avg_speed_mps': stats[..., 4].astype(np.float64).reshape(-1),
                         'std_queue': stats[..., 6].astype(np.float64).reshape(-1),
                         'avg_queue': stats[..., 5].astype(np.float64).reshape(-1)})


def trip_frame(trips):
    """Trip rows of envs/env.py `collect_tripinfo`: trips[k] = BatchedSim.trips(k) of episode k + 1."""
    import pandas as pd
    if sum(len(t) for t in trips) == 0:
        return pd.DataFrame([])                               # what the env writes when no vehicle arrived
    ep = np.concatenate([np.full(len(t), k + 1, np.int64) for k, t in enumerate(trips)] + [np.zeros(0, np.int64)])
    rows = np.concatenate([np.asarray(t, np.int64).reshape(-1, 5) for t in trips] + [np.zeros((0, 5), np.int64)])
    dep, arr, route, wsec, wcnt = rows.T
    return pd.DataFrame({'episode': ep, 'id': ['r%d.%d' % (r, d) for r, d in zip(route, dep)],
                         'depart_sec': dep.astype(np.float64), 'arrival_sec': arr.astype(np.float64),
                         'duration_sec': (arr - dep).astype(np.float64), 'wait_step': wcnt,
                         'wait_sec': wsec.astype(np.float64)})


def episode_summary(env, policy_type, mean, std, traffic=None, trip=None):
    """Evaluator.summary of the episodes played on `env`'s test seeds (mean / std: one entry per episode)."""
    out = {'scenario': env.name, 'agent': env.agent, 'policy_type': policy_type,
           'seeds': [int(s) for s in env.test_seeds], 'episode_length_sec': int(env.episode_length_sec),
           'episode_mean_reward': [float(x) for x in mean], 'episode_std_reward': [float(x) for x in std],
           'mean_reward': float(np.mean(mean)), 'std_reward': float(np.std(mean))}
    if traffic is not None:
        out.update(avg_queue=float(traffic.avg_queue.mean()), avg_speed_mps=float(traffic.avg_speed_mps.mean()),
                   avg_wait_sec=float(traffic.avg_wait_sec.mean()))
    if trip is not None:
        ep = trip.episode.values.astype(np.int64) if len(trip) else np.zeros(0, np.int64)
        n = np.bincount(ep, minlength=len(mean) + 1)[1:]
        out.update(trips_per_episode=[int(x) for x in n], mean_trips=float(np.mean(n)))
    return out


class Evaluator:
    """One model on its env's own simulator (env._ensure_sim()): a `_Group` of one member."""

    def __init__(self, env, model, output_path, demo=False, policy_type='default', seed=None):
        if policy_type not in ('default', 'stochastic', 'deterministic'):
            raise ValueError("policy_type must be 'default', 'stochastic' or 'deterministic' (got %r)" % (policy_type,))
        if env.n_replicas != env.test_num:
            raise ValueError("the evaluator plays every test seed at once: build the env with n_replicas == test_num "
                             "(%d), got %d" % (env.test_num, env.n_replicas))
        self.env, self.model, self.output_path, self.demo = env, model, output_path, demo
        self.policy_type = policy_type
        self.agent = env.agent
        self.seed = int(env.seed if seed is None else seed)
        self.env.train_mode = False
        self.test_num = env.test_num
        self.group = _Group([env], [model], [self.seed], ['Evaluator'], policy_type, sim=env._ensure_sim())
        self.sim, self.R, self.T = self.group.sim, self.group.R, self.group.T
        self.family = self.group.fwd[0][0]
        self.recorded = None          # (control, traffic, trip) frames written by the last output_data()

    # ---- reference interface ----------------------------------------------------------------------
    def perform_all(self):
        """Batched Tester.perform: (mean_reward [R], std_reward [R]) float64, np.mean / np.std of each replica's
        per-step global rewards (utils.py:230-234).  IQL: with policy_type 'stochastic' a row whose normalised q is not
        a distribution raises the ValueError np.random.choice raises in the reference."""
        self.group.episode()
        failed = self.group.failed()
        if failed:
            raise ValueError(failed[0])
        return self.group.rewards()[0]

    def run(self):
        """Evaluator.run (utils.py:376-388): every test seed, then the CSVs when the env records."""
        env = self.env
        env.cur_episode = 0
        if env.is_record:
            env.init_data(True, env.record_stats, self.output_path)
        mean, std = self.perform_all()
        for k in range(self.R):
            logging.info('test %i, avg reward %.2f' % (k, mean[k]))
        env.cur_episode = self.R
        if env.is_record:
            self.output_data()
        return mean, std

    def summary(self, mean, std, traffic=None, trip=None):
        """The quantities of the reference's recorded-evaluation table (BASELINE.md §1): mean and std over episodes of the
        per-episode mean step reward; with the recorded frames also the means of avg_queue / avg_speed_mps /
        avg_wait_sec over all recorded seconds and the completed trips per episode."""
        return episode_summary(self.env, self.policy_type, mean, std, traffic, trip)

    def frames(self):
        """(control, traffic, trip) DataFrames of the last recorded episode set."""
        return self.group.frames(0)

    def output_data(self):
        """The reference's three CSVs (envs/env.py output_data): <output_path><scenario>_<agent>_{control,traffic,trip}.csv"""
        if not self.env.is_record or self.group.stats is None:
            logging.error('Evaluator: no record to output!')
            return None
        self.recorded = self.group.output_data(0, self.output_path)
        return self.recorded


# ---- several agents at once ---------------------------------------------------------------------------------------------
# the combined replicas of one shared simulator: the recorded per-second statistics alone take T * ci * 32 bytes per
# replica (115 KB at the grid's 720 control steps of 5 s), so 65536 replicas keep the record under 8 GB
MAX_GROUP_REPLICAS = 1 << 16

CONTROLLERS = ('greedy', 'maxpressure', 'fixedtime', 'actuated')       # agent directories without a checkpoint
PROGRAMS = ('fixedtime', 'actuated')           # controllers the simulator runs itself, with no action launch
NO_A2C = "batched evaluation covers greedy, maxpressure, fixedtime, actuated, ia2c, ma2c and IQL (got agent 'a2c')"


def entry_model(agent):
    """The model an agent directory's name selects (main.py:179-190, scripts/evaluate.py): 'greedy', 'maxpressure',
    'fixedtime', 'actuated', 'ia2c', 'ma2c', 'a2c', 'iqld' -> IQL 'dqn', any other name -> IQL 'lr'."""
    if agent in CONTROLLERS + ('ia2c', 'ma2c', 'a2c'):
        return agent
    return 'dqn' if agent == 'iqld' else 'lr'


def build_model(agent, agent_dir, env, config, policy='lstm', device=0):
    """The model of an agent directory for `env`: `agent` as entry_model gives it, `config` the directory's config.
    The controllers are built without touching the simulator (the evaluators set their programs); IA2C, MA2C and IQL are
    built from [MODEL_CONFIG] and load the checkpoint under agent_dir/model/."""
    import os
    from ..envs import greedy_controller, maxpressure_controller
    from ..envs.actuated import ActuatedController
    from ..envs.fixedtime import FixedTimeController
    from .models import IA2C, IQL, MA2C
    if agent == 'greedy':
        return greedy_controller(env)
    if agent == 'maxpressure':
        return maxpressure_controller(env)
    if agent == 'fixedtime':
        return FixedTimeController(env)
    if agent == 'actuated':
        return ActuatedController(env)
    if agent == 'a2c':
        raise ValueError(NO_A2C)
    mc = config['MODEL_CONFIG']
    kw = dict(n_replicas=1, obs_off=env._tables.node_obs_off, policy=policy, device=device)
    if agent == 'ma2c':
        m = MA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, env.n_f_ls, 0, mc, **kw)
    elif agent == 'ia2c':
        m = IA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, 0, mc, **kw)
    else:
        m = IQL(env.n_s_ls, env.n_a_ls, env.n_w_ls, 0, mc, seed=0, model_type=agent, device=torch.device('cuda', device))
    if not m.load(os.path.join(agent_dir, 'model') + '/'):
        raise RuntimeError('%s: the checkpoint under %s/model/ does not load' % (agent_dir, agent_dir))
    return m


def find_checkpoint(model_dir):
    """True when `model_dir` holds a checkpoint the models' load() takes (checkpoint-<step>.npz, or .pt for A2C)."""
    import os
    import re
    return os.path.isdir(model_dir) and any(re.fullmatch(r'checkpoint-\d+\.(npz|pt)', f) for f in os.listdir(model_dir))


def _frozen(v):
    if isinstance(v, np.ndarray):
        return (v.dtype.str, v.shape, v.tobytes())
    if isinstance(v, dict):
        return tuple((k, _frozen(x)) for k, x in sorted(v.items()))
    if isinstance(v, (list, tuple)):
        return tuple(_frozen(x) for x in v)
    return v


def sim_key(env, demand=False):
    """Equal for two envs whose simulators are built identically: the scenario, the simulator parameters and every net
    table, compared on the built objects.  MA2C leaves out coop_gamma (parameter and observation scale): members that
    differ only there share a simulator through per-replica coop_gamma.  The env seed is not part of the simulator (it
    keys only the policies' sampling).  `demand` leaves out the demand tables (net.tables.DEMAND_FIELDS) as well:
    members that differ only there share a simulator through per-replica demand (tsc_set_replica_demand)."""
    import dataclasses
    from ..net.tables import DEMAND_FIELDS
    net, par = env._tables, env._params
    ma2c = par.agent == 'ma2c'
    c = par.as_c()
    cfg = tuple((n, getattr(c, n)) for n, _ in type(c)._fields_ if not (ma2c and n == 'coop_gamma'))
    tables = tuple((f.name, _frozen(getattr(net, f.name))) for f in dataclasses.fields(net)
                   if not (ma2c and f.name == 'obs_scale') and not (demand and f.name in DEMAND_FIELDS))
    return env.name, cfg, tables


class GroupEntry:
    """One agent directory of a GroupEvaluator: `label` (its name on the command line), `agent` (the directory's name),
    `model` (entry_model), `output_path`; after the checks `env` (its own one-seed-set env, no simulator), `config`,
    `seed` ([ENV_CONFIG] seed), and `error` when it was skipped; `demand`, the {key: value} demand level it runs at
    (None: its config's own).  After run(): mean / std per episode, the three frames and `summary`."""

    def __init__(self, agent_dir, model, output_path, demand=None):
        import os
        self.agent_dir = agent_dir.rstrip('/')
        self.agent = os.path.basename(self.agent_dir)
        self.label = self.agent_dir
        self.model, self.output_path = model, output_path
        self.env = self.config = self.error = None
        self.demand = demand
        self.mean = self.std = self.recorded = self.summary = None


class GroupEvaluator:
    """Several trained agents on the same test seeds in one process: the reference's `main.py evaluate --agents`
    (main.py:158-222) on shared simulators.

        GroupEvaluator(entries, seeds, policy_type='default', policy='lstm').run()

    `entries`: (agent directory, model, output path) triples, model as entry_model gives it.  The constructor only
    checks and groups, on the host: an entry whose directory, config or checkpoint (none for greedy, maxpressure,
    fixedtime and actuated) is
    missing is logged as an error and skipped (`skipped`); an `a2c` entry, or a simulator whose combined replicas exceed MAX_GROUP_REPLICAS, is refused
    with a ValueError naming the entry.  Entries whose simulators would be built identically (sim_key) share one
    simulator, len(seeds) consecutive replicas per entry, and run() evaluates each simulator's entries as one `_Group`
    (one launch per forward family and control step).  The greedy and maxpressure launches write every row of their
    simulator, and a fixed-time or actuated program governs every replica of its simulator, so entries of these
    controllers, which would otherwise share one, get a simulator each (fixedtime or actuated entries of one program
    share one; for actuated entries the program includes the loop tables).
    Each entry's reward trace, frames and summary are those `Evaluator` gives for its directory alone: member k samples
    with its own [ENV_CONFIG] seed and member-local replica index, ma2c members their own coop_gamma
    (tsc_set_replica_coop_gamma).

    `share_demand`: entries whose simulators differ only in their demand tables (sim_key(demand=True)) share one
    simulator too, each still at its own config's demand (tsc_set_replica_demand).  `demand_levels`: a list of
    {[ENV_CONFIG] key: value} demand overrides (keys of the entry scenario's envs.DEMAND_KEYS; a key a level does not
    name keeps the entry's value); implies share_demand.  Every entry is then evaluated at every level, as one member
    per (entry, level) pair, and the output path of an entry is a list with one path per level.  `entries` (and
    `groups`) then hold one GroupEntry per pair, with `demand` set to its level."""

    def __init__(self, entries, seeds, policy_type='default', policy='lstm', device=0, max_replicas=MAX_GROUP_REPLICAS,
                 share_demand=False, demand_levels=None):
        import configparser
        import glob
        import os
        from ..envs import check_demand_tables, demand_keys, make_env
        if policy_type not in ('default', 'stochastic', 'deterministic'):
            raise ValueError("policy_type must be 'default', 'stochastic' or 'deterministic' (got %r)" % (policy_type,))
        self.seeds = [int(s) for s in seeds]
        if not self.seeds:
            raise ValueError('GroupEvaluator: no evaluation seeds')
        self.policy_type, self.policy, self.device = policy_type, policy, device
        levels = None if demand_levels is None else [dict((str(k), str(v)) for k, v in lv.items()) for lv in demand_levels]
        if levels is not None and not levels:
            raise ValueError('GroupEvaluator: demand_levels is an empty list')
        self.share_demand = bool(share_demand) or levels is not None
        if levels is None:
            self.entries = [GroupEntry(d, m, o) for d, m, o in entries]
        else:
            self.entries = []
            for d, m, o in entries:
                if isinstance(o, str) or len(o) != len(levels):
                    raise ValueError('%s: with %d demand levels, the output path is a list of %d paths'
                                     % (d, len(levels), len(levels)))
                self.entries += [GroupEntry(d, m, oj, demand=lv) for oj, lv in zip(o, levels)]
        for e in self.entries:
            if e.model == 'a2c':
                raise ValueError('%s: %s' % (e.label, NO_A2C))
        self.skipped = []
        for e in self.entries:
            inis = sorted(glob.glob(os.path.join(e.agent_dir, 'data', '*.ini')))
            if not os.path.isdir(e.agent_dir):
                e.error = 'no agent directory %s' % e.agent_dir
            elif not inis:
                e.error = 'no config under %s/data/' % e.agent_dir
            elif e.model not in CONTROLLERS and not find_checkpoint(os.path.join(e.agent_dir, 'model')):
                e.error = 'no checkpoint under %s/model/' % e.agent_dir
            if e.error:
                logging.error('%s: %s, skipped' % (e.label, e.error))
                self.skipped.append(e)
                continue
            e.config = configparser.ConfigParser()
            e.config.read(inis[0])
            cfg = e.config['ENV_CONFIG']
            cfg['test_seeds'] = ','.join(str(s) for s in self.seeds)
            cfg['agent'] = e.agent
            e.seed = cfg.getint('seed')
            if e.demand is not None:
                allowed = demand_keys(cfg)
                for key in e.demand:
                    if key not in allowed:
                        raise ValueError('%s: %r is not a demand key of its scenario %r (demand keys: %s)'
                                         % (e.label, key, cfg.get('scenario'), ', '.join(allowed) or 'none'))
                own = make_env(cfg, len(self.seeds), e.output_path, device=device)._tables
                for key, v in e.demand.items():
                    cfg[key] = v
                e.env = make_env(cfg, len(self.seeds), e.output_path, device=device)
                check_demand_tables(own, e.env._tables, e.label, ignore=())
                continue
            e.env = make_env(cfg, len(self.seeds), e.output_path, device=device)
        self.groups = []                                 # [[entry, ...]] per shared simulator, in entry order
        keys = []
        for e in self.entries:
            if e.error:
                continue
            k = (sim_key(e.env, demand=self.share_demand), e.model if e.model in CONTROLLERS else '',
                 _program_key(e.env, e.model))
            if k in keys:
                self.groups[keys.index(k)].append(e)
            else:
                keys.append(k)
                self.groups.append([e])
        for g in self.groups:
            if len(g) * len(self.seeds) > max_replicas:
                raise ValueError('%s: the %d entries sharing its simulator need %d replicas (%d seeds each), more than '
                                 '%d' % (g[-1].label, len(g), len(g) * len(self.seeds), len(self.seeds), max_replicas))

    # ---- device work ----------------------------------------------------------------------------------------------
    def run(self):
        """Every group, one after another; then each entry's CSVs and summary when its env records.  Returns the entries
        that were evaluated."""
        done = []
        for g in self.groups:
            done += self._run_group(g)
        return done

    def _run_group(self, entries):
        models = [build_model(e.model, e.agent_dir, e.env, e.config, self.policy, self.device) for e in entries]
        grp = _Group([e.env for e in entries], models, [e.seed for e in entries], [e.label for e in entries],
                     self.policy_type, device=self.device, share_demand=self.share_demand)
        grp.episode()
        failed = grp.failed()
        done = []
        for k, (mean, std) in enumerate(grp.rewards()):
            e = entries[grp.order[k]]
            if k in failed:
                e.error = failed[k]
                logging.error('%s: %s' % (e.label, e.error))
                continue
            e.mean, e.std = mean, std
            for i in range(grp.S):
                logging.info('%s: test %i, avg reward %.2f' % (e.label, i, e.mean[i]))
            e.env.cur_episode = grp.S
            traffic = trip = None
            if grp.record:
                e.recorded = grp.output_data(k, e.output_path)
                _, traffic, trip = e.recorded
            e.summary = episode_summary(e.env, self.policy_type, e.mean, e.std, traffic, trip)
            done.append(e)
        return done


def _layout_key(lay):
    return tuple((k, _frozen(v)) for k, v in sorted(vars(lay).items())
                 if isinstance(v, (int, float, bool, str, list, tuple, np.ndarray)))


def _program_key(env, model):
    """Fixed-time and actuated entries share a simulator only when they run the same program (None for the other
    models)."""
    if model == 'actuated':
        from ..envs.actuated import env_program as actuated_program
        return actuated_program(env).key()
    if model != 'fixedtime':
        return None
    from ..envs.fixedtime import env_program, program_key
    return program_key(env_program(env))


def forward_family(model, net, label):
    """The forward family of `model` on a simulator of the net tables `net`, read from the model alone; members of one
    family share each control step's launch.  (name,) for the controllers; ('q', layout key) for IQL; ('v2', layout
    key) for IA2C / MA2C on the fused tensor-core forward; ('v1', id) and ('fc', id) for the A2C forwards that serve one
    member per launch.  Raises a ValueError naming `label` for a model without a batched evaluation path, or whose
    observation layout differs from the net's."""
    from .layout import QLayout
    name = getattr(model, 'name', None)
    if name in CONTROLLERS:
        return (name,)
    off = np.asarray(net.node_obs_off)
    if name == 'iql':
        n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
        if list(model.n_s_ls) != n_s or list(model.n_a_ls) != [int(a) for a in net.n_a_ls]:
            raise ValueError("%s: the model's observation layout differs from the env's (IQL n_s %s / n_a %s, env "
                             "observation widths %s / n_a %s)" % (label, list(model.n_s_ls), list(model.n_a_ls), n_s,
                                                                  list(net.n_a_ls)))
        return ('q', _layout_key(QLayout.from_iql(model, off, net.n_obs, max_na=net.max_na)))
    b = getattr(model, 'batched', None)
    if b is None or name not in ('ia2c', 'ma2c'):
        raise ValueError("%s: batched evaluation covers the greedy, max-pressure, fixed-time and actuated controllers, "
                         "IA2C / MA2C and IQL; %r stays on the one-replica protocol" % (label, name))
    L = b.lay
    if L.n_obs != net.n_obs or not np.array_equal(L.obs_off, off[:L.A]):
        raise ValueError("%s: the model's observation layout differs from the env's (build the model with "
                         "obs_off=env node_obs_off)" % label)
    if not L.recurrent:
        return ('fc', id(model))
    if not b.use_tc:
        raise ValueError("%s: the fp32 twin forward (use_tc=False) has no batched evaluation path; evaluate the "
                         "tensor-core model" % label)
    if b.paths.forward == 'v2':
        return ('v2', _layout_key(L))
    return ('v1', id(model))


class _Group:
    """One simulator and the forwards of its members.  Member k (`models[k]`, `envs[k]`, sampling seed `seeds[k]`,
    `labels[k]` naming it in errors) plays its env's S test seeds; the members are kept in row order (`order[p]`: the
    index of the member at position p), sorted by forward family so that each launch covers consecutive rows, the
    member at position p on replicas p * S .. (p + 1) * S - 1.  `sim`: the simulator to run on (K * S replicas), or None
    to build one.  ma2c members that differ in coop_gamma take it per replica, and with `share_demand` members that
    differ in their demand tables take their own per replica.  Every per-member result below is indexed by position."""

    def __init__(self, envs, models, seeds, labels, policy_type, sim=None, device=0, share_demand=False):
        from ..sim import BatchedSim
        fam = [forward_family(m, envs[0]._tables, lab) for m, lab in zip(models, labels)]
        self.order = sorted(range(len(models)), key=lambda k: (fam.index(fam[k]), k))
        self.envs = [envs[k] for k in self.order]
        self.models = [models[k] for k in self.order]
        self.seeds = [seeds[k] for k in self.order]
        self.policy_type = policy_type
        K, S = len(models), len(envs[0].test_seeds)
        self.K, self.S, self.R = K, S, K * S
        self.ma2c = self.models[0].name == 'ma2c'
        cg = [e.coop_gamma for e in self.envs] if self.ma2c else None
        env = self.envs[0]
        if cg is not None and len(set(cg)) > 1:
            # the simulator marks the observation entries it scales only when built with a coop_gamma other than 1
            env = next((e for e in self.envs if e.coop_gamma != 1.0), env)
        else:
            cg = None
        self.sim = sim = BatchedSim(env._tables, env._params, self.R, device=device) if sim is None else sim
        if cg is not None:
            sim.set_replica_coop_gamma(np.repeat(np.asarray(cg, np.float32), S))
        if share_demand:
            # members that differ in their demand tables: each member's replicas take its own (identical ones once)
            from ..net.tables import DEMAND_FIELDS
            nets = [e._tables for e in self.envs]
            if any(not np.array_equal(getattr(t, f), getattr(env._tables, f)) for t in nets for f in DEMAND_FIELDS):
                sim.set_replica_demand(nets, np.repeat(np.arange(K), S))
        self.dev = sim.device
        net = env._tables
        self.N, self.n_obs, self.max_na = net.n_nodes, net.n_obs, net.max_na
        self.T, self.ci = int(env.T), int(env.control_interval_sec)
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.obs = torch.zeros(self.R, self.n_obs, **f32)
        self.act = torch.zeros(self.R, self.N, dtype=torch.int32, device=self.dev)
        self.reward = torch.zeros(self.R, self.N, **f32)
        self.done = torch.zeros(self.R, dtype=torch.uint8, device=self.dev)
        self.trace = torch.zeros(self.T, self.R, **f32)
        self.pi = torch.zeros(self.R, self.N, self.max_na, **f32)
        self.stats = self.act_trace = None
        self.record = False
        self.fwd = []                 # (kind, state) per forward family, in row order
        for f, ps in itertools.groupby(range(K), key=lambda p: fam[self.order[p]]):
            ps = list(ps)
            self._add_forward(f[0], ps[0], ps[-1] + 1)
        if self.ma2c:
            u = torch.zeros(self.R, self.N, self.max_na, **f32)
            for a, na in enumerate(net.n_a_ls):
                u[:, a, :na] = 1.0 / int(na)                          # envs/env.py:263-269
            self.fp0 = u

    def _rows(self, i, j):
        S = self.S
        return torch.tensor([(k - i) * S for k in range(i, j + 1)], dtype=torch.int64, device=self.dev)

    def _seeds(self, i, j):
        return torch.tensor(np.array(self.seeds[i:j], dtype=np.uint64).view(np.int64), dtype=torch.int64,
                            device=self.dev)

    def _add_forward(self, kind, i, j):
        """The buffers of the family of the members at positions i .. j - 1; the parameters are read per episode."""
        from .layout import QLayout
        lib, S, f32 = _lib.lib(), self.S, dict(dtype=torch.float32, device=self.dev)
        n, r0 = (j - i) * S, i * S
        st = dict(i=i, j=j, n=n, obs=self.obs[r0:r0 + n], pi=self.pi[r0:r0 + n], act=self.act[r0:r0 + n])
        m0 = self.models[i]
        if kind == 'greedy':
            prog = m0.greedy_program(self.envs[i]._tables.node_obs_off)
            max_cand, off, idx, act = (int(prog[0]),) + tuple(np.ascontiguousarray(a, np.int32) for a in prog[1:])
            _lib.check(lib.tsc_set_greedy_program(
                self.sim._h, max_cand, off.ctypes.data, idx.ctypes.data, act.ctypes.data))
        elif kind == 'actuated':
            self.sim.set_actuated_program(m0.program)
        elif kind == 'q':
            qlay = QLayout.from_iql(m0, np.asarray(self.envs[i]._tables.node_obs_off), self.n_obs, max_na=self.max_na)
            h = C.c_void_p()
            _lib.check(lib.tscl_q_create(C.byref(qlay.as_c()), self.dev.index or 0, C.byref(h)))
            st.update(h=h, qlay=qlay, rows=self._rows(i, j), seeds=self._seeds(i, j),
                      params=torch.zeros(j - i, qlay.n_params, **f32), q=torch.zeros(n, self.N, self.max_na, **f32),
                      bad=torch.full((j - i,), -1, dtype=torch.int64, device=self.dev))
        elif kind == 'v2':
            b0, L = m0.batched, m0.batched.lay
            st.update(b=b0, rows=self._rows(i, j), seeds=self._seeds(i, j),
                      P=b0.P.new_empty((j - i,) + tuple(b0.P.shape)), Wp=b0.Wp.new_empty((j - i,) + tuple(b0.Wp.shape)),
                      c=torch.zeros(L.A, n, L.h, **f32), h=torch.zeros(L.A, n, L.h, **f32))
        elif kind in ('v1', 'fc'):                      # one member, its own launches on its own parameters
            b, L = m0.batched, m0.batched.lay
            st.update(b=b, val=torch.zeros(n, L.A, **f32))
            if kind == 'v1':
                st.update(c=torch.zeros(L.U, n, L.h, **f32), h=torch.zeros(L.U, n, L.h, **f32))
            else:
                st.update(X=torch.empty(L.U, n, L.dx, **f32), H=torch.empty(L.U, n, L.h, **f32))
        self.fwd.append((kind, st))

    def __del__(self):
        for kind, st in getattr(self, 'fwd', []):
            if kind == 'q' and st['h'].value:
                _lib.lib().tscl_q_destroy(st['h'])
                st['h'] = C.c_void_p()

    def _set_programs(self, programs, i):
        """The fixed-time family's programs, one per member from position i on: set_signal_program when they are all
        the same program, else plan p on the replicas of position i + p (set_replica_signal_programs)."""
        from ..envs.fixedtime import program_key
        if len(set(program_key(p) for p in programs)) == 1:
            self.sim.set_signal_program(programs[0])
            return
        plan = np.zeros(self.R, np.int64)
        for p in range(len(programs)):
            plan[(i + p) * self.S:(i + p + 1) * self.S] = p
        self.sim.set_replica_signal_programs(programs, plan)

    def _actions(self, t, stream):
        lib, done, stp = _lib.lib(), 1 if t == 0 else 0, t
        argmax = self.policy_type == 'deterministic'
        for kind, st in self.fwd:
            n, obs, pi, act = st['n'], st['obs'], st['pi'], st['act']
            if kind == 'greedy':
                _lib.check(lib.tsc_greedy_actions(self.sim._h, _p(self.obs), _p(self.act), stream))
            elif kind == 'maxpressure':
                _lib.check(lib.tsc_pressure_actions(self.sim._h, _p(self.act), stream))
            elif kind == 'q':
                _lib.check(lib.tscl_q_step_g(st['h'], _p(st['params']), st['qlay'].n_params, _p(obs), st['j'] - st['i'],
                                             _p(st['rows']), n, _p(st['q']), _p(act),
                                             int(self.policy_type == 'stochastic'), _p(st['seeds']), stp,
                                             _p(st['bad']), stream))
            elif kind == 'v2':
                b = st['b']
                _lib.check(lib.tscl_policy_step_pi_g(
                    b._h, _p(st['P']), st['P'].shape[1], _p(st['Wp']), st['Wp'][0].numel(), _p(obs), st['j'] - st['i'],
                    _p(st['rows']), n, _p(st['c']), _p(st['h']), _p(st['c']), _p(st['h']), _p(pi), _p(act),
                    int(argmax), done, _p(st['seeds']), stp, stream))
            elif kind in ('v1', 'fc'):
                b, seed = st['b'], self.seeds[st['i']]
                a = None if argmax else _p(act)
                if kind == 'v1':
                    _lib.check(lib.tscl_policy_step(b._h, _p(b.P), _p(b.Wp), _p(obs), n, _p(st['c']), _p(st['h']),
                                                    _p(st['c']), _p(st['h']), _p(pi), _p(st['val']), a, done, seed, stp,
                                                    0, None, 0, stream))
                else:
                    _lib.check(lib.tscl_fc_embed(b._h, _p(b.P), _p(obs), n, n, 0, _p(st['X']), stream))
                    _lib.check(lib.tscl_fc_hidden_fwd(b._h, _p(b.P), _p(st['X']), n, _p(st['H']), stream))
                    _lib.check(lib.tscl_heads(b._h, _p(b.P), _p(st['H']), n, _p(pi), _p(st['val']), a, seed, stp, 0,
                                              stream))
                if argmax:
                    _lib.check(lib.tscl_argmax_actions(b._h, _p(pi), n, _p(act), stream))

    def episode(self):
        """One episode of every member on its test seeds: the members' current parameters, then the reward trace and,
        when every member's env records, the per-second statistics and the recorded actions."""
        sim, lib, stream = self.sim, _lib.lib(), _lib.stream(self.dev)
        self.record = all(e.is_record for e in self.envs)
        sim.reset(np.tile(replica_seeds(self.envs[0]), self.K))
        sim.set_train_mode(False)
        if self.record:
            sim.set_record(True)
            self.stats = torch.zeros(self.T, self.R, self.ci, 8, dtype=torch.float32, device=self.dev)
            self.act_trace = torch.zeros(self.T, self.R, self.N, dtype=torch.int32, device=self.dev)
        for kind, st in self.fwd:
            members = self.models[st['i']:st['j']]
            if kind == 'v2':
                for k, m in enumerate(members):
                    st['P'][k].copy_(m.batched.P)
                    st['Wp'][k].copy_(m.batched.Wp)
            elif kind == 'q':
                for k, m in enumerate(members):
                    st['params'][k].copy_(st['qlay'].pack(m.nets))
                st['bad'].fill_(-1)
            elif kind == 'fixedtime':
                self._set_programs([m.program for m in members], st['i'])
            if kind in ('v1', 'v2'):
                st['c'].zero_(); st['h'].zero_()
        fp = self.fp0 if self.ma2c else None
        sim.observe(fp, obs_out=self.obs)
        act = None if self.fwd[0][0] in PROGRAMS else self.act
        fp = self.pi if self.ma2c else None
        for t in range(self.T):
            self._actions(t, stream)
            if self.record:
                _lib.check(lib.tsc_step_record(sim._h, _p(act), _p(fp), _p(self.obs), _p(self.reward),
                                               _p(self.trace[t]), _p(self.done), _p(self.stats[t]), stream))
                _lib.check(lib.tsc_get_counts(sim._h, None, None, None, _p(self.act_trace[t]), stream))
            else:
                _lib.check(lib.tsc_step(sim._h, _p(act), _p(fp), _p(self.obs), _p(self.reward), _p(self.trace[t]),
                                        _p(self.done), stream))
        for e in self.envs:
            e.cur_sec = self.T * self.ci

    def failed(self):
        """{position: message} for the IQL members whose stochastic sample met a q that is not a distribution in the last
        episode: the ValueError np.random.choice raises in the reference."""
        out = {}
        if self.policy_type != 'stochastic':
            return out
        for kind, st in self.fwd:
            if kind != 'q':
                continue
            for k, key in enumerate(st['bad'].cpu().numpy().tolist()):
                if key != -1:
                    r, step, agent = key >> 40, (key >> 16) & 0xFFFFFF, key & 0xFFFF
                    out[st['i'] + k] = ('probabilities are not non-negative: q / sum(q) of agent %d at control step %d '
                                        'of test episode %d (seed %d)'
                                        % (agent, step, r, int(self.envs[st['i'] + k].test_seeds[r])))
        return out

    def rewards(self):
        """Per position, (mean [S], std [S]) float64 of the last episode: np.mean / np.std of each replica's per-step
        global rewards (utils.py:230-234)."""
        tr, S = self.trace.cpu().numpy(), self.S
        out = []
        for k in range(self.K):
            cols = [np.array(tr[:, r], dtype=np.float64) for r in range(k * S, (k + 1) * S)]
            out.append((np.array([np.mean(c) for c in cols]), np.array([np.std(c) for c in cols])))
        return out

    def frames(self, k):
        """(control, traffic, trip) DataFrames of the member at position k in the last recorded episode."""
        S, T = self.S, self.T
        rows = slice(k * S, (k + 1) * S)
        control = control_frame(self.act_trace[:, rows].permute(1, 0, 2).cpu().numpy(),
                                self.trace[:, rows].t().cpu().numpy(), self.ci)
        traffic = traffic_frame(self.stats[:, rows].permute(1, 0, 2, 3).reshape(S, T * self.ci, 8).cpu().numpy())
        trip = trip_frame([self.sim.trips(r) for r in range(rows.start, rows.stop)])
        return control, traffic, trip

    def output_data(self, k, output_path):
        """The reference's three CSVs (envs/env.py output_data) of the member at position k:
        <output_path><scenario>_<agent>_{control,traffic,trip}.csv.  Returns the frames."""
        frames = self.frames(k)
        env = self.envs[k]
        base = output_path + ('%s_%s_' % (env.name, env.agent))
        for kind, frame in zip(('control', 'traffic', 'trip'), frames):
            frame.to_csv(base + kind + '.csv')
        return frames
