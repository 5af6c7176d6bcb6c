"""`train`: the reference's `main.py train` (main.py:82-155) with its `utils.py:Counter` / `Trainer.run`
(utils.py:70-108, 255-308), for R lock-stepped replicas on the device.

    train(config, base_dir, test_mode='no_test', n_replicas=1, policy='lstm', device=0, process_group=None,
          summaries=False)
    train_population(config, base_dir, seeds, ...) / train_sweep([a.ini, b.ini, ...], base_dir, ...)   (ia2c / ma2c
                                                        members, one per seed or config, in one process)
    train_iql_population(config, base_dir, seeds, ...) / train_iql_sweep([a.ini, ...], base_dir, ...)   (the same for
                                                        iqll / iqld)

The four member fronts refuse what they cannot train and then run one members driver (`_train_members`), built from
the solo run's parts: the same trainer construction (`_trainer`), summary set-up (`_summaries`) and log set-up
(`init_log`).

leaves the reference's agent directory: `data/` with a copy of the config and `train_reward.csv`, `model/checkpoint-<step>`
and `log/<time>.log`; with `after_train_test` / `all_test` also `data/<scenario>_<agent>_{control,traffic,trip}.csv`;
with `summaries` also the TensorBoard event file `log/events.out.tfevents.<time>.<host>` (`Summaries`).
`scripts/evaluate.py --agent-dir base_dir` reads that directory back.

With a `process_group` of W ranks, one agent trains on `n_replicas` replicas in all: rank k steps the global replicas
[k*R/W, (k+1)*R/W) on its device, and the learner all-reduces its gradient once per update (A2C) or per round (IQL).
Seeds, actions and replay draws are keyed by the global replica, so a run over W ranks plays the episodes of the
one-process run with the same n_replicas; only the order in which the gradient is summed differs.  Rank 0 owns every
file and runs every test; the other ranks write nothing under base_dir and log WARNING and above to stderr.

Protocol (the reference's, applied to R replicas):
* the global step counts control steps of the lock-step: one episode of all replicas advances it by T, so a run of
  `total_step` makes as many updates as the reference's one-environment run, each on R times the data;
* before every episode set: a test when `in_train_test` and `cur_step - last_test_step >= test_interval`; the run stops
  when `cur_step >= total_step`, checked only between episodes;
* one `train_reward.csv` row per episode set (test_id -1): avg_reward = mean and std_reward = np.std of the per-step
  global reward pooled over every replica and step; one row per test seed (test_id k) with that seed's mean / std.
  Over W > 1 ranks rank 0 gathers the [T, R] trace of all global replicas first (`training_row`).
The training loop itself is `BatchedTrainer` / `BatchedIQLTrainer`; the tests run on the batched `Evaluator` over an
env of its own (`ENV_CONFIG.test_seeds`, test mode, policy_type 'default'), which reads the learner's live weights on
the device and leaves the training sim and the learner's recurrent state alone.
"""
from __future__ import annotations

import configparser
import copy
import hashlib
import json
import logging
import os
import shutil
import time
import types

import numpy as np

from .. import dist as _dist

TEST_MODES = ('no_test', 'in_train_test', 'after_train_test', 'all_test')


def init_dir(base_dir, pathes=('log', 'data', 'model')):
    """utils.py:30-39: {name: '<base_dir>/<name>/'}, created when missing."""
    dirs = {}
    for path in pathes:
        dirs[path] = os.path.join(base_dir, path) + os.sep
        os.makedirs(dirs[path], exist_ok=True)
    return dirs


def init_log(log_dirs):
    """utils.py:42-48: INFO records to `<log_dir>/<time>.log` of every directory in `log_dirs` and to stderr.  File k
    takes the records of member k (`extra={'member': k}`, a population's) and those of no member in particular, so one
    directory takes every record.  The handlers are added to the root logger and returned, so that a caller that trains
    more than once in a process can remove them."""
    fmt = logging.Formatter('%(asctime)s [%(levelname)s] %(message)s')
    handlers = []
    for k, d in enumerate(log_dirs):
        handlers.append(logging.FileHandler(os.path.join(d, '%d.log' % time.time())))
        handlers[-1].addFilter(lambda rec, k=k: getattr(rec, 'member', k) == k)
    handlers.append(logging.StreamHandler())
    root = logging.getLogger()
    for h in handlers:
        h.setFormatter(fmt)
        root.addHandler(h)
    root.setLevel(logging.INFO)
    return handlers


def init_rank_log(rank):
    """A rank other than 0 writes no log file: WARNING records and above go to stderr, prefixed with the rank."""
    h = logging.StreamHandler()
    h.setLevel(logging.WARNING)
    h.setFormatter(logging.Formatter('[rank %d] %%(asctime)s [%%(levelname)s] %%(message)s' % rank))
    logging.getLogger().addHandler(h)
    return [h]


def init_test_flag(test_mode):
    """utils.py:51-60: (in-training tests, post-training test)."""
    if test_mode not in TEST_MODES:
        raise ValueError('test_mode must be one of %s (got %r)' % (', '.join(TEST_MODES), test_mode))
    return test_mode in ('in_train_test', 'all_test'), test_mode in ('after_train_test', 'all_test')


def model_spec(agent):
    """main.py:110-121: ('ia2c' | 'ma2c', None) for the A2C agents, ('iql', 'dqn') for iqld and ('iql', 'lr') for every
    other name.  greedy, fixedtime and actuated have nothing to train; the centralised a2c (a joint action space of
    prod(n_a) actions) has no batched learner."""
    if agent in ('greedy', 'fixedtime', 'actuated'):
        raise ValueError("agent %r has no model to train" % agent)
    if agent == 'a2c':
        raise ValueError("agent 'a2c' (the centralised A2C) has no batched learner; train ia2c, ma2c or an IQL agent")
    if agent in ('ia2c', 'ma2c'):
        return agent, None
    return 'iql', 'dqn' if agent == 'iqld' else 'lr'


class Counter:
    """utils.py:70-107 with the step advanced by one episode set at a time."""

    def __init__(self, total_step, test_step, log_step):
        self.cur_step = 0
        self.cur_test_step = 0
        self.total_step, self.test_step, self.log_step = total_step, test_step, log_step

    def next(self, n_step):
        self.cur_step += n_step
        return self.cur_step

    def should_test(self):
        if self.cur_step - self.cur_test_step >= self.test_step:
            self.cur_test_step = self.cur_step
            return True
        return False

    def should_log(self, prev_step):
        """A multiple of log_interval lies in (prev_step, cur_step]: the reference logs at `cur_step % log_step == 0`
        and the step advances by T here."""
        return self.log_step > 0 and prev_step // self.log_step < self.cur_step // self.log_step

    def should_stop(self):
        return self.cur_step >= self.total_step


class Summaries:
    """The reference's TensorBoard log of a training run (utils.py:129-140, 255-306; agents/policies.py:62-72, 331-338):
    agent 0's scalars of every update (A2C: policy / value / total loss and gradient norm at the step of the backward,
    and with a teacher the imitation loss;
    IQL: loss, mean q, mean target and gradient norm of round k at that step + k), `train_reward` once per episode set
    (the training row's avg_reward, at the step of its last update) and `test_reward` once per in-training test (the
    mean over test seeds of the per-seed means, at the step of the test).

    The learners keep each update's record on the device (the trainers' `summary_rec`); the driver reads it once per
    episode set, where it reads the reward trace, and writes that set's events then (wall_time: the time of writing).
    Over W > 1 ranks the A2C loss terms are each rank's partial sums, so rank 0 adds them over the ranks
    (`dist.sum_partials`); the gradient norms and the IQL records are global after the gradient all-reduce.  `writer` is
    the SummaryWriter on rank 0 and None on the other ranks, which only take part in the sums."""

    def __init__(self, writer, name, kind, n_step):
        self.writer, self.name, self.kind, self.n_step = writer, name, kind, int(n_step)

    def record(self, trainer, group=None):
        """This episode set's records on rank 0 (A2C [n_updates, 4], IQL agent 0's [n_updates, rounds, 4]), None on
        the other ranks; every rank of `group` must call it."""
        if self.kind == 'iql':
            return None if self.writer is None else trainer.summary_rec[:, :, 0, :].cpu().numpy()
        rec = trainer.summary_rec.cpu().numpy()
        if group is not None:
            cols = [0, 1, 2] + ([4] if rec.shape[1] > 4 else [])      # loss terms (with a teacher also imitation)
            loss = _dist.sum_partials(rec[:, cols], group)
            if loss is None:
                return None
            rec = rec.astype(np.float64)
            rec[:, cols] = loss
        return rec

    def episode_set(self, rec, ran, prev_step, step, train_reward):
        from .summary import a2c_events, iql_events
        first = prev_step + self.n_step
        events = iql_events(self.name, rec, ran, first, self.n_step) if self.kind == 'iql' else \
            a2c_events(self.name, rec, first, self.n_step)
        now = time.time()
        for st, values in events:
            self.writer.add_scalars(values, st, now)
        self.writer.add_scalar('train_reward', train_reward, step, now)
        self.writer.flush()

    def test_reward(self, value, step):
        self.writer.add_scalar('test_reward', value, step)
        self.writer.flush()


def training_row(rewards):
    """(avg_reward, std_reward) of a training row over W > 1 ranks from the gathered [T, R_total] trace: the float64
    mean over global replicas of each replica's episode mean, and np.std of the very array a one-process run holds.
    avg_reward can differ in the last bits from the one-process row, which takes the trainer's float32
    `episode_rewards[-1]`."""
    rewards = np.asarray(rewards, np.float64)
    return float(rewards.mean(axis=0).mean()), float(np.std(rewards))


# data/train_reward_demand.csv of a run on a mixture of demand levels: train_reward.csv's columns and the level's label
DEMAND_ROW_COLUMNS = ('agent', 'step', 'test_id', 'demand', 'avg_reward', 'std_reward')


class Trainer:
    """utils.py:Trainer.run / Tester.run_offline over a batched trainer (`run(n)`, `T_episode`, `episode_rewards`,
    `greward_trace` [T_episode, R]) and a batched `Evaluator` (`perform_all()`, `run()`, `env`).

    `group`: None for one process; over W > 1 ranks a group that takes CPU tensors (gloo).  Every rank then runs the
    same schedule; rank 0 gathers the traces, holds the rows, runs the tests (only it has an evaluator) and writes the
    CSV, and all ranks meet at a barrier after each test.
    `summary`: None, or the `Summaries` of the run (the trainer then keeps a `summary_rec`).
    `log_extra`: the `extra` of its log records (a population member's tag, see `train_population`).
    `levels`: a run on a mixture of L demand levels (`demand_mix_levels`), a list of (label, evaluator at that level or
    None); global replica g runs at level g mod L.  The driver then also keeps `level_data`, the rows of
    `train_reward_demand.csv`: per episode set one training row per level (`training_row` over that level's columns of
    the [T, R_total] trace), per test one row per level and seed, and the post-training test writes each level's CSVs
    into <output_path>/<label>/.
    `run_schedule` runs one schedule for several drivers that share a batched trainer and counter."""

    def __init__(self, trainer, evaluator, counter: Counter, agent: str, run_test: bool, output_path: str,
                 group=None, summary=None, log_extra=None, levels=None):
        if trainer.greward_trace is None:
            raise ValueError('the driver needs the trainer to keep a greward_trace')
        self.trainer, self.evaluator, self.counter = trainer, evaluator, counter
        self.agent, self.run_test, self.output_path = agent, run_test, output_path
        self.group, self.summary = group, summary
        self.levels, self.level_data, self.level_post = levels, [], None
        self.log_extra = dict(log_extra or {})
        if group is None:
            self.rank0 = True
        else:
            import torch.distributed as dist
            self.rank0 = dist.get_rank(group) == 0
        self.T = int(trainer.T_episode)
        self.data = []
        self.n_episode_sets = 0
        if run_test and self.rank0:
            logging.info('Testing: total test num: %d' % evaluator.test_num, extra=self.log_extra)

    def _barrier(self):
        if self.group is not None:
            import torch.distributed as dist
            dist.barrier(group=self.group)

    def test(self):
        if self.rank0:
            step = self.counter.cur_step
            t0 = time.time()
            mean, std = self.evaluator.perform_all()
            for k in range(len(mean)):
                self.data.append({'agent': self.agent, 'step': step, 'test_id': k, 'avg_reward': float(mean[k]),
                                  'std_reward': float(std[k])})
            logging.info('Testing: global step %d, avg R: %.2f (%.2f s)' % (step, np.mean(mean), time.time() - t0),
                         extra=self.log_extra)
            if self.summary is not None:
                self.summary.test_reward(float(np.mean(mean)), step)
            for label, ev in self.levels or ():
                t0 = time.time()
                mean, std = ev.perform_all()
                for k in range(len(mean)):
                    self.level_data.append({'agent': self.agent, 'step': step, 'test_id': k, 'demand': label,
                                            'avg_reward': float(mean[k]), 'std_reward': float(std[k])})
                logging.info('Testing: global step %d, demand %s, avg R: %.2f (%.2f s)'
                             % (step, label, np.mean(mean), time.time() - t0), extra=self.log_extra)
        self._barrier()

    def run(self):
        run_schedule([self])

    def episode_set(self, prev, step):
        """The training row (and the summaries) of the episode set that took the step from prev to step."""
        c = self.counter
        self.n_episode_sets += 1
        rec = self.summary.record(self.trainer, self.group) if self.summary is not None else None
        if self.group is None:
            rewards = np.asarray(self.trainer.greward_trace.cpu().numpy(), np.float64)
            mean, std = float(self.trainer.episode_rewards[-1]), float(np.std(rewards))
        else:
            rewards = _dist.gather_traces(self.trainer.greward_trace.cpu(), self.group)
            if rewards is None:
                return
            mean, std = training_row(rewards)
        self.data.append({'agent': self.agent, 'step': step, 'test_id': -1, 'avg_reward': mean, 'std_reward': std})
        if self.levels is not None:
            from .trainer import mix_level_of
            L = len(self.levels)
            level_of = mix_level_of(0, rewards.shape[1], L)
            for j, (label, _) in enumerate(self.levels):
                m, s = training_row(rewards[:, level_of == j])
                self.level_data.append({'agent': self.agent, 'step': step, 'test_id': -1, 'demand': label,
                                        'avg_reward': m, 'std_reward': s})
        if self.summary is not None:
            self.summary.episode_set(rec, self.trainer.summary_ran, prev, step, mean)
        if c.should_log(prev):
            logging.info('Training: global step %d, episode set %d, avg R: %.2f, std R: %.2f'
                         % (step, self.n_episode_sets, mean, std), extra=self.log_extra)

    def write_rows(self):
        if self.rank0:
            import pandas as pd
            pd.DataFrame(self.data).to_csv(self.output_path + 'train_reward.csv')
            if self.levels is not None:
                pd.DataFrame(self.level_data, columns=DEMAND_ROW_COLUMNS).to_csv(
                    self.output_path + 'train_reward_demand.csv')

    def run_offline(self):
        """Tester.run_offline: every test seed in record mode, the three CSVs into output_path (and, on a mixture of
        demand levels, each level's into output_path/<label>/, its (mean, std) into `level_post`).  Returns the
        per-seed (mean, std) on rank 0, None on the other ranks."""
        out = None
        if self.rank0:
            self.evaluator.env.init_data(True, False, self.output_path)
            mean, std = self.evaluator.run()
            logging.info('Offline testing: avg R: %.2f' % np.mean(mean), extra=self.log_extra)
            out = mean, std
            if self.levels is not None:
                self.level_post = []
                for label, ev in self.levels:
                    path = os.path.join(self.output_path, label) + os.sep
                    os.makedirs(path, exist_ok=True)
                    ev.env.init_data(True, False, path)
                    self.level_post.append(ev.run())
                    logging.info('Offline testing: demand %s, avg R: %.2f' % (label, np.mean(self.level_post[-1][0])),
                                 extra=self.log_extra)
        self._barrier()
        return out


def run_schedule(drivers):
    """utils.py:Trainer.run for drivers that share one batched trainer and counter (drivers[0]'s): the tests before an
    episode set, one episode of every replica, then each driver's training row; finally each driver's CSV.  One driver
    is `Trainer.run`; a population has one driver per member, each over its member's view of the trainer."""
    d0 = drivers[0]
    c = d0.counter
    while not c.should_stop():
        if d0.run_test and c.should_test():
            for d in drivers:
                d.test()
        prev = c.cur_step
        d0.trainer.run(d0.T)                                          # one episode of every replica
        step = c.next(d0.T)
        for d in drivers:
            d.episode_set(prev, step)
    for d in drivers:
        d.write_rows()


def build_model(agent, env, model_config, total_step, n_replicas, policy='lstm', seed=0, device=0, replica0=0,
                total_replicas=None, process_group=None, seeds=None, member_configs=None, deterministic=False):
    """main.py:110-121 on the batched learners: IA2C / MA2C wrappers (seed = ENV_CONFIG.seed) or BatchedIQL (seed 0).
    `n_replicas` are this rank's replicas, the global ones [replica0, replica0 + n_replicas) of `total_replicas`; the
    learner all-reduces its gradient over `process_group` when one is given.  `seeds`: an A2C population, one member
    per seed on n_replicas replicas each (`BatchedA2C`); with `member_configs` (one [MODEL_CONFIG] per seed) a sweep.
    `deterministic`: the A2C update adds in a fixed order (`BatchedA2C(deterministic=True)`); IQL's TD kernel already
    reduces in a fixed order, so for iqll / iqld it changes nothing.  For iqll / iqld, `seeds` and `member_configs`
    give a `BatchedIQL` with members (each with learner seed 0, as the solo run)."""
    kind, model_type = model_spec(agent)
    t = env._tables
    if kind != 'iql':
        from .models import IA2C, MA2C
        kw = dict(seed=seed, n_replicas=n_replicas, obs_off=t.node_obs_off, policy=policy, device=device)
        if process_group is not None:
            kw.update(replica0=replica0, total_replicas=total_replicas, process_group=process_group)
        if seeds is not None:
            kw.update(seeds=seeds)
        if member_configs is not None:
            kw.update(member_configs=member_configs)
        if deterministic:
            kw.update(deterministic=True)
        if kind == 'ma2c':
            return MA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, env.n_f_ls, total_step, model_config, **kw)
        return IA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, total_step, model_config, **kw)
    from .layout import QLayout
    from .learner_iql import BatchedIQL
    off = np.asarray(t.node_obs_off)
    n_fc = model_config.getint('num_fc', fallback=0) if model_type == 'dqn' else 0
    n_h = model_config.getint('num_h', fallback=0) if model_type == 'dqn' else 0
    lay = QLayout(model_type, [int(off[i + 1] - off[i]) for i in range(t.n_nodes)], t.n_a_ls, t.n_w_ls, off, t.n_obs,
                  n_fc=n_fc, n_ft=n_fc // 4, n_h=n_h, max_na=t.max_na)          # q_fct width: agents/policies.py:383
    return BatchedIQL(lay, n_replicas, model_config, model_type, seed=0, device=device, replica0=replica0,
                      total_replicas=total_replicas, pg=process_group, seeds=seeds, member_configs=member_configs)


def parse_seeds(text):
    """'12,13,14' -> [12, 13, 14]: the member seeds of a population run (distinct non-negative integers)."""
    try:
        seeds = [int(x) for x in str(text).split(',') if x.strip()]
    except ValueError:
        raise ValueError('seeds must be comma-separated integers (got %r)' % (text,))
    if not seeds:
        raise ValueError('no seed in %r' % (text,))
    if len(set(seeds)) != len(seeds):
        raise ValueError('population seeds must be distinct (got %s)' % seeds)
    if min(seeds) < 0:
        raise ValueError('population seeds must be non-negative (got %s)' % seeds)
    return seeds


def member_dir(base_dir, seed, agent):
    """The agent directory of the population member with `seed`: <base_dir>/seed<seed>/<agent>."""
    return os.path.join(base_dir, 'seed%d' % int(seed), agent)


def demand_mix_levels(config, demand_mix, n_replicas):
    """The L levels of a run on a mixture of demand levels, checked before any directory or device work: a namespace
    with `levels` (the {[ENV_CONFIG] key: value} dicts, in order), `labels` (envs.demand_label), `configs` (`config`
    edited to each level; a key a level leaves out keeps the config's value) and `nets` (each level's NetTables, built
    on the host).  Refused with a ValueError naming the level, key or count: no level, a scenario without demand keys,
    a key outside the scenario's envs.DEMAND_KEYS, a level that repeats another (same values of every demand key), a
    level whose net differs from the config's in more than its demand tables (`check_demand_tables`), and a replica
    count that is not a multiple of L (each level weighs the same in every gradient)."""
    from ..envs import check_demand_tables, demand_keys, demand_label, make_env
    levels = [dict((str(k), str(v)) for k, v in dict(lv).items()) for lv in demand_mix]
    if not levels:
        raise ValueError('demand_mix: a mixture needs at least one demand level')
    env_cfg = config['ENV_CONFIG']
    keys = demand_keys(env_cfg)
    if not keys:
        raise ValueError('demand_mix: the scenario %r has no demand keys, so it has no demand levels to mix'
                         % env_cfg.get('scenario'))
    labels = [demand_label(lv) for lv in levels]
    cfgs, values = [], []
    for j, lv in enumerate(levels):
        for key in lv:
            if key not in keys:
                raise ValueError('demand level %s: %r is not a demand key of the scenario %r (demand keys: %s)'
                                 % (labels[j], key, env_cfg.get('scenario'), ', '.join(keys)))
        c = copy.deepcopy(config)
        for key, v in lv.items():
            c['ENV_CONFIG'][key] = v
        vals = [c['ENV_CONFIG'].get(key, fallback=None) for key in keys]
        for i, prev in enumerate(values):
            if all(_same(a, b) for a, b in zip(prev, vals)):
                raise ValueError('demand level %s repeats level %s: a mixture takes each level once'
                                 % (labels[j], labels[i]))
        cfgs.append(c)
        values.append(vals)
    L = len(levels)
    if int(n_replicas) % L:
        raise ValueError('%d replicas do not split evenly over %d demand levels: n_replicas must be a multiple of %d'
                         % (int(n_replicas), L, L))
    base = make_env(env_cfg, 1, '', is_record=False)._tables
    nets = []
    for c, label in zip(cfgs, labels):
        nets.append(make_env(c['ENV_CONFIG'], 1, '', is_record=False)._tables)
        check_demand_tables(base, nets[-1], 'demand level %s' % label)
    return types.SimpleNamespace(levels=levels, labels=labels, configs=cfgs, nets=nets)


def train(config, base_dir, test_mode='no_test', n_replicas=1, policy='lstm', device=0, process_group=None,
          summaries=False, seeds=None, deterministic=False, demand_mix=None):
    """main.py train.  `config`: the path of a reference config (copied into data/) or a parsed ConfigParser (written
    to data/config.ini), with [ENV_CONFIG], [MODEL_CONFIG] and [TRAIN_CONFIG].  Returns a namespace with final_step,
    episode_sets, env_samples (= final_step * n_replicas), wall_sec, world, rank, data (the train_reward.csv rows),
    post_test (the per-seed (mean, std) of the post-training test or None), and the live model and trainer.

    `process_group`: None trains in this process alone.  A group of W > 1 ranks trains one agent on `n_replicas`
    replicas in all, R/W on each rank (W must divide n_replicas), on `device`; every rank of the group calls train()
    with the same arguments.  Rank 0 writes every file and runs every test; `data` and `post_test` are None on the
    other ranks.  The host-side gathers and barriers run on the group itself when its backend is gloo, else on a gloo
    group over the same ranks, which torch.distributed.new_group makes every process of the default group enter.

    The post-training test follows what the reference intends (main.py:147-150) rather than what its code does: its
    `Tester.__init__` calls `Trainer.__init__` without `run_test`, and `run_offline` is passed an argument it does not
    take, so both raise TypeError and the reference's after_train_test never runs.  Here the model is saved first, then
    every test seed is played once in record mode and the three CSVs go into data/.

    `summaries`: also write the reference's TensorBoard event file into log/ (`Summaries`; rank 0 only).  Off by default:
    the run then allocates, launches and writes nothing for it.

    `seeds`: train a population instead, one member per seed, each on `n_replicas` replicas, in one process
    (`train_population`).  Returns its namespace.

    `deterministic`: the A2C update adds its gradients, loss sums and clip norms in a fixed order
    (`BatchedA2C(deterministic=True)`), so two runs with the same config, seeds, replicas, world size, build and GPU
    model leave the same bits: checkpoint, CSVs and summaries.  The LSTM policy only (refused for policy='fc' before any
    directory is made); a no-op for IQL, whose update is already reproducible.

    `demand_mix`: train the one agent on a mixture of traffic demand levels, a list of L {[ENV_CONFIG] demand key:
    value} dicts (`demand_mix_levels` checks them, on every rank, before any directory or device work).  Global replica
    g runs at level g mod L (the config edited to that level; a key a level leaves out keeps the config's value), so
    n_replicas must be a multiple of L.  The directory holds what it holds without a mixture, with the same meaning:
    the config (at its own demand), train_reward.csv (training rows pooled over every replica, test rows at the
    config's demand), the checkpoint and the post-training CSVs.  Added: data/demand_mix.json (the levels and their
    labels), data/train_reward_demand.csv (`DEMAND_ROW_COLUMNS`: one training row per level and episode set, one row
    per level and seed per in-training test) and, with a post-training test, each level's three CSVs in
    data/<label>/.  Not with `seeds`."""
    if deterministic and policy != 'lstm':
        raise ValueError("deterministic=True needs the LSTM policy's lean update (got policy=%r)" % (policy,))
    cfg, path = _read_config(config)
    _check_imitation([cfg])
    mix = None
    if demand_mix is not None:
        if seeds is not None:
            raise ValueError('demand_mix trains one agent: it does not combine with seeds (a population)')
        mix = demand_mix_levels(cfg, demand_mix, n_replicas)
    if seeds is not None:
        if process_group is not None:
            raise ValueError('a population trains in one process: seeds and process_group exclude each other')
        return train_population(config, base_dir, seeds, test_mode, n_replicas, policy, device, summaries,
                                deterministic=deterministic)
    t0 = time.time()
    in_test, post_test = init_test_flag(test_mode)
    world, rank = 1, 0
    if process_group is not None:
        import torch.distributed as dist
        world, rank = dist.get_world_size(process_group), dist.get_rank(process_group)
    pg = process_group if world > 1 else None
    _dist.replica_range(rank, world, int(n_replicas))                 # every rank rejects an uneven split alike
    if rank == 0:
        dirs = init_dir(base_dir)
        handlers = init_log([dirs['log']])
    else:
        dirs = {k: os.path.join(base_dir, k) + os.sep for k in ('log', 'data', 'model')}
        handlers = init_rank_log(rank)
    try:
        if rank == 0:
            _save_config(dirs['data'], cfg, path)
            if mix is not None:
                with open(os.path.join(dirs['data'], 'demand_mix.json'), 'w') as f:
                    json.dump({'levels': mix.levels, 'labels': mix.labels}, f, indent=1)
        out = _train(cfg, dirs, in_test, post_test, int(n_replicas), policy, device, pg, bool(summaries),
                     bool(deterministic), mix)
    finally:
        for h in handlers:
            logging.getLogger().removeHandler(h)
            h.close()
    out.wall_sec = time.time() - t0
    return out


def host_group(pg):
    """The group of the driver's host-side gathers and barriers: `pg` itself when its backend is gloo, else a new gloo
    group over the same ranks.  Keeps them off the learner's NCCL stream and lets CPU tensors through."""
    import torch.distributed as dist
    if dist.get_backend(pg) == 'gloo':
        return pg, False
    return dist.new_group(ranks=dist.get_process_group_ranks(pg), backend='gloo'), True


def state_digest(model):
    """SHA-256 of the learner state every rank must hold bit for bit: the weights and the optimiser slots (RMSProp ms,
    or Adam m, v and step count)."""
    if model.name == 'iql':
        tensors, extra = (model.P, model.M, model.V), np.int64(model.t).tobytes()
    else:
        tensors, extra = (model.batched.P, model.batched.MS), b''
    h = hashlib.sha256(extra)
    for t in tensors:
        h.update(t.detach().cpu().numpy().tobytes())
    return h.digest()


def check_ranks_agree(model, group):
    """Raise on every rank unless all ranks of `group` (gloo) hold bit-identical learner state.  The ranks apply the
    same all-reduced gradient to the same weights, so a difference means one of them drifted."""
    import torch
    import torch.distributed as dist
    mine = torch.frombuffer(bytearray(state_digest(model)), dtype=torch.uint8)
    all_ = [torch.empty_like(mine) for _ in range(dist.get_world_size(group))]
    dist.all_gather(all_, mine, group=group)
    differ = [k for k, d in enumerate(all_) if not torch.equal(d, all_[0])]
    if differ:
        raise RuntimeError('the learner state of rank(s) %s differs from rank 0\'s: the ranks no longer train one '
                           'model' % differ)


def teacher_kwargs(model, env, sweep=False):
    """The `BatchedTrainer` arguments of a model with a teacher ({} without one): the imitation coefficient's schedule
    (one per member in a sweep) and, for the greedy teacher, the training env's greedy program: the greedy rule on the
    own-wave entries of the observation the student sees, normalised and clipped by the training config."""
    teacher = getattr(model, 'teacher', None)
    if not teacher:
        return {}
    kw = dict(imit=model.imit_schedulers if sweep else model.imit_scheduler)
    if teacher == 'greedy':
        from ..envs import greedy_controller
        kw['greedy_program'] = greedy_controller(env).greedy_program(env._tables.node_obs_off)
    return kw


def _check_imitation(cfgs):
    """check_imitation on the [MODEL_CONFIG] of every config (before any directory or device work)."""
    from .models import check_imitation
    for c in cfgs:
        check_imitation(c['MODEL_CONFIG'], c['ENV_CONFIG'].get('agent'))


def _schedule(config, env):
    """(total_step, Counter, episode length T) of a run; T must be a multiple of batch_size (utils.py:121)."""
    total_step = int(config.getfloat('TRAIN_CONFIG', 'total_step'))
    counter = Counter(total_step, int(config.getfloat('TRAIN_CONFIG', 'test_interval')),
                      int(config.getfloat('TRAIN_CONFIG', 'log_interval')))
    T, n_step = int(env.T), config['MODEL_CONFIG'].getint('batch_size')
    if T % n_step:
        raise ValueError('episode length T = %d is not a multiple of batch_size = %d' % (T, n_step))
    return total_step, counter, T


def _read_config(config):
    """(ConfigParser, its path or None) of a config path or a parsed ConfigParser."""
    if isinstance(config, configparser.ConfigParser):
        return config, None
    c = configparser.ConfigParser()
    if not c.read(config):
        raise FileNotFoundError(config)
    return c, config


def _save_config(data_dir, cfg, path=None, name='config.ini'):
    """A run's config into its data/: a copy of the file `path` (as main.py copies it), else `cfg` written as `name`."""
    if path is not None:
        shutil.copy(path, data_dir)
        return
    with open(os.path.join(data_dir, name), 'w') as f:
        cfg.write(f)


def _summaries(model, agent, policy, T, log_dirs, device):
    """(summary_rec, [Summaries]) of a run with summaries over K = len(log_dirs) members: the record the trainer fills
    (A2C [T / n_step, 4], 5 columns with a teacher; IQL [ceil(T / n_step), N_ROUNDS, n_agent, 4]; with K > 1 a member
    axis after the first) and one `Summaries` per log directory, with no writer for a directory of None."""
    import torch
    from .summary import SummaryWriter, summary_name
    n_step, K = int(model.n_step), len(log_dirs)
    if model.name == 'iql':
        from .learner_iql import N_ROUNDS
        tail = (N_ROUNDS, model.n_agent, 4)
    else:
        tail = (5 if getattr(model, 'teacher', None) else 4,)
    rec = torch.zeros((-(-T // n_step),) + ((K,) if K > 1 else ()) + tail, dtype=torch.float32, device=device)
    name = summary_name(agent, policy, getattr(model, 'model_type', None))
    kind = 'iql' if model.name == 'iql' else 'a2c'
    return rec, [Summaries(None if d is None else SummaryWriter(d), name, kind, n_step) for d in log_dirs]


def _trainer(model, env, cfgs, total_step, T, rec, seed0, replica0=0, demand=None, demand_mix=None, coop_gamma=None,
             sweep=False):
    """The batched trainer of `model` on env's simulator, keeping a [T, R] reward trace: `BatchedIQLTrainer` with one
    lr / ε schedule pair per config of cfgs (`member_schedulers`), or `BatchedTrainer` with the model's lr / β
    schedules (one per member in a sweep), its teacher's arguments and the members' coop_gamma."""
    import torch
    sim = env._ensure_sim()
    kw = dict(seed0=seed0, replica0=replica0, summary_rec=rec, demand=demand, demand_mix=demand_mix,
              greward_trace=torch.zeros(T, sim.R, dtype=torch.float32, device=sim.device))
    if model.name == 'iql':
        from .learner_iql import BatchedIQLTrainer
        lr, eps = member_schedulers([c['MODEL_CONFIG'] for c in cfgs], total_step)
        return BatchedIQLTrainer(sim, model, lr, eps, **kw)
    from .trainer import BatchedTrainer
    lr, beta = (model.lr_schedulers, model.beta_schedulers) if sweep else (model.lr_scheduler, model.beta_scheduler)
    return BatchedTrainer(sim, model.batched, model.name, lr, beta, coop_gamma=coop_gamma, **kw,
                          **teacher_kwargs(model, env, sweep))


def _evaluator(env_cfg, n_seeds, path, model, device):
    """The batched Evaluator of `model` on a test env of its own (n_seeds test seeds), writing into `path`."""
    from ..envs import make_env
    from .evaluator import Evaluator
    return Evaluator(make_env(env_cfg, n_seeds, path, is_record=False, device=device), model, path,
                     policy_type='default')


def _train(config, dirs, in_test, post_test, R_total, policy, device, pg, summaries=False, deterministic=False,
           mix=None):
    import torch
    from ..envs import make_env
    env_cfg, mc = config['ENV_CONFIG'], config['MODEL_CONFIG']
    agent = env_cfg.get('agent')
    model_spec(agent)                                                 # reject greedy / a2c before any device work
    world, rank = 1, 0
    if pg is not None:
        import torch.distributed as dist
        world, rank = dist.get_world_size(pg), dist.get_rank(pg)
    replica0, R = _dist.replica_range(rank, world, R_total)
    env = make_env(env_cfg, R, dirs['data'], is_record=False, device=device)
    logging.info('Training: s dim: %d, s dim ls: %r, a dim ls: %r, replicas: %d'
                 % (env.n_s, env.n_s_ls, env.n_a_ls, R_total) + (' over %d ranks' % world if world > 1 else ''))
    if mix is not None:
        logging.info('Training: %d demand levels %s, replica g at level g mod %d'
                     % (len(mix.labels), mix.labels, len(mix.labels)))
    total_step, counter, T = _schedule(config, env)
    seed = env_cfg.getint('seed')
    group, own_group = host_group(pg) if pg is not None else (None, False)
    summ = []
    try:
        model = build_model(agent, env, mc, total_step, R, policy=policy, seed=seed, device=device, replica0=replica0,
                            total_replicas=R_total, process_group=pg, deterministic=deterministic)
        sim = env._ensure_sim()
        rec = None
        if summaries:
            rec, summ = _summaries(model, agent, policy, T, [dirs['log'] if rank == 0 else None], sim.device)
            if rank == 0:
                logging.info('Summaries: TensorBoard events into %s' % summ[0].writer.path)
        trainer = _trainer(model, env, [config], total_step, T, rec, seed, replica0=replica0,
                           demand_mix=None if mix is None else mix.nets)
        evaluator = None
        levels = None if mix is None else [(label, None) for label in mix.labels]
        if (in_test or post_test) and rank == 0:
            n = len(env.test_seeds)
            evaluator = _evaluator(env_cfg, n, dirs['data'], model, device)
            if mix is not None:                     # one evaluator per level, on the config edited to that level
                levels = [(label, _evaluator(c['ENV_CONFIG'], n, os.path.join(dirs['data'], label) + os.sep, model,
                                             device)) for label, c in zip(mix.labels, mix.configs)]
        driver = Trainer(trainer, evaluator, counter, agent, in_test, dirs['data'], group=group,
                         summary=summ[0] if summ else None, levels=levels)
        driver.run()
        final_step = counter.cur_step
        if group is not None:
            check_ranks_agree(model, group)
        if rank == 0:
            logging.info('Training: save final model at step %d ...' % final_step)
            model.save(dirs['model'], final_step)
        post = driver.run_offline() if post_test else None
        torch.cuda.synchronize(sim.device)
    finally:
        for s in summ:
            if s.writer is not None:
                s.writer.close()
        if own_group:
            import torch.distributed as dist
            dist.destroy_process_group(group)
    return types.SimpleNamespace(final_step=final_step, episode_sets=driver.n_episode_sets,
                                 env_samples=final_step * R_total, world=world, rank=rank,
                                 data=driver.data if rank == 0 else None, post_test=post, model=model,
                                 trainer=trainer, demand_data=driver.level_data if mix is not None and rank == 0 else None,
                                 demand_post_test=driver.level_post)


def _a2c_agent(config, what, policy):
    """The agent of an A2C population or sweep (`what`): refused for IQL agents and for the FC policy."""
    agent = config['ENV_CONFIG'].get('agent')
    if model_spec(agent)[0] == 'iql':
        raise ValueError("a %s trains an A2C agent (ia2c or ma2c), not %r; train_iql_%s trains IQL members"
                         % (what, agent, what))
    if policy != 'lstm':
        raise ValueError("a %s trains the LSTM policy only (got policy=%r)" % (what, policy))
    return agent


def _iql_agent(config, what):
    agent = config['ENV_CONFIG'].get('agent')
    if model_spec(agent)[0] != 'iql':
        raise ValueError("%s trains an IQL agent (iqll or iqld), not %r; train(seeds=) and train_sweep train A2C "
                         "members" % (what, agent))
    return agent


def _population(config, base_dir, seeds, agent_of):
    """(seeds, member configs, member directories, name of their configs in data/) of a population: the seeds parsed,
    the config read and its agent checked by agent_of(config), which returns it; member k's config is the config with
    `[ENV_CONFIG] seed = seeds[k]` and its directory `member_dir(base_dir, seeds[k], agent)`."""
    seeds = parse_seeds(seeds if isinstance(seeds, str) else ','.join(str(int(x)) for x in seeds))
    config, path = _read_config(config)
    agent = agent_of(config)
    cfgs = []
    for s in seeds:
        cfgs.append(copy.deepcopy(config))
        cfgs[-1]['ENV_CONFIG']['seed'] = str(s)
    return seeds, cfgs, [member_dir(base_dir, s, agent) for s in seeds], os.path.basename(path) if path else 'config.ini'


def train_population(config, base_dir, seeds, test_mode='no_test', n_replicas=1, policy='lstm', device=0,
                     summaries=False, deterministic=False):
    """Train K = len(seeds) members of one A2C agent (ia2c / ma2c, LSTM policy) in one process, member k with
    `[ENV_CONFIG] seed = seeds[k]` on `n_replicas` replicas (a multiple of 64).  One simulator launch and one grouped
    policy forward per control step cover all K * n_replicas replicas (`BatchedA2C` with seeds); the update, the
    optimiser step, the tests and every file are per member.  Member k trains what `train(config with seed seeds[k],
    n_replicas=n_replicas)` trains alone, and its directory `member_dir(base_dir, seeds[k], agent)` holds what that
    run leaves: data/ (the config with the member's seed, train_reward.csv, test CSVs), model/checkpoint-<step>.npz,
    log/<time>.log and, with `summaries`, the member's event file.  Returns a namespace like train()'s with per-member
    lists `dirs`, `data`, `post_test` and `members`.  `deterministic`: as in train(); member k then equals its solo
    deterministic run bit for bit."""
    from .learner import check_population
    t0 = time.time()
    in_test, post_test = init_test_flag(test_mode)
    seeds, cfgs, paths, name = _population(config, base_dir, seeds, lambda c: _a2c_agent(c, 'population', policy))
    check_population(seeds, 0, n_replicas, 1024, None)               # before any directory or device work
    _check_imitation(cfgs[:1])
    out = _train_members(cfgs, paths, int(n_replicas), in_test, post_test, device, summaries, policy=policy,
                         deterministic=deterministic, config_name=name)
    out.wall_sec = time.time() - t0
    return out


def train_iql_population(config, base_dir, seeds, test_mode='no_test', n_replicas=1, device=0, summaries=False):
    """Train K = len(seeds) members of one IQL agent (iqll / iqld) in one process, member k with `[ENV_CONFIG] seed =
    seeds[k]` on `n_replicas` replicas.  One simulator launch, one grouped ε-greedy forward per control step and one
    grouped TD / Adam update per round cover all K * n_replicas replicas (`BatchedIQL` with seeds); the schedules, the
    tests and every file are per member.  Member k's directory `member_dir(base_dir, seeds[k], agent)` is, bit for bit,
    what `train(config with seed seeds[k], n_replicas=n_replicas)` leaves (the log's times aside).  Everything is
    checked before any directory is made.  Returns a namespace like train_population's."""
    t0 = time.time()
    in_test, post_test = init_test_flag(test_mode)
    seeds, cfgs, paths, name = _population(config, base_dir, seeds, lambda c: _iql_agent(c, 'train_iql_population'))
    _check_imitation(cfgs[:1])
    out = _train_members(cfgs, paths, int(n_replicas), in_test, post_test, device, summaries, config_name=name)
    out.wall_sec = time.time() - t0
    return out


# the config keys a sweep's members may set for themselves; every other key must be equal in all of them
SWEEP_CONFIG_KEYS = {
    'ENV_CONFIG': ('seed', 'coop_gamma'),
    'MODEL_CONFIG': ('lr_init', 'lr_decay', 'lr_min', 'entropy_coef_init', 'entropy_decay', 'entropy_coef_min',
                     'entropy_ratio', 'value_coef', 'max_grad_norm', 'rmsp_alpha', 'rmsp_epsilon', 'gamma',
                     'reward_norm', 'reward_clip')}
# the imitation keys the members of an A2C sweep may set for themselves as well (`train_sweep`); `teacher` must be the same
IMITATION_SWEEP_KEYS = ('imitation_coef_init', 'imitation_decay', 'imitation_coef_min', 'imitation_ratio')
# the same for an IQL sweep (`train_iql_sweep`): IQL reads no coop_gamma, and its ring and networks are shared
IQL_SWEEP_CONFIG_KEYS = {
    'ENV_CONFIG': ('seed',),
    'MODEL_CONFIG': ('lr_init', 'lr_decay', 'lr_min', 'epsilon_init', 'epsilon_min', 'epsilon_decay', 'epsilon_ratio',
                     'gamma', 'max_grad_norm', 'reward_norm', 'reward_clip')}


def _same(a, b):
    """Two config values agree: equal text, or equal numbers (5e-4 and 0.0005)."""
    if a == b:
        return True
    try:
        return float(a) == float(b)
    except (TypeError, ValueError):
        return False


def _value(cfg, sec, key):
    return cfg.get(sec, key, fallback=None) if cfg.has_section(sec) else None


def sweep_members(configs, keys=None, demand=False):
    """The members of a sweep as [(name, ConfigParser, path or None)], checked.  `configs`: a list of config paths
    (member name = file stem) or a dict name -> ConfigParser.  Refused with a ValueError: no config, repeated names, a
    key outside `keys` (default SWEEP_CONFIG_KEYS) that differs between two members (naming the key and both members), a
    coop_gamma that differs under ia2c (the reference reads it only for ma2c, envs/env.py:184-188, 595-609), and two
    identical configs.  `demand`: the members may also differ in their scenario's demand keys (envs.DEMAND_KEYS); their
    nets, built on the host, must then differ only in their demand tables (refused naming the member and the field)."""
    from ..envs import demand_keys
    allowed = SWEEP_CONFIG_KEYS if keys is None else keys
    if isinstance(configs, dict):
        items = [(str(n), c, None) for n, c in configs.items()]
    else:
        items = []
        for p in configs:
            c = configparser.ConfigParser()
            if not c.read(p):
                raise FileNotFoundError(p)
            items.append((os.path.splitext(os.path.basename(p))[0], c, p))
    if not items:
        raise ValueError('a sweep needs at least one config')
    names = [n for n, _, _ in items]
    if len(set(names)) != len(names):
        raise ValueError('sweep member names must be distinct (got %s)' % names)
    label = lambda i: items[i][2] or items[i][0]
    c0 = items[0][1]
    agent = _value(c0, 'ENV_CONFIG', 'agent')
    if demand and c0.has_section('ENV_CONFIG'):
        allowed = dict(allowed)
        allowed['ENV_CONFIG'] = tuple(allowed.get('ENV_CONFIG', ())) + tuple(demand_keys(c0['ENV_CONFIG']))
    for i in range(1, len(items)):
        c = items[i][1]
        for sec in sorted(set(c0.sections()) | set(c.sections())):
            keys = set(c0[sec] if c0.has_section(sec) else ()) | set(c[sec] if c.has_section(sec) else ())
            for key in sorted(keys):
                a, b = _value(c0, sec, key), _value(c, sec, key)
                if _same(a, b):
                    continue
                if key not in allowed.get(sec, ()):
                    raise ValueError('[%s] %s differs between %s (%s) and %s (%s): the members of a sweep may differ '
                                     'only in %s' % (sec, key, label(0), a, label(i), b, allowed))
                if key == 'coop_gamma' and agent != 'ma2c':
                    raise ValueError('[ENV_CONFIG] coop_gamma differs between %s and %s, but %s does not use it (only '
                                     'ma2c does)' % (label(0), label(i), agent))
        for j in range(i):
            if all(_same(_value(items[j][1], sec, key), _value(c, sec, key))
                   for sec, ks in allowed.items() for key in ks):
                raise ValueError('%s and %s are identical: a sweep trains each config once' % (label(j), label(i)))
    if demand:
        member_demand([c for _, c, _ in items], [label(i) for i in range(len(items))])
    return items


def member_demand(cfgs, labels=None):
    """The nets of a demand sweep's members (one NetTables per config, built on the host), or None when their demand
    tables are all equal.  Refuses (naming the member and the field) a member whose net differs from the first member's
    in more than its demand tables; ma2c members may differ in coop_gamma as well."""
    from ..envs import check_demand_tables, make_env
    from ..net.tables import DEMAND_FIELDS
    nets = [make_env(c['ENV_CONFIG'], 1, '', is_record=False)._tables for c in cfgs]
    ignore = ('obs_scale',) if cfgs[0]['ENV_CONFIG'].get('agent') == 'ma2c' else ()
    for k in range(1, len(nets)):
        check_demand_tables(nets[0], nets[k], labels[k] if labels else 'member %d' % k, ignore=ignore)
    same = all(np.array_equal(getattr(t, f), getattr(nets[0], f)) for t in nets for f in DEMAND_FIELDS)
    return None if same else nets


def sweep_dir(base_dir, name, agent):
    """The agent directory of the sweep member `name`: <base_dir>/<name>/<agent>."""
    return os.path.join(base_dir, name, agent)


def train_sweep(configs, base_dir, test_mode='no_test', n_replicas=64, device=0, summaries=False, policy='lstm',
                process_group=None, deterministic=False, vary_demand=False):
    """Train a hyperparameter sweep of one A2C agent (ia2c / ma2c, LSTM policy) in one process: one member per config
    (`sweep_members`: the configs may differ only in SWEEP_CONFIG_KEYS and IMITATION_SWEEP_KEYS, with one teacher for
    all), each on `n_replicas` replicas (a multiple of
    64).  One simulator launch and one grouped policy forward per control step cover all K * n_replicas replicas;
    member k runs with its own seed, coop_gamma (ma2c), learner values and lr / entropy schedules, and trains what
    `train(config_k, n_replicas=n_replicas)` trains alone.  Its directory `sweep_dir(base_dir, name_k, agent)` holds
    what that run leaves: data/ (its config, train_reward.csv, test CSVs), model/checkpoint-<step>.npz, log/<time>.log
    and, with `summaries`, its event file.  Everything is checked before any directory or device work.  Returns a
    namespace like train_population's with `names`.  `deterministic`: as in train().  `vary_demand`: the members may
    also differ in their scenario's demand keys (envs.DEMAND_KEYS, `sweep_members(demand=True)`); member k's replicas
    then run at its own demand in the shared simulator."""
    from .learner import check_sweep
    from .models import a2c_hparams
    t0 = time.time()
    in_test, post_test = init_test_flag(test_mode)
    if process_group is not None:
        raise ValueError('a sweep trains in one process: it takes no process_group')
    keys = dict(SWEEP_CONFIG_KEYS, MODEL_CONFIG=SWEEP_CONFIG_KEYS['MODEL_CONFIG'] + IMITATION_SWEEP_KEYS)
    items = sweep_members(configs, keys, demand=vary_demand)
    agent = _a2c_agent(items[0][1], 'sweep', policy)
    cfgs, names = [c for _, c, _ in items], [n for n, _, _ in items]
    _check_imitation(cfgs)
    check_sweep([c['ENV_CONFIG'].getint('seed') for c in cfgs], [a2c_hparams(c['MODEL_CONFIG']) for c in cfgs],
                n_replicas, 1024, None)
    out = _train_members(cfgs, [sweep_dir(base_dir, n, agent) for n in names], int(n_replicas), in_test, post_test,
                         device, summaries, policy=policy, deterministic=deterministic, names=names,
                         srcs=[p for _, _, p in items], demand=member_demand(cfgs) if vary_demand else None)
    out.wall_sec = time.time() - t0
    return out


def train_iql_sweep(configs, base_dir, test_mode='no_test', n_replicas=1, device=0, summaries=False, vary_demand=False):
    """Train a hyperparameter sweep of one IQL agent (iqll / iqld) in one process: one member per config
    (`sweep_members` with IQL_SWEEP_CONFIG_KEYS: the seed, the lr and ε schedules, gamma, max_grad_norm and the reward
    scaling), each on `n_replicas` replicas, sharing the simulator, the replay ring and the grouped kernels.  Member k's
    directory `sweep_dir(base_dir, name_k, agent)` is what `train(config_k, n_replicas=n_replicas)` leaves.  Everything
    is checked before any directory is made.  Returns a namespace like train_sweep's.  `vary_demand`: as in
    train_sweep."""
    t0 = time.time()
    in_test, post_test = init_test_flag(test_mode)
    items = sweep_members(configs, IQL_SWEEP_CONFIG_KEYS, demand=vary_demand)
    agent = _iql_agent(items[0][1], 'train_iql_sweep')
    cfgs, names = [c for _, c, _ in items], [n for n, _, _ in items]
    _check_imitation(cfgs)
    out = _train_members(cfgs, [sweep_dir(base_dir, n, agent) for n in names], int(n_replicas), in_test, post_test,
                         device, summaries, names=names, srcs=[p for _, _, p in items],
                         demand=member_demand(cfgs) if vary_demand else None)
    out.wall_sec = time.time() - t0
    return out


def member_schedulers(model_configs, total_step):
    """(lr, ε) schedulers of IQL members, one `iql_schedulers` pair per member's [MODEL_CONFIG] (a population's are
    equal): two lists, or one pair for one member.  The trainer calls each as the member's solo run calls its own."""
    from .models import iql_schedulers
    pairs = [iql_schedulers(c, total_step) for c in model_configs]
    if len(pairs) == 1:
        return pairs[0]
    return [p[0] for p in pairs], [p[1] for p in pairs]


def _train_members(cfgs, paths, R_m, in_test, post_test, device, summaries, policy='lstm', deterministic=False,
                   config_name='config.ini', names=None, srcs=None, demand=None):
    """The training run of a population, or with `names` a sweep, of A2C or IQL members: member k from cfgs[k] into the
    agent directory paths[k].  The env and the learner (which refuses what it cannot train) are built before any
    directory is made; then the directories with their configs (a copy of srcs[k], else cfgs[k] written as
    `config_name`), member-tagged log files, and one driver per member over one simulator, learner and trainer for all
    K * R_m replicas.  A sweep gives each member its own learner values and schedules and, for ma2c, its own coop_gamma
    in the simulator; `demand` (member_demand) gives member k the demand of demand[k]."""
    import torch
    from ..envs import make_env
    K, sweep = len(cfgs), names is not None
    agent = cfgs[0]['ENV_CONFIG'].get('agent')
    seeds = [c['ENV_CONFIG'].getint('seed') for c in cfgs]
    cg = [c['ENV_CONFIG'].getfloat('coop_gamma') for c in cfgs] if sweep and agent == 'ma2c' else None
    if cg is not None and len(set(cg)) == 1:
        cg = None                                                     # one coop_gamma: the simulator's own
    # the training simulator marks the observation entries it scales only when built with a coop_gamma other than 1
    base = next((k for k in range(K) if cg[k] != 1.0), 0) if cg is not None else 0
    env = make_env(cfgs[base]['ENV_CONFIG'], K * R_m, os.path.join(paths[0], 'data') + os.sep, is_record=False,
                   device=device)
    total_step, counter, T = _schedule(cfgs[0], env)
    model = build_model(agent, env, cfgs[0]['MODEL_CONFIG'], total_step, R_m, seeds=seeds, device=device,
                        member_configs=[c['MODEL_CONFIG'] for c in cfgs] if sweep else None,
                        deterministic=deterministic)
    dirs = [init_dir(p) for p in paths]
    for k, d in enumerate(dirs):
        _save_config(d['data'], cfgs[k], srcs[k] if srcs else None, config_name)
    handlers, summ = init_log([d['log'] for d in dirs]), []
    try:
        what = 'sweep of %d configs %s' % (K, names) if sweep else 'population of %d seeds %s' % (K, seeds)
        logging.info('Training: s dim: %d, s dim ls: %r, a dim ls: %r, %s x %d replicas'
                     % (env.n_s, env.n_s_ls, env.n_a_ls, what, R_m))
        members = [model.member(k) for k in range(K)] if model.name == 'iql' else model.members()
        sim = env._ensure_sim()
        rec = None
        if summaries:
            rec, summ = _summaries(model, agent, policy, T, [d['log'] for d in dirs], sim.device)
        trainer = _trainer(model, env, cfgs, total_step, T, rec, seeds[0], demand=demand, coop_gamma=cg, sweep=sweep)
        drivers = []
        for k in range(K):                  # one driver per member, over its view of the shared trainer
            evaluator = None
            if in_test or post_test:
                evaluator = _evaluator(cfgs[k]['ENV_CONFIG'], len(env.test_seeds), dirs[k]['data'], members[k], device)
            drivers.append(Trainer(trainer.member(k), evaluator, counter, agent, in_test, dirs[k]['data'],
                                   summary=summ[k] if summ else None, log_extra={'member': k}))
        run_schedule(drivers)
        post = [None] * K
        for k, d in enumerate(drivers):
            logging.info('Training: save final model at step %d ...' % counter.cur_step, extra=d.log_extra)
            members[k].save(dirs[k]['model'], counter.cur_step)
            if post_test:
                post[k] = d.run_offline()
        torch.cuda.synchronize(sim.device)
    finally:
        for s in summ:
            s.writer.close()
        for h in handlers:
            logging.getLogger().removeHandler(h)
            h.close()
    out = types.SimpleNamespace(final_step=counter.cur_step, episode_sets=drivers[0].n_episode_sets,
                                env_samples=counter.cur_step * K * R_m, world=1, rank=0, seeds=seeds,
                                data=[d.data for d in drivers], post_test=post, model=model, members=members,
                                trainer=trainer, dirs=paths)
    if sweep:
        out.names = names
    return out
