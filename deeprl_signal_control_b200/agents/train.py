"""`train`: the reference's `main.py train` (main.py:82-155) with its `utils.py:Counter` / `Trainer.run`
(utils.py:70-108, 255-308), for R lock-stepped replicas on the device.

    train(config, base_dir, test_mode='no_test', n_replicas=1, policy='lstm', device=0, process_group=None,
          summaries=False)
    train_sweep([a.ini, b.ini, ...], base_dir, ...)   (one member per config in one process, `train_sweep`)

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
import hashlib
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


def init_log(log_dir):
    """utils.py:42-48: INFO records to `<log_dir>/<time>.log` and to stderr.  The handlers are added to the root logger
    and returned, so that a caller that trains more than once in a process can remove them."""
    fmt = logging.Formatter('%(asctime)s [%(levelname)s] %(message)s')
    handlers = [logging.FileHandler(os.path.join(log_dir, '%d.log' % time.time())), logging.StreamHandler()]
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
    other name.  greedy has nothing to train; the centralised a2c (a joint action space of prod(n_a) actions) has no
    batched learner."""
    if agent == 'greedy':
        raise ValueError("agent 'greedy' has no model to train")
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
    agent 0's scalars of every update (A2C: policy / value / total loss and gradient norm at the step of the backward;
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
            loss = _dist.sum_partials(rec[:, :3], group)
            if loss is None:
                return None
            rec = np.concatenate([loss, rec[:, 3:]], 1)
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


class Trainer:
    """utils.py:Trainer.run / Tester.run_offline over a batched trainer (`run(n)`, `T_episode`, `episode_rewards`,
    `greward_trace` [T_episode, R]) and a batched `Evaluator` (`perform_all()`, `run()`, `env`).

    `group`: None for one process; over W > 1 ranks a group that takes CPU tensors (gloo).  Every rank then runs the
    same schedule; rank 0 gathers the traces, holds the rows, runs the tests (only it has an evaluator) and writes the
    CSV, and all ranks meet at a barrier after each test.
    `summary`: None, or the `Summaries` of the run (the trainer then keeps a `summary_rec`).
    `log_extra`: the `extra` of its log records (a population member's tag, see `train_population`).
    `run_schedule` runs one schedule for several drivers that share a batched trainer and counter."""

    def __init__(self, trainer, evaluator, counter: Counter, agent: str, run_test: bool, output_path: str,
                 group=None, summary=None, log_extra=None):
        if trainer.greward_trace is None:
            raise ValueError('the driver needs the trainer to keep a greward_trace')
        self.trainer, self.evaluator, self.counter = trainer, evaluator, counter
        self.agent, self.run_test, self.output_path = agent, run_test, output_path
        self.group, self.summary = group, summary
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
        if self.summary is not None:
            self.summary.episode_set(rec, self.trainer.summary_ran, prev, step, mean)
        if c.should_log(prev):
            logging.info('Training: global step %d, episode set %d, avg R: %.2f, std R: %.2f'
                         % (step, self.n_episode_sets, mean, std), extra=self.log_extra)

    def write_rows(self):
        if self.rank0:
            import pandas as pd
            pd.DataFrame(self.data).to_csv(self.output_path + 'train_reward.csv')

    def run_offline(self):
        """Tester.run_offline: every test seed in record mode, the three CSVs into output_path.  Returns the per-seed
        (mean, std) on rank 0, None on the other ranks."""
        out = None
        if self.rank0:
            self.evaluator.env.init_data(True, False, self.output_path)
            mean, std = self.evaluator.run()
            logging.info('Offline testing: avg R: %.2f' % np.mean(mean), extra=self.log_extra)
            out = mean, std
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
    reduces in a fixed order, so for iqll / iqld it changes nothing."""
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
                      total_replicas=total_replicas, pg=process_group)


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


def train(config, base_dir, test_mode='no_test', n_replicas=1, policy='lstm', device=0, process_group=None,
          summaries=False, seeds=None, deterministic=False):
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
    directory is made); a no-op for IQL, whose update is already reproducible."""
    if deterministic and policy != 'lstm':
        raise ValueError("deterministic=True needs the LSTM policy's lean update (got policy=%r)" % (policy,))
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
        handlers = init_log(dirs['log'])
    else:
        dirs = {k: os.path.join(base_dir, k) + os.sep for k in ('log', 'data', 'model')}
        handlers = init_rank_log(rank)
    try:
        if isinstance(config, configparser.ConfigParser):
            if rank == 0:
                with open(os.path.join(dirs['data'], 'config.ini'), 'w') as f:
                    config.write(f)
        else:
            if rank == 0:
                shutil.copy(config, dirs['data'])
            path, config = config, configparser.ConfigParser()
            if not config.read(path):
                raise FileNotFoundError(path)
        out = _train(config, dirs, in_test, post_test, int(n_replicas), policy, device, pg, bool(summaries),
                     bool(deterministic))
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


def _schedule(config, env):
    """(total_step, Counter, episode length T) of a run; T must be a multiple of batch_size (utils.py:121)."""
    total_step = int(config.getfloat('TRAIN_CONFIG', 'total_step'))
    counter = Counter(total_step, int(config.getfloat('TRAIN_CONFIG', 'test_interval')),
                      int(config.getfloat('TRAIN_CONFIG', 'log_interval')))
    T, n_step = int(env.T), config['MODEL_CONFIG'].getint('batch_size')
    if T % n_step:
        raise ValueError('episode length T = %d is not a multiple of batch_size = %d' % (T, n_step))
    return total_step, counter, T


def _train(config, dirs, in_test, post_test, R_total, policy, device, pg, summaries=False, deterministic=False):
    import torch
    from ..envs import make_env
    from .evaluator import Evaluator
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
    total_step, counter, T = _schedule(config, env)
    seed = env_cfg.getint('seed')
    group, own_group = host_group(pg) if pg is not None else (None, False)
    writer = None
    try:
        model = build_model(agent, env, mc, total_step, R, policy=policy, seed=seed, device=device, replica0=replica0,
                            total_replicas=R_total, process_group=pg, deterministic=deterministic)
        sim = env._ensure_sim()
        trace = torch.zeros(T, R, dtype=torch.float32, device=sim.device)
        summary, srec = None, {}
        if summaries:
            from .summary import SummaryWriter, summary_name
            n_step = int(model.n_step)
            if model.name == 'iql':
                from .learner_iql import N_ROUNDS
                shape = (-(-T // n_step), N_ROUNDS, model.n_agent, 4)
            else:
                shape = (T // n_step, 4)
            srec = dict(summary_rec=torch.zeros(shape, dtype=torch.float32, device=sim.device))
            if rank == 0:
                writer = SummaryWriter(dirs['log'])
                logging.info('Summaries: TensorBoard events into %s' % writer.path)
            summary = Summaries(writer, summary_name(agent, policy, getattr(model, 'model_type', None)),
                                'iql' if model.name == 'iql' else 'a2c', n_step)
        if model.name == 'iql':
            from .learner_iql import BatchedIQLTrainer
            from .models import iql_schedulers
            lr_s, eps_s = iql_schedulers(mc, total_step)
            trainer = BatchedIQLTrainer(sim, model, lr_s, eps_s, seed0=seed, replica0=replica0, greward_trace=trace,
                                        **srec)
        else:
            from .trainer import BatchedTrainer
            trainer = BatchedTrainer(sim, model.batched, agent, model.lr_scheduler, model.beta_scheduler, seed0=seed,
                                     replica0=replica0, greward_trace=trace, **srec)
        evaluator = None
        if (in_test or post_test) and rank == 0:
            test_env = make_env(env_cfg, len(env.test_seeds), dirs['data'], is_record=False, device=device)
            evaluator = Evaluator(test_env, model, dirs['data'], policy_type='default')
        driver = Trainer(trainer, evaluator, counter, agent, in_test, dirs['data'], group=group, summary=summary)
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
        if writer is not None:
            writer.close()
        if own_group:
            import torch.distributed as dist
            dist.destroy_process_group(group)
    return types.SimpleNamespace(final_step=final_step, episode_sets=driver.n_episode_sets,
                                 env_samples=final_step * R_total, world=world, rank=rank,
                                 data=driver.data if rank == 0 else None, post_test=post, model=model,
                                 trainer=trainer)


def _member_filter(k):
    """Log records of member k, and those of no member in particular, go to member k's log file."""
    return lambda rec: getattr(rec, 'member', k) == k


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
    import copy
    from .learner import check_population
    t0 = time.time()
    in_test, post_test = init_test_flag(test_mode)
    seeds = parse_seeds(','.join(str(int(x)) for x in seeds)) if not isinstance(seeds, str) else parse_seeds(seeds)
    if isinstance(config, configparser.ConfigParser):
        name = 'config.ini'
    else:
        path, name, config = config, os.path.basename(config), configparser.ConfigParser()
        if not config.read(path):
            raise FileNotFoundError(path)
    agent = config['ENV_CONFIG'].get('agent')
    kind, _ = model_spec(agent)
    if kind == 'iql':
        raise ValueError("a population trains an A2C agent (ia2c or ma2c), not %r" % agent)
    if policy != 'lstm':
        raise ValueError("a population trains the LSTM policy only (got policy=%r)" % policy)
    check_population(seeds, 0, n_replicas, 1024, None)               # before any directory or device work
    cfgs, dirs = [], []
    for s in seeds:
        cfg = copy.deepcopy(config)
        cfg['ENV_CONFIG']['seed'] = str(s)
        d = init_dir(member_dir(base_dir, s, agent))
        with open(os.path.join(d['data'], name), 'w') as f:
            cfg.write(f)
        cfgs.append(cfg); dirs.append(d)
    out = _train_members(cfgs, dirs, agent, seeds, int(n_replicas), in_test, post_test, policy, device, summaries,
                         'population of %d seeds %s' % (len(seeds), seeds), deterministic=deterministic)
    out.dirs, out.wall_sec = [member_dir(base_dir, s, agent) for s in seeds], time.time() - t0
    return out


def _train_members(cfgs, dirs, agent, seeds, R_m, in_test, post_test, policy, device, summaries, what, sweep=False,
                   deterministic=False):
    """The training run of a population or a sweep, member k from cfgs[k] (seed seeds[k]) into the agent directory
    dirs[k] (init_dir's dict): member-tagged log files, one simulator and one learner for all K * R_m replicas, one
    driver per member.  A sweep gives each member its own learner values and schedules (`IA2C(member_configs=...)`)
    and, for ma2c, its own coop_gamma in the simulator."""
    import torch
    from ..envs import make_env
    from .evaluator import Evaluator
    from .trainer import BatchedTrainer
    K = len(cfgs)
    handlers = []
    fmt = logging.Formatter('%(asctime)s [%(levelname)s] %(message)s')
    for k, d in enumerate(dirs):
        h = logging.FileHandler(os.path.join(d['log'], '%d.log' % time.time()))
        h.setFormatter(fmt)
        h.addFilter(_member_filter(k))
        handlers.append(h)
    handlers.append(logging.StreamHandler())
    handlers[-1].setFormatter(fmt)
    root = logging.getLogger()
    for h in handlers:
        root.addHandler(h)
    root.setLevel(logging.INFO)
    writers = []
    cg = [c['ENV_CONFIG'].getfloat('coop_gamma') for c in cfgs] if sweep and agent == 'ma2c' else None
    if cg is not None and len(set(cg)) == 1:
        cg = None                                                     # one coop_gamma: the simulator's own
    # the training simulator marks the observation entries it scales only when built with a coop_gamma other than 1
    base = next((k for k in range(K) if cg[k] != 1.0), 0) if cg is not None else 0
    try:
        env_cfg, mc = cfgs[base]['ENV_CONFIG'], cfgs[0]['MODEL_CONFIG']
        env = make_env(env_cfg, K * R_m, dirs[0]['data'], is_record=False, device=device)
        logging.info('Training: s dim: %d, s dim ls: %r, a dim ls: %r, %s x %d replicas'
                     % (env.n_s, env.n_s_ls, env.n_a_ls, what, R_m))
        total_step, counter, T = _schedule(cfgs[0], env)
        model = build_model(agent, env, mc, total_step, R_m, seeds=seeds, device=device,
                            member_configs=[c['MODEL_CONFIG'] for c in cfgs] if sweep else None,
                            deterministic=deterministic)
        members = model.members()
        sim = env._ensure_sim()
        trace = torch.zeros(T, K * R_m, dtype=torch.float32, device=sim.device)
        srec, summ = {}, None
        if summaries:
            from .summary import SummaryWriter, summary_name
            shape = (T // model.n_step,) + ((K,) if K > 1 else ()) + (4,)
            srec = dict(summary_rec=torch.zeros(shape, dtype=torch.float32, device=sim.device))
            writers = [SummaryWriter(d['log']) for d in dirs]
            summ = [Summaries(w, summary_name(agent, policy), 'a2c', model.n_step) for w in writers]
        lr, beta = (model.lr_schedulers, model.beta_schedulers) if sweep else (model.lr_scheduler, model.beta_scheduler)
        trainer = BatchedTrainer(sim, model.batched, agent, lr, beta, seed0=seeds[0], greward_trace=trace,
                                 coop_gamma=cg, **srec)
        drivers = []
        for k in range(K):                  # one driver per member, over its view of the shared trainer
            evaluator = None
            if in_test or post_test:
                test_env = make_env(cfgs[k]['ENV_CONFIG'], len(env.test_seeds), dirs[k]['data'], is_record=False,
                                    device=device)
                evaluator = Evaluator(test_env, members[k], dirs[k]['data'], policy_type='default')
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
        for w in writers:
            w.close()
        for h in handlers:
            root.removeHandler(h)
            h.close()
    return types.SimpleNamespace(final_step=counter.cur_step, episode_sets=drivers[0].n_episode_sets,
                                 env_samples=counter.cur_step * K * R_m, world=1, rank=0, seeds=seeds,
                                 data=[d.data for d in drivers], post_test=post, model=model, members=members,
                                 trainer=trainer)


# the config keys a sweep's members may set for themselves; every other key must be equal in all of them
SWEEP_CONFIG_KEYS = {
    'ENV_CONFIG': ('seed', 'coop_gamma'),
    'MODEL_CONFIG': ('lr_init', 'lr_decay', 'lr_min', 'entropy_coef_init', 'entropy_decay', 'entropy_coef_min',
                     'entropy_ratio', 'value_coef', 'max_grad_norm', 'rmsp_alpha', 'rmsp_epsilon', 'gamma',
                     'reward_norm', 'reward_clip')}


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


def sweep_members(configs):
    """The members of a sweep as [(name, ConfigParser, path or None)], checked.  `configs`: a list of config paths
    (member name = file stem) or a dict name -> ConfigParser.  Refused with a ValueError: no config, repeated names, a
    key outside SWEEP_CONFIG_KEYS that differs between two members (naming the key and both members), a coop_gamma that
    differs under ia2c (the reference reads it only for ma2c, envs/env.py:184-188, 595-609), and two identical configs."""
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
    for i in range(1, len(items)):
        c = items[i][1]
        for sec in sorted(set(c0.sections()) | set(c.sections())):
            keys = set(c0[sec] if c0.has_section(sec) else ()) | set(c[sec] if c.has_section(sec) else ())
            for key in sorted(keys):
                a, b = _value(c0, sec, key), _value(c, sec, key)
                if _same(a, b):
                    continue
                if key not in SWEEP_CONFIG_KEYS.get(sec, ()):
                    raise ValueError('[%s] %s differs between %s (%s) and %s (%s): the members of a sweep may differ '
                                     'only in %s' % (sec, key, label(0), a, label(i), b, SWEEP_CONFIG_KEYS))
                if key == 'coop_gamma' and agent != 'ma2c':
                    raise ValueError('[ENV_CONFIG] coop_gamma differs between %s and %s, but %s does not use it (only '
                                     'ma2c does)' % (label(0), label(i), agent))
        for j in range(i):
            if all(_same(_value(items[j][1], sec, key), _value(c, sec, key))
                   for sec, keys in SWEEP_CONFIG_KEYS.items() for key in keys):
                raise ValueError('%s and %s are identical: a sweep trains each config once' % (label(j), label(i)))
    return items


def sweep_dir(base_dir, name, agent):
    """The agent directory of the sweep member `name`: <base_dir>/<name>/<agent>."""
    return os.path.join(base_dir, name, agent)


def train_sweep(configs, base_dir, test_mode='no_test', n_replicas=64, device=0, summaries=False, policy='lstm',
                process_group=None, deterministic=False):
    """Train a hyperparameter sweep of one A2C agent (ia2c / ma2c, LSTM policy) in one process: one member per config
    (`sweep_members`: the configs may differ only in SWEEP_CONFIG_KEYS), each on `n_replicas` replicas (a multiple of
    64).  One simulator launch and one grouped policy forward per control step cover all K * n_replicas replicas;
    member k runs with its own seed, coop_gamma (ma2c), learner values and lr / entropy schedules, and trains what
    `train(config_k, n_replicas=n_replicas)` trains alone.  Its directory `sweep_dir(base_dir, name_k, agent)` holds
    what that run leaves: data/ (its config, train_reward.csv, test CSVs), model/checkpoint-<step>.npz, log/<time>.log
    and, with `summaries`, its event file.  Everything is checked before any directory or device work.  Returns a
    namespace like train_population's with `names`.  `deterministic`: as in train()."""
    from .learner import check_sweep
    from .models import a2c_hparams
    t0 = time.time()
    in_test, post_test = init_test_flag(test_mode)
    if process_group is not None:
        raise ValueError('a sweep trains in one process: it takes no process_group')
    items = sweep_members(configs)
    agent = items[0][1]['ENV_CONFIG'].get('agent')
    kind, _ = model_spec(agent)
    if kind == 'iql':
        raise ValueError("a sweep trains an A2C agent (ia2c or ma2c), not %r" % agent)
    if policy != 'lstm':
        raise ValueError("a sweep trains the LSTM policy only (got policy=%r)" % policy)
    cfgs = [c for _, c, _ in items]
    seeds = [c['ENV_CONFIG'].getint('seed') for c in cfgs]
    check_sweep(seeds, [a2c_hparams(c['MODEL_CONFIG']) for c in cfgs], n_replicas, 1024, None)
    names, dirs = [n for n, _, _ in items], []
    for name, cfg, path in items:
        d = init_dir(sweep_dir(base_dir, name, agent))
        if path is not None:
            shutil.copy(path, d['data'])                              # as train() copies its config
        else:
            with open(os.path.join(d['data'], 'config.ini'), 'w') as f:
                cfg.write(f)
        dirs.append(d)
    out = _train_members(cfgs, dirs, agent, seeds, int(n_replicas), in_test, post_test, policy, device, summaries,
                         'sweep of %d configs %s' % (len(cfgs), names), sweep=True, deterministic=deterministic)
    out.names, out.dirs = names, [sweep_dir(base_dir, n, agent) for n in names]
    out.wall_sec = time.time() - t0
    return out
