"""`train`: the reference's `main.py train` (main.py:82-155) with its `utils.py:Counter` / `Trainer.run`
(utils.py:70-108, 255-308), for R lock-stepped replicas on the device.

    train(config, base_dir, test_mode='no_test', n_replicas=1, policy='lstm', device=0)

leaves the reference's agent directory: `data/` with a copy of the config and `train_reward.csv`, `model/checkpoint-<step>`
and `log/<time>.log`; with `after_train_test` / `all_test` also `data/<scenario>_<agent>_{control,traffic,trip}.csv`.
`scripts/evaluate.py --agent-dir base_dir` reads that directory back.

Protocol (the reference's, applied to R replicas):
* the global step counts control steps of the lock-step: one episode of all replicas advances it by T, so a run of
  `total_step` makes as many updates as the reference's one-environment run, each on R times the data;
* before every episode set: a test when `in_train_test` and `cur_step - last_test_step >= test_interval`; the run stops
  when `cur_step >= total_step`, checked only between episodes;
* one `train_reward.csv` row per episode set (test_id -1): avg_reward = mean and std_reward = np.std of the per-step
  global reward pooled over every replica and step; one row per test seed (test_id k) with that seed's mean / std.
The training loop itself is `BatchedTrainer` / `BatchedIQLTrainer`; the tests run on the batched `Evaluator` over an
env of its own (`ENV_CONFIG.test_seeds`, test mode, policy_type 'default'), which reads the learner's live weights on
the device and leaves the training sim and the learner's recurrent state alone.
"""
from __future__ import annotations

import configparser
import logging
import os
import shutil
import time
import types

import numpy as np

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


class Trainer:
    """utils.py:Trainer.run / Tester.run_offline over a batched trainer (`run(n)`, `T_episode`, `episode_rewards`,
    `greward_trace` [T_episode, R]) and a batched `Evaluator` (`perform_all()`, `run()`, `env`)."""

    def __init__(self, trainer, evaluator, counter: Counter, agent: str, run_test: bool, output_path: str):
        if trainer.greward_trace is None:
            raise ValueError('the driver needs the trainer to keep a greward_trace')
        self.trainer, self.evaluator, self.counter = trainer, evaluator, counter
        self.agent, self.run_test, self.output_path = agent, run_test, output_path
        self.T = int(trainer.T_episode)
        self.data = []
        self.n_episode_sets = 0
        if run_test:
            logging.info('Testing: total test num: %d' % evaluator.test_num)

    def test(self):
        step = self.counter.cur_step
        t0 = time.time()
        mean, std = self.evaluator.perform_all()
        for k in range(len(mean)):
            self.data.append({'agent': self.agent, 'step': step, 'test_id': k, 'avg_reward': float(mean[k]),
                              'std_reward': float(std[k])})
        logging.info('Testing: global step %d, avg R: %.2f (%.2f s)' % (step, np.mean(mean), time.time() - t0))

    def run(self):
        c = self.counter
        while not c.should_stop():
            if self.run_test and c.should_test():
                self.test()
            prev = c.cur_step
            self.trainer.run(self.T)                                  # one episode of every replica
            step = c.next(self.T)
            self.n_episode_sets += 1
            rewards = np.asarray(self.trainer.greward_trace.cpu().numpy(), np.float64)
            mean, std = float(self.trainer.episode_rewards[-1]), float(np.std(rewards))
            self.data.append({'agent': self.agent, 'step': step, 'test_id': -1, 'avg_reward': mean, 'std_reward': std})
            if c.should_log(prev):
                logging.info('Training: global step %d, episode set %d, avg R: %.2f, std R: %.2f'
                             % (step, self.n_episode_sets, mean, std))
        import pandas as pd
        pd.DataFrame(self.data).to_csv(self.output_path + 'train_reward.csv')

    def run_offline(self):
        """Tester.run_offline: every test seed in record mode, the three CSVs into output_path.  Returns the per-seed
        (mean, std)."""
        self.evaluator.env.init_data(True, False, self.output_path)
        mean, std = self.evaluator.run()
        logging.info('Offline testing: avg R: %.2f' % np.mean(mean))
        return mean, std


def build_model(agent, env, model_config, total_step, n_replicas, policy='lstm', seed=0, device=0):
    """main.py:110-121 on the batched learners: IA2C / MA2C wrappers (seed = ENV_CONFIG.seed) or BatchedIQL (seed 0)."""
    kind, model_type = model_spec(agent)
    t = env._tables
    if kind != 'iql':
        from .models import IA2C, MA2C
        kw = dict(seed=seed, n_replicas=n_replicas, obs_off=t.node_obs_off, policy=policy, device=device)
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
    return BatchedIQL(lay, n_replicas, model_config, model_type, seed=0, device=device)


def train(config, base_dir, test_mode='no_test', n_replicas=1, policy='lstm', device=0):
    """main.py train.  `config`: the path of a reference config (copied into data/) or a parsed ConfigParser (written
    to data/config.ini), with [ENV_CONFIG], [MODEL_CONFIG] and [TRAIN_CONFIG].  Returns a namespace with final_step,
    episode_sets, env_samples (= final_step * n_replicas), wall_sec, data (the train_reward.csv rows), post_test (the
    per-seed (mean, std) of the post-training test or None), and the live model and trainer.

    The post-training test follows what the reference intends (main.py:147-150) rather than what its code does: its
    `Tester.__init__` calls `Trainer.__init__` without `run_test`, and `run_offline` is passed an argument it does not
    take, so both raise TypeError and the reference's after_train_test never runs.  Here the model is saved first, then
    every test seed is played once in record mode and the three CSVs go into data/."""
    t0 = time.time()
    in_test, post_test = init_test_flag(test_mode)
    dirs = init_dir(base_dir)
    handlers = init_log(dirs['log'])
    try:
        if isinstance(config, configparser.ConfigParser):
            with open(os.path.join(dirs['data'], 'config.ini'), 'w') as f:
                config.write(f)
        else:
            shutil.copy(config, dirs['data'])
            path, config = config, configparser.ConfigParser()
            if not config.read(path):
                raise FileNotFoundError(path)
        out = _train(config, dirs, in_test, post_test, int(n_replicas), policy, device)
    finally:
        for h in handlers:
            logging.getLogger().removeHandler(h)
            h.close()
    out.wall_sec = time.time() - t0
    return out


def _train(config, dirs, in_test, post_test, R, policy, device):
    import torch
    from ..envs import make_env
    from .evaluator import Evaluator
    env_cfg, mc = config['ENV_CONFIG'], config['MODEL_CONFIG']
    agent = env_cfg.get('agent')
    model_spec(agent)                                                 # reject greedy / a2c before any device work
    env = make_env(env_cfg, R, dirs['data'], is_record=False, device=device)
    logging.info('Training: s dim: %d, s dim ls: %r, a dim ls: %r, replicas: %d'
                 % (env.n_s, env.n_s_ls, env.n_a_ls, R))
    total_step = int(config.getfloat('TRAIN_CONFIG', 'total_step'))
    counter = Counter(total_step, int(config.getfloat('TRAIN_CONFIG', 'test_interval')),
                      int(config.getfloat('TRAIN_CONFIG', 'log_interval')))
    seed = env_cfg.getint('seed')
    model = build_model(agent, env, mc, total_step, R, policy=policy, seed=seed, device=device)
    sim = env._ensure_sim()
    T = int(env.T)
    if T % mc.getint('batch_size'):                                   # utils.py:121
        raise ValueError('episode length T = %d is not a multiple of batch_size = %d' % (T, mc.getint('batch_size')))
    trace = torch.zeros(T, R, dtype=torch.float32, device=sim.device)
    if model.name == 'iql':
        from .learner_iql import BatchedIQLTrainer
        from .models import iql_schedulers
        lr_s, eps_s = iql_schedulers(mc, total_step)
        trainer = BatchedIQLTrainer(sim, model, lr_s, eps_s, seed0=seed, greward_trace=trace)
    else:
        from .trainer import BatchedTrainer
        trainer = BatchedTrainer(sim, model.batched, agent, model.lr_scheduler, model.beta_scheduler, seed0=seed,
                                 greward_trace=trace)
    evaluator = None
    if in_test or post_test:
        test_env = make_env(env_cfg, len(env.test_seeds), dirs['data'], is_record=False, device=device)
        evaluator = Evaluator(test_env, model, dirs['data'], policy_type='default')
    driver = Trainer(trainer, evaluator, counter, agent, in_test, dirs['data'])
    driver.run()
    final_step = counter.cur_step
    logging.info('Training: save final model at step %d ...' % final_step)
    model.save(dirs['model'], final_step)
    post = driver.run_offline() if post_test else None
    torch.cuda.synchronize(sim.device)
    return types.SimpleNamespace(final_step=final_step, episode_sets=driver.n_episode_sets,
                                 env_samples=final_step * R, data=driver.data, post_test=post, model=model,
                                 trainer=trainer)
