"""CPU: the training driver (agents/train.py) — its schedule of tests, training rows and stop against a restatement of
the reference's Counter + Trainer.run (utils.py:70-107, 255-308) stepped one control step at a time, the
train_reward.csv format, the agent -> model map of main.py and the shared IQL scheduler builder."""
import configparser
import itertools
import logging

import numpy as np
import pytest
import torch

from deeprl_signal_control_b200.agents import train as drv


def reference_schedule(total_step, test_step, log_step, T, n_step, run_test, post_test):
    """utils.py:Counter and Trainer.run with explore() cut at n_step steps or done, the episode ending after T steps:
    the events (kind, step) in order, and the steps the reference logs at."""
    counter, cur, cur_test = itertools.count(1), 0, 0
    events, logged = [], []
    while not cur >= total_step:
        if run_test and cur - cur_test >= test_step:
            cur_test = cur
            events.append(("test", cur))
        t, done = 0, False
        while not done:
            for _ in range(n_step):
                cur = next(counter)
                t += 1
                if cur % log_step == 0:
                    logged.append(cur)
                done = t == T
                if done:
                    break
        events.append(("train", cur))
    if post_test:
        events.append(("offline", cur))
    return events, cur, logged


class StubTrainer:
    def __init__(self, T, R):
        self.T_episode, self.R = T, R
        self.greward_trace = torch.zeros(T, R)
        self.episode_rewards = []
        self.episode = 0

    def run(self, n):
        assert n == self.T_episode
        self.episode += 1
        g = torch.arange(self.T_episode * self.R, dtype=torch.float32).reshape(self.T_episode, self.R)
        self.greward_trace.copy_(-(g % 7) * self.episode)
        self.episode_rewards.append(float(self.greward_trace.double().mean()))


class StubEnv:
    def __init__(self):
        self.records = []

    def init_data(self, is_record, record_stats, output_path):
        self.records.append((is_record, record_stats, output_path))


class StubEvaluator:
    def __init__(self, n_seeds, trainer):
        self.test_num, self.trainer, self.env = n_seeds, trainer, StubEnv()
        self.calls = []

    def perform_all(self):
        e = self.trainer.episode
        self.calls.append(("perform_all", e))
        return np.arange(self.test_num) - 10.0 * e, np.arange(self.test_num) + 0.5 * e

    def run(self):
        self.calls.append(("run", self.trainer.episode))
        return self.perform_all()


def _drive(tmp_path, total_step, test_step, log_step, T, mode):
    in_test, post_test = drv.init_test_flag(mode)
    tr = StubTrainer(T, 3)
    ev = StubEvaluator(2, tr)
    d = drv.Trainer(tr, ev, drv.Counter(total_step, test_step, log_step), "ma2c", in_test, str(tmp_path) + "/")
    d.run()
    post = d.run_offline() if post_test else None
    return d, tr, ev, post


@pytest.mark.parametrize("mode", drv.TEST_MODES)
@pytest.mark.parametrize("total_step,test_step,T,n_step", [
    (300, 50, 120, 120),        # total_step not a multiple of T, tests more often than episodes
    (360, 120, 120, 20),        # test_interval == T
    (1000, 250, 120, 40),       # test_interval > T and not a multiple of it
    (1e4, 2e4, 720, 120),       # the shipped grid configs' ratio: no in-training test before step 2e4
    (240, 0, 120, 120),         # test_interval 0: a test before every episode, the first at step 0
])
def test_schedule_matches_reference_counter_and_run(tmp_path, caplog, mode, total_step, test_step, T, n_step):
    log_step = 100
    in_test, post_test = drv.init_test_flag(mode)
    want, final, logged = reference_schedule(total_step, test_step, log_step, T, n_step, in_test, post_test)
    with caplog.at_level(logging.INFO):
        d, tr, ev, post = _drive(tmp_path, total_step, test_step, log_step, T, mode)
    got = [("train" if row["test_id"] == -1 else "test", row["step"]) for row in d.data if row["test_id"] <= 0]
    if post is not None:
        got.append(("offline", d.counter.cur_step))
    assert got == want
    assert d.counter.cur_step == final and d.n_episode_sets == len([e for e in want if e[0] == "train"])
    # every test seed gets a row, at the step of its test; tests read the learner between episode sets
    tests = [e for e in want if e[0] == "test"]
    assert [c for c in ev.calls if c[0] == "perform_all"][:len(tests)] == \
        [("perform_all", s // T) for _, s in tests]
    assert len([r for r in d.data if r["test_id"] >= 0]) == 2 * len(tests)
    assert ev.env.records == ([(True, False, str(tmp_path) + "/")] if post_test else [])
    # one 'Training:' line per episode set in which the reference logs at least once
    steps = [s for k, s in want if k == "train"]
    want_log = [s for p, s in zip([0] + steps[:-1], steps) if any(p < x <= s for x in logged)]
    got_log = [int(r.getMessage().split()[3].rstrip(",")) for r in caplog.records
               if r.getMessage().startswith("Training: global step")]
    assert got_log == want_log


def test_training_rows_pool_every_replica_and_step(tmp_path):
    d, tr, ev, _ = _drive(tmp_path, 240, 120, 100, 120, "in_train_test")
    rows = [r for r in d.data if r["test_id"] == -1]
    assert [r["step"] for r in rows] == [120, 240]
    g = -(np.arange(120 * 3).reshape(120, 3) % 7) * 2.0                # episode 2 of the stub
    assert rows[1]["avg_reward"] == tr.episode_rewards[1]
    assert rows[1]["std_reward"] == np.std(g)
    test_rows = [r for r in d.data if r["test_id"] >= 0]
    assert [(r["step"], r["test_id"], r["avg_reward"], r["std_reward"]) for r in test_rows] == \
        [(120, 0, -10.0, 0.5), (120, 1, -9.0, 1.5)]


def test_train_reward_csv_has_the_reference_columns(tmp_path):
    import pandas as pd
    _drive(tmp_path, 240, 120, 100, 120, "in_train_test")
    lines = open(tmp_path / "train_reward.csv").read().splitlines()
    assert lines[0] == ",agent,step,test_id,avg_reward,std_reward"
    assert [ln.split(",")[:4] for ln in lines[1:]] == [["0", "ma2c", "120", "-1"], ["1", "ma2c", "120", "0"],
                                                      ["2", "ma2c", "120", "1"], ["3", "ma2c", "240", "-1"]]
    df = pd.read_csv(tmp_path / "train_reward.csv", index_col=0)
    assert list(df.columns) == ["agent", "step", "test_id", "avg_reward", "std_reward"]
    assert list(df.index) == [0, 1, 2, 3]


def test_agent_names_map_to_models_like_main():
    assert drv.model_spec("ia2c") == ("ia2c", None)
    assert drv.model_spec("ma2c") == ("ma2c", None)
    assert drv.model_spec("iqld") == ("iql", "dqn")
    assert drv.model_spec("iqll") == ("iql", "lr")
    assert drv.model_spec("my_agent") == ("iql", "lr")            # main.py:119-121: every other name is IQL-LR
    with pytest.raises(ValueError, match="greedy"):
        drv.model_spec("greedy")
    with pytest.raises(ValueError, match="a2c"):
        drv.model_spec("a2c")


def test_test_modes():
    assert [drv.init_test_flag(m) for m in drv.TEST_MODES] == [(False, False), (True, False), (False, True),
                                                             (True, True)]
    with pytest.raises(ValueError):
        drv.init_test_flag("sometimes")


def test_counter_logs_at_crossings():
    c = drv.Counter(1000, 100, 250)
    crossed = []
    for _ in range(8):
        prev = c.cur_step
        c.next(120)
        crossed.append(c.should_log(prev))
    assert crossed == [False, False, True, False, True, False, True, False]   # 250, 500, 750 in steps 3, 5, 7


def test_driver_refuses_a_trainer_without_a_trace():
    tr = StubTrainer(120, 2)
    tr.greward_trace = None
    with pytest.raises(ValueError, match="greward_trace"):
        drv.Trainer(tr, None, drv.Counter(240, 120, 100), "ma2c", False, "")


def test_train_rejects_greedy_before_device_work(tmp_path):
    cp = configparser.ConfigParser()
    cp.read_string("[ENV_CONFIG]\nagent = greedy\n[MODEL_CONFIG]\n[TRAIN_CONFIG]\n")
    with pytest.raises(ValueError, match="greedy"):
        drv.train(cp, str(tmp_path / "greedy"))
    assert (tmp_path / "greedy" / "data" / "config.ini").exists() and (tmp_path / "greedy" / "log").is_dir()


IQL_INI = """[MODEL_CONFIG]
lr_init = %s
lr_decay = %s
lr_min = 1e-5
epsilon_init = 1.0
epsilon_min = 0.01
epsilon_decay = %s
epsilon_ratio = 0.5
"""


def _old_iql_schedulers(mc, total_step):
    """models.IQL.__init__'s scheduler construction as it read before iql_schedulers() was factored out"""
    from deeprl_signal_control_b200.agents.utils import Scheduler
    lr_init = mc.getfloat('lr_init')
    lr_decay = mc.get('lr_decay')
    lr = Scheduler(lr_init, decay=lr_decay) if lr_decay == 'constant' else \
        Scheduler(lr_init, mc.getfloat('lr_min'), total_step, decay=lr_decay)
    eps_init = mc.getfloat('epsilon_init')
    eps_decay = mc.get('epsilon_decay')
    eps = Scheduler(eps_init, decay=eps_decay) if eps_decay == 'constant' else \
        Scheduler(eps_init, mc.getfloat('epsilon_min'), total_step * mc.getfloat('epsilon_ratio'), decay=eps_decay)
    return lr, eps


@pytest.mark.parametrize("lr_decay,eps_decay", [("constant", "linear"), ("linear", "constant"), ("linear", "linear")])
def test_iql_scheduler_builder_matches_the_old_construction(lr_decay, eps_decay):
    from deeprl_signal_control_b200.agents.models import IQL, iql_schedulers
    cp = configparser.ConfigParser()
    cp.read_string(IQL_INI % ("1e-4", lr_decay, eps_decay)
                   + "max_grad_norm = 40\ngamma = 0.99\nbatch_size = 20\nbuffer_size = 1000\nreward_norm = 3000.0\n"
                   "reward_clip = 2.0\n")
    mc, total = cp["MODEL_CONFIG"], 6000
    old = _old_iql_schedulers(mc, total)
    new = iql_schedulers(mc, total)
    m = IQL([4, 6], [2, 3], [0, 0], total, mc, seed=0, model_type="lr", device="cpu")
    for o, n, k in zip(old, new, (m.lr_scheduler, m.eps_scheduler)):
        assert (o.val, o.val_min, o.N, o.decay) == (n.val, n.val_min, n.N, n.decay) == (k.val, k.val_min, k.N, k.decay)
        for step in (1, 20, 1, 500, 2000, 4000):
            assert o.get(step) == n.get(step) == k.get(step)
