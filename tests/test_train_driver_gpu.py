"""GPU: the training driver (agents/train.py, scripts/train.py) on the grid shortened to T = 120 control steps — the
agent directory it leaves, its training rows against the per-step global rewards recorded by hand, its final weights
against the same run wired by hand, the round trip with scripts/evaluate.py, and in-training tests that equal the
post-training test of a shorter run and leave training unchanged."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 16
T = 120                                   # episode_length_sec 600 / control_interval_sec 5
SEEDS = [10000, 20000]

A2C_MODEL = """[MODEL_CONFIG]
rmsp_alpha = 0.99
rmsp_epsilon = 1e-5
max_grad_norm = 40
gamma = 0.99
lr_init = 5e-4
lr_decay = constant
entropy_coef_init = 0.01
entropy_coef_min = 0.01
entropy_decay = constant
entropy_ratio = 0.5
value_coef = 0.5
num_fw = 128
num_ft = 32
num_lstm = 64
num_fp = 64
batch_size = 120
reward_norm = 2000.0
reward_clip = 2.0
"""
IQL_MODEL = """[MODEL_CONFIG]
max_grad_norm = 40
gamma = 0.99
lr_init = 1e-4
lr_decay = constant
epsilon_init = 1.0
epsilon_min = 0.01
epsilon_decay = linear
epsilon_ratio = 0.5
num_fc = 128
num_h = 64
batch_size = 20
buffer_size = 1000
reward_norm = 3000.0
reward_clip = 2.0
"""
TRAIN = """
[TRAIN_CONFIG]
total_step = %d
test_interval = %d
log_interval = 200
"""
GRID = """
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = %s
coop_gamma = 0.9
data_path = ./large_grid/data/
episode_length_sec = 600
norm_wave = 5.0
norm_wait = 100.0
coef_wait = 0.2
peak_flow1 = 1100
peak_flow2 = 925
init_density = 0
objective = hybrid
scenario = large_grid
seed = 12
test_seeds = %s
yellow_interval_sec = 2
"""


def _ini(agent, total_step, test_interval, eps_decay="linear"):
    model = A2C_MODEL if agent in ("ia2c", "ma2c") else IQL_MODEL.replace("linear", eps_decay)
    return model + TRAIN % (total_step, test_interval) + GRID % (agent, ",".join(map(str, SEEDS)))


def _run(tmp_path, tag, agent, mode, total_step=360, test_interval=240, policy="lstm", eps_decay="linear"):
    """train() into <tmp>/<tag>/<agent> from <tmp>/<tag>/config_<agent>_large.ini"""
    from deeprl_signal_control_b200.agents.train import train
    d = tmp_path / tag
    d.mkdir()
    cfg = d / ("config_%s_large.ini" % agent)
    cfg.write_text(_ini(agent, total_step, test_interval, eps_decay))
    base = d / agent
    return base, train(str(cfg), str(base), mode, n_replicas=R, policy=policy)


def _rows(base):
    return pd.read_csv(base / "data" / "train_reward.csv", index_col=0, float_precision="round_trip")


def _weights(model):
    return (model.batched.P if model.name != "iql" else model.P).clone()


@pytest.mark.parametrize("agent,policy", [("ma2c", "lstm"), ("ia2c", "lstm"), ("ia2c", "fc"), ("iqll", "lstm"),
                                          ("iqld", "lstm")])
def test_all_test_leaves_the_agent_directory(tmp_path, monkeypatch, agent, policy):
    from deeprl_signal_control_b200.sim import BatchedSim
    rec = []                                  # every training step's global reward, recorded by hand
    step = BatchedSim.step

    def recording_step(self, *a, **k):
        out = step(self, *a, **k)
        rec.append(out[2].double().cpu().numpy().copy())
        return out
    monkeypatch.setattr(BatchedSim, "step", recording_step)
    base, out = _run(tmp_path, "run", agent, "all_test", policy=policy)
    monkeypatch.undo()
    data = base / "data"
    assert (data / ("config_%s_large.ini" % agent)).read_text() == _ini(agent, 360, 240)
    assert (base / "model" / "checkpoint-360.npz").exists()
    for kind in ("control", "traffic", "trip"):
        assert (data / ("large_grid_%s_%s.csv" % (agent, kind))).exists(), kind
    logs = glob.glob(str(base / "log" / "*.log"))
    assert len(logs) == 1 and "Training: global step 240" in open(logs[0]).read()
    assert out.final_step == 360 and out.episode_sets == 3 and out.env_samples == 360 * R
    # test at 240 (240 - 0 >= test_interval) before the third episode set; the run stops at 360 >= total_step
    df = _rows(base)
    assert list(df.columns) == ["agent", "step", "test_id", "avg_reward", "std_reward"]
    assert list(zip(df.step, df.test_id)) == [(120, -1), (240, -1), (240, 0), (240, 1), (360, -1)]
    assert (df.agent == agent).all()
    # training rows: mean / std of the per-step global rewards pooled over replicas and steps
    assert len(rec) == 3 * T
    train_rows = df[df.test_id == -1]
    for e in range(3):
        g = np.stack(rec[e * T:(e + 1) * T])                       # [T, R]
        row = train_rows.iloc[e]
        np.testing.assert_allclose(row.avg_reward, out.trainer.episode_rewards[e], rtol=1e-5)
        np.testing.assert_allclose(row.avg_reward, np.mean(g), rtol=1e-5)
        np.testing.assert_allclose(row.std_reward, np.std(g), rtol=1e-12)
    mean, std = out.post_test
    assert mean.shape == (2,) and np.isfinite(mean).all() and (std > 0).all()


def _hand_wired(agent, total_step):
    """main.py's model, seeds and schedulers wired by hand: BatchedTrainer / BatchedIQLTrainer on an R-replica env"""
    import configparser
    from deeprl_signal_control_b200.agents.utils import Scheduler
    from deeprl_signal_control_b200.envs.large_grid_env import LargeGridEnv
    cp = configparser.ConfigParser()
    cp.read_string(_ini(agent, total_step, 10 ** 9))
    env = LargeGridEnv(cp["ENV_CONFIG"], n_replicas=R)
    sim = env._ensure_sim()
    if agent == "ma2c":
        from deeprl_signal_control_b200.agents.models import MA2C
        from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
        m = MA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, env.n_f_ls, total_step, cp["MODEL_CONFIG"], seed=12, n_replicas=R,
                 obs_off=env._tables.node_obs_off)
        tr = BatchedTrainer(sim, m.batched, "ma2c", lr=Scheduler(5e-4, decay="constant"),
                            beta=Scheduler(0.01, decay="constant"), seed0=12)
    else:
        from deeprl_signal_control_b200.agents.layout import QLayout
        from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL, BatchedIQLTrainer
        t = env._tables
        off = np.asarray(t.node_obs_off)
        kind = "dqn" if agent == "iqld" else "lr"
        lay = QLayout(kind, [int(off[i + 1] - off[i]) for i in range(t.n_nodes)], t.n_a_ls, t.n_w_ls, off, t.n_obs,
                      n_fc=128, n_ft=32, n_h=64, max_na=t.max_na)
        m = BatchedIQL(lay, R, cp["MODEL_CONFIG"], kind, seed=0)
        tr = BatchedIQLTrainer(sim, m, Scheduler(1e-4, decay="constant"),
                               Scheduler(1.0, 0.01, total_step * 0.5, decay="linear"), seed0=12)
    tr.run(total_step)
    torch.cuda.synchronize()
    return m, tr


@pytest.mark.parametrize("agent", ["ma2c", "iqld", "iqll"])
def test_driver_equals_the_hand_wired_loop(tmp_path, agent):
    _, out = _run(tmp_path, "run", agent, "no_test")
    m, tr = _hand_wired(agent, 360)
    assert tr.n_env_steps == out.trainer.n_env_steps == 360 and tr.n_updates == out.trainer.n_updates
    got, want = _weights(out.model), _weights(m)
    if agent == "ma2c":
        # the weight-gradient kernels add with atomics: two runs of one build differ by a few 1e-8 (DESIGN.md §5)
        assert float((got - want).abs().max()) <= 1e-6
        np.testing.assert_allclose(out.trainer.episode_rewards, tr.episode_rewards, rtol=1e-5)
    else:
        assert torch.equal(got, want) and out.trainer.episode_rewards == tr.episode_rewards
        assert torch.equal(out.model.M, m.M) and torch.equal(out.model.V, m.V) and out.model.t == m.t > 0


@pytest.mark.parametrize("agent", ["ma2c", "iqld"])
def test_post_training_test_equals_evaluate_script(tmp_path, agent):
    base, out = _run(tmp_path, "run", agent, "after_train_test", total_step=240)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", str(base),
                        "--evaluation-policy-type", "default"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    got = json.load(open(base / "eva_data" / ("%s_summary.json" % agent)))
    mean, std = out.post_test
    assert got["seeds"] == SEEDS
    assert got["episode_mean_reward"] == [float(x) for x in mean]
    assert got["episode_std_reward"] == [float(x) for x in std]
    for kind in ("control", "traffic"):
        name = "large_grid_%s_%s.csv" % (agent, kind)
        assert (base / "data" / name).read_text() == (base / "eva_data" / name).read_text(), kind


def test_in_training_tests_equal_a_shorter_runs_post_test_and_leave_training_alone(tmp_path):
    # a constant ε: the linear schedule decays over total_step * epsilon_ratio, so runs of different total_step would
    # not train alike up to step 240
    base, a = _run(tmp_path, "a", "iqll", "in_train_test", total_step=360, test_interval=120, eps_decay="constant")
    df = _rows(base)
    assert list(zip(df.step, df.test_id)) == [(120, -1), (120, 0), (120, 1), (240, -1), (240, 0), (240, 1), (360, -1)]
    _, b = _run(tmp_path, "b", "iqll", "after_train_test", total_step=240, eps_decay="constant")
    assert b.trainer.episode_rewards == a.trainer.episode_rewards[:2]
    at240 = df[(df.step == 240) & (df.test_id >= 0)]
    assert list(at240.avg_reward) == [float(x) for x in b.post_test[0]]
    assert list(at240.std_reward) == [float(x) for x in b.post_test[1]]
    _, c = _run(tmp_path, "c", "iqll", "no_test", total_step=360, eps_decay="constant")
    assert torch.equal(a.model.P, c.model.P) and torch.equal(a.model.M, c.model.M)
    assert a.trainer.episode_rewards == c.trainer.episode_rewards
    assert list(df[df.test_id == -1].avg_reward) == c.trainer.episode_rewards


def test_train_script_round_trip(tmp_path):
    """scripts/train.py --base-dir DIR train ... then scripts/evaluate.py --agent-dir DIR"""
    cfg = tmp_path / "config_ia2c_large.ini"
    cfg.write_text(_ini("ia2c", 240, 120))
    base = tmp_path / "ia2c"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "train.py"), "--base-dir", str(base), "train",
                        "--config-dir", str(cfg), "--test-mode", "all_test", "--replicas", "8", "--policy", "fc"],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert (line["final_step"], line["episode_sets"], line["env_samples"]) == (240, 2, 240 * 8)
    assert "Testing: global step 120" in r.stderr
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", str(base),
                        "--policy", "fc"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    assert (base / "eva_data" / "large_grid_ia2c_control.csv").read_text() == \
        (base / "data" / "large_grid_ia2c_control.csv").read_text()
