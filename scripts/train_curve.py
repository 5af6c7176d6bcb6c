"""Training curves of the device-resident learner on the restated simulator, and the greedy controller's score on the
same episodes (reference utils.py:296-305: mean over the 720 control steps of the global reward, averaged over replicas).

  python scripts/train_curve.py --replicas 512 --episodes 300 --agent ma2c [--scenario grid|real] [--policy lstm|fc]
                                [--fp32] [--reward-norm X] [--lr X] [--tag NAME] [--greedy]
  python scripts/train_curve.py --replicas 4096 --episodes 20 --agent iqll|iqld [--scenario grid|real] [--eval-seeds S,..]

--agent iqll / iqld  IQL-LR / IQL-DQN on the batched IQL learner (agents/learner_iql.py) with the MODEL_CONFIG of the
               reference's config_iql{l,d}_{large,real}.ini, then test-mode evaluation of the trained weights on
               --eval-seeds through the batched evaluator
--fp32         plain fp32 learner kernels (no tensor cores, no bf16 activation store): the A/B partner of the default path
--reward-norm  override MODEL_CONFIG.reward_norm (reference: 2000 for MA2C on the grid, config/config_ma2c_large.ini)
--greedy       no learning: the reference's greedy controller (envs/large_grid_env.py:56-60, envs/real_net_env.py:78-111)
               on the same seeds, through the batched evaluator (agents/evaluator.py)
Writes $OUT/train_curve_<tag>.json (OUT defaults to results/).
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from deeprl_signal_control_b200.agents.layout import PolicyLayout
from deeprl_signal_control_b200.agents.learner import BatchedA2C
from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
from deeprl_signal_control_b200.dist import episode_seeds
from deeprl_signal_control_b200.net.large_grid import build_large_grid
from deeprl_signal_control_b200.net.tables import EnvParams
from deeprl_signal_control_b200.sim import BatchedSim



GREEDY_INI = {"grid": """
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = greedy
coop_gamma = 0.9
data_path = ./large_grid/data/
episode_length_sec = 3600
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
""", "real": """
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = greedy
coop_gamma = 0.9
data_path = ./real_net/data/
episode_length_sec = 3600
norm_wave = 5.0
norm_wait = 30.0
coef_wait = 0
flow_rate = 325
objective = queue
scenario = real_net
seed = 12
test_seeds = %s
yellow_interval_sec = 2
"""}


def out_path(tag):
    out = os.environ.get("OUT", "results")
    os.makedirs(out, exist_ok=True)
    return os.path.join(out, "train_curve_%s.json" % tag)


p = argparse.ArgumentParser()
p.add_argument("--replicas", type=int, default=512)
p.add_argument("--episodes", type=int, default=24)
p.add_argument("--agent", default="ma2c")
p.add_argument("--scenario", default="grid", choices=["grid", "real"])
p.add_argument("--policy", default="lstm", choices=["lstm", "fc"])
p.add_argument("--fp32", action="store_true")
p.add_argument("--reward-norm", type=float, default=None)
p.add_argument("--lr", type=float, default=None, help="default 5e-4 (A2C), 1e-4 (IQL)")
p.add_argument("--eval-seeds", default="10000,20000", help="IQL: test seeds of the evaluation after training")
p.add_argument("--seed", type=int, default=1)
p.add_argument("--tag", default=None)
p.add_argument("--greedy", action="store_true")
a = p.parse_args()
R, agent = a.replicas, a.agent
tag = a.tag or ("%s_%s" % (agent, a.scenario) if agent in ("iqll", "iqld") else
                "%s_%s_%s%s" % (agent, a.scenario, a.policy, "_fp32" if a.fp32 else ""))

if a.scenario == "real":
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    net = real_net_tables("greedy" if a.greedy else agent)
    par = EnvParams(agent="greedy" if a.greedy else agent, objective="queue", norm_wave=5.0, norm_wait=30.0, clip_wave=2.0,
                    clip_wait=2.0, coef_wait=0.0, coop_gamma=0.9, teleport_sec=300, real_net_norm=True, use_wait=False,
                    det_len=-1.0, halt_speed=0.1, queue_cap=10)
    n_step, reward_norm = 40, 1.0
else:
    net = build_large_grid(agent="greedy" if a.greedy else agent)
    par = EnvParams(agent="greedy" if a.greedy else agent)
    n_step, reward_norm = 120, 2000.0 if agent == "ma2c" else 3000.0
if a.reward_norm is not None:
    reward_norm = a.reward_norm
sim = BatchedSim(net, par, R)
t0 = time.time()

if a.greedy:
    # the batched evaluator's greedy path (tsc_greedy_actions) on the training seeds of every episode; the greedy agent's
    # rewards are the same in train and test mode (local rewards, envs/env.py:591-594)
    import configparser
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    cp = configparser.ConfigParser()
    cp.read_string(GREEDY_INI[a.scenario] % ",".join(["0"] * R))
    if a.scenario == "real":
        from deeprl_signal_control_b200.envs.real_net_env import RealNetController, RealNetEnv
        env = RealNetEnv(cp["ENV_CONFIG"], n_replicas=R)
        ctrl = RealNetController(env.node_names, env.nodes)
    else:
        from deeprl_signal_control_b200.envs.large_grid_env import LargeGridController, LargeGridEnv
        env = LargeGridEnv(cp["ENV_CONFIG"], n_replicas=R)
        ctrl = LargeGridController(env.node_names)
    ev = Evaluator(env, ctrl, "", policy_type="deterministic")
    curve = []
    for ep in range(a.episodes):
        env.init_test_seeds([int(x) for x in episode_seeds(12, ep, 0, R, R)])
        mean, _ = ev.perform_all()
        curve.append(float(np.mean(mean)))
        print("greedy episode %3d  mean step reward %9.2f" % (ep + 1, curve[-1]), flush=True)
    json.dump({"agent": "greedy", "scenario": a.scenario, "replicas": R, "episodes": len(curve), "mean_episode_reward": curve,
               "wall_s": time.time() - t0}, open(out_path(tag), "w"))
    sys.exit(0)

if agent in ("iqll", "iqld"):
    # reference config/config_iql{l,d}_{large,real}.ini, MODEL_CONFIG
    import configparser
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    from deeprl_signal_control_b200.agents.layout import QLayout
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL, BatchedIQLTrainer
    from deeprl_signal_control_b200.agents.utils import Scheduler
    kind = "dqn" if agent == "iqld" else "lr"
    lr = 1e-4 if a.lr is None else a.lr
    rn = (1.0 if a.scenario == "real" else 3000.0) if a.reward_norm is None else a.reward_norm
    cp = configparser.ConfigParser()
    cp.read_string("[MODEL_CONFIG]\nmax_grad_norm = 40\ngamma = 0.99\nnum_fc = 128\nnum_h = 64\nbatch_size = 20\n"
                   "buffer_size = 1000\nreward_norm = %r\nreward_clip = 2.0\n" % rn)
    total_step = 1e6
    off = np.asarray(net.node_obs_off)
    qlay = QLayout(kind, [int(off[i + 1] - off[i]) for i in range(net.n_nodes)], net.n_a_ls, net.n_w_ls, off, net.n_obs,
                   n_fc=128, n_ft=32, n_h=64, max_na=net.max_na)
    model = BatchedIQL(qlay, R, cp["MODEL_CONFIG"], kind, seed=a.seed)
    tr = BatchedIQLTrainer(sim, model, Scheduler(lr, decay="constant"), Scheduler(1.0, 0.01, total_step * 0.5), seed0=12)
    curve = []
    while len(tr.episode_rewards) < a.episodes:
        tr.run(tr.T_episode)
        torch.cuda.synchronize()
        curve = list(tr.episode_rewards)
        print("episode %3d  mean step reward %9.2f   loss[0] %.4g   grad-norm[0] %.3f   %.1fs" %
              (len(curve), curve[-1], float(model.losses[-1, 0]), float(model.norms[-1, 0]), time.time() - t0), flush=True)
    seeds = [int(x) for x in a.eval_seeds.split(",")]
    ecp = configparser.ConfigParser()
    ecp.read_string(GREEDY_INI[a.scenario].replace("agent = greedy", "agent = " + agent) % ",".join(map(str, seeds)))
    if a.scenario == "real":
        from deeprl_signal_control_b200.envs.real_net_env import RealNetEnv as Env
    else:
        from deeprl_signal_control_b200.envs.large_grid_env import LargeGridEnv as Env
    env = Env(ecp["ENV_CONFIG"], n_replicas=len(seeds))
    mean, std = Evaluator(env, model, "", policy_type="default").perform_all()
    print("evaluation on seeds %s: mean step reward %s" % (seeds, np.round(mean, 2).tolist()), flush=True)
    json.dump({"agent": agent, "scenario": a.scenario, "replicas": R, "episodes": len(curve), "lr": lr, "reward_norm": rn,
               "mean_episode_reward": curve, "eval_seeds": seeds, "eval_mean": [float(x) for x in mean],
               "eval_std": [float(x) for x in std], "wall_s": time.time() - t0, "env_steps": tr.n_env_steps},
              open(out_path(tag), "w"))
    sys.exit(0)

a.lr = 5e-4 if a.lr is None else a.lr
lay = PolicyLayout(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, net.node_obs_off, net.n_obs, fw=128, ft=32,
                   ff=64 if agent == "ma2c" else 0, h=64, max_na=net.max_na, recurrent=a.policy != "fc")
kw = dict(use_tc=False, allow_tf32=False) if a.fp32 else {}
if a.policy == "fc":
    from deeprl_signal_control_b200.agents.learner_fc import BatchedFcA2C as Learner
    kw = {}
else:
    Learner = BatchedA2C
model = Learner(lay, R, n_step=n_step, gamma=0.99, v_coef=0.5, max_grad_norm=40.0, alpha=0.99, eps=1e-5,
                reward_norm=reward_norm, reward_clip=2.0, seed=a.seed, chunk=min(R, 1024), **kw)
tr = BatchedTrainer(sim, model, agent, lr=a.lr, beta=0.01, seed0=12)
curve = []
while len(tr.episode_rewards) < a.episodes:
    tr.run(720)
    torch.cuda.synchronize()
    curve = list(tr.episode_rewards)
    if len(curve) % 10 == 0 or len(curve) == a.episodes:
        print("episode %3d  mean step reward %9.2f   grad-norm[0] %.3f   %.1fs" %
              (len(curve), curve[-1], float(model.norms[0]), time.time() - t0), flush=True)
json.dump({"agent": agent, "scenario": a.scenario, "policy": a.policy, "replicas": R, "episodes": len(curve),
           "fp32": bool(a.fp32), "reward_norm": reward_norm, "lr": a.lr, "mean_episode_reward": curve,
           "wall_s": time.time() - t0, "env_steps": tr.n_env_steps},
          open(out_path(tag), "w"))
