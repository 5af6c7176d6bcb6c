"""Measure batched test-mode evaluation (deeprl_signal_control_b200/agents/evaluator.py) on the GPU:

    python scripts/profile_evaluate.py [--launches N] [--ref-seconds S]

1. The pi-only policy forward (tscl_policy_step_pi, argmax actions) against the training forward without the activation
   store (tscl_policy_step_v2, both networks, sampled actions), on the same inputs: grid MA2C (R = 4096) and Monaco MA2C
   (R = 2048), N launches each after a warm-up, CUDA events; the HBM bytes each has to move (computed from the shapes:
   every operand read once, every result written once) and the achieved GB/s.
2. Evaluation throughput of whole 3600-s episodes (one untimed episode first), timed from the first launch to the
   synchronising copy of the reward trace: grid MA2C deterministic at R = 4096 with and without record mode, Monaco
   MA2C at R = 2048, grid greedy at R = 4096; agent-env-steps/s = R x agents x control steps / time, and episodes/hour.
3. The one-seed-at-a-time reference protocol (utils.py:Tester.perform on the one-replica env + MA2C wrapper) on the grid:
   the user-visible "before", timed over the first S seconds of one episode and scaled to 720 control steps.
4. IQL: the fp32 Q forward (tscl_q_step, argmax actions) alone for LR and DQN, grid R = 4096 and Monaco R = 2048, CUDA
   events, with the FLOPs and HBM bytes of one launch computed from the shapes; and whole 3600-s episodes of grid IQL-LR
   / IQL-DQN at R = 4096 and Monaco IQL-LR / IQL-DQN at R = 2048 (--iql-only: this part alone).
The card and its power limit are read in the same run.
"""
import argparse
import configparser
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import build_scenario, make_layout  # noqa: E402
from deeprl_signal_control_b200 import _lib  # noqa: E402
from deeprl_signal_control_b200.agents.learner import BatchedA2C, _p  # noqa: E402

MODEL_INI = """
[MODEL_CONFIG]
rmsp_alpha = 0.99
rmsp_epsilon = 1e-5
max_grad_norm = 40
gamma = 0.99
value_coef = 0.5
num_fw = 128
num_ft = 32
num_lstm = 64
num_fp = 64
batch_size = 120
reward_norm = 2000.0
reward_clip = 2.0
"""
ENV_INI = {"large_grid": """
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = %s
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
""", "real_net": """
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = %s
coop_gamma = 0.9
data_path = ./real_net/data/
episode_length_sec = 3600
norm_wave = 5.0
norm_wait = 100.0
coef_wait = 0
flow_rate = 325
objective = queue
scenario = real_net
seed = 42
test_seeds = %s
yellow_interval_sec = 2
"""}


def forward_bytes(lay, R, units):
    """Essential HBM traffic of one launch (bytes): observations, c/h in and out of `units` networks, pi + one int32
    action per agent, and the value per agent when both networks run."""
    b = R * lay.n_obs * 4 + 4 * units * R * lay.h * 4 + R * lay.A * (lay.max_na * 4 + 4)
    return b + (R * lay.A * 4 if units == lay.U else 0)


def time_kernels(scenario, R, launches, warmup):
    class _A:
        agent, policy = "ma2c", "lstm"
    _A.scenario = scenario
    lay = make_layout(build_scenario(_A)[0], _A)
    m = BatchedA2C(lay, R, n_step=2, seed=1, chunk=1024, store_acts=False)
    assert m.tc_v2
    g = torch.Generator(device="cuda").manual_seed(0)
    obs = torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2
    c, h = torch.zeros(lay.A, R, lay.h, device="cuda"), torch.zeros(lay.A, R, lay.h, device="cuda")
    pi, act = torch.zeros_like(m.pi), torch.zeros_like(m.act)
    lib = _lib.lib()

    def full():
        _lib.check(lib.tscl_policy_step_v2(m._h, _p(m.P), _p(m.Wp), _p(obs), R, _p(m.c_fw), _p(m.h_fw), _p(m.c_fw),
                                           _p(m.h_fw), _p(m.pi), _p(m.val), _p(m.act), 0, 1, 0, 0, None, None, None,
                                           None, None, 0, 1, R, m._st()))

    def pi_only():
        _lib.check(lib.tscl_policy_step_pi(m._h, _p(m.P), _p(m.Wp), _p(obs), R, _p(c), _p(h), _p(c), _p(h), _p(pi),
                                           _p(act), 1, 0, 1, 0, 0, 0, 0, m._st()))

    res = {}
    for rep in range(2):                       # alternate the two kernels; report the second round
        for name, fn, units in (("v2 (pi + V, no store)", full, lay.U), ("pi-only", pi_only, lay.A)):
            for _ in range(warmup):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                fn()
            e1.record()
            torch.cuda.synchronize()
            res[name] = (e0.elapsed_time(e1) / launches, forward_bytes(lay, R, units))
    for name, (ms, b) in res.items():
        print("  %-22s %s R = %d, dx = %d: %.4f ms per launch (%d launches), %.0f MB, %.0f GB/s"
              % (name, scenario, R, lay.dx, ms, launches, b / 1e6, b / (ms * 1e-3) / 1e9))
    print("  pi-only / v2 time: %.3f" % (res["pi-only"][0] / res["v2 (pi + V, no store)"][0]))


def make(scenario, agent, R, record):
    from deeprl_signal_control_b200.agents.models import MA2C
    cp = configparser.ConfigParser()
    cp.read_string(ENV_INI[scenario] % (agent, ",".join(str(10000 + 7 * k) for k in range(R))) + MODEL_INI)
    if scenario == "large_grid":
        from deeprl_signal_control_b200.envs.large_grid_env import LargeGridController, LargeGridEnv as Env
    else:
        from deeprl_signal_control_b200.envs.real_net_env import RealNetController, RealNetEnv as Env
    env = Env(cp["ENV_CONFIG"], output_path="", is_record=record, n_replicas=R)
    if agent == "greedy":
        model = LargeGridController(env.node_names) if scenario == "large_grid" else RealNetController(env.node_names, env.nodes)
    else:
        model = MA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, env.n_f_ls, 0, cp["MODEL_CONFIG"], seed=1, n_replicas=1,
                     obs_off=env._tables.node_obs_off)
    return env, model


def time_evaluation(name, scenario, agent, R, record):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    env, model = make(scenario, agent, R, record)
    ev = Evaluator(env, model, "", policy_type="deterministic")
    ev.perform_all()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mean, _ = ev.perform_all()               # ends with the device -> host copy of the reward trace
    el = time.perf_counter() - t0
    steps = R * env._tables.n_nodes * ev.T
    print("  %-40s R = %d: %.3f s per episode set (%d control steps), %.3g agent-env-steps/s, %.0f episodes/hour; "
          "mean step reward %.2f" % (name, R, el, ev.T, steps / el, R / el * 3600, float(np.mean(mean))))
    del ev, env, model
    torch.cuda.empty_cache()


def time_reference(budget_s):
    """Tester.perform (utils.py:195-234) on the one-replica env: forward 'p' + host argmax + env.step per control step."""
    env, model = make("large_grid", "ma2c", 1, False)
    env.train_mode = False
    ob = env.reset(test_ind=0)
    done, n = True, 0
    model.reset()
    t0 = time.perf_counter()
    while time.perf_counter() - t0 < budget_s and n < 720:
        policy = model.forward(ob, done, 'p')
        env.update_fingerprint(policy)
        ob, reward, done, greward = env.step([int(np.argmax(np.array(p))) for p in policy])
        n += 1
    el = time.perf_counter() - t0
    per_ep = el / n * 720
    print("  one-seed reference protocol, grid MA2C: %d control steps in %.2f s -> %.1f s per 720-step episode, "
          "%.3g agent-env-steps/s, %.0f episodes/hour" % (n, el, per_ep, 25 * 720 / per_ep, 3600 / per_ep))


IQL_INI = """
[MODEL_CONFIG]
gamma = 0.99
max_grad_norm = 40
batch_size = 20
reward_norm = 2000.0
reward_clip = 2.0
num_fc = 128
num_h = 64
"""


def q_cost(lay, R):
    """(FLOPs, HBM bytes) of one tscl_q_step launch: 2 x multiply-adds of every layer; observations read once, q, the
    actions and the parameters moved once"""
    mac = 0
    for i in range(lay.A):
        n_s, n_a, n_w = int(lay.n_s[i]), int(lay.n_a[i]), int(lay.n_w[i])
        if lay.model_type == "lr":
            mac += n_s * n_a
        else:
            ft = lay.n_ft if n_w > 0 else 0
            mac += (n_s - n_w) * lay.n_fc + n_w * ft + (lay.n_fc + ft) * lay.n_h + lay.n_h * n_a
    return 2 * R * mac, R * lay.n_obs * 4 + R * lay.A * (lay.max_na + 1) * 4 + lay.n_params * 4


def make_iql(scenario, agent, R):
    from deeprl_signal_control_b200.agents.models import IQL
    cp = configparser.ConfigParser()
    cp.read_string(ENV_INI[scenario] % (agent, ",".join(str(10000 + 7 * k) for k in range(R))) + IQL_INI)
    if scenario == "large_grid":
        from deeprl_signal_control_b200.envs.large_grid_env import LargeGridEnv as Env
    else:
        from deeprl_signal_control_b200.envs.real_net_env import RealNetEnv as Env
    env = Env(cp["ENV_CONFIG"], output_path="", is_record=False, n_replicas=R)
    model = IQL(env.n_s_ls, env.n_a_ls, env.n_w_ls, 0, cp["MODEL_CONFIG"], seed=1,
                model_type="dqn" if agent == "iqld" else "lr", device="cuda")
    return env, model


def time_q_kernel(scenario, agent, R, launches, warmup):
    from deeprl_signal_control_b200.agents.layout import QLayout
    env, model = make_iql(scenario, agent, 1)
    net = env._tables
    lay = QLayout.from_iql(model, net.node_obs_off, net.n_obs, max_na=net.max_na)
    h = C.c_void_p()
    lib = _lib.lib()
    _lib.check(lib.tscl_q_create(C.byref(lay.as_c()), 0, C.byref(h)))
    P = lay.pack(model.nets)
    g = torch.Generator(device="cuda").manual_seed(0)
    obs = torch.rand(R, net.n_obs, device="cuda", generator=g) * 2
    q = torch.zeros(R, lay.A, lay.max_na, device="cuda")
    act = torch.zeros(R, lay.A, dtype=torch.int32, device="cuda")
    st = _lib.stream()

    def fn():
        _lib.check(lib.tscl_q_step(h, _p(P), _p(obs), R, _p(q), _p(act), 0, 1, 0, 0, None, st))
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / launches
    flops, b = q_cost(lay, R)
    print("  Q forward %-4s %s R = %d: %.4f ms per launch (%d launches), %.2f GFLOP, %.1f MB -> %.1f TFLOP/s, %.0f GB/s"
          % (lay.model_type, scenario, R, ms, launches, flops / 1e9, b / 1e6, flops / (ms * 1e-3) / 1e12,
             b / (ms * 1e-3) / 1e9))
    lib.tscl_q_destroy(h)


def time_iql_evaluation(name, scenario, agent, R):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    env, model = make_iql(scenario, agent, R)
    ev = Evaluator(env, model, "", policy_type="default")
    ev.perform_all()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mean, _ = ev.perform_all()
    el = time.perf_counter() - t0
    steps = R * env._tables.n_nodes * ev.T
    print("  %-40s R = %d: %.3f s per episode set (%d control steps), %.3g agent-env-steps/s, %.0f episodes/hour; "
          "mean step reward %.2f" % (name, R, el, ev.T, steps / el, R / el * 3600, float(np.mean(mean))))
    del ev, env, model
    torch.cuda.empty_cache()


def time_iql(launches, warmup):
    print("IQL Q forward alone (fp32 SIMT, argmax actions):")
    for scenario, R in (("large_grid", 4096), ("real_net", 2048)):
        for agent in ("iqll", "iqld"):
            time_q_kernel(scenario, agent, R, launches, warmup)
    print("IQL evaluation, whole 3600-s episodes (untrained weights):")
    time_iql_evaluation("grid IQL-LR", "large_grid", "iqll", 4096)
    time_iql_evaluation("grid IQL-DQN", "large_grid", "iqld", 4096)
    time_iql_evaluation("Monaco IQL-LR", "real_net", "iqll", 2048)
    time_iql_evaluation("Monaco IQL-DQN", "real_net", "iqld", 2048)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--launches", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--ref-seconds", type=float, default=20.0)
    p.add_argument("--iql-only", action="store_true")
    a = p.parse_args()
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("card: %s" % smi)
    if a.iql_only:
        time_iql(a.launches, a.warmup)
        return
    print("policy forward alone:")
    time_kernels("large_grid", 4096, a.launches, a.warmup)
    time_kernels("real_net", 2048, a.launches, a.warmup)
    print("evaluation, whole 3600-s episodes (untrained weights: the work per step does not depend on them):")
    time_evaluation("grid MA2C deterministic", "large_grid", "ma2c", 4096, False)
    time_evaluation("grid MA2C deterministic, record mode", "large_grid", "ma2c", 4096, True)
    time_evaluation("Monaco MA2C deterministic", "real_net", "ma2c", 2048, False)
    time_evaluation("grid greedy", "large_grid", "greedy", 4096, False)
    print("before:")
    time_reference(a.ref_seconds)
    time_iql(a.launches, a.warmup)


if __name__ == "__main__":
    main()
