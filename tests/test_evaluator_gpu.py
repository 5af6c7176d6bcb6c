"""GPU: batched test-mode evaluation (agents/evaluator.py) — the pi-only policy forward (tscl_policy_step_pi) against the
training forward, the greedy-controller kernel (tsc_greedy_actions) against the controllers, end-to-end parity of the
evaluator with the reference's one-seed-at-a-time protocol (utils.py:Tester.perform / Evaluator.run), isolation from a
live learner, and scripts/evaluate.py on a saved checkpoint."""
import configparser
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "fixtures"))

MODEL_INI = """
[MODEL_CONFIG]
rmsp_alpha = 0.99
rmsp_epsilon = 1e-5
max_grad_norm = 40
gamma = 0.99
lr_init = 5e-4
lr_decay = constant
entropy_coef_init = 0.01
entropy_decay = constant
value_coef = 0.5
num_fw = 128
num_ft = 32
num_lstm = 64
num_fp = 64
batch_size = 20
reward_norm = 2000.0
reward_clip = 2.0
"""
GRID_INI = """
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = %s
coop_gamma = 0.9
data_path = ./large_grid/data/
episode_length_sec = %d
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
REAL_INI = """
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = %s
coop_gamma = 0.9
data_path = ./real_net/data/
episode_length_sec = %d
norm_wave = 5.0
norm_wait = 100.0
coef_wait = 0
flow_rate = 325
objective = queue
scenario = real_net
seed = 42
test_seeds = %s
yellow_interval_sec = 2
"""


def _pmix(h):
    h = h ^ (h >> np.uint32(16)); h = h * np.uint32(0x7feb352d); h = h ^ (h >> np.uint32(15))
    h = h * np.uint32(0x846ca68b); return h ^ (h >> np.uint32(16))


def _reference_actions(pi, n_a, seed, step, replica0):
    """inverse-CDF sample of the kernel: hash of (seed, step, replica, agent), cumulative sum of pi in fp32"""
    with np.errstate(over="ignore"):
        R, A, _ = pi.shape
        r = np.arange(R, dtype=np.uint64) + np.uint64(replica0)
        h0 = _pmix(np.uint32(seed & 0xFFFFFFFF) ^ (np.uint32(step) * np.uint32(0x9E3779B1)))
        h1 = _pmix(h0 ^ np.uint32(seed >> 32) ^ (r.astype(np.uint32) * np.uint32(0x85EBCA77)))
        act = np.zeros((R, A), np.int32)
        for a in range(A):
            h = _pmix(h1 ^ np.uint32(a * 0xC2B2AE3D & 0xFFFFFFFF))
            uu = (h >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
            na = int(n_a[a])
            cum = np.cumsum(pi[:, a, :na], axis=1, dtype=np.float32)
            hit = uu[:, None] < cum
            act[:, a] = np.where(hit.any(1), hit.argmax(1), na - 1)
    return act


def _argmax(pi, n_a):
    return np.stack([np.argmax(pi[:, a, :int(na)], axis=1) for a, na in enumerate(n_a)], 1).astype(np.int32)


def _pi_step(m, obs, c, h, c_out, h_out, pi, act, mode, done, step, r0=0, n=None, ld=0):
    """tscl_policy_step_pi on replicas [r0, r0 + n) (compact state [A][R][h])"""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    L, R = m.lay, m.R
    n = R if n is None else n
    off = lambda t, per_row: C.c_void_p(t.data_ptr() + r0 * per_row * t.element_size())
    _lib.check(_lib.lib().tscl_policy_step_pi(
        m._h, _p(m.P), _p(m.Wp), off(obs, L.n_obs), C.c_int64(n), off(c, L.h), off(h, L.h), off(c_out, L.h),
        off(h_out, L.h), off(pi, L.A * L.max_na), off(act, L.A), C.c_int32(mode), C.c_int32(int(done)),
        C.c_uint64(m.seed), C.c_int64(step), C.c_int64(r0), C.c_int64(ld), C.c_int64(r0 if ld else 0), m._st()))


@pytest.mark.parametrize("scenario,agent,R", [("large_grid", "ma2c", 4096), ("real_net", "ma2c", 2048),
                                              ("large_grid", "ia2c", 4096)])
def test_pi_only_forward_matches_training_forward(scenario, agent, R):
    from bench import build_scenario, make_layout
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import BatchedA2C, _p

    class A:
        policy = "lstm"
    A.scenario, A.agent = scenario, agent
    lay = make_layout(build_scenario(A)[0], A)
    m = BatchedA2C(lay, R, n_step=2, seed=5, chunk=1024, store_acts=False)
    assert m.tc_v2 and lay.dx == {"ma2c": 224 if scenario == "large_grid" else 192, "ia2c": 160}[agent]
    g = torch.Generator(device="cuda").manual_seed(3)
    m.P.add_(torch.randn(m.P.shape, device="cuda", generator=g) * 0.02)     # weights away from the initialisation
    m.pack_weights()
    m.h_fw.copy_(torch.rand(m.h_fw.shape, device="cuda", generator=g) * 2 - 1)
    m.c_fw.copy_(torch.randn(m.c_fw.shape, device="cuda", generator=g))
    c, h = m.c_fw[0::2].clone(), m.h_fw[0::2].clone()
    c1, h1 = torch.empty_like(c), torch.empty_like(h)
    pi = torch.empty_like(m.pi)
    act_max = torch.empty_like(m.act); act_smp = torch.empty_like(m.act)
    for step, done in enumerate([True, False, False]):
        obs = torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2
        _lib.check(_lib.lib().tscl_policy_step_v2(
            m._h, _p(m.P), _p(m.Wp), _p(obs), C.c_int64(R), _p(m.c_fw), _p(m.h_fw), _p(m.c_tmp), _p(m.h_tmp), _p(m.pi),
            _p(m.val), _p(m.act), C.c_int32(int(done)), C.c_uint64(m.seed), C.c_int64(step), C.c_int64(0), None,
            None, None, None, None, C.c_int32(0), C.c_int32(2), C.c_int64(R), m._st()))
        pi.fill_(float("nan")); c1.fill_(float("nan")); h1.fill_(float("nan"))
        _pi_step(m, obs, c, h, c1, h1, pi, act_max, 1, done, step)
        pi2, c2, h2 = torch.empty_like(pi), torch.empty_like(c1), torch.empty_like(h1)
        _pi_step(m, obs, c, h, c2, h2, pi2, act_smp, 0, done, step)
        torch.cuda.synchronize()
        # bit-identical to the pi units of the training forward
        assert torch.equal(pi, m.pi) and torch.equal(pi2, m.pi)
        assert torch.equal(c1, m.c_tmp[0::2]) and torch.equal(h1, m.h_tmp[0::2])
        assert torch.equal(c2, c1) and torch.equal(h2, h1)
        p = pi.cpu().numpy()
        np.testing.assert_array_equal(act_max.cpu().numpy(), _argmax(p, lay.n_a))
        np.testing.assert_array_equal(act_smp.cpu().numpy(), _reference_actions(p, lay.n_a, m.seed, step, 0))
        assert torch.equal(act_smp, m.act)
        # uneven replica ranges reproduce the full launch bit for bit, in both action modes
        for mode, want in ((1, act_max), (0, act_smp)):
            cr, hr, pr = (torch.full_like(x, float("nan")) for x in (c1, h1, pi))
            ar = torch.full_like(act_max, -1)
            bounds = [0, R // 4 - 24, R // 2 + 52, 3 * R // 4 + 7, R]
            for r0, r1 in zip(bounds[:-1], bounds[1:]):
                _pi_step(m, obs, c, h, cr, hr, pr, ar, mode, done, step, r0=r0, n=r1 - r0, ld=R)
            torch.cuda.synchronize()
            assert torch.equal(cr, c1) and torch.equal(hr, h1) and torch.equal(pr, pi) and torch.equal(ar, want)
        m.c_fw.copy_(m.c_tmp); m.h_fw.copy_(m.h_tmp)
        c.copy_(c1); h.copy_(h1)


def _controller(scenario, env=None, net=None, tmp_path=None):
    from deeprl_signal_control_b200.envs.env import Node
    from deeprl_signal_control_b200.envs.large_grid_env import LargeGridController
    from deeprl_signal_control_b200.envs.real_net_env import RealNetController
    from deeprl_signal_control_b200.envs.small_grid_env import SmallGridController
    if scenario == "grid":
        return LargeGridController(net.node_names)
    if scenario == "small":
        return SmallGridController(net.node_names)
    nodes = {}
    for name in net.node_names:
        nd = Node(name)
        nd.lanes_in, nd.ilds_in = net.lanes_in[name], net.ilds_in[name]
        nodes[name] = nd
    return RealNetController(net.node_names, nodes)


def _forward(ctrl, net, obs):
    off = net.node_obs_off
    return np.array([[int(a) for a in ctrl.forward([row[off[i]:off[i + 1]].astype(np.float64) for i in range(net.n_nodes)])]
                     for row in obs], np.int32)


@pytest.mark.parametrize("scenario", ["grid", "monaco", "small", "mini_sumo"])
def test_greedy_kernel_equals_controllers_on_simulated_observations(scenario, tmp_path):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    if scenario == "grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid
        net, par = build_large_grid(agent="greedy"), EnvParams(agent="greedy")
        ctrl = _controller(scenario, net=net)
    elif scenario == "monaco":
        from deeprl_signal_control_b200.net.real_net import real_net_tables
        from tests.test_real_net_cpu import real_params
        net, par = real_net_tables("greedy"), real_params("greedy")
        ctrl = _controller(scenario, net=net)
    elif scenario == "small":
        from deeprl_signal_control_b200.net.small_grid import build_small_grid
        net = build_small_grid(agent="greedy")
        par = EnvParams(agent="greedy", norm_wave=1.0, norm_wait=1.0, clip_wave=1000.0, clip_wait=1000.0)
        ctrl = _controller(scenario, net=net)
    else:
        from tests.test_evaluator_cpu import _mini_sumo
        ctrl, net = _mini_sumo(tmp_path)
        par = EnvParams(agent="greedy", episode_length_sec=900)
    R = 1024
    sim = BatchedSim(net, par, R)
    sim.reset(np.arange(R, dtype=np.uint64) * np.uint64(3) + np.uint64(101)); sim.set_train_mode(False)
    prog = ctrl.greedy_program(net.node_obs_off)
    ip = lambda a: np.ascontiguousarray(a, np.int32).ctypes.data_as(C.POINTER(C.c_int32))
    arrs = [np.ascontiguousarray(a, np.int32) for a in prog[1:]]
    _lib.check(_lib.lib().tsc_set_greedy_program(sim._h, C.c_int32(prog[0]), ip(arrs[0]), ip(arrs[1]), ip(arrs[2])))
    act = torch.zeros(R, net.n_nodes, dtype=torch.int32, device="cuda")
    obs = sim.observe()
    checked = 0
    for t in range(55):                # inside the shortest demand horizon (300 s)
        _lib.check(_lib.lib().tsc_greedy_actions(sim._h, _p(obs), _p(act), sim._stream()))
        if t in (0, 5, 25, 54):
            o = obs.cpu().numpy()
            np.testing.assert_array_equal(act.cpu().numpy(), _forward(ctrl, net, o))
            checked += int((o != 0).any())
        obs = sim.step(act)[0]
    assert checked >= 3                # the comparison saw loaded networks


def _train(scenario, agent, policy="lstm", updates=2, fw=128):
    """weights after a few device-resident training updates, as a one-replica reference wrapper"""
    from deeprl_signal_control_b200.agents.models import IA2C, MA2C
    from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    if scenario == "large_grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid
        net, par = build_large_grid(agent=agent), EnvParams(agent=agent)
    else:
        from deeprl_signal_control_b200.net.real_net import real_net_tables
        from tests.test_real_net_cpu import real_params
        net, par = real_net_tables(agent), real_params(agent)
    cp = configparser.ConfigParser(); cp.read_string(MODEL_INI)
    cp["MODEL_CONFIG"]["num_fw"] = str(fw)
    mk = lambda R: (MA2C(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, 0, cp["MODEL_CONFIG"], seed=1, n_replicas=R,
                         obs_off=net.node_obs_off) if agent == "ma2c" else
                    IA2C(net.n_s_ls, net.n_a_ls, net.n_w_ls, 0, cp["MODEL_CONFIG"], seed=1, n_replicas=R,
                         obs_off=net.node_obs_off, policy=policy))
    big, one = mk(32), mk(1)
    sim = BatchedSim(net, par, 32)
    tr = BatchedTrainer(sim, big.batched, agent, lr=5e-4, beta=0.01)
    p0 = big.batched.P.clone()
    tr.run(20 * updates)
    torch.cuda.synchronize()
    assert tr.n_updates == updates and not torch.equal(p0, big.batched.P)
    one.batched.P.copy_(big.batched.P)
    one.batched.pack_weights()
    return one, big, sim, tr


def _env(scenario, agent, seeds, episode_sec, out, n_replicas, record=True):
    cp = configparser.ConfigParser()
    ini = GRID_INI if scenario == "large_grid" else REAL_INI
    cp.read_string(ini % (agent, episode_sec, ",".join(str(s) for s in seeds)))
    if scenario == "large_grid":
        from deeprl_signal_control_b200.envs.large_grid_env import LargeGridEnv as Env
    else:
        from deeprl_signal_control_b200.envs.real_net_env import RealNetEnv as Env
    return Env(cp["ENV_CONFIG"], output_path=out, is_record=record, n_replicas=n_replicas)


def _reference_run(env, model, ctrl):
    """reference utils.py:Evaluator.run / Tester.perform with policy_type='deterministic' on the one-replica env"""
    env.train_mode = False
    env.cur_episode = 0
    env.init_data(True, False, env.output_path)
    means, stds = [], []
    for k in range(env.test_num):
        ob = env.reset(test_ind=k)
        done = True
        if model is not None:
            model.reset()
        rewards = []
        while True:
            if ctrl is not None:
                action = ctrl.forward(ob)
            else:
                policy = model.forward(ob, done, 'p')
                if env.agent == 'ma2c':
                    env.update_fingerprint(policy)
                action = [np.argmax(np.array(pi)) for pi in policy]
            next_ob, reward, done, global_reward = env.step(action)
            rewards.append(global_reward)
            if done:
                break
            ob = next_ob
        means.append(np.mean(np.array(rewards))); stds.append(np.std(np.array(rewards)))
        env.collect_tripinfo()
    env.output_data()
    return np.array(means), np.array(stds)


def _read(path):
    import pandas as pd
    return pd.read_csv(path, index_col=0)


# (scenario, agent, policy, num_fw) -> forward family: Monaco has no wait block, so IA2C there has dx = num_fw: the
# reference's num_fw = 128 and 160 are fused v2 widths.  The grid IA2C with num_fw = 64 (dx = 96, outside the v2 widths)
# runs the v1 forward.
CASES = {("large_grid", "ma2c", "lstm", 128): "v2", ("large_grid", "ia2c", "fc", 128): "fc",
         ("large_grid", "ia2c", "lstm", 64): "v1",
         ("real_net", "ma2c", "lstm", 128): "v2", ("real_net", "ia2c", "lstm", 128): "v2",
         ("real_net", "ia2c", "lstm", 160): "v2", ("large_grid", "greedy", None, 0): None, ("real_net", "greedy", None, 0): None}


@pytest.mark.parametrize("scenario,agent,policy,fw", list(CASES))
def test_evaluator_matches_reference_protocol(scenario, agent, policy, fw, tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    seeds, sec = [10000, 20000, 30000, 40000, 50000], 600
    d1, d2 = str(tmp_path / "one") + os.sep, str(tmp_path / "batched") + os.sep
    os.makedirs(d1); os.makedirs(d2)
    env1 = _env(scenario, agent, seeds, sec, d1, 1)
    envb = _env(scenario, agent, seeds, sec, d2, len(seeds))
    if agent == "greedy":
        from deeprl_signal_control_b200.envs.large_grid_env import LargeGridController
        from deeprl_signal_control_b200.envs.real_net_env import RealNetController
        mk = (lambda e: LargeGridController(e.node_names)) if scenario == "large_grid" else \
            (lambda e: RealNetController(e.node_names, e.nodes))
        model, ctrl1, ctrlb = None, mk(env1), mk(envb)
    else:
        model = _train(scenario, agent, policy, fw=fw)[0]
        family = "fc" if policy == "fc" else ("v2" if model.batched.tc_v2 else "v1")
        assert family == CASES[(scenario, agent, policy, fw)]
        ctrl1 = None
        ctrlb = model
    mean1, std1 = _reference_run(env1, model, ctrl1)
    ev = Evaluator(envb, ctrlb, d2, policy_type="deterministic")
    assert getattr(ev, "family", None) == CASES[(scenario, agent, policy, fw)]
    meanb, stdb = ev.run()
    np.testing.assert_array_equal(meanb, mean1)
    np.testing.assert_array_equal(stdb, std1)
    base = "%s_%s_" % (env1.name, agent)
    for kind in ("control", "traffic"):
        assert open(d1 + base + kind + ".csv").read() == open(d2 + base + kind + ".csv").read(), kind
    # trips: the same rows; the order of arrivals within one second is thread order (test_record_gpu.py)
    if open(d1 + base + "trip.csv").read() != open(d2 + base + "trip.csv").read():
        key = ["episode", "arrival_sec", "depart_sec", "id"]
        t1 = _read(d1 + base + "trip.csv").sort_values(key).reset_index(drop=True)
        tb = _read(d2 + base + "trip.csv").sort_values(key).reset_index(drop=True)
        assert t1.equals(tb)


def test_evaluation_leaves_a_live_learner_unchanged(tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    _, big, sim, tr = _train("large_grid", "ma2c", updates=1)
    b = big.batched
    tr.run(7)                              # in the middle of a rollout
    torch.cuda.synchronize()
    assert 0 < b.t < b.T and b.store_acts
    names = ["P", "MS", "c_fw", "h_fw", "c_bw", "h_bw", "obs_hist", "act_hist", "st_x", "st_g", "st_c", "st_h", "Wp"]
    before = {k: getattr(b, k).clone() for k in names}
    t, nf = b.t, b.n_forward
    env = _env("large_grid", "ma2c", [7, 8, 9], 300, str(tmp_path) + os.sep, 3)
    mean, std = Evaluator(env, big, str(tmp_path) + os.sep, policy_type="default").run()
    torch.cuda.synchronize()
    assert np.isfinite(mean).all() and (std > 0).all()
    for k in names:
        assert torch.equal(getattr(b, k), before[k]), k
    assert b.t == t and b.n_forward == nf
    tr.run(b.T - b.t)                      # and the rollout completes into its update
    assert tr.n_updates == 2


def test_evaluate_script_reproduces_in_memory_summary(tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    one = _train("large_grid", "ma2c")[0]
    agent_dir = tmp_path / "ma2c"
    (agent_dir / "data").mkdir(parents=True); (agent_dir / "model").mkdir()
    seeds = [11, 12, 13, 14]
    ini = GRID_INI % ("ma2c", 600, ",".join(str(s) for s in seeds)) + MODEL_INI
    (agent_dir / "data" / "config_ma2c_large.ini").write_text(ini)
    one.save(str(agent_dir / "model"), 40)
    out = tmp_path / "eva"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", str(agent_dir),
                        "--evaluation-policy-type", "deterministic", "--output-dir", str(out)],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    got = json.load(open(out / "ma2c_summary.json"))
    env = _env("large_grid", "ma2c", seeds, 600, str(tmp_path) + os.sep, len(seeds))
    ev = Evaluator(env, one, str(tmp_path) + os.sep, policy_type="deterministic")
    mean, std = ev.run()
    want = ev.summary(mean, std, *ev.recorded[1:])
    assert got == json.loads(json.dumps(want))
    for k in ("control", "traffic", "trip"):
        assert (out / ("large_grid_ma2c_%s.csv" % k)).exists()
    assert got["avg_speed_mps"] > 0 and len(got["trips_per_episode"]) == len(seeds)
