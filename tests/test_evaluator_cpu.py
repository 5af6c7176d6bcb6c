"""CPU: the pieces of the batched evaluator (agents/evaluator.py) that need no device — the greedy programs of the four
controllers against the controllers themselves (through a numpy restatement of tsc_greedy_kernel), the seed-to-replica
mapping, the CSV row assembly against the one-replica env's own row writers, and the new ABI symbols."""
import configparser
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tests", "fixtures"))

GRID_INI = """
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = greedy
coop_gamma = 0.9
data_path = ./large_grid/data/
episode_length_sec = 300
norm_wave = 5.0
norm_wait = 100.0
coef_wait = 0.2
peak_flow1 = 1100
peak_flow2 = 925
init_density = 0
objective = hybrid
scenario = large_grid
seed = 12
test_seeds = 10000,20000,30000
yellow_interval_sec = 2
"""


def greedy_np(prog, obs):
    """tsc_greedy_kernel restated: per node, float64 sums of the listed float32 observation entries in table order,
    first maximum over the candidates that exist."""
    max_cand, off, idx, act = prog
    R, N = obs.shape[0], (len(off) - 1) // max_cand
    out = np.zeros((R, N), np.int32)
    for i in range(N):
        best = np.full(R, -np.inf)
        for c in range(max_cand):
            k = i * max_cand + c
            if act[k] < 0:
                continue
            s = np.zeros(R, np.float64)
            for e in idx[off[k]:off[k + 1]]:
                s = s + obs[:, e].astype(np.float64)
            take = (s > best) | (best == -np.inf)
            out[take, i] = act[k]
            best = np.where(take, s, best)
    return out


def _controllers():
    """(controller, node_obs_off, n_obs, recorded observations or None) of each scenario"""
    from deeprl_signal_control_b200.envs.env import Node
    from deeprl_signal_control_b200.envs.large_grid_env import LargeGridController
    from deeprl_signal_control_b200.envs.real_net_env import RealNetController
    from deeprl_signal_control_b200.envs.small_grid_env import SmallGridController
    from deeprl_signal_control_b200.envs.sumo_env import SumoNetController
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    from deeprl_signal_control_b200.net.small_grid import build_small_grid
    out = {}
    net = build_large_grid(agent="greedy")
    out["grid"] = (LargeGridController(net.node_names), net, np.load(os.path.join(GOLD, "env_greedy_test.npz"))["obs"])
    net = real_net_tables("greedy")
    nodes = {}
    for name in net.node_names:
        nd = Node(name)
        nd.lanes_in, nd.ilds_in = net.lanes_in[name], net.ilds_in[name]
        nodes[name] = nd
    out["monaco"] = (RealNetController(net.node_names, nodes), net, np.load(os.path.join(GOLD, "real_greedy_test.npz"))["obs"])
    z = np.load(os.path.join(GOLD, "small_greedy_test.npz"))
    meta = json.loads(str(z["meta"]))
    net = build_small_grid(int(meta["cfg"]["num_extra_car_per_hour"]), agent="greedy", coop_gamma=float(meta["cfg"]["coop_gamma"]))
    out["small"] = (SmallGridController(net.node_names), net, z["obs"])
    return out


def _mini_sumo(tmp_path):
    import make_mini_sumo
    from deeprl_signal_control_b200.envs.sumo_env import SumoNetController, SumoNetEnv
    net_file, rou_file = make_mini_sumo.write(str(tmp_path))
    cp = configparser.ConfigParser()
    cp.read_string(GRID_INI.replace("scenario = large_grid", "scenario = mini") + "net_file = %s\nroute_file = %s\n"
                   % (net_file, rou_file))
    env = SumoNetEnv(cp["ENV_CONFIG"])
    ctl = SumoNetController(env.node_names, env.nodes, {n: env.phase_map.phases[n].phases for n in env.node_names})
    return ctl, env._tables


def _forward(ctrl, net, obs):
    """the controller's own forward on each row (float64 copies of the float32 observation, as env._split_obs)"""
    off = net.node_obs_off
    return np.array([[int(a) for a in ctrl.forward([row[off[i]:off[i + 1]].astype(np.float64) for i in range(net.n_nodes)])]
                     for row in obs], np.int32)


def _random_obs(rng, n, n_obs):
    """few distinct values, so that exact ties are common, plus values whose float64 sums tie or not depending on the
    summation precision"""
    vals = np.array([0.0, 0.2, 0.4, 0.6, 1.0, 2.0, 0.1, 0.3, 1e-8, 0.2 + 1e-8, 16777216.0, 1.0 + 2 ** -23], np.float32)
    obs = rng.choice(vals, size=(n, n_obs)).astype(np.float32)
    cont = rng.random((n // 2, n_obs), dtype=np.float32) * 2
    return np.concatenate([obs, cont])


@pytest.mark.parametrize("scenario", ["grid", "monaco", "small"])
def test_greedy_program_equals_controller_on_recorded_observations(scenario):
    ctrl, net, rec = _controllers()[scenario]
    prog = ctrl.greedy_program(net.node_obs_off)
    assert len(prog[1]) == net.n_nodes * prog[0] + 1 and len(prog[3]) == net.n_nodes * prog[0]
    obs = rec.astype(np.float32)
    assert obs.shape[1] == net.n_obs
    np.testing.assert_array_equal(greedy_np(prog, obs), _forward(ctrl, net, obs))


@pytest.mark.parametrize("scenario", ["grid", "monaco", "small", "mini_sumo"])
def test_greedy_program_equals_controller_with_ties(scenario, tmp_path):
    if scenario == "mini_sumo":
        ctrl, net = _mini_sumo(tmp_path)
    else:
        ctrl, net, _ = _controllers()[scenario]
    prog = ctrl.greedy_program(net.node_obs_off)
    rng = np.random.default_rng(7)
    obs = _random_obs(rng, 2000 if scenario != "monaco" else 600, net.n_obs)
    got, want = greedy_np(prog, obs), _forward(ctrl, net, obs)
    np.testing.assert_array_equal(got, want)
    # the planted values produced ties that the first-maximum rule had to break
    assert (want == 0).mean() > 0.1


def test_mini_sumo_program_from_recorded_oracle_observations(tmp_path):
    from deeprl_signal_control_b200.net.tables import EnvParams
    from oracle.sim_ref import RefSim
    ctrl, net = _mini_sumo(tmp_path)
    par = EnvParams(agent="greedy", episode_length_sec=300)
    sim = RefSim(net, par, 2)
    sim.reset(np.array([3, 4], np.uint64)); sim.set_train_mode(False)
    prog = ctrl.greedy_program(net.node_obs_off)
    obs, rows = sim.observe(), []
    for _ in range(60):
        act = greedy_np(prog, obs)
        np.testing.assert_array_equal(act, _forward(ctrl, net, obs))
        rows.append(obs.copy())
        obs = sim.step(act, None)[0]
    assert np.concatenate(rows).max() > 0


def _grid_env(tmp_path, R=1, record=True):
    from deeprl_signal_control_b200.envs.large_grid_env import LargeGridEnv
    cp = configparser.ConfigParser()
    cp.read_string(GRID_INI)
    return LargeGridEnv(cp["ENV_CONFIG"], output_path=str(tmp_path) + os.sep, is_record=record, n_replicas=R)


def test_replica_k_plays_test_seed_k(tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import replica_seeds
    one, many = _grid_env(tmp_path), _grid_env(tmp_path, R=3)
    one.train_mode = False
    seeds = replica_seeds(many)
    assert seeds.dtype == np.uint64 and len(seeds) == many.test_num == 3
    for k in range(3):     # env.reset(test_ind=k) of the one-replica env: seed test_seeds[k], no replica offset
        assert one._episode_seeds(one.test_seeds[k])[0] == seeds[k]
    # and not the training mapping seed + r of a multi-replica env.reset
    assert not np.array_equal(many._episode_seeds(many.test_seeds[0]), seeds)


def test_csv_rows_match_the_one_replica_env(tmp_path):
    """Synthetic traces of R episodes: the evaluator's frames equal, as CSV text, what the one-replica env's row writers
    produce when the episodes run one after another."""
    import pandas as pd
    from deeprl_signal_control_b200.agents.evaluator import control_frame, traffic_frame, trip_frame
    env = _grid_env(tmp_path)
    R, T, ci, N = 3, 7, env.control_interval_sec, 25
    rng = np.random.default_rng(3)
    acts = rng.integers(0, 5, (R, T, N)).astype(np.int32)
    grew = (rng.standard_normal((R, T)) * 50).astype(np.float32)
    dep = np.cumsum(rng.integers(0, 4, (R, T * ci)), axis=1)
    arr = np.minimum(np.cumsum(rng.integers(0, 3, (R, T * ci)), axis=1), dep)
    stats = np.zeros((R, T * ci, 8), np.float32)
    stats[..., 0] = dep - arr; stats[..., 1] = dep; stats[..., 2] = arr
    stats[..., 3:7] = rng.random((R, T * ci, 4), dtype=np.float32) * 10
    trips = [np.stack([rng.integers(0, 100, n), rng.integers(100, 300, n), rng.integers(0, 16, n), rng.integers(0, 60, n),
                       rng.integers(0, 5, n)], 1) for n in (5, 0, 9)]

    class _Sim:
        k = 0

        def trips(self, replica):
            return trips[self.k]
    env._sim = _Sim()
    env.cur_episode = 0
    for k in range(R):                        # the one-replica env's bookkeeping of reset / step / collect_tripinfo
        env.cur_episode += 1
        env.cur_sec = 0
        env._n_dep_prev = env._n_arr_prev = 0
        for t in range(T):
            env._record_traffic(stats[k, t * ci:(t + 1) * ci], env.cur_sec)
            env.cur_sec += ci
            env._record_control(acts[k, t], grew[k, t])
        env._sim.k = k
        env.collect_tripinfo()
    want = [pd.DataFrame(d).to_csv() for d in (env.control_data, env.traffic_data, env.trip_data)]
    got = [f.to_csv() for f in (control_frame(acts, grew, ci), traffic_frame(stats), trip_frame(trips))]
    for g, w in zip(got, want):
        assert g == w


def test_evaluator_abi_is_exported():
    from deeprl_signal_control_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build_native()
    lib = C.CDLL(_lib.LIB_PATH)
    for name in ("tsc_set_greedy_program", "tsc_greedy_actions", "tscl_policy_step_pi", "tscl_argmax_actions"):
        assert hasattr(lib, name) and name in _lib.SYMBOLS
