"""Cost of the max-pressure controller (tsc_pressure_actions) next to the greedy one (tsc_greedy_actions), and the mean
episode reward of both controllers at three demand levels.

  python scripts/time_pressure.py [--iters 500] [--pairs 5]

* kernels: per-launch time of tsc_pressure_actions and tsc_greedy_actions on the grid (R = 4096) and Monaco
  (R = 2048), each replica loaded by 60 control steps of random actions; CUDA events around `--iters` launches after a
  warm-up, the two arms alternating `--pairs` times (median, min and max over the pairs).
* evaluate.py: wall time of one `scripts/evaluate.py` process (start-up included) for a greedy and a maxpressure agent
  directory on the grid and Monaco, 3600 s episodes, the reference's 10 evaluation seeds (10000 .. 100000).
* rewards: `scripts/evaluate_agents.py --agents greedy,maxpressure` on the same seeds at the configured demand and at
  the x0.6 / x1.4 levels (grid: peak_flow1 / peak_flow2, Monaco: flow_rate): mean and std over episodes of the
  per-episode mean step reward, and the mean queue.
Prints one JSON line per measurement, each with the card's name and power limit, and writes them to
$OUT/time_pressure.json (OUT defaults to results/).
"""
import argparse
import configparser
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.time_population import card  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS = ",".join(str(s) for s in range(10000, 100001, 10000))     # main.py:40-41
LEVELS = {"large_grid": [{"peak_flow1": "1100", "peak_flow2": "925"}, {"peak_flow1": "660", "peak_flow2": "555"},
                         {"peak_flow1": "1540", "peak_flow2": "1295"}],
          "real_net": [{"flow_rate": "325"}, {"flow_rate": "195"}, {"flow_rate": "455"}]}
FACTORS = (1.0, 0.6, 1.4)


def time_kernels(iters, pairs):
    import numpy as np
    import torch
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.envs.env import Node
    from deeprl_signal_control_b200.envs.large_grid_env import LargeGridController
    from deeprl_signal_control_b200.envs.real_net_env import RealNetController
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    from tests.test_real_net_cpu import real_params
    out = []
    for scen, R in (("large_grid", 4096), ("real_net", 2048)):
        if scen == "large_grid":
            net, par = build_large_grid(agent="greedy"), EnvParams(agent="greedy")
            ctrl = LargeGridController(net.node_names)
        else:
            net, par = real_net_tables("greedy"), real_params("greedy")
            nodes = {}
            for name in net.node_names:
                nd = Node(name)
                nd.lanes_in, nd.ilds_in = net.lanes_in[name], net.ilds_in[name]
                nodes[name] = nd
            ctrl = RealNetController(net.node_names, nodes)
        sim = BatchedSim(net, par, R)
        sim.reset(np.arange(R, dtype=np.uint64) + np.uint64(12))
        sim.set_train_mode(False)
        g = torch.Generator(device="cuda").manual_seed(3)
        for _ in range(60):
            sim.step(torch.stack([torch.randint(0, int(na), (R,), device="cuda", generator=g, dtype=torch.int32)
                                  for na in net.node_n_phases], 1).contiguous())
        obs = sim.observe()
        prog = ctrl.greedy_program(net.node_obs_off)
        arrs = [np.ascontiguousarray(a, np.int32) for a in prog[1:]]
        _lib.check(_lib.lib().tsc_set_greedy_program(sim._h, int(prog[0]), *(a.ctypes.data for a in arrs)))
        act = torch.zeros(R, net.n_nodes, dtype=torch.int32, device="cuda")
        st = sim._stream()
        arms = {"tsc_greedy_actions": lambda: _lib.lib().tsc_greedy_actions(sim._h, obs.data_ptr(), act.data_ptr(), st),
                "tsc_pressure_actions": lambda: _lib.lib().tsc_pressure_actions(sim._h, act.data_ptr(), st)}
        times = {k: [] for k in arms}
        for p in range(pairs + 1):                              # pair 0 warms both arms up
            for k, fn in arms.items():
                for _ in range(20):
                    _lib.check(fn())
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                if p:
                    times[k].append(e0.elapsed_time(e1) * 1000.0 / iters)
        live = sim.mean_live()
        for k, ts in times.items():
            out.append(dict(what=k, scenario=scen, replicas=R, nodes=net.n_nodes, iters=iters, pairs=pairs,
                            us_per_launch_median=round(statistics.median(ts), 3), us_min=round(min(ts), 3),
                            us_max=round(max(ts), 3), mean_live_vehicles=round(live, 1)))
    return out


def _cfg(path, scenario, agent, level=None):
    from tests.test_evaluator_gpu import GRID_INI, REAL_INI
    c = configparser.ConfigParser()
    c.read_string((GRID_INI if scenario == "large_grid" else REAL_INI) % (agent, 3600, SEEDS))
    for k, v in (level or {}).items():
        c["ENV_CONFIG"][k] = v
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        c.write(f)


def _proc(*args):
    t0 = time.time()
    r = subprocess.run([sys.executable] + list(args), capture_output=True, text=True, cwd=ROOT)
    if r.returncode:
        raise SystemExit(r.stdout + r.stderr)
    return time.time() - t0, r.stdout


def time_eval_and_rewards():
    from deeprl_signal_control_b200.envs import demand_label
    rows = []
    for scen in ("large_grid", "real_net"):
        base = tempfile.mkdtemp(prefix="time_pressure_")
        try:
            for agent in ("greedy", "maxpressure"):
                _cfg(os.path.join(base, agent, "data", "config.ini"), scen, agent)
                sec, _ = _proc(os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", os.path.join(base, agent))
                rows.append(dict(what="evaluate.py", scenario=scen, agent=agent, seeds=10, episode_sec=3600,
                                 wall_sec=round(sec, 2)))
            dem = sum((["--demand", ",".join("%s=%s" % kv for kv in lv.items())] for lv in LEVELS[scen]), [])
            _, text = _proc(os.path.join(ROOT, "scripts", "evaluate_agents.py"), "--base-dir", base, "--agents",
                            "greedy,maxpressure", "--evaluation-seeds", SEEDS, *dem)
            factor = {demand_label(lv): f for lv, f in zip(LEVELS[scen], FACTORS)}
            for line in text.splitlines():
                if line.startswith("{"):
                    r = json.loads(line)
                    rows.append(dict(what="reward", scenario=scen, agent=r["entry"], demand=r["demand"],
                                     demand_factor=factor[r["demand"]], seeds=10, episode_sec=3600,
                                     mean_reward=round(r["mean_reward"], 2), std_reward=round(r["std_reward"], 2),
                                     avg_queue=round(r["avg_queue"], 3), mean_trips=r["mean_trips"]))
        finally:
            shutil.rmtree(base, ignore_errors=True)
    return rows


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=500)
    p.add_argument("--pairs", type=int, default=5)
    a = p.parse_args()
    info = card()
    rows = time_kernels(a.iters, a.pairs) + time_eval_and_rewards()
    out_dir = os.environ.get("OUT", "results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_pressure.json"), "w") as f:
        for r in rows:
            r["card"] = info
            print(json.dumps(r), flush=True)
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
