"""Cost of vehicle-actuated control (the ACTUATED instantiation of tsc_step_kernel) next to the fixed-time and the
greedy-driven control step, and the mean episode reward of greedy, max-pressure, fixed-time and actuated control at
three demand levels.

  python scripts/time_actuated.py [--iters 500] [--pairs 5]

* step: time of one control step in actuated mode (tsc_step, action = NULL) against fixed mode (tsc_step, action =
  NULL) and tsc_greedy_actions + tsc_step, on the grid (R = 4096) and Monaco (R = 2048).  Before every timed window
  each handle is reset and loaded by 60 control steps; CUDA events around `--iters` steps after 20 warm-up steps, the
  three arms alternating `--pairs` times after a warm-up round (median, min and max over the rounds).  The arms carry
  different traffic, so the difference is the controllers' as much as the kernels'.
* evaluate.py: wall time of one `scripts/evaluate.py` process (start-up included) for each controller's agent
  directory on the grid and Monaco, 3600 s episodes, the reference's 10 evaluation seeds.
* rewards: `scripts/evaluate_agents.py --agents greedy,maxpressure,fixedtime,actuated` on the same seeds at the
  configured demand and at the x0.6 / x1.4 levels: mean and std over episodes of the per-episode mean step reward, the
  mean queue and the mean trips per episode.
Prints one JSON line per measurement, each with the card's name and power limit, and writes them to
$OUT/time_actuated.json (OUT defaults to results/).
"""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.time_population import card  # noqa: E402
from scripts.time_pressure import FACTORS, LEVELS, ROOT, SEEDS, _cfg, _proc  # noqa: E402

AGENTS = ("greedy", "maxpressure", "fixedtime", "actuated")


def time_steps(iters, pairs):
    import numpy as np
    import torch
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.envs.actuated import actuated_tables
    from deeprl_signal_control_b200.envs.env import Node
    from deeprl_signal_control_b200.envs.fixedtime import program_tables
    from deeprl_signal_control_b200.envs.large_grid_env import LargeGridController
    from deeprl_signal_control_b200.envs.real_net_env import RealNetController
    from deeprl_signal_control_b200.net import large_grid
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    from tests.test_real_net_cpu import real_params
    lib = _lib.lib()
    out = []
    for scen, R in (("large_grid", 4096), ("real_net", 2048)):
        if scen == "large_grid":
            net, par = large_grid.build_large_grid(agent="greedy"), EnvParams(agent="greedy")
            ctrl, programs = LargeGridController(net.node_names), large_grid.tls_programs()
        else:
            net, par = real_net_tables("greedy"), real_params("greedy")
            nodes = {}
            for name in net.node_names:
                nd = Node(name)
                nd.lanes_in, nd.ilds_in = net.lanes_in[name], net.ilds_in[name]
                nodes[name] = nd
            ctrl = RealNetController(net.node_names, nodes)
            with open(os.path.join(ROOT, "deeprl_signal_control_b200", "net", "data", "real_net_programs.json")) as f:
                programs = json.load(f)
        actuated, fixed, greedy = BatchedSim(net, par, R), BatchedSim(net, par, R), BatchedSim(net, par, R)
        fixed.set_signal_program(program_tables(net.node_names, [len(net.phases[n][0]) for n in net.node_names],
                                                programs))
        actuated.set_actuated_program(actuated_tables(net, programs))
        gp = ctrl.greedy_program(net.node_obs_off)
        arrs = [np.ascontiguousarray(a, np.int32) for a in gp[1:]]
        _lib.check(lib.tsc_set_greedy_program(greedy._h, int(gp[0]), *(a.ctypes.data for a in arrs)))
        act = torch.zeros(R, net.n_nodes, dtype=torch.int32, device="cuda")
        st = fixed._stream()

        def program_step(sim):
            return lambda: lib.tsc_step(sim._h, None, None, sim.obs.data_ptr(), sim.reward.data_ptr(),
                                        sim.greward.data_ptr(), sim.done.data_ptr(), st)

        def greedy_step():
            rc = lib.tsc_greedy_actions(greedy._h, greedy.obs.data_ptr(), act.data_ptr(), st)
            return rc or lib.tsc_step(greedy._h, act.data_ptr(), None, greedy.obs.data_ptr(), greedy.reward.data_ptr(),
                                      greedy.greward.data_ptr(), greedy.done.data_ptr(), st)

        arms = {"actuated step": (actuated, program_step(actuated)), "fixedtime step": (fixed, program_step(fixed)),
                "greedy actions + step": (greedy, greedy_step)}
        times, live = {k: [] for k in arms}, {k: [] for k in arms}
        for p in range(pairs + 1):                              # round 0 warms every arm up
            for k, (sim, fn) in arms.items():
                sim.reset(np.arange(R, dtype=np.uint64) + np.uint64(12 + p))
                sim.set_train_mode(False)
                sim.observe()
                for _ in range(80):                             # 60 loading steps, then 20 warm-up steps
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
                    live[k].append(sim.mean_live())
        for k, ts in times.items():
            out.append(dict(what=k, scenario=scen, replicas=R, nodes=net.n_nodes, iters=iters, pairs=pairs,
                            us_per_step_median=round(statistics.median(ts), 2), us_min=round(min(ts), 2),
                            us_max=round(max(ts), 2), mean_live_vehicles_end=round(statistics.mean(live[k]), 1)))
    return out


def time_eval_and_rewards():
    from deeprl_signal_control_b200.envs import demand_label
    rows = []
    for scen in ("large_grid", "real_net"):
        base = tempfile.mkdtemp(prefix="time_actuated_")
        try:
            for agent in AGENTS:
                _cfg(os.path.join(base, agent, "data", "config.ini"), scen, agent)
                sec, _ = _proc(os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", os.path.join(base, agent))
                rows.append(dict(what="evaluate.py", scenario=scen, agent=agent, seeds=10, episode_sec=3600,
                                 wall_sec=round(sec, 2)))
            dem = sum((["--demand", ",".join("%s=%s" % kv for kv in lv.items())] for lv in LEVELS[scen]), [])
            _, text = _proc(os.path.join(ROOT, "scripts", "evaluate_agents.py"), "--base-dir", base, "--agents",
                            ",".join(AGENTS), "--evaluation-seeds", SEEDS, *dem)
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
    rows = time_steps(a.iters, a.pairs) + time_eval_and_rewards()
    out_dir = os.environ.get("OUT", "results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_actuated.json"), "w") as f:
        for r in rows:
            r["card"] = info
            print(json.dumps(r), flush=True)
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
