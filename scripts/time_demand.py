"""Cost of per-replica traffic demand (tsc_set_replica_demand) in the simulator, and wall time of evaluating agents at
several demand levels in one process against one `scripts/evaluate.py` run per (agent, level).

  python scripts/time_demand.py [--replicas 4096] [--iters 200] [--pairs 5] [--eval-seeds 10]

* tsc_step: grid MA2C (5x5 grid, 3600 s horizon) on `--replicas` replicas, CUDA events around `--iters` control steps
  of random actions after a warm-up, with no demand set, with one level (every replica at the configured level) and with
  8 levels in blocks of R / 8 replicas (peak flows x0.6 .. x2.0).  The three arms alternate `--pairs` times; the median
  per-step time of each arm is reported with its spread.
* evaluation: greedy and a briefly trained ma2c grid agent (600 s episodes) at 3 demand levels on `--eval-seeds` seeds, one
  `scripts/evaluate_agents.py --demand ... x3` process against the 6 `scripts/evaluate.py` processes on copies of the
  agent directories whose configs carry each level (wall time of the processes, start-up included).
Prints one JSON line per measurement, each with the card's name and power limit, and writes them to
$OUT/time_demand.json (OUT defaults to results/).
"""
import argparse
import configparser
import glob
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
LEVELS = (0.6, 0.8, 1.0, 1.2, 1.4, 1.6, 1.8, 2.0)          # peak-flow factors of the 8-level arm
EVAL_LEVELS = ({"peak_flow1": "1100", "peak_flow2": "925"}, {"peak_flow1": "1400", "peak_flow2": "1180"},
               {"peak_flow1": "1700", "peak_flow2": "1430"})


def time_step(R, iters, pairs):
    import numpy as np
    import torch
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    net, par = build_large_grid(agent="ma2c"), EnvParams(agent="ma2c")
    levels = [build_large_grid(int(1100 * f), int(925 * f), agent="ma2c") for f in LEVELS]
    sims = {"none": BatchedSim(net, par, R), "one_level": BatchedSim(net, par, R), "eight_levels": BatchedSim(net, par, R)}
    sims["one_level"].set_replica_demand([net], np.zeros(R, np.int64))
    sims["eight_levels"].set_replica_demand(levels, np.repeat(np.arange(8), R // 8))
    g = torch.Generator(device="cuda").manual_seed(3)
    acts = [torch.randint(0, 5, (R, net.n_nodes), device="cuda", generator=g, dtype=torch.int32) for _ in range(iters)]
    fp = torch.rand(R, net.n_nodes, net.max_na, device="cuda", generator=g)
    seeds = np.arange(R, dtype=np.uint64) + np.uint64(12)
    times = {k: [] for k in sims}
    for p in range(pairs + 1):                              # pair 0 warms every arm up
        for k, s in sims.items():
            s.reset(seeds)
            for a in acts[:20]:                             # fill the network before timing
                s.step(a, fp)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for a in acts:
                s.step(a, fp)
            e1.record()
            torch.cuda.synchronize()
            if p:
                times[k].append(e0.elapsed_time(e1) / iters)
    live = {k: s.mean_live() for k, s in sims.items()}
    out = []
    for k, ts in times.items():
        out.append(dict(what="tsc_step", arm=k, replicas=R, iters=iters, pairs=pairs,
                        ms_per_step_median=round(statistics.median(ts), 4), ms_min=round(min(ts), 4),
                        ms_max=round(max(ts), 4), mean_live_vehicles=round(live[k], 1)))
    return out


def _cfg(path, agent, level=None):
    from tests.test_train_driver_gpu import _ini
    c = configparser.ConfigParser()
    c.read_string(_ini("ma2c", 120, 240))
    c["ENV_CONFIG"]["agent"] = agent
    for k, v in (level or {}).items():
        c["ENV_CONFIG"][k] = v
    with open(path, "w") as f:
        c.write(f)


def _proc(*args):
    t0 = time.time()
    r = subprocess.run([sys.executable] + list(args), capture_output=True, text=True, cwd=ROOT)
    if r.returncode:
        raise SystemExit(r.stdout + r.stderr)
    return time.time() - t0


def time_eval(n_seeds):
    from deeprl_signal_control_b200.agents.train import train
    base = tempfile.mkdtemp(prefix="time_demand_")
    try:
        os.makedirs(os.path.join(base, "greedy", "data"))
        _cfg(os.path.join(base, "greedy", "data", "config.ini"), "greedy")
        _cfg(os.path.join(base, "ma2c.ini"), "ma2c")
        train(os.path.join(base, "ma2c.ini"), os.path.join(base, "ma2c"), "no_test", n_replicas=64)
        seeds = ",".join(str(10000 * (i + 1)) for i in range(n_seeds))
        dem = sum((["--demand", ",".join("%s=%s" % kv for kv in lv.items())] for lv in EVAL_LEVELS), [])
        grouped = _proc(os.path.join(ROOT, "scripts", "evaluate_agents.py"), "--base-dir", base, "--agents",
                        "greedy,ma2c", "--evaluation-seeds", seeds, *dem)
        separate = 0.0
        for agent in ("greedy", "ma2c"):
            for j, lv in enumerate(EVAL_LEVELS):
                d = os.path.join(base, "sep%d" % j, agent)
                shutil.copytree(os.path.join(base, agent), d, ignore=shutil.ignore_patterns("eva_data"))
                for ini in glob.glob(os.path.join(d, "data", "*.ini")):
                    _cfg(ini, agent, lv)
                separate += _proc(os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", d, "--evaluation-seeds",
                                  seeds)
        return [dict(what="evaluation", agents=2, levels=len(EVAL_LEVELS), seeds=n_seeds,
                     grouped_wall_sec=round(grouped, 2), separate_wall_sec=round(separate, 2),
                     speedup=round(separate / grouped, 2))]
    finally:
        shutil.rmtree(base, ignore_errors=True)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--replicas", type=int, default=4096)
    p.add_argument("--iters", type=int, default=200)
    p.add_argument("--pairs", type=int, default=5)
    p.add_argument("--eval-seeds", type=int, default=10)
    a = p.parse_args()
    info = card()
    rows = time_step(a.replicas, a.iters, a.pairs) + time_eval(a.eval_seeds)
    out_dir = os.environ.get("OUT", "results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_demand.json"), "w") as f:
        for r in rows:
            r["card"] = info
            print(json.dumps(r))
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
