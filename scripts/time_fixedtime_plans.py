"""Cost and benefit of per-replica fixed-time plans (tsc_set_replica_signal_programs) and of the plan search
(agents/tune_fixedtime.py).

  python scripts/time_fixedtime_plans.py [--iters 300] [--pairs 5] [--generations 30] [--candidates 512]

* step: one control step (tsc_step, action = NULL) with one shared program against K distinct plans (random green
  durations and offsets of the search space), grid R = 4096 with K = 512 and Monaco R = 2048 with K = 256; two more
  arms split the difference: the shared program set through tsc_set_replica_signal_programs (the plan-index load
  alone) and the first random plan shared by every replica (its traffic alone).  Every handle is reset and loaded by 60
  control steps before every window; CUDA events around `--iters` steps after 20 warm-up steps, the arms taking turns
  `--pairs` times after a warm-up round (median, min and max over the rounds).
* tune: `tune_fixedtime` at its defaults (512 candidates, 30 generations, 8 tuning seeds 1001..1008, 3600-s episodes)
  on the grid and Monaco at configured demand: wall time of the run and per generation, shipped and final score.
* rewards: `scripts/evaluate_agents.py --agents greedy,maxpressure,fixedtime,actuated,tuned/fixedtime` on the
  reference's 10 evaluation seeds at the configured demand and at the x0.6 / x1.4 levels, the tuned plan being the one
  tuned at x1; each tuned row also carries the plan's score on the tuning seeds.
Prints one JSON line per measurement, each with the card's name and power limit, and writes them to
$OUT/time_fixedtime_plans.json (OUT defaults to results/).
"""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.time_population import card  # noqa: E402
from scripts.time_pressure import FACTORS, LEVELS, ROOT, SEEDS, _cfg, _proc  # noqa: E402

AGENTS = ("greedy", "maxpressure", "fixedtime", "actuated", "tuned/fixedtime")
TUNE_SEEDS = list(range(1001, 1009))


def _net(scen):
    import json as js
    from deeprl_signal_control_b200.envs.fixedtime import program_tables
    from deeprl_signal_control_b200.net import large_grid
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    from deeprl_signal_control_b200.net.tables import EnvParams
    from tests.test_real_net_cpu import real_params
    if scen == "large_grid":
        net, par, programs = large_grid.build_large_grid(agent="fixedtime"), EnvParams(agent="fixedtime"), \
            large_grid.tls_programs()
    else:
        net, par = real_net_tables("fixedtime"), real_params("fixedtime")
        with open(os.path.join(ROOT, "deeprl_signal_control_b200", "net", "data", "real_net_programs.json")) as f:
            programs = js.load(f)
    return net, par, program_tables(net.node_names, [len(net.phases[n][0]) for n in net.node_names], programs)


def time_steps(iters, pairs):
    import numpy as np
    import torch
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.tune_fixedtime import offsets_of, search_space
    from deeprl_signal_control_b200.sim import BatchedSim
    lib = _lib.lib()
    out = []
    for scen, R, K in (("large_grid", 4096, 512), ("real_net", 2048, 256)):
        net, par, prog = _net(scen)
        space = search_space(prog)
        rng = np.random.default_rng(0)
        plans = []
        for _ in range(K):
            g = rng.integers(space.lo, space.hi + 1)
            plans.append(space.program(g, offsets_of(space, g, rng.random(space.n_nodes))))
        shared, per, index, one = (BatchedSim(net, par, R) for _ in range(4))
        shared.set_signal_program(prog)
        per.set_replica_signal_programs(plans, np.repeat(np.arange(K), R // K))
        index.set_replica_signal_programs([prog], np.zeros(R, np.int64))     # the per-replica path, one plan
        one.set_signal_program(plans[0])                                    # one of the random plans, shared
        st = shared._stream()

        def stepper(sim):
            return lambda: lib.tsc_step(sim._h, None, None, sim.obs.data_ptr(), sim.reward.data_ptr(),
                                        sim.greward.data_ptr(), sim.done.data_ptr(), st)
        arms = {"one shared program": (shared, stepper(shared)), "%d distinct plans" % K: (per, stepper(per)),
                "the shared program through the plan index": (index, stepper(index)),
                "one of the random plans, shared": (one, stepper(one))}
        times, live = {k: [] for k in arms}, {k: [] for k in arms}
        for p in range(pairs + 1):                              # pair 0 warms both arms up
            for k, (sim, fn) in arms.items():
                sim.reset(np.arange(R, dtype=np.uint64) + np.uint64(12 + p))
                sim.set_train_mode(False)
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
            out.append(dict(what="step: " + k, scenario=scen, replicas=R, nodes=net.n_nodes, iters=iters, pairs=pairs,
                            us_per_step_median=round(statistics.median(ts), 2), us_min=round(min(ts), 2),
                            us_max=round(max(ts), 2), mean_live_vehicles_end=round(statistics.mean(live[k]), 1)))
        del shared, per, index, one
    return out


def tune_and_rewards(candidates, generations):
    from deeprl_signal_control_b200.agents.tune_fixedtime import tune_fixedtime
    from deeprl_signal_control_b200.envs import demand_label
    rows = []
    for scen in ("large_grid", "real_net"):
        base = tempfile.mkdtemp(prefix="time_fixedtime_plans_")
        try:
            for agent in AGENTS[:4]:
                _cfg(os.path.join(base, agent, "data", "config.ini"), scen, agent)
            cfg = os.path.join(base, "fixedtime", "data", "config.ini")
            t0 = time.time()
            res = tune_fixedtime(cfg, os.path.join(base, "tuned"), TUNE_SEEDS, candidates=candidates,
                                 generations=generations)
            sec = time.time() - t0
            rows.append(dict(what="tune", scenario=scen, candidates=candidates, generations=generations,
                             tuning_seeds=len(TUNE_SEEDS), episode_sec=3600, wall_sec=round(sec, 1),
                             sec_per_generation=round(sec / max(generations, 1), 2),
                             shipped_score=round(res["shipped_score"], 2), final_score=round(res["best_score"], 2)))
            dem = sum((["--demand", ",".join("%s=%s" % kv for kv in lv.items())] for lv in LEVELS[scen]), [])
            _, text = _proc(os.path.join(ROOT, "scripts", "evaluate_agents.py"), "--base-dir", base, "--agents",
                            ",".join(AGENTS), "--evaluation-seeds", SEEDS, *dem)
            factor = {demand_label(lv): f for lv, f in zip(LEVELS[scen], FACTORS)}
            for line in text.splitlines():
                if line.startswith("{"):
                    r = json.loads(line)
                    row = dict(what="reward", scenario=scen, agent=r["entry"], demand=r["demand"],
                               demand_factor=factor[r["demand"]], seeds=10, episode_sec=3600,
                               mean_reward=round(r["mean_reward"], 2), std_reward=round(r["std_reward"], 2),
                               avg_queue=round(r["avg_queue"], 3), mean_trips=r["mean_trips"])
                    if r["entry"] == "tuned/fixedtime":
                        row["tuning_seed_score_x1"] = round(res["best_score"], 2)
                    rows.append(row)
        finally:
            shutil.rmtree(base, ignore_errors=True)
    return rows


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=300)
    p.add_argument("--pairs", type=int, default=5)
    p.add_argument("--candidates", type=int, default=512)
    p.add_argument("--generations", type=int, default=30)
    p.add_argument("--steps-only", action="store_true")
    a = p.parse_args()
    import logging
    logging.basicConfig(level=logging.INFO, format="%(message)s")
    info = card()
    out_dir = os.environ.get("OUT", "results")
    os.makedirs(out_dir, exist_ok=True)
    rows = time_steps(a.iters, a.pairs) + ([] if a.steps_only else tune_and_rewards(a.candidates, a.generations))
    with open(os.path.join(out_dir, "time_fixedtime_plans.json"), "w") as f:
        for r in rows:
            r["card"] = info
            print(json.dumps(r), flush=True)
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
