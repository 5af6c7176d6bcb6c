"""Tune a scenario's fixed-time signal plan on the device: a cross-entropy search over its green durations and offsets
(deeprl_signal_control_b200/agents/tune_fixedtime.py), each generation's candidate plans one episode of one simulator.

  python scripts/tune_fixedtime.py --base-dir runs/tuned --config-dir config_greedy_large.ini
                                   --seeds 1001,1002,1003,1004,1005,1006,1007,1008
                                   [--candidates 512] [--generations 30] [--elite-frac 0.1] [--min-green 5]
                                   [--max-green 60] [--rng-seed 0] [--device 0]

Writes the agent directory B/fixedtime/ (data/<config name> with tll_file set to data/tuned.tll.xml, the log
data/tune_log.csv and data/tune.json), which the evaluation scripts run as any `fixedtime` directory:

  python scripts/evaluate_agents.py --base-dir runs --agents greedy,maxpressure,fixedtime,actuated,tuned/fixedtime

The tuning seeds may not be the config's test_seeds or the evaluation scripts' default seeds (10000 .. 100000).
"""
import argparse
import json
import logging
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--base-dir", required=True, help="the tuned directory is written to BASE_DIR/fixedtime/")
    p.add_argument("--config-dir", required=True, help="the scenario's config (.ini), as in main.py")
    p.add_argument("--seeds", required=True, help="comma-separated tuning seeds")
    p.add_argument("--candidates", type=int, default=512)
    p.add_argument("--generations", type=int, default=30)
    p.add_argument("--elite-frac", type=float, default=0.1)
    p.add_argument("--min-green", type=int, default=5)
    p.add_argument("--max-green", type=int, default=60)
    p.add_argument("--rng-seed", type=int, default=0)
    p.add_argument("--device", type=int, default=0)
    a = p.parse_args(argv)
    try:
        a.seeds = [int(s) for s in a.seeds.split(",") if s.strip()]
    except ValueError:
        p.error("--seeds takes comma-separated integers (got %r)" % a.seeds)
    return a


def main(argv=None):
    a = parse_args(argv)
    logging.basicConfig(level=logging.INFO, format="%(message)s")
    from deeprl_signal_control_b200.agents.tune_fixedtime import tune_fixedtime
    res = tune_fixedtime(a.config_dir, a.base_dir, a.seeds, candidates=a.candidates, generations=a.generations,
                         elite_frac=a.elite_frac, min_green=a.min_green, max_green=a.max_green, rng_seed=a.rng_seed,
                         device=a.device)
    print(json.dumps({"dir": res["dir"], "shipped_score": res["shipped_score"], "best_score": res["best_score"]}))
    return res


if __name__ == "__main__":
    main()
