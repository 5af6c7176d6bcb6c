"""Test-mode evaluation of a trained agent on every evaluation seed at once: the reference's `main.py evaluate`
(main.py:35-43, 158-198) on the batched device evaluator (deeprl_signal_control_b200/agents/evaluator.py).

  python scripts/evaluate.py --agent-dir DIR [--evaluation-policy-type default|stochastic|deterministic]
                             [--evaluation-seeds 2000,2001,... | --n-seeds N --seed0 S] [--output-dir OUT]
                             [--policy lstm|fc]

DIR holds `data/*.ini` (the run's config, [ENV_CONFIG] + [MODEL_CONFIG]) and, unless the agent is a controller,
`model/checkpoint-<step>.npz` as written by IA2C.save / MA2C.save / IQL.save.  The agent is the directory's name, as in
the reference (main.py:179-190; agents/evaluator.py:entry_model and build_model): ia2c, ma2c, the controllers greedy, maxpressure (envs.maxpressure), fixedtime (the
net's fixed-time signal programs, envs.fixedtime) and actuated (vehicle-actuated control on the net's programs,
envs.actuated), iqld
(IQL with DeepQPolicy) or any other name, e.g. iqll (IQL with LRQPolicy).  The controllers ignore
--evaluation-policy-type and --policy.  Writes the reference's `<scenario>_<agent>_{control,traffic,trip}.csv` and
`<agent>_summary.json` (mean / std over episodes of the per-episode mean step reward, mean avg_queue / avg_speed_mps /
avg_wait_sec, completed trips per episode) into OUT (default: DIR/eva_data).
"""
import argparse
import configparser
import glob
import json
import logging
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deeprl_signal_control_b200.envs import make_env  # noqa: E402


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--agent-dir", required=True)
    p.add_argument("--evaluation-policy-type", default="default", choices=["default", "stochastic", "deterministic"])
    p.add_argument("--evaluation-seeds", default=None, help="comma-separated seeds (default: [ENV_CONFIG] test_seeds)")
    p.add_argument("--n-seeds", type=int, default=None, help="evaluate seeds seed0 .. seed0 + n - 1")
    p.add_argument("--seed0", type=int, default=2000)
    p.add_argument("--output-dir", default=None)
    p.add_argument("--policy", default="lstm", choices=["lstm", "fc"])
    return p.parse_args(argv)


def main(argv=None):
    a = parse_args(argv)
    logging.basicConfig(level=logging.INFO, format="%(message)s")
    agent_dir = a.agent_dir.rstrip("/")
    agent = os.path.basename(agent_dir)
    inis = sorted(glob.glob(os.path.join(agent_dir, "data", "*.ini")))
    if not inis:
        raise SystemExit("no config under %s/data/" % agent_dir)
    config = configparser.ConfigParser()
    config.read(inis[0])
    cfg = config["ENV_CONFIG"]
    if a.n_seeds is not None:
        seeds = [a.seed0 + i for i in range(a.n_seeds)]
    elif a.evaluation_seeds:
        seeds = [int(s) for s in a.evaluation_seeds.split(",")]
    else:
        seeds = [int(s) for s in cfg.get("test_seeds").split(",")]
    cfg["test_seeds"] = ",".join(str(s) for s in seeds)
    cfg["agent"] = agent
    out = a.output_dir or os.path.join(agent_dir, "eva_data")
    os.makedirs(out, exist_ok=True)
    out = out.rstrip("/") + "/"
    env = make_env(cfg, len(seeds), out)
    from deeprl_signal_control_b200.agents.evaluator import Evaluator, build_model, entry_model
    model = build_model(entry_model(agent), agent_dir, env, config, a.policy)
    ev = Evaluator(env, model, out, policy_type=a.evaluation_policy_type)
    mean, std = ev.run()
    control, traffic, trip = ev.recorded
    summary = ev.summary(mean, std, traffic, trip)
    with open(os.path.join(out, "%s_summary.json" % agent), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps({k: summary[k] for k in ("mean_reward", "std_reward", "avg_queue", "avg_speed_mps", "avg_wait_sec",
                                              "mean_trips")}))
    return summary


if __name__ == "__main__":
    main()
