"""Train one agent into a reference agent directory: the reference's `main.py train` (main.py:21-48, 82-155) on the
device-resident learners (deeprl_signal_control_b200/agents/train.py).

  python scripts/train.py --base-dir DIR train --config-dir CFG.ini
                          [--test-mode no_test|in_train_test|after_train_test|all_test] [--replicas N] [--policy lstm|fc]

The agent is `[ENV_CONFIG] agent` of the config: ia2c, ma2c, iqld (IQL with DeepQPolicy) or any other name, e.g. iqll
(IQL with LRQPolicy).  `--replicas` lock-stepped environments train together (default 1, the reference's single
environment); the step counts control steps of the lock-step, so `total_step` gives as many updates as the reference's
run, each on N times the data.  DIR receives data/<config>.ini, data/train_reward.csv, model/checkpoint-<step>.npz and
log/<time>.log, and with after_train_test / all_test the three evaluation CSVs in data/.  Name DIR after the agent
and `scripts/evaluate.py --agent-dir DIR` evaluates the result.  Prints one JSON line: final step, episode sets, env
samples (steps x replicas) and wall seconds.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--base-dir", required=True, help="experiment base dir")
    sub = p.add_subparsers(dest="option", help="train")
    sp = sub.add_parser("train", help="train a single agent under base dir")
    sp.add_argument("--test-mode", default="no_test", help="test mode during training",
                    choices=["no_test", "in_train_test", "after_train_test", "all_test"])
    sp.add_argument("--config-dir", default="./config/config_test_large.ini", help="experiment config path")
    sp.add_argument("--replicas", type=int, default=1, help="lock-stepped environments (default 1)")
    sp.add_argument("--policy", default="lstm", choices=["lstm", "fc"])
    a = p.parse_args(argv)
    if not a.option:
        p.print_help()
        raise SystemExit(1)
    return a


def main(argv=None):
    a = parse_args(argv)
    from deeprl_signal_control_b200.agents.train import train
    out = train(a.config_dir, a.base_dir, a.test_mode, n_replicas=a.replicas, policy=a.policy)
    print(json.dumps({"final_step": out.final_step, "episode_sets": out.episode_sets, "env_samples": out.env_samples,
                      "replicas": a.replicas, "wall_sec": round(out.wall_sec, 3)}))
    return out


if __name__ == "__main__":
    main()
