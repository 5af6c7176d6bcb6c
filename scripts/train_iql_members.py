"""Train several seeds or configs of one IQL agent (iqll / iqld) in one process (deeprl_signal_control_b200/agents/
train.py: train_iql_population, train_iql_sweep).

  python scripts/train_iql_members.py --base-dir DIR (--config-dir CFG.ini --seeds 12,13,... | --sweep a.ini,b.ini,...)
                                      --replicas R_m [--test-mode no_test|in_train_test|after_train_test|all_test]
                                      [--summaries] [--vary-demand]

`--seeds` trains a population: one member per seed (its [ENV_CONFIG] seed) into DIR/seed<s>/<agent>/.  `--sweep` trains
one member per config into DIR/<config stem>/<agent>/; the configs may differ only in [ENV_CONFIG] seed and the
[MODEL_CONFIG] lr and ε schedules, gamma, max_grad_norm and reward scaling (agents/train.py: IQL_SWEEP_CONFIG_KEYS).
Every member trains on `--replicas` replicas; all members share one simulator, one replay ring and one grouped
ε-greedy forward and TD / Adam update, and each member's directory is the one `scripts/train.py train` leaves for it
alone, bit for bit.  At most 64 members; not under torchrun.  Prints one JSON line as scripts/train.py does, with
"seeds" or "members".  `--vary-demand` (with --sweep) lets the configs also differ in their scenario's demand keys
(envs.DEMAND_KEYS, as `scripts/train.py train --sweep ... --vary-demand`).
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--base-dir", required=True, help="experiment base dir")
    p.add_argument("--config-dir", default=None, help="experiment config path (with --seeds)")
    p.add_argument("--seeds", default=None,
                   help="comma-separated seeds: train one population member per seed into DIR/seed<s>/<agent>/")
    p.add_argument("--sweep", default=None,
                   help="comma-separated configs: train one sweep member per config into DIR/<config stem>/<agent>/")
    p.add_argument("--replicas", type=int, required=True, help="lock-stepped environments per member")
    p.add_argument("--test-mode", default="no_test", help="test mode during training",
                   choices=["no_test", "in_train_test", "after_train_test", "all_test"])
    p.add_argument("--summaries", action="store_true",
                   help="also write the reference's TensorBoard event file into each member's log/")
    p.add_argument("--vary-demand", action="store_true",
                   help="with --sweep: the configs may also differ in their scenario's traffic demand keys")
    a = p.parse_args(argv)
    if (a.seeds is None) == (a.sweep is None):
        p.error("give exactly one of --seeds (with --config-dir) and --sweep")
    if a.sweep is not None:
        if a.config_dir is not None:
            p.error("--sweep takes each member's config from the list; it takes no --config-dir")
        a.sweep = [x.strip() for x in a.sweep.split(",") if x.strip()]
        if not a.sweep:
            p.error("--sweep needs at least one config")
    else:
        if a.config_dir is None:
            p.error("--seeds needs --config-dir")
        if a.vary_demand:
            p.error("--vary-demand applies to a --sweep")
        from deeprl_signal_control_b200.agents.train import parse_seeds
        try:
            a.seeds = parse_seeds(a.seeds)
        except ValueError as e:
            p.error(str(e))
    return a


def main(argv=None):
    a = parse_args(argv)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise SystemExit("train_iql_members.py trains its members in one process; it does not run under torchrun")
    from deeprl_signal_control_b200.agents.train import train_iql_population, train_iql_sweep
    if a.sweep is not None:
        out = train_iql_sweep(a.sweep, a.base_dir, a.test_mode, n_replicas=a.replicas, summaries=a.summaries,
                              vary_demand=a.vary_demand)
        key, val = "members", out.names
    else:
        out = train_iql_population(a.config_dir, a.base_dir, a.seeds, a.test_mode, n_replicas=a.replicas,
                                   summaries=a.summaries)
        key, val = "seeds", out.seeds
    print(json.dumps({"final_step": out.final_step, "episode_sets": out.episode_sets, key: val,
                      "env_samples": out.env_samples, "replicas": a.replicas, "wall_sec": round(out.wall_sec, 3)}))
    return out


if __name__ == "__main__":
    main()
