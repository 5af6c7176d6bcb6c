"""Test-mode evaluation of a trained agent on every evaluation seed at once: the reference's `main.py evaluate`
(main.py:35-43, 158-198) on the batched device evaluator (deeprl_signal_control_b200/agents/evaluator.py).

  python scripts/evaluate.py --agent-dir DIR [--evaluation-policy-type default|stochastic|deterministic]
                             [--evaluation-seeds 2000,2001,... | --n-seeds N --seed0 S] [--output-dir OUT]
                             [--policy lstm|fc]

DIR holds `data/*.ini` (the run's config, [ENV_CONFIG] + [MODEL_CONFIG]) and, unless the agent is greedy,
`model/checkpoint-<step>.npz` as written by IA2C.save / MA2C.save / IQL.save.  The agent is the directory's name, as in
the reference (main.py:179-190): ia2c, ma2c, greedy, iqld (IQL with DeepQPolicy) or any other name, e.g. iqll (IQL with
LRQPolicy).  Writes the reference's `<scenario>_<agent>_{control,traffic,trip}.csv` and
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

from deeprl_signal_control_b200.envs import greedy_controller, make_env  # noqa: E402


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


def iql_model_type(agent):
    """main.py:185-190: 'iqld' is the DeepQPolicy IQL, every other agent name that is not an A2C variant or greedy the
    LRQPolicy one."""
    return 'dqn' if agent == 'iqld' else 'lr'


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
    if agent == "greedy":
        model = greedy_controller(env)
    else:
        from deeprl_signal_control_b200.agents.models import IA2C, IQL, MA2C
        mc = config["MODEL_CONFIG"]
        kw = dict(n_replicas=1, obs_off=env._tables.node_obs_off, policy=a.policy)
        if agent == "ma2c":
            model = MA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, env.n_f_ls, 0, mc, **kw)
        elif agent == "ia2c":
            model = IA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, 0, mc, **kw)
        elif agent == "a2c":
            raise SystemExit("batched evaluation covers greedy, ia2c, ma2c and IQL (got %r)" % agent)
        else:
            model = IQL(env.n_s_ls, env.n_a_ls, env.n_w_ls, 0, mc, seed=0, model_type=iql_model_type(agent))
        if not model.load(os.path.join(agent_dir, "model") + "/"):
            raise SystemExit("no checkpoint under %s/model/" % agent_dir)
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
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
