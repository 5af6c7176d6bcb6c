"""Test-mode evaluation of several trained agents on the same seeds in one process: the reference's
`main.py --base-dir B evaluate --agents ...` (main.py:35-43, 158-222) on the grouped device evaluator
(deeprl_signal_control_b200/agents/evaluator.py:GroupEvaluator).

  python scripts/evaluate_agents.py --base-dir B --agents greedy,ia2c,ma2c,seed12/ma2c,seed13/ma2c
                                    [--evaluation-policy-type default|stochastic|deterministic]
                                    [--evaluation-seeds 10000,20000,...,100000] [--policy lstm|fc]

Each entry is an agent directory under B holding `data/*.ini` and, unless the agent is greedy, `model/checkpoint-*`.
The agent is the entry's last path component (ia2c, ma2c, greedy, iqld = IQL with DeepQPolicy, any other name = IQL
with LRQPolicy; a2c is refused).  An entry without a `/` writes the reference's
`<scenario>_<agent>_{control,traffic,trip}.csv` into B/eva_data/, an entry p/<agent> into B/eva_data/p/, each next to
`<agent>_summary.json` (as scripts/evaluate.py writes it).  B/eva_data/summary.csv compares the entries (one row each:
mean / std reward, avg queue, speed, wait and mean trips); the log goes to B/eva_log/.  A missing directory, config or
checkpoint is logged as an error and the entry skipped.
"""
import argparse
import csv
import json
import logging
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# main.py:40-41: the reference's default evaluation seeds
DEFAULT_SEEDS = ",".join(str(s) for s in range(10000, 100001, 10000))
SUMMARY_COLUMNS = ("mean_reward", "std_reward", "avg_queue", "avg_speed_mps", "avg_wait_sec", "mean_trips")


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--base-dir", required=True)
    p.add_argument("--agents", required=True, help="comma-separated agent directories under the base directory")
    p.add_argument("--evaluation-policy-type", default="default", choices=["default", "stochastic", "deterministic"])
    p.add_argument("--evaluation-seeds", default=DEFAULT_SEEDS, help="comma-separated seeds")
    p.add_argument("--policy", default="lstm", choices=["lstm", "fc"])
    return p.parse_args(argv)


def entries(base_dir, agents):
    """[(label, agent directory, output directory)] of the --agents list: entry `a` writes into base/eva_data/, entry
    `p/a` into base/eva_data/p/.  Refuses repeated entries."""
    labels = [a.strip().strip("/") for a in agents.split(",") if a.strip()]
    if len(set(labels)) != len(labels):
        raise SystemExit("repeated entries in --agents: %s" % labels)
    out = []
    for lab in labels:
        sub = os.path.dirname(lab)
        out.append((lab, os.path.join(base_dir, lab), os.path.join(base_dir, "eva_data", sub).rstrip("/") + "/"))
    return out


def main(argv=None):
    a = parse_args(argv)
    from deeprl_signal_control_b200.agents.evaluator import GroupEvaluator, entry_model
    base = a.base_dir.rstrip("/")
    log_dir = os.path.join(base, "eva_log")
    os.makedirs(log_dir, exist_ok=True)
    root = logging.getLogger()
    root.setLevel(logging.INFO)
    handlers = [logging.FileHandler(os.path.join(log_dir, "%d.log" % time.time())), logging.StreamHandler()]
    for h in handlers:
        h.setFormatter(logging.Formatter("%(asctime)s [%(levelname)s] %(message)s"))
        root.addHandler(h)
    try:
        ent = entries(base, a.agents)
        for _, _, out in ent:
            os.makedirs(out, exist_ok=True)
        seeds = [int(s) for s in a.evaluation_seeds.split(",")]
        ge = GroupEvaluator([(d, entry_model(os.path.basename(d)), out) for _, d, out in ent], seeds,
                            policy_type=a.evaluation_policy_type, policy=a.policy)
        labels = {d: lab for lab, d, _ in ent}
        logging.info("Evaluation: %d entries on %d seeds, %d shared simulators"
                     % (len(ge.entries) - len(ge.skipped), len(seeds), len(ge.groups)))
        results = []
        for e in ge.run():
            with open(os.path.join(e.output_path, "%s_summary.json" % e.agent), "w") as f:
                json.dump(e.summary, f, indent=1)
            results.append((labels[e.agent_dir], e.summary))
        order = {lab: i for i, (lab, _, _) in enumerate(ent)}
        results.sort(key=lambda r: order[r[0]])
        with open(os.path.join(base, "eva_data", "summary.csv"), "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(("entry",) + SUMMARY_COLUMNS)
            for lab, s in results:
                w.writerow((lab,) + tuple(s.get(k, "") for k in SUMMARY_COLUMNS))
        for lab, s in results:
            print(json.dumps(dict(entry=lab, **{k: s.get(k) for k in SUMMARY_COLUMNS})))
        return results
    finally:
        for h in handlers:
            root.removeHandler(h)
            h.close()


if __name__ == "__main__":
    main()
