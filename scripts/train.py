"""Train one agent into a reference agent directory: the reference's `main.py train` (main.py:21-48, 82-155) on the
device-resident learners (deeprl_signal_control_b200/agents/train.py).

  python scripts/train.py --base-dir DIR train --config-dir CFG.ini
                          [--test-mode no_test|in_train_test|after_train_test|all_test] [--replicas N] [--policy lstm|fc]
                          [--summaries] [--seeds 12,13,14,15 | --sweep a.ini,b.ini,...]
  torchrun --nproc-per-node W scripts/train.py --base-dir DIR train --config-dir CFG.ini --replicas N
                          [--backend nccl|gloo] ...

The agent is `[ENV_CONFIG] agent` of the config: ia2c, ma2c, iqld (IQL with DeepQPolicy) or any other name, e.g. iqll
(IQL with LRQPolicy).  `--replicas` lock-stepped environments train together (default 1, the reference's single
environment); the step counts control steps of the lock-step, so `total_step` gives as many updates as the reference's
run, each on N times the data.  DIR receives data/<config>.ini, data/train_reward.csv, model/checkpoint-<step>.npz and
log/<time>.log, and with after_train_test / all_test the three evaluation CSVs in data/.  Name DIR after the agent
and `scripts/evaluate.py --agent-dir DIR` evaluates the result.  Prints one JSON line: final step, episode sets, env
samples (steps x replicas) and wall seconds.  `--summaries` also writes the reference's TensorBoard event file into
log/ (agent 0's per-update losses and gradient norm, train_reward, test_reward): `tensorboard --logdir DIR/log`, or
`scripts/extract_summaries.py --log-dir DIR/log --scalar-name TAG` for a CSV.

Under torchrun with W > 1 processes, the N replicas are split over the W ranks (W must divide N), one GPU per rank
(LOCAL_RANK), and the learner all-reduces its gradient once per update over `--backend` (default nccl).  Rank 0 writes
the directory and prints the JSON line, with "world": W; the run plays the episodes of a one-process run with the same
--replicas.

`--seeds s1,s2,...` trains a population in one process: one member of the agent per seed (its [ENV_CONFIG] seed), each
on `--replicas` replicas (a multiple of 64), all in one lock-step.  Member s gets the complete agent directory
DIR/seed<s>/<agent>/ of a one-seed run, so `scripts/evaluate.py --agent-dir DIR/seed<s>/<agent>` reads it.  ia2c / ma2c
with the LSTM policy only, and not under torchrun.  The JSON line gains "seeds".

`--sweep a.ini,b.ini,...` trains a hyperparameter sweep in one process: one member per config, each on `--replicas`
replicas (a multiple of 64), all in one lock-step.  The configs may differ only in [ENV_CONFIG] seed / coop_gamma (ma2c)
and the [MODEL_CONFIG] learning-rate, entropy, value / gradient-norm, RMSProp, gamma and reward-scaling keys
(agents/train.py: SWEEP_CONFIG_KEYS).  Member a.ini gets the complete agent directory DIR/a/<agent>/ of
`train --config-dir a.ini`.  Not with --seeds, and not under torchrun.  The JSON line gains "members".
"""
import argparse
import datetime
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# The longest wait at a collective is the other ranks' at the barrier while rank 0 runs a test; a rank that fails ends
# the run after this long instead of leaving the others waiting.
TIMEOUT = datetime.timedelta(minutes=10)


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--base-dir", required=True, help="experiment base dir")
    sub = p.add_subparsers(dest="option", help="train")
    sp = sub.add_parser("train", help="train a single agent under base dir")
    sp.add_argument("--test-mode", default="no_test", help="test mode during training",
                    choices=["no_test", "in_train_test", "after_train_test", "all_test"])
    sp.add_argument("--config-dir", default="./config/config_test_large.ini", help="experiment config path")
    sp.add_argument("--replicas", type=int, default=1, help="lock-stepped environments in all ranks (default 1)")
    sp.add_argument("--policy", default="lstm", choices=["lstm", "fc"])
    sp.add_argument("--summaries", action="store_true",
                    help="also write the reference's TensorBoard event file into log/")
    sp.add_argument("--backend", default="nccl", choices=["nccl", "gloo"],
                    help="gradient all-reduce backend under torchrun (default nccl)")
    sp.add_argument("--seeds", default=None,
                    help="comma-separated seeds: train one population member per seed into DIR/seed<s>/<agent>/")
    sp.add_argument("--sweep", default=None,
                    help="comma-separated configs: train one sweep member per config into DIR/<config stem>/<agent>/")
    a = p.parse_args(argv)
    if not a.option:
        p.print_help()
        raise SystemExit(1)
    if a.sweep is not None:
        if a.seeds is not None:
            p.error("--sweep and --seeds exclude each other (a sweep takes each member's seed from its config)")
        a.sweep = [x.strip() for x in a.sweep.split(",") if x.strip()]
        if not a.sweep:
            p.error("--sweep needs at least one config")
    if a.seeds is not None:
        from deeprl_signal_control_b200.agents.train import parse_seeds
        try:
            a.seeds = parse_seeds(a.seeds)
        except ValueError as e:
            p.error(str(e))
    return a


def main(argv=None):
    a = parse_args(argv)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if a.sweep is not None:
        if world > 1:
            raise SystemExit("--sweep trains a sweep in one process; it does not run under torchrun")
        from deeprl_signal_control_b200.agents.train import train_sweep
        out = train_sweep(a.sweep, a.base_dir, a.test_mode, n_replicas=a.replicas, summaries=a.summaries,
                          policy=a.policy)
        print(json.dumps({"final_step": out.final_step, "episode_sets": out.episode_sets, "members": out.names,
                          "env_samples": out.env_samples, "replicas": a.replicas, "wall_sec": round(out.wall_sec, 3)}))
        return out
    if a.seeds is not None:
        if world > 1:
            raise SystemExit("--seeds trains a population in one process; it does not run under torchrun")
        from deeprl_signal_control_b200.agents.train import train
        out = train(a.config_dir, a.base_dir, a.test_mode, n_replicas=a.replicas, policy=a.policy,
                    summaries=a.summaries, seeds=a.seeds)
        print(json.dumps({"final_step": out.final_step, "episode_sets": out.episode_sets, "seeds": out.seeds,
                          "env_samples": out.env_samples, "replicas": a.replicas, "wall_sec": round(out.wall_sec, 3)}))
        return out
    if world <= 1:
        from deeprl_signal_control_b200.agents.train import train
        out = train(a.config_dir, a.base_dir, a.test_mode, n_replicas=a.replicas, policy=a.policy,
                    summaries=a.summaries)
        print(json.dumps({"final_step": out.final_step, "episode_sets": out.episode_sets,
                          "env_samples": out.env_samples, "replicas": a.replicas, "wall_sec": round(out.wall_sec, 3)}))
        return out
    local_rank = int(os.environ["LOCAL_RANK"])
    from deeprl_signal_control_b200.dist import bind_to_gpu_numa
    bind_to_gpu_numa(local_rank)                  # before torch allocates anything page-locked
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(local_rank)
    kw = {"device_id": torch.device("cuda", local_rank)} if a.backend == "nccl" else {}
    dist.init_process_group(a.backend, timeout=TIMEOUT, **kw)
    try:
        from deeprl_signal_control_b200.agents.train import train
        out = train(a.config_dir, a.base_dir, a.test_mode, n_replicas=a.replicas, policy=a.policy, device=local_rank,
                    process_group=dist.group.WORLD, summaries=a.summaries)
    finally:
        dist.destroy_process_group()
    if out.rank == 0:
        print(json.dumps({"final_step": out.final_step, "episode_sets": out.episode_sets,
                          "env_samples": out.env_samples, "replicas": a.replicas, "world": world,
                          "wall_sec": round(out.wall_sec, 3)}))
    return out


if __name__ == "__main__":
    main()
