"""Wall time of a training run with and without the TensorBoard summaries (`train(..., summaries=True)`).

  python scripts/time_summaries.py [--replicas 1024] [--total-step 3600] [--pairs 3]

Trains MA2C on the grid with the settings of the reference's config_ma2c_large.ini (3600 s episodes, batch_size 120),
`total_step` control steps, no tests, R replicas, into temporary directories: one warm-up run, then `--pairs` pairs of
runs alternating off / on in one process.  Prints one JSON line with every wall time, the card's name and its power
limit, and writes it to $OUT/time_summaries.json (OUT defaults to results/).
"""
import argparse
import configparser
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODEL = dict(rmsp_alpha="0.99", rmsp_epsilon="1e-5", max_grad_norm="40", gamma="0.99", lr_init="5e-4",
             lr_decay="constant", entropy_coef_init="0.01", entropy_coef_min="0.01", entropy_decay="constant",
             entropy_ratio="0.5", value_coef="0.5", num_fw="128", num_ft="32", num_lstm="64", num_fp="64",
             batch_size="120", reward_norm="2000.0", reward_clip="2.0")
ENV = dict(clip_wave="2.0", clip_wait="2.0", control_interval_sec="5", agent="ma2c", coop_gamma="0.9",
           data_path="./large_grid/data/", episode_length_sec="3600", norm_wave="5.0", norm_wait="100.0",
           coef_wait="0.2", peak_flow1="1100", peak_flow2="925", init_density="0", objective="hybrid",
           scenario="large_grid", seed="12", test_seeds="10000,20000", yellow_interval_sec="2")


def config(total_step):
    cp = configparser.ConfigParser()
    cp["MODEL_CONFIG"] = MODEL
    cp["TRAIN_CONFIG"] = dict(total_step=str(total_step), test_interval="1e9", log_interval="1e4")
    cp["ENV_CONFIG"] = ENV
    return cp


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--replicas", type=int, default=1024)
    p.add_argument("--total-step", type=int, default=3600)
    p.add_argument("--pairs", type=int, default=3)
    a = p.parse_args()
    import logging
    import torch
    from deeprl_signal_control_b200.agents.train import train
    if not torch.cuda.is_available():
        raise SystemExit("time_summaries.py needs a CUDA device")
    logging.disable(logging.INFO)
    runs = {"off": [], "on": []}
    with tempfile.TemporaryDirectory() as tmp:
        train(config(720), os.path.join(tmp, "warmup"), "no_test", n_replicas=a.replicas)
        for i in range(a.pairs):
            for mode in ("off", "on"):
                out = train(config(a.total_step), os.path.join(tmp, "%s%d" % (mode, i)), "no_test",
                            n_replicas=a.replicas, summaries=mode == "on")
                torch.cuda.synchronize()
                runs[mode].append(round(out.wall_sec, 3))
    res = {"card": card(), "replicas": a.replicas, "total_step": a.total_step, "wall_sec": runs,
           "min_off": min(runs["off"]), "min_on": min(runs["on"])}
    line = json.dumps(res)
    print(line)
    out_dir = os.environ.get("OUT", "results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_summaries.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
