"""Time IQL members (BatchedIQL with seeds, tscl_q_*_g) against the same members trained one after another.

  python scripts/time_iql_population.py [--agents iqld,iqll] [--members 1,4,8] [--replicas 256,512] [--episode-sec 300]
                                        [--buffer-size 200] [--rounds 20] [--pairs 3] [--out DIR]

For each agent (grid layout), member count K and replicas per member R_m:
* round: one TD + clip / Adam round of all K members (tscl_q_td_g, tscl_q_adam_g) against K solo rounds in sequence,
  on the same filled ring, CUDA events around `--rounds` rounds; the two arms alternate `--pairs` times;
* episode set: one episode of the population trainer (K * R_m replicas) against K solo trainers' episodes in sequence,
  host clock around work that ends in a device synchronise, arms alternating `--pairs` times (the first episode of each
  arm is a warm-up and is not timed);
* peak device memory of each arm: torch.cuda.max_memory_allocated over its set-up and warm-up episode, less what the
  other arm already held.
Episodes are shortened to `--episode-sec` simulated seconds and the ring to `--buffer-size` slots, so that the largest
shape fits next to its solo arm; the update cadence (batch_size 20, 10 rounds) is the reference's.  Prints one JSON line
per shape with medians and the (min, max) spread, plus the card's name and power limit, and writes them to
DIR/time_iql_population.json when --out is given.
"""
import argparse
import configparser
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODEL = """[MODEL_CONFIG]
max_grad_norm = 40
gamma = 0.99
lr_init = 1e-4
lr_decay = constant
epsilon_init = 1.0
epsilon_min = 0.01
epsilon_decay = linear
epsilon_ratio = 0.5
num_fc = 128
num_h = 64
batch_size = 20
buffer_size = %d
reward_norm = 3000.0
reward_clip = 2.0
"""


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


def run_shape(agent, K, R_m, args, torch):
    from deeprl_signal_control_b200.agents.layout import QLayout
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL, BatchedIQLTrainer
    from deeprl_signal_control_b200.agents.models import iql_schedulers
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    kind = "dqn" if agent == "iqld" else "lr"
    net = build_large_grid(agent=agent)
    off = np.asarray(net.node_obs_off)
    n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
    cp = configparser.ConfigParser(); cp.read_string(MODEL % args.buffer_size)
    mc = cp["MODEL_CONFIG"]
    lay = QLayout(kind, n_s, net.n_a_ls, net.n_w_ls, off, net.n_obs, n_fc=128 if kind == "dqn" else 0,
                  n_ft=32 if kind == "dqn" else 0, n_h=64 if kind == "dqn" else 0, max_na=net.max_na)
    par = EnvParams(agent=agent, episode_length_sec=args.episode_sec)
    seeds = [12 + k for k in range(K)]
    res = {"agent": agent, "K": K, "R_m": R_m, "episode_steps": int(args.episode_sec // 5),
           "buffer_size": args.buffer_size}

    def sched():
        return iql_schedulers(mc, 10 ** 6)

    # ---- episode sets ----
    def pop_arm():
        m = BatchedIQL(lay, R_m, mc, kind, seeds=seeds if K > 1 else None)
        sc = [sched() for _ in range(K)]
        lr, eps = ([s[0] for s in sc], [s[1] for s in sc]) if K > 1 else sc[0]
        tr = BatchedIQLTrainer(BatchedSim(net, par, K * R_m, device=0), m, lr, eps, seed0=seeds[0])
        return [(tr, m)]

    def solo_arm():
        out = []
        for s in seeds:
            m = BatchedIQL(lay, R_m, mc, kind)
            lr, eps = sched()
            out.append((BatchedIQLTrainer(BatchedSim(net, par, R_m, device=0), m, lr, eps, seed0=s), m))
        return out

    T = res["episode_steps"]
    times, mem = {"population": [], "solo": []}, {}
    for name, make in (("population", pop_arm), ("solo", solo_arm)):
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()                      # the other arm, still resident
        arm = make()
        for tr, _ in arm:
            tr.run(T)                                             # warm-up episode (the ring fills)
        torch.cuda.synchronize()
        mem[name] = (torch.cuda.max_memory_allocated() - base) / 1e9
        times[name + "_arm"] = arm
    for _ in range(args.pairs):
        for name in ("population", "solo"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for tr, _ in times[name + "_arm"]:
                tr.run(T)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
    res["episode_set_sec"] = {"population": stats(times["population"]), "solo_in_sequence": stats(times["solo"])}
    res["peak_gb"] = {"population": round(mem["population"], 3), "solo_in_sequence": round(mem["solo"], 3)}

    # ---- rounds on the filled rings ----
    pop = times["population_arm"][0][1]
    solos = [m for _, m in times["solo_arm"]]
    lr = [1e-4] * K if K > 1 else 1e-4
    ev = lambda: torch.cuda.Event(enable_timing=True)
    rt = {"grouped": [], "solo": []}
    for _ in range(args.pairs):
        for name in ("grouped", "solo"):
            e0, e1 = ev(), ev()
            e0.record()
            for r in range(args.rounds):
                if name == "grouped":
                    pop.td_round(r % 10, lr)
                else:
                    for m in solos:
                        m.td_round(r % 10, 1e-4)
            e1.record()
            torch.cuda.synchronize()
            rt[name].append(e0.elapsed_time(e1) / args.rounds)
    res["round_ms"] = {"grouped": stats(rt["grouped"]), "solo_in_sequence": stats(rt["solo"])}
    del times
    return res


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--agents", default="iqld,iqll")
    p.add_argument("--members", default="1,4,8")
    p.add_argument("--replicas", default="256,512")
    p.add_argument("--episode-sec", type=int, default=300)
    p.add_argument("--buffer-size", type=int, default=200)
    p.add_argument("--rounds", type=int, default=20)
    p.add_argument("--pairs", type=int, default=3)
    p.add_argument("--out", default=None)
    a = p.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_iql_population.py measures on the GPU; no CUDA device is visible")
    dev = card()
    rows = []
    for agent in a.agents.split(","):
        for R_m in [int(x) for x in a.replicas.split(",")]:
            for K in [int(x) for x in a.members.split(",")]:
                r = run_shape(agent, K, R_m, a, torch)
                r["device"] = dev
                print(json.dumps(r), flush=True)
                rows.append(r)
                import gc
                gc.collect()
                torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_iql_population.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
