"""Batched IQL training on the device (agents/learner_iql.py): ms per control step split into rollout and update, and
the fused TD kernel's time and achieved fp32 FLOP/s, for grid R = 4096 and Monaco R = 2048, LR and DQN.

    python scripts/profile_iql_train.py [--steps 200] [--td-reps 20]
"""
import argparse
import configparser
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FP32_PEAK = 67e12            # NVIDIA H100 SXM data sheet, dense fp32 (700 W part)
CFG = """[MODEL_CONFIG]
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
buffer_size = 1000
reward_norm = 3000.0
reward_clip = 2.0
"""


def td_flops(lay, R, batch):
    """FMA-counted FLOPs of one tscl_q_td call: forward of s and s1, backward (weight and input gradients) of s."""
    rows = R * batch
    total = 0
    for i in range(lay.A):
        n_s, n_a, n_w = int(lay.n_s[i]), int(lay.n_a[i]), int(lay.n_w[i])
        if lay.model_type == "dqn":
            fwd = (n_s - n_w) * lay.n_fc + n_w * (lay.n_ft if n_w else 0)
            h1 = lay.n_fc + (lay.n_ft if n_w else 0)
            fwd += h1 * lay.n_h + lay.n_h * n_a
            bwd = fwd + h1 * lay.n_h          # weight gradients of every layer + dh1
        else:
            fwd = n_s * n_a
            bwd = fwd
        total += 2 * rows * (2 * fwd + bwd)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--td-reps", type=int, default=20)
    args = ap.parse_args()
    from deeprl_signal_control_b200.agents.layout import QLayout
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL, BatchedIQLTrainer
    from deeprl_signal_control_b200.agents.utils import Scheduler
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("card:", smi)
    cp = configparser.ConfigParser(); cp.read_string(CFG)
    cfg = cp["MODEL_CONFIG"]
    for scen, R in (("large_grid", 4096), ("real_net", 2048)):
        for kind in ("lr", "dqn"):
            agent = "iql" + kind[0]
            net = build_large_grid(agent=agent) if scen == "large_grid" else real_net_tables(agent)
            off = np.asarray(net.node_obs_off)
            n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
            lay = QLayout(kind, n_s, net.n_a_ls, net.n_w_ls, off, net.n_obs, n_fc=128, n_ft=32, n_h=64)
            m = BatchedIQL(lay, R, cfg, kind, seed=0, device=0)
            sim = BatchedSim(net, EnvParams(agent=agent), R, device=0)
            tr = BatchedIQLTrainer(sim, m, Scheduler(1e-4, decay="constant"), Scheduler(1.0, 0.01, 5e5, decay="linear"))
            tr.run(2 * m.n_step)                               # warm-up, fills the ring past batch_size
            tr.sim_events, tr.update_events = [], []
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            tr.run(args.steps)
            e1.record(); torch.cuda.synchronize()
            total = e0.elapsed_time(e1) / args.steps
            roll = sum(a.elapsed_time(b) for a, b in tr.sim_events) / args.steps
            upd = sum(a.elapsed_time(b) for a, b in tr.update_events) / args.steps
            # TD kernel (tscl_q_td: TD kernel + fixed-order reduction) alone over many launches
            m.sample(0)
            torch.cuda.synchronize()
            from deeprl_signal_control_b200 import _lib
            p = _lib.ptr
            lib = _lib.lib()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.td_reps):
                _lib.check(lib.tscl_q_td(m._h, p(m.P), p(m.s), p(m.s1), p(m.a), p(m.r), p(m.done), p(m.idx), R, 20,
                                         0.99, 1.0 / (20 * R), p(m.grad), m._st()))
            t1.record(); torch.cuda.synchronize()
            td_ms = t0.elapsed_time(t1) / args.td_reps
            fl = td_flops(lay, R, 20)
            print(json.dumps(dict(scenario=scen, R=R, model=kind, ms_per_step=round(total, 3),
                                  rollout_ms=round(roll, 3), update_ms_per_step=round(upd, 3),
                                  td_ms=round(td_ms, 3), td_gflop=round(fl / 1e9, 2),
                                  td_tflops=round(fl / td_ms / 1e9, 2), td_share_of_fp32_peak=round(fl / td_ms / 1e-3 / FP32_PEAK, 3),
                                  peak_mem_gb=round(torch.cuda.max_memory_allocated() / 1e9, 1))), flush=True)
            del tr, m, sim
            torch.cuda.empty_cache(); torch.cuda.reset_peak_memory_stats()


if __name__ == "__main__":
    main()
