"""Cost of the deterministic A2C update (BatchedA2C(deterministic=True), tscl_set_deterministic) against the atomic one.

  python scripts/time_deterministic.py [--pairs 3] [--out results/time_deterministic.json]

At the bench workload (grid MA2C, 4096 replicas, chunk 1024, T = 120) and at Monaco MA2C (2048 replicas, T = 40), one
learner fills its rollout with seeded random observations and rewards, then runs whole updates (backward(): returns,
BPTT + heads, weight gradients, clip + RMSProp, repack) alternately in the two modes, --pairs pairs after one warm-up
pair, each timed with CUDA events.  A torch.profiler pass over one update per mode gives each kernel's device time, so
every deterministic kernel and reduce step stands beside its atomic counterpart.  The partial slabs' memory is the drop
in free device memory over the first deterministic update.  Prints the card name and power limit read in the same run,
one table per workload, and writes the numbers as JSON.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WORKLOADS = [("grid_ma2c", "large_grid", "ma2c", 4096, 120), ("monaco_ma2c", "real_net", "ma2c", 2048, 40)]
CHUNK = 1024


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


def layout(scenario, agent):
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    if scenario == "large_grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid
        net = build_large_grid(agent=agent)
    else:
        from deeprl_signal_control_b200.net.real_net import real_net_tables
        net = real_net_tables(agent=agent)
    return PolicyLayout(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, net.node_obs_off, net.n_obs, fw=128, ft=32,
                        ff=64 if agent == "ma2c" else 0, h=64)


def fill(m, g):
    for t in range(m.T):
        m.obs_slot().copy_(torch.rand(m.obs_slot().shape, generator=g, device=m.dev))
        m.forward(m.obs_slot(), False, to_hist=True)
        m.add_transition(torch.randn(m.R, m.lay.A, generator=g, device=m.dev) * 1000.0, False, False)


def run(name, scenario, agent, R, T, pairs):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    lib = _lib.lib()
    m = BatchedA2C(layout(scenario, agent), R, T, chunk=CHUNK, seed=1, reward_norm=2000.0, reward_clip=2.0,
                   deterministic=True)
    g = torch.Generator(device=m.dev).manual_seed(0)

    def update(on):
        _lib.check(lib.tscl_set_deterministic(m._h, on, 0))
        fill(m, g)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        m.backward(None, 5e-4, 0.01)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    update(0)
    free0 = torch.cuda.mem_get_info()[0]
    update(1)                                               # warm-up pair; the first deterministic update makes the slabs
    slab = free0 - torch.cuda.mem_get_info()[0]
    times = {0: [], 1: []}
    for _ in range(pairs):
        for on in (0, 1):
            times[on].append(update(on))
    kern = {}
    from torch.profiler import ProfilerActivity, profile
    for on in (0, 1):
        _lib.check(lib.tscl_set_deterministic(m._h, on, 0))
        fill(m, g)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m.backward(None, 5e-4, 0.01)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" and ev.count:
                k = ev.key.split("(")[0][:60]
                kern.setdefault(k, {0: 0.0, 1: 0.0})[on] += ev.device_time_total / 1000.0
    m.close()
    return dict(workload=name, replicas=R, T=T, chunk=CHUNK, update_ms_atomic=times[0], update_ms_det=times[1],
                slab_bytes=int(slab), kernels_ms={k: [v[0], v[1]] for k, v in sorted(kern.items())})


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--pairs", type=int, default=3)
    p.add_argument("--out", default="results/time_deterministic.json")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_deterministic.py needs a CUDA device")
    res = dict(card=card(), workloads=[])
    print("card, power limit, max SM clock:", res["card"])
    for w in WORKLOADS:
        r = run(*w, a.pairs)
        res["workloads"].append(r)
        at, de = sorted(r["update_ms_atomic"]), sorted(r["update_ms_det"])
        print("\n%s: %d replicas, T = %d, chunk %d; slabs %.1f MB" % (r["workload"], r["replicas"], r["T"], CHUNK,
                                                                   r["slab_bytes"] / 1e6))
        print("  whole update ms   atomic %s   deterministic %s   median ratio %.3f"
              % (["%.2f" % x for x in r["update_ms_atomic"]], ["%.2f" % x for x in r["update_ms_det"]],
                 de[len(de) // 2] / at[len(at) // 2]))
        print("  %-60s %10s %10s" % ("kernel (one update)", "atomic ms", "det ms"))
        for k, (x, y) in r["kernels_ms"].items():
            print("  %-60s %10.3f %10.3f" % (k, x, y))
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
