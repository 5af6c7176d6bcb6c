"""Wall time of one agent trained on a mixture of traffic demand levels against the same run at the configured level.

  python scripts/time_demand_mix.py [--replicas 1024] [--pairs 3]

Grid MA2C with the settings of the reference's config_ma2c_large.ini (3600 s episodes = 720 control steps, batch_size
120, num_fw 128 / num_ft 32 / num_fp 64 / num_lstm 64) on `--replicas` replicas, two arms with one learner and one
simulator each:
* "configured": every replica at the configured peak flows (1100 / 925 veh/h), no demand levels set;
* "mix3": a 3-level mixture at x0.6, x1 and x1.4 of the peak flows, replica g at level g mod 3 (`BatchedTrainer` with
  demand_mix, as train(demand_mix=...) sets it up).  At R = 1024 the levels hold 342 / 341 / 341 replicas: train()
  asks for a multiple of L so that every level weighs the same, but the cost per replica does not depend on it.
Each arm first plays one untimed episode set, sampling the mean number of live vehicles per replica after every update;
then the arms alternate `--pairs` times, one timed episode set (720 control steps, 6 updates; host clock around work
that ends in a device synchronise) per arm and pair.  Prints one JSON line per arm (median, min and max seconds per
episode set, mean live vehicles) with the card's name and power limit, and writes them to $OUT/time_demand_mix.json
(OUT defaults to results/).
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.time_population import card  # noqa: E402

SEED0 = 12
N_STEP = 120                                         # config_ma2c_large.ini batch_size
FACTORS = (0.6, 1.0, 1.4)                            # peak-flow factors of the mixture


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--replicas", type=int, default=1024)
    p.add_argument("--pairs", type=int, default=3)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_demand_mix.py needs a CUDA device")
    from bench import build_scenario, make_layout
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.sim import BatchedSim

    class A:
        agent, policy, scenario = "ma2c", "lstm", "large_grid"
    net, par, _, reward_norm = build_scenario(A)
    lay = make_layout(net, A)
    R = a.replicas
    levels = [build_large_grid(int(1100 * f), int(925 * f), agent="ma2c") for f in FACTORS]

    def arm(mix):
        m = BatchedA2C(lay, R, N_STEP, gamma=0.99, v_coef=0.5, max_grad_norm=40.0, alpha=0.99, eps=1e-5,
                       reward_norm=reward_norm, reward_clip=2.0, seed=SEED0)
        sim = BatchedSim(net, par, R)
        tr = BatchedTrainer(sim, m, "ma2c", lr=5e-4, beta=0.01, seed0=SEED0, demand_mix=levels if mix else None)
        assert tr.T_episode == 720
        live = []
        for _ in range(tr.T_episode // N_STEP - 1):     # the last update ends the episode and resets the simulator
            tr.run(N_STEP)
            live.append(sim.mean_live())
        tr.run(N_STEP)
        torch.cuda.synchronize()
        return tr, statistics.mean(live)

    arms = {"configured": arm(False), "mix3": arm(True)}
    times = {k: [] for k in arms}
    for _ in range(a.pairs):
        for k, (tr, _) in arms.items():
            t0 = time.perf_counter()
            tr.run(tr.T_episode)
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    name = card()
    lines = []
    for k, ts in times.items():
        lines.append(dict(arm=k, replicas=R, levels=[1.0] if k == "configured" else list(FACTORS), pairs=a.pairs,
                          episode_set_s_median=round(statistics.median(ts), 3), s_min=round(min(ts), 3),
                          s_max=round(max(ts), 3), mean_live_vehicles=round(arms[k][1], 1), card=name))
    lines.append(dict(what="mix3 / configured", ratio_of_medians=round(lines[1]["episode_set_s_median"] /
                                                                     lines[0]["episode_set_s_median"], 4), card=name))
    out_dir = os.environ.get("OUT", "results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_demand_mix.json"), "w") as f:
        for r in lines:
            print(json.dumps(r), flush=True)
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
