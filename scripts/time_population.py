"""Wall time of a population (K members of grid MA2C in one process) against the same K runs one after another.

  python scripts/time_population.py [--members 1,4,8] [--replicas 512,1024] [--reps 3] [--forward-iters 50]

Grid MA2C with the settings of the reference's config_ma2c_large.ini (3600 s episodes = 720 control steps, batch_size
120, num_fw 128 / num_ft 32 / num_fp 64 / num_lstm 64).  For every K x R_m:
* episode set: one warm-up episode set, then the fastest of `--reps` timed episode sets (720 control steps, 6 updates,
  host clock around work that ends in a device synchronise) of the population `BatchedA2C(seeds=...)` +
  `BatchedTrainer` on K * R_m replicas, and of each of the K solo learners on R_m replicas; "solo_seq" is the sum of
  the K solo times;
* forward: CUDA events around `--forward-iters` grouped forwards (tscl_policy_step_v2g, store on, sampled actions)
  against the same number of rounds of K per-member launches (tscl_policy_step_v2 on R_m replicas), per launch/round.
A population whose activation store does not fit the card is reported as such.  Prints one JSON line per shape, each
with the card's name and power limit, and writes them to $OUT/time_population.json (OUT defaults to results/).
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SEED0 = 12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--members", default="1,4,8")
    p.add_argument("--replicas", default="512,1024")
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--forward-iters", type=int, default=50)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_population.py needs a CUDA device")
    from bench import build_scenario, make_layout
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
    from deeprl_signal_control_b200.sim import BatchedSim

    class A:
        agent, policy, scenario = "ma2c", "lstm", "large_grid"
    net, par, _, reward_norm = build_scenario(A)
    lay = make_layout(net, A)
    kw = dict(gamma=0.99, v_coef=0.5, max_grad_norm=40.0, alpha=0.99, eps=1e-5, reward_norm=reward_norm,
              reward_clip=2.0)
    n_step = 120                                        # config_ma2c_large.ini batch_size

    def episode_set(seeds, Rm):
        """(fastest timed episode set after a warm-up one in seconds, learner, sim) of a population (list of seeds)
        or a solo run (one seed)"""
        pop = isinstance(seeds, list)
        m = BatchedA2C(lay, Rm, n_step, seeds=seeds, **kw) if pop else BatchedA2C(lay, Rm, n_step, seed=seeds, **kw)
        sim = BatchedSim(net, par, m.R)
        tr = BatchedTrainer(sim, m, "ma2c", lr=5e-4, beta=0.01, seed0=seeds[0] if pop else seeds)
        tr.run(tr.T_episode)
        torch.cuda.synchronize()
        best = float("inf")
        for _ in range(a.reps):
            t0 = time.perf_counter()
            tr.run(tr.T_episode)
            torch.cuda.synchronize()
            best = min(best, time.perf_counter() - t0)
        assert tr.T_episode == 720
        return best, m, sim

    def forward_ms(learners, obs_parts):
        """ms per round of one forward per learner (rollout slot 0, store on, sampled actions)"""
        for m, o in zip(learners, obs_parts):
            m.t = 0
            m.forward(o, False)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.forward_iters):
            for m, o in zip(learners, obs_parts):
                m.forward(o, False)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.forward_iters

    name = card()
    lines = []
    for Rm in [int(x) for x in a.replicas.split(",")]:
        for K in [int(x) for x in a.members.split(",")]:
            seeds = [SEED0 + k for k in range(K)]
            res = {"K": K, "R_m": Rm, "card": name}
            try:
                t_pop, m, sim = episode_set(seeds, Rm)
            except ValueError as e:
                res["population"] = "rejected: %s" % e
                lines.append(res); print(json.dumps(res), flush=True)
                continue
            obs = torch.rand(m.R, lay.n_obs, device=m.dev) * 2
            res["pop_forward_ms"] = round(forward_ms([m], [obs]), 4)
            res["pop_episode_set_s"] = round(t_pop, 3)
            del m, sim
            torch.cuda.empty_cache()
            solo_t, solos = [], []
            for k, s in enumerate(seeds):
                t, m, sim = episode_set(s, Rm)
                solo_t.append(round(t, 3))
                solos.append(m)
                del sim
            res["solo_forward_ms"] = round(forward_ms(solos, [obs[k * Rm:(k + 1) * Rm].contiguous()
                                                              for k in range(K)]), 4)
            del solos
            torch.cuda.empty_cache()
            res["solo_episode_set_s"] = solo_t
            res["solo_seq_s"] = round(sum(solo_t), 3)
            res["speedup"] = round(sum(solo_t) / t_pop, 3)
            lines.append(res)
            print(json.dumps(res), flush=True)
    out_dir = os.environ.get("OUT", "results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_population.json"), "w") as f:
        for r in lines:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
