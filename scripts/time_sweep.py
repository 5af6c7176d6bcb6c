"""Wall time of a hyperparameter sweep (K members of grid MA2C in one process) against the same K runs one after another.

  python scripts/time_sweep.py [--members 4,8] [--replicas 512,1024] [--reps 3] [--kernel-iters 200]

Grid MA2C with the settings of the reference's config_ma2c_large.ini (3600 s episodes = 720 control steps, batch_size
120, num_fw 128 / num_ft 32 / num_fp 64 / num_lstm 64).  Member k differs from the others in lr, entropy coefficient,
gamma and coop_gamma (MEMBER_VALUES).  For every K x R_m:
* episode set: one warm-up episode set, then the fastest of `--reps` timed episode sets (720 control steps, 6 updates,
  host clock around work that ends in a device synchronise) of the sweep (`BatchedA2C(seeds=..., hparams=...)` +
  `BatchedTrainer` with per-member schedules and coop_gamma) on K * R_m replicas, and of each member's solo run on R_m
  replicas on a simulator built with its coop_gamma; "solo_seq" is the sum of the K solo times;
* kernels: CUDA events around `--kernel-iters` launches of tscl_returns_g and tscl_device_transition_g on the sweep's
  rollout buffers against as many rounds of K one-member launches on R_m-replica buffers, per launch / round.
A sweep whose activation store does not fit the card is reported as such.  Prints one JSON line per shape, each with
the card's name and power limit, and writes them to $OUT/time_sweep.json (OUT defaults to results/).
"""
import argparse
import ctypes as C
import dataclasses
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.time_population import card  # noqa: E402

SEED0 = 12
N_STEP = 120                                         # config_ma2c_large.ini batch_size


def member_values(k):
    """(lr, beta, gamma, coop_gamma) of member k: a grid around the config_ma2c_large.ini values"""
    return 5e-4 * (1.0, 2.0, 0.5, 1.5)[k % 4], 0.01 * (1.0, 0.5)[(k // 4) % 2], (0.99, 0.95)[k % 2], (0.9, 0.75)[(k // 2) % 2]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--members", default="4,8")
    p.add_argument("--replicas", default="512,1024")
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--kernel-iters", type=int, default=200)
    a = p.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_sweep.py needs a CUDA device")
    from bench import build_scenario, make_layout
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
    from deeprl_signal_control_b200.sim import BatchedSim

    class A:
        agent, policy, scenario = "ma2c", "lstm", "large_grid"
    net, par, _, reward_norm = build_scenario(A)
    lay = make_layout(net, A)
    hp = lambda gamma: dict(gamma=gamma, v_coef=0.5, max_grad_norm=40.0, alpha=0.99, eps=1e-5, reward_norm=reward_norm,
                            reward_clip=2.0)

    def scenario(cg):
        scaled = np.asarray(net.obs_scale) != 1.0
        return (dataclasses.replace(net, obs_scale=np.where(scaled, np.float32(cg), np.float32(1)).astype(np.float32)),
                dataclasses.replace(par, coop_gamma=cg))

    def timed(tr):
        tr.run(tr.T_episode)
        torch.cuda.synchronize()
        best = float("inf")
        for _ in range(a.reps):
            t0 = time.perf_counter()
            tr.run(tr.T_episode)
            torch.cuda.synchronize()
            best = min(best, time.perf_counter() - t0)
        assert tr.T_episode == 720
        return best

    def sweep(K, Rm):
        vals = [member_values(k) for k in range(K)]
        m = BatchedA2C(lay, Rm, N_STEP, seeds=[SEED0 + k for k in range(K)], hparams=[hp(v[2]) for v in vals])
        n_, p_ = scenario(vals[0][3])
        sim = BatchedSim(n_, p_, m.R)
        tr = BatchedTrainer(sim, m, "ma2c", lr=[v[0] for v in vals], beta=[v[1] for v in vals], coop_gamma=[v[3] for v in vals])
        return timed(tr), m

    def solo(k, Rm):
        lr, beta, gamma, cg = member_values(k)
        m = BatchedA2C(lay, Rm, N_STEP, seed=SEED0 + k, **hp(gamma))
        sim = BatchedSim(*scenario(cg), Rm)
        return timed(BatchedTrainer(sim, m, "ma2c", lr=lr, beta=beta, seed0=SEED0 + k))

    def kernel_ms(m, K, Rm):
        """(grouped, per-member) ms of the returns and of the reward hand-over on the sweep learner's buffers"""
        lib, st = _lib.lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
        ptr = lambda t: C.c_void_p(t.data_ptr())
        T, R, A_ = m.T, m.R, m.lay.A
        dpost = torch.zeros(T, device=m.dev)
        rew, grew, acc = torch.randn(R, A_, device=m.dev), torch.randn(R, device=m.dev), torch.zeros(R, device=m.dev)
        Rm_rows = lambda t, k: ptr(t[k * Rm:])          # member k's rows of a [R, ...] buffer
        calls = {
            "returns_g": lambda: lib.tscl_returns_g(m._h, ptr(m.rew_hist), ptr(m.val_hist), ptr(m.boot), ptr(dpost),
                                                    ptr(m.gamma_dev), C.c_int32(K), C.c_int32(T), C.c_int64(R), ptr(m.Rs),
                                                    ptr(m.Adv), st),
            # K one-member launches on R_m-replica buffers (the layout of K solo learners)
            "returns_solo": lambda: [lib.tscl_returns(m._h, ptr(sr[k]), ptr(sv[k]), ptr(sb[k]), ptr(dpost),
                                                      C.c_float(0.99), C.c_int32(T), C.c_int64(Rm), ptr(sR[k]), ptr(sA[k]),
                                                      st) for k in range(K)],
            "transition_g": lambda: lib.tscl_device_transition_g(m._h, ptr(rew), ptr(m.rew_hist[0]), C.c_int64(R * A_),
                                                                 ptr(m.rnorm_dev), ptr(m.rclip_dev), C.c_int32(K),
                                                                 ptr(grew), ptr(acc), C.c_int64(R), st),
            "transition_solo": lambda: [lib.tscl_device_transition(m._h, Rm_rows(rew, k), Rm_rows(m.rew_hist[0], k),
                                                                   C.c_int64(Rm * A_), C.c_float(reward_norm),
                                                                   C.c_float(2.0), Rm_rows(grew, k), Rm_rows(acc, k),
                                                                   C.c_int64(Rm), st) for k in range(K)],
        }
        sr, sv, sR, sA = ([torch.randn(T, Rm, A_, device=m.dev) for _ in range(K)] for _ in range(4))
        sb = [torch.randn(Rm, A_, device=m.dev) for _ in range(K)]
        if m.rnorm_dev is None:                     # the timing sweep shares the reward scaling: time the kernel anyway
            m.rnorm_dev = torch.full((K,), reward_norm, device=m.dev)
            m.rclip_dev = torch.full((K,), 2.0, device=m.dev)
        out = {}
        for name, fn in calls.items():
            fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.kernel_iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            out[name + "_ms"] = round(e0.elapsed_time(e1) / a.kernel_iters, 4)
        return out

    name = card()
    lines = []
    for Rm in [int(x) for x in a.replicas.split(",")]:
        for K in [int(x) for x in a.members.split(",")]:
            res = {"K": K, "R_m": Rm, "card": name, "members": [member_values(k) for k in range(K)]}
            try:
                t_sw, m = sweep(K, Rm)
            except ValueError as e:
                res["sweep"] = "rejected: %s" % e
                lines.append(res); print(json.dumps(res), flush=True)
                continue
            res["sweep_episode_set_s"] = round(t_sw, 3)
            res.update(kernel_ms(m, K, Rm))
            del m
            torch.cuda.empty_cache()
            solo_t = [round(solo(k, Rm), 3) for k in range(K)]
            torch.cuda.empty_cache()
            res["solo_episode_set_s"] = solo_t
            res["solo_seq_s"] = round(sum(solo_t), 3)
            res["speedup"] = round(sum(solo_t) / t_sw, 3)
            lines.append(res)
            print(json.dumps(res), flush=True)
    out_dir = os.environ.get("OUT", "results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_sweep.json"), "w") as f:
        for r in lines:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
