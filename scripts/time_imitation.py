"""Cost of imitation of a signal controller in the A2C update (BatchedA2C(teacher=...), DESIGN §5 Imitation).

  python scripts/time_imitation.py [--pairs 5] [--iters 5]

* backward: one BatchedA2C.backward() at the bench shape (grid MA2C, R = 4096, n_step 120, chunks of 1024) of a learner
  with the max-pressure teacher (lam = 0.5), and of the same learner with its teacher switched off (it then launches
  what a learner without a teacher launches; two learners' activation stores do not both fit), the arms alternating
  `--pairs` times, CUDA events around `--iters` updates each (median, min and max of the per-update time over the pairs);
* fused kernel: tscl_lstm_seq_bwd_tc_heads against tscl_lstm_seq_bwd_tc_heads_imit over the same four chunks, alone;
* control step: BatchedTrainer.control_step() on the grid at R = 4096 without a teacher and with the max-pressure and
  greedy teachers (one label launch each), updates excluded (CUDA events around each step that is not followed by one).
Prints one JSON line per measurement, each with the card's name and power limit, and writes them to
$OUT/time_imitation.json (OUT defaults to results/).
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.time_population import card  # noqa: E402


def _stat(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs))


def _learner(teacher, R=4096, T=120):
    import torch
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from tests.test_update_bench_size_gpu import _layout
    lay = _layout("grid")
    m = BatchedA2C(lay, R, n_step=T, seed=7, chunk=1024, reward_norm=2000.0, reward_clip=2.0, teacher=teacher)
    g = torch.Generator(device="cuda").manual_seed(3)
    for t in range(T):
        m.obs_slot().copy_(torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2)
        m.forward(m.obs_slot(), t == 0)
        m.add_transition(torch.randn(R, lay.A, device="cuda", generator=g) * 3000, t == 0, False)
    if teacher:
        na = torch.as_tensor(lay.n_a, device="cuda")
        m.teach_hist.copy_((torch.rand(T, R, lay.A, device="cuda", generator=g) * na).long().clamp_max(na - 1))
    return m


def time_backward(pairs, iters):
    import torch
    m = _learner("maxpressure")
    assert m.store_acts
    arms = ("no teacher", "maxpressure teacher")

    def one(k):
        m.t, m._acts_ok = m.T, [True] * m.T                   # the same rollout again
        if k == "no teacher":
            m.teacher = None
            m.backward(None, 0.0, 0.01)
            m.teacher = "maxpressure"
        else:
            m.backward(None, 0.0, 0.01, 0.5)
    for k in arms:
        one(k)
    res = {k: [] for k in arms}
    for _ in range(pairs):
        for k in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                one(k)
            e1.record()
            torch.cuda.synchronize()
            res[k].append(e0.elapsed_time(e1) / iters)
    out = [dict(what="backward", arm=k, R=4096, n_step=120, ms=_stat(v)) for k, v in res.items()]
    # the fused kernel alone, on the last rollout's store
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    R, T, A = m.R, m.T, m.lay.A
    dz, G, st = m._dz_all_buf(), torch.zeros_like(m.G), torch.zeros(4, device="cuda")
    dpre = torch.zeros(T, device="cuda")
    base = (m._h, _p(m.Wt), _p(m.P), _p(m.st_g[0]), _p(m.st_c[0]), _p(m.st_h[0]), _p(m.c_bw), _p(dpre), _p(m.act_hist[0]),
            _p(m.Rs[0]), _p(m.Adv[0]), T, m.chunk, R // m.chunk, R, 0, R * A, 0.5, 0.01, 1.0 / (T * R), _p(dz), _p(st),
            _p(G))
    arms = {"tscl_lstm_seq_bwd_tc_heads": lambda: _lib.lib().tscl_lstm_seq_bwd_tc_heads(*base, m._st()),
            "tscl_lstm_seq_bwd_tc_heads_imit": lambda: _lib.lib().tscl_lstm_seq_bwd_tc_heads_imit(
                *base, _p(m.teach_hist[0]), 0.5, m._st())}
    for f in arms.values():
        _lib.check(f())
    res = {k: [] for k in arms}
    for _ in range(pairs):
        for k, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters * 4):
                _lib.check(f())
            e1.record()
            torch.cuda.synchronize()
            res[k].append(e0.elapsed_time(e1) / (iters * 4))
    out += [dict(what="fused heads + BPTT kernel", arm=k, R=4096, n_step=120, ms=_stat(v)) for k, v in res.items()]
    m.close()
    return out


def time_control_step(pairs, steps=19):
    import configparser
    import torch
    from deeprl_signal_control_b200.agents.train import build_model, teacher_kwargs
    from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
    from tests.test_evaluator_gpu import GRID_INI, MODEL_INI
    R = 4096
    trainers = {}
    for teacher in (None, "maxpressure", "greedy"):
        c = configparser.ConfigParser()
        c.read_string(GRID_INI % ("ma2c", 3600, "10000") + MODEL_INI)
        if teacher:
            c["MODEL_CONFIG"]["teacher"], c["MODEL_CONFIG"]["imitation_coef_init"] = teacher, "0.5"
        from deeprl_signal_control_b200.envs import make_env
        env = make_env(c["ENV_CONFIG"], R, "", is_record=False)
        model = build_model("ma2c", env, c["MODEL_CONFIG"], 3600, R, seed=3)
        trainers[teacher or "none"] = BatchedTrainer(env._ensure_sim(), model.batched, "ma2c", 5e-4, 0.01, seed0=5,
                                                     **teacher_kwargs(model, env))
    for tr in trainers.values():
        tr.run(2 * tr.model.T)                                   # warm-up, through an update
    res = {k: [] for k in trainers}
    for _ in range(pairs):
        for k, tr in trainers.items():
            times = []
            while len(times) < steps:
                if tr.model.t == tr.model.T - 1:                 # the next step updates: not timed
                    tr.control_step()
                    continue
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                tr.control_step()
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            res[k].append(statistics.median(times) * 1000.0)
    return [dict(what="control step", arm="teacher " + k, R=R, us=_stat(v)) for k, v in res.items()]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--pairs", type=int, default=5)
    p.add_argument("--iters", type=int, default=5)
    a = p.parse_args()
    gpu = card()
    out_dir = os.environ.get("OUT", "results")
    os.makedirs(out_dir, exist_ok=True)
    rows = time_backward(a.pairs, a.iters) + time_control_step(a.pairs)
    with open(os.path.join(out_dir, "time_imitation.json"), "w") as f:
        for r in rows:
            r["gpu"] = gpu
            print(json.dumps(r))
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
