"""Wall time of evaluating K grid MA2C agent directories (a sweep's members: distinct seeds and coop_gammas) on S seeds:

* grouped   one GroupEvaluator run (scripts/evaluate_agents.py's path: one simulator, one tscl_policy_step_pi_g per step);
* serial    K in-process `Evaluator` runs one after another (scripts/evaluate.py's path without the process start);
* procs     K `scripts/evaluate.py` processes one after another (K <= --proc-max-k only: each pays CUDA start-up);
* kernels   CUDA events around tscl_policy_step_pi_g against K tscl_policy_step_pi launches on the same inputs, and
            tscl_q_step_g against K tscl_q_step launches (IQL LR, grid), each over --iters launches.

  python scripts/time_evaluate_agents.py [--ks 4,8,32] [--ss 10,1000] [--episode-sec 3600] [--repeats 3] [--out DIR]

Prints one JSON line per (K, S) with the card and its power limit, the median and spread of --repeats runs; writes them
to OUT/time_evaluate_agents.json (default results/).  The directories hold randomly initialised checkpoints: the timing
does not depend on the weights.
"""
import argparse
import configparser
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MODEL = """[MODEL_CONFIG]
rmsp_alpha = 0.99
rmsp_epsilon = 1e-5
max_grad_norm = 40
gamma = 0.99
lr_init = 5e-4
lr_decay = constant
entropy_coef_init = 0.01
entropy_coef_min = 0.01
entropy_decay = constant
entropy_ratio = 0.5
value_coef = 0.5
num_fw = 128
num_ft = 32
num_lstm = 64
num_fp = 64
batch_size = 120
reward_norm = 2000.0
reward_clip = 2.0
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = ma2c
coop_gamma = %s
data_path = ./large_grid/data/
episode_length_sec = %d
norm_wave = 5.0
norm_wait = 100.0
coef_wait = 0.2
peak_flow1 = 1100
peak_flow2 = 925
init_density = 0
objective = hybrid
scenario = large_grid
seed = %d
test_seeds = 10000
yellow_interval_sec = 2
"""


def make_dirs(base, K, episode_sec):
    from deeprl_signal_control_b200.agents.models import MA2C
    from deeprl_signal_control_b200.envs import make_env
    dirs = []
    for k in range(K):
        d = os.path.join(base, "m%d" % k, "ma2c")
        os.makedirs(os.path.join(d, "data")); os.makedirs(os.path.join(d, "model"))
        c = configparser.ConfigParser()
        c.read_string(MODEL % ((0.9, 0.75, 0.5)[k % 3], episode_sec, 12 + k))
        with open(os.path.join(d, "data", "config.ini"), "w") as f:
            c.write(f)
        env = make_env(c["ENV_CONFIG"], 1, d + "/", is_record=False)
        m = MA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, env.n_f_ls, 0, c["MODEL_CONFIG"], n_replicas=1,
                 obs_off=env._tables.node_obs_off, seed=k)
        m.save(os.path.join(d, "model"), 0)
        dirs.append(d)
    return dirs


def run_grouped(dirs, seeds, out):
    import torch
    from deeprl_signal_control_b200.agents.evaluator import GroupEvaluator
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    GroupEvaluator([(d, "ma2c", out + "/") for d in dirs], seeds).run()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def run_serial(dirs, seeds, out):
    import torch
    ev = _load("evaluate")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for d in dirs:
        ev.main(["--agent-dir", d, "--output-dir", out, "--evaluation-seeds", ",".join(map(str, seeds))])
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def run_procs(dirs, seeds, out):
    t0 = time.perf_counter()
    for d in dirs:
        subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", d, "--output-dir",
                        out, "--evaluation-seeds", ",".join(map(str, seeds))], check=True, capture_output=True)
    return time.perf_counter() - t0


def _load(name):
    import importlib.util
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "scripts", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _events(fn, iters):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3          # us per call


def time_kernels(K, S, iters):
    """(grouped, K member launches) in us per step for the pi-only forward (grid MA2C) and the Q forward (grid LR)."""
    import numpy as np
    import torch
    from bench import build_scenario, make_layout
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.layout import QLayout
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from deeprl_signal_control_b200.agents.models import IQL
    lib, st = _lib.lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())
    R = K * S

    class A:
        scenario, agent, policy = "large_grid", "ma2c", "lstm"
    net = build_scenario(A)[0]
    lay = make_layout(net, A)
    ms = [BatchedA2C(lay, 64, n_step=2, seed=k, chunk=64, store_acts=False) for k in range(K)]
    P, Wp = torch.stack([m.P for m in ms]).contiguous(), torch.stack([m.Wp for m in ms]).contiguous()
    rows = torch.arange(0, R + 1, S, dtype=torch.int64, device="cuda")
    seeds = torch.arange(K, dtype=torch.int64, device="cuda")
    obs = torch.rand(R, lay.n_obs, device="cuda")
    c, h = torch.zeros(lay.A, R, lay.h, device="cuda"), torch.zeros(lay.A, R, lay.h, device="cuda")
    pi = torch.zeros(R, lay.A, lay.max_na, device="cuda")
    act = torch.zeros(R, lay.A, dtype=torch.int32, device="cuda")
    cm, hm = torch.zeros(lay.A, S, lay.h, device="cuda"), torch.zeros(lay.A, S, lay.h, device="cuda")
    grouped = lambda: _lib.check(lib.tscl_policy_step_pi_g(
        ms[0]._h, p(P), C.c_int64(P.shape[1]), p(Wp), C.c_int64(Wp[0].numel()), p(obs), C.c_int32(K), p(rows), C.c_int64(R),
        p(c), p(h), p(c), p(h), p(pi), p(act), C.c_int32(0), C.c_int32(0), p(seeds), C.c_int64(1), st))

    def members():
        for k, m in enumerate(ms):
            _lib.check(lib.tscl_policy_step_pi(m._h, p(m.P), p(m.Wp), p(obs[k * S:(k + 1) * S]), C.c_int64(S), p(cm), p(hm),
                                               p(cm), p(hm), p(pi[k * S:]), p(act[k * S:]), C.c_int32(0), C.c_int32(0),
                                               C.c_uint64(k), C.c_int64(1), C.c_int64(0), C.c_int64(0), C.c_int64(0), st))
    out = {"pi_g_us": _events(grouped, iters), "pi_members_us": _events(members, iters)}
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    qnet = build_large_grid(agent="iqll")
    cp = configparser.ConfigParser()
    cp.read_string("[M]\nmax_grad_norm = 40\ngamma = 0.99\nnum_fc = 128\nnum_h = 64\nbatch_size = 20\n"
                   "buffer_size = 1000\nreward_norm = 3000.0\nreward_clip = 2.0\n")
    qm = IQL(qnet.n_s_ls, qnet.n_a_ls, qnet.n_w_ls, 0, cp["M"], seed=0, model_type="lr", device="cuda")
    ql = QLayout.from_iql(qm, np.asarray(qnet.node_obs_off), qnet.n_obs, max_na=qnet.max_na)
    hq = C.c_void_p()
    _lib.check(lib.tscl_q_create(C.byref(ql.as_c()), C.c_int32(0), C.byref(hq)))
    QP = ql.pack(qm.nets).cuda().repeat(K, 1).contiguous()
    qobs = torch.rand(R, qnet.n_obs, device="cuda")
    q = torch.zeros(R, ql.A, ql.max_na, device="cuda")
    qact = torch.zeros(R, ql.A, dtype=torch.int32, device="cuda")
    qg = lambda: _lib.check(lib.tscl_q_step_g(hq, p(QP), C.c_int64(ql.n_params), p(qobs), C.c_int32(K), p(rows),
                                              C.c_int64(R), p(q), p(qact), C.c_int32(0), p(seeds), C.c_int64(1), None, st))

    def qmembers():
        for k in range(K):
            _lib.check(lib.tscl_q_step(hq, p(QP[k]), p(qobs[k * S:]), C.c_int64(S), p(q[k * S:]), p(qact[k * S:]),
                                       C.c_int32(0), C.c_uint64(k), C.c_int64(1), C.c_int64(0), None, st))
    out.update(q_g_us=_events(qg, iters), q_members_us=_events(qmembers, iters))
    lib.tscl_q_destroy(hq)
    return out


def _stats(xs):
    xs = sorted(xs)
    return {"median": xs[len(xs) // 2], "min": xs[0], "max": xs[-1], "runs": len(xs)}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="4,8,32")
    ap.add_argument("--ss", default="10,1000")
    ap.add_argument("--episode-sec", type=int, default=3600)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--proc-max-k", type=int, default=8)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=os.path.join(ROOT, "results"))
    a = ap.parse_args(argv)
    import logging
    logging.disable(logging.INFO)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    res = []
    with tempfile.TemporaryDirectory() as tmp:
        for K in [int(x) for x in a.ks.split(",")]:
            dirs = make_dirs(os.path.join(tmp, "K%d" % K), K, a.episode_sec)
            for S in [int(x) for x in a.ss.split(",")]:
                seeds = [10000 + 10000 * i for i in range(S)]
                out = os.path.join(tmp, "out")
                os.makedirs(out, exist_ok=True)
                run_grouped(dirs, seeds, out)            # warm-up: module loads, first launches
                r = {"card": card, "K": K, "S": S, "episode_sec": a.episode_sec,
                     "grouped_s": _stats([run_grouped(dirs, seeds, out) for _ in range(a.repeats)]),
                     "serial_s": _stats([run_serial(dirs, seeds, out) for _ in range(a.repeats)])}
                if K <= a.proc_max_k:
                    r["procs_s"] = _stats([run_procs(dirs, seeds, out) for _ in range(a.repeats)])
                r.update(time_kernels(K, S, a.iters))
                print(json.dumps(r), flush=True)
                res.append(r)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_evaluate_agents.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
