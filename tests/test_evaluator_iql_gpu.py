"""GPU: batched test-mode evaluation of IQL agents — the fp32 Q forward (tscl_q_step) against a float64 forward at the
evaluation shapes, its normalised-q sampling against a numpy restatement, end-to-end parity of the evaluator with the
reference's one-seed-at-a-time protocol (utils.py:Tester.perform with IQL.forward), isolation from a live IQL, and
scripts/evaluate.py on IQL checkpoints."""
import configparser
import ctypes as C
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.test_evaluator_gpu import GRID_INI, _env, _read, _reference_actions
from tests.test_evaluator_iql_cpu import INI, q_forward_ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# max |q - q_float64| / row scale over all (replica, agent) rows of a launch, ~3x the largest value observed on an H100
# (DESIGN.md §5); the row scale is max_j (|b_j| + sum_k |x_k W_kj|) of the output layer (q_forward_ref)
Q_BOUND = {"lr": 8e-7, "dqn": 1.2e-6}


def _net(scenario, agent):
    if scenario == "large_grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid
        return build_large_grid(agent=agent)
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    return real_net_tables(agent)


def _iql(net, kind, seed=0, total_step=0):
    from deeprl_signal_control_b200.agents.models import IQL
    cp = configparser.ConfigParser(); cp.read_string(INI)
    m = IQL(net.n_s_ls, net.n_a_ls, net.n_w_ls, total_step, cp["MODEL_CONFIG"], seed=seed, model_type=kind, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(seed + 11)
    for p in m.nets:
        for k, v in p.items():
            if k.endswith("/b"):       # biases N(0, 0.1): no two actions tie exactly
                v.data.copy_(torch.randn(v.shape, device="cuda", generator=g) * 0.1)
    return m


class _Q:
    """tscl_q handle over an IQL's packed weights, observation rows of stride n_obs"""

    def __init__(self, m, net, n_obs):
        from deeprl_signal_control_b200 import _lib
        from deeprl_signal_control_b200.agents.layout import QLayout
        self.lib, self.check = _lib.lib(), _lib.check
        self.lay = QLayout.from_iql(m, net.node_obs_off, n_obs, max_na=net.max_na)
        self.h = C.c_void_p()
        self.check(self.lib.tscl_q_create(C.byref(self.lay.as_c()), C.c_int32(0), C.byref(self.h)))
        self.P = self.lay.pack(m.nets).cuda()

    def step(self, obs, q, act, mode, seed, step, r0=0, n=None, bad=None):
        L = self.lay
        n = obs.shape[0] - r0 if n is None else n
        off = lambda t, per_row: C.c_void_p(t.data_ptr() + r0 * per_row * t.element_size())
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.check(self.lib.tscl_q_step(self.h, C.c_void_p(self.P.data_ptr()), off(obs, L.n_obs), C.c_int64(n),
                                        off(q, L.A * L.max_na), off(act, L.A), C.c_int32(mode), C.c_uint64(seed),
                                        C.c_int64(step), C.c_int64(r0), None if bad is None else C.c_void_p(bad.data_ptr()),
                                        st))

    def close(self):
        self.lib.tscl_q_destroy(self.h)


def _q64(m, lay, obs):
    """float64 q [R][A][max_na] (zero padded) of the observation rows and the row scales [R][A]"""
    o = np.asarray(obs, np.float64)
    R = o.shape[0]
    out, scale = np.zeros((R, lay.A, lay.max_na)), np.zeros((R, lay.A))
    for i in range(lay.A):
        w = {k: v.detach().cpu().numpy() for k, v in m.nets[i].items()}
        s = o[:, int(lay.obs_off[i]):int(lay.obs_off[i]) + int(lay.n_s[i])]
        out[:, i, :int(lay.n_a[i])], scale[:, i] = q_forward_ref(
            m.model_type, w, s, int(m.n_w_ls[i]) if m.model_type == "dqn" else 0, with_scale=True)
    return out, scale


def _rel_err(q, q64, scale, n_a):
    return max(float((np.abs(q[:, i, :na] - q64[:, i, :na]).max(1) / scale[:, i]).max()) for i, na in enumerate(n_a))


def _sample_ref(q, n_a, seed, step, replica0):
    """qs / np.sum(qs) in fp32 (sum in index order), then the kernel's inverse CDF at the counter-hash uniform"""
    R, A, mna = q.shape
    p = np.zeros_like(q, dtype=np.float32)
    for a in range(A):
        s = np.zeros(R, np.float32)
        for j in range(int(n_a[a])):
            s = s + q[:, a, j]
        p[:, a, :int(n_a[a])] = q[:, a, :int(n_a[a])] / s[:, None]
    return _reference_actions(p, n_a, seed, step, replica0)


@pytest.mark.parametrize("scenario,R", [("large_grid", 4096), ("real_net", 2048)])
@pytest.mark.parametrize("kind", ["lr", "dqn"])
def test_q_kernel_matches_float64_forward(scenario, R, kind):
    agent = "iqll" if kind == "lr" else "iqld"
    net = _net(scenario, agent)
    m = _iql(net, kind, seed=3)
    pad = 5                                             # observation columns that belong to no agent: NaN
    qk = _Q(m, net, net.n_obs + pad)
    g = torch.Generator(device="cuda").manual_seed(1)
    q = torch.empty(R, net.n_nodes, net.max_na, device="cuda")
    act = torch.empty(R, net.n_nodes, dtype=torch.int32, device="cuda")
    worst = 0.0
    for step in range(3):
        obs = torch.rand(R, net.n_obs + pad, device="cuda", generator=g) * 2
        obs[:, net.n_obs:] = float("nan")
        q.fill_(float("nan")); act.fill_(-1)
        qk.step(obs, q, act, 0, 7, step)
        torch.cuda.synchronize()
        qn, an = q.cpu().numpy(), act.cpu().numpy()
        assert np.isfinite(qn).all()
        for i, na in enumerate(net.n_a_ls):
            assert (qn[:, i, na:] == 0).all()
        q64, scale = _q64(m, qk.lay, obs.cpu().numpy())
        err = _rel_err(qn, q64, scale, net.n_a_ls)
        worst = max(worst, err)
        print("Q kernel %s %s step %d: max error / row scale %.3g" % (scenario, kind, step, err))
        assert err <= Q_BOUND[kind], err
        # actions: the float64 argmax wherever the top-2 gap is wider than twice the bound
        n_cmp = 0
        for i, na in enumerate(net.n_a_ls):
            ref = q64[:, i, :na]
            srt = np.sort(ref, 1)
            clear = (srt[:, -1] - srt[:, -2]) > 2 * Q_BOUND[kind] * scale[:, i]
            np.testing.assert_array_equal(an[clear, i], np.argmax(ref, 1)[clear])
            np.testing.assert_array_equal(an[:, i], np.argmax(qn[:, i, :na], 1))     # np.argmax of the q it wrote
            n_cmp += int(clear.sum())
        assert n_cmp > 0.999 * R * net.n_nodes
        # uneven replica ranges reproduce one full launch bit for bit, in both action modes
        for mode in (0, 1):
            qa, aa = torch.empty_like(q), torch.empty_like(act)
            bad_a = torch.full((1,), -1, dtype=torch.int64, device="cuda")
            qk.step(obs, qa, aa, mode, 7, step, bad=bad_a)
            qr, ar = torch.full_like(q, float("nan")), torch.full_like(act, -1)
            bad_r = torch.full((1,), -1, dtype=torch.int64, device="cuda")
            bounds = [0, R // 4 - 24, R // 2 + 52, 3 * R // 4 + 7, R]
            for r0, r1 in zip(bounds[:-1], bounds[1:]):
                qk.step(obs, qr, ar, mode, 7, step, r0=r0, n=r1 - r0, bad=bad_r)
            torch.cuda.synchronize()
            assert torch.equal(qr, qa) and torch.equal(ar, aa) and torch.equal(bad_r, bad_a)
            assert torch.equal(qa, q)
    qk.close()
    print("Q kernel %s %s R=%d: max error / row scale %.3g (bound %.1g)" % (scenario, kind, R, worst, Q_BOUND[kind]))


@pytest.mark.parametrize("kind", ["lr", "dqn"])
def test_q_sampling_matches_numpy_restatement(kind):
    net = _net("large_grid", "iqll" if kind == "lr" else "iqld")
    R, A = 4096, net.n_nodes
    seed = (5 << 32) | 77
    for sign in (1.0, -1.0):
        m = _iql(net, kind, seed=4)
        for p in m.nets:                                 # every q of one sign
            p["q/b"].data.add_(sign * 100.0)
        qk = _Q(m, net, net.n_obs)
        g = torch.Generator(device="cuda").manual_seed(2)
        obs = torch.rand(R, net.n_obs, device="cuda", generator=g) * 2
        q = torch.empty(R, A, net.max_na, device="cuda")
        act = torch.empty(R, A, dtype=torch.int32, device="cuda")
        bad = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        for step in (0, 9):
            qk.step(obs, q, act, 1, seed, step, bad=bad)
            torch.cuda.synchronize()
            qn = q.cpu().numpy()
            assert ((qn > 0) if sign > 0 else (qn < 0))[:, 0, :5].all()
            np.testing.assert_array_equal(act.cpu().numpy(), _sample_ref(qn, net.n_a_ls, seed, step, 0))
            assert int(bad.item()) == -1
            a_np = act.cpu().numpy()
            assert len(np.unique(a_np[:, 0])) == int(net.n_a_ls[0])         # a sample, not an argmax
        # a planted mixed-sign row: flag with (replica, step, agent), action 0; the other rows unchanged
        obs2 = obs.clone()
        r_bad, a_bad = 1234, 7
        o0 = int(net.node_obs_off[a_bad]); n_s = int(net.n_s_ls[a_bad])
        rng = np.random.default_rng(0)
        for _ in range(100):                             # a large observation row whose q has both signs
            obs2[r_bad, o0:o0 + n_s] = torch.from_numpy(rng.normal(0.0, 300.0, n_s).astype(np.float32)).cuda()
            q64 = _q64(m, qk.lay, obs2[r_bad:r_bad + 1].cpu().numpy())[0][0, a_bad, :int(net.n_a_ls[a_bad])]
            if (q64 > 0).any() and (q64 < 0).any():
                break
        assert (q64 > 0).any() and (q64 < 0).any()
        act2 = torch.empty_like(act)
        qk.step(obs, q, act, 1, seed, 3)
        qk.step(obs2, q, act2, 1, seed, 3, bad=bad)
        torch.cuda.synchronize()
        key = int(bad.item())
        assert (key >> 40, (key >> 16) & 0xFFFFFF, key & 0xFFFF) == (r_bad, 3, a_bad)
        a1, a2 = act.cpu().numpy(), act2.cpu().numpy()
        assert a2[r_bad, a_bad] == 0
        a2[r_bad, a_bad] = a1[r_bad, a_bad]
        np.testing.assert_array_equal(a1, a2)
        qk.close()


def _reference_iql_run(env, model):
    """reference utils.py:Evaluator.run / Tester.perform for a value-based agent (policy_type 'default' -> argmax of q)
    on the one-replica env, with the float64 top-2 margin / row scale of every decision"""
    env.train_mode = False
    env.cur_episode = 0
    env.init_data(True, False, env.output_path)
    means, stds, margins = [], [], []
    w = [{k: v.detach().cpu().numpy() for k, v in p.items()} for p in model.nets]
    for k in range(env.test_num):
        ob = env.reset(test_ind=k)
        model.reset()
        rewards = []
        while True:
            action, _ = model.forward(ob)
            for i, o in enumerate(ob):
                q64, scale = q_forward_ref(model.model_type, w[i], np.asarray(o, np.float32)[None],
                                           int(model.n_w_ls[i]) if model.model_type == "dqn" else 0, with_scale=True)
                top = np.sort(q64[0])[::-1]
                margins.append((top[0] - top[1]) / scale[0])
            next_ob, reward, done, global_reward = env.step(action)
            rewards.append(global_reward)
            if done:
                break
            ob = next_ob
        means.append(np.mean(np.array(rewards))); stds.append(np.std(np.array(rewards)))
        env.collect_tripinfo()
    env.output_data()
    return np.array(means), np.array(stds), np.array(margins)


@pytest.mark.parametrize("scenario,agent", [("large_grid", "iqll"), ("large_grid", "iqld"), ("real_net", "iqll"),
                                            ("real_net", "iqld")])
def test_evaluator_matches_reference_protocol_for_iql(scenario, agent, tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    kind = "dqn" if agent == "iqld" else "lr"
    seeds, sec = [10000, 20000, 30000, 40000], 600
    d1, d2 = str(tmp_path / "one") + os.sep, str(tmp_path / "batched") + os.sep
    os.makedirs(d1); os.makedirs(d2)
    env1 = _env(scenario, agent, seeds, sec, d1, 1)
    envb = _env(scenario, agent, seeds, sec, d2, len(seeds))
    model = _iql(_net(scenario, agent), kind, seed=6)
    mean1, std1, margins = _reference_iql_run(env1, model)
    assert margins.min() >= 10 * Q_BOUND[kind], margins.min()      # equality below is expected, not lucky
    ev = Evaluator(envb, model, d2, policy_type="default")
    assert ev.family == "q"
    meanb, stdb = ev.run()
    np.testing.assert_array_equal(meanb, mean1)
    np.testing.assert_array_equal(stdb, std1)
    base = "%s_%s_" % (env1.name, agent)
    for k in ("control", "traffic"):
        assert open(d1 + base + k + ".csv").read() == open(d2 + base + k + ".csv").read(), k
    if open(d1 + base + "trip.csv").read() != open(d2 + base + "trip.csv").read():
        key = ["episode", "arrival_sec", "depart_sec", "id"]
        t1 = _read(d1 + base + "trip.csv").sort_values(key).reset_index(drop=True)
        tb = _read(d2 + base + "trip.csv").sort_values(key).reset_index(drop=True)
        assert t1.equals(tb)
    print("IQL e2e %s %s: %d decisions, smallest float64 top-2 margin / row scale %.3g" %
          (scenario, agent, len(margins), margins.min()))


def _state(m):
    """everything of an IQL that training reads: weights, Adam moments and step, replay buffers, exploration RNG"""
    t = lambda d: {k: v.detach().cpu().numpy() for k, v in d.items()}
    return pickle.dumps(([t(p) for p in m.nets], [(s["t"], t(s["m"]), t(s["v"])) for s in m.adam],
                         [b.__dict__ for b in m.trans_buffer_ls], m._np_rng.get_state()))


def test_evaluating_a_live_iql_leaves_it_unchanged(tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    net = _net("large_grid", "iqld")
    m = _iql(net, "dqn", seed=8, total_step=10000)
    rng = np.random.default_rng(0)
    for t in range(45):                                  # fill the replay buffers past one minibatch, two updates
        obs = [rng.random(n).astype(np.float32) for n in net.n_s_ls]
        act, _ = m.forward(obs, mode="explore")
        m.add_transition(obs, act, rng.normal(size=len(obs)), obs, t % 20 == 19)
        if t % 20 == 19:
            m.backward(None, t)
    assert m.adam[0]["t"] > 0 and m.trans_buffer_ls[0].size == 45
    before = _state(m)
    nets = [{k: v.detach().clone() for k, v in p.items()} for p in m.nets]
    env = _env("large_grid", "iqld", [7, 8, 9], 300, str(tmp_path) + os.sep, 3)
    for pt in ("default", "stochastic"):
        if pt == "stochastic":                           # needs q > 0 everywhere; restored exactly below
            for p in m.nets:
                p["q/b"].data.add_(100.0)
        mean, std = Evaluator(env, m, str(tmp_path) + os.sep, policy_type=pt).run()
        for p, p0 in zip(m.nets, nets):
            p["q/b"].data.copy_(p0["q/b"])
        assert np.isfinite(mean).all() and (std > 0).all()
    torch.cuda.synchronize()
    for p, p0 in zip(m.nets, nets):
        for k in p:
            assert torch.equal(p[k], p0[k]) and p[k].requires_grad, k
    assert _state(m) == before


def _agent_dir(tmp_path, agent, model, seeds):
    d = tmp_path / agent
    (d / "data").mkdir(parents=True); (d / "model").mkdir()
    (d / "data" / ("config_%s_large.ini" % agent)).write_text(GRID_INI % (agent, 600, ",".join(map(str, seeds))) + INI)
    model.save(str(d / "model"), 1000)
    return d


def _run_script(d, out, policy_type):
    return subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", str(d),
                           "--evaluation-policy-type", policy_type, "--output-dir", str(out)],
                          capture_output=True, text=True, cwd=ROOT)


@pytest.mark.parametrize("agent", ["iqll", "iqld"])
def test_evaluate_script_runs_iql_checkpoints(agent, tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    kind = "dqn" if agent == "iqld" else "lr"
    m = _iql(_net("large_grid", agent), kind, seed=9)
    seeds = [11, 12, 13]
    d = _agent_dir(tmp_path, agent, m, seeds)
    out = tmp_path / "eva"
    r = _run_script(d, out, "default")
    assert r.returncode == 0, r.stdout + r.stderr
    got = json.load(open(out / ("%s_summary.json" % agent)))
    env = _env("large_grid", agent, seeds, 600, str(tmp_path) + os.sep, len(seeds))
    ev = Evaluator(env, m, str(tmp_path) + os.sep, policy_type="default")
    mean, std = ev.run()
    assert got == json.loads(json.dumps(ev.summary(mean, std, *ev.recorded[1:])))
    for k in ("control", "traffic", "trip"):
        assert (out / ("large_grid_%s_%s.csv" % (agent, k))).exists()
    # stochastic evaluation of a model whose q has mixed signs: the reference's np.random.choice error
    for p in m.nets:
        p["q/b"].data.copy_(torch.linspace(-5.0, 5.0, p["q/b"].numel(), device="cuda"))
        p["q/w"].data.zero_()
    d2 = _agent_dir(tmp_path / "mixed", agent, m, seeds)
    r = _run_script(d2, tmp_path / "eva2", "stochastic")
    assert r.returncode != 0 and "ValueError: probabilities are not non-negative" in r.stderr, r.stderr[-2000:]
