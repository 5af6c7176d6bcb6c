"""GPU: batched IQL training (agents/learner_iql.py, csrc/tsc_q.cu) — the TD / Adam kernels on the TF1-shim golden
minibatches, one round at the bench shapes against the float64 q_td_ref, bit-reproducibility, the sampler and the
ε-greedy forward against their numpy restatements, and a short training run."""
import configparser
import os

import numpy as np
import pytest
import torch

from tests.test_iql_batched_cpu import explore_ref, golden_batches, golden_weights, q_td_ref, sample_ref
from tests.test_learner_reference_golden_cpu import INI

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cfg():
    cp = configparser.ConfigParser(); cp.read_string(INI)
    return cp["MODEL_CONFIG"]


def _learner(n_s, n_a, n_w, kind, R, seed=0, n_obs=None, obs_off=None, **kw):
    from deeprl_signal_control_b200.agents.layout import QLayout
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL
    cfg = _cfg()
    off = np.concatenate([[0], np.cumsum(n_s)]) if obs_off is None else obs_off
    lay = QLayout(kind, n_s, n_a, n_w, off, int(off[len(n_s)]) if n_obs is None else n_obs,
                  n_fc=cfg.getint("num_fc"), n_ft=cfg.getint("num_fc") // 4, n_h=cfg.getint("num_h"))
    return BatchedIQL(lay, R, cfg, kind, seed=seed, device=0, **kw)


@pytest.mark.parametrize("kind", ["lr", "dqn"])
def test_td_and_adam_kernels_on_the_golden_minibatches(kind):
    z = np.load(os.path.join(GOLD, "learner_iql.npz"))
    m = _learner([24, 36], [5, 4], [0, 0], kind, 1)
    for i in range(2):
        for k, v in golden_weights(z, kind, 0, i).items():
            m.nets[i][k].copy_(torch.from_numpy(v))
    idx = torch.arange(40, dtype=torch.int32, device="cuda").reshape(2, 1, 20)
    m.cum_size = 40
    off = [0, 24, 60]
    for k in range(3):
        for i in range(2):
            S, A, S1, Rw, D = golden_batches(z, kind, k, i)
            rows = slice(20 * i, 20 * i + 20)
            m.s[rows, 0, off[i]:off[i + 1]] = torch.tensor(S, dtype=torch.float32)
            m.s1[rows, 0, off[i]:off[i + 1]] = torch.tensor(S1, dtype=torch.float32)
            m.a[rows, 0, i] = torch.tensor(A, dtype=torch.int8)
            m.r[rows, 0, i] = torch.tensor(Rw, dtype=torch.float32)
            m.done[rows, 0] = torch.tensor(D, dtype=torch.uint8)
        m.td_round(k, 1e-4, idx=idx)
        torch.cuda.synchronize()
        for i in range(2):
            pre = "%s/k%d/a%d" % (kind, k, i)
            np.testing.assert_allclose(float(m.losses[k, i]), float(z[pre + "/loss"]), rtol=5e-5)
            np.testing.assert_allclose(float(m.norms[k, i]), float(z[pre + "/grad_norm"]), rtol=5e-5)
            G = m.lay.views(m.grad[:m.lay.n_params])[i]
            for name, g in G.items():
                ref = z["%s/g/%s_%da_q/%s" % (pre, kind, i, name)]
                err = np.abs(g.cpu().numpy() - ref).max()
                assert err <= 5e-4 * np.abs(ref).max(), (pre, name, err)
    for i in range(2):
        for name, ref in golden_weights(z, kind, 3, i).items():
            np.testing.assert_allclose(m.nets[i][name].cpu().numpy(), ref, rtol=0, atol=3e-6, err_msg=name)


def _net(scenario, agent):
    if scenario == "large_grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid
        return build_large_grid(agent=agent)
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    return real_net_tables(agent)


# gradient rel-L2 and loss rel error of one round at the bench shapes against float64, worst agent: about 3x the value
# observed on an H100 (DESIGN.md, K10).  The DQN values are those of the same round in plain fp32 torch, to 3 digits.
ROUND_BOUND = {("large_grid", "dqn"): 2e-5, ("large_grid", "lr"): 8e-7, ("real_net", "dqn"): 9e-5,
               ("real_net", "lr"): 5e-7}


def _rel_l2(G, ref):
    num = sum(((np.asarray(G[k], np.float64) - ref[k]) ** 2).sum() for k in ref)
    return float(np.sqrt(num / sum((ref[k] ** 2).sum() for k in ref)))


def _fp32_grads(w, kind, n_w, S, A, S1, Rw, D, gamma, n_total):
    """the round's weight gradients in float32 torch on the CPU (no kernel involved)"""
    from tests.test_iql_batched_cpu import q_net64
    p = {k: torch.tensor(np.asarray(v, np.float32), requires_grad=True) for k, v in w.items()}
    St, S1t = torch.tensor(np.array(S, np.float32)), torch.tensor(np.array(S1, np.float32))
    q0 = q_net64(p, kind, n_w, St).gather(1, torch.tensor(np.asarray(A, np.int64))[:, None])[:, 0]
    with torch.no_grad():
        Rt = torch.tensor(np.asarray(Rw, np.float32))
        tq = torch.where(torch.tensor(np.asarray(D).astype(bool)), Rt, Rt + gamma * q_net64(p, kind, n_w, S1t).max(1)[0])
    loss = ((q0 - tq) ** 2).sum() / n_total
    return {k: g.numpy() for k, g in zip(p, torch.autograd.grad(loss, list(p.values())))}


@pytest.mark.parametrize("scenario,R,kind", [("large_grid", 4096, "dqn"), ("large_grid", 4096, "lr"),
                                             ("real_net", 2048, "dqn"), ("real_net", 2048, "lr")])
def test_one_round_at_the_bench_shapes_against_float64(scenario, R, kind):
    net = _net(scenario, "iql" + kind[0])
    off = np.asarray(net.node_obs_off)
    n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
    B = 64                                 # a short ring: the kernels see the same strides as with buffer_size
    m = _learner(n_s, list(net.n_a_ls), list(net.n_w_ls), kind, R, n_obs=net.n_obs, obs_off=off)
    m.B = B
    m.s, m.s1 = m.s[:B], m.s1[:B]
    m.a, m.r, m.done = m.a[:B], m.r[:B], m.done[:B]
    g = torch.Generator(device="cuda").manual_seed(1)
    m.s.copy_(torch.rand(m.s.shape, device="cuda", generator=g) * 2)
    m.s1.copy_(torch.rand(m.s1.shape, device="cuda", generator=g) * 2)
    na = torch.tensor(net.n_a_ls, device="cuda")
    m.a.copy_((torch.rand(m.a.shape, device="cuda", generator=g) * na).to(torch.int8))
    m.r.copy_(torch.randn(m.r.shape, device="cuda", generator=g))
    m.done.copy_((torch.rand(m.done.shape, device="cuda", generator=g) < 0.1).to(torch.uint8))
    m.cum_size = B + 7
    P0 = m.P.clone()
    m.td_round(0, 1e-4)
    torch.cuda.synchronize()
    idx = m.idx.cpu().numpy()
    assert np.array_equal(idx, sample_ref(net.n_nodes, R, 20, B, m.seed, 0, 0, 0))
    P1, grad1 = m.P.clone(), m.grad.clone()
    s, s1 = m.s.cpu().numpy(), m.s1.cpu().numpy()
    a, r, d = m.a.cpu().numpy(), m.r.cpu().numpy(), m.done.cpu().numpy()
    w0 = m.lay.views(P0.cpu().numpy())
    G = m.lay.views(grad1[:m.lay.n_params].cpu().numpy())
    rr = np.repeat(np.arange(R), 20)
    errs = []
    for i in range(net.n_nodes):
        sl = idx[i].reshape(-1)
        o = slice(int(off[i]), int(off[i]) + n_s[i])
        batch = (s[sl, rr, o], a[sl, rr, i], s1[sl, rr, o], r[sl, rr, i], d[sl, rr])
        ref = q_td_ref(w0[i], kind, int(m.lay.n_w[i]), *batch, 0.99)
        rel = _rel_l2(G[i], ref["grads"])
        lerr = abs(float(m.losses[0, i]) - ref["loss"]) / ref["loss"]
        errs.append((max(rel, lerr), i, rel, lerr))
    worst, i, rel, lerr = max(errs)
    sl, o = idx[i].reshape(-1), slice(int(off[i]), int(off[i]) + n_s[i])
    batch = (s[sl, rr, o], a[sl, rr, i], s1[sl, rr, o], r[sl, rr, i], d[sl, rr])
    ref = q_td_ref(w0[i], kind, int(m.lay.n_w[i]), *batch, 0.99)
    # the same round in plain fp32 torch (IQL.td_update's arithmetic) on the worst agent: how much of the error is fp32
    # summation over R * batch rows of near-cancelling terms rather than the kernel
    f32 = _rel_l2(_fp32_grads(w0[i], kind, int(m.lay.n_w[i]), *batch, 0.99, R * 20), ref["grads"])
    print("worst rel error %s R=%d %s: %.3g (agent %d: gradient %.3g, loss %.3g; fp32 torch on the same rows %.3g)"
          % (scenario, R, kind, worst, i, rel, lerr, f32))
    assert worst <= ROUND_BOUND[(scenario, kind)], (i, rel, lerr)
    assert rel <= 2 * f32 + 3e-7, (i, rel, f32)            # no worse than fp32 arithmetic itself
    # same seed, same ring: bit-identical weights
    m.P.copy_(P0); m.M.zero_(); m.V.zero_(); m.t = 0
    m.td_round(0, 1e-4)
    assert torch.equal(m.P, P1) and torch.equal(m.grad, grad1)


@pytest.mark.parametrize("kind", ["lr", "dqn"])
def test_explore_forward_against_the_restated_draws(kind):
    from deeprl_signal_control_b200 import _lib
    import ctypes as C
    net = _net("large_grid", "iql" + kind[0])
    off = np.asarray(net.node_obs_off)
    n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
    R = 1024
    m = _learner(n_s, list(net.n_a_ls), list(net.n_w_ls), kind, R, seed=3, n_obs=net.n_obs, obs_off=off)
    obs = torch.rand(R, net.n_obs, device="cuda") * 2
    q0 = torch.zeros_like(m.q); act0 = torch.zeros_like(m.act)
    _lib.check(_lib.lib().tscl_q_step(m._h, C.c_void_p(m.P.data_ptr()), C.c_void_p(obs.data_ptr()), C.c_int64(R),
                                      C.c_void_p(q0.data_ptr()), C.c_void_p(act0.data_ptr()), C.c_int32(0),
                                      C.c_uint64(0), C.c_int64(0), C.c_int64(0), None, m._st()))
    m.explore(obs, 0.0, 5)
    torch.cuda.synchronize()
    assert torch.equal(m.q, q0) and torch.equal(m.act, act0)
    assert torch.equal(m.s[0], obs) and torch.equal(m.a[0].to(torch.int32), act0)
    for eps in (1.0, 0.3):
        m.explore(obs, eps, 17)
        torch.cuda.synchronize()
        ref = explore_ref(m.q.cpu().numpy(), list(net.n_a_ls), eps, 3, 17, 0)
        assert np.array_equal(m.act.cpu().numpy(), ref)


def test_sampler_after_wrap_matches_the_restatement():
    m = _learner([24, 36], [5, 4], [0, 0], "lr", 300, seed=4000000007, replica0=77, total_replicas=1000)
    m.cum_size = 1234                      # wrapped: size = buffer_size
    m.n_updates = 3
    idx = m.sample(4)
    torch.cuda.synchronize()
    assert np.array_equal(idx.cpu().numpy(), sample_ref(2, 300, 20, 1000, 4000000007, 3, 4, 77))


def test_short_training_run_on_the_grid():
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQLTrainer
    from deeprl_signal_control_b200.agents.utils import Scheduler
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    net = _net("large_grid", "iqld")
    par = EnvParams(agent="iqld", episode_length_sec=200)
    off = np.asarray(net.node_obs_off)
    n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
    m = _learner(n_s, list(net.n_a_ls), list(net.n_w_ls), "dqn", 64, n_obs=net.n_obs, obs_off=off)
    sim = BatchedSim(net, par, 64, device=0)
    tr = BatchedIQLTrainer(sim, m, Scheduler(1e-4, decay="constant"), Scheduler(1.0, 0.01, 100, decay="linear"))
    P0 = m.P.clone()
    tr.run(80)                             # two 40-step episodes
    torch.cuda.synchronize()
    assert tr.n_updates == 4 and len(tr.episode_rewards) == 2
    assert bool(torch.isfinite(m.losses).all()) and float(m.norms.min()) > 0
    assert not torch.equal(P0, m.P) and bool(torch.isfinite(m.P).all())
    assert m.cum_size == 80
    # the ring's s1 of a step is the next step's s, except across the episode end
    assert torch.equal(m.s[1:40], m.s1[0:39]) and not torch.equal(m.s[40], m.s1[39])


def test_replica_ranges_split_the_draws_and_the_gradient():
    """two learners on [0, R/2) and [R/2, R) with total_replicas = R: the same draws as one learner on R, and their
    gradients (and loss sums) add up to its gradient: the data-parallel split of a multi-rank run"""
    net = _net("large_grid", "iqld")
    off = np.asarray(net.node_obs_off)
    n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
    R, h = 256, 128
    mk = lambda n, r0: _learner(n_s, list(net.n_a_ls), list(net.n_w_ls), "dqn", n, seed=9, n_obs=net.n_obs,
                                obs_off=off, replica0=r0, total_replicas=R)
    full, lo, hi = mk(R, 0), mk(h, 0), mk(h, h)
    g = torch.Generator(device="cuda").manual_seed(2)
    full.s.copy_(torch.rand(full.s.shape, device="cuda", generator=g))
    full.s1.copy_(torch.rand(full.s1.shape, device="cuda", generator=g))
    full.a.copy_((torch.rand(full.a.shape, device="cuda", generator=g) * 5).to(torch.int8))
    full.r.copy_(torch.randn(full.r.shape, device="cuda", generator=g))
    full.done.copy_((torch.rand(full.done.shape, device="cuda", generator=g) < 0.1).to(torch.uint8))
    for part, sl in ((lo, slice(0, h)), (hi, slice(h, R))):
        for name in ("s", "s1", "a", "r", "done"):
            getattr(part, name).copy_(getattr(full, name)[:, sl])
    for m in (full, lo, hi):
        m.cum_size = 1500
        m.td_round(3, 1e-4)
    torch.cuda.synchronize()
    assert torch.equal(torch.cat([lo.idx, hi.idx], 1), full.idx)
    summed = (lo.grad.double() + hi.grad.double())
    rel = float((summed - full.grad.double()).norm() / full.grad.double().norm())
    print("replica-range gradient sum rel-L2 %.3g" % rel)
    assert rel <= 1e-6


def test_protocol_at_one_replica_matches_the_one_replica_iql():
    """BatchedIQLTrainer at R = 1 with every transition mirrored into the one-replica IQL (agents/models.py): the ring
    holds what IQL.add_transition stores, the actions are the restated ε-greedy draws, every round's loss and norm equal
    IQL.td_update's on the read-back indices, and the weights stay together"""
    import configparser
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQLTrainer
    from deeprl_signal_control_b200.agents.models import IQL
    from deeprl_signal_control_b200.agents.utils import Scheduler
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    cp = configparser.ConfigParser(); cp.read_string(INI.replace("reward_norm = 3.0", "reward_norm = 30.0"))
    cfg = cp["MODEL_CONFIG"]
    net = _net("large_grid", "iqld")
    off = np.asarray(net.node_obs_off)
    n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
    from deeprl_signal_control_b200.agents.layout import QLayout
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL
    lay = QLayout("dqn", n_s, net.n_a_ls, net.n_w_ls, off, net.n_obs, n_fc=128, n_ft=32, n_h=64, max_na=net.max_na)
    m = BatchedIQL(lay, 1, cfg, "dqn", seed=5, device=0)
    ref = IQL(n_s, list(net.n_a_ls), list(net.n_w_ls), 1000, cfg, seed=5, model_type="dqn", device="cpu")
    assert all(torch.equal(m.nets[i][k].cpu(), v.detach()) for i, p in enumerate(ref.nets) for k, v in p.items())
    sim = BatchedSim(net, EnvParams(agent="iqld", episode_length_sec=150), 1, device=0)     # 30-step episodes
    tr = BatchedIQLTrainer(sim, m, ref.lr_scheduler, ref.eps_scheduler, seed0=12)
    eps_ref = Scheduler(1.0, 0.01, 1000 * 0.5, decay="linear")
    rounds = []
    orig = m.td_round

    def record(rnd, lr, idx=None):
        orig(rnd, lr, idx)
        rounds.append((m.idx.cpu().numpy().copy(), lr, m.losses[rnd].cpu().numpy().copy(),
                       m.norms[rnd].cpu().numpy().copy()))
    m.td_round = record
    rewards = []
    orig_add = m.add_transition

    def keep_reward(reward, *args):
        rewards.append(reward[0].cpu().numpy().copy())
        orig_add(reward, *args)
    m.add_transition = keep_reward
    worst_loss = worst_norm = 0.0
    n_clipped = 0
    for step in range(60):
        eps = eps_ref.get(1)
        rounds.clear()
        tr.control_step()
        k = (m.cum_size - 1) % m.B
        s, s1 = m.s[k, 0].cpu().numpy(), m.s1[k, 0].cpu().numpy()
        act = m.a[k, 0].cpu().numpy().astype(np.int64)
        assert np.array_equal(act, explore_ref(m.q.cpu().numpy(), list(net.n_a_ls), eps, 5, step, 0)[0])
        done = (step + 1) % 30 == 0
        ref.add_transition([s[o:o + w] for o, w in zip(off, n_s)], list(act), rewards[-1],
                           [s1[o:o + w] for o, w in zip(off, n_s)], done)
        for i in range(net.n_nodes):
            ob, a_i, r_i, nob, d = ref.trans_buffer_ls[i]._slots[k]
            assert np.float32(r_i) == m.r[k, 0, i].cpu().numpy(), (step, i)
            n_clipped += abs(r_i) == 2.0
        assert bool(m.done[k, 0]) == done
        if step > 0 and step % 30 != 0:                  # s1 of the previous step is this step's s, except at a reset
            assert np.array_equal(m.s1[k - 1, 0].cpu().numpy(), s)
        elif step == 30:
            assert not np.array_equal(m.s1[k - 1, 0].cpu().numpy(), s)
        for idx, lr, loss, norm in rounds:
            for i in range(net.n_nodes):
                b = ref.trans_buffer_ls[i]
                pick = [b._slots[j] for j in idx[i, 0]]
                f = lambda c: np.asarray([x[c] for x in pick])
                l_ref, n_ref = ref.td_update(i, f(0), f(1), f(3), f(4), f(2), lr)
                worst_loss = max(worst_loss, abs(loss[i] - l_ref) / abs(l_ref))
                worst_norm = max(worst_norm, abs(norm[i] - n_ref) / abs(n_ref))
    assert tr.n_updates == 4 and len(tr.episode_rewards) == 2
    assert 0 < n_clipped < 60 * net.n_nodes           # both normalised-only and clipped rewards occurred
    wdiff = max(float((m.nets[i][k].cpu() - v.detach()).abs().max()) for i, p in enumerate(ref.nets) for k, v in p.items())
    print("R=1 protocol: worst loss rel %.3g, norm rel %.3g, final weight max |diff| %.3g" % (worst_loss, worst_norm, wdiff))
    assert worst_loss <= PROTOCOL_BOUND["loss"] and worst_norm <= PROTOCOL_BOUND["norm"]
    assert wdiff <= PROTOCOL_BOUND["weights"]


# fp32 device kernels against IQL.td_update's fp32 torch ops over 4 backwards (40 Adam steps per agent): about 4x the
# values observed on an H100 (DESIGN.md, K10)
PROTOCOL_BOUND = {"loss": 1e-6, "norm": 1e-6, "weights": 1e-6}


def test_checkpoints_and_evaluator_interop(tmp_path):
    """BatchedIQL.save is read by IQL.load and by BatchedIQL.load (weights and Adam state), and the batched evaluator
    gives the same results on the BatchedIQL as on the IQL loaded from its checkpoint"""
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    from deeprl_signal_control_b200.agents.models import IQL
    from tests.test_evaluator_gpu import _env
    net = _net("large_grid", "iqld")
    off = np.asarray(net.node_obs_off)
    n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
    m = _learner(n_s, list(net.n_a_ls), list(net.n_w_ls), "dqn", 4, seed=3, n_obs=net.n_obs, obs_off=off)
    g = torch.Generator(device="cuda").manual_seed(4)
    m.P.add_(torch.randn(m.P.shape, device="cuda", generator=g) * 0.05)
    m.M.copy_(torch.randn(m.M.shape, device="cuda", generator=g))
    m.V.copy_(torch.rand(m.V.shape, device="cuda", generator=g))
    m.t = 7
    d = str(tmp_path / "ck")
    os.makedirs(d)
    m.save(d, 11)
    ref = IQL(n_s, list(net.n_a_ls), list(net.n_w_ls), 0, _cfg(), seed=99, model_type="dqn", device="cuda")
    assert ref.load(d)
    for i, p in enumerate(ref.nets):
        for k, v in p.items():
            assert torch.equal(v.detach(), m.nets[i][k]), (i, k)
    m2 = _learner(n_s, list(net.n_a_ls), list(net.n_w_ls), "dqn", 4, seed=1, n_obs=net.n_obs, obs_off=off)
    assert m2.load(d)
    assert torch.equal(m2.P, m.P) and torch.equal(m2.M, m.M) and torch.equal(m2.V, m.V) and m2.t == 7
    out = str(tmp_path) + os.sep
    mean_b, std_b = Evaluator(_env("large_grid", "iqld", [7, 8], 300, out, 2, record=False), m, out).run()
    mean_r, std_r = Evaluator(_env("large_grid", "iqld", [7, 8], 300, out, 2, record=False), ref, out).run()
    np.testing.assert_array_equal(mean_b, mean_r)
    np.testing.assert_array_equal(std_b, std_r)
