"""CPU: the float64 restatement of one batched IQL round (q_td_ref) against the TF1-shim goldens and autograd, planted
defects, numpy restatements of the device's minibatch sampler and ε-greedy draws, and BatchedIQL's initial weights."""
import configparser
import os

import numpy as np
import pytest
import torch

from tests.test_learner_reference_golden_cpu import INI

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
M32 = 0xFFFFFFFF


# ---- float64 reference of one round -------------------------------------------------------------------------------
def q_net64(w, kind, n_w, S):
    """q of DeepQPolicy / LRQPolicy in float64 torch (w: {name: tensor})"""
    if kind != "dqn":
        return S @ w["q/w"] + w["q/b"]
    n_wave = S.shape[1] - n_w
    h = torch.relu(S[:, :n_wave] @ w["q_fcw/w"] + w["q_fcw/b"])
    if n_w > 0:
        h = torch.cat([h, torch.relu(S[:, n_wave:] @ w["q_fct/w"] + w["q_fct/b"])], 1)
    h = torch.relu(h @ w["q_fc_0/w"] + w["q_fc_0/b"])
    return h @ w["q/w"] + w["q/b"]


def q_td_ref(w, kind, n_w, S, A, S1, Rw, D, gamma, n_total=None, max_norm=40.0, adam=None, lr=None,
             mutate=None):
    """One round of IQL.td_update for one agent in float64: loss = sum over the rows of (q(s)[a] - tq)^2 / n_total
    (n_total = rows of all replicas; default the rows given), tq = done ? r : r + gamma max q(s1) without gradient.
    Returns (q, err = the TD errors, loss, grads, norm) and, with adam = {'t', 'm', 'v'} and lr, the new weights (TF1 Adam after the global
    norm clip).  `mutate` plants a defect: 'no_done', 'grad_tq', 's_for_s1'."""
    w = {k: torch.as_tensor(np.asarray(v, np.float64)).clone().requires_grad_(True) for k, v in w.items()}
    S = torch.tensor(np.array(S, np.float64)); S1 = torch.tensor(np.array(S1, np.float64))
    A = torch.as_tensor(np.asarray(A, np.int64)); Rw = torch.as_tensor(np.asarray(Rw, np.float64))
    D = torch.as_tensor(np.asarray(D).astype(bool))
    n_total = S.shape[0] if n_total is None else n_total
    q = q_net64(w, kind, n_w, S)
    q1 = q_net64(w, kind, n_w, S if mutate == "s_for_s1" else S1).max(1)[0]
    if mutate != "grad_tq":
        q1 = q1.detach()
    tq = Rw + gamma * q1 if mutate == "no_done" else torch.where(D, Rw, Rw + gamma * q1)
    err = q.gather(1, A[:, None])[:, 0] - tq
    loss = (err ** 2).sum() / n_total
    keys = list(w)
    g = dict(zip(keys, torch.autograd.grad(loss, [w[k] for k in keys])))
    norm = float(torch.sqrt(sum((x * x).sum() for x in g.values())))
    out = dict(q=q.detach().numpy(), err=err.detach().numpy(), loss=float(loss.detach()), grads={k: v.numpy() for k, v in g.items()}, norm=norm)
    if adam is not None:
        new_w, new_adam = adam_ref({k: v.detach().numpy() for k, v in w.items()}, out["grads"], norm, adam, lr, max_norm)
        out.update(w=new_w, adam=new_adam)
    return out


def adam_ref(w, grads, norm, adam, lr, max_norm):
    """tf.clip_by_global_norm of grads (global norm `norm`) and one TF1 Adam step from adam = {'t', 'm', 'v'}, float64:
    (new weights, new adam state)"""
    scale = max_norm / max(norm, max_norm) if max_norm > 0 else 1.0
    t = adam["t"] + 1
    lr_t = lr * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
    new_w, m, v = {}, {}, {}
    for k in w:
        gk = np.asarray(grads[k], np.float64) * scale
        m[k] = adam["m"][k] + (gk - adam["m"][k]) * 0.1
        v[k] = adam["v"][k] + (gk * gk - adam["v"][k]) * 0.001
        new_w[k] = np.asarray(w[k], np.float64) - lr_t * m[k] / (np.sqrt(v[k]) + 1e-8)
    return new_w, dict(t=t, m=m, v=v)


def golden_batches(z, kind, k, i):
    pre = "%s/k%d/a%d" % (kind, k, i)
    return (z[pre + "/obs"], z[pre + "/acts"], z[pre + "/next_obs"], z[pre + "/rs"], z[pre + "/dones"])


def golden_weights(z, kind, step, i):
    pre = "%s/w%d/%s_%da_q/" % (kind, step, kind, i)
    return {k[len(pre):]: z[k] for k in z.files if k.startswith(pre)}


@pytest.mark.parametrize("kind", ["lr", "dqn"])
def test_q_td_ref_reproduces_the_golden_rounds(kind):
    z = np.load(os.path.join(GOLD, "learner_iql.npz"))
    w = [golden_weights(z, kind, 0, i) for i in range(2)]
    adam = [dict(t=0, m={k: 0 * v.astype(np.float64) for k, v in w[i].items()},
                 v={k: 0 * v.astype(np.float64) for k, v in w[i].items()}) for i in range(2)]
    for k in range(3):
        for i in range(2):
            S, A, S1, Rw, D = golden_batches(z, kind, k, i)
            pre = "%s/k%d/a%d" % (kind, k, i)
            out = q_td_ref(w[i], kind, 0, S, A, S1, Rw, D, 0.99, adam=adam[i], lr=1e-4)
            np.testing.assert_allclose(out["q"], z[pre + "/q"], rtol=1e-7, atol=1e-7)
            np.testing.assert_allclose(out["loss"], float(z[pre + "/loss"]), rtol=1e-7)
            np.testing.assert_allclose(out["norm"], float(z[pre + "/grad_norm"]), rtol=1e-7)
            gpre = "%s/g/%s_%da_q/" % (pre, kind, i)
            for name, g in out["grads"].items():
                ref = z[gpre + name]
                assert np.abs(g - ref).max() <= 1e-7 * max(1.0, np.abs(ref).max()), name
            w[i], adam[i] = out["w"], out["adam"]
        for i in range(2):
            for name, ref in golden_weights(z, kind, k + 1, i).items():
                np.testing.assert_allclose(w[i][name], ref, rtol=0, atol=1e-6, err_msg=name)


def _ragged_weights(rng, n_s, n_w, n_a, n_fc=32, n_h=16):
    w = {"q_fcw/w": rng.standard_normal((n_s - n_w, n_fc)) * 0.3, "q_fcw/b": rng.standard_normal(n_fc) * 0.1,
         "q_fc_0/w": rng.standard_normal((n_fc + (n_fc // 4 if n_w else 0), n_h)) * 0.3,
         "q_fc_0/b": rng.standard_normal(n_h) * 0.1, "q/w": rng.standard_normal((n_h, n_a)) * 0.3,
         "q/b": rng.standard_normal(n_a) * 0.1}
    if n_w:
        w.update({"q_fct/w": rng.standard_normal((n_w, n_fc // 4)) * 0.3, "q_fct/b": rng.standard_normal(n_fc // 4) * 0.1})
    return w


def _batch(rng, n, n_s, n_a):
    return (rng.standard_normal((n, n_s)), rng.integers(0, n_a, n), rng.standard_normal((n, n_s)),
            rng.standard_normal(n), rng.random(n) < 0.3)


def test_q_td_ref_matches_autograd_with_a_wait_block():
    """IQL.td_update's own torch graph (float64) on a layout with n_w > 0"""
    from deeprl_signal_control_b200.agents.models import IQL
    rng = np.random.default_rng(3)
    cp = configparser.ConfigParser(); cp.read_string(INI)
    cfg = cp["MODEL_CONFIG"]
    m = IQL([30, 24], [5, 3], [6, 0], 0, cfg, seed=1, model_type="dqn", device="cpu")
    for i, (n_s, n_w, n_a) in enumerate([(30, 6, 5), (24, 0, 3)]):
        w = {k: v.detach().numpy().astype(np.float64) for k, v in m.nets[i].items()}
        S, A, S1, Rw, D = _batch(rng, 20, n_s, n_a)
        out = q_td_ref(w, "dqn", n_w, S, A, S1, Rw, D, 0.99)
        p = {k: torch.tensor(v, requires_grad=True) for k, v in w.items()}
        St, S1t = torch.tensor(S), torch.tensor(S1)
        q0 = q_net64(p, "dqn", n_w, St).gather(1, torch.tensor(A)[:, None])[:, 0]
        with torch.no_grad():
            tq = torch.where(torch.tensor(D), torch.tensor(Rw), torch.tensor(Rw) + 0.99 * q_net64(p, "dqn", n_w, S1t).max(1)[0])
        loss = ((q0 - tq) ** 2).mean()
        grads = torch.autograd.grad(loss, list(p.values()))
        assert abs(out["loss"] - float(loss)) <= 1e-12 * abs(float(loss))
        for k, g in zip(p, grads):
            np.testing.assert_allclose(out["grads"][k], g.numpy(), rtol=1e-10, atol=1e-14, err_msg=k)


# the GPU bounds of tests/test_iql_train_gpu.py: loss rel 5e-5, gradient 5e-4 of each tensor's max
def _rel_change(a, b):
    return max(np.abs(a["grads"][k] - b["grads"][k]).max() / max(np.abs(a["grads"][k]).max(), 1e-30) for k in a["grads"])


def test_planted_defects_move_the_loss_or_gradient_far_beyond_the_gpu_bound():
    rng = np.random.default_rng(5)
    n_s, n_w, n_a = 30, 6, 5
    w = _ragged_weights(rng, n_s, n_w, n_a)
    S, A, S1, Rw, D = _batch(rng, 40, n_s, n_a)
    base = q_td_ref(w, "dqn", n_w, S, A, S1, Rw, D, 0.99)
    bound = 5e-4
    for mut in ("no_done", "grad_tq", "s_for_s1"):
        bad = q_td_ref(w, "dqn", n_w, S, A, S1, Rw, D, 0.99, mutate=mut)
        moved = max(abs(bad["loss"] - base["loss"]) / base["loss"], _rel_change(base, bad))
        assert moved >= 10 * bound, (mut, moved)
    # s1 taken from the next ring slot (at an episode end that is the reset observation, not the terminal one)
    S1_next = np.roll(S, -1, axis=0)
    bad = q_td_ref(w, "dqn", n_w, S, A, S1_next, Rw, D, 0.99)
    assert max(abs(bad["loss"] - base["loss"]) / base["loss"], _rel_change(base, bad)) >= 10 * bound
    # the wrong agent's observation slice
    obs = rng.standard_normal((40, 2 * n_s))
    good = q_td_ref(w, "dqn", n_w, obs[:, :n_s], A, obs[:, :n_s][::-1], Rw, D, 0.99)
    bad = q_td_ref(w, "dqn", n_w, obs[:, n_s:], A, obs[:, n_s:][::-1], Rw, D, 0.99)
    assert max(abs(bad["loss"] - good["loss"]) / good["loss"], _rel_change(good, bad)) >= 10 * bound


# ---- numpy restatements of the device's counter-hash draws --------------------------------------------------------
def qmix32(h):
    h = np.asarray(h, np.uint64) & M32
    h ^= h >> 16; h = (h * 0x7feb352d) & M32
    h ^= h >> 15; h = (h * 0x846ca68b) & M32
    h ^= h >> 16
    return h


def row_hash(seed, step, replica, a):
    lo, hi = seed & M32, seed >> 32
    h = qmix32(lo ^ ((step * 0x9E3779B1) & M32))
    h = qmix32(h ^ hi ^ ((np.asarray(replica, np.uint64) * 0x85EBCA77) & M32))
    return qmix32(h ^ ((a * 0xC2B2AE3D) & M32))


def explore_ref(q, n_a, eps, seed, step, replica0):
    """tscl_q_explore's actions: first argmax, or the uniform action when u < eps.  q [R][A][max_na]"""
    R, A = q.shape[:2]
    act = np.zeros((R, A), np.int64)
    for a in range(A):
        h = row_hash(seed, step, np.arange(R) + replica0, a)
        u = (h >> 8).astype(np.float32) * np.float32(1.0 / 16777216.0)
        rnd = ((qmix32(h ^ 0x5BD1E995) * np.uint64(n_a[a])) >> 32).astype(np.int64)
        greedy = np.argmax(q[:, a, :n_a[a]], axis=1)
        act[:, a] = np.where(u < np.float32(eps), rnd, greedy)
    return act


def sample_ref(A, R, batch, size, seed, update, rnd, replica0):
    """tscl_q_sample: idx [A][R][batch], Floyd's algorithm with multiply-shift draws"""
    lo, hi = seed & M32, seed >> 32
    out = np.zeros((A, R, batch), np.int64)
    for a in range(A):
        rep = np.arange(R, dtype=np.uint64) + np.uint64(replica0)
        h = qmix32(lo ^ ((update * 0x9E3779B1) & M32))
        h = qmix32(h ^ hi ^ ((rep * 0x85EBCA77) & M32))
        key = qmix32(h ^ ((a * 0xC2B2AE3D) & M32) ^ ((rnd * 0x27D4EB2F) & M32))
        for d in range(batch):
            j = size - batch + d
            x = qmix32(key ^ (((d + 1) * 0x165667B1) & M32))
            t = ((x * np.uint64(j + 1)) >> 32).astype(np.int64)
            taken = (out[a, :, :d] == t[:, None]).any(axis=1)
            out[a, :, d] = np.where(taken, j, t)
    return out


@pytest.mark.parametrize("size", [20, 37, 1000])
def test_sampler_draws_are_distinct_and_in_range(size):
    idx = sample_ref(3, 256, 20, size, 7, 4, 2, 100)
    assert idx.min() >= 0 and idx.max() < size
    for row in idx.reshape(-1, 20):
        assert len(set(row.tolist())) == 20
    if size == 1000:       # roughly uniform over the ring
        counts = np.bincount(idx.ravel(), minlength=size)
        assert counts.min() > 0 and counts.max() < 3 * counts.mean()


def test_explore_draws_follow_eps():
    rng = np.random.default_rng(0)
    q = rng.standard_normal((4096, 3, 5)).astype(np.float32)
    n_a = [5, 3, 4]
    greedy = explore_ref(q, n_a, 0.0, 9, 11, 0)
    assert all((greedy[:, a] == np.argmax(q[:, a, :n_a[a]], 1)).all() for a in range(3))
    rand = explore_ref(q, n_a, 1.0, 9, 11, 0)
    for a in range(3):
        c = np.bincount(rand[:, a], minlength=n_a[a])
        assert len(c) == n_a[a] and c.min() > 0.7 * 4096 / n_a[a]


@pytest.mark.parametrize("kind", ["lr", "dqn"])
def test_initial_weights_equal_iql_seed(kind):
    from deeprl_signal_control_b200.agents.layout import QLayout
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL
    from deeprl_signal_control_b200.agents.models import IQL
    cp = configparser.ConfigParser(); cp.read_string(INI)
    cfg = cp["MODEL_CONFIG"]
    n_s, n_a, n_w = [30, 24, 36], [5, 3, 4], [6, 0, 6]
    m = IQL(n_s, n_a, n_w, 0, cfg, seed=4, model_type=kind, device="cpu")
    lay = QLayout.from_iql(m, np.concatenate([[0], np.cumsum(n_s)]), int(sum(n_s)))
    flat = BatchedIQL.initial_params(lay, cfg, kind, 4)
    assert np.array_equal(flat, lay.pack(m.nets).numpy())
