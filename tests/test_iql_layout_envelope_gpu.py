"""GPU: the IQL Q kernels (csrc/tsc_q.cu) at every layout class they accept (tests/iql_layout_envelope.py), against
float64, at R = 300 replicas (not a multiple of the 64-row tile) and batch 20 (6000 TD rows per agent: a partial tile):

  * evaluation forward (tscl_q_step, both action modes) against q_forward_ref with NaN in the observation columns no
    agent owns, padded q columns exactly 0, sampled actions against _sample_ref, and the grouped launch on ragged members
    bit-identical to per-member launches;
  * the ε-greedy explore forward against explore_ref at ε 0, 0.3 and 1, with the ring slot's s and a for every row;
  * one TD round on a wrapped ring: the draws against sample_ref, every agent's named gradients, loss, mean q and mean tq
    against q_td_ref, each within 2x the error of the same round in fp32 torch plus a floor and within a bound per model;
  * the clip + Adam step with max_grad_norm between the agents' norms (some clipped, some not) against float64 Adam on
    the reference's and on the kernel's own gradient; the round repeated from the same state is bit-identical;
  * planted defects of the edge layouts (tests/iql_layout_envelope.py:agent_batch) land at least 10x outside the bounds;
  * short training runs on small_grid and mini SUMO whose learner and checkpoint evaluate identically;
  * layouts one past a limit refused at construction, the TD limit found with tscl_q_info.

Bounds are about 3x the worst value seen on an H100 80GB HBM3 (700 W power limit); the OBSERVED lines print them."""
import configparser
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests.iql_layout_envelope import (BEYOND, DEFECTS, EDGES, FC32_NO_WAIT, GRAD_BOUND, LOSS_BOUND, SCENARIOS, SPARE,
                                       TD_WAVE_MAX, Case, agent_batch, moved, rel_l2, scenario_case, synthetic_case)
from tests.test_evaluator_iql_cpu import q_forward_ref
from tests.test_evaluator_iql_gpu import Q_BOUND, _sample_ref
from tests.test_iql_batched_cpu import adam_ref, explore_ref, q_net64, q_td_ref, sample_ref

pytestmark = pytest.mark.gpu

R, BATCH, B, GAMMA, LR = 300, 20, 64, 0.99, 1e-3
MEMBERS = (1, 63, 65, 171)                 # ragged members of one grouped launch: R rows
CASES = ["%s/%s" % c for c in SCENARIOS] + list(EDGES)
# a kernel error within 2x the fp32 torch error of the same rows plus this floor (rel-L2 of a named gradient, relative
# loss / mean q / mean tq error; the excess over 2x fp32 torch observed at most 2.4e-7)
FLOOR = 7.5e-7
# Adam after one round against the float64 round: rel-L2 of m (observed lr 1.9e-7, dqn 7.8e-6), v (lr 3.5e-7, dqn 1.2e-6)
# and the weight step (lr 1.6e-5, dqn 1.4e-5)
ADAM_M_BOUND = {"lr": 6e-7, "dqn": 2.5e-5}
ADAM_V_BOUND = {"lr": 1.1e-6, "dqn": 4e-6}
STEP_BOUND = {"lr": 5e-5, "dqn": 5e-5}


def _lib():
    from deeprl_signal_control_b200 import _lib as L
    return L


def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _case(name, tmp_path):
    if name in EDGES:
        return synthetic_case(**EDGES[name])
    if name in BEYOND:
        return synthetic_case(**BEYOND[name][0])
    c = scenario_case(*name.split("/"), str(tmp_path))
    c.n_obs += SPARE                       # observation columns that belong to no agent
    return c


def _model(c, seed):
    """the case's IQL with weights off the initialisation and biases away from zero (no exact argmax ties)"""
    m = c.iql(seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for p in m.nets:
        for v in p.values():
            v.data.add_(torch.randn(v.shape, generator=g) * 0.05)
    return m


def _shifted(lay, P, delta):
    """P with every q/b raised by delta: q > 0 everywhere for the normalised-q sample"""
    P = P.clone()
    for v in lay.views(P):
        v["q/b"].add_(delta)
    return P


def _unowned(lay):
    own = np.zeros(lay.n_obs, bool)
    for o, n in zip(lay.obs_off, lay.n_s):
        own[int(o):int(o) + int(n)] = True
    return np.flatnonzero(~own)


class _H:
    """a tscl_q handle on a QLayout"""

    def __init__(self, lay):
        self.lib, self.check = _lib().lib(), _lib().check
        self.lay, self.h = lay, C.c_void_p()
        self.check(self.lib.tscl_q_create(C.byref(lay.as_c()), C.c_int32(0), C.byref(self.h)))

    def info(self):
        f, t = C.c_int64(), C.c_int64()
        self.check(self.lib.tscl_q_info(self.h, C.byref(f), C.byref(t)))
        return f.value, t.value

    def step(self, P, obs, q, act, mode, seed, step, bad=None):
        self.check(self.lib.tscl_q_step(self.h, _p(P), _p(obs), C.c_int64(obs.shape[0]), _p(q), _p(act), C.c_int32(mode),
                                        C.c_uint64(seed), C.c_int64(step), C.c_int64(0),
                                        None if bad is None else _p(bad), _st()))

    def step_g(self, Ps, obs, rows, q, act, mode, seeds, step, bad):
        self.check(self.lib.tscl_q_step_g(self.h, _p(Ps), C.c_int64(Ps.shape[1]), _p(obs), C.c_int32(Ps.shape[0]),
                                          _p(rows), C.c_int64(obs.shape[0]), _p(q), _p(act), C.c_int32(mode), _p(seeds),
                                          C.c_int64(step), _p(bad), _st()))

    def close(self):
        self.lib.tscl_q_destroy(self.h)


def _q64(m, lay, obs):
    o = np.asarray(obs, np.float64)
    q, scale = np.zeros((o.shape[0], lay.A, lay.max_na)), np.zeros((o.shape[0], lay.A))
    for i in range(lay.A):
        w = {k: v.detach().cpu().numpy() for k, v in m.nets[i].items()}
        s = o[:, int(lay.obs_off[i]):int(lay.obs_off[i]) + int(lay.n_s[i])]
        q[:, i, :int(lay.n_a[i])], scale[:, i] = q_forward_ref(lay.model_type, w, s, int(lay.n_w[i]), with_scale=True)
    return q, scale


def _forward_error(lay, q, q64, scale):
    return max(float((np.abs(q[:, i, :na] - q64[:, i, :na]).max(1) / scale[:, i]).max()) for i, na in enumerate(lay.n_a))


# ---- evaluation forward ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES + ["td_wave_beyond"])
def test_evaluation_forward(name, tmp_path):
    c = _case(name, tmp_path)
    m = _model(c, 3)
    lay = c.layout(m)
    kind = lay.model_type
    h = _H(lay)
    P = lay.pack(m.nets).cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    obs = torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2
    nan_cols = _unowned(lay)
    assert len(nan_cols) >= SPARE
    obs[:, torch.from_numpy(nan_cols).cuda()] = float("nan")
    q = torch.full((R, lay.A, lay.max_na), float("nan"), device="cuda")
    act = torch.full((R, lay.A), -1, dtype=torch.int32, device="cuda")
    h.step(P, obs, q, act, 0, 7, 2)
    torch.cuda.synchronize()
    qn, an = q.cpu().numpy(), act.cpu().numpy()
    assert np.isfinite(qn).all()
    for i, na in enumerate(lay.n_a):
        assert (qn[:, i, na:] == 0).all(), i
        np.testing.assert_array_equal(an[:, i], np.argmax(qn[:, i, :na], 1))
    q64, scale = _q64(m, lay, obs.cpu().numpy())
    err = _forward_error(lay, qn, q64, scale)
    n_clear = n_all = 0
    for i, na in enumerate(lay.n_a):
        srt = np.sort(q64[:, i, :na], 1)
        clear = (srt[:, -1] - srt[:, -2]) > 2 * Q_BOUND[kind] * scale[:, i]
        np.testing.assert_array_equal(an[clear, i], np.argmax(q64[:, i, :na], 1)[clear])
        n_clear += int(clear.sum()); n_all += R
    # mode 1: the normalised-q sample on weights whose q is positive everywhere
    Ppos = _shifted(lay, P, 100.0)
    bad = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    h.step(Ppos, obs, q, act, 1, (3 << 32) | 99, 4, bad)
    torch.cuda.synchronize()
    qp = q.cpu().numpy()
    assert (qp[:, :, 0] > 0).all() and int(bad.item()) == -1
    np.testing.assert_array_equal(act.cpu().numpy(), _sample_ref(qp, lay.n_a, (3 << 32) | 99, 4, 0))
    # grouped launch: ragged members with their own weights and seeds, bit-identical to one launch per member
    K = len(MEMBERS)
    rows = torch.tensor(np.concatenate([[0], np.cumsum(MEMBERS)]), dtype=torch.int64, device="cuda")
    assert int(rows[-1]) == R
    seeds = torch.tensor([11 + 1000 * k for k in range(K)], dtype=torch.int64, device="cuda")
    for mode, base in ((0, P), (1, Ppos)):
        Ps = torch.stack([base * (1.0 + 0.01 * k) for k in range(K)])
        qg, ag = torch.full_like(q, float("nan")), torch.full_like(act, -1)
        badg = torch.full((K,), -1, dtype=torch.int64, device="cuda")
        h.step_g(Ps, obs, rows, qg, ag, mode, seeds, 6, badg)
        qs, as_ = torch.full_like(q, float("nan")), torch.full_like(act, -1)
        bads = torch.full((K,), -1, dtype=torch.int64, device="cuda")
        for k in range(K):
            r0, r1 = int(rows[k]), int(rows[k + 1])
            h.step(Ps[k], obs[r0:r1], qs[r0:r1], as_[r0:r1], mode, int(seeds[k]), 6, bads[k:k + 1])
        torch.cuda.synchronize()
        assert torch.equal(qg, qs) and torch.equal(ag, as_) and torch.equal(badg, bads), mode
        assert int(badg.max()) == -1
    h.close()
    print("OBSERVED forward %-22s %s: max |q - q64| / row scale %.3g (bound %.2g, %.1fx margin); %d of %d argmax "
          "decisions clear of the bound" % (name, kind, err, Q_BOUND[kind], Q_BOUND[kind] / max(err, 1e-30), n_clear, n_all))
    assert err <= Q_BOUND[kind], err
    assert n_clear > 0.99 * n_all


# ---- explore, one TD round, clip + Adam ----------------------------------------------------------------------------
def _learner(c, lay, P, seed=11):
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL
    m = BatchedIQL(lay, R, c.cfg(buffer_size=B), lay.model_type, seed=seed, device=0)
    m.P.copy_(P)
    return m


def _fp32_round(w, kind, n_w, S, A, S1, Rw, D, n_total):
    """the round in float32 torch on the CPU (IQL.td_update's arithmetic): grads, loss, mean q, mean tq"""
    p = {k: torch.tensor(np.asarray(v, np.float32), requires_grad=True) for k, v in w.items()}
    St, S1t = torch.tensor(np.asarray(S, np.float32)), torch.tensor(np.asarray(S1, np.float32))
    q0 = q_net64(p, kind, n_w, St).gather(1, torch.tensor(np.asarray(A, np.int64))[:, None])[:, 0]
    with torch.no_grad():
        Rt = torch.tensor(np.asarray(Rw, np.float32))
        tq = torch.where(torch.tensor(np.asarray(D).astype(bool)), Rt, Rt + GAMMA * q_net64(p, kind, n_w, S1t).max(1)[0])
    loss = ((q0 - tq) ** 2).sum() / n_total
    grads = torch.autograd.grad(loss, list(p.values()))
    return dict(grads={k: g.numpy() for k, g in zip(p, grads)}, loss=float(loss.detach()),
                q=float(q0.detach().sum()) / n_total, tq=float(tq.sum()) / n_total)


def _fill_ring(m, lay, g):
    m.s.copy_(torch.rand(m.s.shape, device="cuda", generator=g) * 2)
    m.s1.copy_(torch.rand(m.s1.shape, device="cuda", generator=g) * 2)
    na = torch.tensor(lay.n_a, device="cuda")
    m.a.copy_((torch.rand(m.a.shape, device="cuda", generator=g) * na).to(torch.int8))
    m.r.copy_(torch.randn(m.r.shape, device="cuda", generator=g))
    m.done.copy_((torch.rand(m.done.shape, device="cuda", generator=g) < 0.15).to(torch.uint8))
    m.cum_size = B + 7                     # wrapped: the draws cover the whole ring


def _check_explore(m, h, lay, P, g):
    obs = torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2
    q0, a0 = torch.empty_like(m.q), torch.empty_like(m.act)
    h.step(P, obs, q0, a0, 0, 0, 0)
    for k, eps in enumerate((0.0, 0.3, 1.0)):
        m.cum_size = k
        m.s[k].fill_(-1.0); m.a[k].fill_(-1)
        m.explore(obs, eps, 5 + k)
        torch.cuda.synchronize()
        assert torch.equal(m.s[k], obs), eps                      # every row, the tail tile's included
        assert torch.equal(m.a[k].to(torch.int32), m.act), eps
        ref = explore_ref(m.q.cpu().numpy(), lay.n_a, eps, m.seed, 5 + k, 0)
        assert np.array_equal(m.act.cpu().numpy(), ref), eps
        assert torch.equal(m.q, q0), eps
        if eps == 0.0:
            assert torch.equal(m.act, a0)
        elif eps == 1.0:                   # uniform draws: every action of every agent occurs
            an = m.act.cpu().numpy()
            assert all(len(np.unique(an[:, i])) == lay.n_a[i] for i in range(lay.A))


def _split_threshold(norms):
    """a max_grad_norm with some agents' norms above it and some below, as far from every norm as possible"""
    s = np.sort(np.asarray(norms))
    j = int(np.argmax(s[1:] / s[:-1]))
    assert s[j + 1] / s[j] > 1.01, s
    return float(np.sqrt(s[j] * s[j + 1]))


@pytest.mark.parametrize("name", CASES)
def test_training_round(name, tmp_path):
    c = _case(name, tmp_path)
    mdl = _model(c, 5)
    lay = c.layout(mdl)
    kind = lay.model_type
    P0 = lay.pack(mdl.nets).cuda()
    m = _learner(c, lay, P0)
    h = _H(lay)
    assert h.info()[1] > 0 and h.info() == lay.smem_bytes()
    g = torch.Generator(device="cuda").manual_seed(21)
    _check_explore(m, h, lay, P0, g)
    h.close()

    _fill_ring(m, lay, g)
    idx = m.sample(0)
    torch.cuda.synchronize()
    idx = idx.cpu().numpy()
    assert np.array_equal(idx, sample_ref(lay.A, R, BATCH, B, m.seed, 0, 0, 0))
    s, s1 = m.s.cpu().numpy(), m.s1.cpu().numpy()
    a, r, d = m.a.cpu().numpy(), m.r.cpu().numpy(), m.done.cpu().numpy()
    rr = np.repeat(np.arange(R), BATCH)
    n_total = R * BATCH
    P64 = P0.double().cpu().numpy()
    refs, batches = [], []
    for i in range(lay.A):
        sl = idx[i].reshape(-1)
        w, n_w, S, S1, _ = agent_batch(lay, P64, i, s[sl, rr], s1[sl, rr])
        batches.append((s[sl, rr], s1[sl, rr], a[sl, rr, i].astype(np.int64), r[sl, rr, i], d[sl, rr]))
        refs.append(q_td_ref(w, kind, n_w, S, batches[-1][2], S1, batches[-1][3], batches[-1][4], GAMMA,
                             n_total=n_total))
    m.max_grad_norm = _split_threshold([x["norm"] for x in refs])
    rec = torch.zeros(lay.A, 4, device="cuda")
    m.td_round(0, LR, idx=torch.from_numpy(idx.astype(np.int32)).cuda(), rec=rec)
    torch.cuda.synchronize()
    P1, M1, V1, grad1 = m.P.clone(), m.M.clone(), m.V.clone(), m.grad.clone()
    G = lay.views(grad1[:lay.n_params].double().cpu().numpy())
    rec = rec.double().cpu().numpy()
    W1, Mv, Vv = (lay.views(x.double().cpu().numpy()) for x in (P1, M1, V1))
    W0 = lay.views(P64)

    worst = dict(grad=(0.0, ""), loss=(0.0, ""), over_fp32=-np.inf, m=0.0, v=0.0, step=0.0)
    clipped = []
    for i in range(lay.A):
        ref, n_w = refs[i], int(lay.n_w[i])
        w, _, S, S1, _ = agent_batch(lay, P64, i, batches[i][0], batches[i][1])
        f32 = _fp32_round(w, kind, n_w, S, batches[i][2], S1, batches[i][3], batches[i][4], n_total)
        q_ref = float(ref["q"][np.arange(len(batches[i][2])), batches[i][2]].sum()) / n_total
        tq_all = ref["q"][np.arange(len(batches[i][2])), batches[i][2]] - ref["err"]
        scale_q = float(np.abs(ref["q"][np.arange(len(batches[i][2])), batches[i][2]]).mean())
        scale_tq = float(np.abs(tq_all).mean())
        errs = {"loss": (abs(rec[i, 0] - ref["loss"]) / ref["loss"], abs(f32["loss"] - ref["loss"]) / ref["loss"]),
                "mean q": (abs(rec[i, 1] - q_ref) / scale_q, abs(f32["q"] - q_ref) / scale_q),
                "mean tq": (abs(rec[i, 2] - tq_all.sum() / n_total) / scale_tq,
                            abs(f32["tq"] - tq_all.sum() / n_total) / scale_tq)}
        for k, gref in ref["grads"].items():
            errs[k] = (rel_l2(G[i][k], gref), rel_l2(f32["grads"][k], gref))
        for k, (e, f) in errs.items():
            grad = k in ref["grads"]
            bound = GRAD_BOUND[kind] if grad else LOSS_BOUND[kind]
            assert e <= 2 * f + FLOOR, (i, k, e, f)
            assert e <= bound, (i, k, e, bound)
            key = "grad" if grad else "loss"
            worst[key] = max(worst[key], (e, "agent %d %s" % (i, k)))
            worst["over_fp32"] = max(worst["over_fp32"], e - 2 * f)
        norm_k = float(rec[i, 3])
        assert abs(norm_k - ref["norm"]) <= GRAD_BOUND[kind] * ref["norm"], (i, norm_k, ref["norm"])
        is_clipped = ref["norm"] > m.max_grad_norm
        assert (norm_k > m.max_grad_norm) == is_clipped
        clipped.append(is_clipped)
        # Adam against the float64 round, and against float64 Adam on the kernel's own gradient
        zero = {k: 0 * v for k, v in ref["grads"].items()}
        w_ref, ad = adam_ref(W0[i], ref["grads"], ref["norm"], dict(t=0, m=zero, v=zero), LR, m.max_grad_norm)
        cat = lambda d: np.concatenate([np.ravel(d[k]) for k in ref["grads"]])
        worst["m"] = max(worst["m"], rel_l2(cat(Mv[i]), cat(ad["m"])))
        worst["v"] = max(worst["v"], rel_l2(cat(Vv[i]), cat(ad["v"])))
        worst["step"] = max(worst["step"], rel_l2(cat(W1[i]) - cat(W0[i]), cat(w_ref) - cat(W0[i])))
        gk = {k: np.asarray(G[i][k]) for k in ref["grads"]}
        w_own, ad_own = adam_ref(W0[i], gk, float(np.sqrt(sum((x * x).sum() for x in gk.values()))),
                                 dict(t=0, m=zero, v=zero), LR, m.max_grad_norm)
        for k in ref["grads"]:
            step = np.abs(w_own[k] - W0[i][k])
            assert (np.abs(W1[i][k] - w_own[k]) <= 2.0 ** -23 * np.abs(W0[i][k]) + 1e-5 * step + 1e-30).all(), (i, k)
            assert np.abs(Mv[i][k] - ad_own["m"][k]).max() <= 1e-5 * max(np.abs(ad_own["m"][k]).max(), 1e-30), (i, k)
    assert any(clipped) and not all(clipped), clipped
    assert worst["m"] <= ADAM_M_BOUND[kind] and worst["v"] <= ADAM_V_BOUND[kind], worst
    assert worst["step"] <= STEP_BOUND[kind], worst
    print("OBSERVED round %-22s %s: worst gradient rel-L2 %.3g (%s; bound %.2g), worst loss/q/tq rel %.3g (%s; bound "
          "%.2g), worst (error - 2x fp32 torch) %.3g" % (name, kind, worst["grad"][0], worst["grad"][1], GRAD_BOUND[kind],
                                                          worst["loss"][0], worst["loss"][1], LOSS_BOUND[kind],
                                                          worst["over_fp32"]))
    print("OBSERVED adam  %-22s %s: max_grad_norm %.4g clips %d of %d agents; m rel-L2 %.3g, v %.3g, weight step %.3g "
          "(bounds %.2g / %.2g / %.2g)" % (name, kind, m.max_grad_norm, sum(clipped), lay.A, worst["m"], worst["v"],
                                           worst["step"], ADAM_M_BOUND[kind], ADAM_V_BOUND[kind], STEP_BOUND[kind]))
    # the same round from the same state: bit-identical
    m.P.copy_(P0); m.M.zero_(); m.V.zero_(); m.t = 0
    m.td_round(0, LR, idx=torch.from_numpy(idx.astype(np.int32)).cuda())
    torch.cuda.synchronize()
    assert torch.equal(m.P, P1) and torch.equal(m.M, M1) and torch.equal(m.V, V1) and torch.equal(m.grad, grad1)

    if name in EDGES:                      # planted defects: the kernel's round lands far outside each
        got = [dict(loss=float(rec[i, 0]), grads=G[i]) for i in range(lay.A)]
        seen = {}
        for defect in DEFECTS:
            for i in range(lay.A):
                b = agent_batch(lay, P64, i, batches[i][0], batches[i][1], defect)
                if b is None:
                    continue
                bad = q_td_ref(b[0], kind, b[1], b[2], batches[i][2], b[3], batches[i][3], batches[i][4], GAMMA,
                               n_total=n_total, mutate=b[4])
                ratio, what = moved(got[i], bad, kind)
                assert ratio >= 10, (defect, i, what, ratio)
                seen[defect] = min(seen.get(defect, (np.inf, "")), (ratio, what))
        for defect, (ratio, what) in seen.items():
            print("OBSERVED defect %-22s %-46s moves %s by %.0fx its bound" % (name, defect, what, ratio))
        assert "done mask dropped" in seen and "next agent's observation slice" in seen


# ---- end to end ---------------------------------------------------------------------------------------------------
SMALL_ENV = """
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = %s
coop_gamma = 0.75
data_path = ./small_grid/data/
episode_length_sec = 300
norm_wave = 5.0
norm_wait = 100.0
coef_wait = 0.2
num_extra_car_per_hour = 1000
objective = hybrid
scenario = small_grid
seed = 42
test_seeds = 10000,20000
yellow_interval_sec = 2
"""
MINI_ENV = """
[ENV_CONFIG]
clip_wave = 2.0
clip_wait = 2.0
control_interval_sec = 5
agent = %s
coop_gamma = 0.9
episode_length_sec = 300
norm_wave = 5.0
norm_wait = 100.0
coef_wait = 0.2
objective = hybrid
scenario = mini
seed = 5
test_seeds = 100,200
yellow_interval_sec = 2
net_file = %s
route_file = %s
"""


def _env(scenario, agent, tmp_path, out):
    os.makedirs(str(tmp_path), exist_ok=True)
    cp = configparser.ConfigParser()
    if scenario == "small_grid":
        from deeprl_signal_control_b200.envs.small_grid_env import SmallGridEnv as Env
        cp.read_string(SMALL_ENV % agent)
    else:
        import sys
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "fixtures"))
        import make_mini_sumo
        from deeprl_signal_control_b200.envs.sumo_env import SumoNetEnv as Env
        cp.read_string(MINI_ENV % ((agent,) + tuple(make_mini_sumo.write(str(tmp_path)))))
    return Env(cp["ENV_CONFIG"], output_path=out, is_record=False, n_replicas=2)


@pytest.mark.parametrize("scenario", ["small_grid", "mini_sumo"])
@pytest.mark.parametrize("agent", ["iqll", "iqld"])
def test_trains_and_evaluates_end_to_end(scenario, agent, tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL, BatchedIQLTrainer
    from deeprl_signal_control_b200.agents.utils import Scheduler
    from deeprl_signal_control_b200.sim import BatchedSim
    out = str(tmp_path) + os.sep
    env = _env(scenario, agent, tmp_path, out)
    net = env._tables
    off = np.asarray(net.node_obs_off)
    kind = "dqn" if agent == "iqld" else "lr"
    c = Case(kind, [int(off[i + 1] - off[i]) for i in range(net.n_nodes)], net.n_a_ls, net.n_w_ls, off, net.n_obs,
             net.max_na)
    lay = c.layout()
    if kind == "dqn":
        assert any(lay.n_w) and lay.n_ft == 32
    m = BatchedIQL(lay, 16, c.cfg(), kind, seed=3, device=0)
    sim = BatchedSim(net, env._params, 16, device=0)
    tr = BatchedIQLTrainer(sim, m, Scheduler(1e-3, decay="constant"), Scheduler(1.0, 0.01, 40, decay="linear"))
    P0 = m.P.clone()
    tr.run(60)                             # one 60-step episode, three backwards
    torch.cuda.synchronize()
    assert tr.n_updates == 3 and len(tr.episode_rewards) == 1
    assert bool(torch.isfinite(m.losses).all()) and float(m.norms.min()) > 0
    assert bool(torch.isfinite(m.P).all()) and not torch.equal(P0, m.P)
    d = str(tmp_path / "ck")
    os.makedirs(d)
    m.save(d, 60)
    ref = c.iql(seed=99, device="cuda")
    assert ref.load(d)
    for i, p in enumerate(ref.nets):
        for k, v in p.items():
            assert torch.equal(v.detach(), m.nets[i][k]), (i, k)
    mean_b, std_b = Evaluator(env, m, out).run()
    mean_r, std_r = Evaluator(_env(scenario, agent, tmp_path / "again", out), ref, out).run()
    print("OBSERVED e2e %s %s: episode reward %s, evaluation means %s" % (scenario, agent, tr.episode_rewards, mean_b))
    assert np.isfinite(mean_b).all()
    np.testing.assert_array_equal(mean_b, mean_r)
    np.testing.assert_array_equal(std_b, std_r)


# ---- refusals -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(BEYOND))
def test_beyond_the_limits_is_refused_at_construction(name):
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL
    kw, msg = BEYOND[name]
    c = synthetic_case(**kw)
    lay = c.layout()
    err = ValueError if name == "td_wave_beyond" else RuntimeError
    with pytest.raises(err, match=msg) as e:
        BatchedIQL(lay, 8, c.cfg(buffer_size=B), c.kind, device=0)
    if name == "td_wave_beyond":           # names the bytes needed and available
        assert str(lay.smem_bytes()[1]) in str(e.value)
        assert str(torch.cuda.get_device_properties(0).shared_memory_per_block_optin) in str(e.value)
    if name == "fc32_wait":                # the same width without wait inputs trains
        c = synthetic_case(**FC32_NO_WAIT)
        m = BatchedIQL(c.layout(), 8, c.cfg(buffer_size=B), c.kind, device=0)
        m.cum_size = B
        m.td_round(0, LR)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(m.P).all()) and float(m.norms[0].min()) > 0


def test_td_limit_found_with_the_query():
    """a wave block W next to 6 wait inputs at the reference widths: tscl_q_info reports the TD kernel's bytes up to
    W = TD_WAVE_MAX and 0 from the next W on, while the forward keeps fitting; the reported bytes are QLayout.smem_bytes"""
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    first_over = None
    for W in range(TD_WAVE_MAX - 8, TD_WAVE_MAX + 9):
        lay = synthetic_case(n_wave=[W, 21], n_wait=[6, 0], n_a=[4, 3]).layout()
        h = _H(lay)
        fwd, td = h.info()
        h.close()
        want = lay.smem_bytes()
        assert fwd == want[0] and td == (want[1] if want[1] <= optin else 0), (W, fwd, td, want)
        if td == 0 and first_over is None:
            first_over = W
        assert (td == 0) == (first_over is not None), W
    print("OBSERVED TD limit: wave block %d (+6 wait) fits in %d bytes of opt-in shared memory, %d does not"
          % (first_over - 1, optin, first_over))
    assert first_over == TD_WAVE_MAX + 1
