"""GPU: `BatchedA2C` with its default settings at every layout class it accepts (tests/layout_envelope.py), against
float64.  Each case runs a T = 12 rollout from nonzero recurrent states with dones at interior steps, R = 320, then
backward(lr=0), and checks:

  * the selected forward family and update path (learner_paths), so that a silent change of path fails;
  * every forward step: the fused v2 forward against a restatement of its bf16 arithmetic (X within one bf16 ulp of the
    float64 fc front end on bf16 operands, c / h from bf16 operands, the activation store, pi / value from the kernel's
    h), the v1 forward against the float64 step on its bf16 GEMM operands; actions against the inverse-CDF sample of
    pi; pi exactly 0 in the padded action columns;
  * test-mode evaluation: the Evaluator's family is the training forward's, and its launch gives the same pi bit for bit;
  * the gradient G against float64 references that round where the chosen path rounds (oracle/learner_ref.py):
    update_ref on the kernel's own activation store ('lean': bf16 operands throughout; 'store': dX = dZ . Wx^T by a
    TF32 torch product and fp32 fc weight gradients), and the recompute reference for 'recompute' — rel-L2 per named
    tensor and overall;
  * planted defects of the edge layouts, built by perturbing the reference's inputs: each moves some named tensor of G by
    at least 10x its bound;
  * a population of K = 2 where selection allows one (the wave block that fills its tile): every member's forward is
    bit-identical to its solo learner, its first gradient within the spread of two solo runs.

Layouts one past a kernel limit must be refused at construction, and the reference's Monaco IA2C configuration trains
and evaluates end to end.  Bounds are about 3x the worst value seen on an H100 80GB HBM3 (700 W power limit)."""
import copy
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.layout_envelope import BEYOND, EDGES, ROOT, net_tables, scenario_layout, synthetic_layout
from tests.test_evaluator_gpu import REAL_INI, _pi_step
from tests.test_policy_forward_bench_size_gpu import _reference_actions
from tests.test_update_recompute_bench_size_gpu import (GROUPS_LSTM, _check_returns, _per_tensor, _recompute_reference,
                                                        _rel_l2)
from tests.update_fallback_bounds import RECOMPUTE_G_REL_L2, RECOMPUTE_TENSOR_REL_L2

pytestmark = pytest.mark.gpu

T, R, GAMMA, BETA = 12, 320, 0.99, 0.01
DONES = (4, 9)
KW = dict(gamma=GAMMA, v_coef=0.5, max_grad_norm=40.0, reward_norm=2000.0, reward_clip=2.0)
# G rel-L2 bounds (overall, worst named tensor) per update path.  Observed: lean 8.0e-5 / 1.8e-4 (mini SUMO MA2C, fcf_w),
# store 2.2e-5 / 3.6e-5 (wh), recompute 3.5e-4 / 5.4e-4 (grid IA2C fw 64, wh; the bench-shape bounds of
# update_fallback_bounds.py).  The planted defects move a named tensor by 52x (bias slot) to 6000x its bound.
BOUNDS = {"lean": (2.5e-4, 6e-4), "store": (7e-5, 1.2e-4), "recompute": (RECOMPUTE_G_REL_L2, RECOMPUTE_TENSOR_REL_L2)}
# forward: max |delta| of c / h (tanh.approx, bf16 flips of X; observed 1.1e-5 from the store's X, 8.3e-4 from X
# restated without a store, 2.3e-3 for v1), of pi / value from the kernel's own h (observed 9.4e-8 / 2.3e-7), and of the
# stored gate activations (observed 3.9e-3: one bf16 ulp below 1)
CH_MAX, HEAD_MAX, ST_G_MAX = 7e-3, 1e-6, 1e-2


def _bf(x):
    return x.to(torch.bfloat16).to(x.dtype)


def _layout(case, tmp_path):
    if case in EDGES or case == "limits_tail_chunk":
        return synthetic_layout(**EDGES["limits" if case == "limits_tail_chunk" else case][0])
    scenario, agent, fw = CASES[case][3]
    return scenario_layout(net_tables(scenario, agent, str(tmp_path)), agent, fw)


# case -> (forward, update the case runs, chunk, (scenario, agent, fw) or None)
CASES = {
    "monaco_ia2c": ("v2", "lean", 1024, ("real_net", "ia2c", 128)),     # dx 128, wave block 48
    "grid_ia2c_fw64": ("v1", "recompute", 1024, ("large_grid", "ia2c", 64)),
    "wave32_wait": ("v2", "store", 1024, None),
    "wave48_fp": ("v2", "store", 1024, None),
    "limits": ("v2", "lean", 1024, None),
    "limits_tail_chunk": ("v2", "recompute", 96, None),                # 96 does not divide 320: no store
    "mini_sumo_ma2c": ("v2", "lean", 1024, ("mini_sumo", "ma2c", 128)),
    "mini_sumo_ia2c": ("v2", "lean", 1024, ("mini_sumo", "ia2c", 128)),
}

# planted defects per edge case: perturbations of the reference's observations / layout
DEFECTS = {"wave32_wait": ["last wave input dropped"], "wave48_fp": ["last wave input dropped"],
           "limits": ["last wave input dropped", "bias slot read as an input", "padded actions in the softmax",
                      "wait block read at the fingerprint offset"]}


def _plant(name, lay, obs):
    """(layout, obs [.., n_obs]) the reference reads with defect `name`"""
    ob = obs.clone()
    for a in range(lay.A):
        o0, nw, nt = int(lay.obs_off[a]), int(lay.n_wave[a]), int(lay.n_wait[a])
        if name == "last wave input dropped":
            ob[..., o0 + nw - 1] = 0.0
        elif name == "bias slot read as an input":          # the ones column lands on the last wave input
            ob[..., o0 + nw - 1] = 1.0
        elif name == "wait block read at the fingerprint offset" and nt > 0:
            src = torch.clamp(torch.arange(o0 + nw + nt, o0 + nw + 2 * nt, device=obs.device), max=lay.n_obs - 1)
            ob[..., o0 + nw:o0 + nw + nt] = obs[..., src]
    if name == "padded actions in the softmax":
        lay = copy.copy(lay)
        lay.n_a = np.full(lay.A, lay.max_na, np.int32)
    return lay, ob


def _store_rows(st, t, U):
    """slot t of an activation-store array [R/rc][U][T][rc][w] as [U][R][w]"""
    return st[:, :, t].transpose(0, 1).reshape(U, -1, st.shape[-1]).double()


def _check_forward(lay, m, obs, done, c0, h0, step, t, err):
    """one committed forward step of a one-member learner (state c0 / h0 before it) against its float64 restatement"""
    from oracle.learner_ref import fc_front
    U, H = lay.U, lay.h
    v = lay.views(m.P.double())
    ob = obs.double()
    if m.tc_v2:                    # the v2 fc front end multiplies bf16 observations and fc weights
        ob = _bf(ob)
        v = {k: (_bf(x) if k[:3] in ("fcw", "fcf", "fct") and "_w" in k else x) for k, x in v.items()}
    X = _bf(torch.stack([fc_front(v, lay, u, ob) for u in range(U)]))
    store = m.tc_v2 and m.store_acts
    if store:                      # fp32 sums in another order: a rounding flip moves an element by one bf16 ulp
        st_x = _store_rows(m.st_x, t, U)
        assert bool(((st_x - X).abs() <= X.abs() * 2 ** -7 + 1e-6).all())
        assert float((st_x != X).double().mean()) < 1e-2
        X = st_x
    keep = 0.0 if done else 1.0
    vd = lay.views(m.P.double())
    z = X @ _bf(vd["wx"]) + _bf(h0.double() * keep) @ _bf(vd["wh"]) + vd["bl"][:, None, :]
    gi, gf, go, gu = (torch.sigmoid(z[..., :H]), torch.sigmoid(z[..., H:2 * H]), torch.sigmoid(z[..., 2 * H:3 * H]),
                      torch.tanh(z[..., 3 * H:]))
    c = gf * c0.double() * keep + gi * gu
    h = go * torch.tanh(c)
    err["c/h"] = max(err.get("c/h", 0.0), float((m.c_fw.double() - c).abs().max()), float((m.h_fw.double() - h).abs().max()))
    if store:
        g = torch.cat([gi, gf, go, gu], -1)
        err["st_g"] = max(err.get("st_g", 0.0), float((_store_rows(m.st_g, t, U) - _bf(g)).abs().max()))
        assert torch.equal(_store_rows(m.st_c, t, U), _bf(m.c_fw.double()))
        assert torch.equal(_store_rows(m.st_h, t, U), _bf(m.h_fw.double()))
    lg = m.h_fw.double() @ vd["wo"] + vd["bo"][:, None, :]
    for a in range(lay.A):
        na = int(lay.n_a[a])
        err["pi"] = max(err.get("pi", 0.0), float((m.pi[:, a, :na].double() - torch.softmax(lg[2 * a, :, :na], -1)).abs().max()))
        err["value"] = max(err.get("value", 0.0), float((m.val[:, a].double() - lg[2 * a + 1, :, 0]).abs().max()))
        assert not bool(m.pi[:, a, na:].any()), "padded pi columns of agent %d are not 0" % a
    act_ref = _reference_actions(m.pi.cpu().numpy(), lay.n_a, m.seed, step, 0)
    assert np.array_equal(m.act.cpu().numpy(), act_ref)


def _check_evaluation_step(lay, m, obs, done, c0, h0, step):
    """the Evaluator's launch for the learner's family (agents/evaluator.py:_actions, sampling) on the state before a
    committed training step gives that step's pi and actions bit for bit"""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    pi, act = torch.full_like(m.pi, float("nan")), torch.full_like(m.act, -1)
    if m.paths.forward == "v2":
        c1, h1 = torch.empty_like(c0[0::2]), torch.empty_like(h0[0::2])
        _pi_step(m, obs, c0[0::2].contiguous(), h0[0::2].contiguous(), c1, h1, pi, act, 0, done, step)
        torch.cuda.synchronize()
        assert torch.equal(c1, m.c_fw[0::2]) and torch.equal(h1, m.h_fw[0::2])
    else:
        assert m.paths.forward == "v1"
        c, h = c0.clone(), h0.clone()
        val = torch.empty_like(m.val)
        _lib.check(_lib.lib().tscl_policy_step(m._h, _p(m.P), _p(m.Wp), _p(obs), C.c_int64(m.R), _p(c), _p(h), _p(c),
                                               _p(h), _p(pi), _p(val), _p(act), C.c_int32(int(done)),
                                               C.c_uint64(m.seed), C.c_int64(step), C.c_int64(0), None, C.c_int32(0),
                                               m._st()))
        torch.cuda.synchronize()
    assert torch.equal(pi, m.pi) and torch.equal(act, m.act)


def _init_state(ms, rows, g):
    """the same nonzero recurrent state in every learner of `ms`: learner i takes rows[i] of one draw"""
    c0 = torch.randn(ms[0].c_fw.shape[0], max(r.stop for r in rows), ms[0].c_fw.shape[2], device="cuda", generator=g)
    h0 = torch.tanh(torch.randn(c0.shape, device="cuda", generator=g)) * 0.5
    for m, r in zip(ms, rows):
        m.c_fw.copy_(c0[:, r] * 0.5); m.h_fw.copy_(h0[:, r])
        m.c_bw.copy_(m.c_fw); m.h_bw.copy_(m.h_fw)


def _rollout(lay, ms, rows, g, check=None):
    """T steps of one rollout through every learner of `ms`, learner i on rows[i] of the same observations, rewards and
    initial states; `check(m, t, obs, done, c0, h0, step)` after each step.  Returns (dpre, dpost, bootstrap values)."""
    Rt = max(r.stop for r in rows)
    _init_state(ms, rows, g)
    dpre = [1.0 if t in DONES else 0.0 for t in range(T)]
    dpost = dpre[1:] + [0.0]
    for t in range(T):
        obs = torch.rand(Rt, lay.n_obs, device="cuda", generator=g) * 2
        rew = torch.randn(Rt, lay.A, device="cuda", generator=g) * 3000
        for m, r in zip(ms, rows):
            m.obs_slot().copy_(obs[r])
            cs, hs, step = m.c_fw.clone(), m.h_fw.clone(), m.n_forward
            m.forward(m.obs_slot(), bool(dpre[t]))
            torch.cuda.synchronize()
            if check is not None:
                check(m, t, m.obs_slot(), bool(dpre[t]), cs, hs, step)
            m.add_transition(rew[r], bool(dpre[t]), bool(dpost[t]))
    nxt = torch.rand(Rt, lay.n_obs, device="cuda", generator=g) * 2
    boot = torch.randn(Rt, lay.A, device="cuda", generator=g)
    for m, r in zip(ms, rows):
        m.obs_hist[T].copy_(nxt[r])
    return dpre, dpost, boot


def _reference_G(lay, m, path, obs, c_bw, h_bw, dpre, defect=None):
    from oracle.learner_ref import update_ref
    if defect is not None:
        lay, obs = _plant(defect, lay, obs)
    if path == "recompute":
        return _recompute_reference(lay, m, obs, c_bw, h_bw, dpre, T, m.R, m.chunk, BETA, tf32=m.allow_tf32)
    store = lambda ci: (m.st_x[ci], m.st_g[ci], m.st_c[ci], m.st_h[ci])
    kw = dict(dx_product="tf32" if m.allow_tf32 else "fp32", fc_fp32=True) if path == "store" else {}
    return update_ref(lay, m.P, store, obs[:T], m.act_hist, m.Rs, m.Adv, c_bw, h_bw, dpre, 1.0 / (T * m.R), 0.5, BETA,
                      m.chunk, agents_per_group=4, **kw)[0]


@pytest.mark.parametrize("case", list(CASES))
def test_layout_matches_float64(case, tmp_path):
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    forward, path, chunk, _ = CASES[case]
    lay = _layout(case, tmp_path)
    m = BatchedA2C(lay, R, n_step=T, seed=7, chunk=chunk, **KW)
    err = {}

    def check(m_, t, obs, done, c0, h0, step):
        _check_forward(lay, m_, obs, done, c0, h0, step, t, err)
        if t in (0, 1):
            _check_evaluation_step(lay, m_, obs, done, c0, h0, step)
    g = torch.Generator(device="cuda").manual_seed(41)
    dpre, dpost, boot = _rollout(lay, [m], [slice(0, R)], g, check)
    print("OBSERVED forward %s (%s, dx %d): max |delta| %s" % (case, forward, lay.dx,
                                                                ", ".join("%s %.2e" % kv for kv in err.items())))
    assert err["c/h"] <= CH_MAX and err["pi"] <= HEAD_MAX and err["value"] <= HEAD_MAX, err
    assert err.get("st_g", 0.0) <= ST_G_MAX, err
    c_bw, h_bw, obs = m.c_bw.clone(), m.h_bw.clone(), m.obs_hist.clone()
    m.backward(boot, lr=0.0, beta=BETA)
    torch.cuda.synchronize()
    _check_returns(m, dpost, boot, GAMMA)
    # the path: selected by learner_paths, and the store on exactly where the case expects it
    from deeprl_signal_control_b200.agents.learner import learner_paths
    p = learner_paths(lay)
    assert vars(m.paths) == vars(p)
    assert m.paths.forward == forward and m.store_acts == (path in ("lean", "store"))
    assert (m.paths.update if m.store_acts else "recompute") == path
    Gref = _reference_G(lay, m, path, obs, c_bw, h_bw, dpre)
    worst = _per_tensor(lay, m.G, Gref, GROUPS_LSTM)
    overall = _rel_l2(m.G, Gref)
    print("OBSERVED update %s (%s): overall rel-L2 %.3e; per tensor %s" % (
        case, path, overall, ", ".join("%s %.2e" % kv for kv in worst.items())))
    b_all, b_t = BOUNDS[path]
    assert overall <= b_all and max(worst.values()) <= b_t, (overall, worst)
    for name in DEFECTS.get(case, []):
        Gm = _reference_G(lay, m, path, obs, c_bw, h_bw, dpre, defect=name)
        moved = _per_tensor(lay, Gm, Gref, GROUPS_LSTM)
        k = max(moved, key=moved.get)
        print("OBSERVED defect %-42s moves %s by rel-L2 %.3e = %.0fx the bound" % (name, k, moved[k], moved[k] / b_t))
        assert moved[k] >= 10 * b_t, (name, moved)
    m.close()


def test_population_on_the_store_path():
    """wave block 32 with wait inputs: no spare slot for the bias column, so the update unpacks the store and multiplies
    dX = dZ . Wx^T with each member's own Wx.  K = 2 members of 320 replicas against solo learners of their seeds."""
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    lay = synthetic_layout(**EDGES["wave32_wait"][0])
    seeds = [7, 11]
    pop = BatchedA2C(lay, R, n_step=T, seeds=seeds, chunk=R, **KW)
    solos = [BatchedA2C(lay, R, n_step=T, seed=s, chunk=R, **KW) for s in seeds + [seeds[0]]]
    rows = [slice(0, 2 * R), slice(0, R), slice(R, 2 * R), slice(0, R)]
    last = {}

    def check(m, t, obs, done, c0, h0, step):
        if m is pop:            # the population steps first, then each solo learner on its member's rows
            last.update(pi=m.pi.clone(), val=m.val.clone(), act=m.act.clone(), c=m.c_fw.clone(), h=m.h_fw.clone())
            return
        r = rows[1 + [id(s) for s in solos].index(id(m))]
        assert torch.equal(last["pi"][r], m.pi) and torch.equal(last["val"][r], m.val), t
        assert torch.equal(last["act"][r], m.act), t
        assert torch.equal(last["c"][:, r], m.c_fw) and torch.equal(last["h"][:, r], m.h_fw), t
    g = torch.Generator(device="cuda").manual_seed(5)
    _, _, boot = _rollout(lay, [pop] + solos, rows, g, check)
    for m, r in zip([pop] + solos, rows):
        m.backward(boot[r], lr=0.0, beta=BETA)
    torch.cuda.synchronize()
    assert pop.store_acts and pop.paths.update == "store" and all(s.paths.update == "store" for s in solos)
    spread = float((solos[0].G - solos[2].G).abs().max())
    scale = float(solos[0].G.abs().max())
    bound = max(2 * spread, 1e-6 * scale)
    for k in (0, 1):
        d = float((pop.G[k] - solos[k].G).abs().max())
        print("OBSERVED population member %d: max |dG| %.3g, two-solo spread %.3g, max |G| %.3g" % (k, d, spread, scale))
        assert d <= bound, (k, d, bound)
    assert not torch.equal(pop.G[0], pop.G[1])


@pytest.mark.parametrize("name", list(BEYOND))
def test_beyond_the_kernel_limits_is_refused(name):
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    kw, msg = BEYOND[name]
    with pytest.raises((ValueError, RuntimeError), match=msg):
        BatchedA2C(synthetic_layout(**kw), 64, n_step=2, use_tc=True)


def test_monaco_ia2c_trains_and_evaluates(tmp_path):
    """train() of the reference's Monaco IA2C configuration (num_fw 128, num_ft 32: dx 128) for one update at R = 64
    with the post-training test, then scripts/evaluate.py on the directory: the same control and traffic CSVs"""
    from deeprl_signal_control_b200.agents.train import train
    from tests.test_train_driver_gpu import A2C_MODEL, TRAIN
    seeds = [10000, 20000]
    cfg = tmp_path / "config_ia2c_real.ini"
    cfg.write_text(A2C_MODEL + TRAIN % (120, 240) + REAL_INI % ("ia2c", 600, ",".join(map(str, seeds))))
    base = tmp_path / "ia2c"
    out = train(str(cfg), str(base), "after_train_test", n_replicas=64)
    assert out.final_step == 120 and out.trainer.n_updates == 1
    assert out.model.batched.paths.forward == "v2" and out.model.layout.dx == 128
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", str(base),
                        "--evaluation-policy-type", "default"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    got = json.load(open(base / "eva_data" / "ia2c_summary.json"))
    mean, std = out.post_test
    assert got["seeds"] == seeds and got["episode_mean_reward"] == [float(x) for x in mean]
    for kind in ("control", "traffic"):
        name = "real_net_ia2c_%s.csv" % kind
        assert (base / "data" / name).read_text() == (base / "eva_data" / name).read_text(), kind
