"""GPU: learner kernels (through the C ABI) vs the float64 CPU restatement (oracle/learner_ref.py,
autograd as the differentiation oracle).  fp32 kernels vs fp64 oracle: rtol 2e-4 / atol 2e-5 on
activations, gradients compared relative to the largest gradient entry of each tensor (3e-4)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _layout(ff=64):
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    if ff == "monaco":
        # Monaco shapes (real_net): no wait block (ft = 0), up to 34 wave inputs, 6 phases
        n_w, n_f, n_wave = [0, 0, 0], [16, 4, 9], [34, 5, 33]
        n_s = [w + f for w, f in zip(n_wave, n_f)]
        off = np.concatenate([[0], np.cumsum(n_s)]).astype(np.int32)
        return PolicyLayout(n_s, [6, 2, 4], n_w, n_f, off, int(off[-1]) + 2, fw=128, ft=0, ff=64, h=64, max_na=6)
    # three agents with the three grid shapes: corner / edge / interior (n_s 32 / 42 / 52)
    n_w = [6, 6, 6]
    n_f = [8, 12, 16] if ff else [0, 0, 0]
    n_wave = [18, 24, 30]
    n_s = [w + t + f for w, t, f in zip(n_wave, n_w, n_f)]
    off = np.concatenate([[0], np.cumsum(n_s)]).astype(np.int32)
    return PolicyLayout(n_s, [5, 4, 5], n_w, n_f, off, int(off[-1]) + 3, fw=128, ft=32, ff=ff, h=64, max_na=5)


def _ref_views(lay, P):
    return lay.views(torch.from_numpy(P.astype(np.float64)))


@pytest.mark.parametrize("ff", [64, 0, "monaco"])
def test_forward_matches_oracle(ff):
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from oracle.learner_ref import unit_forward
    lay = _layout(ff)
    R = 37
    m = BatchedA2C(lay, R, n_step=4, seed=3, allow_tf32=False, use_tc=False)
    P = m.P.cpu().numpy()
    # non-zero biases so that they are exercised
    P = P + np.random.default_rng(0).normal(0, 0.05, P.shape).astype(np.float32) * (P == 0)
    mask = np.ones_like(P)
    v = lay.views(mask)
    for u in range(lay.U):
        n_out = int(lay.n_a[u // 2]) if u % 2 == 0 else 1
        v["wo"][u][:, n_out:] = 0; v["bo"][u][n_out:] = 0
    P = P * mask
    m.P.copy_(torch.from_numpy(P))
    rng = np.random.default_rng(1)
    vr = _ref_views(lay, P)
    c = [torch.zeros(R, 64, dtype=torch.float64) for _ in range(lay.U)]
    h = [torch.zeros(R, 64, dtype=torch.float64) for _ in range(lay.U)]
    for step, done in enumerate([True, False, False, True, False]):
        obs = rng.random((R, lay.n_obs)).astype(np.float32) * 2
        pi, val, act = m.forward(torch.from_numpy(obs).cuda(), done)
        torch.cuda.synchronize()
        o64 = torch.from_numpy(obs.astype(np.float64))[None]
        for a in range(lay.A):
            p_ref, _, c[2 * a], h[2 * a] = unit_forward(vr, lay, 2 * a, o64, [float(done)], c[2 * a], h[2 * a])
            v_ref, _, c[2 * a + 1], h[2 * a + 1] = unit_forward(vr, lay, 2 * a + 1, o64, [float(done)], c[2 * a + 1], h[2 * a + 1])
            na = int(lay.n_a[a])
            np.testing.assert_allclose(pi[:, a, :na].cpu().numpy(), p_ref[0].numpy(), rtol=2e-4, atol=2e-5)
            assert float(pi[:, a, na:].abs().max()) == 0.0 if na < lay.max_na else True
            np.testing.assert_allclose(val[:, a].cpu().numpy(), v_ref[0].numpy(), rtol=2e-4, atol=2e-5)
            assert int(act[:, a].max()) < na and int(act[:, a].min()) >= 0
        # 'v' forward must not advance the recurrent state (agents/policies.py:127-135)
        cf = m.c_fw.clone()
        m.forward(torch.from_numpy(obs).cuda(), False, out_type="v")
        assert torch.equal(cf, m.c_fw)
    np.testing.assert_allclose(m.c_fw[1].cpu().numpy(), c[1].numpy(), rtol=2e-4, atol=2e-5)


def test_sampling_follows_policy():
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    lay = _layout(64)
    R = 4096
    m = BatchedA2C(lay, R, n_step=4, seed=5, use_tc=False)
    obs = torch.rand(1, lay.n_obs, device="cuda").expand(R, -1).contiguous()
    pi, val, act = m.forward(obs, True)
    torch.cuda.synchronize()
    for a in range(lay.A):
        p = pi[0, a].cpu().numpy()
        freq = np.bincount(act[:, a].cpu().numpy(), minlength=lay.max_na) / R
        assert np.abs(freq - p).max() < 0.03


@pytest.mark.parametrize("ff,chunk", [(64, 16), (0, 64), ("monaco", 37)])
def test_backward_gradients_match_autograd(ff, chunk):
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from oracle.learner_ref import a2c_loss, nstep_returns
    lay = _layout(ff)
    R, T = 37, 6
    gamma, v_coef, beta = 0.99, 0.5, 0.01
    m = BatchedA2C(lay, R, n_step=T, gamma=gamma, v_coef=v_coef, max_grad_norm=0.0, seed=7, chunk=chunk,
                   reward_norm=3.0, reward_clip=2.0, allow_tf32=False, use_tc=False)
    rng = np.random.default_rng(2)
    P0 = m.P.cpu().numpy().copy()
    # start the rollout from a non-zero recurrent state
    m.c_fw.copy_(torch.from_numpy(rng.normal(0, 0.3, tuple(m.c_fw.shape)).astype(np.float32)))
    m.h_fw.copy_(torch.tanh(m.c_fw) * 0.5)
    m.c_bw.copy_(m.c_fw); m.h_bw.copy_(m.h_fw)
    c0, h0 = m.c_bw.cpu().double(), m.h_bw.cpu().double()
    dones_pre = [0.0, 0.0, 1.0, 0.0, 0.0, 0.0]
    dones_post = dones_pre[1:] + [0.0]
    obs_all, act_all, rew_all, val_all = [], [], [], []
    for t in range(T):
        obs = rng.random((R, lay.n_obs)).astype(np.float32) * 2
        m.obs_slot().copy_(torch.from_numpy(obs))
        pi, val, act = m.forward(m.obs_slot(), bool(dones_pre[t]))
        rew = rng.normal(0, 4, (R, lay.A)).astype(np.float32)
        obs_all.append(obs); act_all.append(act.cpu().numpy().copy()); val_all.append(val.cpu().numpy().copy())
        rew_all.append(np.clip(rew / 3.0, -2.0, 2.0))
        m.add_transition(torch.from_numpy(rew).cuda(), bool(dones_pre[t]), bool(dones_post[t]))
    boot = rng.normal(0, 1, (R, lay.A)).astype(np.float32)
    m.backward(torch.from_numpy(boot).cuda(), lr=0.0, beta=beta)
    torch.cuda.synchronize()
    G = m.G.cpu().numpy().astype(np.float64)
    assert np.array_equal(m.P.cpu().numpy(), P0)               # lr = 0
    # returns kernel vs restatement (agents/utils.py:202-214)
    rew_np, val_np = np.stack(rew_all), np.stack(val_all)
    Rs_ref, Adv_ref = nstep_returns(list(rew_np.astype(np.float64)), list(val_np.astype(np.float64)), dones_post,
                                    boot.astype(np.float64), gamma)
    np.testing.assert_allclose(m.Rs.cpu().numpy(), Rs_ref, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(m.Adv.cpu().numpy(), Adv_ref, rtol=1e-5, atol=1e-5)
    # autograd oracle (float64)
    P = torch.from_numpy(P0.astype(np.float64)).requires_grad_(True)
    loss, parts = a2c_loss(P, lay, torch.from_numpy(np.stack(obs_all).astype(np.float64)),
                           torch.from_numpy(np.stack(act_all)), torch.from_numpy(m.Rs.cpu().numpy().astype(np.float64)),
                           torch.from_numpy(m.Adv.cpu().numpy().astype(np.float64)), dones_pre,
                           [c0[u] for u in range(lay.U)], [h0[u] for u in range(lay.U)], v_coef, beta)
    loss.backward()
    Gref = P.grad.numpy()
    gv, rv = lay.views(G), lay.views(Gref)
    for k in gv:
        if rv[k].size == 0:
            continue
        scale = max(np.abs(rv[k]).max(), 1e-8)
        err = np.abs(gv[k] - rv[k]).max() / scale
        assert err < 3e-4, (k, err, scale)
    st = m.stats.cpu().numpy()
    np.testing.assert_allclose(st[:3], np.array(parts[0]), rtol=1e-3, atol=1e-5)   # agent-0 summaries
    # states_bw refreshed from states_fw (agents/policies.py:153)
    assert torch.equal(m.c_bw, m.c_fw) and m.t == 0


def test_clip_rmsprop_matches_tf1_semantics():
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import BatchedA2C, _p
    from oracle.learner_ref import clip_rmsprop
    import ctypes as C
    lay = _layout(64)
    m = BatchedA2C(lay, 8, n_step=2, seed=1)
    rng = np.random.default_rng(4)
    G = rng.normal(0, 1.0, lay.n_params).astype(np.float32)
    G[lay.agent_of == 1] *= 1e-3                                  # agent 1 stays below the clip norm
    P0, MS0 = m.P.cpu().numpy().copy(), m.MS.cpu().numpy().copy()
    assert np.all(MS0 == 1.0)
    m.G.copy_(torch.from_numpy(G))
    for it in range(2):
        _lib.check(_lib.lib().tscl_clip_rmsprop(m._h, _p(m.P), _p(m.G), _p(m.MS), _p(m.agent_of), C.c_float(40.0),
                                                C.c_float(5e-4), C.c_float(0.99), C.c_float(1e-5), _p(m.norms), m._st()))
        P0, MS0, norms = clip_rmsprop(P0, G, MS0, lay.agent_of, 40.0, 5e-4, 0.99, 1e-5, lay.A)
    torch.cuda.synchronize()
    np.testing.assert_allclose(m.norms.cpu().numpy(), norms, rtol=1e-4)
    np.testing.assert_allclose(m.MS.cpu().numpy(), MS0, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(m.P.cpu().numpy(), P0, rtol=1e-5, atol=1e-6)
    assert norms[0] > 40.0 > norms[1]


def _fc_layout():
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    n_w, n_wave = [6, 6, 6], [18, 24, 30]
    n_s = [w + t for w, t in zip(n_wave, n_w)]
    off = np.concatenate([[0], np.cumsum(n_s)]).astype(np.int32)
    return PolicyLayout(n_s, [5, 4, 5], n_w, [0, 0, 0], off, int(off[-1]) + 3, fw=128, ft=32, ff=0, h=64, max_na=5,
                        recurrent=False)


def test_fc_policy_forward_and_gradients_match_oracle():
    """FcACPolicy (agents/policies.py:214-256, BASELINE config 2): forward vs the float64 restatement, gradients vs
    float64 autograd (rel. 3e-4 of each tensor's max), with the fp32 front-end gradient kernel and the wgmma one."""
    from deeprl_signal_control_b200.agents.learner_fc import BatchedFcA2C
    from oracle.learner_ref import a2c_loss, nstep_returns, unit_forward
    lay = _fc_layout()
    R, T = 37, 5
    gamma, v_coef, beta = 0.99, 0.5, 0.01
    for fc_tc in (False, True):
        m = BatchedFcA2C(lay, R, n_step=T, gamma=gamma, v_coef=v_coef, max_grad_norm=0.0, seed=7, chunk=16,
                         reward_norm=3.0, reward_clip=2.0, allow_tf32=False)
        m.fc_bwd_tc = fc_tc and lay.fc_bwd_tc_ok
        rng = np.random.default_rng(2)
        P0 = m.P.cpu().numpy().copy()
        P0 = P0 + rng.normal(0, 0.05, P0.shape).astype(np.float32) * (P0 == 0)       # non-zero biases
        mask = np.ones_like(P0); vm = lay.views(mask)
        for u in range(lay.U):
            n_out = int(lay.n_a[u // 2]) if u % 2 == 0 else 1
            vm["wo"][u][:, n_out:] = 0; vm["bo"][u][n_out:] = 0
        P0 = P0 * mask
        m.P.copy_(torch.from_numpy(P0))
        vr = lay.views(torch.from_numpy(P0.astype(np.float64)))
        dones_pre = [0.0, 1.0, 0.0, 0.0, 0.0]
        dones_post = dones_pre[1:] + [0.0]
        obs_all, act_all, rew_all, val_all = [], [], [], []
        for t in range(T):
            obs = rng.random((R, lay.n_obs)).astype(np.float32) * 2
            m.obs_slot().copy_(torch.from_numpy(obs))
            pi, val, act = m.forward(m.obs_slot(), bool(dones_pre[t]))
            torch.cuda.synchronize()
            o64 = torch.from_numpy(obs.astype(np.float64))[None]
            for a in range(lay.A):
                p_ref = unit_forward(vr, lay, 2 * a, o64, [0.0], None, None)[0]
                v_ref = unit_forward(vr, lay, 2 * a + 1, o64, [0.0], None, None)[0]
                na = int(lay.n_a[a])
                np.testing.assert_allclose(pi[:, a, :na].cpu().numpy(), p_ref[0].numpy(), rtol=2e-4, atol=2e-5)
                np.testing.assert_allclose(val[:, a].cpu().numpy(), v_ref[0].numpy(), rtol=2e-4, atol=2e-5)
                assert int(act[:, a].max()) < na and int(act[:, a].min()) >= 0
            rew = rng.normal(0, 4, (R, lay.A)).astype(np.float32)
            obs_all.append(obs); act_all.append(act.cpu().numpy().copy()); val_all.append(val.cpu().numpy().copy())
            rew_all.append(np.clip(rew / 3.0, -2.0, 2.0))
            m.add_transition(torch.from_numpy(rew).cuda(), bool(dones_pre[t]), bool(dones_post[t]))
        boot = rng.normal(0, 1, (R, lay.A)).astype(np.float32)
        m.backward(torch.from_numpy(boot).cuda(), lr=0.0, beta=beta)
        torch.cuda.synchronize()
        G = m.G.cpu().numpy().astype(np.float64)
        Rs_ref, Adv_ref = nstep_returns(list(np.stack(rew_all).astype(np.float64)), list(np.stack(val_all).astype(np.float64)),
                                        dones_post, boot.astype(np.float64), gamma)
        np.testing.assert_allclose(m.Rs.cpu().numpy(), Rs_ref, rtol=1e-5, atol=1e-5)
        P = torch.from_numpy(P0.astype(np.float64)).requires_grad_(True)
        zeros = [None] * lay.U
        loss, parts = a2c_loss(P, lay, torch.from_numpy(np.stack(obs_all).astype(np.float64)),
                               torch.from_numpy(np.stack(act_all)), torch.from_numpy(m.Rs.cpu().numpy().astype(np.float64)),
                               torch.from_numpy(m.Adv.cpu().numpy().astype(np.float64)), dones_pre, zeros, zeros, v_coef, beta)
        loss.backward()
        gv, rv = lay.views(G), lay.views(P.grad.numpy())
        tol = 2e-2 if m.fc_bwd_tc else 3e-4           # the wgmma kernel multiplies bf16-rounded operands
        for k in gv:
            if rv[k].size == 0 or (m.fc_bwd_tc and not k.startswith("fc")):
                continue
            scale = max(np.abs(rv[k]).max(), 1e-8)
            assert np.abs(gv[k] - rv[k]).max() / scale < tol, (k, fc_tc)
        assert m.t == 0
