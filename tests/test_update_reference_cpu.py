"""CPU: the float64 reference of the tensor-core update from the activation store (oracle/learner_ref.py: heads_ref,
bptt_ref, lstm_grads_ref, fc_grads_ref, update_ref) is itself right, and a comparison against it can see the defects a
BPTT kernel can plausibly have.

With round_bf16=False and the store taken from the float64 forward, the chained reference must equal autograd of
a2c_loss (the restatement of agents/policies.py:41-52 that the reference goldens pin) to 1e-9 per tensor: several
chunks with r0 > 0, per-replica initial states, done at t = 0, inside the rollout and at t = T-1, and one row whose taken
action has pi < 1e-10, where the TF clip makes the policy gradient of that row zero."""
import numpy as np
import pytest
import torch

from oracle.learner_ref import a2c_loss, bptt_mutations, bptt_ref, store_forward, update_ref
from tests.test_learner_gpu import _layout
from tests.test_update_bench_size_gpu import DZ_REL_L2, dz_errors     # the GPU comparison of dZ


def _problem(lay, R, T, dones, seed):
    """Parameters (nonzero biases, wide policy heads), per-replica initial states, observations, float64 store."""
    rng = np.random.default_rng(seed)
    P = lay.init_params(seed).astype(np.float64)
    v = lay.views(P)
    for k in ("bl", "bo"):
        v[k][...] = rng.normal(0, 0.1, v[k].shape)
    for u in range(lay.U):
        v["fcw_b%d" % u][...] = rng.normal(0, 0.1, lay.fw)
        n_out = int(lay.n_a[u // 2]) if u % 2 == 0 else 1
        v["wo"][u][:, :n_out] = rng.normal(0, 0.2 if u % 2 else 3.0, (lay.h, n_out))     # logits spread over ~1e-20 .. 1
        v["wo"][u][:, n_out:] = 0.0
        v["bo"][u][n_out:] = 0.0
    P = torch.from_numpy(P)
    c0 = torch.from_numpy(rng.normal(0, 0.5, (lay.U, R, lay.h)))
    h0 = torch.tanh(torch.from_numpy(rng.normal(0, 0.7, (lay.U, R, lay.h))))
    obs = torch.from_numpy(rng.random((T, R, lay.n_obs)) * 2)
    vt = lay.views(P)
    st = [store_forward(vt, lay, u, obs, dones, c0[u], h0[u]) for u in range(lay.U)]
    store = [torch.stack([s[k] for s in st]) for k in range(4)]           # X, gates, c, h: [U][T][R][w]
    return P, c0, h0, obs, store, rng


@pytest.mark.parametrize("ff", [64, 0, "monaco"])
def test_reference_update_equals_autograd(ff):
    lay = _layout(ff)
    R, T, chunk = 11, 6, 4                      # chunks r0 = 0, 4, 8 (the last one ragged)
    dones = [1.0, 0.0, 0.0, 1.0, 0.0, 1.0]
    v_coef, beta = 0.5, 0.01
    P, c0, h0, obs, store, rng = _problem(lay, R, T, dones, seed=3 + (ff == 0))
    acts = np.stack([rng.integers(0, int(na), (T, R)) for na in lay.n_a], -1).astype(np.int32)   # [T, R, A]
    # one row whose taken action has pi < 1e-10: forward pi of agent 0 from the float64 store
    # (a bias of -40 on action 1 of agent 0; the store does not depend on the heads)
    v = lay.views(P)
    v["bo"][0][1] = -40.0
    H = store[3][0]                                                     # agent 0's policy unit, [T][R][h]
    pi = torch.softmax(H @ v["wo"][0][:, :int(lay.n_a[0])] + v["bo"][0][:int(lay.n_a[0])], -1)
    t_, r_ = 2, 6
    acts[t_, r_, 0] = 1
    assert float(pi[t_, r_, 1]) < 1e-10
    Rs = torch.from_numpy(rng.normal(0, 2, (T, R, lay.A)))
    Adv = torch.from_numpy(rng.normal(0, 2, (T, R, lay.A)))
    Adv[t_, r_, 0] = 5.0                                                # that row would move the gradient a lot
    act = torch.from_numpy(acts)
    scale = 1.0 / (T * R)

    def chunk_store(ci):
        r0 = ci * chunk
        return tuple(s[:, :, r0:r0 + chunk] for s in store)
    G, stats = update_ref(lay, P, chunk_store, obs, act, Rs, Adv, c0, h0, dones, scale, v_coef, beta, chunk,
                          round_bf16=False, agents_per_group=2)
    Pg = P.clone().requires_grad_(True)
    loss, parts = a2c_loss(Pg, lay, obs, act, Rs, Adv, dones, list(c0), list(h0), v_coef, beta)
    loss.backward()
    gv, rv = lay.views(G), lay.views(Pg.grad)
    for k in rv:
        if rv[k].numel() == 0:
            continue
        ref = float(rv[k].abs().max())
        err = float((gv[k] - rv[k]).abs().max())
        assert err <= 1e-9 * max(ref, 1e-300), (k, err, ref)
        assert (ref > 0) or err == 0.0, k
    np.testing.assert_allclose(stats.numpy(), np.array(parts[0]), rtol=1e-12)
    # the bf16-rounding variant (what the GPU tests compare with) stays within bf16 noise of the exact gradient
    Gb, _ = update_ref(lay, P, chunk_store, obs, act, Rs, Adv, c0, h0, dones, scale, v_coef, beta, chunk)
    rel = float((Gb - G).norm() / G.norm())
    assert 1e-5 < rel < 2e-2, rel


def test_bptt_comparison_sees_planted_defects():
    """Each planted defect moves the reference dZ (rel-L2 per unit and step, worst case) by at least 10x the bound of the
    GPU comparison."""
    lay = _layout(64)
    R, T, r0 = 12, 8, 5
    dones = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 1.0, 0.0]
    P, c0, h0, obs, store, rng = _problem(lay, R, T, dones, seed=11)
    v = lay.views(P)
    rc = 6
    us = slice(0, 4)
    gates, c = store[1][us, :, r0:r0 + rc], store[2][us, :, r0:r0 + rc]
    dH = torch.from_numpy(rng.normal(0, 1e-2, (4, T, rc, lay.h)))
    ok, mutants = bptt_mutations(gates, c, c0[us], r0, dH, dones)
    for round_bf16 in (False, True):
        dz = bptt_ref(**ok, wh=v["wh"][us], round_bf16=round_bf16)
        for name, kw in mutants.items():
            dzm = bptt_ref(**kw, wh=v["wh"][us], round_bf16=round_bf16)
            rel = dz_errors(dzm, dz)[0]
            assert rel > 10 * DZ_REL_L2, (name, rel)
