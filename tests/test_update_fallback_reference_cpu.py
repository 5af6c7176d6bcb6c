"""CPU: the float64 references of the two update paths that do not read the activation store are themselves right, and a
comparison against them can see the defects those paths can plausibly have.

  * the recompute update (BatchedA2C.backward with store_acts off): update_ref over the float64 forward of each agent
    group (store_group, store_units=True), with the recompute path's rounding (round_operands, dx_product);
  * the FcACPolicy update (BatchedFcA2C.backward): fc_update_ref.

With all rounding off both must equal autograd of a2c_loss to 1e-9 per tensor: several chunks with r0 > 0 and a ragged
last one, per-replica initial states, done at t = 0, inside the rollout and at t = T-1.  With the rounding on they stay
within bf16 noise of the exact gradient.  Every planted defect (recompute_mutations, FC_DEFECTS) moves G by at least 10x
the bound the GPU comparison is judged by (tests/update_fallback_bounds.py)."""
import numpy as np
import pytest
import torch

from oracle.learner_ref import (FC_DEFECTS, a2c_loss, fc_update_ref, recompute_mutations, store_group, update_ref)
from tests.test_learner_gpu import _layout
from tests.update_fallback_bounds import FC_G_REL_L2, RECOMPUTE_G_REL_L2_FP32

R, T, CHUNK = 11, 6, 4                          # chunks r0 = 0, 4, 8 (the last one ragged)
DONES = [1.0, 0.0, 0.0, 1.0, 0.0, 1.0]
V_COEF, BETA = 0.5, 0.01


def _fc_layout(ff):
    """FcACPolicy layout with the three grid agent shapes (corner / edge / interior), with or without fingerprints."""
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    n_w, n_wave = [6, 6, 6], [18, 24, 30]
    n_f = [8, 12, 16] if ff else [0, 0, 0]
    n_s = [w + t + f for w, t, f in zip(n_wave, n_w, n_f)]
    off = np.concatenate([[0], np.cumsum(n_s)]).astype(np.int32)
    return PolicyLayout(n_s, [5, 4, 5], n_w, n_f, off, int(off[-1]) + 3, fw=128, ft=32, ff=ff, h=64, max_na=5,
                        recurrent=False)


def _problem(lay, seed):
    """Parameters (nonzero biases, wide policy heads), per-replica initial states, T + 1 observation slots, actions,
    returns and advantages, all float64 on the CPU."""
    rng = np.random.default_rng(seed)
    P = lay.init_params(seed).astype(np.float64)
    v = lay.views(P)
    for k in ("bl", "bo"):
        v[k][...] = rng.normal(0, 0.1, v[k].shape)
    for u in range(lay.U):
        v["fcw_b%d" % u][...] = rng.normal(0, 0.1, lay.fw)
        n_out = int(lay.n_a[u // 2]) if u % 2 == 0 else 1
        v["wo"][u][:, n_out:] = 0.0
        v["bo"][u][n_out:] = 0.0
        v["wo"][u][:, :n_out] = rng.normal(0, 0.2 if u % 2 else 1.0, (lay.h, n_out))
    P = torch.from_numpy(P)
    c0 = torch.from_numpy(rng.normal(0, 0.5, (lay.U, R, lay.h)))
    h0 = torch.tanh(torch.from_numpy(rng.normal(0, 0.7, (lay.U, R, lay.h))))
    obs = torch.from_numpy(rng.random((T + 1, R, lay.n_obs)) * 2)
    act = torch.from_numpy(np.stack([rng.integers(0, int(na), (T, R)) for na in lay.n_a], -1).astype(np.int32))
    Rs = torch.from_numpy(rng.normal(0, 2, (T, R, lay.A)))
    Adv = torch.from_numpy(rng.normal(0, 2, (T, R, lay.A)))
    return P, c0, h0, obs, act, Rs, Adv


def _autograd(lay, P, obs, act, Rs, Adv, c0, h0):
    Pg = P.clone().requires_grad_(True)
    cs = list(c0) if c0 is not None else [None] * lay.U
    hs = list(h0) if h0 is not None else [None] * lay.U
    loss, parts = a2c_loss(Pg, lay, obs[:T], act, Rs, Adv, DONES, cs, hs, V_COEF, BETA)
    loss.backward()
    return Pg.grad, parts


def _assert_per_tensor(lay, G, ref):
    gv, rv = lay.views(G), lay.views(ref)
    for k in rv:
        if rv[k].numel() == 0:
            continue
        r = float(rv[k].abs().max())
        err = float((gv[k] - rv[k]).abs().max())
        assert err <= 1e-9 * max(r, 1e-300), (k, err, r)
        assert r > 0 or err == 0.0, k


def _recompute_store(lay, P, fwd_of_chunk):
    """store(ci, us) of update_ref: the float64 forward of the units `us` from the forward inputs of chunk ci."""
    v = lay.views(P.to(torch.float64))
    return lambda ci, us: store_group(v, lay, us, **fwd_of_chunk(ci))


def _recompute_G(lay, P, obs, act, Rs, Adv, c0, h0, fwd_of_chunk, dones=DONES, **kw):
    return update_ref(lay, P, _recompute_store(lay, P, fwd_of_chunk), obs[:T], act, Rs, Adv, c0, h0, dones, 1.0 / (T * R),
                      V_COEF, BETA, CHUNK, agents_per_group=2, store_units=True, **kw)


@pytest.mark.parametrize("ff", [64, 0, "monaco"])
def test_recompute_reference_equals_autograd(ff):
    lay = _layout(ff)
    P, c0, h0, obs, act, Rs, Adv = _problem(lay, seed=5 + (ff == 0))
    fwd = lambda ci: recompute_mutations(obs, c0, h0, DONES, ci * CHUNK, min(CHUNK, R - ci * CHUNK))[0]
    G, stats = _recompute_G(lay, P, obs, act, Rs, Adv, c0, h0, fwd, round_bf16=False)
    ref, parts = _autograd(lay, P, obs, act, Rs, Adv, c0, h0)
    _assert_per_tensor(lay, G, ref)
    np.testing.assert_allclose(stats.numpy(), np.array(parts[0]), rtol=1e-12)
    # the store asked for per (chunk, unit group) gives the bits of the whole-chunk store of the same forward
    v = lay.views(P)
    whole = lambda ci: store_group(v, lay, slice(0, lay.U), **fwd(ci))
    Gw, _ = update_ref(lay, P, whole, obs[:T], act, Rs, Adv, c0, h0, DONES, 1.0 / (T * R), V_COEF, BETA, CHUNK,
                       agents_per_group=2)
    Gu, _ = _recompute_G(lay, P, obs, act, Rs, Adv, c0, h0, fwd)
    assert torch.equal(Gw, Gu)
    # the recompute path's rounding (fp32 / TF32 dX product, bf16 X / Hp operands) stays within bf16 noise of the exact
    # gradient and differs from the store path's rounding
    for dx_product in ("fp32", "tf32"):
        Gr, _ = _recompute_G(lay, P, obs, act, Rs, Adv, c0, h0, fwd, round_operands=True, dx_product=dx_product)
        rel = float((Gr - G).norm() / G.norm())
        assert 1e-5 < rel < 2e-2, (dx_product, rel)
        assert not torch.equal(Gr, Gu)


@pytest.mark.parametrize("ff", [0, 64])
def test_fc_reference_equals_autograd(ff):
    lay = _fc_layout(ff)
    P, _, _, obs, act, Rs, Adv = _problem(lay, seed=9 + ff)
    G, stats = fc_update_ref(lay, P, obs[:T], act, Rs, Adv, 1.0 / (T * R), V_COEF, BETA, CHUNK)
    ref, parts = _autograd(lay, P, obs, act, Rs, Adv, None, None)
    _assert_per_tensor(lay, G, ref)
    np.testing.assert_allclose(stats.numpy(), np.array(parts[0]), rtol=1e-12)
    Gb, _ = fc_update_ref(lay, P, obs[:T], act, Rs, Adv, 1.0 / (T * R), V_COEF, BETA, CHUNK, round_bf16=True)
    rel = float((Gb - G).norm() / G.norm())
    assert 1e-6 < rel < 2e-2, rel


def test_recompute_comparison_sees_planted_defects():
    """Each planted defect of the recompute forward moves G (rel-L2, rounding as on the GPU with fp32 products, where the
    GPU check of these defects runs) by >= 10x the fp32 GPU bound.
    No done at t = 0 here: it would hide the initial state."""
    lay = _layout(64)
    P, c0, h0, obs, act, Rs, Adv = _problem(lay, seed=13)
    dones = [0.0, 0.0, 1.0, 0.0, 0.0, 1.0]
    muts = lambda ci: recompute_mutations(obs, c0, h0, dones, ci * CHUNK, min(CHUNK, R - ci * CHUNK))
    kw = dict(round_operands=True, dx_product="fp32", dones=dones)
    G, _ = _recompute_G(lay, P, obs, act, Rs, Adv, c0, h0, lambda ci: muts(ci)[0], **kw)
    names = list(muts(0)[1])
    assert len(names) == 4
    for name in names:
        Gm, _ = _recompute_G(lay, P, obs, act, Rs, Adv, c0, h0, lambda ci: muts(ci)[1][name], **kw)
        rel = float((Gm - G).norm() / G.norm())
        assert rel >= 10 * RECOMPUTE_G_REL_L2_FP32, (name, rel)


def test_fc_comparison_sees_planted_defects():
    lay = _fc_layout(0)
    P, _, _, obs, act, Rs, Adv = _problem(lay, seed=17)
    args = (lay, P, obs[:T], act, Rs, Adv, 1.0 / (T * R), V_COEF, BETA, CHUNK)
    G, _ = fc_update_ref(*args, round_bf16=True)
    for name in FC_DEFECTS:
        Gm, _ = fc_update_ref(*args, round_bf16=True, defect=name)
        rel = float((Gm - G).norm() / G.norm())
        assert rel >= 10 * FC_G_REL_L2, (name, rel)
