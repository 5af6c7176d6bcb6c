"""GPU: the fused wgmma policy-forward kernel (tscl_policy_step) vs the fp32 kernels / the oracle.

The tensor-core path multiplies bf16-rounded operands with fp32 accumulation, so
  * raw gate accumulators are compared with a torch matmul of the SAME bf16-rounded operands
    (rtol 1e-3, atol 2e-3: only the summation order differs);
  * policy / value / state are compared with the fp32 SIMT path at atol 3e-2 (bf16 operand rounding)."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _layout(ff):
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    if ff == "monaco":
        # Monaco shapes (real_net): no wait block (ft = 0, dx = 192), up to 34 wave inputs -> 48|16 input tile
        n_w, n_f, n_wave = [0, 0, 0], [16, 4, 9], [34, 5, 33]
        n_s = [w + f for w, f in zip(n_wave, n_f)]
        off = np.concatenate([[0], np.cumsum(n_s)]).astype(np.int32)
        return PolicyLayout(n_s, [6, 2, 4], n_w, n_f, off, int(off[-1]) + 2, fw=128, ft=0, ff=64, h=64, max_na=6)
    n_w = [6, 6, 6]
    n_f = [8, 12, 16] if ff else [0, 0, 0]
    n_wave = [18, 24, 30]
    n_s = [w + t + f for w, t, f in zip(n_wave, n_w, n_f)]
    off = np.concatenate([[0], np.cumsum(n_s)]).astype(np.int32)
    return PolicyLayout(n_s, [5, 4, 5], n_w, n_f, off, int(off[-1]) + 3, fw=128, ft=32, ff=ff, h=64, max_na=5)


def _run_tc(m, obs, done, zdbg, swap, v2=False):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    args = (m._h, _p(m.P), _p(m.Wp), _p(obs), C.c_int64(m.R), _p(m.c_fw), _p(m.h_fw), _p(m.c_tmp), _p(m.h_tmp),
            _p(m.pi), _p(m.val), _p(m.act), C.c_int32(int(done)), C.c_uint64(7), C.c_int64(0), C.c_int64(0), _p(zdbg))
    if v2:
        _lib.check(_lib.lib().tscl_policy_step_v2(*args, None, None, None, None, C.c_int32(0), C.c_int32(1), C.c_int64(0), m._st()))
    else:
        _lib.check(_lib.lib().tscl_policy_step(*args, C.c_int32(swap), m._st()))
    torch.cuda.synchronize()


@pytest.mark.parametrize("ff", [64, 0, "monaco"])
def test_gate_accumulators_match_bf16_matmul(ff):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import BatchedA2C, _p
    lay = _layout(ff)
    R = 300                                     # 2 full tiles + a ragged one
    m = BatchedA2C(lay, R, n_step=2, seed=11)
    rng = np.random.default_rng(0)
    m.h_fw.copy_(torch.from_numpy(rng.uniform(-1, 1, tuple(m.h_fw.shape)).astype(np.float32)))
    m.c_fw.copy_(torch.from_numpy(rng.normal(0, 0.5, tuple(m.c_fw.shape)).astype(np.float32)))
    obs = torch.from_numpy((rng.random((R, lay.n_obs)) * 2).astype(np.float32)).cuda()
    # reference operands: X from the fp32 fc kernel, rounded to bf16 exactly like the fused kernel does
    _lib.check(_lib.lib().tscl_fc_embed(m._h, _p(m.P), _p(obs), C.c_int64(R), C.c_int64(R), C.c_int64(0), _p(m.X1), m._st()))
    Xb = m.X1.to(torch.bfloat16).float()
    Hb = m.h_fw.to(torch.bfloat16).float()
    Wx = m.pv["wx"].to(torch.bfloat16).float()
    Wh = m.pv["wh"].to(torch.bfloat16).float()
    torch.backends.cuda.matmul.allow_tf32 = False
    z_ref = torch.bmm(Xb, Wx) + torch.bmm(Hb, Wh)
    zdbg = torch.zeros(lay.U, R, 256, device="cuda")
    if ff == "monaco":                          # v1 keeps the 32-wide wave block and must say so
        with pytest.raises(RuntimeError, match="wave widths"):
            _run_tc(m, obs, False, zdbg, 0)
    else:
        _check_v1(m, obs, zdbg, z_ref, Xb, Wx)
    _check_v2(m, lay, obs, zdbg, Hb, Wx, Wh)


def _check_v1(m, obs, zdbg, z_ref, Xb, Wx):
    _run_tc(m, obs, False, zdbg, 0)
    err0 = float((zdbg - z_ref).abs().max())
    if err0 > 5e-2:                             # diagnose a descriptor-stride mix-up in one GPU run
        z1 = torch.zeros_like(zdbg)
        _run_tc(m, obs, False, z1, 1)
        err1 = float((z1 - z_ref).abs().max())
        raise AssertionError("wgmma gate GEMM mismatch: max err %.4f (LBO/SBO swapped: %.4f)" % (err0, err1))
    torch.testing.assert_close(zdbg, z_ref, rtol=1e-3, atol=2e-3)
    # done flag zeroes h and c inside the cell (agents/utils.py:104-105)
    _run_tc(m, obs, True, zdbg, 0)
    torch.testing.assert_close(zdbg, torch.bmm(Xb, Wx), rtol=1e-3, atol=2e-3)


def _check_v2(m, lay, obs, zdbg, Hb, Wx, Wh):
    # v2 (fc front end on the tensor cores): reference with bf16-rounded observations and fc weights
    v = lay.views(m.P)
    Xs = []
    for u in range(lay.U):
        a = u // 2
        o0 = int(lay.obs_off[a]); nw, nt, nf = int(lay.n_wave[a]), int(lay.n_wait[a]), int(lay.n_fp[a])
        ob = obs.to(torch.bfloat16).float()
        parts = [torch.relu(ob[:, o0:o0 + nw] @ v["fcw_w%d" % u].to(torch.bfloat16).float() + v["fcw_b%d" % u])]
        if lay.ff > 0:
            parts.append(torch.relu(ob[:, o0 + nw + nt:o0 + nw + nt + nf] @ v["fcf_w%d" % u].to(torch.bfloat16).float() + v["fcf_b%d" % u]))
        if lay.ft > 0:
            parts.append(torch.relu(ob[:, o0 + nw:o0 + nw + nt] @ v["fct_w%d" % u].to(torch.bfloat16).float() + v["fct_b%d" % u]))
        Xs.append(torch.cat(parts, 1))
    X2 = torch.stack(Xs).to(torch.bfloat16).float()
    z2_ref = torch.bmm(X2, Wx) + torch.bmm(Hb, Wh)
    z2 = torch.zeros_like(zdbg)
    _run_tc(m, obs, False, z2, 0, v2=True)
    # a bf16 rounding flip of one X element moves z by <= |w| * 2^-8 * |x|: allow a few of them
    assert float((z2 - z2_ref).abs().max()) < 4e-2, float((z2 - z2_ref).abs().max())
    assert float((z2 - z2_ref).abs().mean()) < 2e-3


@pytest.mark.parametrize("ff", [64, 0, "monaco"])
def test_fused_forward_matches_fp32_path(ff):
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    lay = _layout(ff)
    R = 515
    a = BatchedA2C(lay, R, n_step=2, seed=3, use_tc=True)
    b = BatchedA2C(lay, R, n_step=2, seed=3, use_tc=False, allow_tf32=False)
    assert a.use_tc and torch.equal(a.P, b.P)
    rng = np.random.default_rng(1)
    for step, done in enumerate([True, False, False, True, False, False]):
        obs = torch.from_numpy((rng.random((R, lay.n_obs)) * 2).astype(np.float32)).cuda()
        pa, va, aa = a.forward(obs, done)
        pb, vb, ab = b.forward(obs, done)
        torch.cuda.synchronize()
        torch.testing.assert_close(pa, pb, rtol=0, atol=3e-2)
        torch.testing.assert_close(va, vb, rtol=0, atol=5e-2)
        torch.testing.assert_close(a.h_fw, b.h_fw, rtol=0, atol=3e-2)
        torch.testing.assert_close(a.c_fw, b.c_fw, rtol=0, atol=6e-2)
        assert int(aa.min()) >= 0 and all(int(aa[:, i].max()) < int(lay.n_a[i]) for i in range(lay.A))
        np.testing.assert_allclose(pa.sum(-1).cpu().numpy(), 1.0, rtol=1e-5)
        # value-only forward leaves the recurrent state untouched
        cf = a.c_fw.clone()
        a.forward(obs, False, out_type="v")
        assert torch.equal(cf, a.c_fw)
        # keep the two models on the same trajectory
        a.c_fw.copy_(b.c_fw); a.h_fw.copy_(b.h_fw)
    # identical probabilities -> identical inverse-CDF samples wherever u is not within the bf16 error of a boundary
    assert float((aa == ab).float().mean()) > 0.97


def test_update_from_stored_activations_matches_recompute():
    """The update that back-propagates through the rollout's stored bf16 activations must agree with the
    update that recomputes the forward pass (same rollout, same parameters) within bf16 noise."""
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    lay = _layout(64)
    R, T = 200, 6
    kw = dict(n_step=T, gamma=0.99, v_coef=0.5, max_grad_norm=0.0, seed=9, chunk=100, reward_norm=2.0,
              reward_clip=2.0, allow_tf32=False)
    a = BatchedA2C(lay, R, use_tc=True, store_acts=True, **kw)
    b = BatchedA2C(lay, R, use_tc=True, store_acts=False, **kw)
    assert a.store_acts and not b.store_acts
    rng = np.random.default_rng(5)
    dones = [True, False, False, True, False, False]
    for t in range(T):
        obs = torch.from_numpy((rng.random((R, lay.n_obs)) * 2).astype(np.float32)).cuda()
        rew = torch.from_numpy(rng.normal(0, 3, (R, lay.A)).astype(np.float32)).cuda()
        for m in (a, b):
            m.obs_slot().copy_(obs)
            m.forward(m.obs_slot(), dones[t])
            m.add_transition(rew, dones[t], dones[t + 1] if t + 1 < T else False)
    assert torch.equal(a.act_hist, b.act_hist)
    boot = torch.from_numpy(rng.normal(0, 1, (R, lay.A)).astype(np.float32)).cuda()
    a.backward(boot, lr=0.0, beta=0.01); b.backward(boot, lr=0.0, beta=0.01)
    torch.cuda.synchronize()
    ga, gb = lay.views(a.G.cpu().numpy()), lay.views(b.G.cpu().numpy())
    worst = 1.0
    for k in ga:
        if gb[k].size < 8:
            continue
        x, y = ga[k].ravel().astype(np.float64), gb[k].ravel().astype(np.float64)
        if np.linalg.norm(y) < 1e-12:
            continue
        cos = float(x @ y / (np.linalg.norm(x) * np.linalg.norm(y) + 1e-30))
        rel = float(np.linalg.norm(x - y) / np.linalg.norm(y))
        worst = min(worst, cos)
        assert cos > 0.99 and rel < 0.12, (k, cos, rel)      # per-tensor: bf16 activations vs fp32 recompute
    va, vb = a.G.flatten().double(), b.G.flatten().double()
    assert float(torch.dot(va, vb) / (va.norm() * vb.norm())) > 0.999
    assert float((va - vb).norm() / vb.norm()) < 0.03


def test_bptt_tensor_core_kernel_matches_fp32_kernel():
    """tscl_lstm_seq_bwd_tc (wgmma dz.Wh^T, bf16 operands) vs tscl_lstm_seq_bwd (fp32 SIMT) on the same inputs."""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import BatchedA2C, _p
    lay = _layout(64)
    Rc, T, R = 150, 7, 300
    m = BatchedA2C(lay, R, n_step=T, seed=2)
    U = lay.U
    g = torch.Generator(device="cuda").manual_seed(0)
    gates = torch.rand(U, T * Rc, 256, device="cuda", generator=g)
    gates[..., 192:] = gates[..., 192:] * 2 - 1                      # u gate in (-1, 1)
    Cc = torch.randn(U, T * Rc, 64, device="cuda", generator=g) * 0.7
    dH = torch.randn(U, T * Rc, 64, device="cuda", generator=g) * 1e-3
    m.c_bw.copy_(torch.randn(U, R, 64, device="cuda", generator=g) * 0.5)
    done = torch.tensor([0, 0, 0, 1, 0, 0, 0], dtype=torch.float32, device="cuda")
    r0 = 100
    z1, z2 = gates.clone(), gates.clone()
    lib = _lib.lib()
    _lib.check(lib.tscl_lstm_seq_bwd(m._h, _p(m.P), _p(z1), _p(Cc), _p(dH), _p(m.c_bw), _p(done), C.c_int32(T),
                                     C.c_int64(Rc), C.c_int64(R), C.c_int64(r0), m._st()))
    _lib.check(lib.tscl_lstm_seq_bwd_tc(m._h, _p(m.Wt), _p(z2), _p(Cc), _p(dH), _p(m.c_bw), _p(done), C.c_int32(T),
                                        C.c_int64(Rc), C.c_int64(R), C.c_int64(r0), None, None, None, m._st()))
    # same again with gates / c read from bf16 copies (the activation-store fast path)
    z3 = torch.zeros_like(gates)
    gb, cb = gates.to(torch.bfloat16).contiguous(), Cc.to(torch.bfloat16).contiguous()
    _lib.check(lib.tscl_lstm_seq_bwd_tc(m._h, _p(m.Wt), _p(z3), None, _p(dH), _p(m.c_bw), _p(done), C.c_int32(T),
                                        C.c_int64(Rc), C.c_int64(R), C.c_int64(r0), _p(gb), _p(cb), None, m._st()))
    # ... and with dZ written as bf16 only (no fp32 output at all)
    z4 = torch.zeros(U, T * Rc, 256, dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.tscl_lstm_seq_bwd_tc(m._h, _p(m.Wt), None, None, _p(dH), _p(m.c_bw), _p(done), C.c_int32(T),
                                        C.c_int64(Rc), C.c_int64(R), C.c_int64(r0), _p(gb), _p(cb), _p(z4), m._st()))
    torch.cuda.synchronize()
    assert torch.equal(z4, z3.to(torch.bfloat16))
    assert float((z3 - z1).norm() / z1.norm()) < 2e-2
    assert torch.isfinite(z2).all()
    scale = float(z1.abs().max())
    err = float((z1 - z2).abs().max()) / scale
    rel = float((z1 - z2).norm() / z1.norm())
    assert err < 3e-2 and rel < 1e-2, (err, rel)
    # the last time step has no recurrent carry: identical up to tanh.approx
    last = slice((T - 1) * Rc, T * Rc)
    assert float((z1[:, last] - z2[:, last]).abs().max()) / scale < 2e-3


@pytest.mark.parametrize("ff,use_bf16_x", [(64, True), (0, False), ("monaco", True)])
def test_fc_weight_gradients_tensor_core_kernel(ff, use_bf16_x):
    """tscl_fc_bwd_tc (wgmma, MN-major bf16 operands, reduction over rows) vs
      * a float64 contraction of the SAME bf16-rounded operands (rtol 2e-3: only summation order differs), and
      * tscl_fc_bwd (fp32 SIMT kernel) within the bf16 operand rounding."""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import BatchedA2C, _p
    lay = _layout(ff)
    assert lay.fc_bwd_tc_ok
    T, Rc, R = 5, 333, 400                        # M = 1665 rows: 13 full tiles + a ragged one, chunk at r0 = 40
    m = BatchedA2C(lay, R, n_step=T, seed=4)
    U, M, dx = lay.U, T * Rc, lay.dx
    g = torch.Generator(device="cuda").manual_seed(1)
    obs = torch.rand(T, R, lay.n_obs, device="cuda", generator=g) * 2
    X = torch.relu(torch.randn(U, M, dx, device="cuda", generator=g))
    Xb = X.to(torch.bfloat16).contiguous()
    X = Xb.float()                                 # same mask on both paths
    dXb = (torch.randn(U, M, dx, device="cuda", generator=g) * 1e-2).to(torch.bfloat16).contiguous()
    dX = dXb.float()                               # bf16-representable, so the bf16 and fp32 inputs are the same numbers
    r0 = 40
    obs0 = obs[0, r0:]
    lib = _lib.lib()
    G1, G2 = torch.zeros_like(m.G), torch.zeros_like(m.G)
    _lib.check(lib.tscl_fc_bwd(m._h, _p(obs0), _p(X), _p(dX), C.c_int64(M), C.c_int64(Rc), C.c_int64(R * lay.n_obs),
                               _p(G1), m._st()))

    def run(variant, out):
        _lib.check(lib.tscl_fc_bwd_tc(m._h, _p(obs0), None if use_bf16_x else _p(X), _p(Xb) if use_bf16_x else None,
                                      None if use_bf16_x else _p(dX), _p(dXb) if use_bf16_x else None, C.c_int64(M),
                                      C.c_int64(Rc), C.c_int64(R * lay.n_obs), _p(out), C.c_int32(variant), m._st()))
        torch.cuda.synchronize()
    run(0, G2)
    g1, g2 = lay.views(G1.cpu().numpy()), lay.views(G2.cpu().numpy())
    # float64 reference from bf16-rounded operands
    ob = obs[:, r0:r0 + Rc].reshape(M, lay.n_obs).to(torch.bfloat16).double()
    dXm = (dX * (X > 0)).to(torch.bfloat16).double()
    worst = 0.0
    for u in range(U):
        a = u // 2
        o0, nw, nt, nf = int(lay.obs_off[a]), int(lay.n_wave[a]), int(lay.n_wait[a]), int(lay.n_fp[a])
        blocks = [("fcw", ob[:, o0:o0 + nw], dXm[u][:, :lay.fw])]
        c0 = lay.fw
        if lay.ff > 0:
            blocks.append(("fcf", ob[:, o0 + nw + nt:o0 + nw + nt + nf], dXm[u][:, c0:c0 + lay.ff])); c0 += lay.ff
        if lay.ft > 0:
            blocks.append(("fct", ob[:, o0 + nw:o0 + nw + nt], dXm[u][:, c0:c0 + lay.ft]))
        for name, inp, dd in blocks:
            w_ref = (inp.T @ dd).cpu().numpy()
            b_ref = dd.sum(0).cpu().numpy()
            w_tc, b_tc = g2["%s_w%d" % (name, u)], g2["%s_b%d" % (name, u)]
            e = max(np.abs(w_tc - w_ref).max() / max(np.abs(w_ref).max(), 1e-12),
                    np.abs(b_tc - b_ref).max() / max(np.abs(b_ref).max(), 1e-12))
            worst = max(worst, e)
    if worst > 2e-3:                               # diagnose a descriptor-stride mix-up in one GPU run
        G3 = torch.zeros_like(m.G)
        run(1, G3)
        raise AssertionError("wgmma MN-major fc_bwd mismatch: worst rel err %.4f (LBO/SBO swapped: rel-L2 vs fp32 %.4f)"
                             % (worst, float((G3 - G1).norm() / G1.norm())))
    # untouched parameter ranges stay zero, and the fp32 kernel agrees within bf16 operand rounding
    for k in g1:
        if not k.startswith("fc"):
            assert not g2[k].any()
    rel = float((G2 - G1).norm() / G1.norm())
    assert rel < 1e-2, rel


@pytest.mark.parametrize("ff,from_store", [(64, True), (0, False), ("monaco", True)])
def test_lstm_weight_gradients_tensor_core_kernel(ff, from_store):
    """tscl_wgrad_tc: dWx = X^T dZ, dWh = Hp^T dZ, dbl = 1^T dZ (wgmma, MN-major bf16 operands) vs a float64
    contraction of the same bf16-rounded operands (rtol 2e-3); Hp rebuilt from the bf16 store with the done mask."""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import BatchedA2C, _p
    lay = _layout(ff)
    T, Rc, R, r0 = 5, 333, 400, 40
    m = BatchedA2C(lay, R, n_step=T, seed=4)
    U, M, dx = lay.U, T * Rc, lay.dx
    g = torch.Generator(device="cuda").manual_seed(2)
    Xb = torch.relu(torch.randn(U, M, dx, device="cuda", generator=g)).to(torch.bfloat16).contiguous()
    Hb = torch.tanh(torch.randn(U, T, Rc, 64, device="cuda", generator=g)).to(torch.bfloat16).contiguous()
    h0 = torch.tanh(torch.randn(U, R, 64, device="cuda", generator=g))
    done = torch.tensor([0, 0, 1, 0, 0], dtype=torch.float32, device="cuda")
    dZb = (torch.randn(U, M, 256, device="cuda", generator=g) * 1e-2).to(torch.bfloat16).contiguous()
    dZ = dZb.float()
    # reference Hp (fp32 values of the bf16 operands)
    Hp = torch.empty(U, T, Rc, 64, device="cuda")
    Hp[:, 0] = h0[:, r0:r0 + Rc].to(torch.bfloat16).float()
    Hp[:, 1:] = Hb[:, :-1].float()
    Hp = (Hp * (1 - done)[None, :, None, None]).reshape(U, M, 64).contiguous()
    G = torch.zeros_like(m.G)
    lib = _lib.lib()

    def run(variant, out):
        if from_store:
            _lib.check(lib.tscl_wgrad_tc(m._h, None, _p(dZb), None, _p(Xb), None, _p(Hb), _p(h0), _p(done), C.c_int32(T),
                                         C.c_int64(Rc), C.c_int64(R), C.c_int64(r0), _p(out), C.c_int32(variant), m._st()))
        else:
            Xf = Xb.float().contiguous()
            _lib.check(lib.tscl_wgrad_tc(m._h, _p(dZ), None, _p(Xf), None, _p(Hp), None, None, None, C.c_int32(T),
                                         C.c_int64(Rc), C.c_int64(R), C.c_int64(r0), _p(out), C.c_int32(variant), m._st()))
        torch.cuda.synchronize()
    run(0, G)
    gv = lay.views(G)
    Zb = dZ.to(torch.bfloat16).double()
    wx_ref = torch.bmm(Xb.double().transpose(1, 2), Zb)
    wh_ref = torch.bmm(Hp.double().transpose(1, 2), Zb)
    bl_ref = Zb.sum(1)
    errs = [float((gv["wx"].double() - wx_ref).abs().max() / wx_ref.abs().max()),
            float((gv["wh"].double() - wh_ref).abs().max() / wh_ref.abs().max()),
            float((gv["bl"].double() - bl_ref).abs().max() / bl_ref.abs().max())]
    if max(errs) > 2e-3:
        G3 = torch.zeros_like(m.G)
        run(1, G3)
        e3 = float((lay.views(G3)["wx"].double() - wx_ref).abs().max() / wx_ref.abs().max())
        raise AssertionError("wgmma wgrad mismatch: rel errs wx/wh/bl %s (LBO/SBO swapped: wx %.4f)" % (errs, e3))
    # nothing outside wx / wh / bl is touched
    for k, v in gv.items():
        if k not in ("wx", "wh", "bl"):
            assert not bool(v.any()), k


@pytest.mark.parametrize("ff,M", [(64, 128 * 5 + 37), (0, 300), ("monaco", 4096 + 1), (64, 128 * 400 + 3)])
def test_dx_kernel_matches_bf16_matmul(ff, M):
    """tscl_dx_tc (dX = dZ . Wx^T, warp-specialised wgmma kernel) vs the same product of the bf16-rounded operands in
    fp32: products of bf16 values are exact in fp32, so only the summation order and the final bf16 rounding differ."""
    import ctypes as C
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from tests.test_learner_gpu import _layout
    lay = _layout(ff)
    m = BatchedA2C(lay, 8, n_step=2, seed=5)
    assert m.dx_own
    U, dx = lay.U, lay.dx
    g = torch.Generator(device="cuda").manual_seed(7)
    dZ = (torch.randn(U, M, 256, device="cuda", generator=g) * 0.3).to(torch.bfloat16)
    dX = torch.full((U, M, dx), float("nan"), device="cuda", dtype=torch.bfloat16)
    pad = torch.full((1024,), 7.0, device="cuda", dtype=torch.bfloat16)        # canary right behind the output
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for _ in range(2):          # second call: the persistent state (barriers, accumulator tiles) is set up afresh every launch
        _lib.check(_lib.lib().tscl_dx_tc(m._h, C.c_void_p(dZ.data_ptr()), C.c_void_p(m.Wxt.data_ptr()),
                                         C.c_void_p(dX.data_ptr()), C.c_int64(M), st))
    torch.cuda.synchronize()
    wx = m.pv["wx"].to(torch.bfloat16).float()                 # [U][dx][256]
    ref = torch.bmm(dZ.float(), wx.transpose(1, 2))
    assert torch.isfinite(dX.float()).all()
    err = (dX.float() - ref).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item() + 1e-6, err
    # bf16 rounding of the exact result: at most one bf16 ulp of the value
    assert ((dX.float() - ref).abs() <= ref.abs() * 2.0 ** -7 + 1e-3).all()
    assert (pad == 7.0).all()
