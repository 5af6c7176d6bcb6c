"""GPU: the two update paths that do not read the activation store, at the bench's chunk shape (1024 replicas x 120 steps
on the 5x5 grid, 50 units; 40 steps on Monaco), kernel by kernel and as a whole, against float64 references that round
where the kernels round (oracle/learner_ref.py; tests/test_update_fallback_reference_cpu.py pins them to autograd).

  * the recompute update, which BatchedA2C.backward takes when the activation store is off (it does not fit in half of
    the free device memory, or R is not a multiple of the chunk): tscl_fc_embed -> X . Wx + bl (torch.baddbmm, TF32 when
    allowed) -> tscl_lstm_seq_fwd -> tscl_heads_loss on fp32 H -> tscl_lstm_seq_bwd_tc_dx on fp32 gates / c
    (lstm_bwd_tc_kernel<512>, dZ written fp32 in place) -> tscl_wgrad_tc on fp32 operands (wgrad_tc_kernel) -> dX by
    torch.bmm -> tscl_fc_bwd_tc on fp32 X / dX;
  * the FcACPolicy learner (BatchedFcA2C, bench --policy fc): tscl_fc_embed -> tscl_fc_hidden_fwd -> tscl_heads_loss ->
    tscl_fc_hidden_bwd -> tscl_fc_bwd_tc, and its forward with inverse-CDF sampling (tscl_heads).

Bounds are about 3x the worst value seen on an H100 80GB HBM3 (400 W power limit); the observed values are given beside
each bound.  Every test frees its device memory when it ends."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests.test_update_bench_size_gpu import _layout, dz_errors
from tests.update_fallback_bounds import (RECOMPUTE_G_REL_L2, RECOMPUTE_TENSOR_REL_L2, RECOMPUTE_G_REL_L2_FP32,
                                        RECOMPUTE_TENSOR_REL_L2_FP32, FC_G_REL_L2, FC_FP32_TENSOR_REL_L2,
                                        FC_FRONT_TENSOR_REL_L2, FP32_KERNEL_MAX, HEADS_MAX, FC_FORWARD_MAX,
                                        WGRAD_FP32_MAX, FC_BWD_FP32_MAX, BPTT_FP32_REL_L2, BPTT_FP32_MAX)

pytestmark = pytest.mark.gpu

T_GRID, T_MONACO = 120, 40
R_BENCH, RC, R0 = 2048, 1024, 1024


@pytest.fixture(autouse=True)
def _free_device_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    print("peak device memory %.2f GB" % (torch.cuda.max_memory_allocated() / 2 ** 30))
    torch.cuda.empty_cache()


@pytest.fixture
def restore_tf32():
    """BatchedA2C._mm sets the process-wide TF32 flag of torch matmuls: put it back when the test ends."""
    saved = torch.backends.cuda.matmul.allow_tf32
    yield
    torch.backends.cuda.matmul.allow_tf32 = saved


def _fc_layout():
    """grid IA2C with the FC policy (bench --agent ia2c --policy fc): dx = 160"""
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    net = build_large_grid(agent="ia2c")
    return PolicyLayout(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, net.node_obs_off, net.n_obs, fw=128, ft=32, ff=0,
                        h=64, max_na=net.max_na, recurrent=False)


def _model(kind, R=8, T=2, **kw):
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from deeprl_signal_control_b200.agents.learner_fc import BatchedFcA2C
    if kind == "fc":
        lay = _fc_layout()
        return lay, BatchedFcA2C(lay, R, n_step=T, seed=kw.pop("seed", 3), **kw)
    lay = _layout(kind)
    return lay, BatchedA2C(lay, R, n_step=T, seed=kw.pop("seed", 3), **kw)


def _call(name, *args):
    from deeprl_signal_control_b200 import _lib
    _lib.check(getattr(_lib.lib(), name)(*args))
    torch.cuda.synchronize()


def _p(t):
    from deeprl_signal_control_b200.agents.learner import _p as p_
    return p_(t)


# The comparisons below return inf, never nan, when an output holds a NaN or an inf: Python's max(worst, nan) keeps
# `worst`, so a nan would vanish from the running maxima.  Outputs start as NaN where a kernel should write every element,
# so an unwritten row shows up here too.
def _finite(x):
    return x if math.isfinite(x) else math.inf


def _rel_max(got, ref):
    return _finite(((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item())


def _rel_l2(got, ref):
    return _finite(((got.double() - ref).norm() / ref.norm().clamp_min(1e-300)).item())


def _assert_finite(**outputs):
    for name, t in outputs.items():
        assert bool(torch.isfinite(t).all()), "%s holds %d non-finite values" % (name, int((~torch.isfinite(t)).sum()))


def _only_moved(lay, G, keys):
    """nothing in G outside the named views moved"""
    for k, t in lay.views(G).items():
        if not any(k == n or (k.startswith(n) and k[len(n):].isdigit()) for n in keys):
            assert not bool(t.any()), k


# ------------------------------------------------------------------------------------------------------------------
# kernels of the recompute path, one chunk (r0 = 1024 of R = 2048, or the ragged Rc = 1000 at r0 = 1000 of R = 3000)
SHAPES = [("grid", T_GRID, RC, R_BENCH, R0), ("monaco", T_MONACO, RC, R_BENCH, R0), ("grid_ia2c", T_GRID, RC, R_BENCH, R0),
          ("grid", T_GRID, 1000, 3000, 1000)]


@pytest.mark.parametrize("kind,T,Rc,R,r0", SHAPES)
def test_fc_embed_chunk(kind, T, Rc, R, r0):
    """tscl_fc_embed over the chunk's rows (row stride R * n_obs per step, r0 > 0) vs fc_front in float64."""
    from oracle.learner_ref import fc_front
    lay, m = _model(kind)
    g = torch.Generator(device="cuda").manual_seed(1)
    v = lay.views(m.P)
    for u in range(lay.U):
        v["fcw_b%d" % u].copy_(torch.randn(lay.fw, device="cuda", generator=g) * 0.1)
    obs = torch.rand(T, R, lay.n_obs, device="cuda", generator=g) * 2
    M = T * Rc
    X = torch.full((lay.U, M, lay.dx), float("nan"), device="cuda")
    _call("tscl_fc_embed", m._h, _p(m.P), _p(obs[0, r0:]), C.c_int64(M), C.c_int64(Rc), C.c_int64(R * lay.n_obs), _p(X),
          m._st())
    _assert_finite(X=X)
    vd = lay.views(m.P.double())
    ob = obs[:, r0:r0 + Rc].double()
    worst = max(_rel_max(X[u], fc_front(vd, lay, u, ob).reshape(M, -1)) for u in range(lay.U))
    print("OBSERVED fc_embed %s T=%d Rc=%d r0=%d: max|d|/max|ref| %.3e" % (kind, T, Rc, r0, worst))
    assert worst <= FP32_KERNEL_MAX, worst


@pytest.mark.parametrize("kind,T,Rc,R,r0", SHAPES[:2] + SHAPES[3:])
def test_lstm_seq_fwd_chunk(kind, T, Rc, R, r0):
    """tscl_lstm_seq_fwd over all T steps of the chunk from given pre-activations ZG (x-part + bias), nonzero c_bw / h_bw
    rows r0 .. r0 + Rc, done {0, 37, 90} and {37, 90} (the second lets the initial state through): gates (written over
    ZG), C, H, Hp and the final state vs float64; state rows outside the chunk untouched."""
    lay, m = _model(kind)
    U, H = lay.U, lay.h
    g = torch.Generator(device="cuda").manual_seed(2)
    M = T * Rc
    Z0 = torch.randn(U, M, 4 * H, device="cuda", generator=g)
    c_bw = torch.randn(U, R, H, device="cuda", generator=g) * 0.5
    h_bw = torch.tanh(torch.randn(U, R, H, device="cuda", generator=g))
    wh = m.pv["wh"].double()
    worst = {"gates": 0.0, "C": 0.0, "H": 0.0, "Hp": 0.0, "state": 0.0}
    for pattern in ((0, 37, 90), (37, 90)):
        done = torch.zeros(T, device="cuda")
        done[[s for s in pattern if s < T]] = 1.0
        ZG = Z0.clone()
        Cc, Hh, Hp = (torch.full((U, M, H), float("nan"), device="cuda") for _ in range(3))
        c1, h1 = c_bw.clone(), h_bw.clone()
        _call("tscl_lstm_seq_fwd", m._h, _p(m.P), _p(ZG), _p(Cc), _p(Hh), _p(Hp), _p(c_bw), _p(h_bw), _p(c1), _p(h1),
              _p(done), C.c_int32(T), C.c_int64(Rc), C.c_int64(R), C.c_int64(r0), m._st())
        _assert_finite(gates=ZG, C=Cc, H=Hh, Hp=Hp, c1=c1, h1=h1)
        for u0 in range(0, U, 10):
            us = slice(u0, min(U, u0 + 10))
            c, h = c_bw[us, r0:r0 + Rc].double(), h_bw[us, r0:r0 + Rc].double()
            z0 = Z0[us].double().reshape(-1, T, Rc, 4 * H)
            sh = lambda t_: t_[us].reshape(-1, T, Rc, t_.shape[-1])
            for t in range(T):
                keep = 1.0 - float(done[t])
                c, h = c * keep, h * keep
                worst["Hp"] = max(worst["Hp"], _rel_max(sh(Hp)[:, t], h) if keep else _finite(float(sh(Hp)[:, t].abs().max())))
                z = z0[:, t] + h @ wh[us]
                gt = torch.cat([torch.sigmoid(z[..., :3 * H]), torch.tanh(z[..., 3 * H:])], -1)
                c = gt[..., H:2 * H] * c + gt[..., :H] * gt[..., 3 * H:]
                h = gt[..., 2 * H:3 * H] * torch.tanh(c)
                worst["gates"] = max(worst["gates"], _rel_max(sh(ZG)[:, t], gt))
                worst["C"] = max(worst["C"], _rel_max(sh(Cc)[:, t], c))
                worst["H"] = max(worst["H"], _rel_max(sh(Hh)[:, t], h))
            worst["state"] = max(worst["state"], _rel_max(c1[us, r0:r0 + Rc], c), _rel_max(h1[us, r0:r0 + Rc], h))
            del z0
        out = torch.ones(R, dtype=torch.bool, device="cuda")
        out[r0:r0 + Rc] = False
        assert torch.equal(c1[:, out], c_bw[:, out]) and torch.equal(h1[:, out], h_bw[:, out])
        del ZG, Cc, Hh, Hp
    print("OBSERVED lstm_seq_fwd %s T=%d Rc=%d r0=%d: %s" % (kind, T, Rc, r0,
                                                            ", ".join("%s %.3e" % kv for kv in worst.items())))
    assert max(worst.values()) <= FP32_KERNEL_MAX, worst


def test_heads_loss_fp32_h_chunk():
    """tscl_heads_loss with fp32 H (the recompute and FC paths) for the chunk at r0 = 1024 of R = 2048 (M = 122 880 rows),
    with the planted rows of test_heads_loss_bench_chunk (clipped pi of agent 0's action 1, last action, Adv = 0)."""
    from oracle.learner_ref import heads_ref
    T, R, rc, r0 = T_GRID, R_BENCH, RC, R0
    M = T * rc
    lay, m = _model("grid")
    U, A = lay.U, lay.A
    g = torch.Generator(device="cuda").manual_seed(31)
    v = lay.views(m.P)
    for u in range(U):
        n_out = int(lay.n_a[u // 2]) if u % 2 == 0 else 1
        v["wo"][u][:, :n_out] = torch.randn(64, n_out, device="cuda", generator=g) * 0.5
        v["bo"][u][:n_out] = torch.randn(n_out, device="cuda", generator=g) * 0.1
    v["bo"][0][1] = -40.0
    Hf = torch.tanh(torch.randn(U, M, 64, device="cuda", generator=g) * 1.5)
    na = torch.as_tensor(lay.n_a, device="cuda")
    act = (torch.rand(T, R, A, device="cuda", generator=g) * na).long().clamp_max(na - 1).to(torch.int32)
    act[::3, :, 0] = 1
    act[1::5] = (na - 1).to(torch.int32)
    Rs = torch.randn(T, R, A, device="cuda", generator=g) * 2
    Adv = torch.randn(T, R, A, device="cuda", generator=g) * 2
    Adv[2::7] = 0.0
    scale, v_coef, beta = 1.0 / (T * R), 0.5, 0.01
    dH = torch.empty(U, M, 64, device="cuda")
    G = torch.zeros_like(m.G)
    stats = torch.zeros(4, device="cuda")
    _call("tscl_heads_loss", m._h, _p(m.P), _p(Hf), _p(act[0, r0:]), _p(Rs[0, r0:]), _p(Adv[0, r0:]), C.c_int64(M),
          C.c_int64(rc), C.c_int64(R * A), C.c_float(v_coef), C.c_float(beta), C.c_float(scale), None, _p(dH), _p(stats),
          None, _p(G), m._st())
    _assert_finite(dH=dH, G=G, stats=stats)
    vd, gv = lay.views(m.P.double()), lay.views(G)
    worst = {"dH": 0.0, "wo": 0.0, "bo": 0.0}
    for a in range(A):
        sl = lambda x: x[:, r0:r0 + rc, a].reshape(-1)
        hr = heads_ref(lay, vd, a, Hf[2 * a].double(), Hf[2 * a + 1].double(), sl(act), sl(Rs).double(), sl(Adv).double(),
                       scale, v_coef, beta)
        n = int(lay.n_a[a])
        worst["dH"] = max(worst["dH"], _rel_max(dH[2 * a], hr["dH_pi"]), _rel_max(dH[2 * a + 1], hr["dH_v"]))
        worst["wo"] = max(worst["wo"], _rel_max(gv["wo"][2 * a][:, :n], hr["wo_pi"]),
                          _rel_max(gv["wo"][2 * a + 1][:, 0], hr["wo_v"]))
        worst["bo"] = max(worst["bo"], _rel_max(gv["bo"][2 * a][:n], hr["bo_pi"]),
                          _rel_max(gv["bo"][2 * a + 1][:1], hr["bo_v"].reshape(1)))
        if a == 0:
            np.testing.assert_allclose(stats[:3].cpu().numpy(), hr["stats"].cpu().numpy(), rtol=1e-4)
    print("OBSERVED heads_loss fp32 H: max|d|/max|ref| dH %.3e wo %.3e bo %.3e" % (worst["dH"], worst["wo"], worst["bo"]))
    assert all(worst[k] <= HEADS_MAX[k] for k in worst), worst
    _only_moved(lay, G, ("wo", "bo"))


def _bptt_fp32_inputs(U, T, Rc, ld, done_steps, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(U, T * Rc, 256, device="cuda", generator=g) * 1.5
    gates = torch.cat([torch.sigmoid(z[..., :192]), torch.tanh(z[..., 192:])], -1)
    del z
    cc = torch.randn(U, T * Rc, 64, device="cuda", generator=g) * 0.8
    dH = torch.randn(U, T * Rc, 64, device="cuda", generator=g) * 1e-3
    c_bw = torch.randn(U, ld, 64, device="cuda", generator=g) * 0.5
    done = torch.zeros(T, device="cuda")
    done[list(done_steps)] = 1.0
    return gates, cc, dH, c_bw, done


@pytest.mark.parametrize("kind,T,Rc,ld,r0", [("grid", T_GRID, RC, R_BENCH, R0), ("monaco", T_MONACO, RC, R_BENCH, R0),
                                             ("grid", T_GRID, 1000, 3000, 1000)])
def test_bptt_fp32_gates_matches_float64_reference(kind, T, Rc, ld, r0):
    """tscl_lstm_seq_bwd_tc_dx as the recompute update calls it: fp32 gates / c, dZ written fp32 over ZG
    (lstm_bwd_tc_kernel<512>), vs bptt_ref (recurrent product bf16(dz) . bf16(Wh)^T, dZ unrounded), dz_errors metric of
    the store-path test; done {37, 90} and {0, T-1}; the six planted defects of bptt_mutations."""
    from oracle.learner_ref import bptt_mutations, bptt_ref
    lay, m = _model(kind)
    U = lay.U
    worst_l2 = worst_max = 0.0
    mutation = {}
    for pat, steps in enumerate([(37 % T, 90 % T), (0, T - 1)]):
        gates, cc, dH, c_bw, done = _bptt_fp32_inputs(U, T, Rc, ld, steps, seed=20 + pat)
        ZG = gates.clone()
        _call("tscl_lstm_seq_bwd_tc_dx", m._h, _p(m.Wt), _p(ZG), _p(cc), _p(dH), _p(c_bw), _p(done), C.c_int32(T),
              C.c_int64(Rc), C.c_int64(ld), C.c_int64(r0), None, None, None, None, None, m._st())
        _assert_finite(dZ=ZG)
        d = lambda x, us: x[us].double().reshape(len(range(*us.indices(U))), T, Rc, -1)
        for u0 in range(0, U, 10):
            us = slice(u0, min(U, u0 + 10))
            ref = bptt_ref(d(gates, us), d(cc, us), c_bw[us, r0:r0 + Rc].double(), d(dH, us), done.tolist(),
                           m.pv["wh"][us].double())
            l2, mx = map(_finite, dz_errors(d(ZG, us), ref))
            worst_l2, worst_max = max(worst_l2, l2), max(worst_max, mx)
            del ref
        if kind == "grid" and Rc == RC and pat == 0:
            us = slice(0, 2)
            ok, mutants = bptt_mutations(d(gates, us), d(cc, us), c_bw[us].double(), r0, d(dH, us), done.tolist())
            wh = m.pv["wh"][us].double()
            ref = bptt_ref(**ok, wh=wh)
            for name, kw in mutants.items():
                mutation[name] = dz_errors(bptt_ref(**kw, wh=wh), ref)[0]
                print("OBSERVED mutation %-32s rel-L2 %.3e = %.0fx the bound" % (name, mutation[name],
                                                                                mutation[name] / BPTT_FP32_REL_L2))
            del ok, mutants, ref
        del gates, cc, dH, c_bw, done, ZG
    print("OBSERVED bptt fp32 gates %s T=%d Rc=%d r0=%d: per (unit, step) rel-L2 %.3e, max|d|/max|ref| %.3e" % (
        kind, T, Rc, r0, worst_l2, worst_max))
    assert worst_l2 <= BPTT_FP32_REL_L2 and worst_max <= BPTT_FP32_MAX, (worst_l2, worst_max)
    assert len(mutation) == (6 if kind == "grid" and Rc == RC else 0)
    for name, rel in mutation.items():
        assert rel >= 10 * BPTT_FP32_REL_L2, (name, rel)


@pytest.mark.parametrize("kind,T,Rc", [("grid", T_GRID, RC), ("monaco", T_MONACO, RC), ("grid_ia2c", T_GRID, RC),
                                       ("grid", T_GRID, 1000)])
def test_wgrad_fp32_operands_chunk(kind, T, Rc):
    """tscl_wgrad_tc with fp32 dZ / X / Hp (wgrad_tc_kernel: accumulator tiles in global memory, thousands of tiles per
    CTA) vs the float64 contraction of the operands rounded to bf16 as the kernel converts them; nothing but wx / wh / bl
    moves."""
    lay, m = _model(kind)
    U, dx, M = lay.U, lay.dx, T * Rc
    g = torch.Generator(device="cuda").manual_seed(23)
    X = torch.relu(torch.randn(U, M, dx, device="cuda", generator=g))
    Hp = torch.tanh(torch.randn(U, M, 64, device="cuda", generator=g))
    Hp[:, :Rc] = 0.0                                   # done at t = 0
    dZ = torch.randn(U, M, 256, device="cuda", generator=g) * 1e-2
    G = torch.zeros_like(m.G)
    _call("tscl_wgrad_tc", m._h, _p(dZ), None, _p(X), None, _p(Hp), None, None, None, C.c_int32(T), C.c_int64(Rc),
          C.c_int64(Rc), C.c_int64(0), _p(G), C.c_int32(0), m._st())
    _assert_finite(G=G)
    gv = lay.views(G)
    b = lambda t_: t_.to(torch.bfloat16).double()
    worst = 0.0
    for u in range(U):
        Z = b(dZ[u])
        worst = max(worst, _rel_max(gv["wx"][u], b(X[u]).T @ Z), _rel_max(gv["wh"][u], b(Hp[u]).T @ Z),
                    _rel_max(gv["bl"][u], Z.sum(0)))
    print("OBSERVED wgrad fp32 operands %s T=%d Rc=%d: max|d|/max|ref| %.3e" % (kind, T, Rc, worst))
    assert worst <= WGRAD_FP32_MAX, worst
    _only_moved(lay, G, ("wx", "wh", "bl"))


@pytest.mark.parametrize("kind,T,Rc,R,r0", SHAPES)
def test_fc_bwd_fp32_inputs_chunk(kind, T, Rc, R, r0):
    """tscl_fc_bwd_tc with fp32 X / dX (relu mask from fp32 X, operands converted to bf16) for the chunk at r0 of R
    (observation row stride R * n_obs) vs fc_grads_ref; nothing but the fc front end moves."""
    from oracle.learner_ref import bf16, fc_grads_ref
    lay, m = _model(kind)
    U, dx, M = lay.U, lay.dx, T * Rc
    g = torch.Generator(device="cuda").manual_seed(24)
    obs = torch.rand(T, R, lay.n_obs, device="cuda", generator=g) * 2
    X = torch.relu(torch.randn(U, M, dx, device="cuda", generator=g))
    dX = torch.randn(U, M, dx, device="cuda", generator=g) * 1e-2
    G = torch.zeros_like(m.G)
    _call("tscl_fc_bwd_tc", m._h, _p(obs[0, r0:]), _p(X), None, _p(dX), None, C.c_int64(M), C.c_int64(Rc),
          C.c_int64(R * lay.n_obs), _p(G), C.c_int32(0), m._st())
    _assert_finite(G=G)
    gv = lay.views(G)
    ob = obs[:, r0:r0 + Rc].double()
    worst = 0.0
    for u in range(U):
        ref = fc_grads_ref(lay, u, ob, X[u].double().reshape(T, Rc, dx), bf16(dX[u].double()).reshape(T, Rc, dx))
        for k, r in ref.items():
            worst = max(worst, _rel_max(gv[k], r))
    print("OBSERVED fc_bwd fp32 inputs %s T=%d Rc=%d r0=%d: max|d|/max|ref| %.3e" % (kind, T, Rc, r0, worst))
    assert worst <= FC_BWD_FP32_MAX, worst
    _only_moved(lay, G, ("fcw_w", "fcw_b", "fcf_w", "fcf_b", "fct_w", "fct_b"))


def test_fc_hidden_layer_bench_chunk():
    """tscl_fc_hidden_fwd / tscl_fc_hidden_bwd at dx = 160, M = 122 880 rows per unit (many tiles per persistent CTA, 60
    row splits of the weight gradient): H, the masked dH written back (bit-exact), dX, g.wx and g.bl vs float64."""
    lay, m = _model("fc")
    U, dx, M = lay.U, lay.dx, T_GRID * RC
    assert dx == 160
    g = torch.Generator(device="cuda").manual_seed(25)
    v = lay.views(m.P)
    v["bl"].copy_(torch.randn(U, 64, device="cuda", generator=g) * 0.1)
    X = torch.relu(torch.randn(U, M, dx, device="cuda", generator=g))
    H = torch.full((U, M, 64), float("nan"), device="cuda")
    _call("tscl_fc_hidden_fwd", m._h, _p(m.P), _p(X), C.c_int64(M), _p(H), m._st())
    _assert_finite(H=H)
    dH0 = torch.randn(U, M, 64, device="cuda", generator=g) * 1e-3
    dH = dH0.clone()
    dX = torch.full((U, M, dx), float("nan"), device="cuda")
    G = torch.zeros_like(m.G)
    _call("tscl_fc_hidden_bwd", m._h, _p(m.P), _p(X), _p(H), _p(dH), C.c_int64(M), _p(dX), _p(G), m._st())
    _assert_finite(dX=dX, G=G)
    assert torch.equal(dH, torch.where(H > 0, dH0, torch.zeros_like(dH0)))
    gv = lay.views(G)
    worst = {"H": 0.0, "dX": 0.0, "wx": 0.0, "bl": 0.0}
    for u in range(U):
        Xd, w = X[u].double(), m.pv["wx"][u].double()
        worst["H"] = max(worst["H"], _rel_max(H[u], torch.relu(Xd @ w + m.pv["bl"][u].double())))
        dHm = dH[u].double()
        worst["dX"] = max(worst["dX"], _rel_max(dX[u], dHm @ w.T))
        worst["wx"] = max(worst["wx"], _rel_max(gv["wx"][u], Xd.T @ dHm))
        worst["bl"] = max(worst["bl"], _rel_max(gv["bl"][u], dHm.sum(0)))
    print("OBSERVED fc_hidden dx=160 M=%d: %s" % (M, ", ".join("%s %.3e" % kv for kv in worst.items())))
    assert max(worst.values()) <= FP32_KERNEL_MAX, worst
    _only_moved(lay, G, ("wx", "bl"))


# ------------------------------------------------------------------------------------------------------------------
# whole updates
GROUPS_LSTM = ("wx", "wh", "bl", "wo", "bo", "fcw_w", "fcw_b", "fcf_w", "fcf_b", "fct_w", "fct_b")


def _per_tensor(lay, G, Gref, names):
    gv, rv = lay.views(G.double()), lay.views(Gref)
    worst = {}
    for name in names:
        keys = [name] if name in rv else [name + str(u) for u in range(lay.U)]
        ref = torch.cat([rv[k].reshape(-1) for k in keys])
        if ref.numel() == 0:
            continue
        worst[name] = _rel_l2(torch.cat([gv[k].reshape(-1) for k in keys]), ref)
    return worst


def _rollout(lay, m, T, R, g, done_steps):
    """T steps of random observations / rewards through m.forward / m.add_transition, from nonzero recurrent states
    (LSTM learners); the next observation in slot T.  Returns (dpre, dpost, bootstrap values)."""
    if lay.recurrent:
        m.c_fw.copy_(torch.randn(m.c_fw.shape, device="cuda", generator=g) * 0.5)
        m.h_fw.copy_(torch.tanh(torch.randn(m.h_fw.shape, device="cuda", generator=g)) * 0.5)
        m.c_bw.copy_(m.c_fw); m.h_bw.copy_(m.h_fw)
    dpre = [1.0 if t in done_steps else 0.0 for t in range(T)]
    dpost = dpre[1:] + [0.0]
    for t in range(T):
        m.obs_slot().copy_(torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2)
        m.forward(m.obs_slot(), bool(dpre[t]))
        m.add_transition(torch.randn(R, lay.A, device="cuda", generator=g) * 3000, bool(dpre[t]), bool(dpost[t]))
    m.obs_hist[T].copy_(torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2)
    return dpre, dpost, torch.randn(R, lay.A, device="cuda", generator=g)


def _check_returns(m, dpost, boot, gamma):
    from oracle.learner_ref import nstep_returns
    Rs_ref, Adv_ref = nstep_returns(list(m.rew_hist.double().cpu().numpy()), list(m.val_hist.double().cpu().numpy()),
                                    dpost, boot.double().cpu().numpy(), gamma)
    np.testing.assert_allclose(m.Rs.cpu().numpy(), Rs_ref, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(m.Adv.cpu().numpy(), Adv_ref, rtol=1e-5, atol=1e-5)


def _recompute_reference(lay, m, obs, c_bw, h_bw, dpre, T, R, chunk, beta, tf32, fwd_pick=None, agents=None):
    """update_ref of the recompute path over the float64 forward of each agent group (store_units); `fwd_pick` chooses
    the forward inputs from recompute_mutations (default: the correct ones)."""
    from oracle.learner_ref import recompute_mutations, store_group, update_ref
    vd = lay.views(m.P.double())
    pick = fwd_pick or (lambda ok, mutants: ok)

    def store(ci, us):
        r0 = ci * chunk
        f = pick(*recompute_mutations(obs, c_bw, h_bw, dpre, r0, min(chunk, R - r0)))
        return store_group(vd, lay, us, f["obs"].double(), f["dones"], f["c0"].double(), f["h0"].double())
    return update_ref(lay, m.P, store, obs[:T], m.act_hist, m.Rs, m.Adv, c_bw, h_bw, dpre, 1.0 / (T * R), 0.5, beta, chunk,
                      agents_per_group=3, store_units=True, round_operands=True, dx_product="tf32" if tf32 else "fp32",
                      agents=agents)[0]


def _run_recompute_update(kind, R, chunk, tf32, store_acts, seed=41):
    T = T_MONACO if kind == "monaco" else T_GRID
    gamma, beta = 0.99, 0.01
    lay, m = _model(kind, R=R, T=T, seed=7, chunk=chunk, gamma=gamma, v_coef=0.5, max_grad_norm=40.0,
                    reward_norm=2000.0, reward_clip=2.0, use_tc=True, store_acts=store_acts, allow_tf32=tf32)
    assert not m.store_acts and m.use_tc and m.bwd_tc and m.wgrad_tc and m.fc_bwd_tc
    g = torch.Generator(device="cuda").manual_seed(seed)
    dpre, dpost, boot = _rollout(lay, m, T, R, g, {T // 3, (2 * T) // 3 + 1})
    c_bw, h_bw, obs = m.c_bw.clone(), m.h_bw.clone(), m.obs_hist.clone()
    m.backward(boot, lr=0.0, beta=beta)
    torch.cuda.synchronize()
    assert torch.backends.cuda.matmul.allow_tf32 == tf32
    m._upd_bufs = None                  # the fp32 chunk buffers (22 GB on the grid) are not needed by the reference
    torch.cuda.empty_cache()
    _check_returns(m, dpost, boot, gamma)
    return lay, m, T, dict(obs=obs, c_bw=c_bw, h_bw=h_bw, dpre=dpre, T=T, R=R, chunk=chunk, beta=beta, tf32=tf32)


@pytest.mark.parametrize("tf32", [True, False])
@pytest.mark.parametrize("kind", ["grid", "monaco", "grid_ia2c"])
def test_recompute_update_matches_float64(kind, tf32, restore_tf32):
    """BatchedA2C(use_tc=True, store_acts=False).backward at R = 2048 in two 1024-replica chunks (nonzero initial states,
    interior dones, random rewards) vs update_ref over the float64 forward of the same rollout, with the recompute path's
    rounding; TF32 allowed (the bench default) and not.  Rs / Adv vs nstep_returns, G per named tensor and overall, and
    (grid, fp32 products) the four planted defects of the recompute forward on agents 0-2.  They are judged against the
    fp32 bound: with TF32 the forward product alone moves G by up to 3.7e-4, and a zero initial state, which only matters
    for the 40 steps before the first done, moves it by 6.7e-3.  Observed: 6.3e-3 (state row) to 4.6e-2 (obs slot)."""
    lay, m, T, ref_args = _run_recompute_update(kind, R_BENCH, RC, tf32, store_acts=False)
    G0 = m.G.clone()
    Gref = _recompute_reference(lay, m, **ref_args)
    worst = _per_tensor(lay, G0, Gref, GROUPS_LSTM)
    overall = _rel_l2(G0, Gref)
    print("OBSERVED recompute update %s tf32=%s: overall rel-L2 %.3e; per tensor %s" % (
        kind, tf32, overall, ", ".join("%s %.2e" % kv for kv in worst.items())))
    b_all, b_t = (RECOMPUTE_G_REL_L2, RECOMPUTE_TENSOR_REL_L2) if tf32 else (RECOMPUTE_G_REL_L2_FP32,
                                                                          RECOMPUTE_TENSOR_REL_L2_FP32)
    assert overall <= b_all and max(worst.values()) <= b_t, (overall, worst)
    if kind == "grid" and not tf32:
        agents = range(0, 3)
        mask = torch.as_tensor(lay.agent_of < 3, device="cuda")
        for name in ("recompute from zero state", "state from row r instead of r0 + r", "done one step late",
                     "obs slot t + 1 instead of t"):
            Gm = _recompute_reference(lay, m, fwd_pick=lambda ok, mutants: mutants[name], agents=agents, **ref_args)
            rel = _rel_l2(Gm[mask], Gref[mask])
            print("OBSERVED mutation %-36s G rel-L2 %.3e = %.0fx the bound" % (name, rel, rel / RECOMPUTE_G_REL_L2_FP32))
            assert rel >= 10 * RECOMPUTE_G_REL_L2_FP32, (name, rel)
            del Gm
    m.close()


def test_recompute_fallback_when_chunk_does_not_divide(restore_tf32):
    """store_acts=None at grid R = 2500, chunk 1024: R is not a multiple of the chunk, so the store is off and the update
    recomputes the forward; the tail chunk of 452 replicas runs on dense temporaries.  Same comparison as above."""
    lay, m, T, ref_args = _run_recompute_update("grid", 2500, RC, True, store_acts=None, seed=43)
    Gref = _recompute_reference(lay, m, **ref_args)
    worst = _per_tensor(lay, m.G, Gref, GROUPS_LSTM)
    overall = _rel_l2(m.G, Gref)
    print("OBSERVED recompute fallback grid R=2500: overall rel-L2 %.3e; per tensor %s" % (
        overall, ", ".join("%s %.2e" % kv for kv in worst.items())))
    assert overall <= RECOMPUTE_G_REL_L2 and max(worst.values()) <= RECOMPUTE_TENSOR_REL_L2, (overall, worst)
    m.close()


def test_fc_update_matches_float64(restore_tf32):
    """BatchedFcA2C.backward on grid IA2C-FC at R = 2048, chunk 1024, T = 120 vs fc_update_ref (bf16 obs / dX where the
    tensor-core fc weight-gradient kernel reads them): fp32 tensors and fc front-end tensors (rel-L2 each), G overall,
    and the three FC planted defects on agents 0-2."""
    from oracle.learner_ref import FC_DEFECTS, fc_update_ref
    T, R, gamma, beta = T_GRID, R_BENCH, 0.99, 0.01
    lay, m = _model("fc", R=R, T=T, seed=7, chunk=RC, gamma=gamma, v_coef=0.5, max_grad_norm=40.0, reward_norm=3000.0,
                    reward_clip=2.0)
    assert m.fc_bwd_tc
    g = torch.Generator(device="cuda").manual_seed(45)
    v = lay.views(m.P)
    v["bl"].copy_(torch.randn(lay.U, 64, device="cuda", generator=g) * 0.1)      # some hidden units off, some on
    dpre, dpost, boot = _rollout(lay, m, T, R, g, {T // 3})
    obs = m.obs_hist[:T].clone()
    m.backward(boot, lr=0.0, beta=beta)
    torch.cuda.synchronize()
    _check_returns(m, dpost, boot, gamma)
    args = (lay, m.P, obs, m.act_hist, m.Rs, m.Adv, 1.0 / (T * R), 0.5, beta, RC)
    Gref, stats = fc_update_ref(*args, round_bf16=True)
    np.testing.assert_allclose(m.stats[:3].cpu().numpy(), stats.cpu().numpy(), rtol=1e-4)
    fp32 = _per_tensor(lay, m.G, Gref, ("wx", "bl", "wo", "bo"))
    front = _per_tensor(lay, m.G, Gref, ("fcw_w", "fcw_b", "fct_w", "fct_b"))
    overall = _rel_l2(m.G, Gref)
    print("OBSERVED FC update: overall rel-L2 %.3e; fp32 tensors %s; fc front end %s" % (
        overall, ", ".join("%s %.2e" % kv for kv in fp32.items()), ", ".join("%s %.2e" % kv for kv in front.items())))
    assert overall <= FC_G_REL_L2, overall
    assert max(fp32.values()) <= FC_FP32_TENSOR_REL_L2 and max(front.values()) <= FC_FRONT_TENSOR_REL_L2, (fp32, front)
    mask = torch.as_tensor(lay.agent_of < 3, device="cuda")
    for name in FC_DEFECTS:
        Gm, _ = fc_update_ref(*args, round_bf16=True, agents=range(0, 3), defect=name)
        rel = _rel_l2(Gm[mask], Gref[mask])
        print("OBSERVED mutation %-48s G rel-L2 %.3e = %.0fx the bound" % (name, rel, rel / FC_G_REL_L2))
        assert rel >= 10 * FC_G_REL_L2, (name, rel)
    m.close()


def test_fc_forward_bench_size(restore_tf32):
    """BatchedFcA2C.forward at R = 4096 (grid IA2C-FC): pi and value vs unit_forward in float64, actions bit-exact vs the
    counter-hash inverse-CDF restatement applied to the kernel's pi."""
    from oracle.learner_ref import unit_forward
    from tests.test_policy_forward_bench_size_gpu import _reference_actions
    R = 4096
    lay, m = _model("fc", R=R, T=2, seed=11)
    g = torch.Generator(device="cuda").manual_seed(46)
    v = lay.views(m.P)
    v["bl"].copy_(torch.randn(lay.U, 64, device="cuda", generator=g) * 0.1)
    for u in range(0, lay.U, 2):                      # wider policy heads: not near-uniform
        v["wo"][u][:, :int(lay.n_a[u // 2])].mul_(8.0)
    vd = lay.views(m.P.double())
    worst = {"pi": 0.0, "v": 0.0}
    for step in range(2):
        obs = torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2
        n_fwd = m.n_forward
        pi, val, act = m.forward(obs)
        torch.cuda.synchronize()
        _assert_finite(pi=pi, val=val)
        for a in range(lay.A):
            na = int(lay.n_a[a])
            p_ref = unit_forward(vd, lay, 2 * a, obs.double()[None], [0.0], None, None)[0][0]
            v_ref = unit_forward(vd, lay, 2 * a + 1, obs.double()[None], [0.0], None, None)[0][0]
            worst["pi"] = max(worst["pi"], _rel_max(pi[:, a, :na], p_ref))
            worst["v"] = max(worst["v"], _rel_max(val[:, a], v_ref))
            assert not bool(pi[:, a, na:].any())
        ref_act = _reference_actions(pi.cpu().numpy(), lay.n_a, m.seed, n_fwd, m.replica0)
        assert np.array_equal(act.cpu().numpy(), ref_act), step
    print("OBSERVED FC forward R=4096: max|d|/max|ref| pi %.3e value %.3e" % (worst["pi"], worst["v"]))
    assert max(worst.values()) <= FC_FORWARD_MAX, worst
    m.close()
