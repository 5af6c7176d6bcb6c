"""GPU: the weight-gradient kernels at the bench's update-chunk size (5x5 grid MA2C layout, 50 units, M = 120 x 1024 rows
per unit), where every CTA of tscl_wgrad_tc keeps its accumulator over thousands of tiles and flushes it across unit
boundaries, vs a float64 contraction of the same bf16 operands (rtol 2e-3, as in test_policy_tc_gpu.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T, RC = 120, 1024
M = T * RC


def _model():
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    net = build_large_grid(agent="ma2c")
    lay = PolicyLayout(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, net.node_obs_off, net.n_obs, fw=128, ft=32, ff=64,
                       h=64, max_na=net.max_na)
    return lay, BatchedA2C(lay, 8, n_step=2, seed=3)


def _rel(got, ref):
    return float((got.double() - ref).abs().max() / ref.abs().max())


def test_wgrad_bench_chunk():
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    lay, m = _model()
    U, dx = lay.U, lay.dx
    g = torch.Generator(device="cuda").manual_seed(21)
    Xb = torch.relu(torch.randn(U, M, dx, device="cuda", generator=g)).to(torch.bfloat16)
    Hb = torch.tanh(torch.randn(U, T, RC, 64, device="cuda", generator=g)).to(torch.bfloat16)
    h0 = torch.tanh(torch.randn(U, RC, 64, device="cuda", generator=g))
    done = torch.zeros(T, device="cuda")
    done[[0, 37, 90]] = 1.0
    dZb = (torch.randn(U, M, 256, device="cuda", generator=g) * 1e-2).to(torch.bfloat16)
    G = torch.zeros_like(m.G)
    _lib.check(_lib.lib().tscl_wgrad_tc(m._h, None, _p(dZb), None, _p(Xb), None, _p(Hb), _p(h0), _p(done), C.c_int32(T),
                                        C.c_int64(RC), C.c_int64(RC), C.c_int64(0), _p(G), C.c_int32(0), m._st()))
    torch.cuda.synchronize()
    gv = lay.views(G)
    keep = (1 - done)[:, None, None]
    errs = []
    for u in range(U):
        Hp = torch.cat([h0[u][None].to(torch.bfloat16).double(), Hb[u, :-1].double()]) * keep
        Z = dZb[u].double()
        errs.append(max(_rel(gv["wx"][u], Xb[u].double().T @ Z), _rel(gv["wh"][u], Hp.reshape(M, 64).T @ Z),
                        _rel(gv["bl"][u], Z.sum(0))))
    assert max(errs) < 2e-3, errs
    for k, v in gv.items():
        if k not in ("wx", "wh", "bl"):
            assert not bool(v.any()), k


def test_fc_bwd_bench_chunk():
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    lay, m = _model()
    U, dx = lay.U, lay.dx
    g = torch.Generator(device="cuda").manual_seed(22)
    obs = torch.rand(T, RC, lay.n_obs, device="cuda", generator=g) * 2
    Xb = torch.relu(torch.randn(U, M, dx, device="cuda", generator=g)).to(torch.bfloat16)
    dXb = (torch.randn(U, M, dx, device="cuda", generator=g) * 1e-2).to(torch.bfloat16)
    G = torch.zeros_like(m.G)
    _lib.check(_lib.lib().tscl_fc_bwd_tc(m._h, _p(obs[0]), None, _p(Xb), None, _p(dXb), C.c_int64(M), C.c_int64(RC),
                                         C.c_int64(RC * lay.n_obs), _p(G), C.c_int32(0), m._st()))
    torch.cuda.synchronize()
    gv = lay.views(G.cpu().numpy())
    ob = obs.reshape(M, lay.n_obs).to(torch.bfloat16).double()
    worst = 0.0
    for u in range(U):
        a = u // 2
        o0, nw, nt, nf = int(lay.obs_off[a]), int(lay.n_wave[a]), int(lay.n_wait[a]), int(lay.n_fp[a])
        dd = (dXb[u].double() * (Xb[u] > 0))
        blocks = [("fcw", ob[:, o0:o0 + nw], dd[:, :lay.fw]),
                  ("fcf", ob[:, o0 + nw + nt:o0 + nw + nt + nf], dd[:, lay.fw:lay.fw + lay.ff]),
                  ("fct", ob[:, o0 + nw:o0 + nw + nt], dd[:, lay.fw + lay.ff:])]
        for name, inp, d_ in blocks:
            w_ref, b_ref = (inp.T @ d_).cpu().numpy(), d_.sum(0).cpu().numpy()
            w_tc, b_tc = gv["%s_w%d" % (name, u)], gv["%s_b%d" % (name, u)]
            worst = max(worst, np.abs(w_tc - w_ref).max() / max(np.abs(w_ref).max(), 1e-12),
                        np.abs(b_tc - b_ref).max() / max(np.abs(b_ref).max(), 1e-12))
    assert worst < 2e-3, worst
