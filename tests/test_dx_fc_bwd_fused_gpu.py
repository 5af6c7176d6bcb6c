"""GPU: tscl_dx_fc_bwd_tc (dX = dZ . Wx^T fused into the fc front-end weight gradients, dX never stored) against
  1. the two-kernel path tscl_dx_tc -> tscl_fc_bwd_tc on the same seeded dZ / X / obs: the masked bf16 dX has the same
     bits, so only the order of the fp32 sums (atomics, fragment layout) differs;
  2. a float64 In^T . ((dZ . Wx^T)_bf16 * [X > 0]) at the bound of test_fc_bwd_bench_chunk;
  3. the same float64 reference with planted defects (mask ignored, mask from the wrong row, the wrong agent's observation
     slice), each of which must land far outside that bound;
and it must leave G outside the fc blocks untouched.  Shapes: the bench chunk (grid MA2C, 50 units, 120 x 1024 rows,
dx = 224), Monaco (dx = 192, 40 x 1024), IA2C (dx = 160), a ragged chunk (rc = 1000) and rc = 40."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

BOUND = 2e-3          # test_fc_bwd_bench_chunk: max-abs error relative to the block's max-abs
BLOCKS = ("fcw", "fcf", "fct")


def _grid_model():
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    net = build_large_grid(agent="ma2c")
    lay = PolicyLayout(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, net.node_obs_off, net.n_obs, fw=128, ft=32, ff=64,
                       h=64, max_na=net.max_na)
    return lay, BatchedA2C(lay, 8, n_step=2, seed=3)


def _small_model(ff):
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from tests.test_learner_gpu import _layout
    lay = _layout(ff)
    return lay, BatchedA2C(lay, 8, n_step=2, seed=5)


def _inputs(lay, T, rc, R, seed):
    """dZ, X (bf16 [U][T*rc][.]), obs [T][R][n_obs] whose replicas r0 = R - rc .. R - 1 are the chunk's rows."""
    U, dx, M = lay.U, lay.dx, T * rc
    g = torch.Generator(device="cuda").manual_seed(seed)
    obs = torch.rand(T, R, lay.n_obs, device="cuda", generator=g) * 2
    Xb = torch.relu(torch.randn(U, M, dx, device="cuda", generator=g)).to(torch.bfloat16)
    dZb = (torch.randn(U, M, 256, device="cuda", generator=g) * 1e-2).to(torch.bfloat16)
    return obs, Xb, dZb


def _fused(m, lay, obs, Xb, dZb, T, rc, R):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    G = torch.zeros_like(m.G)
    _lib.check(_lib.lib().tscl_dx_fc_bwd_tc(m._h, _p(obs[0, R - rc:]), _p(Xb), _p(dZb), _p(m.Wxt), C.c_int64(T * rc),
                                            C.c_int64(rc), C.c_int64(R * lay.n_obs), _p(G), m._st()))
    torch.cuda.synchronize()
    return G


def _two_kernel(m, lay, obs, Xb, dZb, T, rc, R):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    M = T * rc
    G = torch.zeros_like(m.G)
    dXb = torch.empty(lay.U, M, lay.dx, dtype=torch.bfloat16, device="cuda")
    _lib.check(_lib.lib().tscl_dx_tc(m._h, _p(dZb), _p(m.Wxt), _p(dXb), C.c_int64(M), m._st()))
    _lib.check(_lib.lib().tscl_fc_bwd_tc(m._h, _p(obs[0, R - rc:]), None, _p(Xb), None, _p(dXb), C.c_int64(M),
                                         C.c_int64(rc), C.c_int64(R * lay.n_obs), _p(G), C.c_int32(0), m._st()))
    torch.cuda.synchronize()
    del dXb
    return G


def _groups(lay, G):
    """fc weight / bias blocks of every unit, concatenated per block kind: {"fcw_w": flat tensor, ...}"""
    gv = lay.views(G)
    out = {}
    for name in BLOCKS:
        for kind in ("w", "b"):
            parts = [gv["%s_%s%d" % (name, kind, u)].reshape(-1) for u in range(lay.U)]
            if sum(p.numel() for p in parts):
                out["%s_%s" % (name, kind)] = torch.cat(parts)
    return out


def _worst_vs_f64(m, lay, obs, Xb, dZb, G, T, rc, R, defect=None):
    """max over units and blocks of max|G - ref| / max|ref|, ref = In^T . ((dZ . Wx^T)_bf16 * [X > 0]) in float64."""
    gv = lay.views(G)
    M = T * rc
    ob = obs[:, R - rc:].reshape(M, lay.n_obs).to(torch.bfloat16).double()
    wx = m.pv["wx"].to(torch.bfloat16).double()                 # [U][dx][256]
    worst = 0.0
    for u in range(lay.U):
        a = u // 2
        if defect == "agent":
            a = (a + 1) % lay.A
        o0, nw, nt, nf = int(lay.obs_off[a]), int(lay.n_wave[a]), int(lay.n_wait[a]), int(lay.n_fp[a])
        dx = (dZb[u].double() @ wx[u].T).float().to(torch.bfloat16).double()
        x = Xb[u]
        if defect == "row":
            x = torch.roll(x, 1, dims=0)
        dd = dx if defect == "mask" else dx * (x > 0)
        blocks = [("fcw", ob[:, o0:o0 + nw], dd[:, :lay.fw]),
                  ("fcf", ob[:, o0 + nw + nt:o0 + nw + nt + nf], dd[:, lay.fw:lay.fw + lay.ff]),
                  ("fct", ob[:, o0 + nw:o0 + nw + nt], dd[:, lay.fw + lay.ff:])]
        for name, inp, d_ in blocks:
            if d_.shape[1] == 0:
                continue
            w_tc, b_tc = gv["%s_w%d" % (name, u)].double(), gv["%s_b%d" % (name, u)].double()
            if inp.shape[1] != w_tc.shape[0]:      # the wrong agent's slice has another width: compare the common rows
                k = min(inp.shape[1], w_tc.shape[0])
                inp, w_tc = inp[:, :k], w_tc[:k]
            w_ref, b_ref = inp.T @ d_, d_.sum(0)
            for got, ref in ((w_tc, w_ref), (b_tc, b_ref)):
                if ref.numel():
                    worst = max(worst, float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-12)))
    return worst


def _check_untouched(lay, G):
    for k, v in lay.views(G).items():
        if not k.startswith(BLOCKS):
            assert not bool(v.any()), k


CASES = [("grid", 120, 1024, 1024), ("monaco", 40, 1024, 1024), (0, 120, 1024, 1024), ("grid", 120, 1000, 1024),
         (64, 40, 40, 64), ("monaco", 40, 1000, 1030)]


@pytest.mark.parametrize("which,T,rc,R", CASES)
def test_fused_matches_two_kernel_path_and_f64(which, T, rc, R):
    lay, m = _grid_model() if which == "grid" else _small_model(which)
    assert lay.dx in (160, 192, 224) and m.dx_fc_fused
    obs, Xb, dZb = _inputs(lay, T, rc, R, seed=31 + T + rc)
    G = _fused(m, lay, obs, Xb, dZb, T, rc, R)
    G2 = _two_kernel(m, lay, obs, Xb, dZb, T, rc, R)
    assert torch.isfinite(G).all()
    fused, ref = _groups(lay, G), _groups(lay, G2)
    rel = {k: float((fused[k] - ref[k]).norm() / ref[k].norm().clamp_min(1e-30)) for k in ref}
    print("dx=%d T=%d rc=%d: rel-L2 vs tscl_dx_tc + tscl_fc_bwd_tc %s" %
          (lay.dx, T, rc, " ".join("%s %.2e" % kv for kv in rel.items())))
    assert max(rel.values()) <= 5e-7, rel
    _check_untouched(lay, G)
    worst = _worst_vs_f64(m, lay, obs, Xb, dZb, G, T, rc, R)
    print("dx=%d T=%d rc=%d: worst block vs float64 %.2e" % (lay.dx, T, rc, worst))
    assert worst < BOUND, worst


@pytest.mark.parametrize("defect", ["mask", "row", "agent"])
def test_planted_defects_leave_the_bound(defect):
    """The float64 reference with one defect planted must miss the kernel's result by far more than BOUND."""
    lay, m = _small_model(64)
    T, rc, R = 40, 256, 256
    obs, Xb, dZb = _inputs(lay, T, rc, R, seed=77)
    G = _fused(m, lay, obs, Xb, dZb, T, rc, R)
    assert _worst_vs_f64(m, lay, obs, Xb, dZb, G, T, rc, R) < BOUND
    off = _worst_vs_f64(m, lay, obs, Xb, dZb, G, T, rc, R, defect=defect)
    print("defect %s: %.2e" % (defect, off))
    assert off > 50 * BOUND, off
