"""GPU: the fused policy forward (tscl_policy_step_v2 / _v2r) at the bench shapes, activation store on.

The other policy-forward tests run at R = 300 and 515: one or two work items per CTA.  Here the grid (R = 4096, dx = 224)
and Monaco (R = 2048, dx = 192) give every CTA many items, unit changes in the middle of a CTA's range, and store
chunks (1024 replicas) beyond the first.  Every output is compared with a torch restatement of the same bf16 arithmetic
(tolerances as in test_policy_tc_gpu.py: only the summation order and the MUFU tanh differ), and replica-range launches
must reproduce one full launch bit for bit."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CHUNK, T, SLOT = 1024, 2, 1


def _model(scenario, R):
    from bench import build_scenario, make_layout
    from deeprl_signal_control_b200.agents.learner import BatchedA2C

    class A:
        agent, policy = "ma2c", "lstm"
    A.scenario = scenario
    lay = make_layout(build_scenario(A)[0], A)
    m = BatchedA2C(lay, R, n_step=T, seed=5, chunk=CHUNK, store_acts=True)
    assert m.tc_v2 and m.store_acts
    return lay, m


def _pmix(h):
    h = h ^ (h >> np.uint32(16)); h = h * np.uint32(0x7feb352d); h = h ^ (h >> np.uint32(15))
    h = h * np.uint32(0x846ca68b); return h ^ (h >> np.uint32(16))


def _reference_actions(pi, n_a, seed, step, replica0):
    """inverse-CDF sample of the kernel: hash of (seed, step, replica, agent), cumulative sum of pi in fp32"""
    with np.errstate(over="ignore"):
        R, A, _ = pi.shape
        r = np.arange(R, dtype=np.uint64) + np.uint64(replica0)
        h0 = _pmix(np.uint32(seed & 0xFFFFFFFF) ^ (np.uint32(step) * np.uint32(0x9E3779B1)))
        h1 = _pmix(h0 ^ np.uint32(seed >> 32) ^ (r.astype(np.uint32) * np.uint32(0x85EBCA77)))
        act = np.zeros((R, A), np.int32)
        for a in range(A):
            h = _pmix(h1 ^ np.uint32(a * 0xC2B2AE3D & 0xFFFFFFFF))
            uu = (h >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
            na = int(n_a[a])
            cum = np.cumsum(pi[:, a, :na], axis=1, dtype=np.float32)
            hit = uu[:, None] < cum
            act[:, a] = np.where(hit.any(1), hit.argmax(1), na - 1)
    return act


@pytest.fixture
def no_tf32():
    """fp32 reference products: TF32 off for the test, the process-wide flag restored afterwards"""
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = saved


def _check_step(lay, m, obs, done, c_prev, h_prev, zdbg, step):
    U, R, H = lay.U, m.R, lay.h
    v = lay.views(m.P)
    bf = lambda t: t.to(torch.bfloat16).float()
    ob = bf(obs)
    # fc front end and X (bf16, as stored in st_x)
    Xs = []
    for u in range(U):
        a = u // 2
        o0 = int(lay.obs_off[a]); nw, nt, nf = int(lay.n_wave[a]), int(lay.n_wait[a]), int(lay.n_fp[a])
        parts = [torch.relu(ob[:, o0:o0 + nw] @ bf(v["fcw_w%d" % u]) + v["fcw_b%d" % u])]
        if lay.ff > 0:
            parts.append(torch.relu(ob[:, o0 + nw + nt:o0 + nw + nt + nf] @ bf(v["fcf_w%d" % u]) + v["fcf_b%d" % u]))
        if lay.ft > 0:
            parts.append(torch.relu(ob[:, o0 + nw:o0 + nw + nt] @ bf(v["fct_w%d" % u]) + v["fct_b%d" % u]))
        Xs.append(torch.cat(parts, 1))
    X = bf(torch.stack(Xs))
    st = lambda s: s[:, :, SLOT].transpose(0, 1).reshape(U, R, -1).float()     # [R/rc][U][rc][w] -> [U][R][w]
    st_x = st(m.st_x)
    # the fp32 sums differ in order only: a rounding flip moves an element by at most one bf16 ulp (<= 2^-7 |x|)
    assert bool(((st_x - X).abs() <= X.abs() * 2 ** -7 + 1e-6).all())
    assert float((st_x != X).float().mean()) < 1e-2
    # gate accumulators, from the kernel's own X (st_x) and the bf16 h_{t-1}
    hp = torch.zeros_like(h_prev) if done else h_prev
    cp = torch.zeros_like(c_prev) if done else c_prev
    z_ref = torch.bmm(st_x, bf(v["wx"])) + torch.bmm(bf(hp), bf(v["wh"]))
    assert float((zdbg - z_ref).abs().max()) < 2e-2 and float((zdbg - z_ref).abs().mean()) < 1e-4
    # LSTM cell from the kernel's accumulators
    zb = zdbg + v["bl"][:, None, :]
    gi, gf, go, gu = torch.sigmoid(zb[..., :H]), torch.sigmoid(zb[..., H:2 * H]), torch.sigmoid(zb[..., 2 * H:3 * H]), \
        torch.tanh(zb[..., 3 * H:])
    c_ref = gf * cp + gi * gu
    h_ref = go * torch.tanh(c_ref)
    torch.testing.assert_close(m.c_tmp, c_ref, rtol=0, atol=5e-3)
    torch.testing.assert_close(m.h_tmp, h_ref, rtol=0, atol=5e-3)
    torch.testing.assert_close(st(m.st_g), bf(torch.cat([gi, gf, go, gu], -1)), rtol=0, atol=1e-2)
    torch.testing.assert_close(st(m.st_c), bf(m.c_tmp), rtol=0, atol=0)
    torch.testing.assert_close(st(m.st_h), bf(m.h_tmp), rtol=0, atol=0)
    # heads from the kernel's h
    lg = torch.bmm(m.h_tmp, v["wo"]) + v["bo"][:, None, :]           # [U][R][max_na]
    for a in range(lay.A):
        na = int(lay.n_a[a])
        p_ref = torch.softmax(lg[2 * a, :, :na], -1)
        torch.testing.assert_close(m.pi[:, a, :na], p_ref, rtol=0, atol=2e-4)
        torch.testing.assert_close(m.val[:, a], lg[2 * a + 1, :, 0], rtol=0, atol=2e-4)
    act_ref = _reference_actions(m.pi.cpu().numpy(), lay.n_a, m.seed, step, 0)
    assert np.array_equal(m.act.cpu().numpy(), act_ref)


@pytest.mark.parametrize("scenario,R", [("large_grid", 4096), ("real_net", 2048)])
def test_fused_forward_at_bench_size(scenario, R, no_tf32):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    lay, m = _model(scenario, R)
    g = torch.Generator(device="cuda").manual_seed(1)
    m.h_fw.copy_(torch.rand(m.h_fw.shape, device="cuda", generator=g) * 2 - 1)
    m.c_fw.copy_(torch.randn(m.c_fw.shape, device="cuda", generator=g))
    zdbg = torch.zeros(lay.U, R, 4 * lay.h, device="cuda")
    for step, done in enumerate([False, True, False]):
        obs = torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2
        for t in (m.st_x, m.st_g, m.st_c, m.st_h):
            t.fill_(float("nan"))
        c_prev, h_prev = m.c_fw.clone(), m.h_fw.clone()
        _lib.check(_lib.lib().tscl_policy_step_v2(
            m._h, _p(m.P), _p(m.Wp), _p(obs), C.c_int64(R), _p(m.c_fw), _p(m.h_fw), _p(m.c_tmp), _p(m.h_tmp), _p(m.pi),
            _p(m.val), _p(m.act), C.c_int32(int(done)), C.c_uint64(m.seed), C.c_int64(step), C.c_int64(0), _p(zdbg),
            _p(m.st_x), _p(m.st_g), _p(m.st_c), _p(m.st_h), C.c_int32(SLOT), C.c_int32(T), C.c_int64(CHUNK), m._st()))
        torch.cuda.synchronize()
        _check_step(lay, m, obs, done, c_prev, h_prev, zdbg, step)
        m.c_fw.copy_(m.c_tmp); m.h_fw.copy_(m.h_tmp)


@pytest.mark.parametrize("scenario,R", [("large_grid", 4096), ("real_net", 2048)])
def test_replica_ranges_match_one_launch(scenario, R):
    lay, m = _model(scenario, R)
    g = torch.Generator(device="cuda").manual_seed(2)
    m.h_fw.copy_(torch.rand(m.h_fw.shape, device="cuda", generator=g) * 2 - 1)
    m.c_fw.copy_(torch.randn(m.c_fw.shape, device="cuda", generator=g))
    m.obs_hist[SLOT].copy_(torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2)
    c0, h0 = m.c_fw.clone(), m.h_fw.clone()
    outs = []
    # four ranges with starts that are not multiples of the 64-row work item: items straddle store chunks
    for bounds in ([0, R], [0, R // 4 - 24, R // 2 + 52, 3 * R // 4 + 7, R]):
        m.c_fw.copy_(c0); m.h_fw.copy_(h0)
        for t in (m.st_x, m.st_g, m.st_c, m.st_h, m.pi, m.val):
            t.fill_(float("nan"))
        m.act.fill_(-1)
        for r0, r1 in zip(bounds[:-1], bounds[1:]):
            m.forward_range(r0, r1 - r0, False, SLOT, 9)
        torch.cuda.synchronize()
        outs.append([x.clone() for x in (m.c_fw, m.h_fw, m.pi, m.val, m.act, m.st_x[:, :, SLOT], m.st_g[:, :, SLOT],
                                         m.st_c[:, :, SLOT], m.st_h[:, :, SLOT])])
    for a, b in zip(*outs):
        assert torch.equal(a, b)
