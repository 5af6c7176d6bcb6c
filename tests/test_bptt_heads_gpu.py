"""GPU: tscl_lstm_seq_bwd_tc_heads, the BPTT kernel that computes the loss gradients at the heads itself, against the pair
it replaces (tscl_heads_loss on the bf16 store followed by the store-path tscl_lstm_seq_bwd_tc), chunk by chunk.

  * dZ is bit-identical, launched once per chunk and launched once over every chunk;
  * the head weight / bias gradients and agent 0's loss sums agree up to summation order;
  * nothing past the dZ of the last chunk is written.

Shapes: the bench's 5x5 grid MA2C (4 chunks of 1024 replicas, T = 120), Monaco MA2C (T = 40), grid IA2C (dx = 160), a
ragged Rc = 1000 and Rc = 40 (one partial 128-row tile).  Agent 0's action 1 has a logit bias of -40, so pi_1 < 1e-10
on every row and the clip rule of log(clip(pi, 1e-10, 1)) is exercised."""
import ctypes as C

import pytest
import torch

from tests.test_update_bench_size_gpu import _model

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _free_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _inputs(m, T, Rc, nc, done_steps, seed):
    lay = m.lay
    U, A = lay.U, lay.A
    R = nc * Rc
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = lay.views(m.P)
    for u in range(U):           # wider heads than the initialisation, so that the policies are not near-uniform
        n_out = int(lay.n_a[u // 2]) if u % 2 == 0 else 1
        v["wo"][u][:, :n_out] = torch.randn(64, n_out, device="cuda", generator=g) * 0.5
        v["bo"][u][:n_out] = torch.randn(n_out, device="cuda", generator=g) * 0.1
    v["bo"][0][1] = -40.0
    m.pack_weights()
    gates = torch.empty(nc, U, T, Rc, 256, dtype=torch.bfloat16, device="cuda")
    for ci in range(nc):
        z = torch.randn(U, T, Rc, 256, device="cuda", generator=g) * 1.5
        gates[ci] = torch.cat([torch.sigmoid(z[..., :192]), torch.tanh(z[..., 192:])], -1).to(torch.bfloat16)
        del z
    cb = (torch.randn(nc, U, T, Rc, 64, device="cuda", generator=g) * 0.8).to(torch.bfloat16)
    hb = torch.tanh(torch.randn(nc, U, T, Rc, 64, device="cuda", generator=g) * 1.5).to(torch.bfloat16)
    c_bw = torch.randn(U, R, 64, device="cuda", generator=g) * 0.5
    done = torch.zeros(T, device="cuda")
    done[list(done_steps)] = 1.0
    na = torch.as_tensor(lay.n_a, device="cuda")
    act = (torch.rand(T, R, A, device="cuda", generator=g) * na).long().clamp_max(na - 1).to(torch.int32)
    act[::3, :, 0] = 1                                          # taken action with pi < 1e-10
    act[1::5] = (na - 1).to(torch.int32)
    Rs = torch.randn(T, R, A, device="cuda", generator=g) * 2
    Adv = torch.randn(T, R, A, device="cuda", generator=g) * 2
    Adv[2::7] = 0.0
    return dict(gates=gates, cb=cb, hb=hb, c_bw=c_bw, done=done, act=act, Rs=Rs, Adv=Adv)


@pytest.mark.parametrize("kind,T,Rc,nc,done_steps", [
    ("grid", 120, 1024, 4, (37, 90)),          # the bench: R = 4096 in chunks of 1024
    ("monaco", 40, 1024, 2, (0, 39)),
    ("grid_ia2c", 120, 1024, 2, tuple(range(120))),
    ("grid", 120, 1000, 2, (37, 90)),
    ("grid", 120, 40, 3, (0, 119)),
])
def test_bptt_heads_matches_two_kernels(kind, T, Rc, nc, done_steps):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    lib = _lib.lib()
    lay, m = _model(kind)
    U, A = lay.U, lay.A
    R = nc * Rc
    x = _inputs(m, T, Rc, nc, done_steps, seed=41)
    scale, v_coef, beta = 1.0 / (T * R), 0.5, 0.01
    M = T * Rc

    # the two-kernel pair, chunk by chunk
    G2, st2 = torch.zeros_like(m.G), torch.zeros(4, device="cuda")
    dZ2 = torch.empty(nc, U, M, 256, dtype=torch.bfloat16, device="cuda")
    dH = torch.empty(U, M, 64, device="cuda")
    for ci in range(nc):
        r0 = ci * Rc
        _lib.check(lib.tscl_heads_loss(m._h, _p(m.P), None, _p(x["act"][0, r0:]), _p(x["Rs"][0, r0:]),
                                       _p(x["Adv"][0, r0:]), C.c_int64(M), C.c_int64(Rc), C.c_int64(R * A),
                                       C.c_float(v_coef), C.c_float(beta), C.c_float(scale), None, _p(dH), _p(st2),
                                       _p(x["hb"][ci]), _p(G2), m._st()))
        _lib.check(lib.tscl_lstm_seq_bwd_tc(m._h, _p(m.Wt), None, None, _p(dH), _p(x["c_bw"]), _p(x["done"]),
                                            C.c_int32(T), C.c_int64(Rc), C.c_int64(R), C.c_int64(r0), _p(x["gates"][ci]),
                                            _p(x["cb"][ci]), _p(dZ2[ci]), m._st()))
    del dH

    def fused(r0, n_chunks, dz, G, st):
        ci = r0 // Rc
        _lib.check(lib.tscl_lstm_seq_bwd_tc_heads(
            m._h, _p(m.Wt), _p(m.P), _p(x["gates"][ci]), _p(x["cb"][ci]), _p(x["hb"][ci]), _p(x["c_bw"]), _p(x["done"]),
            _p(x["act"][0, r0:]), _p(x["Rs"][0, r0:]), _p(x["Adv"][0, r0:]), C.c_int32(T), C.c_int64(Rc),
            C.c_int32(n_chunks), C.c_int64(R), C.c_int64(r0), C.c_int64(R * A), C.c_float(v_coef), C.c_float(beta),
            C.c_float(scale), _p(dz), _p(st), _p(G), m._st()))

    # one launch per chunk
    G1, st1 = torch.zeros_like(m.G), torch.zeros(4, device="cuda")
    dz1 = torch.empty(U, M, 256, dtype=torch.bfloat16, device="cuda")
    for ci in range(nc):
        fused(ci * Rc, 1, dz1, G1, st1)
        torch.cuda.synchronize()
        assert torch.equal(dz1.view(torch.int16), dZ2[ci].view(torch.int16)), "chunk %d" % ci
    del dz1

    # one launch over every chunk, into a buffer with a guard region behind the last chunk
    guard = 1 << 16
    flat = torch.full((nc * U * M * 256 + guard,), -7.0, dtype=torch.bfloat16, device="cuda")
    Ga, sta = torch.zeros_like(m.G), torch.zeros(4, device="cuda")
    fused(0, nc, flat, Ga, sta)
    torch.cuda.synchronize()
    dza = flat[:nc * U * M * 256].view(nc, U, M, 256)
    for ci in range(nc):
        assert torch.equal(dza[ci].view(torch.int16), dZ2[ci].view(torch.int16)), "all-chunk launch, chunk %d" % ci
    assert bool((flat[nc * U * M * 256:] == -7.0).all()), "written past the last chunk"

    # head gradients and loss sums: the same terms, summed in another order
    g2 = lay.views(G2)
    worst = {"wo": 0.0, "bo": 0.0}
    for name, Gx in (("per-chunk", G1), ("all-chunk", Ga)):
        gx = lay.views(Gx)
        for key in ("wo", "bo"):
            ref = g2[key].double()
            d = ((gx[key].double() - ref).abs().max() / ref.abs().max()).item()
            worst[key] = max(worst[key], d)
        others = torch.ones_like(G2, dtype=torch.bool)
        others[lay.off_wo:int(lay.off_fcw_w[0])] = False
        assert not bool(Gx[others].any()), name              # only the heads' gradients are written
    print("OBSERVED %s: head gradients max |d| / max |ref| wo %.2e bo %.2e; stats %s vs %s vs %s" % (
        kind, worst["wo"], worst["bo"], st2[:3].tolist(), st1[:3].tolist(), sta[:3].tolist()))
    # observed on an H100 80GB HBM3 (700 W): wo 4.9e-7 .. 1.5e-6 (Rc = 40), bo 2.1e-7 .. 1.1e-6
    assert worst["wo"] <= 5e-6 and worst["bo"] <= 5e-6, worst
    torch.testing.assert_close(st1[:3], st2[:3], rtol=1e-4, atol=0)
    torch.testing.assert_close(sta[:3], st2[:3], rtol=1e-4, atol=0)
