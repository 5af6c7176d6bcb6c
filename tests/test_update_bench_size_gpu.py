"""GPU: the tensor-core A2C update from the bf16 activation store at the bench's chunk shape (1024 replicas x 120 steps on
the 5x5 grid, 50 units; x 40 steps on Monaco, 56 units), kernel by kernel and as a whole, against the float64 reference of
oracle/learner_ref.py (heads_ref, bptt_ref, lstm_grads_ref, fc_grads_ref, update_ref), which rounds to bf16 exactly where
the kernels do.  tests/test_update_reference_cpu.py pins that reference to autograd of a2c_loss.

Bounds are about 3x the worst value seen on an H100 80GB HBM3 (400 W power limit); the observed values are given beside
each bound.  Every test frees its device memory when it ends."""
import ctypes as C
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# BPTT dZ against bptt_ref, worst over (unit, time step): rel-L2 and max |delta| / max |ref|.  Observed on the H100:
# rel-L2 1.70e-3 (grid, Monaco, Rc = 1000) and 1.93e-3 (Rc = 40), max 3.78e-3 .. 3.87e-3 (bf16 rounding of dZb plus
# tanh.approx).  The planted defects of bptt_mutations move it by 0.31 (c0 row) to 1.42 (dH shifted): >= 52x the bound.
DZ_REL_L2 = 6e-3
DZ_MAX = 1.2e-2


def dz_errors(got, ref):
    """(rel-L2, max |delta| / max |ref|) of dZ [U, T, rc, 4h], each the worst over (unit, time step)."""
    diff = (got - ref).flatten(2)
    r = ref.flatten(2)
    return ((diff.norm(dim=2) / r.norm(dim=2)).max().item(),
            (diff.abs().amax(2) / r.abs().amax(2)).max().item())


@pytest.fixture(autouse=True)
def _free_device_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    print("peak device memory %.2f GB" % (torch.cuda.max_memory_allocated() / 2 ** 30))
    torch.cuda.empty_cache()


def _layout(kind):
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    if kind == "monaco":
        from deeprl_signal_control_b200.net.real_net import real_net_tables
        net, ff = real_net_tables("ma2c"), 64
    else:
        from deeprl_signal_control_b200.net.large_grid import build_large_grid
        net, ff = (build_large_grid(agent="ia2c"), 0) if kind == "grid_ia2c" else (build_large_grid(agent="ma2c"), 64)
    return PolicyLayout(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, net.node_obs_off, net.n_obs, fw=128, ft=32, ff=ff,
                        h=64, max_na=net.max_na)


def _model(kind, **kw):
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    lay = _layout(kind)
    return lay, BatchedA2C(lay, kw.pop("R", 8), n_step=kw.pop("n_step", 2), seed=kw.pop("seed", 3), **kw)


def _bptt_inputs(U, T, Rc, ld, done_steps, seed):
    """Store-path BPTT operands: gate activations / c as bf16 [U][T*Rc][w], dH fp32, c_bw [U][ld][64], done [T]."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(U, T * Rc, 256, device="cuda", generator=g) * 1.5
    gates = torch.cat([torch.sigmoid(z[..., :192]), torch.tanh(z[..., 192:])], -1).to(torch.bfloat16)
    del z
    cb = (torch.randn(U, T * Rc, 64, device="cuda", generator=g) * 0.8).to(torch.bfloat16)
    dH = torch.randn(U, T * Rc, 64, device="cuda", generator=g) * 1e-3
    c_bw = torch.randn(U, ld, 64, device="cuda", generator=g) * 0.5
    done = torch.zeros(T, device="cuda")
    done[list(done_steps)] = 1.0
    return gates, cb, dH, c_bw, done


def _run_bptt(m, gates, cb, dH, c_bw, done, T, Rc, ld, r0, fused_dx=False):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    U = m.lay.U
    dZb = torch.empty(U, T * Rc, 256, dtype=torch.bfloat16, device="cuda")
    dXb = torch.empty(U, T * Rc, m.lay.dx, dtype=torch.bfloat16, device="cuda") if fused_dx else None
    _lib.check(_lib.lib().tscl_lstm_seq_bwd_tc_dx(
        m._h, _p(m.Wt), None, None, _p(dH), _p(c_bw), _p(done), C.c_int32(T), C.c_int64(Rc), C.c_int64(ld),
        C.c_int64(r0), _p(gates), _p(cb), _p(dZb), _p(m.Wxt) if fused_dx else None, _p(dXb), m._st()))
    torch.cuda.synchronize()
    return dZb, dXb


def _bptt_reference(m, gates, cb, dH, c_bw, done, T, Rc, r0, units, **kw):
    from oracle.learner_ref import bptt_ref
    d = lambda x: x[units].double().reshape(len(range(*units.indices(m.lay.U))), T, Rc, -1)
    return bptt_ref(d(gates), d(cb), c_bw[units, r0:r0 + Rc].double(), d(dH), done.tolist(),
                    m.pv["wh"][units].double(), **kw)


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,T,Rc,ld,r0", [("grid", 120, 1024, 2048, 1024), ("monaco", 40, 1024, 2048, 1024),
                                             ("grid", 120, 1000, 3000, 1000), ("grid", 120, 40, 80, 40)])
def test_bptt_matches_float64_reference(kind, T, Rc, ld, r0):
    """tscl_lstm_seq_bwd_tc as the update calls it (gates / c from the bf16 store, dZ written as bf16 only) vs bptt_ref.
    Shapes: the bench chunk at r0 = 1024; Monaco; a ragged Rc = 1000 at r0 = 1000; Rc = 40, one partial 128-row tile
    whose TMA boxes read past the rows of the chunk (and, for the last unit, past the end of the tensors).
    Done patterns {37, 90} (interior) and {0, T-1}."""
    from oracle.learner_ref import bptt_mutations, bptt_ref
    lay, m = _model(kind)
    U = lay.U
    worst_l2 = worst_max = 0.0
    mutation = {}
    for pat, steps in enumerate([(37 % T, 90 % T), (0, T - 1)]):
        gates, cb, dH, c_bw, done = _bptt_inputs(U, T, Rc, ld, steps, seed=10 + pat)
        dZb, _ = _run_bptt(m, gates, cb, dH, c_bw, done, T, Rc, ld, r0)
        for u0 in range(0, U, 10):
            us = slice(u0, min(U, u0 + 10))
            ref = _bptt_reference(m, gates, cb, dH, c_bw, done, T, Rc, r0, us)
            l2, mx = dz_errors(dZb[us].double().reshape(ref.shape), ref)
            worst_l2, worst_max = max(worst_l2, l2), max(worst_max, mx)
            del ref
        if kind == "grid" and Rc == 1024 and pat == 0:
            # every planted defect, on units 0 and 1, moves dZ by >= 10x the bound
            us = slice(0, 2)
            d = lambda x: x[us].double().reshape(2, T, Rc, -1)
            ok, mutants = bptt_mutations(d(gates), d(cb), c_bw[us].double(), r0, d(dH), done.tolist())
            wh = m.pv["wh"][us].double()
            ref = bptt_ref(**ok, wh=wh)
            for name, kw in mutants.items():
                mutation[name] = dz_errors(bptt_ref(**kw, wh=wh), ref)[0]
                print("OBSERVED mutation %-32s rel-L2 %.3e = %.0fx the bound" % (name, mutation[name],
                                                                                mutation[name] / DZ_REL_L2))
            del ok, mutants, ref
        del gates, cb, dH, c_bw, done, dZb
    print("OBSERVED bptt %s T=%d Rc=%d r0=%d: per (unit, step) rel-L2 %.3e, max|d|/max|ref| %.3e" % (
        kind, T, Rc, r0, worst_l2, worst_max))
    assert worst_l2 <= DZ_REL_L2 and worst_max <= DZ_MAX, (worst_l2, worst_max)
    for name, rel in mutation.items():
        assert rel >= 10 * DZ_REL_L2, (name, rel)


# ------------------------------------------------------------------------------------------------------------------
VARIANT_SHAPE = dict(T=120, Rc=300, ld=600, r0=300)


def _variant_digest(out_path):
    """Run the store-path BPTT at VARIANT_SHAPE on seeded inputs; write the sha256 of dZb to out_path (run in a fresh
    process: the kernel-selection switches are read once per process)."""
    s = VARIANT_SHAPE
    lay, m = _model("grid")
    gates, cb, dH, c_bw, done = _bptt_inputs(lay.U, s["T"], s["Rc"], s["ld"], (37, 90), seed=5)
    dZb, _ = _run_bptt(m, gates, cb, dH, c_bw, done, s["T"], s["Rc"], s["ld"], s["r0"])
    with open(out_path, "w") as f:
        f.write(hashlib.sha256(dZb.view(torch.int16).cpu().numpy().tobytes()).hexdigest())


def test_bptt_variants_are_bit_identical(tmp_path):
    """The cp.async staged kernel (TSC_BPTT_TMA=0: also what runs when the driver has no cuTensorMapEncodeTiled), the
    unstaged kernel (TSC_BPTT_STAGED=0) and the 256-thread kernel (TSC_BPTT_THREADS=256) give the dZb of the default
    (TMA-staged) kernel bit for bit."""
    digests = {}
    for name, env in [("default", {}), ("TSC_BPTT_TMA=0", {"TSC_BPTT_TMA": "0"}),
                      ("TSC_BPTT_STAGED=0", {"TSC_BPTT_STAGED": "0"}), ("TSC_BPTT_THREADS=256", {"TSC_BPTT_THREADS": "256"})]:
        out = tmp_path / ("%d.sha" % len(digests))
        e = {k: v for k, v in os.environ.items() if not k.startswith("TSC_BPTT_")}
        e.update(env)
        r = subprocess.run([sys.executable, "-c", "import sys; from tests.test_update_bench_size_gpu import _variant_digest; "
                            "_variant_digest(sys.argv[1])", str(out)], cwd=ROOT, env=e, capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, (name, r.stderr[-3000:])
        digests[name] = out.read_text()
    assert len(set(digests.values())) == 1, digests


@pytest.mark.parametrize("kind", ["grid", "monaco", "grid_ia2c"])
def test_fused_dx_bptt(kind):
    """tscl_lstm_seq_bwd_tc_dx with the Wx^T image (what `dx_fused = True` runs; dx = 224 / 192 / 160): dZb is bit-identical
    to the default kernel's, and dXb is the float64 product bf16(dZb) . bf16(Wx)^T rounded to bf16: within one bf16 ulp."""
    s = VARIANT_SHAPE
    lay, m = _model(kind)
    assert m.dx_fusable and lay.dx == {"grid": 224, "monaco": 192, "grid_ia2c": 160}[kind]
    gates, cb, dH, c_bw, done = _bptt_inputs(lay.U, s["T"], s["Rc"], s["ld"], (37, 90), seed=6)
    dZ0, _ = _run_bptt(m, gates, cb, dH, c_bw, done, s["T"], s["Rc"], s["ld"], s["r0"])
    dZ1, dXb = _run_bptt(m, gates, cb, dH, c_bw, done, s["T"], s["Rc"], s["ld"], s["r0"], fused_dx=True)
    assert torch.equal(dZ0.view(torch.int16), dZ1.view(torch.int16))
    wx = m.pv["wx"].to(torch.bfloat16).double()
    worst = 0.0
    for u in range(lay.U):
        ref = dZ1[u].double() @ wx[u].T
        err = (dXb[u].double() - ref).abs()
        ulp = ref.abs() * 2.0 ** -7 + 1e-6 * ref.abs().max()           # one bf16 ulp of the value, at most
        worst = max(worst, (err / ulp).max().item())
    print("OBSERVED fused dX %s: max |d| = %.3f of the one-ulp bound" % (kind, worst))
    assert worst <= 1.0, worst           # observed 0.498: the exact product rounded to nearest


# ------------------------------------------------------------------------------------------------------------------
def test_heads_loss_bench_chunk():
    """tscl_heads_loss on the store path (h from the bf16 store, head gradients fused) for the second chunk of R = 2048
    (M = 122 880 rows, stride_t = R * A, r0 = 1024), vs heads_ref.  Planted rows: agent 0's action 1 has a logit bias of
    -40, so pi_1 < 1e-10 on every row and rows that took it get no policy gradient (TF clip); rows that took action
    n_a - 1; rows with Adv = 0.  dH, wo, bo relative to each tensor's max (bounds below); stats rtol 1e-4; nothing else
    in G moves."""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    from oracle.learner_ref import heads_ref
    T, R, rc, r0 = 120, 2048, 1024, 1024
    M = T * rc
    lay, m = _model("grid")
    U, A = lay.U, lay.A
    g = torch.Generator(device="cuda").manual_seed(31)
    v = lay.views(m.P)
    for u in range(U):           # wider heads than the initialisation, so that the policies are not near-uniform
        n_out = int(lay.n_a[u // 2]) if u % 2 == 0 else 1
        v["wo"][u][:, :n_out] = torch.randn(64, n_out, device="cuda", generator=g) * 0.5
        v["bo"][u][:n_out] = torch.randn(n_out, device="cuda", generator=g) * 0.1
    v["bo"][0][1] = -40.0
    Hb = torch.tanh(torch.randn(U, T, rc, 64, device="cuda", generator=g) * 1.5).to(torch.bfloat16)
    na = torch.as_tensor(lay.n_a, device="cuda")
    act = (torch.rand(T, R, A, device="cuda", generator=g) * na).long().clamp_max(na - 1).to(torch.int32)
    act[::3, :, 0] = 1                                          # taken action with pi < 1e-10
    act[1::5] = (na - 1).to(torch.int32)                        # last action of every agent
    Rs = torch.randn(T, R, A, device="cuda", generator=g) * 2
    Adv = torch.randn(T, R, A, device="cuda", generator=g) * 2
    Adv[2::7] = 0.0
    scale, v_coef, beta = 1.0 / (T * R), 0.5, 0.01
    dH = torch.empty(U, M, 64, device="cuda")
    G = torch.zeros_like(m.G)
    stats = torch.zeros(4, device="cuda")
    _lib.check(_lib.lib().tscl_heads_loss(m._h, _p(m.P), None, _p(act[0, r0:]), _p(Rs[0, r0:]), _p(Adv[0, r0:]),
                                          C.c_int64(M), C.c_int64(rc), C.c_int64(R * A), C.c_float(v_coef), C.c_float(beta),
                                          C.c_float(scale), None, _p(dH), _p(stats), _p(Hb), _p(G), m._st()))
    torch.cuda.synchronize()
    vd = lay.views(m.P.double())
    gv = lay.views(G)
    rel = lambda got, ref: ((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()
    worst = {"dH": 0.0, "wo": 0.0, "bo": 0.0}
    for a in range(A):
        sl = lambda x: x[:, r0:r0 + rc, a].reshape(-1)
        hr = heads_ref(lay, vd, a, Hb[2 * a].double().reshape(M, 64), Hb[2 * a + 1].double().reshape(M, 64), sl(act),
                       sl(Rs).double(), sl(Adv).double(), scale, v_coef, beta)
        n = int(lay.n_a[a])
        worst["dH"] = max(worst["dH"], rel(dH[2 * a], hr["dH_pi"]), rel(dH[2 * a + 1], hr["dH_v"]))
        worst["wo"] = max(worst["wo"], rel(gv["wo"][2 * a][:, :n], hr["wo_pi"]), rel(gv["wo"][2 * a + 1][:, 0], hr["wo_v"]))
        worst["bo"] = max(worst["bo"], rel(gv["bo"][2 * a][:n], hr["bo_pi"]),
                          rel(gv["bo"][2 * a + 1][:1], hr["bo_v"].reshape(1)))
        if a == 0:
            np.testing.assert_allclose(stats[:3].cpu().numpy(), hr["stats"].cpu().numpy(), rtol=1e-4)
    print("OBSERVED heads_loss: max |d| / max |ref|  dH %.3e  wo %.3e  bo %.3e" % (worst["dH"], worst["wo"], worst["bo"]))
    # observed: dH 5.4e-7, wo 9.5e-7, bo 3.4e-5 (the bias sums cancel); the unclipped formula gave dH 0.91
    assert worst["dH"] <= 2e-6 and worst["wo"] <= 3e-6 and worst["bo"] <= 1e-4, worst
    for k, t in gv.items():
        if k == "wo":
            for u in range(U):
                assert not bool(t[u][:, int(lay.n_a[u // 2]) if u % 2 == 0 else 1:].any())
        elif k == "bo":
            for u in range(U):
                assert not bool(t[u][int(lay.n_a[u // 2]) if u % 2 == 0 else 1:].any())
        else:
            assert not bool(t.any()), k


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["grid", "monaco", "grid_ia2c"])
def test_whole_update_matches_chunked_reference(kind):
    """BatchedA2C(use_tc=True, store_acts=True).backward at R = 2048 (two 1024-replica chunks, accumulated through the
    kernels' atomics) vs update_ref on the same store, states and rollout: nonzero per-replica initial states, dones at
    interior steps, random rewards.  Rs / Adv vs nstep_returns; G per named tensor (rel-L2) and overall; and with
    dx_fused = True the same G up to the order of the atomic additions."""
    from oracle.learner_ref import nstep_returns, update_ref
    T = 40 if kind == "monaco" else 120
    R, chunk = 2048, 1024
    gamma, beta = 0.99, 0.01
    lay, m = _model(kind, R=R, n_step=T, seed=7, chunk=chunk, gamma=gamma, v_coef=0.5, max_grad_norm=40.0,
                    reward_norm=2000.0, reward_clip=2.0, use_tc=True, store_acts=True)
    assert m.store_acts and m.tc_v2
    g = torch.Generator(device="cuda").manual_seed(41)
    m.c_fw.copy_(torch.randn(m.c_fw.shape, device="cuda", generator=g) * 0.5)
    m.h_fw.copy_(torch.tanh(torch.randn(m.h_fw.shape, device="cuda", generator=g)) * 0.5)
    m.c_bw.copy_(m.c_fw); m.h_bw.copy_(m.h_fw)
    done_steps = {T // 3, (2 * T) // 3 + 1}
    dpre = [1.0 if t in done_steps else 0.0 for t in range(T)]
    dpost = dpre[1:] + [0.0]
    for t in range(T):
        m.obs_slot().copy_(torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2)
        m.forward(m.obs_slot(), bool(dpre[t]))
        m.add_transition(torch.randn(R, lay.A, device="cuda", generator=g) * 3000, bool(dpre[t]), bool(dpost[t]))
    boot = torch.randn(R, lay.A, device="cuda", generator=g)
    # backward() refreshes c_bw / h_bw from the forward state and moves obs slot T to slot 0: keep copies
    c_bw, h_bw, obs = m.c_bw.clone(), m.h_bw.clone(), m.obs_hist[:T].clone()
    m.backward(boot, lr=0.0, beta=beta)
    torch.cuda.synchronize()
    G0 = m.G.clone()
    Rs_ref, Adv_ref = nstep_returns(list(m.rew_hist.double().cpu().numpy()), list(m.val_hist.double().cpu().numpy()),
                                    dpost, boot.double().cpu().numpy(), gamma)
    np.testing.assert_allclose(m.Rs.cpu().numpy(), Rs_ref, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(m.Adv.cpu().numpy(), Adv_ref, rtol=1e-5, atol=1e-5)
    store = lambda ci: (m.st_x[ci], m.st_g[ci], m.st_c[ci], m.st_h[ci])
    Gref, _ = update_ref(lay, m.P, store, obs, m.act_hist, m.Rs, m.Adv, c_bw, h_bw, dpre, 1.0 / (T * R), 0.5, beta, chunk,
                         agents_per_group=5)
    gv, rv = lay.views(G0.double()), lay.views(Gref)
    groups = {k: [k] for k in ("wx", "wh", "bl", "wo", "bo")}
    for name in ("fcw_w", "fcw_b", "fcf_w", "fcf_b", "fct_w", "fct_b"):
        groups[name] = [name + str(u) for u in range(lay.U)]
    worst = {}
    for name, keys in groups.items():
        got = torch.cat([gv[k].reshape(-1) for k in keys])
        ref = torch.cat([rv[k].reshape(-1) for k in keys])
        if ref.numel() == 0:
            continue
        worst[name] = ((got - ref).norm() / ref.norm()).item()
    overall = ((G0.double() - Gref).norm() / Gref.norm()).item()
    print("OBSERVED whole update %s: overall rel-L2 %.3e; per tensor %s" % (
        kind, overall, ", ".join("%s %.2e" % kv for kv in worst.items())))
    # observed: overall 1.1e-4 / 4.5e-5 / 9.8e-5 (grid / Monaco / IA2C), worst tensor 1.4e-4 (wx)
    assert max(worst.values()) <= 5e-4 and overall <= 4e-4, (overall, worst)
    del Gref, gv, rv
    # the same update with dX fused into the BPTT kernel
    m.c_bw.copy_(c_bw); m.h_bw.copy_(h_bw); m.obs_hist[0].copy_(obs[0])
    m.t, m._acts_ok, m.dx_fused = T, [True] * T, True
    m.backward(boot, lr=0.0, beta=beta)
    torch.cuda.synchronize()
    fused = ((m.G.double() - G0.double()).norm() / G0.double().norm()).item()
    print("OBSERVED whole update %s: dx_fused vs default rel-L2 %.3e" % (kind, fused))
    assert fused <= 5e-7, fused         # observed 6.7e-8 / 7.5e-8 / 1.0e-7
    m.close()


# ------------------------------------------------------------------------------------------------------------------
def test_clip_rmsprop_grid_layout():
    """tscl_clip_rmsprop on the grid layout (25 agents, 3.93 M floats, the interleaved agent_of map) for two steps, with
    about half of the agents above max_norm, vs oracle.clip_rmsprop."""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    from oracle.learner_ref import clip_rmsprop
    lay, m = _model("grid")
    rng = np.random.default_rng(8)
    Gn = rng.normal(0, 0.2, lay.n_params).astype(np.float32)
    small = rng.permutation(lay.A)[:lay.A // 2]
    for a in small:
        Gn[lay.agent_of == a] *= 1e-2
    P0, MS0 = m.P.cpu().numpy().copy(), m.MS.cpu().numpy().copy()
    m.G.copy_(torch.from_numpy(Gn))
    for _ in range(2):
        _lib.check(_lib.lib().tscl_clip_rmsprop(m._h, _p(m.P), _p(m.G), _p(m.MS), _p(m.agent_of), C.c_float(40.0),
                                                C.c_float(5e-4), C.c_float(0.99), C.c_float(1e-5), _p(m.norms), m._st()))
        P0, MS0, norms = clip_rmsprop(P0, Gn, MS0, lay.agent_of, 40.0, 5e-4, 0.99, 1e-5, lay.A)
    torch.cuda.synchronize()
    above = int((norms > 40.0).sum())
    assert 8 <= above <= 17, norms
    np.testing.assert_allclose(m.norms.cpu().numpy(), norms, rtol=1e-5)
    np.testing.assert_allclose(m.MS.cpu().numpy(), MS0, rtol=1e-6)
    np.testing.assert_allclose(m.P.cpu().numpy(), P0, rtol=1e-6, atol=1e-7)


def test_unpack_store_bench_chunk():
    """tscl_unpack_store (store -> fp32 chunk buffers) for the chunk at r0 = 1024 of R = 2048: X, gates, C, H are exact
    upcasts; Hp[t] = (1 - done[t]) * (H[t-1], or h0[r0 + r] at t = 0), bit for bit.  Done at t = 0 and t = 37."""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    T, R, rc, r0 = 120, 2048, 1024, 1024
    lay, m = _model("grid")
    U, dx, M = lay.U, lay.dx, T * rc
    g = torch.Generator(device="cuda").manual_seed(12)
    bf = lambda *s: torch.randn(*s, device="cuda", generator=g).to(torch.bfloat16)
    sx, sg, sc, sh = bf(U, T, rc, dx), bf(U, T, rc, 256), bf(U, T, rc, 64), bf(U, T, rc, 64)
    h0 = torch.randn(U, R, 64, device="cuda", generator=g)
    done = torch.zeros(T, device="cuda")
    done[[0, 37]] = 1.0
    outs = [torch.full((U, M, w), float("nan"), device="cuda") for w in (dx, 256, 64, 64, 64)]
    _lib.check(_lib.lib().tscl_unpack_store(m._h, _p(sx), _p(sg), _p(sc), _p(sh), *(_p(o) for o in outs), _p(h0), _p(done),
                                            C.c_int32(T), C.c_int64(rc), C.c_int64(R), C.c_int64(r0), m._st()))
    torch.cuda.synchronize()
    X, ZG, Cc, H, Hp = outs
    for got, src in ((X, sx), (ZG, sg), (Cc, sc), (H, sh)):
        assert torch.equal(got, src.float().reshape(got.shape))
    del X, ZG, Cc, sx, sg, sc
    prev = torch.cat([h0[:, r0:r0 + rc].unsqueeze(1), sh[:, :-1].float()], 1)
    ref = torch.where((done == 0)[None, :, None, None], prev, torch.zeros_like(prev)).reshape(U, M, 64)
    assert torch.equal(Hp, ref)
