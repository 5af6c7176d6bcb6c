"""GPU: imitation of a signal controller in the A2C update (BatchedA2C(teacher=...), DESIGN §5 Imitation).

- tscl_heads_loss_imit against the float64 reference on a bench chunk with random teachers and wide heads (pi_1 < 1e-10
  on agent 0, so some teacher actions are clipped): dH, head gradients, stats[0..3].
- tscl_lstm_seq_bwd_tc_heads_imit against the pair it replaces (tscl_heads_loss_imit, then the store-path BPTT): dZ bit
  for bit, head gradients and loss sums up to summation order, atomic and deterministic (two deterministic launches
  bit-identical); at lam = 0 both _imit kernels equal the plain ones.
- One whole update at the bench chunk shape with a teacher, and the FC learner's, against the float64 references.
- Labels: teach_hist[t] equals numpy max-pressure on the lane counts and numpy greedy() on obs_hist[t], on the grid
  and Monaco, for the ia2c and ma2c observation layouts.
- End to end: train() with a teacher (directory, evaluate.py, the imitation tag, deterministic bytes, a deterministic
  sweep member against its solo run), and the term doing its job (argmax agreement with max-pressure rises).
"""
import configparser
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.imitation_ref import fc_update_imit_ref, heads_imit_ref, update_imit_ref
from tests.test_bptt_heads_gpu import _inputs
from tests.test_update_bench_size_gpu import _model

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _free_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _teach(lay, T, R, g, act):
    """Random teacher actions: agent 0's clipped action 1 on every 4th step, b == a on every 5th."""
    na = torch.as_tensor(lay.n_a, device="cuda")
    teach = (torch.rand(T, R, lay.A, device="cuda", generator=g) * na).long().clamp_max(na - 1).to(torch.int32)
    teach[::4, :, 0] = 1
    teach[2::5] = act[2::5]
    return teach


def _rel(got, ref):
    return ((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()


def test_heads_loss_imit_matches_float64():
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    T, R, rc, r0, lam = 120, 2048, 1024, 1024, 0.7
    M = T * rc
    lay, m = _model("grid")
    U, A = lay.U, lay.A
    x = _inputs(m, T, rc, 2, (37,), seed=31)                   # wide heads, pi_1 < 1e-10 on agent 0
    Hb = x["hb"][1]
    teach = _teach(lay, T, R, torch.Generator(device="cuda").manual_seed(5), x["act"])
    scale, v_coef, beta = 1.0 / (T * R), 0.5, 0.01
    dH = torch.empty(U, M, 64, device="cuda")
    G, stats = torch.zeros_like(m.G), torch.zeros(4, device="cuda")
    _lib.check(_lib.lib().tscl_heads_loss_imit(
        m._h, _p(m.P), None, _p(x["act"][0, r0:]), _p(x["Rs"][0, r0:]), _p(x["Adv"][0, r0:]), M, rc, R * A, v_coef, beta,
        scale, None, _p(dH), _p(stats), _p(Hb), _p(G), _p(teach[0, r0:]), lam, m._st()))
    torch.cuda.synchronize()
    vd, gv = lay.views(m.P.double()), lay.views(G)
    worst = {"dH": 0.0, "wo": 0.0, "bo": 0.0}
    for a in range(A):
        sl = lambda t_: t_[:, r0:r0 + rc, a].reshape(-1)
        hr = heads_imit_ref(lay, vd, a, Hb[2 * a].double().reshape(M, 64), Hb[2 * a + 1].double().reshape(M, 64),
                            sl(x["act"]), sl(teach), sl(x["Rs"]).double(), sl(x["Adv"]).double(), scale, v_coef, beta, lam)
        n = int(lay.n_a[a])
        worst["dH"] = max(worst["dH"], _rel(dH[2 * a], hr["dH_pi"]), _rel(dH[2 * a + 1], hr["dH_v"]))
        worst["wo"] = max(worst["wo"], _rel(gv["wo"][2 * a][:, :n], hr["wo_pi"]), _rel(gv["wo"][2 * a + 1][:, 0], hr["wo_v"]))
        worst["bo"] = max(worst["bo"], _rel(gv["bo"][2 * a][:n], hr["bo_pi"]))
        if a == 0:
            print("OBSERVED stats", stats.tolist(), hr["stats"].tolist())
            np.testing.assert_allclose(stats.cpu().numpy(), hr["stats"].cpu().numpy(), rtol=1e-4)
    print("OBSERVED heads_loss_imit: max |d| / max |ref| dH %.3e wo %.3e bo %.3e" % (worst["dH"], worst["wo"], worst["bo"]))
    # the plain kernel's bounds (tests/test_update_bench_size_gpu.py::test_heads_loss_bench_chunk)
    assert worst["dH"] <= 2e-6 and worst["wo"] <= 3e-6 and worst["bo"] <= 1e-4, worst


def _pair(m, x, T, Rc, nc, teach, lam, v_coef, beta, scale):
    """tscl_heads_loss_imit on the bf16 store, then the store-path BPTT, chunk by chunk: (dZ [nc, U, M, 256], G, stats)."""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    lib, U, A, R, M = _lib.lib(), m.lay.U, m.lay.A, nc * Rc, T * Rc
    G, st = torch.zeros_like(m.G), torch.zeros(4, device="cuda")
    dZ = torch.empty(nc, U, M, 256, dtype=torch.bfloat16, device="cuda")
    dH = torch.empty(U, M, 64, device="cuda")
    for ci in range(nc):
        r0 = ci * Rc
        _lib.check(lib.tscl_heads_loss_imit(m._h, _p(m.P), None, _p(x["act"][0, r0:]), _p(x["Rs"][0, r0:]),
                                            _p(x["Adv"][0, r0:]), M, Rc, R * A, v_coef, beta, scale, None, _p(dH), _p(st),
                                            _p(x["hb"][ci]), _p(G), _p(teach[0, r0:]), lam, m._st()))
        _lib.check(lib.tscl_lstm_seq_bwd_tc(m._h, _p(m.Wt), None, None, _p(dH), _p(x["c_bw"]), _p(x["done"]), T, Rc, R,
                                            r0, _p(x["gates"][ci]), _p(x["cb"][ci]), _p(dZ[ci]), m._st()))
    torch.cuda.synchronize()
    return dZ, G, st


def _fused(m, x, T, Rc, nc, teach, lam, v_coef, beta, scale, imit=True):
    """One tscl_lstm_seq_bwd_tc_heads[_imit] launch over every chunk: (dZ, G, stats)."""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    U, A, R, M = m.lay.U, m.lay.A, nc * Rc, T * Rc
    G, st = torch.zeros_like(m.G), torch.zeros(4, device="cuda")
    dZ = torch.empty(nc, U, M, 256, dtype=torch.bfloat16, device="cuda")
    args = (m._h, _p(m.Wt), _p(m.P), _p(x["gates"][0]), _p(x["cb"][0]), _p(x["hb"][0]), _p(x["c_bw"]), _p(x["done"]),
            _p(x["act"][0]), _p(x["Rs"][0]), _p(x["Adv"][0]), T, Rc, nc, R, 0, R * A, v_coef, beta, scale, _p(dZ), _p(st),
            _p(G))
    if imit:
        _lib.check(_lib.lib().tscl_lstm_seq_bwd_tc_heads_imit(*args, _p(teach[0]), lam, m._st()))
    else:
        _lib.check(_lib.lib().tscl_lstm_seq_bwd_tc_heads(*args, m._st()))
    torch.cuda.synchronize()
    return dZ, G, st


def _bits(a):
    return a.view(torch.int16)


def _head_rel(lay, G, Gref):
    g, r = lay.views(G.double()), lay.views(Gref.double())
    return max(((g[k] - r[k]).abs().max() / r[k].abs().max()).item() for k in ("wo", "bo"))


@pytest.mark.parametrize("kind,T,Rc,nc,done_steps", [
    ("grid", 120, 1024, 4, (37, 90)),          # the bench: R = 4096 in chunks of 1024
    ("monaco", 40, 1024, 2, (0, 39)),
    ("grid", 120, 40, 3, (0, 119)),            # one partial 128-row tile per chunk
])
def test_fused_imit_matches_the_pair(kind, T, Rc, nc, done_steps):
    from deeprl_signal_control_b200 import _lib
    lay, m = _model(kind)
    x = _inputs(m, T, Rc, nc, done_steps, seed=41)
    teach = _teach(lay, T, nc * Rc, torch.Generator(device="cuda").manual_seed(7), x["act"])
    scale, v_coef, beta, lam = 1.0 / (T * nc * Rc), 0.5, 0.01, 0.9
    dZ2, G2, st2 = _pair(m, x, T, Rc, nc, teach, lam, v_coef, beta, scale)
    dZ1, G1, st1 = _fused(m, x, T, Rc, nc, teach, lam, v_coef, beta, scale)
    assert torch.equal(_bits(dZ1), _bits(dZ2))
    del dZ1
    rel = _head_rel(lay, G1, G2)
    print("OBSERVED %s atomic: head gradients %.2e; stats %s vs %s" % (kind, rel, st1.tolist(), st2.tolist()))
    assert rel <= 5e-6, rel                  # the plain fused kernel's bound (tests/test_bptt_heads_gpu.py)
    torch.testing.assert_close(st1, st2, rtol=1e-4, atol=0)
    assert float(st2[3]) > 0
    # lam = 0: the _imit kernels give the plain kernels' results
    dZ0, G0, st0 = _fused(m, x, T, Rc, nc, teach, 0.0, v_coef, beta, scale)
    dZp, Gp, stp = _fused(m, x, T, Rc, nc, teach, 0.0, v_coef, beta, scale, imit=False)
    assert torch.equal(_bits(dZ0), _bits(dZp))
    del dZ0, dZp
    assert _head_rel(lay, G0, Gp) <= 5e-6
    torch.testing.assert_close(st0[:3], stp[:3], rtol=1e-5, atol=0)
    assert float(stp[3]) == 0.0 and float(st0[3]) > 0            # the cross-entropy is recorded at lam = 0 too
    dH = torch.empty(lay.U, T * Rc, 64, device="cuda")
    from deeprl_signal_control_b200.agents.learner import _p
    outs = []
    for fn in ("tscl_heads_loss_imit", "tscl_heads_loss"):
        G, st = torch.zeros_like(m.G), torch.zeros(4, device="cuda")
        args = (m._h, _p(m.P), None, _p(x["act"][0]), _p(x["Rs"][0]), _p(x["Adv"][0]), T * Rc, Rc, nc * Rc * lay.A,
                v_coef, beta, scale, None, _p(dH), _p(st), _p(x["hb"][0]), _p(G))
        args = args + ((_p(teach[0]), 0.0) if fn.endswith("imit") else ()) + (m._st(),)
        _lib.check(getattr(_lib.lib(), fn)(*args))
        torch.cuda.synchronize()
        outs.append((dH.clone(), G, st))
    assert torch.equal(outs[0][0], outs[1][0])
    assert _head_rel(lay, outs[0][1], outs[1][1]) <= 5e-6
    del outs, dH
    # deterministic mode: the same dZ bits, and two launches give the same bits everywhere
    _lib.check(_lib.lib().tscl_set_deterministic(m._h, 1, 0))
    dZa, Ga, sta = _fused(m, x, T, Rc, nc, teach, lam, v_coef, beta, scale)
    assert torch.equal(_bits(dZa), _bits(dZ2))
    del dZa
    dZb, Gb, stb = _fused(m, x, T, Rc, nc, teach, lam, v_coef, beta, scale)
    assert torch.equal(_bits(dZb), _bits(dZ2))
    del dZb, dZ2
    assert torch.equal(Ga, Gb) and torch.equal(sta, stb)
    assert _head_rel(lay, Ga, G2) <= 5e-6
    torch.testing.assert_close(sta, st2, rtol=1e-4, atol=0)
    with pytest.raises(RuntimeError, match="tscl_heads_loss_imit"):
        _pair(m, x, T, Rc, 1, teach, lam, v_coef, beta, scale)
    m.close()


@pytest.mark.parametrize("kind", ["grid", "monaco"])
def test_whole_update_with_teacher_matches_float64(kind):
    """BatchedA2C(teacher=...).backward at R = 2048 in two chunks of 1024 (the bench's chunk shape) vs the float64
    backward through its own activation store (update_imit_ref); stats[0..3]."""
    T = 40 if kind == "monaco" else 120
    R, chunk, gamma, beta, lam = 2048, 1024, 0.99, 0.01, 0.8
    lay, m = _model(kind, R=R, n_step=T, seed=7, chunk=chunk, gamma=gamma, v_coef=0.5, max_grad_norm=40.0,
                    reward_norm=2000.0, reward_clip=2.0, teacher="maxpressure")
    assert m.store_acts and m.tc_v2
    g = torch.Generator(device="cuda").manual_seed(41)
    m.c_fw.copy_(torch.randn(m.c_fw.shape, device="cuda", generator=g) * 0.5)
    m.h_fw.copy_(torch.tanh(torch.randn(m.h_fw.shape, device="cuda", generator=g)) * 0.5)
    m.c_bw.copy_(m.c_fw); m.h_bw.copy_(m.h_fw)
    done_steps = {T // 3}
    dpre = [1.0 if t in done_steps else 0.0 for t in range(T)]
    dpost = dpre[1:] + [0.0]
    for t in range(T):
        m.obs_slot().copy_(torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2)
        m.forward(m.obs_slot(), bool(dpre[t]))
        m.add_transition(torch.randn(R, lay.A, device="cuda", generator=g) * 3000, bool(dpre[t]), bool(dpost[t]))
    m.teach_hist.copy_(_teach(lay, T, R, g, m.act_hist))
    boot = torch.randn(R, lay.A, device="cuda", generator=g)
    c_bw, h_bw, obs = m.c_bw.clone(), m.h_bw.clone(), m.obs_hist[:T].clone()
    m.backward(boot, lr=0.0, beta=beta, imit=lam)
    torch.cuda.synchronize()
    store = lambda ci: (m.st_x[ci], m.st_g[ci], m.st_c[ci], m.st_h[ci])
    Gref, st_ref = update_imit_ref(lay, m.P, store, obs, m.act_hist, m.teach_hist, m.Rs, m.Adv, c_bw, h_bw, dpre,
                                   1.0 / (T * R), 0.5, beta, lam, chunk, agents_per_group=5)
    overall = ((m.G.double() - Gref).norm() / Gref.norm()).item()
    print("OBSERVED whole update with teacher %s: overall rel-L2 %.3e; stats %s vs %s" % (
        kind, overall, m.stats.tolist(), st_ref.tolist()))
    assert overall <= 1e-3, overall
    np.testing.assert_allclose(m.stats.cpu().numpy(), st_ref.cpu().numpy(), rtol=2e-4)
    with pytest.raises(ValueError, match="finite"):
        m.t = T
        m.backward(boot, lr=0.0, beta=beta, imit=float("nan"))
    m.close()


def test_fc_update_with_teacher_matches_float64():
    from tests.test_update_recompute_bench_size_gpu import RC, R_BENCH, T_GRID, _model as _rmodel, _rel_l2, _rollout
    T, R, gamma, beta, lam = T_GRID, R_BENCH, 0.99, 0.01, 0.6
    lay, m = _rmodel("fc", R=R, T=T, seed=7, chunk=RC, gamma=gamma, v_coef=0.5, max_grad_norm=40.0, reward_norm=3000.0,
                     reward_clip=2.0, teacher="greedy")
    g = torch.Generator(device="cuda").manual_seed(45)
    dpre, dpost, boot = _rollout(lay, m, T, R, g, {T // 3})
    m.teach_hist.copy_(_teach(lay, T, R, g, m.act_hist))
    obs = m.obs_hist[:T].clone()
    m.backward(boot, lr=0.0, beta=beta, imit=lam)
    torch.cuda.synchronize()
    Gref, st_ref = fc_update_imit_ref(lay, m.P, obs, m.act_hist, m.teach_hist, m.Rs, m.Adv, 1.0 / (T * R), 0.5, beta,
                                      lam, RC, round_bf16=True)
    overall = _rel_l2(m.G, Gref)
    print("OBSERVED FC update with teacher: overall rel-L2 %.3e; stats %s vs %s" % (overall, m.stats.tolist(),
                                                                                    st_ref.tolist()))
    assert overall <= 1e-3, overall
    np.testing.assert_allclose(m.stats.cpu().numpy(), st_ref.cpu().numpy(), rtol=2e-4)
    m.close()


# ---- labels ---------------------------------------------------------------------------------------------------------
def _mc(teacher, **kw):
    from tests.test_evaluator_gpu import MODEL_INI
    c = configparser.ConfigParser()
    c.read_string(MODEL_INI)
    mc = c["MODEL_CONFIG"]
    mc["teacher"], mc["imitation_coef_init"] = teacher, "1.0"
    for k, v in kw.items():
        mc[k] = str(v)
    return mc


@pytest.mark.parametrize("scenario,agent", [("large_grid", "ia2c"), ("large_grid", "ma2c"), ("real_net", "ia2c"),
                                            ("real_net", "ma2c")])
def test_labels_equal_the_numpy_controllers(scenario, agent, tmp_path):
    from deeprl_signal_control_b200.agents.train import build_model, teacher_kwargs
    from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
    from deeprl_signal_control_b200.envs import greedy_controller
    from deeprl_signal_control_b200.envs.maxpressure import pressure_actions
    from tests.test_evaluator_gpu import _env
    R = 256
    check = [0, 1, 77, 128, 200, 255]
    for teacher in ("maxpressure", "greedy"):
        env = _env(scenario, agent, [10000], 3600, str(tmp_path), R, record=False)
        model = build_model(agent, env, _mc(teacher), 3600, R, seed=3)
        sim, b = env._ensure_sim(), model.batched
        tr = BatchedTrainer(sim, b, agent, 0.0, 0.0, seed0=5, **teacher_kwargs(model, env))
        ctrl, off = greedy_controller(env), np.asarray(env._tables.node_obs_off)
        varied = 0
        for step in range(b.T - 1):                              # within one rollout: no update in between
            t = b.t
            cnt = np.stack([sim.dump_state(r)[0] for r in check]) if teacher == "maxpressure" else None
            tr.control_step()
            got = b.teach_hist[t].cpu().numpy()[check]
            if teacher == "maxpressure":
                want = pressure_actions(sim.net, cnt)
            else:
                obs = b.obs_hist[t].cpu().numpy()[check]
                want = np.array([[ctrl.greedy(o[off[i]:off[i + 1]], name) for i, name in enumerate(env.node_names)]
                                 for o in obs])
            np.testing.assert_array_equal(got, want, err_msg="%s step %d" % (teacher, t))
            varied += len(np.unique(got)) > 1
        assert varied >= (b.T - 1) // 2, varied                  # the states were not all alike
        b.close()


# ---- end to end -----------------------------------------------------------------------------------------------------
def _write(path, agent="ma2c", total=240, **mc):
    from tests.test_train_driver_gpu import _ini
    c = configparser.ConfigParser()
    c.read_string(_ini(agent, total, 10 ** 9))
    for k, v in mc.items():
        c["MODEL_CONFIG"][k] = str(v)
    with open(path, "w") as f:
        c.write(f)
    return str(path)


def _tree(d):
    out = {}
    for root, _, files in os.walk(d):
        for f in files:
            p = os.path.join(root, f)
            out[os.path.relpath(p, d)] = open(p, "rb").read()
    return out


def test_train_with_a_teacher_end_to_end(tmp_path):
    from deeprl_signal_control_b200.agents.summary import event_files, read_scalars
    from deeprl_signal_control_b200.agents.train import train, train_sweep
    R = 64
    lam = dict(teacher="maxpressure", imitation_coef_init=1.0, imitation_decay="linear", imitation_ratio=0.5)
    cfg = _write(tmp_path / "config_ma2c_large.ini", **lam)
    plain = _write(tmp_path / "plain.ini")
    ref = train(plain, str(tmp_path / "plain" / "ma2c"), "after_train_test", n_replicas=R)
    out = train(cfg, str(tmp_path / "run" / "ma2c"), "after_train_test", n_replicas=R, summaries=True)
    d = str(tmp_path / "run" / "ma2c")
    layout = lambda x: sorted(k.replace("config_ma2c_large", "plain") for k in _tree(x) if not k.startswith("log"))
    assert layout(d) == layout(str(tmp_path / "plain" / "ma2c"))
    assert out.trainer.summary_rec.shape[-1] == 5
    ev = read_scalars(event_files(os.path.join(d, "log"))[0])
    tag = ev["loss/fplstm_0a_imitation_loss"]
    assert [s for _, s, _ in tag] == [120, 240]
    assert tag[-1][2] == pytest.approx(float(out.model.batched.stats[3]), rel=1e-6)
    assert tag[0][2] > 0
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", d],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    # two deterministic runs write the same checkpoint values and CSV bytes
    from tests.test_deterministic_gpu import _same_dir
    dets = [str(tmp_path / ("det%d" % k) / "ma2c") for k in range(2)]
    for base in dets:
        train(cfg, base, "after_train_test", n_replicas=R, deterministic=True)
    _same_dir(dets[0], dets[1], 240)
    # a deterministic sweep member with its own lam equals its solo run
    (tmp_path / "cfg").mkdir()
    a = _write(tmp_path / "cfg" / "a.ini", **lam)
    b = _write(tmp_path / "cfg" / "b.ini", teacher="maxpressure", imitation_coef_init=0.3)
    train_sweep([a, b], str(tmp_path / "sweep"), "no_test", n_replicas=R, deterministic=True)
    solo = str(tmp_path / "solo_b" / "ma2c")
    train(b, solo, "no_test", n_replicas=R, deterministic=True)
    _same_dir(str(tmp_path / "sweep" / "b" / "ma2c"), solo, 240)
    del ref


def test_imitation_raises_agreement_with_the_teacher(tmp_path):
    """A few deterministic updates with a large lam and beta = 0: the student's argmax agreement with max-pressure on a
    fresh rollout rises well above its agreement at initialisation."""
    from deeprl_signal_control_b200.agents.train import build_model, teacher_kwargs
    from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
    from tests.test_evaluator_gpu import _env
    R = 512

    def agreement(model, sim, seed):
        b = model.batched
        sim.reset(np.arange(R, dtype=np.uint64) + np.uint64(seed))
        sim.set_train_mode(True)
        b.reset()
        obs = torch.zeros(R, b.lay.n_obs, device="cuda")
        teach = torch.zeros(R, b.lay.A, dtype=torch.int32, device="cuda")
        sim.observe(None, obs_out=obs)
        hits, n = 0, 0
        for t in range(60):
            pi, _, _ = b.forward(obs, t == 0, out_type="p", sample=False)
            sim.pressure_actions(teach)
            na = torch.as_tensor(b.lay.n_a, device="cuda")
            masked = torch.where(torch.arange(pi.shape[2], device="cuda")[None, None] < na[None, :, None], pi, -1.0)
            greedy_act = masked.argmax(-1).to(torch.int32)
            hits += int((greedy_act == teach).sum()); n += teach.numel()
            sim.step(greedy_act.contiguous(), None, obs_out=obs)
        return hits / n

    env = _env("large_grid", "ia2c", [10000], 3600, str(tmp_path), R, record=False)
    model = build_model("ia2c", env, _mc("maxpressure", entropy_coef_init=0.0, lr_init=1e-3), 3600, R, seed=3,
                        deterministic=True)
    sim = env._ensure_sim()
    before = agreement(model, sim, 900)
    tr = BatchedTrainer(sim, model.batched, "ia2c", 1e-3, 0.0, seed0=5, imit=5.0)
    tr.run(8 * model.batched.T)
    after = agreement(model, sim, 900)
    print("OBSERVED argmax agreement with max-pressure: %.3f at initialisation, %.3f after %d updates"
          % (before, after, tr.n_updates))
    # observed on an H100 80GB HBM3 (700 W): 0.428 at initialisation, 0.531 after 8 updates
    assert after >= before + 0.05, (before, after)
