"""GPU: deterministic A2C training (`BatchedA2C(deterministic=True)`, tscl_set_deterministic).

* Kernels: at the four reference widths (grid MA2C dx 224, Monaco MA2C 192, grid IA2C 160, Monaco IA2C 128; chunk 1024,
  T = 120, Monaco T = 40) the lean update's gradient, loss sums and clip norms are bit-identical between two runs and
  between the device-sized grid and a 61-CTA cap, and agree with the atomic kernels to summation-order rounding.
* Update: two deterministic learners fed the same rollouts hold equal P, MS, norms and stats after every update.
* Driver: two `train(..., deterministic=True)` runs leave the same checkpoint, CSV bytes and event scalars; a population
  and a sweep member equal its solo deterministic run exactly; two gloo ranks end with the same state digest twice.
"""
import datetime
import gc
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

from tests.layout_envelope import net_tables, scenario_layout
from tests.test_train_driver_gpu import _ini

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _free_device_memory():
    """Each test's learners (their handles own the deterministic slabs) and torch's cached blocks go back to the device
    before the next test, so that later tests in the same process find the memory they size themselves by."""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

CHUNK = 1024
SHAPES = [("large_grid", "ma2c", 120), ("real_net", "ma2c", 40), ("large_grid", "ia2c", 120), ("real_net", "ia2c", 40)]


def _filled(lay, R, T, seed=1, dseed=5):
    """A deterministic learner after one rollout of T storing forward steps on seeded random observations / rewards."""
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    m = BatchedA2C(lay, R, T, chunk=CHUNK, seed=seed, reward_norm=2000.0, reward_clip=2.0, deterministic=True)
    g = torch.Generator(device=m.dev).manual_seed(dseed)
    for t in range(T):
        m.obs_slot().copy_(torch.rand(m.obs_slot().shape, generator=g, device=m.dev))
        m.forward(m.obs_slot(), t == 0)
        m.add_transition(torch.randn(R, lay.A, generator=g, device=m.dev) * 1000.0, False, t == T - 1)
    m.obs_slot().copy_(torch.rand(m.obs_slot().shape, generator=g, device=m.dev))
    return m


def _grads(m, on, n_ctas=0):
    """The lean update's kernels from the learner's rollout (backward without the weight step): (G, stats, norms)."""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200 import dist as _dist
    lib, p, L, T, R = _lib.lib(), _lib.ptr, m.lay, m.T, m.R
    _lib.check(lib.tscl_set_deterministic(m._h, on, n_ctas))
    f32 = dict(dtype=torch.float32, device=m.dev)
    dpre, dpost = torch.tensor(m.done_pre, **f32), torch.tensor(m.done_post, **f32)
    st = _lib.stream(m.dev)
    _lib.check(lib.tscl_returns(m._h, p(m.rew_hist), p(m.val_hist), p(torch.zeros_like(m.boot)), p(dpost), m.gamma, T, R,
                                p(m.Rs), p(m.Adv), st))
    G, stats, norms = torch.zeros_like(m.G), torch.zeros(4, **f32), torch.zeros(L.A, **f32)
    scale = _dist.grad_scale(T, 1, R)
    dz = torch.empty(R // CHUNK, L.U, T * CHUNK, 4 * L.h, dtype=torch.bfloat16, device=m.dev)
    m._bwd_heads(m.P, G, m.Wt, stats, 0, R // CHUNK, m.v_coef, 0.01, scale, dpre, dz)
    for ci, r0 in enumerate(range(0, R, CHUNK)):
        _lib.check(lib.tscl_wgrad_tc(m._h, None, p(dz[ci]), None, p(m.st_x[ci]), None, p(m.st_h[ci]), p(m.h_bw), p(dpre),
                                     T, CHUNK, R, r0, p(G), 0, st))
        _lib.check(lib.tscl_dx_fc_bwd_tc(m._h, p(m.obs_hist[0, r0:]), p(m.st_x[ci]), p(dz[ci]), p(m.Wxt), T * CHUNK, CHUNK,
                                         R * L.n_obs, p(G), st))
    P2, MS2 = m.P.clone(), m.MS.clone()
    _lib.check(lib.tscl_clip_rmsprop(m._h, p(P2), p(G), p(MS2), p(m.agent_of), m.max_grad_norm, 5e-4, m.alpha, m.eps,
                                     p(norms), st))
    _lib.check(lib.tscl_set_deterministic(m._h, 1, 0))
    torch.cuda.synchronize(m.dev)
    return G, stats, norms


@pytest.mark.parametrize("scenario,agent,T", SHAPES)
def test_kernels_repeat_their_bits_on_any_grid(scenario, agent, T):
    from deeprl_signal_control_b200.agents.learner import learner_paths
    lay = scenario_layout(net_tables(scenario, agent), agent)
    if learner_paths(lay).update != "lean":
        with pytest.raises(ValueError, match="lean"):
            _filled(lay, CHUNK, T)
        return
    m = _filled(lay, CHUNK, T)
    a, b, c = _grads(m, 1), _grads(m, 1), _grads(m, 1, 61)
    ref = _grads(m, 0)
    for x, y, z, r, name in zip(a, b, c, ref, ("G", "stats", "norms")):
        assert torch.equal(x, y), name + ": two runs differ"
        assert torch.equal(x, z), name + ": the 61-CTA grid differs"
        # fp32 sums of ~1e5 terms in another order: a few 1e-5 of the largest entry (measured up to 2.2e-5)
        tol = 1e-4 * float(r.abs().max()) + 1e-7
        assert float((x - r).abs().max()) <= tol, name
    assert float(a[0].abs().max()) > 0 and float(a[1][0].abs()) > 0
    # every parameter the atomic update touches, the deterministic one touches
    assert torch.equal(a[0] != 0, ref[0] != 0)
    m.close()


def _update_run(seed_data):
    lay = scenario_layout(net_tables("large_grid", "ma2c"), "ma2c")
    m = _filled(lay, 2 * CHUNK, 8, dseed=seed_data)
    out = []
    g = torch.Generator(device=m.dev).manual_seed(seed_data + 1)
    for u in range(3):
        m.backward(None, 5e-4, 0.01)
        out.append([x.clone() for x in (m.P, m.MS, m.norms, m.stats)])
        for t in range(m.T):
            m.forward(m.obs_slot(), False)
            m.add_transition(torch.randn(m.R, lay.A, generator=g, device=m.dev) * 1000.0, False, False)
    m.close()
    return out


def test_two_learners_hold_equal_state_after_every_update():
    a, b = _update_run(3), _update_run(3)
    for u, (x, y) in enumerate(zip(a, b)):
        for name, s, t in zip(("P", "MS", "norms", "stats"), x, y):
            assert torch.equal(s, t), (u, name)
    assert not torch.equal(a[0][0], a[2][0])


def test_dx_fused_and_unstored_steps_are_refused():
    lay = scenario_layout(net_tables("large_grid", "ma2c"), "ma2c")
    m = _filled(lay, CHUNK, 4)
    m.dx_fused = True
    with pytest.raises(ValueError, match="dx_fused"):
        m.backward(None, 5e-4, 0.01)
    m.dx_fused = False
    m._acts_ok[1] = False
    with pytest.raises(RuntimeError, match="activation store"):
        m.backward(None, 5e-4, 0.01)
    from deeprl_signal_control_b200 import _lib
    with pytest.raises(RuntimeError, match="tscl_heads_loss"):
        _lib.check(_lib.lib().tscl_heads_loss(m._h, _lib.ptr(m.P), None, None, None, None, 1, 1, 1, 0.5, 0.01, 1.0,
                                              None, _lib.ptr(m.G), None, _lib.ptr(m.st_h), None, None))
    m.close()


# ---- driver ------------------------------------------------------------------------------------------------------
def _ckpt(d, step):
    from deeprl_signal_control_b200.agents import checkpoint as ck
    return ck.load_npz(os.path.join(d, "model", "checkpoint-%d.npz" % step))[0]


def _same_dir(a, b, step):
    wa, wb = _ckpt(a, step), _ckpt(b, step)
    assert sorted(wa) == sorted(wb)
    for n in wa:
        assert np.array_equal(wa[n], wb[n]), n
    for name in sorted(os.listdir(os.path.join(a, "data"))):
        if name.endswith(".csv"):
            assert open(os.path.join(a, "data", name), "rb").read() == open(os.path.join(b, "data", name), "rb").read(), name


def _scalars(d):
    from deeprl_signal_control_b200.agents.summary import decode_event, event_files, read_records
    files = event_files(os.path.join(d, "log"))
    assert len(files) == 1
    return [(step, vals) for _, step, _, vals in (decode_event(x) for x in read_records(files[0])[1:])]


def test_two_driver_runs_write_the_same_bytes(tmp_path):
    from deeprl_signal_control_b200.agents.train import train
    cfg = tmp_path / "config_ma2c_large.ini"
    cfg.write_text(_ini("ma2c", 240, 120))
    runs = [str(tmp_path / ("run%d" % k) / "ma2c") for k in range(2)]
    outs = [train(str(cfg), d, "all_test", n_replicas=256, summaries=True, deterministic=True) for d in runs]
    assert [o.episode_sets for o in outs] == [2, 2]
    _same_dir(runs[0], runs[1], 240)
    assert _scalars(runs[0]) == _scalars(runs[1])
    assert len(pd.read_csv(os.path.join(runs[0], "data", "train_reward.csv"))) > 0


def test_population_and_sweep_members_equal_their_solo_runs(tmp_path):
    from deeprl_signal_control_b200.agents.train import member_dir, train, train_sweep
    Rm = 64
    cfg = tmp_path / "config_ma2c_large.ini"
    cfg.write_text(_ini("ma2c", 120, 240))
    pop = train(str(cfg), str(tmp_path / "pop"), "after_train_test", n_replicas=Rm, seeds=[12, 13], deterministic=True)
    for s in (12, 13):
        solo_cfg = tmp_path / ("solo%d.ini" % s)
        solo_cfg.write_text(_ini("ma2c", 120, 240).replace("seed = 12", "seed = %d" % s))
        solo = str(tmp_path / ("solo%d" % s) / "ma2c")
        train(str(solo_cfg), solo, "after_train_test", n_replicas=Rm, deterministic=True)
        _same_dir(member_dir(str(tmp_path / "pop"), s, "ma2c"), solo, 120)
    assert pop.final_step == 120
    a = tmp_path / "a.ini"
    b = tmp_path / "b.ini"
    a.write_text(_ini("ma2c", 120, 240))
    b.write_text(_ini("ma2c", 120, 240).replace("lr_init = 5e-4", "lr_init = 1e-3").replace("gamma = 0.99",
                                                                                              "gamma = 0.95"))
    sw = train_sweep([str(a), str(b)], str(tmp_path / "sweep"), "after_train_test", n_replicas=Rm, deterministic=True)
    for name, path in (("a", a), ("b", b)):
        solo = str(tmp_path / ("solo_" + name) / "ma2c")
        train(str(path), solo, "after_train_test", n_replicas=Rm, deterministic=True)
        _same_dir(os.path.join(str(tmp_path / "sweep"), name, "ma2c"), solo, 120)
    assert sw.names == ["a", "b"]


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _rank_worker(rank, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=2, timeout=datetime.timedelta(seconds=300))
    from deeprl_signal_control_b200.agents.train import state_digest, train
    for run in ("r0", "r1"):
        res = train(os.path.join(out, "config_ma2c_large.ini"), os.path.join(out, run, "ma2c"), "no_test", n_replicas=128,
                    device=0, process_group=dist.group.WORLD, deterministic=True)
        with open(os.path.join(out, "%s_rank%d.digest" % (run, rank)), "wb") as f:
            f.write(state_digest(res.model))
    dist.destroy_process_group()


def test_two_gloo_ranks_end_with_the_same_digest_twice(tmp_path):
    import torch.multiprocessing as mp
    (tmp_path / "config_ma2c_large.ini").write_text(_ini("ma2c", 360, 240))
    mp.spawn(_rank_worker, args=(_free_port(), str(tmp_path)), nprocs=2, join=True)
    d = {(run, k): (tmp_path / ("%s_rank%d.digest" % (run, k))).read_bytes() for run in ("r0", "r1") for k in (0, 1)}
    assert len(set(d.values())) == 1
