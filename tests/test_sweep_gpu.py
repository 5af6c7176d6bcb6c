"""GPU: hyperparameter sweeps (K members of one A2C agent, one config each, in one process).

* Simulator: grid MA2C and Monaco MA2C on R = 3 x 64 replicas with coop_gamma (0.9, 0.75, 0.5) per 64-replica block.
  Over a short train-mode episode, then `observe` in test mode, in record mode and through host-range steps, every
  block's obs / reward / greward / done are bit-identical to a simulator built with that block's coop_gamma.  Setting
  every replica to the configured value, or setting and then clearing, is bit-identical to never calling the setter.
* Kernels: tscl_returns_g and tscl_device_transition_g against the one-member entry points on each member's rows
  copied out, with distinct gamma / reward_norm / reward_clip per member, norm 0 and clip 0 included.
* Solo equivalence (grid MA2C, K = 3 x 512; lr_init, entropy_coef_init, gamma, reward_norm, coop_gamma, value_coef and
  max_grad_norm differ, two members share a seed): each member's first rollout is bit-identical to its solo run (MA2C
  from its config on a simulator built with its coop_gamma) and its first update is within the two-solo spread.  Two
  planted defects (members' gamma swapped; every replica on member 0's coop_gamma) fail that comparison.
* Driver: `train_sweep` with configs differing in lr_init and coop_gamma, and a one-config sweep, leave each member the
  directory of its solo `train()` (file set, first training row, checkpoint, post-training CSVs, event file).
"""
import configparser
import dataclasses
import json
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import torch

from tests.test_population_gpu import CKPT_DRIFT, SPREAD_FLOOR, FirstRollout, _listing
from tests.test_train_driver_gpu import _ini

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CG = (0.9, 0.75, 0.5)
RB = 64                                     # replicas per coop_gamma block in the simulator tests


def _scenario(scenario, cg=0.9, episode_sec=None):
    """(net, params) of grid / Monaco MA2C as bench.py builds them, with coop_gamma = cg: the obs program's scaled
    entries (build_obs_program: the neighbour waves) and the reward's spatial discount"""
    from bench import build_scenario

    class A:
        agent, policy = "ma2c", "lstm"
    A.scenario = scenario
    net, par = build_scenario(A)[:2]
    scaled = np.asarray(net.obs_scale) != 1.0
    assert scaled.any() and np.all(np.asarray(net.obs_scale)[scaled] == np.float32(par.coop_gamma))
    net = dataclasses.replace(net, obs_scale=np.where(scaled, np.float32(cg), np.float32(1.0)).astype(np.float32))
    par = dataclasses.replace(par, coop_gamma=cg, **({} if episode_sec is None else dict(episode_length_sec=episode_sec)))
    return net, par


def _sims(scenario, episode_sec):
    """the sweep simulator (built with CG[0], blocks set to CG) and one simulator per block built with its cg"""
    from deeprl_signal_control_b200.sim import BatchedSim
    net, par = _scenario(scenario, CG[0], episode_sec)
    sweep = BatchedSim(net, par, len(CG) * RB)
    sweep.set_replica_coop_gamma(np.repeat(np.asarray(CG, np.float32), RB))
    solos = [BatchedSim(*_scenario(scenario, cg, episode_sec), RB) for cg in CG]
    return sweep, solos


def _reset(sims, ep):
    seeds = np.arange(len(CG) * RB, dtype=np.uint64) * np.uint64(7) + np.uint64(1000 * ep + 12)
    sims[0].reset(seeds)
    for k, s in enumerate(sims[1]):
        s.reset(seeds[k * RB:(k + 1) * RB])


def _inputs(sim, g):
    n = sim.net
    act = torch.stack([torch.randint(0, int(na), (sim.R,), device="cuda", generator=g, dtype=torch.int32)
                       for na in n.n_a_ls], 1).contiguous()
    fp = torch.rand(sim.R, n.n_nodes, n.max_na, device="cuda", generator=g).contiguous()
    return act, fp


def _same_block(got, want, k, what):
    rows = slice(k * RB, (k + 1) * RB)
    for name, a, b in zip(("obs", "reward", "greward", "done"), got, want):
        assert torch.equal(torch.as_tensor(a)[rows].cpu(), torch.as_tensor(b).cpu()), (what, k, name)


@pytest.mark.parametrize("scenario", ["large_grid", "real_net"])
def test_per_replica_coop_gamma_equals_simulators_built_with_it(scenario):
    sweep, solos = _sims(scenario, episode_sec=150)
    g = torch.Generator(device="cuda").manual_seed(5)
    steps = int(np.ceil(150 / sweep.params.control_interval_sec))
    # one train-mode episode with tsc_step, then observe in test mode
    _reset((sweep, solos), 0)
    for s in [sweep] + solos:
        s.set_train_mode(True)
    for t in range(steps):
        act, fp = _inputs(sweep, g)
        got = [x.clone() for x in sweep.step(act, fp)]
        for k, s in enumerate(solos):
            rows = slice(k * RB, (k + 1) * RB)
            _same_block(got, s.step(act[rows].contiguous(), fp[rows].contiguous()), k, ("step", t))
    assert bool(got[3].all())
    _, fp = _inputs(sweep, g)
    for s in [sweep] + solos:
        s.set_train_mode(False)
    obs = sweep.observe(fp).clone()
    for k, s in enumerate(solos):
        rows = slice(k * RB, (k + 1) * RB)
        assert torch.equal(obs[rows], s.observe(fp[rows].contiguous())), ("observe", k)
    # record mode, train rewards
    _reset((sweep, solos), 1)
    for s in [sweep] + solos:
        s.set_train_mode(True)
        s.set_record(True)
    for t in range(4):
        act, fp = _inputs(sweep, g)
        got = [x.clone() for x in sweep.step_record(act, fp)]
        for k, s in enumerate(solos):
            rows = slice(k * RB, (k + 1) * RB)
            want = s.step_record(act[rows].contiguous(), fp[rows].contiguous())
            _same_block(got[:4], want[:4], k, ("record", t))
            assert torch.equal(got[4][rows], want[4]), ("record stats", t, k)
    for s in [sweep] + solos:
        s.set_record(False)
    # host-range steps: two ranges across the member blocks, synchronous and asynchronous
    _reset((sweep, solos), 2)
    R, n = sweep.R, sweep.net
    pin = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype).pin_memory().numpy()
    out = (pin(R, n.n_obs), pin(R, n.n_nodes), pin(R), pin(R, dtype=torch.uint8))
    for t in range(4):
        act, fp = _inputs(sweep, g)
        a_h, f_h = act.cpu().numpy(), fp.cpu().numpy()
        for r0, cnt, sync in ((0, 96, True), (96, R - 96, False)):
            sl = slice(r0, r0 + cnt)
            sweep.step_host_range(r0, cnt, a_h[sl], f_h[sl], *(o[sl] for o in out), sync=sync)
        torch.cuda.synchronize()
        for k, s in enumerate(solos):
            rows = slice(k * RB, (k + 1) * RB)
            want = [x.copy() for x in s.step_host(a_h[rows], f_h[rows])]
            _same_block([torch.from_numpy(o) for o in out], [torch.from_numpy(w) for w in want], k, ("host range", t))


@pytest.mark.parametrize("scenario", ["large_grid", "real_net"])
def test_setter_at_the_config_value_or_cleared_is_the_plain_simulator(scenario):
    from deeprl_signal_control_b200.sim import BatchedSim
    net, par = _scenario(scenario, 0.9, episode_sec=100)
    R = 2 * RB
    plain, same, cleared = (BatchedSim(net, par, R) for _ in range(3))
    same.set_replica_coop_gamma(np.full(R, 0.9, np.float32))
    cleared.set_replica_coop_gamma(np.linspace(0.2, 0.8, R))
    cleared.set_replica_coop_gamma(None)
    seeds = np.arange(R, dtype=np.uint64) + np.uint64(40)
    g = torch.Generator(device="cuda").manual_seed(8)
    for s in (plain, same, cleared):
        s.reset(seeds)
        s.set_train_mode(True)
    for t in range(int(np.ceil(100 / par.control_interval_sec))):
        act, fp = _inputs(plain, g)
        want = [x.clone() for x in plain.step(act, fp)]
        for s in (same, cleared):
            got = s.step(act, fp)
            for a, b in zip(got, want):
                assert torch.equal(a, b), t
    with pytest.raises(ValueError):
        plain.set_replica_coop_gamma(np.ones(R + 1))


def _learner(R):
    from bench import make_layout
    from deeprl_signal_control_b200.agents.learner import BatchedA2C

    class A:
        agent, policy, scenario = "ma2c", "lstm", "large_grid"
    net, _ = _scenario("large_grid")
    return BatchedA2C(make_layout(net, A), R, 4, seed=1, chunk=R, store_acts=False)


def test_grouped_returns_and_transition_equal_the_member_launches():
    import ctypes as C
    from deeprl_signal_control_b200 import _lib
    lib, K, Rm, T = _lib.lib(), 3, 128, 7
    m = _learner(K * Rm)
    A, R = m.lay.A, K * Rm
    p = lambda t: C.c_void_p(t.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(2)
    f32 = dict(device="cuda", dtype=torch.float32)
    rew, val = (torch.randn(T, R, A, generator=g, **f32) for _ in range(2))
    boot = torch.randn(R, A, generator=g, **f32)
    dpost = torch.tensor([0, 0, 1, 0, 0, 0, 1], **f32)
    gam = torch.tensor([0.99, 0.9, 0.75], **f32)
    Rs, Adv = torch.full_like(rew, float("nan")), torch.full_like(rew, float("nan"))
    _lib.check(lib.tscl_returns_g(m._h, p(rew), p(val), p(boot), p(dpost), p(gam), C.c_int32(K), C.c_int32(T),
                                  C.c_int64(R), p(Rs), p(Adv), st))
    for k in range(K):
        rows = slice(k * Rm, (k + 1) * Rm)
        r, v, b = rew[:, rows].contiguous(), val[:, rows].contiguous(), boot[rows].contiguous()
        Rs1, Adv1 = torch.empty_like(r), torch.empty_like(r)
        _lib.check(lib.tscl_returns(m._h, p(r), p(v), p(b), p(dpost), C.c_float(float(gam[k])), C.c_int32(T),
                                    C.c_int64(Rm), p(Rs1), p(Adv1), st))
        assert torch.equal(Rs[:, rows], Rs1) and torch.equal(Adv[:, rows], Adv1), k
    # reward hand-over: norm 0 (off) and clip 0 (off) among the members
    norms, clips = torch.tensor([2000.0, 0.0, 3.0], **f32), torch.tensor([2.0, 1.5, 0.0], **f32)
    r = torch.randn(R, A, generator=g, **f32) * 4000
    grew = torch.randn(R, generator=g, **f32)
    acc0 = torch.randn(R, generator=g, **f32)
    hist, acc = torch.full_like(r, float("nan")), acc0.clone()
    _lib.check(lib.tscl_device_transition_g(m._h, p(r), p(hist), C.c_int64(R * A), p(norms), p(clips), C.c_int32(K),
                                            p(grew), p(acc), C.c_int64(R), st))
    for k in range(K):
        rows = slice(k * Rm, (k + 1) * Rm)
        r1, gr1, acc1 = r[rows].contiguous(), grew[rows].contiguous(), acc0[rows].clone()
        hist1 = torch.empty_like(r1)
        _lib.check(lib.tscl_device_transition(m._h, p(r1), p(hist1), C.c_int64(Rm * A), C.c_float(float(norms[k])),
                                              C.c_float(float(clips[k])), p(gr1), p(acc1), C.c_int64(Rm), st))
        assert torch.equal(hist[rows], hist1) and torch.equal(acc[rows], acc1), k
    assert float(hist[:Rm].abs().max()) <= 2.0 and float(hist[Rm:2 * Rm].abs().max()) <= 1.5
    assert float(hist[2 * Rm:].abs().max()) > 2.0                 # clip 0 leaves member 2 unclipped
    torch.cuda.synchronize()


# ---- solo equivalence -----------------------------------------------------------------------------------------------
N_STEP = 10
RM = 512
MEMBERS = [   # (seed, coop_gamma, [MODEL_CONFIG] changes); members 0 and 2 share a seed
    (12, 0.9, {}),
    (13, 0.75, dict(lr_init="1e-3", lr_decay="linear", lr_min="1e-5", entropy_coef_init="0.02", gamma="0.95",
                    reward_norm="3000.0", value_coef="0.25", max_grad_norm="20")),
    (12, 0.5, dict(lr_init="2e-4", entropy_coef_init="0.005", gamma="0.9", reward_norm="1000.0", value_coef="1.0",
                   max_grad_norm="5")),
]


def _member_cfg(seed, cg, changes):
    c = configparser.ConfigParser()
    c.read_string(_ini("ma2c", 3600, 3600))
    c["MODEL_CONFIG"]["batch_size"] = str(N_STEP)
    c["ENV_CONFIG"]["seed"], c["ENV_CONFIG"]["coop_gamma"] = str(seed), str(cg)
    for k, v in changes.items():
        c["MODEL_CONFIG"][k] = v
    return c


def _model(net, mc, **kw):
    from deeprl_signal_control_b200.agents.models import MA2C
    return MA2C(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, 3600, mc, n_replicas=RM, obs_off=net.node_obs_off,
                chunk=RM, store_acts=True, **kw)


def _sweep_run(members, sim_cg=None, gammas=None):
    """One rollout and update of the sweep; `sim_cg` / `gammas` plant a defect (simulator blocks / learner gammas)."""
    from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
    from deeprl_signal_control_b200.sim import BatchedSim
    cfgs = [_member_cfg(*m) for m in members]
    net, par = _scenario("large_grid", members[0][1])
    model = _model(net, cfgs[0]["MODEL_CONFIG"], seeds=[m[0] for m in members],
                   member_configs=[c["MODEL_CONFIG"] for c in cfgs])
    b = model.batched
    if gammas is not None:
        b.gamma_dev.copy_(torch.tensor(gammas, device=b.dev))
    sim = BatchedSim(net, par, b.R)
    tr = BatchedTrainer(sim, b, "ma2c", model.lr_schedulers, model.beta_schedulers, seed0=members[0][0],
                        coop_gamma=sim_cg or [m[1] for m in members])
    return _go(tr, b)


def _solo_run(member):
    from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
    from deeprl_signal_control_b200.sim import BatchedSim
    seed, cg, _ = member
    mc = _member_cfg(*member)["MODEL_CONFIG"]
    net, par = _scenario("large_grid", cg)
    model = _model(net, mc, seed=seed)
    sim = BatchedSim(net, par, RM)
    tr = BatchedTrainer(sim, model.batched, "ma2c", model.lr_scheduler, model.beta_scheduler, seed0=seed)
    return _go(tr, model.batched)


def _go(tr, m):
    rec = FirstRollout()
    try:
        tr.run(N_STEP)
    finally:
        rec.restore()
    torch.cuda.synchronize()
    assert tr.n_updates == 1
    return m, rec.snaps[id(m)]


@pytest.fixture(scope="module")
def solo_runs():
    solos = [_solo_run(m) for m in MEMBERS]
    again = _solo_run(MEMBERS[1])
    spread = max(float((solos[1][0].P - again[0].P).abs().max()), float((solos[1][0].MS - again[0].MS).abs().max()))
    return solos, max(2 * spread, SPREAD_FLOOR)


def _mismatches(run, solos, bound):
    (m, snap), out = run, []
    for k, (s, ssnap) in enumerate(solos):
        rows = slice(k * RM, (k + 1) * RM)
        for key in ("obs", "act", "rew"):
            if not torch.equal(snap[key][:, rows], ssnap[key]):
                out.append((k, key))
        dp, dms = float((m.P[k] - s.P).abs().max()), float((m.MS[k] - s.MS).abs().max())
        print("member %d: |dP| %.3g, |dMS| %.3g, bound %.3g" % (k, dp, dms, bound))
        if not (dp <= bound and dms <= bound):
            out.append((k, "update", dp, dms))
    return out


def test_members_replay_their_solo_runs(solo_runs):
    solos, bound = solo_runs
    run = _sweep_run(MEMBERS)
    m = run[0]
    assert m.K == 3 and m.gamma_dev is not None and m.rscale_differs
    assert [m.member(k).gamma for k in range(3)] == [0.99, 0.95, 0.9]
    assert _mismatches(run, solos, bound) == []


def test_swapped_gammas_are_caught(solo_runs):
    solos, bound = solo_runs
    bad = _mismatches(_sweep_run(MEMBERS, gammas=[0.95, 0.99, 0.9]), solos, bound)
    assert {x[0] for x in bad if x[1] == "update"} == {0, 1}, bad


def test_one_coop_gamma_for_every_replica_is_caught(solo_runs):
    solos, bound = solo_runs
    bad = _mismatches(_sweep_run(MEMBERS, sim_cg=[MEMBERS[0][1]] * 3), solos, bound)
    assert (1, "rew") in bad and (2, "rew") in bad and not any(x[0] == 0 for x in bad), bad


# ---- driver ---------------------------------------------------------------------------------------------------------
def _write_cfg(path, changes=None):
    c = configparser.ConfigParser()
    c.read_string(_ini("ma2c", 120, 240))
    for (sec, key), v in (changes or {}).items():
        c[sec][key] = v
    with open(path, "w") as f:
        c.write(f)
    return str(path)


@pytest.mark.parametrize("n_members", [2, 1])
def test_driver_writes_each_members_solo_directory(tmp_path, n_members):
    from deeprl_signal_control_b200.agents import checkpoint as ck
    from deeprl_signal_control_b200.agents.summary import decode_event, event_files, read_records
    from deeprl_signal_control_b200.agents.train import sweep_dir, train, train_sweep
    Rm = 64
    (tmp_path / "cfg").mkdir()
    paths = [_write_cfg(tmp_path / "cfg" / "lr5e-4.ini"),
             _write_cfg(tmp_path / "cfg" / "lr1e-3_cg075.ini",
                        changes={("MODEL_CONFIG", "lr_init"): "1e-3", ("ENV_CONFIG", "coop_gamma"): "0.75"})][:n_members]
    names = [os.path.splitext(os.path.basename(p))[0] for p in paths]
    sw = train_sweep(paths, str(tmp_path / "sweep"), "all_test", n_replicas=Rm, summaries=True)
    assert sw.final_step == 120 and sw.episode_sets == 1 and sw.env_samples == 120 * Rm * n_members
    assert sw.names == names
    for k, (name, path) in enumerate(zip(names, paths)):
        d = sweep_dir(str(tmp_path / "sweep"), name, "ma2c")
        assert d == sw.dirs[k]
        assert open(os.path.join(d, "data", os.path.basename(path))).read() == open(path).read()
        solo_dir = str(tmp_path / ("solo_" + name) / "ma2c")
        solo = train(path, solo_dir, "all_test", n_replicas=Rm, summaries=True)
        assert solo.final_step == 120
        assert _listing(d) == _listing(solo_dir)
        rows = pd.read_csv(os.path.join(d, "data", "train_reward.csv"), index_col=0, float_precision="round_trip")
        srows = pd.read_csv(os.path.join(solo_dir, "data", "train_reward.csv"), index_col=0,
                            float_precision="round_trip")
        assert list(rows.columns) == list(srows.columns)
        assert rows.iloc[0].to_dict() == srows.iloc[0].to_dict(), k
        got_ck, want_ck = (ck.load_npz(os.path.join(x, "model", "checkpoint-120.npz"))[0] for x in (d, solo_dir))
        assert sorted(got_ck) == sorted(want_ck)
        assert max(float(np.abs(got_ck[n] - want_ck[n]).max()) for n in got_ck) <= CKPT_DRIFT
        r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", d],
                           capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stdout + r.stderr
        got = json.load(open(os.path.join(d, "eva_data", "ma2c_summary.json")))
        assert got["episode_mean_reward"] == [float(x) for x in sw.post_test[k][0]]
        for kind in ("control", "traffic", "trip"):
            fname = "large_grid_ma2c_%s.csv" % kind
            assert open(os.path.join(d, "data", fname)).read() == open(os.path.join(d, "eva_data", fname)).read(), kind
        files = event_files(os.path.join(d, "log"))
        assert len(files) == 1
        ev = [decode_event(x) for x in read_records(files[0])[1:]]
        tags = {t: v for _, _, _, vals in ev for t, v in vals}
        assert tags["train_reward"] == pytest.approx(rows.iloc[0].avg_reward, rel=1e-6)
        assert tags["train/fplstm_0a_gradnorm"] == pytest.approx(float(sw.members[k].batched.norms[0]), rel=1e-6)
