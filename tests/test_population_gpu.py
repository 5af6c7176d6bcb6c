"""GPU: population training (K members of one A2C agent in one process, `BatchedA2C(seeds=...)`, `train(seeds=...)`).

* Grouped forward (tscl_policy_step_v2g): grid MA2C K = 4 x 1024 and K = 3 x 512, Monaco MA2C K = 2 x 1024, every member
  with its own weights; done = 1 then 0 with the activation store on, then the bootstrap 'v' forward.  pi, value,
  actions, c / h and the four store arrays are bit-identical to each member's own one-member learner (one
  tscl_policy_step_v2 launch on its slice, seed s_k, replica0 = 0).
* Independence: perturbing member 1's weights leaves members 0 and 2's rollouts bit-identical and their updated weights
  within the spread of two identical runs.
* Solo equivalence (grid MA2C, K = 3 x 512): every member's first n_step observations, actions and rewards are
  bit-identical to its solo `BatchedTrainer` run; after the first update its P and MS match the solo run's within the
  spread of two solo runs (the weight-gradient kernels add with atomics).
* Driver: `train(..., seeds=[12, 13] or [12], test_mode='all_test', summaries=True)` with one update leaves in every
  member directory the file set of the member's solo run, the same first train_reward.csv row bit for bit, a checkpoint
  within the two-run spread of the solo run's, post-training CSVs equal to scripts/evaluate.py's on that directory, and
  an event file with the member's own values.  A one-seed population is its seed's solo run.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import torch

from tests.test_train_driver_gpu import _ini

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_STEP = 10
# floor of the solo-equivalence bound, for a run in which two solo runs happen to agree bit for bit: three orders of
# magnitude above the measured spread of two solo runs (about 2e-12 on P after the first update), far below a
# misapplied member update
SPREAD_FLOOR = 1e-9
# two A2C runs of one build through the driver (one update of 120 steps) differ by a few 1e-8 (test_summary_gpu.py)
CKPT_DRIFT = 1e-6


def _scenario(scenario):
    from bench import build_scenario, make_layout

    class A:
        agent, policy = "ma2c", "lstm"
    A.scenario = scenario
    net, par = build_scenario(A)[:2]
    return net, par, make_layout(net, A)


def _population(lay, Rm, seeds):
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    m = BatchedA2C(lay, Rm, n_step=2, seeds=seeds, chunk=min(1024, Rm), store_acts=True)
    assert m.K == len(seeds) and m.R == len(seeds) * Rm and m.store_acts
    return m


def _solo(lay, Rm, seed):
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    return BatchedA2C(lay, Rm, n_step=2, seed=seed, chunk=min(1024, Rm), store_acts=True)


def _store_slice(st, k, Rm, rc):
    return st[k * (Rm // rc):(k + 1) * (Rm // rc)]


@pytest.mark.parametrize("scenario,K,Rm", [("large_grid", 4, 1024), ("large_grid", 3, 512), ("real_net", 2, 1024)])
def test_grouped_forward_is_bit_identical_to_member_launches(scenario, K, Rm):
    _, _, lay = _scenario(scenario)
    seeds = [12 + 7 * k for k in range(K)]
    m = _population(lay, Rm, seeds)
    solos = [_solo(lay, Rm, s) for s in seeds]
    for k in range(K):
        assert torch.equal(m.P[k], solos[k].P) and torch.equal(m.Wp[k], solos[k].Wp)
    assert not torch.equal(m.P[0], m.P[1])
    g = torch.Generator(device="cuda").manual_seed(3)
    m.h_fw.copy_(torch.rand(m.h_fw.shape, device="cuda", generator=g) * 2 - 1)
    m.c_fw.copy_(torch.randn(m.c_fw.shape, device="cuda", generator=g))
    rows = lambda k: slice(k * Rm, (k + 1) * Rm)
    for k, s in enumerate(solos):
        s.h_fw.copy_(m.h_fw[:, rows(k)]); s.c_fw.copy_(m.c_fw[:, rows(k)])
    for x in [m] + solos:
        for t in (x.st_x, x.st_g, x.st_c, x.st_h):
            t.fill_(float("nan"))
    rc = m.chunk
    for done in (True, False):
        obs = torch.rand(m.R, lay.n_obs, device="cuda", generator=g) * 2
        pi, val, act = (t.clone() for t in m.forward(obs, done))
        for k, s in enumerate(solos):
            spi, sval, sact = s.forward(obs[rows(k)].contiguous(), done)
            assert torch.equal(pi[rows(k)], spi), (done, k)
            assert torch.equal(val[rows(k)], sval), (done, k)
            assert torch.equal(act[rows(k)], sact), (done, k)
            assert torch.equal(m.c_fw[:, rows(k)], s.c_fw) and torch.equal(m.h_fw[:, rows(k)], s.h_fw), (done, k)
            for name in ("st_x", "st_g", "st_c", "st_h"):
                a, b = _store_slice(getattr(m, name), k, Rm, rc), getattr(s, name)
                assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (done, k, name)
    obs = torch.rand(m.R, lay.n_obs, device="cuda", generator=g) * 2
    _, val, _ = m.forward(obs, False, out_type="v")
    for k, s in enumerate(solos):
        _, sval, _ = s.forward(obs[rows(k)].contiguous(), False, out_type="v")
        assert torch.equal(val[rows(k)], sval)
        assert torch.equal(m.c_tmp[:, rows(k)], s.c_tmp) and torch.equal(m.h_tmp[:, rows(k)], s.h_tmp)
    torch.cuda.synchronize()


class FirstRollout:
    """The rollout (obs, actions, rewards) every learner of a class holds at its first backward."""

    def __init__(self):
        from deeprl_signal_control_b200.agents.learner import BatchedA2C
        self.orig, self.snaps = BatchedA2C.backward, {}
        me = self

        def backward(m, boot, lr, beta):
            if id(m) not in me.snaps:
                me.snaps[id(m)] = dict(obs=m.obs_hist.clone(), act=m.act_hist.clone(), rew=m.rew_hist.clone())
            return me.orig(m, boot, lr, beta)
        BatchedA2C.backward = backward

    def restore(self):
        from deeprl_signal_control_b200.agents.learner import BatchedA2C
        BatchedA2C.backward = self.orig


def _run(net, par, lay, Rm, seeds, perturb=None):
    """One rollout of N_STEP steps and its update: a population (list of seeds) or a solo run (one int)."""
    from deeprl_signal_control_b200.agents.learner import BatchedA2C
    from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
    from deeprl_signal_control_b200.sim import BatchedSim
    pop = isinstance(seeds, list)
    kw = dict(gamma=0.99, v_coef=0.5, max_grad_norm=40.0, alpha=0.99, eps=1e-5, reward_norm=2000.0, reward_clip=2.0,
              chunk=512, store_acts=True)
    m = BatchedA2C(lay, Rm, N_STEP, seeds=seeds, **kw) if pop else BatchedA2C(lay, Rm, N_STEP, seed=seeds, **kw)
    if perturb is not None:
        g = torch.Generator(device="cuda").manual_seed(9)
        m.P[perturb].add_(torch.randn(m.P.shape[1], device="cuda", generator=g) * 1e-2)
        m.pack_weights()
    sim = BatchedSim(net, par, m.R)
    tr = BatchedTrainer(sim, m, "ma2c", lr=5e-4, beta=0.01, seed0=seeds[0] if pop else seeds)
    rec = FirstRollout()
    try:
        tr.run(N_STEP)
    finally:
        rec.restore()
    torch.cuda.synchronize()
    assert tr.n_updates == 1
    return m, rec.snaps[id(m)]


@pytest.fixture(scope="module")
def grid():
    return _scenario("large_grid")


@pytest.fixture(scope="module")
def population_runs(grid):
    net, par, lay = grid
    seeds, Rm = [12, 13, 14], 512
    pop = _run(net, par, lay, Rm, seeds)
    solos = [_run(net, par, lay, Rm, s) for s in seeds]
    solo0_again = _run(net, par, lay, Rm, seeds[0])
    return seeds, Rm, pop, solos, solo0_again


def test_members_replay_their_solo_runs(population_runs):
    seeds, Rm, (m, snap), solos, (m0b, _) = population_runs
    spread = max(float((solos[0][0].P - m0b.P).abs().max()), float((solos[0][0].MS - m0b.MS).abs().max()))
    bound = max(2 * spread, SPREAD_FLOOR)
    for k, (s, ssnap) in enumerate(solos):
        rows = slice(k * Rm, (k + 1) * Rm)
        assert torch.equal(snap["obs"][:, rows], ssnap["obs"]), k
        assert torch.equal(snap["act"][:, rows], ssnap["act"]), k
        assert torch.equal(snap["rew"][:, rows], ssnap["rew"]), k
        dp = float((m.P[k] - s.P).abs().max()); dms = float((m.MS[k] - s.MS).abs().max())
        print("member %d (seed %d): |dP| %.3g, |dMS| %.3g, two-solo spread %.3g" % (k, seeds[k], dp, dms, spread))
        assert dp <= bound and dms <= bound, (k, dp, dms, bound)
        assert torch.equal(m.norms[k], m.member(k).norms)


def test_perturbing_one_member_leaves_the_others_alone(grid, population_runs):
    net, par, lay = grid
    seeds, Rm, (m, snap), solos, (m0b, _) = population_runs
    mp, psnap = _run(net, par, lay, Rm, seeds, perturb=1)
    spread = float((solos[0][0].P - m0b.P).abs().max())
    bound = max(2 * spread, SPREAD_FLOOR)
    r1 = slice(Rm, 2 * Rm)
    assert not torch.equal(snap["act"][:, r1], psnap["act"][:, r1])
    for k in (0, 2):
        rows = slice(k * Rm, (k + 1) * Rm)
        for key in ("obs", "act", "rew"):
            assert torch.equal(snap[key][:, rows], psnap[key][:, rows]), (k, key)
        assert float((m.P[k] - mp.P[k]).abs().max()) <= bound
        assert float((m.MS[k] - mp.MS[k]).abs().max()) <= bound


def _listing(d):
    out = {}
    for sub in ("data", "model", "log"):
        names = sorted(os.listdir(os.path.join(d, sub)))
        out[sub] = [("<log>" if n.endswith(".log") else "<events>" if n.startswith("events.") else n) for n in names]
    return out


@pytest.mark.parametrize("seeds", [[12, 13], [12]])
def test_driver_writes_each_members_solo_directory(tmp_path, seeds):
    from deeprl_signal_control_b200.agents import checkpoint as ck
    from deeprl_signal_control_b200.agents.summary import decode_event, event_files, read_records
    from deeprl_signal_control_b200.agents.train import member_dir, train
    Rm = 64
    cfg = tmp_path / "config_ma2c_large.ini"
    cfg.write_text(_ini("ma2c", 120, 240))
    pop = train(str(cfg), str(tmp_path / "pop"), "all_test", n_replicas=Rm, summaries=True, seeds=seeds)
    assert pop.final_step == 120 and pop.episode_sets == 1 and pop.env_samples == 120 * Rm * len(seeds)
    assert [m.batched.seed for m in pop.members] == seeds
    for k, s in enumerate(seeds):
        d = member_dir(str(tmp_path / "pop"), s, "ma2c")
        assert d == pop.dirs[k]
        solo_cfg = tmp_path / ("solo%d" % s) / "config_ma2c_large.ini"
        solo_cfg.parent.mkdir()
        solo_cfg.write_text(open(os.path.join(d, "data", "config_ma2c_large.ini")).read())
        assert "seed = %d" % s in solo_cfg.read_text()
        solo_dir = str(tmp_path / ("solo%d" % s) / "ma2c")
        solo = train(str(solo_cfg), solo_dir, "all_test", n_replicas=Rm, summaries=True)
        assert _listing(d) == _listing(solo_dir)
        rows = pd.read_csv(os.path.join(d, "data", "train_reward.csv"), index_col=0, float_precision="round_trip")
        srows = pd.read_csv(os.path.join(solo_dir, "data", "train_reward.csv"), index_col=0,
                            float_precision="round_trip")
        assert list(rows.columns) == list(srows.columns)
        assert rows.iloc[0].to_dict() == srows.iloc[0].to_dict(), k
        # the checkpoint after the one update, within the drift of two runs (the update sums with atomics)
        got_ck, want_ck = (ck.load_npz(os.path.join(x, "model", "checkpoint-120.npz"))[0] for x in (d, solo_dir))
        assert sorted(got_ck) == sorted(want_ck)
        assert max(float(np.abs(got_ck[n] - want_ck[n]).max()) for n in got_ck) <= CKPT_DRIFT
        # post-training CSVs against scripts/evaluate.py on the member directory
        r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", d],
                           capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stdout + r.stderr
        got = json.load(open(os.path.join(d, "eva_data", "ma2c_summary.json")))
        assert got["episode_mean_reward"] == [float(x) for x in pop.post_test[k][0]]
        for kind in ("control", "traffic", "trip"):
            name = "large_grid_ma2c_%s.csv" % kind
            assert open(os.path.join(d, "data", name)).read() == open(os.path.join(d, "eva_data", name)).read(), kind
        # the member's event file: its own train_reward and gradient norm
        files = event_files(os.path.join(d, "log"))
        assert len(files) == 1
        ev = [decode_event(x) for x in read_records(files[0])[1:]]
        tags = {t: v for _, _, _, vals in ev for t, v in vals}
        assert "train/fplstm_0a_gradnorm" in tags and "loss/fplstm_0a_total_loss" in tags
        assert tags["train_reward"] == pytest.approx(rows.iloc[0].avg_reward, rel=1e-6)
        assert tags["train/fplstm_0a_gradnorm"] == pytest.approx(float(pop.members[k].batched.norms[0]), rel=1e-6)
