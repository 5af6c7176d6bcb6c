"""GPU: IQL members (BatchedIQL with seeds / member_configs, tscl_q_*_g) against solo runs, bit for bit.

* Kernels, through the learner at K = 3 members of R_m = 300 replicas (partial tiles) on the grid and Monaco layouts, LR
  and DQN: the grouped explore forward, TD round (a capped and an uncapped tile-group count), clip + Adam with the
  summary rows, and the per-member reward scaling equal three solo learners fed the same rows.  A perturbed member
  leaves the others' round unchanged.
* Learner: three members over several updates of a rollout equal three solo BatchedIQLTrainer runs.
* Driver: every member directory of train_iql_population / train_iql_sweep equals its solo train() directory: CSV
  bytes, checkpoint arrays with the Adam state, event scalars, and the post-training CSVs scripts/evaluate.py writes.
"""
import configparser
import gc
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.test_learner_reference_golden_cpu import INI

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K, RM, B = 3, 300, 48


@pytest.fixture(autouse=True)
def _free_device_memory():
    """Each test's learners (their handles own the TD partial buffers) and torch's cached blocks go back to the device
    before the next test."""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _net(scenario, agent):
    if scenario == "large_grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid
        return build_large_grid(agent=agent)
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    return real_net_tables(agent)


def _cfgs(**per_member):
    """K [MODEL_CONFIG] sections of the golden INI with a short ring (wrapped within a few episodes), member k with
    per_member[key][k]"""
    out = []
    for k in range(K):
        cp = configparser.ConfigParser(); cp.read_string(INI.replace("buffer_size = 1000", "buffer_size = %d" % B))
        for key, vals in per_member.items():
            cp["MODEL_CONFIG"][key] = str(vals[k])
        out.append(cp["MODEL_CONFIG"])
    return out


def _layout(scenario, kind):
    from deeprl_signal_control_b200.agents.layout import QLayout
    net = _net(scenario, "iql" + kind[0])
    off = np.asarray(net.node_obs_off)
    n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
    cfg = _cfgs()[0]
    return QLayout(kind, n_s, net.n_a_ls, net.n_w_ls, off, net.n_obs, n_fc=cfg.getint("num_fc"),
                   n_ft=cfg.getint("num_fc") // 4, n_h=cfg.getint("num_h"), max_na=net.max_na), net


def _pair(scenario, kind, Rm=RM, **per_member):
    """(members, [solo]): a K-member learner and K solo learners with member k's config, the members' weights perturbed
    apart (each solo learner holds its member's)"""
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL
    lay, net = _layout(scenario, kind)
    cfgs = _cfgs(**per_member)
    pop = BatchedIQL(lay, Rm, cfgs[0], kind, device=0, seeds=[12, 12, 13], member_configs=cfgs)
    solo = [BatchedIQL(lay, Rm, cfgs[k], kind, device=0) for k in range(K)]
    g = torch.Generator(device="cuda").manual_seed(3)
    pop.P.add_(torch.randn(pop.P.shape, device="cuda", generator=g) * 0.05)
    for k, m in enumerate(solo):
        m.P.copy_(pop.P[k])
    return pop, solo, net


def _fill(pop, solo, net, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    pop.s.copy_(torch.rand(pop.s.shape, device="cuda", generator=g) * 2)
    pop.s1.copy_(torch.rand(pop.s1.shape, device="cuda", generator=g) * 2)
    na = torch.tensor(net.n_a_ls, device="cuda")
    pop.a.copy_((torch.rand(pop.a.shape, device="cuda", generator=g) * na).to(torch.int8))
    pop.r.copy_(torch.randn(pop.r.shape, device="cuda", generator=g))
    pop.done.copy_((torch.rand(pop.done.shape, device="cuda", generator=g) < 0.1).to(torch.uint8))
    pop.cum_size = B + 7                                   # wrapped
    Rm = pop.R_m
    for k, m in enumerate(solo):
        for name in ("s", "s1", "a", "r", "done"):
            getattr(m, name).copy_(getattr(pop, name)[:, k * Rm:(k + 1) * Rm])
        m.cum_size = pop.cum_size


LAYOUTS = [("large_grid", "lr"), ("large_grid", "dqn"), ("real_net", "lr"), ("real_net", "dqn")]


@pytest.mark.parametrize("scenario,kind", LAYOUTS)
def test_explore_and_transition_equal_the_solo_launches(scenario, kind):
    pop, solo, net = _pair(scenario, kind, reward_norm=[3.0, 30.0, 0.0], reward_clip=[2.0, 0.0, 0.5])
    assert not pop._one_scaling
    g = torch.Generator(device="cuda").manual_seed(5)
    obs = torch.rand(K * RM, net.n_obs, device="cuda", generator=g) * 2
    rew = torch.randn(K * RM, net.n_nodes, device="cuda", generator=g) * 10
    grew = torch.randn(K * RM, device="cuda", generator=g)
    acc = torch.zeros(K * RM, device="cuda")
    pop.cum_size = 5
    pop.explore(obs, [0.0, 1.0, 0.3], 17)
    pop.add_transition(rew, grew, acc, True)
    for k, m in enumerate(solo):
        rows = slice(k * RM, (k + 1) * RM)
        m.cum_size = 5
        m.explore(obs[rows].contiguous(), [0.0, 1.0, 0.3][k], 17)
        acc_k = torch.zeros(RM, device="cuda")
        m.add_transition(rew[rows].contiguous(), grew[rows].contiguous(), acc_k, True)
        torch.cuda.synchronize()
        assert torch.equal(pop.q[rows], m.q) and torch.equal(pop.act[rows], m.act), k
        assert torch.equal(pop.s[5, rows], m.s[5]) and torch.equal(pop.a[5, rows], m.a[5]), k
        assert torch.equal(pop.r[5, rows], m.r[5]) and torch.equal(pop.done[5, rows], m.done[5]), k
        assert torch.equal(acc[rows], acc_k), k
    # ε = 1 explores every row, ε = 0 none
    greedy = pop.q[RM:2 * RM].argmax(-1).to(torch.int32)
    assert not torch.equal(pop.act[RM:2 * RM], greedy)


@pytest.mark.parametrize("scenario,kind", LAYOUTS)
# R_m = 300: 94 tiles of 64 rows, more than the tile groups a device of 132 SMs gives any layout here (at most 8 CTAs of
# 256 threads per SM over >= 25 agents: <= 43 groups); R_m = 10: 4 tiles, fewer than the >= 5 groups of every layout
@pytest.mark.parametrize("Rm", [RM, 10])
def test_td_and_adam_rounds_equal_the_solo_rounds(scenario, kind, Rm):
    from deeprl_signal_control_b200.agents.learner_iql import N_ROUNDS
    pop, solo, net = _pair(scenario, kind, Rm=Rm, gamma=[0.99, 0.9, 0.5], max_grad_norm=[40, 1e-4, 0],
                           lr_init=[1e-4, 5e-4, 1e-3])
    _fill(pop, solo, net)
    lrs = [1e-4, 5e-4, 1e-3]
    rec = torch.zeros(K, N_ROUNDS, pop.n_agent, 4, device="cuda")
    for rnd in range(2):
        pop.td_round(rnd, lrs, rec=rec[:, rnd])
    for k, m in enumerate(solo):
        rec_k = torch.zeros(N_ROUNDS, m.n_agent, 4, device="cuda")
        for rnd in range(2):
            m.td_round(rnd, lrs[k], rec=rec_k[rnd])
        torch.cuda.synchronize()
        assert torch.equal(pop.idx, m.idx)                 # one draw serves every member
        assert torch.equal(pop.grad[k], m.grad), k
        assert torch.equal(pop.P[k], m.P) and torch.equal(pop.M[k], m.M) and torch.equal(pop.V[k], m.V), k
        assert torch.equal(pop.losses[k], m.losses) and torch.equal(pop.norms[k], m.norms), k
        assert torch.equal(rec[k], rec_k), k
    assert pop.t == solo[0].t == 2
    assert float(pop.norms[1, :2].min()) > 1e-4                 # member 1 is clipped; member 2 has no clip at all


def test_a_perturbed_member_leaves_the_others_alone():
    pop, solo, net = _pair("large_grid", "dqn")
    _fill(pop, solo, net)
    state = [t.clone() for t in (pop.P, pop.M, pop.V)]
    pop.td_round(0, [1e-4] * K)
    ref = [t.clone() for t in (pop.P, pop.M, pop.V, pop.grad)]
    for t, s in zip((pop.P, pop.M, pop.V), state):
        t.copy_(s)
    pop.t = 0
    pop.P[1].add_(0.01)
    pop.td_round(0, [1e-4] * K)
    torch.cuda.synchronize()
    for k in (0, 2):
        for a, b in zip((pop.P, pop.M, pop.V, pop.grad), ref):
            assert torch.equal(a[k], b[k]), k
    assert not torch.equal(pop.grad[1], ref[3][1])


@pytest.mark.parametrize("kind", ["lr", "dqn"])
def test_learner_members_over_several_updates_equal_solo_trainers(kind):
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL, BatchedIQLTrainer
    from deeprl_signal_control_b200.agents.models import iql_schedulers
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    lay, net = _layout("large_grid", kind)
    par = EnvParams(agent="iql" + kind[0], episode_length_sec=100)          # 20-step episodes
    cfgs = _cfgs(gamma=[0.99, 0.9, 0.99], lr_init=[1e-4, 1e-3, 1e-4], epsilon_init=[1.0, 0.5, 1.0],
                 reward_norm=[3.0, 3.0, 30.0])
    seeds = [12, 13, 12]
    pop = BatchedIQL(lay, RM, cfgs[0], kind, device=0, seeds=seeds, member_configs=cfgs)
    sch = [iql_schedulers(c, 1000) for c in cfgs]
    tr = BatchedIQLTrainer(BatchedSim(net, par, K * RM, device=0), pop, [s[0] for s in sch], [s[1] for s in sch])
    tr.run(70)
    torch.cuda.synchronize()
    assert tr.n_updates == 3 and len(tr.episode_rewards) == 3
    for k in range(K):
        m = BatchedIQL(lay, RM, cfgs[k], kind, device=0)
        lr_s, eps_s = iql_schedulers(cfgs[k], 1000)
        t = BatchedIQLTrainer(BatchedSim(net, par, RM, device=0), m, lr_s, eps_s, seed0=seeds[k])
        t.run(70)
        torch.cuda.synchronize()
        v = pop.member(k)
        assert torch.equal(v.P, m.P) and torch.equal(v.M, m.M) and torch.equal(v.V, m.V) and v.t == m.t, k
        assert torch.equal(v.losses, m.losses) and torch.equal(v.norms, m.norms), k
        assert tr.member(k).episode_rewards == t.episode_rewards, k
        del m, t
        gc.collect()


# ---- driver ------------------------------------------------------------------------------------------------------
def _ini(agent, **model):
    from tests.test_train_driver_gpu import _ini as ini
    text = ini(agent, 120, 60).replace("episode_length_sec = 600", "episode_length_sec = 300")   # T = 60
    text = text.replace("buffer_size = 1000", "buffer_size = 200")
    for key, val in model.items():
        text = "\n".join(("%s = %s" % (key, val)) if line.startswith(key + " =") else line for line in text.split("\n"))
    return text


def _same_dir(a, b, step):
    from deeprl_signal_control_b200.agents import checkpoint as ck
    (wa, ea), (wb, eb) = (ck.load_npz(os.path.join(d, "model", "checkpoint-%d.npz" % step)) for d in (a, b))
    assert sorted(wa) == sorted(wb) and sorted(ea) == sorted(eb) and "adam_m" in ea
    for n in wa:
        assert np.array_equal(wa[n], wb[n]), n
    for n in ea:
        assert np.array_equal(ea[n], eb[n]), n
    names = sorted(x for x in os.listdir(os.path.join(a, "data")) if x.endswith(".csv"))
    assert names == sorted(x for x in os.listdir(os.path.join(b, "data")) if x.endswith(".csv")) and len(names) == 4
    for name in names:
        assert open(os.path.join(a, "data", name), "rb").read() == open(os.path.join(b, "data", name), "rb").read(), name
    from tests.test_deterministic_gpu import _scalars
    assert _scalars(a) == _scalars(b)


def _evaluate_script_equals_post_test(d, agent):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", d,
                        "--evaluation-policy-type", "default"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    assert json.load(open(os.path.join(d, "eva_data", "%s_summary.json" % agent)))["seeds"]
    for kind in ("control", "traffic"):
        name = "large_grid_%s_%s.csv" % (agent, kind)
        assert open(os.path.join(d, "data", name)).read() == open(os.path.join(d, "eva_data", name)).read(), kind


@pytest.mark.parametrize("agent", ["iqll", "iqld"])
def test_population_members_equal_their_solo_runs(tmp_path, agent):
    from deeprl_signal_control_b200.agents.train import member_dir, train, train_iql_population
    cfg = tmp_path / ("config_%s_large.ini" % agent)
    cfg.write_text(_ini(agent))
    pop = train_iql_population(str(cfg), str(tmp_path / "pop"), [12, 13], "all_test", n_replicas=64, summaries=True)
    assert pop.final_step == 120 and pop.episode_sets == 2
    for s in (12, 13):
        d = tmp_path / ("solo%d" % s)
        d.mkdir()
        solo_cfg = d / ("config_%s_large.ini" % agent)
        solo_cfg.write_text(_ini(agent).replace("seed = 12", "seed = %d" % s))
        train(str(solo_cfg), str(d / agent), "all_test", n_replicas=64, summaries=True)
        md = member_dir(str(tmp_path / "pop"), s, agent)
        c = configparser.ConfigParser(); c.read(os.path.join(md, "data", solo_cfg.name))
        assert c["ENV_CONFIG"].getint("seed") == s
        _same_dir(md, str(d / agent), 120)
    _evaluate_script_equals_post_test(member_dir(str(tmp_path / "pop"), 13, agent), agent)


def test_sweep_members_equal_their_solo_runs(tmp_path):
    from deeprl_signal_control_b200.agents.train import sweep_dir, train, train_iql_sweep
    a, b = tmp_path / "a.ini", tmp_path / "b.ini"
    a.write_text(_ini("iqld"))
    b.write_text(_ini("iqld", lr_init="5e-4", epsilon_init="0.5", epsilon_decay="constant", gamma="0.9",
                      reward_norm="300.0"))
    sw = train_iql_sweep([str(a), str(b)], str(tmp_path / "sweep"), "all_test", n_replicas=64, summaries=True)
    assert sw.names == ["a", "b"] and not sw.model._one_scaling
    for name, path in (("a", a), ("b", b)):
        solo = str(tmp_path / ("solo_" + name) / "iqld")
        train(str(path), solo, "all_test", n_replicas=64, summaries=True)
        d = sweep_dir(str(tmp_path / "sweep"), name, "iqld")
        assert open(os.path.join(d, "data", name + ".ini")).read() == path.read_text()
        _same_dir(d, solo, 120)
    _evaluate_script_equals_post_test(sweep_dir(str(tmp_path / "sweep"), "b", "iqld"), "iqld")
