"""GPU: traffic demand per replica (tsc_set_replica_demand, BatchedSim.set_replica_demand) and what is built on it.

- Simulator: grid MA2C, Monaco MA2C and small grid, three demand levels (the configured one, one higher, one lower) on
  3 x 64 replicas.  Every replica is bit-identical to a simulator built with its level's tables: a train-mode episode
  (obs, rewards, done, detector counts, traffic statistics, vehicle state), record mode (per-second statistics, trips)
  and host-range steps with rep0 != 0; on the grid with per-replica coop_gamma as well.  Every replica at the
  configured level equals no setting, and clearing returns to the built tables.
- Sweeps: a deterministic grid MA2C demand sweep and an iqll demand sweep leave each member's solo directory exactly;
  the default A2C demand sweep's first rollout is bit-identical to the solo runs'.
- Evaluation: `scripts/evaluate_agents.py --demand` writes, per (entry, level), what `scripts/evaluate.py` writes for a
  copy of the entry whose config carries the level; `--share-demand` groups a demand sweep into one simulator.
Short episodes and at most 192 simulator replicas keep the file small.
"""
import configparser
import dataclasses
import glob
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RB = 64                                     # replicas per demand level in the simulator tests
pytestmark = pytest.mark.gpu


def _levels(scenario):
    """(params, [net at the configured level, higher, lower]) of a scenario's MA2C simulator"""
    from deeprl_signal_control_b200.net.tables import EnvParams
    if scenario == "large_grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid
        nets = [build_large_grid(a, b, agent="ma2c") for a, b in ((1100, 925), (1400, 1180), (800, 675))]
        par = EnvParams(agent="ma2c")
    elif scenario == "real_net":
        from bench import build_scenario

        class A:
            agent, policy, scenario = "ma2c", "lstm", "real_net"
        from deeprl_signal_control_b200.net.real_net import real_net_tables
        par = build_scenario(A)[1]
        nets = [real_net_tables("ma2c", flow_rate=f) for f in (325, 450, 200)]
    else:
        from deeprl_signal_control_b200.net.small_grid import build_small_grid
        nets = [build_small_grid(n, agent="ma2c") for n in (1000, 1500, 500)]
        par = EnvParams(agent="ma2c", coop_gamma=0.75)
    return dataclasses.replace(par, episode_length_sec=150), nets


def _inputs(sim, g):
    n = sim.net
    act = torch.stack([torch.randint(0, int(na), (sim.R,), device="cuda", generator=g, dtype=torch.int32)
                       for na in n.n_a_ls], 1).contiguous()
    fp = torch.rand(sim.R, n.n_nodes, n.max_na, device="cuda", generator=g).contiguous()
    return act, fp


def _reset(shared, solos, ep):
    seeds = np.arange(shared.R, dtype=np.uint64) * np.uint64(7) + np.uint64(1000 * ep + 12)
    shared.reset(seeds)
    for k, s in enumerate(solos):
        s.reset(seeds[k * RB:(k + 1) * RB])


def _same_block(got, want, k, what):
    rows = slice(k * RB, (k + 1) * RB)
    for name, a, b in zip(("obs", "reward", "greward", "done"), got, want):
        assert torch.equal(torch.as_tensor(a)[rows].cpu(), torch.as_tensor(b).cpu()), (what, k, name)


@pytest.mark.parametrize("scenario", ["large_grid", "real_net", "small_grid"])
def test_per_replica_demand_equals_simulators_built_with_it(scenario):
    from deeprl_signal_control_b200.sim import BatchedSim
    par, nets = _levels(scenario)
    K = len(nets)
    shared = BatchedSim(nets[0], par, K * RB)
    shared.set_replica_demand(nets, np.repeat(np.arange(K), RB))
    solos = [BatchedSim(n, par, RB) for n in nets]
    cg = None
    if scenario == "large_grid":                            # demand and coop_gamma per replica together
        cg = (0.9, 0.75, 0.5)
        shared.set_replica_coop_gamma(np.repeat(np.asarray(cg, np.float32), RB))
        for s, c in zip(solos, cg):
            s.set_replica_coop_gamma(np.full(RB, c, np.float32))
    g = torch.Generator(device="cuda").manual_seed(5)
    steps = int(np.ceil(par.episode_length_sec / par.control_interval_sec))
    # a train-mode episode
    _reset(shared, solos, 0)
    for s in [shared] + solos:
        s.set_train_mode(True)
    for t in range(steps):
        act, fp = _inputs(shared, g)
        got = [x.clone() for x in shared.step(act, fp)]
        for k, s in enumerate(solos):
            rows = slice(k * RB, (k + 1) * RB)
            _same_block(got, s.step(act[rows].contiguous(), fp[rows].contiguous()), k, ("step", t))
    assert bool(got[3].all())
    counts, stats = shared.counts(), shared.traffic_stats()
    live = stats[:, 0].view(K, RB).mean(1).tolist()
    assert len(set(live)) == K, live                       # the levels do run at different demand
    for k, s in enumerate(solos):
        rows = slice(k * RB, (k + 1) * RB)
        for a, b in zip(counts, s.counts()):
            assert torch.equal(a[rows], b), ("counts", k)
        assert torch.equal(stats[rows], s.traffic_stats()), ("stats", k)
        for r in (0, RB - 1):
            for a, b in zip(shared.dump_state(k * RB + r), s.dump_state(r)):
                assert np.array_equal(a, b), ("state", k, r)
    # record mode
    _reset(shared, solos, 1)
    for s in [shared] + solos:
        s.set_record(True)
    for t in range(6):
        act, fp = _inputs(shared, g)
        got = [x.clone() for x in shared.step_record(act, fp)]
        for k, s in enumerate(solos):
            rows = slice(k * RB, (k + 1) * RB)
            want = s.step_record(act[rows].contiguous(), fp[rows].contiguous())
            _same_block(got[:4], want[:4], k, ("record", t))
            assert torch.equal(got[4][rows], want[4]), ("record stats", t, k)
    for k, s in enumerate(solos):
        for r in (0, 17, RB - 1):
            # arrivals of one simulated second enter the log in atomic order: the rows compare as a set
            assert sorted(map(tuple, shared.trips(k * RB + r).tolist())) == sorted(map(tuple, s.trips(r).tolist())), \
                ("trips", k, r)
    for s in [shared] + solos:
        s.set_record(False)
    # host-range steps across the level blocks, synchronous and asynchronous
    _reset(shared, solos, 2)
    R, n = shared.R, shared.net
    pin = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype).pin_memory().numpy()
    out = (pin(R, n.n_obs), pin(R, n.n_nodes), pin(R), pin(R, dtype=torch.uint8))
    for t in range(6):
        act, fp = _inputs(shared, g)
        a_h, f_h = act.cpu().numpy(), fp.cpu().numpy()
        for r0, cnt, sync in ((0, 96, True), (96, R - 96, False)):
            sl = slice(r0, r0 + cnt)
            shared.step_host_range(r0, cnt, a_h[sl], f_h[sl], *(o[sl] for o in out), sync=sync)
        torch.cuda.synchronize()
        for k, s in enumerate(solos):
            rows = slice(k * RB, (k + 1) * RB)
            want = [x.copy() for x in s.step_host(a_h[rows], f_h[rows])]
            _same_block([torch.from_numpy(o) for o in out], [torch.from_numpy(w) for w in want], k, ("host range", t))


@pytest.mark.parametrize("scenario", ["large_grid", "small_grid"])
def test_configured_level_or_cleared_is_the_plain_simulator(scenario):
    from deeprl_signal_control_b200.sim import BatchedSim
    par, nets = _levels(scenario)
    R = 2 * RB
    plain, same, cleared = (BatchedSim(nets[0], par, R) for _ in range(3))
    same.set_replica_demand([nets[0]], np.zeros(R, np.int64))
    cleared.set_replica_demand(nets[1:], np.arange(R) % 2)
    cleared.set_replica_demand(None)
    seeds = np.arange(R, dtype=np.uint64) + np.uint64(40)
    g = torch.Generator(device="cuda").manual_seed(8)
    for s in (plain, same, cleared):
        s.reset(seeds)
        s.set_train_mode(True)
    for t in range(int(np.ceil(par.episode_length_sec / par.control_interval_sec))):
        act, fp = _inputs(plain, g)
        want = [x.clone() for x in plain.step(act, fp)]
        for s in (same, cleared):
            for a, b in zip(s.step(act, fp), want):
                assert torch.equal(a, b), t
    with pytest.raises(ValueError):
        plain.set_replica_demand(nets, np.full(R, 3))
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    if scenario == "large_grid":
        with pytest.raises(ValueError, match="not only in its demand"):
            plain.set_replica_demand([build_large_grid(agent="ma2c", init_density=0.1, seed=3)], np.zeros(R))


# ---- sweeps ------------------------------------------------------------------------------------------------------------
def _cfg_text(agent, **env):
    from tests.test_iql_population_gpu import _ini as iql_ini
    from tests.test_train_driver_gpu import _ini
    text = _ini(agent, 120, 240) if agent in ("ia2c", "ma2c") else iql_ini(agent)
    c = configparser.ConfigParser()
    c.read_string(text)
    for k, v in env.items():
        sec = "MODEL_CONFIG" if k in ("reward_norm",) else "ENV_CONFIG"
        c[sec][k] = str(v)
    return c


def _write(path, c):
    with open(path, "w") as f:
        c.write(f)
    return str(path)


def _exact_a2c_dir(a, b, step):
    from deeprl_signal_control_b200.agents import checkpoint as ck
    from tests.test_deterministic_gpu import _scalars
    from tests.test_population_gpu import _listing
    assert _listing(a) == _listing(b)
    wa, wb = (ck.load_npz(os.path.join(d, "model", "checkpoint-%d.npz" % step))[0] for d in (a, b))
    assert sorted(wa) == sorted(wb)
    for n in wa:
        assert np.array_equal(wa[n], wb[n]), n
    for name in sorted(x for x in os.listdir(os.path.join(a, "data")) if x.endswith(".csv")):
        assert open(os.path.join(a, "data", name), "rb").read() == open(os.path.join(b, "data", name), "rb").read(), name
    assert _scalars(a) == _scalars(b)


def test_deterministic_a2c_demand_sweep_members_equal_their_solo_runs(tmp_path):
    from deeprl_signal_control_b200.agents.train import sweep_dir, train, train_sweep
    paths = [_write(tmp_path / "pf1100.ini", _cfg_text("ma2c")),
             _write(tmp_path / "pf1400.ini", _cfg_text("ma2c", peak_flow1=1400, peak_flow2=1180, reward_norm="3000.0"))]
    sw = train_sweep(paths, str(tmp_path / "sweep"), "all_test", n_replicas=64, summaries=True, deterministic=True,
                     vary_demand=True)
    assert sw.names == ["pf1100", "pf1400"] and sw.final_step == 120
    rewards = []
    for name, path in zip(sw.names, paths):
        solo = str(tmp_path / ("solo_" + name) / "ma2c")
        train(path, solo, "all_test", n_replicas=64, summaries=True, deterministic=True)
        d = sweep_dir(str(tmp_path / "sweep"), name, "ma2c")
        _exact_a2c_dir(d, solo, 120)
        rewards.append(open(os.path.join(d, "data", "train_reward.csv")).read())
    assert rewards[0] != rewards[1]


def test_default_a2c_demand_sweep_first_rollout_equals_the_solo_runs(tmp_path, monkeypatch):
    """The first rollout (every step's global reward, before any update) is bit-identical to each member's solo run."""
    from deeprl_signal_control_b200.agents.train import train, train_sweep
    from deeprl_signal_control_b200.sim import BatchedSim
    rec = []
    step = BatchedSim.step

    def recording_step(self, *a, **k):
        out = step(self, *a, **k)
        rec.append(out[2].clone())
        return out
    monkeypatch.setattr(BatchedSim, "step", recording_step)
    paths = [_write(tmp_path / "a.ini", _cfg_text("ma2c")),
             _write(tmp_path / "b.ini", _cfg_text("ma2c", peak_flow1=1400, peak_flow2=1180, reward_norm="3000.0"))]
    sw = train_sweep(paths, str(tmp_path / "sweep"), "no_test", n_replicas=64, vary_demand=True)
    n_step = sw.model.batched.T
    got = torch.stack(rec[:n_step])
    for k, path in enumerate(paths):
        rec.clear()
        train(path, str(tmp_path / ("solo%d" % k) / "ma2c"), "no_test", n_replicas=64)
        assert torch.equal(got[:, k * 64:(k + 1) * 64], torch.stack(rec[:n_step])), k


def test_iql_demand_sweep_members_equal_their_solo_runs(tmp_path):
    from deeprl_signal_control_b200.agents.train import sweep_dir, train, train_iql_sweep
    from tests.test_iql_population_gpu import _same_dir
    paths = [_write(tmp_path / "a.ini", _cfg_text("iqll")),
             _write(tmp_path / "b.ini", _cfg_text("iqll", peak_flow1=1400, peak_flow2=1180, reward_norm="300.0"))]
    sw = train_iql_sweep(paths, str(tmp_path / "sweep"), "all_test", n_replicas=64, summaries=True, vary_demand=True)
    for name, path in zip(sw.names, paths):
        solo = str(tmp_path / ("solo_" + name) / "iqll")
        train(path, solo, "all_test", n_replicas=64, summaries=True)
        _same_dir(sweep_dir(str(tmp_path / "sweep"), name, "iqll"), solo, 120)


# ---- evaluation --------------------------------------------------------------------------------------------------------
def _outputs(d):
    return {os.path.basename(p): open(p, "rb").read() for p in sorted(glob.glob(os.path.join(d, "*"))) if os.path.isfile(p)}


def _trip_rows(text):
    """the rows of a trip CSV without its index column, sorted, and its header"""
    lines = text.decode().splitlines()
    return lines[0], sorted(line.split(",", 1)[1] for line in lines[1:])


def _run(script, *args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", script)] + list(args), capture_output=True,
                       text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    return r


def _trained(base, agent, **env):
    from deeprl_signal_control_b200.agents.train import train
    path = _write(os.path.join(base, "cfg_%s.ini" % agent), _cfg_text(agent, **env))
    d = os.path.join(base, agent)
    if agent == "greedy":
        os.makedirs(os.path.join(d, "data"))
        shutil.copy(path, os.path.join(d, "data"))
    else:
        train(path, d, "no_test", n_replicas=64)
    return d


def test_evaluate_agents_at_demand_levels_equals_evaluate_on_edited_configs(tmp_path, monkeypatch):
    from deeprl_signal_control_b200.agents import evaluator
    base = str(tmp_path / "B")
    os.makedirs(base)
    for agent in ("greedy", "ma2c", "iqll"):
        _trained(base, agent)
    levels = [{"peak_flow1": "1400", "peak_flow2": "1180"}, {"peak_flow1": "800"}]
    labels = ["peak_flow1-1400_peak_flow2-1180", "peak_flow1-800"]
    n_groups = []
    init = evaluator.GroupEvaluator.__init__

    def count(self, *a, **k):
        init(self, *a, **k)
        n_groups.append([len(g) for g in self.groups])
    monkeypatch.setattr(evaluator.GroupEvaluator, "__init__", count)
    spec = __import__("importlib.util").util.spec_from_file_location("ea", os.path.join(ROOT, "scripts", "evaluate_agents.py"))
    mod = __import__("importlib.util").util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    res = mod.main(["--base-dir", base, "--agents", "greedy,ma2c,iqll", "--evaluation-seeds", "10000,20000"] +
                   sum((["--demand", ",".join("%s=%s" % kv for kv in lv.items())] for lv in levels), []))
    assert n_groups == [[2, 2, 2]]                        # greedy, ma2c and iqll each at both levels, one simulator each
    assert len(res) == 6
    head = open(os.path.join(base, "eva_data", "summary.csv")).readline().strip().split(",")
    assert head[:2] == ["entry", "demand"]
    for agent in ("greedy", "ma2c", "iqll"):
        for lv, lab in zip(levels, labels):
            ref = str(tmp_path / "ref" / lab / agent)
            shutil.copytree(os.path.join(base, agent), ref, ignore=shutil.ignore_patterns("eva_data"))
            for ini in glob.glob(os.path.join(ref, "data", "*.ini")):
                c = configparser.ConfigParser()
                c.read(ini)
                for k, v in lv.items():
                    c["ENV_CONFIG"][k] = v
                _write(ini, c)
            _run("evaluate.py", "--agent-dir", ref, "--evaluation-seeds", "10000,20000")
            got = _outputs(os.path.join(base, "eva_data", lab))
            want = _outputs(os.path.join(ref, "eva_data"))
            mine = {k: v for k, v in got.items() if k.startswith(("large_grid_%s_" % agent, "%s_summary" % agent))}
            assert sorted(mine) == sorted(want) and len(want) == 4, (agent, lab, sorted(got), sorted(want))
            for k in want:
                if k.endswith("_trip.csv"):
                    # the arrival log takes the vehicles that arrive in the same simulated second in the order its
                    # threads reach the log (an atomic counter), so the trip rows compare as a set
                    assert _trip_rows(mine[k]) == _trip_rows(want[k]), (agent, lab, k)
                else:
                    assert mine[k] == want[k], (agent, lab, k)


def test_share_demand_groups_a_demand_sweep_without_changing_outputs(tmp_path):
    base = str(tmp_path / "B")
    for sub, pf in (("pf1100", 1100), ("pf1400", 1400)):
        os.makedirs(os.path.join(base, sub))
        d = os.path.join(base, sub)
        _trained(d, "ma2c", peak_flow1=pf)
    from deeprl_signal_control_b200.agents.evaluator import GroupEvaluator
    ents = [(os.path.join(base, s, "ma2c"), "ma2c", str(tmp_path / ("o_" + s)) + "/") for s in ("pf1100", "pf1400")]
    ge = GroupEvaluator(ents, [10000, 20000], share_demand=True)
    assert len(ge.groups) == 1
    assert len(GroupEvaluator(ents, [10000, 20000]).groups) == 2
    outs = {}
    for flag in ([], ["--share-demand"]):
        shutil.rmtree(os.path.join(base, "eva_data"), ignore_errors=True)
        _run("evaluate_agents.py", "--base-dir", base, "--agents", "pf1100/ma2c,pf1400/ma2c", "--evaluation-seeds",
             "10000,20000", *flag)
        outs[bool(flag)] = {s: _outputs(os.path.join(base, "eva_data", s)) for s in ("pf1100", "pf1400")}
        outs[bool(flag)]["summary"] = open(os.path.join(base, "eva_data", "summary.csv"), "rb").read()
    assert outs[True] == outs[False]
    assert outs[True]["pf1100"] != outs[True]["pf1400"]
    assert json.loads(outs[True]["pf1100"]["ma2c_summary.json"])
