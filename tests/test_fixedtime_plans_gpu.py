"""GPU: per-replica fixed-time plans (tsc_set_replica_signal_programs) and the plan search (agents/tune_fixedtime.py).

- On the grid, Monaco, the small grid and the mini SUMO net, with 3-5 random plans (durations 1-40 s, random offsets,
  different phase counts) spread unevenly over 8 x SMs + 5 replicas, over more than one cycle of the longest plan,
  every replica equals a tsc_set_signal_program handle running its plan on the same seed: obs, reward, greward, done,
  detector counts, the phase tap and the vehicle state of sampled replicas, through tsc_step, tsc_step_record (per-
  second statistics and trips) and two tsc_step_host_range calls.  A few replicas equal the oracle's fixed mode
  (tests/fixedtime_ref.c) running their plan, and tsc_get_program_phase equals phase_at of each replica's plan.
- Per-replica plans with per-replica demand at two levels.
- Switching: per-replica plans -> one program, -> NULL (action-driven), and an actuated program turning them off.
- The search on a short grid episode: the scores of the best and two other candidates equal the mean_reward
  scripts/evaluate.py reports for a fixedtime directory running that plan, generation 0's incumbent equals the plain
  fixedtime directory's, the incumbent never gets worse, two runs write the same bytes, the output directory evaluates
  alike through evaluate.py and evaluate_agents.py, and --generations 0 reproduces the plain fixedtime outputs.  The
  first equality once on Monaco.
"""
import configparser
import json
import os
import shutil

import numpy as np
import pytest
import torch

from tests.test_fixedtime_gpu import _case, _program, _record_step
from tests.test_fixedtime_plans_cpu import _random_plan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _np(t):
    return t.cpu().numpy()


def _plans(net, programs, n, seed):
    rng = np.random.default_rng(seed)
    out = [_program(net, _random_plan(rng, programs)) for _ in range(n)]
    assert len({tuple(p.n_phases) for p in out}) > 1                # different phase counts
    return out


def _uneven(R, n, seed):
    w = np.arange(1, n + 1, dtype=np.float64) ** 2
    plan = np.random.default_rng(seed).choice(n, R, p=w / w.sum())
    assert len(np.unique(plan)) == n
    return plan


class _Step:
    """one handle's step outputs through the device API"""

    def __init__(self, sim, R, N, n_obs):
        from deeprl_signal_control_b200 import _lib
        self.sim, self.lib, self.st = sim, _lib.lib(), torch.cuda.current_stream().cuda_stream
        self.obs = torch.zeros(R, n_obs, device="cuda"); self.rew = torch.zeros(R, N, device="cuda")
        self.grw = torch.zeros(R, device="cuda"); self.done = torch.zeros(R, dtype=torch.uint8, device="cuda")

    def step(self):
        from deeprl_signal_control_b200 import _lib
        _lib.check(self.lib.tsc_step(self.sim._h, None, None, self.obs.data_ptr(), self.rew.data_ptr(),
                                     self.grw.data_ptr(), self.done.data_ptr(), self.st))
        return tuple(_np(x) for x in (self.obs, self.rew, self.grw, self.done))

    def host(self, R, n_obs, N):
        """two host ranges that cover the handle"""
        out = (np.zeros((R, n_obs), np.float32), np.zeros((R, N), np.float32), np.zeros(R, np.float32),
               np.zeros(R, np.uint8))
        k = R // 3
        for r0, n in ((0, k), (k, R - k)):
            self.sim.step_host_range(r0, n, None, None, *(x[r0:r0 + n] for x in out))
        return out


@pytest.mark.parametrize("scenario", ["grid", "monaco", "small", "mini_sumo"])
def test_replica_plans_equal_one_program_handles(scenario, tmp_path):
    from deeprl_signal_control_b200.envs.fixedtime import phase_at
    from deeprl_signal_control_b200.sim import BatchedSim
    from tests.fixedtime_ref import FixedRefSim
    net, par, programs = _case(scenario, tmp_path)
    n_plans = {"grid": 3, "monaco": 4, "small": 5, "mini_sumo": 4}[scenario]
    plans = _plans(net, programs, n_plans, 7 + n_plans)
    ci, N = par.control_interval_sec, net.n_nodes
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    R = n_sm * 8 + 5
    plan_of = _uneven(R, n_plans, 3)
    n_steps = int(max(p.cycle.max() for p in plans)) // ci + 3
    seeds = np.arange(R, dtype=np.uint64) * np.uint64(5) + np.uint64(77)
    sim, rec = BatchedSim(net, par, R), BatchedSim(net, par, R)
    one = [BatchedSim(net, par, R) for _ in plans]
    one_rec = [BatchedSim(net, par, R) for _ in plans]
    oracle = [int(np.flatnonzero(plan_of == p)[-1]) for p in range(n_plans)][:3]
    refs = [FixedRefSim(net, par, 1) for _ in oracle]
    for s in [sim, rec] + one + one_rec:
        s.reset(seeds); s.set_train_mode(False)
    for s in [rec] + one_rec:
        s.set_record(True)
    for j, r in enumerate(oracle):
        refs[j].reset(seeds[[r]]); refs[j].set_train_mode(False)
    sim.set_replica_signal_programs(plans, plan_of)
    rec.set_replica_signal_programs(plans, plan_of)
    for p, (a, b) in enumerate(zip(one, one_rec)):
        a.set_signal_program(plans[p]); b.set_signal_program(plans[p])
    steps = [_Step(s, R, N, net.n_obs) for s in [sim] + one]
    rows = [np.flatnonzero(plan_of == p) for p in range(n_plans)]
    check = sorted({0, R // 2, R - 1} | set(oracle))
    host_step = n_steps // 2
    for t in range(n_steps):
        want_phase = np.stack([phase_at(plans[p], t * ci) for p in plan_of])
        np.testing.assert_array_equal(_np(sim.program_phase()), want_phase)
        if t == host_step:
            got = steps[0].host(R, net.n_obs, N)
            want = [s.host(R, net.n_obs, N) for s in steps[1:]]
        else:
            got = steps[0].step()
            want = [s.step() for s in steps[1:]]
        for p in range(n_plans):
            for x, y in zip(want[p], got):
                np.testing.assert_array_equal(x[rows[p]], y[rows[p]])
        cg = [_np(x) for x in sim.counts()]
        cw = [[_np(x) for x in s.counts()] for s in one]
        for p in range(n_plans):
            for x, y in zip(cw[p], cg):
                np.testing.assert_array_equal(x[rows[p]], y[rows[p]])
        np.testing.assert_array_equal(cg[3], np.stack([phase_at(plans[p], t * ci) for p in plan_of]))
        for j, r in enumerate(oracle):
            wo = refs[j].step_fixed(plans[plan_of[r]])
            for x, y in zip(wo[:4], got):
                np.testing.assert_array_equal(x[0], y[r])
            np.testing.assert_array_equal(wo[4][0], cg[3][r])
        gr = _record_step(rec, steps[0].lib, steps[0].st, R, N, net.n_obs, ci)
        for p in range(n_plans):
            wr = _record_step(one_rec[p], steps[0].lib, steps[0].st, R, N, net.n_obs, ci)
            for x, y in zip(wr, gr):
                np.testing.assert_array_equal(x[rows[p]], y[rows[p]])
        if t in (host_step, n_steps - 1):
            for r in check:
                for x, y in zip(one[plan_of[r]].dump_state(r), sim.dump_state(r)):
                    np.testing.assert_array_equal(x, y)
                for x, y in zip(one_rec[plan_of[r]].dump_state(r), rec.dump_state(r)):
                    np.testing.assert_array_equal(x, y)
            for j, r in enumerate(oracle):
                for x, y in zip(refs[j].dump_state(0), sim.dump_state(r)):
                    np.testing.assert_array_equal(x, y)
    key = lambda a: a[np.lexsort(a.T[::-1])]
    for r in check:
        np.testing.assert_array_equal(key(one_rec[plan_of[r]].trips(r)), key(rec.trips(r)))
    assert sum(len(rec.trips(r)) for r in check) > 0


def test_replica_plans_with_replica_demand(tmp_path):
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.sim import BatchedSim
    net, par, programs = _case("grid", tmp_path)
    levels = [net, build_large_grid(agent="fixedtime", peak_flow1=1400, peak_flow2=1180)]
    plans = _plans(net, programs, 3, 21)
    R, N = 300, net.n_nodes
    plan_of, level_of = _uneven(R, 3, 4), np.arange(R) % 2
    seeds = np.arange(R, dtype=np.uint64) + np.uint64(40)
    sim = BatchedSim(net, par, R)
    one = [BatchedSim(net, par, R) for _ in plans]
    for p, s in enumerate([sim] + one):
        s.reset(seeds)
        s.set_replica_demand(levels, level_of)
        if p == 0:
            s.set_replica_signal_programs(plans, plan_of)
        else:
            s.set_signal_program(plans[p - 1])
    steps = [_Step(s, R, N, net.n_obs) for s in [sim] + one]
    for t in range(40):
        got = steps[0].step()
        for p in range(3):
            want, rows = steps[p + 1].step(), plan_of == p
            for x, y in zip(want, got):
                np.testing.assert_array_equal(x[rows], y[rows])
    for r in (0, 1, R - 2, R - 1):
        for x, y in zip(one[plan_of[r]].dump_state(r), sim.dump_state(r)):
            np.testing.assert_array_equal(x, y)


def test_switching_modes(tmp_path):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.envs.actuated import actuated_tables
    from deeprl_signal_control_b200.sim import BatchedSim
    net, par, programs = _case("grid", tmp_path)
    plans = _plans(net, programs, 3, 5)
    R, N = 256, net.n_nodes
    plan_of = _uneven(R, 3, 8)
    seeds = np.arange(R, dtype=np.uint64) + np.uint64(3)
    dummy = torch.zeros(R, N, dtype=torch.int32, device="cuda")

    def same(a, b, steps, act=None):
        for _ in range(steps):
            x = act() if act else dummy
            want = [v.clone() for v in a.step(x)]
            for v, w in zip(want, b.step(x)):
                assert torch.equal(v, w)
            for v, w in zip(a.counts(), b.counts()):
                assert torch.equal(v, w)

    a, b = BatchedSim(net, par, R), BatchedSim(net, par, R)
    # per-replica plans, then one program: the one-program run
    b.reset(seeds); b.set_replica_signal_programs(plans, plan_of)
    for _ in range(4):
        b.step(dummy)
    a.reset(seeds); b.reset(seeds)                               # the setting persists over the reset
    a.set_signal_program(plans[1])
    b.set_signal_program(plans[1])
    same(a, b, 25)
    # ... and back to per-replica plans after a reset, which persist over the next reset
    b.set_replica_signal_programs(plans, plan_of)
    b.reset(seeds)
    assert torch.equal(b.program_phase(), _phases0(plans, plan_of))
    # NULL: action-driven stepping
    a.reset(seeds); a.set_signal_program(None)
    b.set_replica_signal_programs(None)
    g = torch.Generator(device="cuda").manual_seed(4)
    same(a, b, 20, lambda: torch.randint(0, 5, (R, N), device="cuda", generator=g, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="tsc_get_program_phase: no signal program is set"):
        b.program_phase()
    # an actuated program turns the plans off
    ap = actuated_tables(net, programs)
    a.reset(seeds); b.reset(seeds)
    b.set_replica_signal_programs(plans, plan_of)
    a.set_actuated_program(ap); b.set_actuated_program(ap)
    same(a, b, 25)
    b.set_actuated_program(None)
    with pytest.raises(RuntimeError, match="tsc_step: bad argument"):
        _lib.check(_lib.lib().tsc_step(b._h, None, None, None, None, None, None, None))
    # refusals name the plan and leave the setting as it was
    b.reset(seeds); b.set_replica_signal_programs(plans, plan_of)
    bad = _program(net, _random_plan(np.random.default_rng(1), programs))
    bad.dur[2, 0] = 0
    with pytest.raises(RuntimeError, match="tsc_set_replica_signal_programs: plan 1: node 2: phase 0 lasts less than 1 s"):
        b.set_replica_signal_programs([plans[0], bad], np.zeros(R, np.int64))
    bad_plan = plan_of.astype(np.int32).copy()
    bad_plan[7] = 3
    n = np.stack([p.n_phases for p in plans]).astype(np.int32)
    P = max(p.max_phases for p in plans)
    pad = lambda x: np.ascontiguousarray(np.stack([np.pad(getattr(p, x), ((0, 0), (0, P - p.max_phases)))
                                                   for p in plans]))
    tabs = [pad("dur").astype(np.int32), pad("open").astype(np.uint32), pad("major").astype(np.uint32),
            pad("yellow").astype(np.uint32), np.ascontiguousarray(np.stack([p.offset for p in plans]).astype(np.int32))]
    with pytest.raises(RuntimeError, match=r"replica 7 has plan index 3, outside \[0, 3\)"):
        _lib.check(_lib.lib().tsc_set_replica_signal_programs(b._h, 3, P, n.ctypes.data, *(x.ctypes.data for x in tabs),
                                                              bad_plan.ctypes.data))
    np.testing.assert_array_equal(_np(b.program_phase()), _np(_phases0(plans, plan_of)))


def _phases0(plans, plan_of):
    from deeprl_signal_control_b200.envs.fixedtime import phase_at
    return torch.from_numpy(np.stack([phase_at(plans[p], 0) for p in plan_of]).astype(np.int32)).cuda()


# ---- the search -----------------------------------------------------------------------------------------------------
SEEDS = [1001, 1002]


def _config(tmp_path, scenario, sec):
    from tests.test_evaluator_gpu import GRID_INI, REAL_INI
    ini = (GRID_INI if scenario == "large_grid" else REAL_INI) % ("greedy", sec, "10000,20000")
    c = configparser.ConfigParser()
    c.read_string(ini)
    path = str(tmp_path / ("config_greedy_%s.ini" % scenario))
    with open(path, "w") as f:
        c.write(f)
    return path


def _evaluate(agent_dir, out):
    """scripts/evaluate.py on the tuning seeds: its summary and output files"""
    from tests.test_demand_gpu import _outputs
    from tests.test_pressure_cpu import _script
    s = _script("evaluate").main(["--agent-dir", agent_dir, "--evaluation-seeds", ",".join(map(str, SEEDS)),
                                  "--output-dir", out])
    return s, _outputs(out)


def _plan_dir(tmp_path, name, config, programs=None):
    """a fixedtime directory of `config`, running `programs` ({id: program}) through its tll_file when given"""
    from deeprl_signal_control_b200.envs.fixedtime import write_tll
    d = str(tmp_path / name / "fixedtime")
    os.makedirs(os.path.join(d, "data"))
    c = configparser.ConfigParser()
    c.read(config)
    if programs is not None:
        c["ENV_CONFIG"]["tll_file"] = write_tll(programs, os.path.join(d, "data", "plan.tll.xml"))
    with open(os.path.join(d, "data", os.path.basename(config)), "w") as f:
        c.write(f)
    return d


def _files(d):
    return {f: open(os.path.join(d, "data", f), "rb").read() for f in ("tuned.tll.xml", "tune_log.csv", "tune.json")}


def test_search_scores_are_the_evaluators(tmp_path):
    from deeprl_signal_control_b200.agents.tune_fixedtime import search_space, written_programs
    from deeprl_signal_control_b200.agents.tune_fixedtime import tune_fixedtime
    from deeprl_signal_control_b200.envs import make_env
    from deeprl_signal_control_b200.envs.fixedtime import env_program
    from tests.test_demand_gpu import _outputs, _run
    from tests.test_pressure_gpu import _same_outputs
    cfg = _config(tmp_path, "large_grid", 600)
    kw = dict(candidates=16, generations=2, elite_frac=0.25, rng_seed=3)
    res = tune_fixedtime(cfg, str(tmp_path / "t1"), SEEDS, **kw)
    res2 = tune_fixedtime(cfg, str(tmp_path / "t2"), SEEDS, **kw)
    assert _files(res["dir"]) == _files(res2["dir"])
    log = open(os.path.join(res["dir"], "data", "tune_log.csv")).read().splitlines()
    assert len(log) == 3 and log[0].split(",")[:2] == ["generation", "incumbent_reward"]
    inc = [float(r.split(",")[1]) for r in log[1:]]
    assert inc[0] <= inc[1] == res["best_score"]
    assert res["scores"][1][0] == inc[0]
    # the scores are what scripts/evaluate.py reports for directories running those plans
    c = configparser.ConfigParser(); c.read(cfg)
    c["ENV_CONFIG"]["test_seeds"] = ",".join(map(str, SEEDS))
    env = make_env(c["ENV_CONFIG"], len(SEEDS), str(tmp_path) + os.sep, is_record=False)
    space = search_space(env_program(env), 5, 60)
    plain, plain_out = _evaluate(_plan_dir(tmp_path, "plain", cfg), str(tmp_path / "plain_out"))
    assert res["scores"][0][0] == res["shipped_score"] == plain["mean_reward"]
    g = int(np.argmax([s.max() for s in res["scores"]]))
    k_best = int(np.argmax(res["scores"][g]))
    picks = [(g, k_best), (0, 5), (1, 11)]
    for gi, k in picks:
        prog = space.program(res["greens"][gi][k], res["offsets"][gi][k])
        d = _plan_dir(tmp_path, "c%d_%d" % (gi, k), cfg, written_programs(env, prog))
        s, _ = _evaluate(d, str(tmp_path / ("c%d_%d_out" % (gi, k))))
        assert s["mean_reward"] == res["scores"][gi][k], (gi, k)
    assert res["scores"][g][k_best] == res["best_score"]
    assert len({float(res["scores"][gi][k]) for gi, k in picks}) > 1
    # the tuned directory evaluates alike through both scripts
    s, tuned_out = _evaluate(res["dir"], str(tmp_path / "tuned_out"))
    assert s["mean_reward"] == res["best_score"]
    _run("evaluate_agents.py", "--base-dir", str(tmp_path), "--agents", "t1/fixedtime", "--evaluation-seeds",
         ",".join(map(str, SEEDS)))
    got = _outputs(os.path.join(str(tmp_path), "eva_data", "t1"))
    _same_outputs(got, tuned_out, "tuned")
    # --generations 0 writes the shipped plan: the plain fixedtime outputs, byte for byte
    _run("tune_fixedtime.py", "--base-dir", str(tmp_path / "g0"), "--config-dir", cfg, "--seeds",
         ",".join(map(str, SEEDS)), "--candidates", "4", "--generations", "0")
    info = json.load(open(str(tmp_path / "g0" / "fixedtime" / "data" / "tune.json")))
    assert info["shipped_score"] == info["final_score"] == plain["mean_reward"]
    _, g0_out = _evaluate(str(tmp_path / "g0" / "fixedtime"), str(tmp_path / "g0_out"))
    _same_outputs(g0_out, plain_out, "generations 0")


def test_search_score_is_the_evaluators_on_monaco(tmp_path):
    from deeprl_signal_control_b200.agents.tune_fixedtime import tune_fixedtime
    cfg = _config(tmp_path, "real_net", 300)
    res = tune_fixedtime(cfg, str(tmp_path / "t"), SEEDS, candidates=8, generations=1, elite_frac=0.25, rng_seed=1)
    s, _ = _evaluate(res["dir"], str(tmp_path / "out"))
    assert s["mean_reward"] == res["best_score"]
    assert os.path.exists(os.path.join(res["dir"], "data", "config_greedy_real_net.ini"))
    shutil.rmtree(res["dir"])
