"""GPU: fixed-time signal control on the device (the FIXED instantiations of tsc_step_kernel, tsc_set_signal_program)
and in the evaluators.

- CUDA equals the oracle's fixed mode (tests/fixedtime_ref.c) bit for bit on the grid, Monaco, the small grid and the
  mini SUMO net, over more than one whole cycle: obs, reward, greward, done, detector counts and full per-vehicle
  state, at a replica count above one wave of resident CTAs, the oracle following replicas spread over the waves.
  tsc_step, tsc_step_record (with its per-second statistics and trips) and tsc_step_host_range (two ranges covering
  the handle) are covered, all with action = NULL; the phase tap equals phase_at at every control step.
- On the device, a program reproducing a random action sequence equals the action-driven tsc_step.
- Turning the program off after a reset returns the handle to action-driven stepping.
- `Evaluator` with the fixed-time controller equals the one-replica controller loop on the grid and Monaco.
- A `scripts/evaluate_agents.py` fixedtime entry, alone and at two `--demand` levels, writes what `scripts/evaluate.py`
  writes for its directory.
"""
import configparser
import glob
import json
import os
import shutil

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(scenario, tmp_path):
    """(net, params, programs) of one scenario"""
    from deeprl_signal_control_b200.net.tables import EnvParams
    if scenario == "grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid, tls_programs
        return build_large_grid(agent="fixedtime"), EnvParams(agent="fixedtime"), tls_programs()
    if scenario == "monaco":
        from deeprl_signal_control_b200.envs.fixedtime import _MONACO_CACHE
        from deeprl_signal_control_b200.net.real_net import real_net_tables
        from tests.test_real_net_cpu import real_params
        return real_net_tables("fixedtime"), real_params("fixedtime"), json.load(open(_MONACO_CACHE))
    if scenario == "small":
        from deeprl_signal_control_b200.net.small_grid import build_small_grid, tls_programs
        return build_small_grid(agent="fixedtime"), EnvParams(agent="fixedtime"), tls_programs()
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests", "fixtures"))
    import make_mini_sumo
    from deeprl_signal_control_b200.net.sumo_ingest import read_signal_programs
    from tests.test_evaluator_cpu import _mini_sumo
    net = _mini_sumo(tmp_path)[1]
    net_file, _ = make_mini_sumo.write(str(tmp_path))
    return net, EnvParams(agent="fixedtime", episode_length_sec=900), read_signal_programs(net_file)


def _program(net, programs):
    from deeprl_signal_control_b200.envs.fixedtime import program_tables
    return program_tables(net.node_names, [len(net.phases[n][0]) for n in net.node_names], programs)


def _np(t):
    return t.cpu().numpy()


@pytest.mark.parametrize("scenario", ["grid", "monaco", "small", "mini_sumo"])
def test_cuda_equals_oracle_fixed_mode(scenario, tmp_path):
    from deeprl_signal_control_b200.envs.fixedtime import phase_at
    from deeprl_signal_control_b200.sim import BatchedSim
    from tests.fixedtime_ref import FixedRefSim
    net, par, programs = _case(scenario, tmp_path)
    prog = _program(net, programs)
    ci, N = par.control_interval_sec, net.n_nodes
    n_steps = int(prog.cycle.max()) // ci + 3                     # a whole cycle and more
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    R = n_sm * 8 + 5                                              # more CTAs than one wave (<= 8 resident per SM)
    check = sorted({0, 1, n_sm - 1, n_sm, 5 * n_sm + 3, R // 2, R - 2, R - 1})
    seeds = np.arange(R, dtype=np.uint64) * np.uint64(3) + np.uint64(101)
    sim, rec = BatchedSim(net, par, R), BatchedSim(net, par, R)
    ref, ref_rec = FixedRefSim(net, par, len(check)), FixedRefSim(net, par, len(check))
    for s in (sim, rec, ref, ref_rec):
        s.reset(seeds if s in (sim, rec) else seeds[check])
        s.set_train_mode(False)
    rec.set_record(True); ref_rec.set_record(True)
    sim.set_signal_program(prog); rec.set_signal_program(prog)
    from deeprl_signal_control_b200 import _lib
    lib, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    obs = torch.zeros(R, net.n_obs, device="cuda"); rew = torch.zeros(R, N, device="cuda")
    grw = torch.zeros(R, device="cuda"); done = torch.zeros(R, dtype=torch.uint8, device="cuda")
    h_obs, h_rew = np.zeros((R, net.n_obs), np.float32), np.zeros((R, N), np.float32)
    h_grw, h_done = np.zeros(R, np.float32), np.zeros(R, np.uint8)
    host_step = n_steps // 2
    loaded = 0
    for t in range(n_steps):
        want = ref.step_fixed(prog)
        if t == host_step:                                        # two host ranges that cover the handle
            k = R // 3
            for r0, n in ((0, k), (k, R - k)):
                sim.step_host_range(r0, n, None, None, h_obs[r0:r0 + n], h_rew[r0:r0 + n], h_grw[r0:r0 + n],
                                    h_done[r0:r0 + n])
            got = (h_obs, h_rew, h_grw, h_done)
        else:
            _lib.check(lib.tsc_step(sim._h, None, None, obs.data_ptr(), rew.data_ptr(), grw.data_ptr(),
                                    done.data_ptr(), st))
            got = tuple(_np(x) for x in (obs, rew, grw, done))
        for x, y in zip(want[:4], got):
            np.testing.assert_array_equal(x, y[check])
        veh, halt, wait, phase = (_np(x) for x in sim.counts())
        wv, wh, ww, wp = ref.counts()
        for x, y in ((wv, veh), (wh, halt), (ww, wait)):
            np.testing.assert_array_equal(x, y[check])
        np.testing.assert_array_equal(phase, np.repeat(phase_at(prog, t * ci)[None], R, axis=0))
        np.testing.assert_array_equal(want[4], phase[check])
        # record mode: same step, per-second statistics, and the trips at the end
        wr = ref_rec.step_fixed(prog, record=True)
        for x, y in zip(wr[:4] + (wr[5],), _record_step(rec, lib, st, R, N, net.n_obs, ci)):
            np.testing.assert_array_equal(x, y[check])
        if t in (host_step, n_steps - 1):
            for j, r in enumerate(check):
                for x, y in zip(ref.dump_state(j), sim.dump_state(r)):
                    np.testing.assert_array_equal(x, y)
                for x, y in zip(ref_rec.dump_state(j), rec.dump_state(r)):
                    np.testing.assert_array_equal(x, y)
                loaded += int(sim.dump_state(r)[0].sum() > 0)
    # trips: the same rows; arrivals within one second enter the device log in thread order
    rows = lambda a: a[np.lexsort(a.T[::-1])]
    for j, r in enumerate(check):
        np.testing.assert_array_equal(rows(ref_rec.trips(j)), rows(rec.trips(r)))
    assert loaded >= len(check)


def _record_step(sim, lib, st, R, N, n_obs, ci):
    from deeprl_signal_control_b200 import _lib
    obs = torch.zeros(R, n_obs, device="cuda"); rew = torch.zeros(R, N, device="cuda")
    grw = torch.zeros(R, device="cuda"); done = torch.zeros(R, dtype=torch.uint8, device="cuda")
    stats = torch.zeros(R, ci, 8, device="cuda")
    _lib.check(lib.tsc_step_record(sim._h, None, None, obs.data_ptr(), rew.data_ptr(), grw.data_ptr(), done.data_ptr(),
                                   stats.data_ptr(), st))
    return tuple(_np(x) for x in (obs, rew, grw, done, stats))


def test_reproducing_program_equals_the_action_path_on_the_device(tmp_path):
    from deeprl_signal_control_b200.envs.fixedtime import env_program
    from deeprl_signal_control_b200.sim import BatchedSim
    from tests.test_fixedtime_cpu import _grid_env, _write, reproducing_tll
    T, R = 30, 300
    plain = _grid_env(tmp_path)
    actions = np.random.default_rng(21).integers(0, 5, (T, len(plain.node_names)), dtype=np.int32)
    env = _grid_env(tmp_path, _write(str(tmp_path / "plan.tll.xml"), reproducing_tll(plain, actions)))
    net, par = env._tables, env._params
    a, b = BatchedSim(net, par, R), BatchedSim(net, par, R)
    seeds = np.arange(R, dtype=np.uint64) + np.uint64(9)
    a.reset(seeds); b.reset(seeds)
    b.set_signal_program(env_program(env))
    dummy = torch.full((R, net.n_nodes), 7, dtype=torch.int32, device="cuda")   # not read in fixed mode
    for t in range(T):
        want = [x.clone() for x in a.step(torch.from_numpy(np.repeat(actions[t][None], R, 0)).cuda())]
        got = b.step(dummy)
        for x, y in zip(want, got):
            assert torch.equal(x, y), t
        for x, y in zip(a.counts()[:3], b.counts()[:3]):
            assert torch.equal(x, y)
    for r in (0, R // 2, R - 1):
        for x, y in zip(a.dump_state(r), b.dump_state(r)):
            np.testing.assert_array_equal(x, y)
    assert a.mean_live() > 0


def test_program_off_returns_to_action_stepping(tmp_path):
    from deeprl_signal_control_b200.net.large_grid import build_large_grid, tls_programs
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    net, par = build_large_grid(agent="fixedtime"), EnvParams(agent="fixedtime")
    R = 64
    a, b = BatchedSim(net, par, R), BatchedSim(net, par, R)
    seeds = np.arange(R, dtype=np.uint64) + np.uint64(5)
    b.reset(seeds)
    b.set_signal_program(_program(net, tls_programs()))
    for _ in range(6):
        b.step(torch.zeros(R, net.n_nodes, dtype=torch.int32, device="cuda"))
    a.reset(seeds); b.reset(seeds)
    b.set_signal_program(None)
    g = torch.Generator(device="cuda").manual_seed(2)
    for _ in range(20):
        act = torch.randint(0, 5, (R, net.n_nodes), device="cuda", generator=g, dtype=torch.int32)
        want = [x.clone() for x in a.step(act)]
        got = b.step(act)
        for x, y in zip(want, got):
            assert torch.equal(x, y)
        for x, y in zip(a.counts(), b.counts()):
            assert torch.equal(x, y)
    with pytest.raises(RuntimeError, match="tsc_step: bad argument"):
        from deeprl_signal_control_b200 import _lib
        _lib.check(_lib.lib().tsc_step(b._h, None, None, None, None, None, None, None))


@pytest.mark.parametrize("scenario", ["large_grid", "real_net"])
def test_evaluator_matches_the_one_replica_controller(scenario, tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    from deeprl_signal_control_b200.envs import fixedtime_controller
    from tests.test_evaluator_gpu import _env, _read, _reference_run
    seeds, sec = [10000, 20000, 30000, 40000, 50000], 600
    d1, d2 = str(tmp_path / "one") + os.sep, str(tmp_path / "batched") + os.sep
    os.makedirs(d1); os.makedirs(d2)
    env1 = _env(scenario, "fixedtime", seeds, sec, d1, 1)
    envb = _env(scenario, "fixedtime", seeds, sec, d2, len(seeds))
    mean1, std1 = _reference_run(env1, None, fixedtime_controller(env1))
    ev = Evaluator(envb, fixedtime_controller(envb), d2, policy_type="deterministic")
    assert ev.family == "fixedtime"
    meanb, stdb = ev.run()
    np.testing.assert_array_equal(meanb, mean1)
    np.testing.assert_array_equal(stdb, std1)
    base = "%s_fixedtime_" % env1.name
    for kind in ("control", "traffic"):
        assert open(d1 + base + kind + ".csv").read() == open(d2 + base + kind + ".csv").read(), kind
    actions = _read(d2 + base + "control.csv").action.str.split(",", expand=True).astype(int).values
    assert len(np.unique(actions)) > 1
    key = ["episode", "arrival_sec", "depart_sec", "id"]
    t1 = _read(d1 + base + "trip.csv").sort_values(key).reset_index(drop=True)
    tb = _read(d2 + base + "trip.csv").sort_values(key).reset_index(drop=True)
    assert t1.equals(tb) and len(tb) > 0


def test_evaluate_agents_entry_equals_evaluate_script(tmp_path):
    from tests.test_demand_gpu import _outputs, _run
    from tests.test_pressure_gpu import _controller_dir, _same_outputs
    base = str(tmp_path / "B")
    os.makedirs(base)
    for agent in ("greedy", "maxpressure", "fixedtime"):
        _controller_dir(base, agent)
    _run("evaluate_agents.py", "--base-dir", base, "--agents", "greedy,maxpressure,fixedtime", "--evaluation-seeds",
         "10000,20000,30000", "--evaluation-policy-type", "deterministic")
    got = {k: v for k, v in _outputs(os.path.join(base, "eva_data")).items()
           if k.startswith(("large_grid_fixedtime_", "fixedtime_summary"))}
    ref = str(tmp_path / "ref" / "fixedtime")
    shutil.copytree(os.path.join(base, "fixedtime"), ref, ignore=shutil.ignore_patterns("eva_data"))
    _run("evaluate.py", "--agent-dir", ref, "--evaluation-seeds", "10000,20000,30000", "--evaluation-policy-type",
         "deterministic")
    _same_outputs(got, _outputs(os.path.join(ref, "eva_data")), "fixedtime")
    rows = open(os.path.join(base, "eva_data", "summary.csv")).read().splitlines()
    assert [r.split(",")[0] for r in rows] == ["entry", "greedy", "maxpressure", "fixedtime"]
    s = json.loads(got["fixedtime_summary.json"])
    assert s["agent"] == "fixedtime" and s["mean_trips"] > 0


def test_evaluate_agents_at_demand_levels_equals_evaluate_on_edited_configs(tmp_path):
    from tests.test_demand_gpu import _outputs, _run, _write
    from tests.test_pressure_gpu import _controller_dir, _same_outputs
    base = str(tmp_path / "B")
    os.makedirs(base)
    _controller_dir(base, "fixedtime")
    _controller_dir(base, "greedy")
    levels = [{"peak_flow1": "1400", "peak_flow2": "1180"}, {"peak_flow1": "800"}]
    labels = ["peak_flow1-1400_peak_flow2-1180", "peak_flow1-800"]
    _run("evaluate_agents.py", "--base-dir", base, "--agents", "greedy,fixedtime", "--evaluation-seeds", "10000,20000",
         *sum((["--demand", ",".join("%s=%s" % kv for kv in lv.items())] for lv in levels), []))
    outs = []
    for lv, lab in zip(levels, labels):
        ref = str(tmp_path / "ref" / lab / "fixedtime")
        shutil.copytree(os.path.join(base, "fixedtime"), ref, ignore=shutil.ignore_patterns("eva_data"))
        for ini in glob.glob(os.path.join(ref, "data", "*.ini")):
            c = configparser.ConfigParser()
            c.read(ini)
            for k, v in lv.items():
                c["ENV_CONFIG"][k] = v
            _write(ini, c)
        _run("evaluate.py", "--agent-dir", ref, "--evaluation-seeds", "10000,20000")
        got = {k: v for k, v in _outputs(os.path.join(base, "eva_data", lab)).items()
               if k.startswith(("large_grid_fixedtime_", "fixedtime_summary"))}
        _same_outputs(got, _outputs(os.path.join(ref, "eva_data")), lab)
        outs.append(got)
    assert outs[0]["fixedtime_summary.json"] != outs[1]["fixedtime_summary.json"]
