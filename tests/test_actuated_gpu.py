"""GPU: vehicle-actuated signal control on the device (the ACTUATED instantiations of tsc_step_kernel,
tsc_set_actuated_program, tsc_get_program_phase) and in the evaluators.

- CUDA equals the oracle's actuated mode (tests/actuated_ref.c) bit for bit on the grid, Monaco, the small grid and the
  mini SUMO net, over two whole cycles at maximum durations: obs, reward, greward, done, detector counts, the phase
  tap, the actuated state and full per-vehicle state.  One CTA per replica, R = 8 x SMs + 5 (more CTAs than one
  resident wave), per-replica demand at x1, x1.4 and x0.6 (the mini net at x1), tsc_step, tsc_step_record (with its
  per-second statistics and trips), two tsc_step_host_range calls, and a tsc_reset mid-run.
- tsc_get_program_phase before each step equals the phase tap the step leaves.
- On the device, a program of fixed phases equals the fixed-time kernel.
- `Evaluator` with the actuated controller equals the one-replica controller loop on the grid and Monaco.
- A `scripts/evaluate_agents.py` actuated entry, alone and at two `--demand` levels, writes what `scripts/evaluate.py`
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

from tests.test_actuated_cpu import case, with_durations

pytestmark = pytest.mark.gpu


def _levels(scenario, tmp_path):
    """(params, [net at x1, x1.4, x0.6], programs); the mini net has one level"""
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    from deeprl_signal_control_b200.net.small_grid import build_small_grid
    net, par, programs = case(scenario, tmp_path)
    if scenario == "grid":
        return par, [net, build_large_grid(1540, 1295, agent="actuated"), build_large_grid(660, 555, agent="actuated")], \
            programs
    if scenario == "monaco":
        return par, [net, real_net_tables("actuated", flow_rate=455), real_net_tables("actuated", flow_rate=195)], programs
    if scenario == "small":
        return par, [net, build_small_grid(1400, agent="actuated"), build_small_grid(600, agent="actuated")], programs
    return par, [net], programs


def _np(t):
    return t.cpu().numpy()


def _record_step(sim, lib, st, R, N, n_obs, ci):
    from deeprl_signal_control_b200 import _lib
    obs = torch.zeros(R, n_obs, device="cuda"); rew = torch.zeros(R, N, device="cuda")
    grw = torch.zeros(R, device="cuda"); done = torch.zeros(R, dtype=torch.uint8, device="cuda")
    stats = torch.zeros(R, ci, 8, device="cuda")
    _lib.check(lib.tsc_step_record(sim._h, None, None, obs.data_ptr(), rew.data_ptr(), grw.data_ptr(), done.data_ptr(),
                                   stats.data_ptr(), st))
    return tuple(_np(x) for x in (obs, rew, grw, done, stats))


@pytest.mark.parametrize("scenario", ["grid", "monaco", "small", "mini_sumo"])
def test_cuda_equals_oracle_actuated_mode(scenario, tmp_path):
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.envs.actuated import actuated_tables
    from deeprl_signal_control_b200.sim import BatchedSim
    from tests.actuated_ref import ActuatedRefSim
    par, nets, programs = _levels(scenario, tmp_path)
    net = nets[0]
    prog = actuated_tables(net, programs)
    ci, N, K = par.control_interval_sec, net.n_nodes, len(nets)
    cycle = int(max(prog.max_dur[i, :prog.n_phases[i]].sum() for i in range(N)))
    n_steps = 2 * cycle // ci + 3                                   # two whole cycles at maximum durations and more
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    R = n_sm * 8 + 5                                                # more CTAs than one wave (<= 8 resident per SM)
    level_of = np.arange(R) % K
    check = sorted({0, 1, n_sm - 1, n_sm, 5 * n_sm + 3, R // 2, R - 2, R - 1})
    seeds0 = np.arange(R, dtype=np.uint64) * np.uint64(3) + np.uint64(101)
    sim, rec = BatchedSim(net, par, R), BatchedSim(net, par, R)
    if K > 1:
        sim.set_replica_demand(nets, level_of); rec.set_replica_demand(nets, level_of)
    # one oracle per (demand level, mode) over the checked replicas of that level
    rows = [[j for j, r in enumerate(check) if level_of[r] == k] for k in range(K)]
    refs = [ActuatedRefSim(nets[k], par, len(rows[k]), prog) for k in range(K)]
    ref_recs = [ActuatedRefSim(nets[k], par, len(rows[k]), prog) for k in range(K)]
    chk = np.asarray(check)

    def reset(seeds):
        for s in [sim, rec]:
            s.reset(seeds)
            s.set_train_mode(False)
        for k in range(K):
            for s in (refs[k], ref_recs[k]):
                s.reset(seeds[chk[rows[k]]])
                s.set_train_mode(False)

    reset(seeds0)
    rec.set_record(True)
    for s in ref_recs:
        s.set_record(True)
    sim.set_actuated_program(prog); rec.set_actuated_program(prog)
    lib, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    obs = torch.zeros(R, net.n_obs, device="cuda"); rew = torch.zeros(R, N, device="cuda")
    grw = torch.zeros(R, device="cuda"); done = torch.zeros(R, dtype=torch.uint8, device="cuda")
    h_obs, h_rew = np.zeros((R, net.n_obs), np.float32), np.zeros((R, N), np.float32)
    h_grw, h_done = np.zeros(R, np.float32), np.zeros(R, np.uint8)
    host_step, reset_step = n_steps // 3, 2 * n_steps // 3
    loaded = 0

    def merge(outs):
        """the per-level oracle results in `check` order"""
        full = []
        for f in range(len(outs[0])):
            parts = [outs[k][f] for k in range(K)]
            x = np.zeros((len(check),) + parts[0].shape[1:], parts[0].dtype)
            for k in range(K):
                x[rows[k]] = parts[k]
            full.append(x)
        return full

    for t in range(n_steps + 4):
        if t == reset_step:                                       # a reset mid-run restores the initial state
            reset(seeds0 + np.uint64(7))
            rec.set_record(True)                                  # a fresh arrival log on both sides
            for s in ref_recs:
                s.set_record(True)
        before = _np(sim.program_phase())
        want = merge([r.step_actuated() for r in refs])
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
        np.testing.assert_array_equal(want[4], phase[check])
        np.testing.assert_array_equal(before, phase)               # tsc_get_program_phase = the next interval's tap
        wc = merge([r.counts() for r in refs])
        for x, y in zip(wc[:3], (veh, halt, wait)):
            np.testing.assert_array_equal(x, y[check])
        # record mode: same step, per-second statistics, and the trips at the end
        wr = merge([r.step_actuated(record=True) for r in ref_recs])
        grec = _record_step(rec, lib, st, R, N, net.n_obs, ci)
        for x, y in zip(wr[:4] + [wr[5]], grec):
            np.testing.assert_array_equal(x, y[check])
        np.testing.assert_array_equal(wr[4], _np(rec.counts()[3])[check])
        if t in (host_step, reset_step - 1, n_steps + 3):
            for k in range(K):
                for j, jj in enumerate(rows[k]):
                    r = check[jj]
                    for x, y in zip(refs[k].dump_state(j), sim.dump_state(r)):
                        np.testing.assert_array_equal(x, y)
                    for x, y in zip(ref_recs[k].dump_state(j), rec.dump_state(r)):
                        np.testing.assert_array_equal(x, y)
                    loaded += int(sim.dump_state(r)[0].sum() > 0)
            np.testing.assert_array_equal(merge([(r.state,) for r in refs])[0][:, :, 0],
                                          _np(sim.program_phase())[check])
    rows_of = lambda a: a[np.lexsort(a.T[::-1])]
    for k in range(K):
        for j, jj in enumerate(rows[k]):
            np.testing.assert_array_equal(rows_of(ref_recs[k].trips(j)), rows_of(rec.trips(check[jj])))
    assert loaded >= len(check)
    assert (refs[0].gap < 255).any()


def test_fixed_phases_equal_the_fixed_time_kernel(tmp_path):
    from deeprl_signal_control_b200.envs.actuated import actuated_tables, fixed_program
    from deeprl_signal_control_b200.sim import BatchedSim
    for scenario in ("grid", "monaco"):
        net, par, programs = case(scenario, tmp_path)
        p = actuated_tables(net, programs)
        ap = with_durations(p, p.dur, p.dur)
        R = 512
        a, b = BatchedSim(net, par, R), BatchedSim(net, par, R)
        seeds = np.arange(R, dtype=np.uint64) + np.uint64(9)
        a.reset(seeds); b.reset(seeds)
        a.set_signal_program(fixed_program(ap))
        b.set_actuated_program(ap)
        dummy = torch.full((R, net.n_nodes), 7, dtype=torch.int32, device="cuda")     # not read under a program
        for t in range(60):
            assert torch.equal(a.program_phase(), b.program_phase()), (scenario, t)
            want = [x.clone() for x in a.step(dummy)]
            got = b.step(dummy)
            for x, y in zip(want, got):
                assert torch.equal(x, y), (scenario, t)
            for x, y in zip(a.counts(), b.counts()):
                assert torch.equal(x, y), (scenario, t)
        for r in (0, R // 2, R - 1):
            for x, y in zip(a.dump_state(r), b.dump_state(r)):
                np.testing.assert_array_equal(x, y)
        # the two programs exclude each other; NULL turns the actuated one off
        a.set_actuated_program(ap)
        b.set_actuated_program(None)
        from deeprl_signal_control_b200 import _lib
        with pytest.raises(RuntimeError, match="tsc_get_program_phase: no signal program is set"):
            b.program_phase()
        with pytest.raises(RuntimeError, match="tsc_step: bad argument"):
            _lib.check(_lib.lib().tsc_step(b._h, None, None, None, None, None, None, None))


@pytest.mark.parametrize("scenario", ["large_grid", "real_net"])
def test_evaluator_matches_the_one_replica_controller(scenario, tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    from deeprl_signal_control_b200.envs import actuated_controller
    from tests.test_evaluator_gpu import _env, _read, _reference_run
    seeds, sec = [10000, 20000, 30000, 40000, 50000], 600
    d1, d2 = str(tmp_path / "one") + os.sep, str(tmp_path / "batched") + os.sep
    os.makedirs(d1); os.makedirs(d2)
    env1 = _env(scenario, "actuated", seeds, sec, d1, 1)
    envb = _env(scenario, "actuated", seeds, sec, d2, len(seeds))
    mean1, std1 = _reference_run(env1, None, actuated_controller(env1))
    ev = Evaluator(envb, actuated_controller(envb), d2, policy_type="deterministic")
    assert ev.family == "actuated"
    meanb, stdb = ev.run()
    np.testing.assert_array_equal(meanb, mean1)
    np.testing.assert_array_equal(stdb, std1)
    base = "%s_actuated_" % env1.name
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
    for agent in ("greedy", "fixedtime", "actuated"):
        _controller_dir(base, agent)
    _run("evaluate_agents.py", "--base-dir", base, "--agents", "greedy,fixedtime,actuated", "--evaluation-seeds",
         "10000,20000,30000", "--evaluation-policy-type", "deterministic")
    got = {k: v for k, v in _outputs(os.path.join(base, "eva_data")).items()
           if k.startswith(("large_grid_actuated_", "actuated_summary"))}
    ref = str(tmp_path / "ref" / "actuated")
    shutil.copytree(os.path.join(base, "actuated"), ref, ignore=shutil.ignore_patterns("eva_data"))
    _run("evaluate.py", "--agent-dir", ref, "--evaluation-seeds", "10000,20000,30000", "--evaluation-policy-type",
         "deterministic")
    _same_outputs(got, _outputs(os.path.join(ref, "eva_data")), "actuated")
    rows = open(os.path.join(base, "eva_data", "summary.csv")).read().splitlines()
    assert [r.split(",")[0] for r in rows] == ["entry", "greedy", "fixedtime", "actuated"]
    s = json.loads(got["actuated_summary.json"])
    assert s["agent"] == "actuated" and s["mean_trips"] > 0


def test_evaluate_agents_at_demand_levels_equals_evaluate_on_edited_configs(tmp_path):
    from tests.test_demand_gpu import _outputs, _run, _write
    from tests.test_pressure_gpu import _controller_dir, _same_outputs
    base = str(tmp_path / "B")
    os.makedirs(base)
    _controller_dir(base, "actuated")
    _controller_dir(base, "greedy")
    levels = [{"peak_flow1": "1400", "peak_flow2": "1180"}, {"peak_flow1": "800"}]
    labels = ["peak_flow1-1400_peak_flow2-1180", "peak_flow1-800"]
    _run("evaluate_agents.py", "--base-dir", base, "--agents", "greedy,actuated", "--evaluation-seeds", "10000,20000",
         *sum((["--demand", ",".join("%s=%s" % kv for kv in lv.items())] for lv in levels), []))
    outs = []
    for lv, lab in zip(levels, labels):
        ref = str(tmp_path / "ref" / lab / "actuated")
        shutil.copytree(os.path.join(base, "actuated"), ref, ignore=shutil.ignore_patterns("eva_data"))
        for ini in glob.glob(os.path.join(ref, "data", "*.ini")):
            c = configparser.ConfigParser()
            c.read(ini)
            for k, v in lv.items():
                c["ENV_CONFIG"][k] = v
            _write(ini, c)
        _run("evaluate.py", "--agent-dir", ref, "--evaluation-seeds", "10000,20000")
        got = {k: v for k, v in _outputs(os.path.join(base, "eva_data", lab)).items()
               if k.startswith(("large_grid_actuated_", "actuated_summary"))}
        _same_outputs(got, _outputs(os.path.join(ref, "eva_data")), lab)
        outs.append(got)
    assert outs[0]["actuated_summary.json"] != outs[1]["actuated_summary.json"]
