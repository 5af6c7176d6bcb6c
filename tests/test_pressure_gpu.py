"""GPU: the max-pressure controller on the device (tsc_pressure_actions) and in the evaluators.

- The kernel equals the numpy definition (envs/maxpressure.py) exactly, on the lane counts tsc_dump_state reads back:
  straight after reset and after a few dozen random-action control steps, on the grid, Monaco, the small grid and the
  ingested mini SUMO net, at a replica count whose CTAs exceed one full wave of resident CTAs on every SM, for a spread
  of replicas including the first and last of a CTA and the last replica.
- `Evaluator` with the max-pressure controller gives the per-episode (mean, std) and the CSVs of the one-replica env
  driven by `maxpressure_controller(env).forward`, on the grid and Monaco.
- `scripts/evaluate_agents.py --agents greedy,maxpressure,ma2c` writes, for its maxpressure entry, what
  `scripts/evaluate.py` writes for that directory; with `--demand` at two levels, what it writes for copies whose config
  carries each level.
"""
import configparser
import glob
import os
import shutil

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RESIDENT_CTAS = 2048 // 256        # CTAs of 256 threads resident per SM (threads bound)


def _net(scenario, tmp_path):
    from deeprl_signal_control_b200.net.tables import EnvParams
    if scenario == "grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid
        return build_large_grid(agent="maxpressure"), EnvParams(agent="maxpressure")
    if scenario == "monaco":
        from deeprl_signal_control_b200.net.real_net import real_net_tables
        from tests.test_real_net_cpu import real_params
        return real_net_tables("maxpressure"), real_params("maxpressure")
    if scenario == "small":
        from deeprl_signal_control_b200.net.small_grid import build_small_grid
        return build_small_grid(agent="maxpressure"), EnvParams(agent="maxpressure")
    from tests.test_evaluator_cpu import _mini_sumo
    return _mini_sumo(tmp_path)[1], EnvParams(agent="maxpressure", episode_length_sec=900)


@pytest.mark.parametrize("scenario", ["grid", "monaco", "small", "mini_sumo"])
def test_kernel_equals_definition_on_simulated_lane_counts(scenario, tmp_path):
    from deeprl_signal_control_b200.envs.maxpressure import pressure_actions
    from deeprl_signal_control_b200.sim import BatchedSim
    net, par = _net(scenario, tmp_path)
    lpad = (net.n_lanes + 15) // 16 * 16
    per_cta = min(256 // net.n_nodes, 48 * 1024 // lpad)       # replicas per CTA of tsc_pressure_actions
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    R = per_cta * (n_sm * RESIDENT_CTAS + 5)
    sim = BatchedSim(net, par, R)
    sim.reset(np.arange(R, dtype=np.uint64) * np.uint64(5) + np.uint64(77))
    sim.set_train_mode(False)
    rng = np.random.default_rng(3)
    check = sorted(set([0, 1, per_cta - 1, per_cta, 2 * per_cta - 1, R // 2, R - per_cta - 1, R - per_cta, R - 2, R - 1]
                       + rng.integers(0, R, 6).tolist()))
    act = torch.full((R, net.n_nodes), -1, dtype=torch.int32, device="cuda")
    sim.pressure_actions(act)                                    # straight after reset: every lane is empty
    assert not act.any()
    g = torch.Generator(device="cuda").manual_seed(11)
    n_a = [int(a) for a in net.node_n_phases]
    loaded = 0
    for t in range(40):                                          # inside the shortest demand horizon (300 s)
        a = torch.stack([torch.randint(0, na, (R,), device="cuda", generator=g, dtype=torch.int32) for na in n_a], 1)
        sim.step(a.contiguous())
        if t in (19, 39):
            act.fill_(-1)
            sim.pressure_actions(act)
            got = act.cpu().numpy()
            cnt = np.stack([sim.dump_state(r)[0] for r in check])
            np.testing.assert_array_equal(got[check], pressure_actions(net, cnt))
            loaded += int(cnt.any(1).sum())
            assert (got >= 0).all() and (got < np.asarray(n_a)[None]).all()
            # observe leaves the state, and with it the actions, as they were
            sim.observe()
            again = sim.pressure_actions()
            assert torch.equal(again, act)
    assert loaded >= len(check)                                  # the comparison saw loaded networks
    assert len(np.unique(got)) > 1


@pytest.mark.parametrize("scenario", ["large_grid", "real_net"])
def test_evaluator_matches_the_one_replica_controller(scenario, tmp_path):
    from deeprl_signal_control_b200.agents.evaluator import Evaluator
    from deeprl_signal_control_b200.envs import maxpressure_controller
    from tests.test_evaluator_gpu import _env, _read, _reference_run
    seeds, sec = [10000, 20000, 30000, 40000, 50000], 600
    d1, d2 = str(tmp_path / "one") + os.sep, str(tmp_path / "batched") + os.sep
    os.makedirs(d1); os.makedirs(d2)
    env1 = _env(scenario, "maxpressure", seeds, sec, d1, 1)
    envb = _env(scenario, "maxpressure", seeds, sec, d2, len(seeds))
    mean1, std1 = _reference_run(env1, None, maxpressure_controller(env1))
    ev = Evaluator(envb, maxpressure_controller(envb), d2, policy_type="deterministic")
    assert ev.family == "maxpressure"
    meanb, stdb = ev.run()
    np.testing.assert_array_equal(meanb, mean1)
    np.testing.assert_array_equal(stdb, std1)
    base = "%s_maxpressure_" % env1.name
    for kind in ("control", "traffic"):
        assert open(d1 + base + kind + ".csv").read() == open(d2 + base + kind + ".csv").read(), kind
    actions = _read(d2 + base + "control.csv").action.str.split(",", expand=True).astype(int).values
    assert len(np.unique(actions)) > 1                           # the controller switched phases
    # trips: the same rows; the order of arrivals within one second is thread order (test_record_gpu.py)
    key = ["episode", "arrival_sec", "depart_sec", "id"]
    t1 = _read(d1 + base + "trip.csv").sort_values(key).reset_index(drop=True)
    tb = _read(d2 + base + "trip.csv").sort_values(key).reset_index(drop=True)
    assert t1.equals(tb) and len(tb) > 0


def _controller_dir(base, agent, **env):
    from tests.test_demand_gpu import _cfg_text, _write
    d = os.path.join(base, agent)
    os.makedirs(os.path.join(d, "data"))
    _write(os.path.join(d, "data", "config_%s_large.ini" % agent), _cfg_text(agent, **env))
    return d


def _same_outputs(got, want, what):
    from tests.test_demand_gpu import _trip_rows
    assert sorted(got) == sorted(want) and len(want) == 4, (what, sorted(got), sorted(want))
    for k in want:
        if k.endswith("_trip.csv"):
            # vehicles that arrive in the same simulated second enter the arrival log in thread order
            assert _trip_rows(got[k]) == _trip_rows(want[k]), (what, k)
        else:
            assert got[k] == want[k], (what, k)


def test_evaluate_agents_entry_equals_evaluate_script(tmp_path):
    from tests.test_demand_gpu import _outputs, _run, _trained
    base = str(tmp_path / "B")
    os.makedirs(base)
    _controller_dir(base, "greedy")
    _controller_dir(base, "maxpressure")
    _trained(base, "ma2c")
    _run("evaluate_agents.py", "--base-dir", base, "--agents", "greedy,maxpressure,ma2c", "--evaluation-seeds",
         "10000,20000,30000", "--evaluation-policy-type", "deterministic")
    got = {k: v for k, v in _outputs(os.path.join(base, "eva_data")).items()
           if k.startswith(("large_grid_maxpressure_", "maxpressure_summary"))}
    ref = str(tmp_path / "ref" / "maxpressure")
    shutil.copytree(os.path.join(base, "maxpressure"), ref, ignore=shutil.ignore_patterns("eva_data"))
    _run("evaluate.py", "--agent-dir", ref, "--evaluation-seeds", "10000,20000,30000", "--evaluation-policy-type",
         "deterministic")
    _same_outputs(got, _outputs(os.path.join(ref, "eva_data")), "maxpressure")
    rows = open(os.path.join(base, "eva_data", "summary.csv")).read().splitlines()
    assert [r.split(",")[0] for r in rows] == ["entry", "greedy", "maxpressure", "ma2c"]
    import json
    s = json.loads(got["maxpressure_summary.json"])
    assert s["agent"] == "maxpressure" and s["mean_trips"] > 0


def test_evaluate_agents_at_demand_levels_equals_evaluate_on_edited_configs(tmp_path):
    from tests.test_demand_gpu import _outputs, _run, _write
    base = str(tmp_path / "B")
    os.makedirs(base)
    _controller_dir(base, "maxpressure")
    _controller_dir(base, "greedy")
    levels = [{"peak_flow1": "1400", "peak_flow2": "1180"}, {"peak_flow1": "800"}]
    labels = ["peak_flow1-1400_peak_flow2-1180", "peak_flow1-800"]
    _run("evaluate_agents.py", "--base-dir", base, "--agents", "greedy,maxpressure", "--evaluation-seeds", "10000,20000",
         *sum((["--demand", ",".join("%s=%s" % kv for kv in lv.items())] for lv in levels), []))
    outs = []
    for lv, lab in zip(levels, labels):
        ref = str(tmp_path / "ref" / lab / "maxpressure")
        shutil.copytree(os.path.join(base, "maxpressure"), ref, ignore=shutil.ignore_patterns("eva_data"))
        for ini in glob.glob(os.path.join(ref, "data", "*.ini")):
            c = configparser.ConfigParser()
            c.read(ini)
            for k, v in lv.items():
                c["ENV_CONFIG"][k] = v
            _write(ini, c)
        _run("evaluate.py", "--agent-dir", ref, "--evaluation-seeds", "10000,20000")
        got = {k: v for k, v in _outputs(os.path.join(base, "eva_data", lab)).items()
               if k.startswith(("large_grid_maxpressure_", "maxpressure_summary"))}
        _same_outputs(got, _outputs(os.path.join(ref, "eva_data")), lab)
        outs.append(got)
    assert outs[0]["maxpressure_summary.json"] != outs[1]["maxpressure_summary.json"]
