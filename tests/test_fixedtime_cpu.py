"""CPU: fixed-time signal control's host side (envs/fixedtime.py) and its oracle.

- The grid's and the small grid's programs equal what the reference generators write (tests/golden/tls_programs.json);
  the Monaco cache equals a fresh ingest of tests/golden/monaco_sumo/most.net.xml.gz.
- The link masks read the state strings, on the grid, Monaco, the small grid and the mini SUMO net.
- Every refusal names the tlLogic id and the reason.
- `phase_at` on hand-made programs: window edges, a non-zero offset, a cycle longer than the episode.
- On the oracle, the fixed mode (tests/fixedtime_ref.c) running a program that reproduces a random action sequence,
  passed through a `tll_file`, equals the action-driven run bit for bit.
- `entry_model`, the directory checks, the `train` refusal and the command lines of scripts/evaluate.py and
  scripts/evaluate_agents.py.
"""
import configparser
import json
import logging
import os
import sys

import numpy as np
import pytest

from tests.test_evaluate_agents_cpu import _dir, _ge, _labels, no_device  # noqa: F401
from tests.test_evaluator_cpu import GRID_INI
from tests.test_pressure_cpu import _script

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "fixtures"))


def _norm(programs):
    """programs with whole-number attributes as ints (the XML gives strings, the restated data ints)"""
    return {k: {"type": v["type"], "offset": int(float(v["offset"])),
                "phases": [[int(float(d)), s] for d, s in v["phases"]]} for k, v in programs.items()}


def _write(path, text):
    with open(path, "w") as f:
        f.write(text)
    return path


@pytest.mark.parametrize("scenario", ["large_grid", "small_grid"])
def test_grid_programs_are_the_reference_generators(scenario, tmp_path):
    from deeprl_signal_control_b200.net import large_grid, small_grid
    from deeprl_signal_control_b200.net.sumo_ingest import read_signal_programs
    text = json.load(open(os.path.join(ROOT, "tests", "golden", "tls_programs.json")))[scenario]
    got = read_signal_programs(_write(str(tmp_path / "exp.tll.xml"), text))
    mine = (large_grid if scenario == "large_grid" else small_grid).tls_programs()
    assert _norm(got) == _norm(mine)
    assert len(mine) == (25 if scenario == "large_grid" else 6)


def test_monaco_cache_is_a_fresh_ingest():
    from deeprl_signal_control_b200.envs.fixedtime import _MONACO_CACHE
    from deeprl_signal_control_b200.net.sumo_ingest import read_signal_programs
    fresh = read_signal_programs(os.path.join(ROOT, "tests", "golden", "monaco_sumo", "most.net.xml.gz"))
    assert json.load(open(_MONACO_CACHE)) == fresh
    assert len(fresh) == 28 and {p["type"] for p in fresh.values()} == {"static"}
    assert {sum(int(d) for d, _ in p["phases"]) for p in fresh.values()} == {90}


def _nets_and_programs(tmp_path):
    from deeprl_signal_control_b200.net import large_grid, small_grid
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    from deeprl_signal_control_b200.net.sumo_ingest import read_signal_programs
    from deeprl_signal_control_b200.envs.fixedtime import _MONACO_CACHE
    import make_mini_sumo
    from tests.test_evaluator_cpu import _mini_sumo
    net_file, _ = make_mini_sumo.write(str(tmp_path))
    return {"grid": (large_grid.build_large_grid(agent="fixedtime"), large_grid.tls_programs()),
            "monaco": (real_net_tables("fixedtime"), json.load(open(_MONACO_CACHE))),
            "small": (small_grid.build_small_grid(agent="fixedtime"), small_grid.tls_programs()),
            "mini_sumo": (_mini_sumo(tmp_path)[1], read_signal_programs(net_file))}


@pytest.mark.parametrize("scenario", ["grid", "monaco", "small", "mini_sumo"])
def test_masks_read_the_state_strings(scenario, tmp_path):
    from deeprl_signal_control_b200.envs.fixedtime import program_tables
    net, programs = _nets_and_programs(tmp_path)[scenario]
    n_links = [len(net.phases[n][0]) for n in net.node_names]
    p = program_tables(net.node_names, n_links, programs)
    n_yellow = 0
    for i, name in enumerate(net.node_names):
        phases = programs[name]["phases"]
        assert int(p.n_phases[i]) == len(phases) and int(p.offset[i]) == int(float(programs[name]["offset"]))
        for k, (d, state) in enumerate(phases):
            assert int(p.dur[i, k]) == int(float(d))
            o, m, y = (int(x[i, k]) for x in (p.open, p.major, p.yellow))
            back = "".join("y" if (y >> j) & 1 else ("G" if (m >> j) & 1 else "g") if (o >> j) & 1 else "r"
                           for j in range(len(state)))
            assert back == state, (name, k)
            assert o >> len(state) == 0 and y & o == 0 and m & ~o == 0
            n_yellow += y != 0
        assert not p.dur[i, len(phases):].any()
    assert n_yellow > 0


def _one(state="GrGr", dur=10, **kw):
    prog = {"type": "static", "offset": "0", "phases": [[str(dur), state], ["3", "yryr"]]}
    prog.update(kw)
    return prog


def test_refusals_name_the_id_and_the_reason():
    from deeprl_signal_control_b200.envs.fixedtime import program_tables
    ok = program_tables(["a"], [4], {"a": _one()})
    assert ok.n_phases.tolist() == [2] and ok.dur[0].tolist() == [10, 3]
    cases = [({"a": _one(type="actuated")}, "tlLogic 'a': type 'actuated' is not static"),
             ({"a": _one(state="GrOr")}, "tlLogic 'a': state 'GrOr' has the character 'O'"),
             ({"a": _one(state="GruY")}, "has the character 'u'"),
             ({"a": _one(dur="2.5")}, "tlLogic 'a': duration '2.5' is not a whole number"),
             ({"a": _one(dur="x")}, "tlLogic 'a': duration 'x' is not a number"),
             ({"a": _one(dur="0")}, "tlLogic 'a': duration '0' is below 1"),
             ({"a": _one(offset="1.5")}, "tlLogic 'a': offset '1.5' is not a whole number"),
             ({"a": _one(state="GrG")}, "tlLogic 'a': state 'GrG' has 3 links, the node has 4"),
             ({"a": _one(state="G" * 33)}, "has 33 links, more than TSC_MAX_NODE_LINKS = 32"),
             ({}, "tlLogic 'a': the signalised node has no program"),
             ({"a": _one(), "zz": _one()}, "tlLogic 'zz' names no signalised node of the env")]
    for programs, msg in cases:
        with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(".", r"\.")):
            program_tables(["a"], [4], programs)


def test_phase_at_on_hand_made_programs():
    from deeprl_signal_control_b200.envs.fixedtime import phase_at, program_tables
    p = program_tables(["a", "b", "c"], [2, 2, 2], {
        "a": {"type": "static", "offset": 0, "phases": [[30, "Gr"], [3, "yr"], [30, "rG"], [3, "ry"]]},
        "b": {"type": "static", "offset": 7, "phases": [[30, "Gr"], [3, "yr"], [30, "rG"], [3, "ry"]]},
        "c": {"type": "static", "offset": 0, "phases": [[5000, "Gr"], [1, "rG"]]}})
    at = lambda s: phase_at(p, s).tolist()
    assert at(0) == [0, 2, 0] and at(29) == [0, 0, 0] and at(30) == [1, 0, 0] and at(32) == [1, 0, 0]
    assert at(33) == [2, 0, 0] and at(36) == [2, 0, 0] and at(37) == [2, 1, 0] and at(40) == [2, 2, 0]
    assert at(62) == [2, 2, 0] and at(63) == [3, 2, 0] and at(65) == [3, 2, 0] and at(66) == [0, 2, 0]
    assert at(99) == [2, 0, 0] and at(-1) == [3, 2, 1]
    # offset 7 delays every phase by 7 s: second s shows what the undelayed program shows at s - 7
    for s in range(200):
        assert phase_at(p, s)[1] == phase_at(p, (s - 7) % 66)[0]
    assert at(3599) == [at(3599 % 66)[0], at((3599 - 7) % 66)[0], 0] and at(5000)[2] == 1 and at(5001)[2] == 0
    assert phase_at(p, 0).dtype == np.int32


# ---- the fixed mode on the oracle against the action-driven run ----------------------------------------------------
def _node_state(phases, a, p, yellow):
    """node_signal's signal (envs/env.py:128-152) as a state string: action a after p, in a yellow sub-step or not"""
    g1, g0 = phases[a], phases[p]
    out = []
    for j, ch in enumerate(g1):
        sw_red = g0[j] in "Gg" and ch not in "Gg"
        if yellow and p != a and any(x in "Gg" and y not in "Gg" for x, y in zip(g0, g1)):
            out.append("y" if sw_red else ("r" if g0[j] not in "Gg" and ch in "Gg" else ch))
        else:
            out.append(ch)
    return "".join(out)


def reproducing_tll(env, actions):
    """<additional> text of the program that reproduces `actions` [T][N] on `env`: per interval the first
    yellow_interval_sec seconds show node_signal's yellow signal (a phase of its own where it differs from the green
    one), the rest the action's phase string; prev_action starts at 0 (reset)."""
    ci, ys = env.control_interval_sec, env.yellow_interval_sec
    text = "<additional>\n"
    for i, name in enumerate(env.node_names):
        phases = env._tables.phases[name]
        text += '  <tlLogic id="%s" type="static" programID="x" offset="0">\n' % name
        prev = 0
        for a in actions[:, i]:
            y, g = _node_state(phases, int(a), prev, True), _node_state(phases, int(a), prev, False)
            seq = [(ys, y), (ci - ys, g)] if y != g else [(ci, g)]
            for d, st in seq:
                text += '    <phase duration="%d" state="%s"/>\n' % (d, st)
            prev = int(a)
        text += "  </tlLogic>\n"
    return text + "</additional>\n"


def _grid_env(tmp_path, tll=None, agent="fixedtime"):
    from deeprl_signal_control_b200.envs.large_grid_env import LargeGridEnv
    cp = configparser.ConfigParser()
    cp.read_string(GRID_INI.replace("agent = greedy", "agent = %s" % agent)
                   + ("tll_file = %s\n" % tll if tll else ""))
    return LargeGridEnv(cp["ENV_CONFIG"], output_path=str(tmp_path) + os.sep)


def test_oracle_fixed_mode_reproduces_an_action_sequence(tmp_path):
    from deeprl_signal_control_b200.envs.fixedtime import env_program
    from oracle.sim_ref import RefSim
    from tests.fixedtime_ref import FixedRefSim
    T, R = 24, 3
    rng = np.random.default_rng(4)
    plain = _grid_env(tmp_path)
    actions = rng.integers(0, 5, (T, len(plain.node_names)), dtype=np.int32)
    actions[3] = actions[2]                                     # a repeated action: no yellow in that interval
    tll = _write(str(tmp_path / "plan.tll.xml"), reproducing_tll(plain, actions))
    env = _grid_env(tmp_path, tll)
    program = env_program(env)
    assert (program.cycle == T * env.control_interval_sec).all() and program.yellow.any()
    net, par = env._tables, env._params
    a, b = RefSim(net, par, R), FixedRefSim(net, par, R)
    seeds = np.arange(R, dtype=np.uint64) + np.uint64(31)
    a.reset(seeds); b.reset(seeds)
    a.set_train_mode(False); b.set_train_mode(False)
    for t in range(T):
        want = a.step(np.repeat(actions[t][None], R, axis=0))
        got = b.step_fixed(program)
        for x, y in zip(want, got[:4]):
            np.testing.assert_array_equal(x, y)
        wc, gc = a.counts(), b.counts()
        for x, y in zip(wc[:3], gc[:3]):
            np.testing.assert_array_equal(x, y)
        assert not gc[3].any()                                 # prev_action is left as reset set it
        np.testing.assert_array_equal(got[4], phase_index(program, t * env.control_interval_sec, R))
        for r in range(R):
            for x, y in zip(a.dump_state(r), b.dump_state(r)):
                np.testing.assert_array_equal(x, y)
    assert a.misc(0)["live"] > 0


def phase_index(program, sec, R):
    from deeprl_signal_control_b200.envs.fixedtime import phase_at
    return np.repeat(phase_at(program, sec)[None], R, axis=0)


def test_oracle_fixed_mode_records_as_the_action_path(tmp_path):
    """record mode: per-second statistics and trips of the fixed mode equal the action-driven step_record's"""
    from deeprl_signal_control_b200.envs.fixedtime import env_program
    from oracle.sim_ref import RefSim
    from tests.fixedtime_ref import FixedRefSim
    T, R = 50, 2
    plain = _grid_env(tmp_path)
    actions = np.random.default_rng(9).integers(0, 5, (T, len(plain.node_names)), dtype=np.int32)
    env = _grid_env(tmp_path, _write(str(tmp_path / "rec.tll.xml"), reproducing_tll(plain, actions)))
    program, net, par = env_program(env), env._tables, env._params
    a, b = RefSim(net, par, R), FixedRefSim(net, par, R)
    seeds = np.array([7, 8], np.uint64)
    a.reset(seeds); b.reset(seeds)
    a.set_record(True); b.set_record(True)
    for t in range(T):
        want = a.step_record(np.repeat(actions[t][None], R, axis=0))
        got = b.step_fixed(program, record=True)
        for x, y in zip(want, got[:4] + (got[5],)):
            np.testing.assert_array_equal(x, y)
    for r in range(R):
        np.testing.assert_array_equal(a.trips(r), b.trips(r))
    assert len(a.trips(0)) > 0


def test_grid_env_program_and_tll_override(tmp_path):
    from deeprl_signal_control_b200.envs.fixedtime import FixedTimeController, env_program, phase_at
    env = _grid_env(tmp_path)
    p = env_program(env)
    assert p.n_phases.tolist() == [6] * 25 and (p.cycle == 99).all() and not p.offset.any()
    own = ('<additional><tlLogic id="nt7" type="static" offset="5"><phase duration="20" state="GGgrrrGGgrrr"/>'
           '<phase duration="20" state="rrrGGGrrrrrr"/></tlLogic></additional>')
    env2 = _grid_env(tmp_path, _write(str(tmp_path / "own.tll.xml"), own))
    q = env_program(env2)
    i = env2.node_names.index("nt7")
    assert q.n_phases[i] == 2 and q.offset[i] == 5 and q.cycle[i] == 40
    keep = [k for k in range(25) if k != i]
    assert (q.dur[keep, :6] == p.dur[keep]).all() and (q.open[keep, :6] == p.open[keep]).all()
    ctrl = FixedTimeController(env2)
    assert ctrl.name == "fixedtime"
    env2.cur_sec = 25
    np.testing.assert_array_equal(ctrl.forward(None), phase_at(q, 25))
    assert ctrl.forward(None)[i] == 1 and ctrl.forward(None)[0] == 0
    bad = _write(str(tmp_path / "bad.tll.xml"), own.replace("nt7", "nt99"))
    with pytest.raises(ValueError, match="tlLogic 'nt99' names no signalised node"):
        env_program(_grid_env(tmp_path, bad))


def test_entry_model_and_directory_checks(tmp_path, no_device, caplog):  # noqa: F811
    from deeprl_signal_control_b200.agents.evaluator import entry_model
    assert entry_model("fixedtime") == "fixedtime"
    base = str(tmp_path)
    _dir(base, "fixedtime", checkpoint=False)                 # a controller needs no checkpoint
    _dir(base, "greedy", checkpoint=False)
    _dir(base, "maxpressure", checkpoint=False)
    _dir(base, "s13/fixedtime", {"seed": "13"}, checkpoint=False)
    _dir(base, "pf/fixedtime", {"peak_flow1": "1000"}, checkpoint=False)
    tll = _write(str(tmp_path / "own.tll.xml"), '<additional><tlLogic id="nt1" type="static" offset="0">'
                 '<phase duration="40" state="GGgrrrGGgrrr"/><phase duration="20" state="rrrGGGrrrrrr"/>'
                 '</tlLogic></additional>')
    _dir(base, "own/fixedtime", {"tll_file": tll}, checkpoint=False)
    os.makedirs(os.path.join(base, "nocfg", "fixedtime", "data"))
    with caplog.at_level(logging.ERROR):
        ge = _ge(base, ["greedy", "maxpressure", "fixedtime", "s13/fixedtime", "pf/fixedtime", "own/fixedtime",
                        "nocfg/fixedtime"])
    ge.base = base
    assert [os.path.relpath(e.agent_dir, base) for e in ge.skipped] == ["nocfg/fixedtime"]
    assert "no config" in caplog.text
    # the three controllers take a simulator each; fixedtime entries of one program share one
    assert _labels(ge) == [["greedy"], ["maxpressure"], ["fixedtime", "s13/fixedtime"], ["pf/fixedtime"],
                           ["own/fixedtime"]]
    e = ge.groups[2][0]
    assert e.env.agent == "fixedtime" and e.env._params.as_c().agent_mode == 0
    assert np.array_equal(e.env._tables.obs_idx, ge.groups[0][0].env._tables.obs_idx)   # observes what greedy does


def test_monaco_tables_for_fixedtime_are_greedys():
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    a, b = real_net_tables("fixedtime"), real_net_tables("greedy")
    for name in ("obs_idx", "obs_kind", "node_obs_off", "link_from", "node_green", "src_due"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name


def test_train_refuses_fixedtime(tmp_path):
    from deeprl_signal_control_b200.agents.train import model_spec
    with pytest.raises(ValueError, match="agent 'fixedtime' has no model to train"):
        model_spec("fixedtime")
    with pytest.raises(ValueError, match="agent 'greedy' has no model to train"):
        model_spec("greedy")


def test_command_lines():
    ev = _script("evaluate")
    a = ev.parse_args(["--agent-dir", "runs/fixedtime", "--evaluation-policy-type", "stochastic"])
    assert a.agent_dir == "runs/fixedtime" and a.evaluation_policy_type == "stochastic"
    ea = _script("evaluate_agents")
    a = ea.parse_args(["--base-dir", "B", "--agents", "greedy,maxpressure,fixedtime", "--demand", "peak_flow1=1400",
                       "--demand", "peak_flow1=800", "--share-demand"])
    assert a.demand == [{"peak_flow1": "1400"}, {"peak_flow1": "800"}] and a.share_demand
    assert ea.entries("B", a.agents)[2] == ("fixedtime", "B/fixedtime", "B/eva_data/")
    assert ea.entries("B", "p/fixedtime", a.demand) == [
        ("p/fixedtime", "B/p/fixedtime", ["B/eva_data/peak_flow1-1400/p/", "B/eva_data/peak_flow1-800/p/"])]


def test_evaluate_script_refuses_a_directory_without_config(tmp_path):
    os.makedirs(tmp_path / "fixedtime" / "data")
    with pytest.raises(SystemExit, match="no config"):
        _script("evaluate").main(["--agent-dir", str(tmp_path / "fixedtime")])
