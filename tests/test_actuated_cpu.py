"""CPU: vehicle-actuated signal control's host side (envs/actuated.py) and its oracle (tests/actuated_ref.c).

- Parsing: SUMO's minDur / maxDur defaults, the static -> actuated conversion, the <param>s, every refusal by name and
  the [ENV_CONFIG] overrides.
- Loop positions on the grid, Monaco, the small grid and the mini SUMO net, short lanes included.
- Hand-computed traces on the mini SUMO net: one vehicle at known positions covers the loop in predicted seconds
  (boundaries exact to 1/64 m), and the gap and the gap-out second follow by hand; on the empty net every actuated
  phase gaps out at min_dur.
- Three identities on the oracle, on each net and in record mode: a program of fixed phases equals the fixed-time
  oracle bit for bit; max_gap = 0 equals fixed-time at min_dur; max_gap = 256 equals fixed-time at max_dur.
- `entry_model`, the directory checks, the `train` refusal and both command lines.
"""
import configparser
import json
import logging
import os
import re
import sys

import numpy as np
import pytest

from tests.test_evaluate_agents_cpu import _dir, _ge, _labels, no_device  # noqa: F401
from tests.test_evaluator_cpu import GRID_INI
from tests.test_fixedtime_cpu import _write
from tests.test_pressure_cpu import _script

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "fixtures"))
SCENARIOS = ["grid", "monaco", "small", "mini_sumo"]


def case(scenario, tmp_path):
    """(net, params, programs) of one scenario, the actuated agent's tables"""
    from deeprl_signal_control_b200.net.tables import EnvParams
    if scenario == "grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid, tls_programs
        return build_large_grid(agent="actuated"), EnvParams(agent="actuated"), tls_programs()
    if scenario == "monaco":
        from deeprl_signal_control_b200.envs.fixedtime import _MONACO_CACHE
        from deeprl_signal_control_b200.net.real_net import real_net_tables
        from tests.test_real_net_cpu import real_params
        return real_net_tables("actuated"), real_params("actuated"), json.load(open(_MONACO_CACHE))
    if scenario == "small":
        from deeprl_signal_control_b200.net.small_grid import build_small_grid, tls_programs
        return build_small_grid(agent="actuated"), EnvParams(agent="actuated"), tls_programs()
    import make_mini_sumo
    from deeprl_signal_control_b200.net.sumo_ingest import read_signal_programs
    from tests.test_evaluator_cpu import _mini_sumo
    net = _mini_sumo(tmp_path)[1]
    net_file, _ = make_mini_sumo.write(str(tmp_path))
    return net, EnvParams(agent="actuated", episode_length_sec=900), read_signal_programs(net_file)


def with_durations(program, lo, hi):
    """a copy of `program` with min_dur = lo, max_dur = hi (arrays [N][P])"""
    import dataclasses
    return dataclasses.replace(program, min_dur=np.ascontiguousarray(lo, np.int32),
                               max_dur=np.ascontiguousarray(hi, np.int32))


# ---- parsing ----------------------------------------------------------------------------------------------------
def _one(typ="actuated", attrs=None, params=None, dur=10, state="GrGr"):
    prog = {"type": typ, "offset": "0", "phases": [[str(dur), state], ["3", "yryr"], ["20", "rGrG"]]}
    if attrs is not None:
        prog["phase_attrs"] = attrs
    if params is not None:
        prog["params"] = params
    return prog


def test_sumo_defaults_and_static_conversion():
    from deeprl_signal_control_b200.envs.actuated import UNBOUNDED, phase_durations
    # minDur defaults to duration; maxDur to duration without minDur, else unbounded
    got = phase_durations("a", _one(attrs=[{"minDur": "5", "maxDur": "40"}, {}, {"minDur": "8"}]))
    assert got == [(5, 40), (3, 3), (8, UNBOUNDED)]
    assert phase_durations("a", _one(attrs=[{"maxDur": "60"}, {}, {}])) == [(10, 60), (3, 3), (20, 20)]
    # a maxDur beyond 2^30 s is unbounded
    assert phase_durations("a", _one(attrs=[{"maxDur": str(1 << 40)}, {}, {}]))[0] == (10, UNBOUNDED)
    # static: a phase with an open link and no yellow one gets [5, 50], every other phase stays fixed
    static = {"type": "static", "offset": "0", "phases": [["30", "GgrG"], ["3", "yyrG"], ["2", "rrrr"], ["30", "rrGr"]]}
    assert phase_durations("a", static) == [(5, 50), (3, 3), (2, 2), (5, 50)]
    assert phase_durations("a", static, 7, 70) == [(7, 70), (3, 3), (2, 2), (7, 70)]


def test_read_signal_programs_keeps_the_attributes(tmp_path):
    from deeprl_signal_control_b200.net.sumo_ingest import read_signal_programs
    text = ('<additional><tlLogic id="a" type="actuated" offset="0"><param key="max-gap" value="2.5"/>'
            '<phase duration="10" minDur="5" maxDur="40" state="GrGr"/><phase duration="3" state="yryr"/></tlLogic>'
            '<tlLogic id="b" type="static" offset="0"><phase duration="10" state="GrGr"/></tlLogic></additional>')
    got = read_signal_programs(_write(str(tmp_path / "a.add.xml"), text))
    assert got["a"] == {"type": "actuated", "offset": "0", "phases": [["10", "GrGr"], ["3", "yryr"]],
                        "phase_attrs": [{"minDur": "5", "maxDur": "40"}, {}], "params": {"max-gap": "2.5"}}
    assert got["b"] == {"type": "static", "offset": "0", "phases": [["10", "GrGr"]]}     # the fixed-time form


def test_refusals_name_the_id_and_the_reason(tmp_path):
    from deeprl_signal_control_b200.envs.actuated import actuated_tables, phase_durations
    cases = [(_one(typ="delay_based"), "tlLogic 'a': type 'delay_based' is neither static nor actuated"),
             (_one(typ="NEMA"), "type 'NEMA' is neither"), (_one(typ="off"), "type 'off' is neither"),
             (_one(attrs=[{"minDur": "12", "maxDur": "11"}, {}, {}]), "tlLogic 'a': minDur 12 is above maxDur 11"),
             (_one(attrs=[{"minDur": "2.5"}, {}, {}]), "tlLogic 'a': minDur '2.5' is not a whole number"),
             (_one(attrs=[{"minDur": "0"}, {}, {}]), "tlLogic 'a': minDur '0' is below 1"),
             (_one(attrs=[{"maxDur": "0"}, {}, {}]), "tlLogic 'a': maxDur '0' is below 1"),
             (_one(dur="0"), "tlLogic 'a': duration '0' is below 1"),
             (_one(dur="1.5"), "duration '1.5' is not a whole number"),
             (_one(dur="inf"), "tlLogic 'a': duration 'inf' is not a finite number"),
             (_one(attrs=[{"minDur": "nan"}, {}, {}]), "tlLogic 'a': minDur 'nan' is not a finite number"),
             (_one(attrs=[{"maxDur": "-inf"}, {}, {}]), "tlLogic 'a': maxDur '-inf' is not a finite number"),
             (_one(attrs=[{"minDur": str((1 << 30) + 1), "maxDur": str((1 << 30) + 1)}, {}, {}]),
              "tlLogic 'a': minDur '1073741825' is above 2^30 s"),
             (_one(dur=str((1 << 30) + 1)), "tlLogic 'a': duration '1073741825' is above 2^30 s")]
    for attr in ("next", "earliestEnd", "latestEnd", "vehext", "yellow", "red"):
        cases.append((_one(attrs=[{attr: "1"}, {}, {}]), "tlLogic 'a': the phase attribute '%s' is not supported" % attr))
    for prog, msg in cases:
        with pytest.raises(ValueError, match=re.escape(msg)):
            phase_durations("a", prog)
    # <param>s and the gap values, through the tables of a real net; program_tables' refusals still hold
    net = case("grid", tmp_path)[0]
    base = case("grid", tmp_path)[2]
    name = net.node_names[0]

    def tables(params=None, **kw):
        p = dict(base)
        p[name] = dict(base[name], type="actuated", **kw)
        if params is not None:
            p[name]["params"] = params
        return actuated_tables(net, p)
    ok = tables({"max-gap": "2.5", "detector-gap": "0", "show-detectors": "true", "file": "x", "freq": "60"})
    assert ok.max_gap[0] == 3 and ok.max_gap_s[0] == 2.5 and ok.detector_gap[0] == 0
    for key in ("passing-time", "jam-threshold", "inactive-threshold", "detector-length", "coordinated",
                "linkMinDur:3", "linkMaxDur:3"):
        with pytest.raises(ValueError, match="tlLogic '%s': the <param> '%s' is not supported" % (name, key)):
            tables({key: "1"})
    for key, value, msg in (("max-gap", "0", "max-gap '0' must be above 0"), ("max-gap", "-1", "max-gap '-1' must be above 0"),
                            ("detector-gap", "-0.5", "detector-gap '-0.5' must be at least 0"),
                            ("max-gap", "x", "max-gap 'x' is not a number")):
        with pytest.raises(ValueError, match="tlLogic '%s': %s" % (name, msg)):
            tables({key: value})
    with pytest.raises(ValueError, match="tlLogic '%s': state 'GrOr' has the character 'O'" % name):
        tables(phases=[["10", "GrOr"]])
    with pytest.raises(ValueError, match="tlLogic 'zz' names no signalised node"):
        actuated_tables(net, dict(base, zz=base[name]))
    with pytest.raises(ValueError, match="actuated_min_dur 9 is above actuated_max_dur 8"):
        actuated_tables(net, base, {"actuated_min_dur": 9.0, "actuated_max_dur": 8.0})


def _grid_env(tmp_path, extra="", agent="actuated"):
    from deeprl_signal_control_b200.envs.large_grid_env import LargeGridEnv
    cp = configparser.ConfigParser()
    cp.read_string(GRID_INI.replace("agent = greedy", "agent = %s" % agent) + extra)
    return LargeGridEnv(cp["ENV_CONFIG"], output_path=str(tmp_path) + os.sep)


def test_env_config_overrides(tmp_path):
    from deeprl_signal_control_b200.envs.actuated import env_program
    p = env_program(_grid_env(tmp_path))
    green = p.open.astype(bool) & ~p.yellow.astype(bool)
    assert (p.min_dur[green & (p.yellow == 0)] == 5).all() and (p.max_dur[p.min_dur == 5] == 50).all()
    assert (p.max_gap == 3).all() and (p.detector_gap == 2.0).all()
    q = env_program(_grid_env(tmp_path, "actuated_min_dur = 8\nactuated_max_dur = 44\nactuated_max_gap = 4.5\n"
                                        "actuated_detector_gap = 1\n"))
    assert set(q.min_dur[p.min_dur == 5].tolist()) == {8} and set(q.max_dur[p.max_dur == 50].tolist()) == {44}
    assert (q.max_gap == 5).all() and (q.max_gap_s == 4.5).all() and (q.detector_gap == 1.0).all()
    assert ((q.loop_pos >= p.loop_pos) | (p.loop_pos < 0)).all() and (q.loop_pos != p.loop_pos).any()
    # the keys are read only by an actuated env
    assert not hasattr(_grid_env(tmp_path, "actuated_min_dur = 8\n", agent="fixedtime"), "actuated_cfg")
    # an actuated tll_file replaces the named programs, SUMO defaults applied
    own = ('<additional><tlLogic id="nt7" type="actuated" offset="0"><param key="detector-gap" value="0.5"/>'
           '<phase duration="20" minDur="6" maxDur="30" state="GGgrrrGGgrrr"/><phase duration="3" state="yyyrrryyyrrr"/>'
           '<phase duration="20" minDur="7" state="rrrGGGrrrrrr"/></tlLogic></additional>')
    env = _grid_env(tmp_path, "tll_file = %s\n" % _write(str(tmp_path / "own.tll.xml"), own))
    r = env_program(env)
    i = env.node_names.index("nt7")
    assert r.n_phases[i] == 3 and r.min_dur[i, :3].tolist() == [6, 3, 7]
    assert r.max_dur[i, :3].tolist() == [30, 3, 1 << 30] and r.detector_gap[i] == 0.5


# ---- loops --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scenario", SCENARIOS)
def test_loop_positions(scenario, tmp_path):
    from deeprl_signal_control_b200.envs.actuated import actuated_tables, loop_positions
    net, _, programs = case(scenario, tmp_path)
    p = actuated_tables(net, programs)
    ctl = {int(f) for f, nd in zip(net.link_from, net.link_node) if f >= 0 and nd >= 0}
    assert ctl and {int(l) for l in np.flatnonzero(p.loop_pos >= 0)} == ctl
    for l in ctl:
        x = max(0.0, float(net.lane_len[l]) - 2.0 * float(net.lane_vmax[l]))
        assert p.loop_pos[l] == int(np.floor(x * 64.0)) and p.loop_pos[l] <= 65535
    # lanes shorter than detector_gap * vmax put their loop at the lane start
    far = loop_positions(net, np.full(net.n_nodes, 100.0))
    assert (far[sorted(ctl)] == 0).all() and (far[far < 0].size == p.loop_pos[p.loop_pos < 0].size)
    short = [l for l in ctl if net.lane_len[l] < 10.0 * net.lane_vmax[l]]
    mid = loop_positions(net, np.full(net.n_nodes, 10.0))
    assert all(mid[l] == 0 for l in short)


# ---- a hand-computed trace ------------------------------------------------------------------------------------------
def test_hand_computed_trace_on_the_empty_mini_net(tmp_path):
    """With no demand no loop is ever covered, so every gap stays 255 and every actuated phase gaps out at min_dur:
    the phase sequence is the program's with min_dur for each actuated phase, predicted here by hand per second."""
    import dataclasses
    from deeprl_signal_control_b200.envs.actuated import actuated_tables
    from tests.actuated_ref import ActuatedRefSim
    net, par, programs = case("mini_sumo", tmp_path)
    p = actuated_tables(net, programs)
    empty = dataclasses.replace(net, src_due=np.zeros_like(net.src_due))
    sim = ActuatedRefSim(empty, par, 1, p)
    sim.reset(np.array([3], np.uint64))
    ci = par.control_interval_sec
    for i in range(net.n_nodes):
        assert (p.min_dur[i, :p.n_phases[i]] < p.max_dur[i, :p.n_phases[i]]).any()
    for t in range(40):
        want = []
        for i in range(net.n_nodes):            # by hand: walk the phases at min_dur from the initial state
            k, e = (int(x) for x in p.init[i])
            for _ in range((t + 1) * ci):
                e += 1
                if e >= p.min_dur[i, k]:
                    k, e = (k + 1) % int(p.n_phases[i]), 0
            want.append([k, e])
        sim.step_actuated()
        assert sim.state[0].tolist() == want, t
    assert (sim.gap[0] == 255).all()


# One vehicle on the mini net, by hand.  Lane NA_A_0 (129 m, 13.89 m/s) enters node A, whose initial phase 0
# ('GGgrrrGGgrrr') opens its straight link (index 1) and its left turn; it is the only loop lane open in phase 0 that the
# net holds.  Its loop is at X = floor((129 - 2 * 13.89) * 64) = 6478 (1/64 m).  The vehicle is put at rest on the lane's
# route with speedFactor 1, sigma = 0 and no other traffic, so it moves 5, 10, then 13.89 m per second (accel 5 m/s^2,
# lane speed 13.89, no junction speed limit) and crosses the stop line in its fifth second.  Lq = 5 m = 320.
# (start xq - X, seconds in which it covers the loop):
_VEHICLE_CASES = [
    # passes over the loop: s2 front 5749 -> 6637 (reaches X), s3 back 6637 - 320 = 6317 <= X (back still over it)
    (-1689, {2, 3}),
    # at rest with its back exactly on the loop: s0 xq - Lq = X (covered); s1 back at X + 320 (not)
    (320, {0}),
    (321, set()),                 # back one unit past the loop: never covered
    # front reaches the loop exactly at the end of s0 (xnq = X), and s1 starts with it on the loop
    (-320, {0, 1}),
    (-321, {1}),                  # front one unit short of the loop after s0
]


@pytest.mark.parametrize("start,covered", _VEHICLE_CASES)
@pytest.mark.parametrize("max_gap", [2, 3, 5])
def test_one_vehicle_gap_out_by_hand(start, covered, max_gap, tmp_path):
    """Per second: the vehicle's position, the lane's gap and node A's (phase, elapsed) equal the prediction.  gap is
    255 until the first covered second, 0 after a covered one, +1 after each uncovered one; phase 0 (minDur 5, maxDur
    50) ends after second s, the first s >= 4 whose gap is >= max_gap, then the 3-s yellow and the next green, whose
    lanes are empty, follow; node B, with no vehicle, ends phase 0 at minDur."""
    import dataclasses
    from deeprl_signal_control_b200.envs.actuated import actuated_tables
    from tests.actuated_ref import ActuatedRefSim
    net, par, programs = case("mini_sumo", tmp_path)
    par = dataclasses.replace(par, control_interval_sec=1, yellow_interval_sec=1, sigma=0.0)
    net = dataclasses.replace(net, src_due=np.zeros_like(net.src_due))
    p = actuated_tables(net, programs)
    lane = net.lane_names.index("NA_A_0")
    A, B = net.node_names.index("A"), net.node_names.index("B")
    X = p.loop_pos[lane]
    assert X == 6478 and net.lane_len[lane] == 129.0
    route = [r for r in range(len(net.route_lane)) if net.route_lane[r][0] == lane and net.route_link[r][0] >= 0]
    link = int(net.route_link[route[0]][0])
    assert net.link_node[link] == A and net.link_tlidx[link] == 1 and net.link_vmax[link] > 1e8
    assert p.init[A].tolist() == [0, 0] and (p.min_dur[A, 0], p.max_dur[A, 0]) == (5, 50)
    sim = ActuatedRefSim(net, par, 1, p, max_gap=np.full(net.n_nodes, max_gap, np.int32))
    sim.reset(np.array([1], np.uint64))
    sim.put_vehicle(0, lane, X + start, route[0])
    x, v, gap, phase, el = (X + start) / 64.0, 0.0, 255, 0, 0
    end_a = end_b = None
    for s in range(12):
        sim.step_actuated()
        v = min(v + 5.0, 13.89)
        x += v
        gap = 0 if s in covered else min(gap + 1, 255)
        el += 1
        if phase == 0 and el >= 5 and gap >= max_gap:
            phase, el, end_a = 1, 0, s
        elif (phase, el) in ((1, 3), (2, 5)):           # the fixed 3-s yellow; the next green has no vehicle
            phase, el = phase + 1, 0
        cnt, veh = sim.dump_state(0)[:2]
        if x < 129.0:                                   # still on the lane, the only vehicle of the net
            pos = float(np.asarray(veh, np.uint32).view(np.float32)[0][0])
            # stored positions are truncated to 1/64 m each second, so the hand sum runs ahead by < 1/64 m a second
            assert cnt[lane] == 1 and 0 <= x - pos < (s + 1) / 64.0, (s, pos, x)
        assert sim.gap[0][lane] == gap, (s, sim.gap[0][lane], gap)
        assert sim.state[0][A].tolist() == [phase, el], (s, sim.state[0][A].tolist(), [phase, el])
        if sim.state[0][B][0] != 0 and end_b is None:
            end_b = s
    # phase 0 of A ends after second max(4, last covered second + max_gap); B's after second 4 (minDur)
    assert end_a == max(4, max(covered, default=-255) + max_gap) and end_b == 4


# ---- the oracle identities ------------------------------------------------------------------------------------------
def _identity(scenario, tmp_path, kind, record, n_steps=None):
    from deeprl_signal_control_b200.envs.actuated import actuated_tables, fixed_program
    from tests.actuated_ref import ActuatedRefSim
    from tests.fixedtime_ref import FixedRefSim
    net, par, programs = case(scenario, tmp_path)
    p = actuated_tables(net, programs)
    assert (p.min_dur < p.max_dur).any()
    if kind == "fixed":
        ap, mg, fp = with_durations(p, p.dur, p.dur), None, fixed_program(with_durations(p, p.dur, p.dur))
    elif kind == "gap0":
        ap, mg, fp = p, np.zeros(net.n_nodes, np.int32), fixed_program(with_durations(p, p.min_dur, p.min_dur))
    else:
        ap, mg, fp = p, np.full(net.n_nodes, 256, np.int32), fixed_program(with_durations(p, p.max_dur, p.max_dur))
    R, ci = 2, par.control_interval_sec
    n_steps = n_steps or int(fp.cycle.max()) // ci * 2 + 2
    a, b = ActuatedRefSim(net, par, R, ap, max_gap=mg), FixedRefSim(net, par, R)
    seeds = np.array([5, 17], np.uint64)
    for s in (a, b):
        s.reset(seeds)
        s.set_train_mode(False)
        if record:
            s.set_record(True)
    from deeprl_signal_control_b200.envs.fixedtime import phase_at
    for t in range(n_steps):
        got, want = a.step_actuated(record=record), b.step_fixed(fp, record=record)
        for x, y in zip(got, want):
            np.testing.assert_array_equal(x, y)
        np.testing.assert_array_equal(got[4][0], phase_at(fp, t * ci))
        for x, y in zip(a.counts(), b.counts()):
            np.testing.assert_array_equal(x, y)
    for r in range(R):
        for x, y in zip(a.dump_state(r), b.dump_state(r)):
            np.testing.assert_array_equal(x, y)
        if record:
            np.testing.assert_array_equal(a.trips(r), b.trips(r))
    assert a.misc(0)["live"] > 0


@pytest.mark.parametrize("scenario", SCENARIOS)
@pytest.mark.parametrize("kind", ["fixed", "gap0", "gap256"])
def test_oracle_identities(scenario, kind, tmp_path):
    _identity(scenario, tmp_path, kind, record=False)


@pytest.mark.parametrize("scenario", ["grid", "mini_sumo"])
@pytest.mark.parametrize("kind", ["fixed", "gap0", "gap256"])
def test_oracle_identities_in_record_mode(scenario, kind, tmp_path):
    _identity(scenario, tmp_path, kind, record=True, n_steps=30)


def test_actuation_changes_the_run(tmp_path):
    """with the default max_gap the actuated run differs from both bounds, and it stays within them"""
    from deeprl_signal_control_b200.envs.actuated import actuated_tables
    from tests.actuated_ref import ActuatedRefSim
    net, par, programs = case("grid", tmp_path)
    p = actuated_tables(net, programs)
    sim = ActuatedRefSim(net, par, 2, p)
    sim.reset(np.array([1, 2], np.uint64))
    seen = []
    for t in range(120):
        before = sim.state.copy()
        sim.step_actuated()
        seen.append(sim.state[:, :, 0].copy())
        assert (sim.state[:, :, 1] < 50).all()
        assert ((sim.state[:, :, 0] == before[:, :, 0]) | (sim.state[:, :, 1] <= 5)).all()
    ph = np.stack(seen)
    assert (sim.gap < 255).any() and (sim.gap == 0).any()
    durs = []                        # lengths of completed green phases: some gap out between 5 and 50
    for r in range(2):
        for i in range(net.n_nodes):
            run = np.flatnonzero(np.diff(ph[:, r, i]) != 0)
            durs += list(np.diff(run) * par.control_interval_sec)
    assert min(durs) < 50 and max(durs) > 5


# ---- evaluation plumbing --------------------------------------------------------------------------------------------
def test_entry_model_and_directory_checks(tmp_path, no_device, caplog):  # noqa: F811
    from deeprl_signal_control_b200.agents.evaluator import entry_model
    assert entry_model("actuated") == "actuated"
    base = str(tmp_path)
    _dir(base, "actuated", checkpoint=False)                  # a controller needs no checkpoint
    _dir(base, "fixedtime", checkpoint=False)
    _dir(base, "s13/actuated", {"seed": "13"}, checkpoint=False)
    _dir(base, "gap/actuated", {"actuated_max_gap": "5"}, checkpoint=False)
    _dir(base, "pf/actuated", {"peak_flow1": "1000"}, checkpoint=False)
    os.makedirs(os.path.join(base, "nocfg", "actuated", "data"))
    with caplog.at_level(logging.ERROR):
        ge = _ge(base, ["fixedtime", "actuated", "s13/actuated", "gap/actuated", "pf/actuated", "nocfg/actuated"])
    ge.base = base
    assert [os.path.relpath(e.agent_dir, base) for e in ge.skipped] == ["nocfg/actuated"]
    # actuated entries of one program share a simulator; another max_gap is another program
    assert _labels(ge) == [["fixedtime"], ["actuated", "s13/actuated"], ["gap/actuated"], ["pf/actuated"]]
    e = ge.groups[1][0]
    assert e.env.agent == "actuated" and e.env._params.as_c().agent_mode == 0
    assert np.array_equal(e.env._tables.obs_idx, ge.groups[0][0].env._tables.obs_idx)


def test_monaco_tables_for_actuated_are_greedys():
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    a, b = real_net_tables("actuated"), real_net_tables("greedy")
    for name in ("obs_idx", "obs_kind", "node_obs_off", "link_from", "node_green", "src_due"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name


def test_train_refuses_actuated():
    from deeprl_signal_control_b200.agents.train import model_spec
    with pytest.raises(ValueError, match="agent 'actuated' has no model to train"):
        model_spec("actuated")


def test_command_lines():
    ev = _script("evaluate")
    a = ev.parse_args(["--agent-dir", "runs/actuated", "--evaluation-policy-type", "stochastic"])
    assert a.agent_dir == "runs/actuated"
    ea = _script("evaluate_agents")
    a = ea.parse_args(["--base-dir", "B", "--agents", "greedy,fixedtime,actuated", "--demand", "peak_flow1=1400",
                       "--demand", "peak_flow1=800", "--share-demand"])
    assert a.share_demand and ea.entries("B", a.agents)[2] == ("actuated", "B/actuated", "B/eva_data/")
    assert ea.entries("B", "p/actuated", a.demand) == [
        ("p/actuated", "B/p/actuated", ["B/eva_data/peak_flow1-1400/p/", "B/eva_data/peak_flow1-800/p/"])]


def test_evaluate_script_refuses_a_directory_without_config(tmp_path):
    os.makedirs(tmp_path / "actuated" / "data")
    with pytest.raises(SystemExit, match="no config"):
        _script("evaluate").main(["--agent-dir", str(tmp_path / "actuated")])
