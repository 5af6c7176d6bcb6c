"""CPU: the max-pressure controller's host side (envs/maxpressure.py) — the per-node link lists against each node's phase
strings, the numpy definition on hand-made lane counts and against a literal loop over the links, the maxpressure entry
of the evaluators (entry_model, the directory checks, its own simulator) and the command lines of scripts/evaluate.py
and scripts/evaluate_agents.py."""
import configparser
import importlib.util
import logging
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from tests.test_evaluate_agents_cpu import _dir, _ge, _labels, no_device  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "fixtures"))


def _nets(tmp_path):
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    from deeprl_signal_control_b200.net.small_grid import build_small_grid
    from tests.test_evaluator_cpu import _mini_sumo
    return {"grid": build_large_grid(agent="maxpressure"), "monaco": real_net_tables("maxpressure"),
            "small": build_small_grid(agent="maxpressure"), "mini_sumo": _mini_sumo(tmp_path)[1]}


@pytest.mark.parametrize("scenario", ["grid", "monaco", "small", "mini_sumo"])
def test_link_lists_read_the_phase_strings(scenario, tmp_path):
    from deeprl_signal_control_b200.envs.maxpressure import pressure_links
    net = _nets(tmp_path)[scenario]
    off, fr, to, tl = pressure_links(net)
    node, lane_to = np.asarray(net.link_node), np.asarray(net.link_to)
    assert off[0] == 0 and off[-1] == len(fr) == int(((node >= 0) & (lane_to >= 0)).sum())
    assert (np.asarray(net.link_from) >= 0).all()
    if scenario == "monaco":
        assert int(((node >= 0) & (lane_to < 0)).sum()) == 4      # connections to lanes outside the passenger net
    inl_off, inl = np.asarray(net.lane_inl_off), np.asarray(net.lane_inl)
    entering = {}                                        # link -> the lanes whose incoming links list it
    for lane in range(net.n_lanes):
        for q in range(inl_off[lane], inl_off[lane + 1]):
            entering.setdefault(int(inl[q]), set()).add(net.lane_names[lane])
    green = np.asarray(net.node_green).reshape(net.n_nodes, -1)
    n_green = 0
    for i, name in enumerate(net.node_names):
        phases = net.phases[name]
        assert int(net.node_n_phases[i]) == len(phases)
        mine = [l for l in range(net.n_links) if node[l] == i and lane_to[l] >= 0]
        # node i's entries are its controlled links in index order: from lane = the phase string's controlled lane at the
        # link's position, to lane = one of the lanes whose incoming links list the link
        want = [(net.lanes_in[name][net.link_tlidx[l]], int(net.link_tlidx[l])) for l in mine]
        got = [(net.lane_names[f], int(x)) for f, x in zip(fr[off[i]:off[i + 1]], tl[off[i]:off[i + 1]])]
        assert got == want, name
        assert all(net.lane_names[t] in entering[l] for l, t in zip(mine, to[off[i]:off[i + 1]])), name
        for p, s in enumerate(phases):
            by_string = [e for e in got if s[e[1]] in "Gg"]
            by_mask = [e for e in got if (int(green[i, p]) >> e[1]) & 1]
            assert by_string == by_mask, (name, p)
            n_green += len(by_string)
    assert n_green > 0


def _toy(phases, links, n_lanes):
    """A one-node net: phase strings, links (from, to, node, tlidx)."""
    from deeprl_signal_control_b200.net.tables import phase_masks
    g, _ = phase_masks(phases)
    fr, to, nd, tl = (np.array(c, np.int32) for c in zip(*links))
    return SimpleNamespace(n_nodes=1, n_lanes=n_lanes, link_from=fr, link_to=to, link_node=nd, link_tlidx=tl,
                           node_green=np.array(g, np.uint32).reshape(1, -1), node_n_phases=np.array([len(phases)]))


def test_definition_on_hand_made_counts():
    from deeprl_signal_control_b200.envs.maxpressure import pressure_actions
    # lanes 0, 1 enter the node, 2, 3 leave it; link k sits at position k of the phase strings
    net = _toy(["Gr", "rG"], [(0, 2, 0, 0), (1, 3, 0, 1)], 4)
    act = lambda *cnt: int(pressure_actions(net, np.array(cnt))[0])
    assert act(0, 0, 0, 0) == 0                          # an empty net: every phase scores 0, the first one wins
    assert act(3, 5, 0, 0) == 1 and act(5, 3, 0, 0) == 0
    assert act(4, 4, 0, 0) == 0                          # a tie resolves to the first phase
    assert act(2, 2, 0, 3) == 0                          # the outgoing queue counts: phase 1 scores 2 - 3 = -1 < 0
    assert act(0, 0, 6, 1) == 1                          # both pressures negative: the larger (-1) wins
    # permissive 'g' counts as green
    assert int(pressure_actions(_toy(["gr", "rG"], [(0, 2, 0, 0), (1, 3, 0, 1)], 4), np.array([5, 3, 0, 0]))[0]) == 0
    # an uncontrolled link at the same position does not count, nor does a link into a lane outside the net
    unc = _toy(["Gr", "rG"], [(0, 2, 0, 0), (1, 3, 0, 1), (1, 2, -1, 0), (1, -1, 0, 0)], 4)
    assert int(pressure_actions(unc, np.array([1, 9, 0, 0]))[0]) == 1
    # a phase with no green link scores 0 and wins over negative pressures; batched counts keep their leading shape
    three = _toy(["Gr", "rG", "rr"], [(0, 2, 0, 0), (1, 3, 0, 1)], 4)
    got = pressure_actions(three, np.array([[[0, 0, 5, 5], [3, 0, 0, 0]]]))
    assert got.shape == (1, 2, 1) and got.dtype == np.int32 and got[0, :, 0].tolist() == [2, 0]


@pytest.mark.parametrize("scenario", ["grid", "monaco", "small", "mini_sumo"])
def test_definition_equals_a_loop_over_the_links(scenario, tmp_path):
    from deeprl_signal_control_b200.envs.maxpressure import pressure_actions
    net = _nets(tmp_path)[scenario]
    rng = np.random.default_rng(7)
    cnt = np.concatenate([rng.integers(0, 4, (40, net.n_lanes)), rng.integers(0, 60, (40, net.n_lanes)),
                          np.zeros((1, net.n_lanes), np.int64)])
    green = np.asarray(net.node_green).reshape(net.n_nodes, -1)
    want = np.zeros((len(cnt), net.n_nodes), np.int32)
    for r in range(len(cnt)):
        for i in range(net.n_nodes):
            best = None
            for p in range(int(net.node_n_phases[i])):
                s = sum(int(cnt[r, net.link_from[l]]) - int(cnt[r, net.link_to[l]]) for l in range(net.n_links)
                        if net.link_node[l] == i and net.link_to[l] >= 0 and (int(green[i, p]) >> int(net.link_tlidx[l])) & 1)
                if best is None or s > best:
                    best, want[r, i] = s, p
    got = pressure_actions(net, cnt)
    np.testing.assert_array_equal(got, want)
    assert len(np.unique(got)) > 1 and not got[-1].any()


def test_entry_model_and_directory_checks(tmp_path, no_device, caplog):  # noqa: F811
    from deeprl_signal_control_b200.agents.evaluator import entry_model
    assert entry_model("maxpressure") == "maxpressure" and entry_model("greedy") == "greedy"
    base = str(tmp_path)
    _dir(base, "maxpressure", checkpoint=False)              # a controller needs no checkpoint
    _dir(base, "greedy", checkpoint=False)
    _dir(base, "pf/maxpressure", {"peak_flow1": "1000"}, checkpoint=False)
    _dir(base, "s13/maxpressure", {"seed": "13"}, checkpoint=False)
    os.makedirs(os.path.join(base, "nocfg", "maxpressure", "data"))
    with caplog.at_level(logging.ERROR):
        ge = _ge(base, ["greedy", "maxpressure", "pf/maxpressure", "s13/maxpressure", "nocfg/maxpressure"])
    ge.base = base
    assert [os.path.relpath(e.agent_dir, base) for e in ge.skipped] == ["nocfg/maxpressure"]
    assert "nocfg/maxpressure" in caplog.text and "no config" in caplog.text
    # greedy and maxpressure would build the same simulator; each controller launch writes all of its rows, so they
    # take one each
    assert _labels(ge) == [["greedy"], ["maxpressure", "s13/maxpressure"], ["pf/maxpressure"]]
    e = ge.groups[1][0]
    assert e.env.agent == "maxpressure" and e.env._params.as_c().agent_mode == 0
    greedy_net = ge.groups[0][0].env._tables
    assert np.array_equal(e.env._tables.obs_idx, greedy_net.obs_idx)            # maxpressure observes what greedy does


def test_monaco_tables_for_maxpressure_are_greedys():
    from deeprl_signal_control_b200.net.real_net import real_net_tables
    a, b = real_net_tables("maxpressure"), real_net_tables("greedy")
    for name in ("obs_idx", "obs_kind", "node_obs_off", "link_from", "link_to", "node_green", "src_due"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name


def _script(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "scripts", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_command_lines():
    ev = _script("evaluate")
    a = ev.parse_args(["--agent-dir", "runs/maxpressure", "--evaluation-policy-type", "stochastic"])
    assert a.agent_dir == "runs/maxpressure" and a.evaluation_policy_type == "stochastic"
    ea = _script("evaluate_agents")
    a = ea.parse_args(["--base-dir", "B", "--agents", "greedy,maxpressure,ma2c", "--demand", "peak_flow1=1400",
                       "--demand", "peak_flow1=800", "--share-demand"])
    assert a.demand == [{"peak_flow1": "1400"}, {"peak_flow1": "800"}] and a.share_demand
    assert ea.entries("B", a.agents) == [("greedy", "B/greedy", "B/eva_data/"),
                                         ("maxpressure", "B/maxpressure", "B/eva_data/"), ("ma2c", "B/ma2c", "B/eva_data/")]
    assert ea.entries("B", "p/maxpressure", a.demand) == [
        ("p/maxpressure", "B/p/maxpressure", ["B/eva_data/peak_flow1-1400/p/", "B/eva_data/peak_flow1-800/p/"])]


def test_evaluate_script_refuses_a_directory_without_config(tmp_path):
    os.makedirs(tmp_path / "maxpressure" / "data")
    with pytest.raises(SystemExit, match="no config"):
        _script("evaluate").main(["--agent-dir", str(tmp_path / "maxpressure")])
