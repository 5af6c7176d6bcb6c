"""CPU: the host side of traffic demand levels — which net tables a demand key changes (net/tables.py:demand_mismatch),
the Monaco table cache honouring flow_rate, demand sweeps' key checks and refusals (agents/train.py:sweep_members with
demand=True, the --vary-demand flags), and the grouped evaluator's demand levels (agents/evaluator.py, the --demand
parsing, labels and output paths of scripts/evaluate_agents.py)."""
import configparser
import gzip
import os
import shutil
import sys

import numpy as np
import pytest

from tests.test_evaluate_agents_cpu import _cli, _dir, no_device  # noqa: F401
from tests.test_sweep_cpu import _cfg, _write

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_NET = os.path.join(ROOT, "tests", "golden", "monaco_sumo", "most.net.xml.gz")


def _fields_that_differ(a, b):
    import dataclasses
    from deeprl_signal_control_b200.net.tables import _same_value
    return [f.name for f in dataclasses.fields(a) if not _same_value(getattr(a, f.name), getattr(b, f.name))]


def test_grid_peak_flows_change_only_src_due():
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import demand_mismatch
    a, b = build_large_grid(1100, 925, agent="ma2c"), build_large_grid(1400, 1180, agent="ma2c")
    assert _fields_that_differ(a, b) == ["src_due"]
    assert demand_mismatch(a, b) is None


def test_small_grid_demand_changes_only_src_phi():
    from deeprl_signal_control_b200.net.small_grid import build_small_grid
    from deeprl_signal_control_b200.net.tables import demand_mismatch
    a, b = build_small_grid(1000, agent="ma2c"), build_small_grid(1500, agent="ma2c")
    assert _fields_that_differ(a, b) == ["src_phi"]
    assert demand_mismatch(a, b) is None


def test_init_density_is_not_demand():
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import DEMAND_FIELDS, demand_mismatch
    a, b = build_large_grid(agent="ma2c"), build_large_grid(agent="ma2c", init_density=0.1, seed=12)
    f = demand_mismatch(a, b)
    assert f is not None and f not in DEMAND_FIELDS and f.startswith(("src_", "route_"))


def _mini(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests", "fixtures"))
    import make_mini_sumo
    return make_mini_sumo.write(str(tmp_path))


def _sumo_env(net_file, rou_file, tmp_path):
    from deeprl_signal_control_b200.envs import make_env
    c = _cfg("ma2c")["ENV_CONFIG"]
    c["scenario"], c["net_file"], c["route_file"] = "mini", net_file, rou_file
    c["episode_length_sec"] = "600"
    return make_env(c, 1, str(tmp_path) + "/", is_record=False)


def test_sumo_route_file_is_demand_only_when_the_routes_stay(tmp_path):
    from deeprl_signal_control_b200.envs import check_demand_tables
    net_file, rou = _mini(tmp_path)
    text = open(rou).read()
    more = str(tmp_path / "more.rou.xml")
    with open(more, "w") as f:                              # the same flows at other rates
        f.write(text.replace('vehsPerHour="600"', 'vehsPerHour="900"').replace('vehsPerHour="240"', 'vehsPerHour="300"'))
    other = str(tmp_path / "other.rou.xml")
    with open(other, "w") as f:                             # one flow on another route
        f.write(text.replace('to="B_E" via="A_B"', 'to="B_SB" via="A_B"'))
    base = _sumo_env(net_file, rou, tmp_path)
    check_demand_tables(base._tables, _sumo_env(net_file, more, tmp_path)._tables, "more")
    with pytest.raises(ValueError, match=r"other: the net differs in '(\w+)'") as e:
        check_demand_tables(base._tables, _sumo_env(net_file, other, tmp_path)._tables, "other")
    assert str(e.value).split("'")[1] not in ("src_due", "src_plo", "src_phi")


def test_demand_keys_per_scenario():
    from deeprl_signal_control_b200.envs import DEMAND_KEYS, demand_keys
    assert DEMAND_KEYS == {"large_grid": ("peak_flow1", "peak_flow2"), "real_net": ("flow_rate",),
                           "small_grid": ("num_extra_car_per_hour",)}
    c = configparser.ConfigParser()
    c.read_string("[ENV_CONFIG]\nscenario = mini\nnet_file = a.net.xml\n")
    assert demand_keys(c["ENV_CONFIG"]) == ("route_file",)
    c["ENV_CONFIG"]["scenario"] = "real_net"
    assert demand_keys(c["ENV_CONFIG"]) == ("flow_rate",)


@pytest.mark.parametrize("agent", ["greedy", "ia2c", "ma2c"])
def test_monaco_cache_at_325_is_the_shipped_table(agent):
    from deeprl_signal_control_b200.net import real_net as rn
    shipped = rn.load_tables(rn._CACHE % agent)
    net = rn.real_net_tables(agent, flow_rate=325)
    assert net.src_due.dtype == np.uint8 and np.array_equal(net.src_due, shipped.src_due)
    assert int(net.src_due.sum()) == 2464
    assert _fields_that_differ(net, shipped) == []


def test_monaco_cache_honours_flow_rate(tmp_path):
    from deeprl_signal_control_b200.net import real_net as rn
    cached = rn.real_net_tables("ma2c", flow_rate=450)
    assert int(cached.src_due.sum()) == 3344
    assert _fields_that_differ(cached, rn.real_net_tables("ma2c")) == ["src_due"]
    if not os.path.exists(GOLD_NET):
        pytest.skip("no Monaco net file")
    net_file = str(tmp_path / "most.net.xml")
    with gzip.open(GOLD_NET, "rb") as fi, open(net_file, "wb") as fo:
        shutil.copyfileobj(fi, fo)
    built = rn.build_real_net(net_file, flow_rate=450, agent="ma2c")
    assert np.array_equal(built.src_due, cached.src_due)
    assert rn.real_net_tables("ma2c", net_file, flow_rate=450).src_due.tobytes() == cached.src_due.tobytes()


# ---- sweeps over demand ------------------------------------------------------------------------------------------------
DEMAND_VALUES = {"large_grid": {"peak_flow1": "1400", "peak_flow2": "1180"}, "real_net": {"flow_rate": "450"},
                 "small_grid": {"num_extra_car_per_hour": "1500"}}


def _scenario_cfg(scenario, agent="ma2c", changes=None):
    c = _cfg(agent)
    e = c["ENV_CONFIG"]
    e["scenario"] = scenario
    if scenario == "real_net":
        e["flow_rate"] = "325"
        e["data_path"] = "/nonexistent/"
    elif scenario == "small_grid":
        e["num_extra_car_per_hour"] = "1000"
    for k, v in (changes or {}).items():
        e[k] = v
    return c


@pytest.mark.parametrize("scenario", sorted(DEMAND_VALUES))
def test_sweep_accepts_the_scenario_demand_keys(scenario):
    from deeprl_signal_control_b200.agents.train import member_demand, sweep_members
    a, b = _scenario_cfg(scenario), _scenario_cfg(scenario, changes=DEMAND_VALUES[scenario])
    items = sweep_members({"lo": a, "hi": b}, demand=True)
    assert [n for n, _, _ in items] == ["lo", "hi"]
    nets = member_demand([a, b])
    assert nets is not None and len(nets) == 2
    assert member_demand([a, _scenario_cfg(scenario, changes={"seed": "13"})]) is None    # one demand: none to set
    with pytest.raises(ValueError, match=sorted(DEMAND_VALUES[scenario])[0]):              # not without the flag
        sweep_members({"lo": a, "hi": b})


def test_demand_combines_with_coop_gamma_and_reward_norm():
    from deeprl_signal_control_b200.agents.train import sweep_members
    b = _scenario_cfg("large_grid", changes={"peak_flow1": "1400", "coop_gamma": "0.75"})
    b["MODEL_CONFIG"]["reward_norm"] = "3000.0"
    assert len(sweep_members({"a": _scenario_cfg("large_grid"), "b": b}, demand=True)) == 2


@pytest.mark.parametrize("sec,key,value", [("ENV_CONFIG", "init_density", "0.1"), ("MODEL_CONFIG", "num_lstm", "32"),
                                           ("ENV_CONFIG", "flow_rate", "450"), ("ENV_CONFIG", "episode_length_sec", "1800"),
                                           ("ENV_CONFIG", "num_extra_car_per_hour", "1500")])
def test_demand_sweep_still_refuses_other_keys_by_name_and_file(tmp_path, sec, key, value):
    from deeprl_signal_control_b200.agents.train import sweep_members
    a = _write(tmp_path, "a", _scenario_cfg("large_grid"))
    bc = _scenario_cfg("large_grid", changes={"peak_flow1": "1400"})
    bc[sec][key] = value
    b = _write(tmp_path, "b", bc)
    with pytest.raises(ValueError, match=key) as e:
        sweep_members([a, b], demand=True)
    assert a in str(e.value) and b in str(e.value)


@pytest.mark.parametrize("script", ["train", "iql"])
def test_vary_demand_refusals_leave_no_directory(tmp_path, script):
    import importlib.util
    agent = "ma2c" if script == "train" else "iqll"
    a = _write(tmp_path, "a", _scenario_cfg("large_grid", agent))
    bc = _scenario_cfg("large_grid", agent, changes={"peak_flow1": "1400"})
    bc["ENV_CONFIG"]["init_density"] = "0.1"
    b = _write(tmp_path, "b", bc)
    base = tmp_path / "runs"
    name = "train.py" if script == "train" else "train_iql_members.py"
    spec = importlib.util.spec_from_file_location("m_" + script, os.path.join(ROOT, "scripts", name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    argv = (["--base-dir", str(base), "train", "--sweep", "%s,%s" % (a, b), "--replicas", "64", "--vary-demand"]
            if script == "train" else
            ["--base-dir", str(base), "--sweep", "%s,%s" % (a, b), "--replicas", "64", "--vary-demand"])
    with pytest.raises(ValueError, match="init_density"):
        mod.main(argv)
    assert not base.exists()
    # the flag is refused without a sweep; with it but equal demand keys, peak_flow1 is refused as before
    with pytest.raises(SystemExit):
        mod.parse_args((["--base-dir", str(base), "train", "--config-dir", a, "--seeds", "1,2", "--vary-demand"])
                       if script == "train" else
                       ["--base-dir", str(base), "--config-dir", a, "--seeds", "1,2", "--replicas", "1",
                        "--vary-demand"])
    c = _write(tmp_path, "c", _scenario_cfg("large_grid", agent, changes={"peak_flow1": "1400"}))
    with pytest.raises(ValueError, match="peak_flow1"):
        mod.main([x if x != "%s,%s" % (a, b) else "%s,%s" % (a, c) for x in argv if x != "--vary-demand"])
    assert not base.exists()


def test_vary_demand_train_sweep_refuses_before_directories(tmp_path):
    from deeprl_signal_control_b200.agents.train import train_iql_sweep, train_sweep
    a = _scenario_cfg("large_grid")
    b = _scenario_cfg("large_grid", changes={"peak_flow1": "1400", "init_density": "0.1"})
    with pytest.raises(ValueError, match="init_density"):
        train_sweep({"a": a, "b": b}, str(tmp_path / "x"), n_replicas=64, vary_demand=True)
    ai, bi = _scenario_cfg("large_grid", "iqll"), _scenario_cfg("large_grid", "iqll", changes={"flow_rate": "450"})
    with pytest.raises(ValueError, match="flow_rate"):
        train_iql_sweep({"a": ai, "b": bi}, str(tmp_path / "y"), n_replicas=64, vary_demand=True)
    assert not (tmp_path / "x").exists() and not (tmp_path / "y").exists()


# ---- evaluation across demand levels ---------------------------------------------------------------------------------
def test_demand_parsing_labels_and_output_paths():
    cli = _cli()
    a = cli.parse_args(["--base-dir", "B", "--agents", "ma2c", "--demand", "peak_flow1=1400,peak_flow2=1180",
                        "--demand", "peak_flow1=1700"])
    assert a.demand == [{"peak_flow1": "1400", "peak_flow2": "1180"}, {"peak_flow1": "1700"}]
    assert [cli.demand_label(lv) for lv in a.demand] == ["peak_flow1-1400_peak_flow2-1180", "peak_flow1-1700"]
    assert cli.parse_args(["--base-dir", "B", "--agents", "ma2c"]).demand is None
    assert not cli.parse_args(["--base-dir", "B", "--agents", "ma2c"]).share_demand
    for bad in ("peak_flow1", "=3", "peak_flow1=1,peak_flow1=2", ","):
        with pytest.raises(SystemExit):
            cli.parse_args(["--base-dir", "B", "--agents", "ma2c", "--demand", bad])
    with pytest.raises(SystemExit):                                            # one level twice
        cli.parse_args(["--base-dir", "B", "--agents", "ma2c", "--demand", "flow_rate=4", "--demand", "flow_rate=4"])
    ent = cli.entries("B", "greedy,pf/ma2c", a.demand)
    assert ent == [("greedy", "B/greedy", ["B/eva_data/peak_flow1-1400_peak_flow2-1180/", "B/eva_data/peak_flow1-1700/"]),
                   ("pf/ma2c", "B/pf/ma2c", ["B/eva_data/peak_flow1-1400_peak_flow2-1180/pf/",
                                             "B/eva_data/peak_flow1-1700/pf/"])]
    assert cli.entries("B", "greedy,pf/ma2c") == [("greedy", "B/greedy", "B/eva_data/"),
                                                   ("pf/ma2c", "B/pf/ma2c", "B/eva_data/pf/")]


def _ge(base, entries, levels=None, **kw):
    from deeprl_signal_control_b200.agents.evaluator import GroupEvaluator, entry_model
    out = (lambda e: str(base) + "/") if levels is None else (lambda e: [str(base) + "/L%d/" % j for j in range(len(levels))])
    return GroupEvaluator([(os.path.join(base, e), entry_model(os.path.basename(e)), out(e)) for e in entries],
                          [10000, 20000], demand_levels=levels, **kw)


def test_demand_levels_group_every_entry_at_every_level(tmp_path, no_device):  # noqa: F811
    from deeprl_signal_control_b200.agents.evaluator import sim_key
    base = str(tmp_path)
    for e in ("greedy", "ma2c", "iqll", "ia2c"):
        _dir(base, e)
    levels = [{"peak_flow1": "1100", "peak_flow2": "925"}, {"peak_flow1": 1400, "peak_flow2": 1180}, {"peak_flow1": 800}]
    ge = _ge(base, ["greedy", "ma2c", "iqll", "ia2c"], levels)
    assert len(ge.entries) == 12 and not ge.skipped
    # greedy, ma2c and the ia2c / iqll observation layout: one simulator each, holding every level
    assert [[(os.path.basename(e.agent_dir), e.demand["peak_flow1"]) for e in g] for g in ge.groups] == [
        [("greedy", "1100"), ("greedy", "1400"), ("greedy", "800")],
        [("ma2c", "1100"), ("ma2c", "1400"), ("ma2c", "800")],
        [("iqll", "1100"), ("iqll", "1400"), ("iqll", "800"), ("ia2c", "1100"), ("ia2c", "1400"), ("ia2c", "800")]]
    g = ge.groups[1]
    assert g[2].env.peak_flow1 == 800 and g[2].env.peak_flow2 == g[0].env.peak_flow2        # unnamed keys keep their value
    assert [e.output_path for e in g] == [base + "/L0/", base + "/L1/", base + "/L2/"]
    assert sim_key(g[0].env) != sim_key(g[1].env) and sim_key(g[0].env, demand=True) == sim_key(g[1].env, demand=True)


def test_share_demand_groups_a_demand_sweep(tmp_path, no_device):  # noqa: F811
    base = str(tmp_path)
    _dir(base, "pf1100/ma2c", {"peak_flow1": "1100"})
    _dir(base, "pf1400/ma2c", {"peak_flow1": "1400"})
    _dir(base, "id/ma2c", {"init_density": "0.1"})
    assert len(_ge(base, ["pf1100/ma2c", "pf1400/ma2c"]).groups) == 2
    ge = _ge(base, ["pf1100/ma2c", "pf1400/ma2c", "id/ma2c"], share_demand=True)
    assert [len(g) for g in ge.groups] == [2, 1] and ge.groups[0][1].env.peak_flow1 == 1400


def test_a_level_key_outside_the_scenario_is_refused_naming_entry_and_key(tmp_path, no_device):  # noqa: F811
    base = str(tmp_path)
    _dir(base, "ma2c")
    with pytest.raises(ValueError, match=r"ma2c: 'flow_rate' is not a demand key") as e:
        _ge(base, ["ma2c"], [{"peak_flow1": "1400"}, {"flow_rate": "450"}])
    assert os.path.join(base, "ma2c") in str(e.value)
    with pytest.raises(ValueError, match="init_density"):
        _ge(base, ["ma2c"], [{"init_density": "0.1"}])
    with pytest.raises(ValueError, match="one path per level|list of 2 paths"):
        from deeprl_signal_control_b200.agents.evaluator import GroupEvaluator
        GroupEvaluator([(os.path.join(base, "ma2c"), "ma2c", base + "/")], [1], demand_levels=[{}, {}])


def test_group_replicas_count_entries_times_levels(tmp_path, no_device):  # noqa: F811
    base = str(tmp_path)
    _dir(base, "ma2c")
    with pytest.raises(ValueError, match="6 replicas"):
        _ge(base, ["ma2c"], [{"peak_flow1": str(1000 + 100 * j)} for j in range(3)], max_replicas=5)
