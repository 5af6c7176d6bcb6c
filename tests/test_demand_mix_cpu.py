"""CPU: one agent trained on a mixture of traffic demand levels (agents/train.py: train(demand_mix=...),
demand_mix_levels; agents/trainer.py: mix_level_of) — every refusal, made before any directory or device work and naming
the level, key or option; the interleaved level assignment over ranks; the per-level training rows; and the
`--train-demand` parsing of scripts/train.py next to the unchanged `--demand` of scripts/evaluate_agents.py."""
import os
import sys

import numpy as np
import pytest

from tests.test_demand_cpu import _scenario_cfg
from tests.test_evaluate_agents_cpu import _cli as _eval_cli, no_device  # noqa: F401
from tests.test_sweep_cpu import _cfg, _cli, _write

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = [{"peak_flow1": "660", "peak_flow2": "555"}, {"peak_flow1": "1100"}, {"peak_flow1": "1540", "peak_flow2": "1295"}]


def test_levels_are_the_config_edited_to_each_level():
    from deeprl_signal_control_b200.agents.train import demand_mix_levels
    mix = demand_mix_levels(_cfg("ma2c"), LEVELS, 192)
    assert mix.labels == ["peak_flow1-660_peak_flow2-555", "peak_flow1-1100", "peak_flow1-1540_peak_flow2-1295"]
    assert [(c["ENV_CONFIG"]["peak_flow1"], c["ENV_CONFIG"]["peak_flow2"]) for c in mix.configs] == \
        [("660", "555"), ("1100", "925"), ("1540", "1295")]                # an unnamed key keeps the config's value
    assert len(mix.nets) == 3 and not np.array_equal(mix.nets[0].src_due, mix.nets[2].src_due)
    assert np.array_equal(mix.nets[1].src_due, demand_mix_levels(_cfg("ma2c"), [{"peak_flow1": "1100"}], 1).nets[0].src_due)
    # a single level, even the config's own, is a valid mixture
    assert demand_mix_levels(_cfg("iqll"), [{"peak_flow2": "925"}], 7).labels == ["peak_flow2-925"]


def _refused(tmp_path, config, levels, match, n_replicas=192, **kw):
    from deeprl_signal_control_b200.agents.train import train
    base = tmp_path / "run"
    with pytest.raises(ValueError, match=match):
        train(config, str(base), "all_test", n_replicas=n_replicas, demand_mix=levels, **kw)
    assert not base.exists()


@pytest.mark.parametrize("agent", ["ma2c", "iqld"])
def test_refusals_leave_no_directory(tmp_path, no_device, agent):  # noqa: F811
    path = _write(tmp_path, "cfg", _cfg(agent))
    _refused(tmp_path, path, LEVELS, r"128 replicas .* 3 demand levels", n_replicas=128)
    _refused(tmp_path, path, [{"peak_flow1": "900"}, {"flow_rate": "450"}], r"demand level flow_rate-450: 'flow_rate'")
    _refused(tmp_path, path, [{"peak_flow1": "900"}, {"init_density": "0.1"}], "'init_density' is not a demand key")
    _refused(tmp_path, path, [{"peak_flow1": "900"}, {"peak_flow1": "900.0"}],
             "demand level peak_flow1-900.0 repeats level peak_flow1-900")
    _refused(tmp_path, path, [{"peak_flow2": "925"}, {"peak_flow1": "1100"}],            # both are the config's level
             "demand level peak_flow1-1100 repeats level peak_flow2-925")
    _refused(tmp_path, path, [], "at least one demand level")
    _refused(tmp_path, path, LEVELS[:1], "does not combine with seeds", seeds=[1, 2])


def test_a_scenario_without_demand_keys_is_refused(tmp_path, no_device):  # noqa: F811
    from deeprl_signal_control_b200.agents.train import demand_mix_levels
    c = _cfg("ma2c")
    c["ENV_CONFIG"]["scenario"] = "mini"                              # a SUMO-file scenario name without a net_file
    with pytest.raises(ValueError, match="scenario 'mini' has no demand keys"):
        demand_mix_levels(c, [{"route_file": "a.rou.xml"}], 64)


def test_a_route_file_level_must_keep_every_route(tmp_path, no_device):  # noqa: F811
    sys.path.insert(0, os.path.join(ROOT, "tests", "fixtures"))
    import make_mini_sumo
    net_file, rou = make_mini_sumo.write(str(tmp_path))
    text = open(rou).read()
    more, other = str(tmp_path / "more.rou.xml"), str(tmp_path / "other.rou.xml")
    with open(more, "w") as f:                              # the same flows at other rates
        f.write(text.replace('vehsPerHour="600"', 'vehsPerHour="900"'))
    with open(other, "w") as f:                             # one flow on another route
        f.write(text.replace('to="B_E" via="A_B"', 'to="B_SB" via="A_B"'))
    c = _cfg("ma2c")
    e = c["ENV_CONFIG"]
    e["scenario"], e["net_file"], e["route_file"], e["episode_length_sec"] = "mini", net_file, rou, "600"
    from deeprl_signal_control_b200.agents.train import demand_mix_levels
    assert demand_mix_levels(c, [{"route_file": rou}, {"route_file": more}], 2).labels == \
        ["route_file-mini.rou.xml", "route_file-more.rou.xml"]
    _refused(tmp_path, c, [{"route_file": more}, {"route_file": other}],
             r"demand level route_file-other.rou.xml: the net differs in", n_replicas=2)


@pytest.mark.parametrize("scenario", ["real_net", "small_grid"])
def test_other_scenarios_take_their_own_keys(scenario):
    from deeprl_signal_control_b200.agents.train import demand_mix_levels
    from tests.test_demand_cpu import DEMAND_VALUES
    high = DEMAND_VALUES[scenario]
    low = {k: str(int(v) // 2) for k, v in high.items()}
    mix = demand_mix_levels(_scenario_cfg(scenario), [high, low], 128)
    assert len(mix.nets) == 2 and any(not np.array_equal(getattr(mix.nets[0], f), getattr(mix.nets[1], f))
                                      for f in ("src_due", "src_phi"))
    with pytest.raises(ValueError, match="'peak_flow1' is not a demand key"):
        demand_mix_levels(_scenario_cfg(scenario), [{"peak_flow1": "1400"}], 64)


@pytest.mark.parametrize("R,W,L", [(192, 1, 3), (192, 2, 3), (384, 4, 3), (128, 2, 4), (96, 3, 2), (64, 2, 1)])
def test_ranks_hold_the_one_process_assignment(R, W, L):
    from deeprl_signal_control_b200 import dist
    from deeprl_signal_control_b200.agents.trainer import mix_level_of
    one = mix_level_of(0, R, L)
    assert np.array_equal(one, np.arange(R) % L)
    parts = []
    for rank in range(W):
        r0, r = dist.replica_range(rank, W, R)
        parts.append(mix_level_of(r0, r, L))
        assert set(parts[-1].tolist()) == set(range(L))                   # every rank holds every level
    assert np.array_equal(np.concatenate(parts), one)
    for t in range(0, R, 64):                                             # and every 64-replica tile
        assert set(one[t:t + 64].tolist()) == set(range(L))


class _Tr:
    def __init__(self, trace):
        import torch
        self.greward_trace = torch.as_tensor(trace)
        self.T_episode, self.summary_ran = trace.shape[0], None
        self.episode_rewards = [float(trace.astype(np.float32).mean(0).mean())]


def test_per_level_training_rows_are_numpy_over_the_level_columns(tmp_path):
    from deeprl_signal_control_b200.agents.train import Counter, Trainer
    rng = np.random.default_rng(3)
    L, R, T = 3, 48, 20
    trace = (rng.standard_normal((T, R)) * 5 - 40).astype(np.float32)
    levels = [("a", None), ("b", None), ("c", None)]
    d = Trainer(_Tr(trace), None, Counter(20, 10 ** 9, 0), "ma2c", False, str(tmp_path) + "/", levels=levels)
    d.episode_set(0, 20)
    rows = d.level_data
    assert [(r["step"], r["test_id"], r["demand"]) for r in rows] == [(20, -1, "a"), (20, -1, "b"), (20, -1, "c")]
    for j, r in enumerate(rows):
        cols = trace[:, np.arange(R) % L == j].astype(np.float64)           # that level's replicas
        assert r["avg_reward"] == pytest.approx(np.mean(cols), rel=1e-12, abs=0)
        assert r["std_reward"] == np.std(cols)
    assert d.data[0]["std_reward"] == np.std(trace.astype(np.float64))  # the pooled row is unchanged
    d.write_rows()
    import pandas as pd
    df = pd.read_csv(tmp_path / "train_reward_demand.csv", index_col=0)
    assert list(df.columns) == ["agent", "step", "test_id", "demand", "avg_reward", "std_reward"]
    assert list(df.demand) == ["a", "b", "c"]


def test_train_demand_cli():
    cli = _cli()
    a = cli.parse_args(["--base-dir", "b", "train", "--train-demand", "peak_flow1=660,peak_flow2=555",
                        "--train-demand", "peak_flow1=1540", "--replicas", "128"])
    assert a.train_demand == [{"peak_flow1": "660", "peak_flow2": "555"}, {"peak_flow1": "1540"}]
    assert cli.parse_args(["--base-dir", "b", "train"]).train_demand is None
    for extra in (["--seeds", "1,2"], ["--sweep", "a.ini,b.ini"], ["--sweep", "a.ini,b.ini", "--vary-demand"],
                  ["--vary-demand"]):
        with pytest.raises(SystemExit):
            cli.parse_args(["--base-dir", "b", "train", "--train-demand", "peak_flow1=660"] + extra)
    for bad in ("peak_flow1", "=3", "peak_flow1=1,peak_flow1=2", ","):
        with pytest.raises(SystemExit):
            cli.parse_args(["--base-dir", "b", "train", "--train-demand", bad])
    with pytest.raises(SystemExit):                                            # one level twice
        cli.parse_args(["--base-dir", "b", "train", "--train-demand", "peak_flow1=7", "--train-demand", "peak_flow1=7"])


def test_cli_messages_name_their_option(capsys):
    for cli, argv, opt in ((_cli(), ["--base-dir", "b", "train"], "--train-demand"),
                           (_eval_cli(), ["--base-dir", "b", "--agents", "ma2c"], "--demand")):
        for bad, msg in (("peak_flow1", "%s takes KEY=VALUE pairs separated by ',' (got 'peak_flow1')"),
                         ("a=1,a=2", "%s 'a=1,a=2' names a twice"), (",", "%s ',' names no key")):
            with pytest.raises(SystemExit):
                cli.parse_args(argv + [opt, bad])
            assert capsys.readouterr().err.rstrip().endswith("error: " + msg % opt)


def test_evaluate_agents_keeps_its_names():
    from deeprl_signal_control_b200 import envs
    cli = _eval_cli()
    assert cli.parse_demand is envs.parse_demand and cli.demand_label is envs.demand_label
    assert cli.parse_demand("peak_flow1=1400, peak_flow2=1180") == {"peak_flow1": "1400", "peak_flow2": "1180"}
    assert cli.demand_label({"route_file": "/x/y/more.rou.xml", "a": "1"}) == "route_file-more.rou.xml_a-1"
    with pytest.raises(ValueError) as e:
        cli.parse_demand("x")
    assert str(e.value) == "--demand takes KEY=VALUE pairs separated by ',' (got 'x')"
