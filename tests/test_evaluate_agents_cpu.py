"""CPU: the host side of evaluating several agents in one process (agents/evaluator.py:GroupEvaluator,
scripts/evaluate_agents.py) — which entries share a simulator, where each entry writes, the command line's defaults,
the a2c refusal, and a missing checkpoint skipped with an error before any device work while the other entries stay."""
import configparser
import importlib.util
import logging
import os

import pytest

from tests.test_train_driver_gpu import A2C_MODEL, GRID, IQL_MODEL, TRAIN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cli():
    spec = importlib.util.spec_from_file_location("evaluate_agents", os.path.join(ROOT, "scripts", "evaluate_agents.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _dir(base, entry, changes=None, checkpoint=True):
    agent = os.path.basename(entry)
    c = configparser.ConfigParser()
    model = A2C_MODEL if agent in ("ia2c", "ma2c", "greedy", "a2c") else IQL_MODEL
    c.read_string(model + TRAIN % (120, 120) + GRID % (agent, "10000,20000"))
    for k, v in (changes or {}).items():
        c["ENV_CONFIG"][k] = v
    d = os.path.join(base, entry)
    os.makedirs(os.path.join(d, "data"))
    os.makedirs(os.path.join(d, "model"))
    with open(os.path.join(d, "data", "config.ini"), "w") as f:
        c.write(f)
    if checkpoint:
        open(os.path.join(d, "model", "checkpoint-120.npz"), "wb").close()
    return d


@pytest.fixture
def no_device(monkeypatch):
    """Any simulator or CUDA initialisation fails the test."""
    import torch
    from deeprl_signal_control_b200 import sim

    def refuse(*a, **k):
        raise AssertionError("device work before the checks")
    monkeypatch.setattr(sim.BatchedSim, "__init__", refuse)
    monkeypatch.setattr(torch.cuda, "init", refuse)


def _ge(base, entries, **kw):
    from deeprl_signal_control_b200.agents.evaluator import GroupEvaluator, entry_model
    return GroupEvaluator([(os.path.join(base, e), entry_model(os.path.basename(e)), str(base) + "/") for e in entries],
                          [10000, 20000], **kw)


def _labels(ge):
    return [[os.path.relpath(e.agent_dir, ge.base) for e in g] for g in ge.groups]


def test_simulator_grouping(tmp_path, no_device):
    base = str(tmp_path)
    spec = [("greedy", {}), ("ia2c", {}), ("iqll", {}), ("iqld", {}), ("ma2c", {}), ("s13/ma2c", {"seed": "13"}),
            ("cg75/ma2c", {"coop_gamma": "0.75"}), ("cg1/ma2c", {"coop_gamma": "1.0"}),
            ("pf/ma2c", {"peak_flow1": "1000"}), ("pf/ia2c", {"peak_flow1": "1000"}), ("s20/iqld", {"seed": "20"})]
    for e, ch in spec:
        _dir(base, e, ch)
    ge = _ge(base, [e for e, _ in spec])
    ge.base = base
    # ia2c / iqll / iqld share (seed aside); ma2c members differing in seed or coop_gamma share; a differing peak_flow1
    # splits; greedy has no wait block and stays apart
    assert _labels(ge) == [["greedy"], ["ia2c", "iqll", "iqld", "s20/iqld"], ["ma2c", "s13/ma2c", "cg75/ma2c", "cg1/ma2c"],
                           ["pf/ma2c"], ["pf/ia2c"]]
    assert not ge.skipped
    assert [e.seed for e in ge.groups[2]] == [12, 13, 12, 12]


def test_ia2c_coop_gamma_is_part_of_its_simulator(tmp_path, no_device):
    """coop_gamma is left out of the comparison only for ma2c, whose members take it per replica."""
    from deeprl_signal_control_b200.agents.evaluator import sim_key
    base = str(tmp_path)
    _dir(base, "ia2c")
    _dir(base, "cg/ia2c", {"coop_gamma": "0.5"})
    ge = _ge(base, ["ia2c", "cg/ia2c"])
    a, b = (e.env for e in ge.entries)
    assert (sim_key(a) == sim_key(b)) == (a._params.as_c().coop_gamma == b._params.as_c().coop_gamma)


def test_output_paths_and_cli_defaults(tmp_path):
    cli = _cli()
    a = cli.parse_args(["--base-dir", "B", "--agents", "ma2c"])
    assert a.evaluation_policy_type == "default" and a.policy == "lstm"
    assert [int(s) for s in a.evaluation_seeds.split(",")] == list(range(10000, 100001, 10000))
    ent = cli.entries("B", "greedy,ma2c,seed12/ma2c,seed13/ma2c,lr_hi/ma2c/")
    assert ent == [("greedy", "B/greedy", "B/eva_data/"), ("ma2c", "B/ma2c", "B/eva_data/"),
                   ("seed12/ma2c", "B/seed12/ma2c", "B/eva_data/seed12/"),
                   ("seed13/ma2c", "B/seed13/ma2c", "B/eva_data/seed13/"),
                   ("lr_hi/ma2c", "B/lr_hi/ma2c", "B/eva_data/lr_hi/")]
    files = [os.path.join(out, "large_grid_%s_control.csv" % os.path.basename(lab)) for lab, _, out in ent]
    assert len(set(files)) == len(files)                                   # no two entries write the same file
    with pytest.raises(SystemExit):
        cli.entries("B", "ma2c,ma2c")
    from deeprl_signal_control_b200.agents.evaluator import entry_model
    assert [entry_model(a) for a in ("greedy", "ia2c", "ma2c", "a2c", "iqld", "iqll", "iql")] == \
        ["greedy", "ia2c", "ma2c", "a2c", "dqn", "lr", "lr"]


def test_a2c_is_refused_naming_the_entry(tmp_path, no_device):
    base = str(tmp_path)
    _dir(base, "ma2c")
    _dir(base, "p/a2c")
    with pytest.raises(ValueError, match="p/a2c"):
        _ge(base, ["ma2c", "p/a2c"])


def test_missing_checkpoint_is_skipped_before_device_work(tmp_path, no_device, caplog):
    base = str(tmp_path)
    _dir(base, "greedy", checkpoint=False)                   # greedy needs no checkpoint
    _dir(base, "ma2c")
    _dir(base, "s13/ma2c", {"seed": "13"}, checkpoint=False)
    _dir(base, "ia2c")
    with caplog.at_level(logging.ERROR):
        ge = _ge(base, ["greedy", "ma2c", "s13/ma2c", "ia2c", "nothere/iqll"])
    ge.base = base
    assert [os.path.relpath(e.agent_dir, base) for e in ge.skipped] == ["s13/ma2c", "nothere/iqll"]
    assert "s13/ma2c" in caplog.text and "checkpoint" in caplog.text and "nothere/iqll" in caplog.text
    assert _labels(ge) == [["greedy"], ["ma2c"], ["ia2c"]]


def test_combined_replicas_must_fit(tmp_path, no_device):
    base = str(tmp_path)
    _dir(base, "ma2c")
    _dir(base, "s13/ma2c", {"seed": "13"})
    with pytest.raises(ValueError, match="s13/ma2c"):
        _ge(base, ["ma2c", "s13/ma2c"], max_replicas=3)
