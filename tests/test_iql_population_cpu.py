"""CPU: the host side of IQL members (train_iql_population, train_iql_sweep, BatchedIQL with seeds) — every refusal
before any directory or device allocation, member directories, each member's schedules and Adam step sizes against its
solo run's, and the command line."""
import configparser
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

from tests.test_train_driver_gpu import _ini


def _write(tmp_path, name, agent, **model):
    text = _ini(agent, 120, 240)
    for key, val in model.items():
        text = "\n".join(("%s = %s" % (key, val)) if line.startswith(key + " =") else line for line in text.split("\n"))
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def test_driver_refusals_leave_no_directory(tmp_path, monkeypatch):
    from deeprl_signal_control_b200.agents.train import train_iql_population, train_iql_sweep
    base = str(tmp_path / "b")
    iqld = _write(tmp_path, "iqld.ini", "iqld")
    with pytest.raises(ValueError, match="IQL agent"):
        train_iql_population(_write(tmp_path, "ma2c.ini", "ma2c"), base, [1, 2], n_replicas=64)
    with pytest.raises(ValueError, match="IQL agent"):
        train_iql_sweep([_write(tmp_path, "a.ini", "ia2c"), _write(tmp_path, "b.ini", "ia2c", gamma=0.9)], base)
    with pytest.raises(ValueError, match="distinct"):
        train_iql_population(iqld, base, [1, 1], n_replicas=64)
    with pytest.raises(ValueError, match="at most 64"):
        train_iql_population(iqld, base, list(range(65)), n_replicas=4)
    for key, val in (("batch_size", 40), ("buffer_size", 500), ("num_fc", 64), ("num_h", 32), ("coop_gamma", 0.5)):
        other = _write(tmp_path, "x_%s.ini" % key, "iqld", **{key: val})
        with pytest.raises(ValueError, match=r"\] %s differs between .*iqld.ini.*x_%s.ini" % (key, key)):
            train_iql_sweep([iqld, other], base)
    import torch
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda dev=None: (1 << 20, 1 << 20))
    with pytest.raises(ValueError, match="replay rings need"):
        train_iql_population(iqld, base, [1, 2], n_replicas=64)
    with pytest.raises(ValueError, match="replay rings need"):
        train_iql_sweep([iqld, _write(tmp_path, "g.ini", "iqld", gamma=0.9)], base, n_replicas=64)
    assert not os.path.exists(base)


def test_learner_refusals():
    from deeprl_signal_control_b200.agents.layout import QLayout
    from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL, check_members
    cp = configparser.ConfigParser(); cp.read_string(_ini("iqld", 120, 240))
    mc = cp["MODEL_CONFIG"]
    lay = QLayout("lr", [4, 4], [2, 2], [0, 0], np.array([0, 4, 8]), 8)
    with pytest.raises(ValueError, match="process group"):
        BatchedIQL(lay, 64, mc, "lr", seeds=[1, 2], pg=object())
    with pytest.raises(ValueError, match="distinct"):
        BatchedIQL(lay, 64, mc, "lr", seeds=[1, 1])
    with pytest.raises(ValueError, match="at most 64"):
        BatchedIQL(lay, 64, mc, "lr", seeds=list(range(65)))
    assert check_members(None, None, mc, object()) == 1                  # the solo learner keeps its process group
    assert check_members([1, 1], [mc, mc], mc, None) == 2                 # a sweep's seeds may repeat
    c2 = configparser.ConfigParser(); c2.read_string(_ini("iqld", 120, 240).replace("batch_size = 20", "batch_size = 40"))
    with pytest.raises(ValueError, match="batch_size differs"):
        check_members([1, 2], [mc, c2["MODEL_CONFIG"]], mc, None)


def test_member_dirs():
    from deeprl_signal_control_b200.agents.train import member_dir, sweep_dir
    assert member_dir("/x/b", 12, "iqld") == os.path.join("/x/b", "seed12", "iqld")
    assert sweep_dir("/x/b", "a", "iqll") == os.path.join("/x/b", "a", "iqll")


def test_member_schedulers_are_the_solo_runs():
    from deeprl_signal_control_b200.agents.models import iql_schedulers
    from deeprl_signal_control_b200.agents.train import member_schedulers
    cfgs = []
    for text in (_ini("iqld", 120, 240),
                 _ini("iqld", 120, 240, eps_decay="constant").replace("lr_init = 1e-4", "lr_init = 3e-4"),
                 _ini("iqld", 120, 240).replace("lr_decay = constant", "lr_decay = linear\nlr_min = 1e-5")):
        c = configparser.ConfigParser(); c.read_string(text)
        cfgs.append(c["MODEL_CONFIG"])
    lr_s, eps_s = member_schedulers(cfgs, 1000)
    assert len(lr_s) == len(eps_s) == 3
    one = member_schedulers(cfgs[:1], 1000)
    assert not isinstance(one[0], list)
    for k, c in enumerate(cfgs):
        lr_ref, eps_ref = iql_schedulers(c, 1000)
        for _ in range(30):                              # as the trainer calls them: ε per step, lr per update
            for _ in range(20):
                assert eps_s[k].get(1) == eps_ref.get(1)
            assert lr_s[k].get(20) == lr_ref.get(20)


def test_member_lr_t_is_td_rounds_value():
    from deeprl_signal_control_b200.agents.learner_iql import member_lr_t
    lrs = [1e-4, 5e-4, 3.3e-4, 1e-3]
    for t in range(1, 200):
        got = member_lr_t(lrs, t)
        assert got.dtype == np.float32
        for k, lr in enumerate(lrs):
            solo = lr * np.sqrt(1.0 - 0.999 ** t) / (1.0 - 0.9 ** t)    # td_round's float, rounded by its call
            assert got[k] == np.float32(C.c_float(solo).value)


def _cli():
    spec = importlib.util.spec_from_file_location("train_iql_members", os.path.join(
        os.path.dirname(__file__), "..", "scripts", "train_iql_members.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    return cli


def test_cli_parses_and_refuses_torchrun(monkeypatch):
    cli = _cli()
    a = cli.parse_args(["--base-dir", "b", "--config-dir", "c.ini", "--seeds", "12,13", "--replicas", "300"])
    assert a.seeds == [12, 13] and a.sweep is None and a.replicas == 300 and a.test_mode == "no_test"
    a = cli.parse_args(["--base-dir", "b", "--sweep", "a.ini, b.ini", "--replicas", "64", "--test-mode", "all_test",
                        "--summaries"])
    assert a.sweep == ["a.ini", "b.ini"] and a.seeds is None and a.summaries
    for bad in (["--seeds", "12,12", "--config-dir", "c.ini"], ["--seeds", "12"], ["--sweep", "a.ini", "--seeds", "1"],
                ["--sweep", "a.ini", "--config-dir", "c.ini"], []):
        with pytest.raises(SystemExit):
            cli.parse_args(["--base-dir", "b", "--replicas", "64"] + bad)
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit, match="torchrun"):
        cli.main(["--base-dir", "b", "--config-dir", "c.ini", "--seeds", "12,13", "--replicas", "64"])
