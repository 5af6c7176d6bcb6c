"""CPU: the host side of population training — seed-list parsing, member directories, each member's episode seeds
against its solo run's, and every combination a population rejects before any device work."""
import configparser
import os

import numpy as np
import pytest

from tests.test_train_driver_gpu import _ini


def test_parse_seeds_and_member_dirs():
    from deeprl_signal_control_b200.agents.train import member_dir, parse_seeds
    assert parse_seeds("12,13,14,15") == [12, 13, 14, 15]
    assert parse_seeds(" 7, 3 ") == [7, 3]
    for bad in ("", "12,12", "a,b", "-1,2"):
        with pytest.raises(ValueError):
            parse_seeds(bad)
    assert member_dir("/x/base", 12, "ma2c") == os.path.join("/x/base", "seed12", "ma2c")


def test_cli_parses_seeds_and_refuses_torchrun(monkeypatch):
    import importlib.util
    spec = importlib.util.spec_from_file_location("train_cli", os.path.join(os.path.dirname(__file__), "..", "scripts",
                                                                           "train.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    a = cli.parse_args(["--base-dir", "b", "train", "--seeds", "12,13", "--replicas", "512"])
    assert a.seeds == [12, 13] and a.replicas == 512
    assert cli.parse_args(["--base-dir", "b", "train"]).seeds is None
    with pytest.raises(SystemExit):
        cli.parse_args(["--base-dir", "b", "train", "--seeds", "12,12"])
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit, match="torchrun"):
        cli.main(["--base-dir", "b", "train", "--seeds", "12,13", "--replicas", "64"])


def test_member_episode_seeds_are_the_solo_runs():
    from deeprl_signal_control_b200.agents.trainer import member_episode_seeds
    from deeprl_signal_control_b200.dist import episode_seeds
    seeds, Rm = [12, 13, 40], 512
    for ep in range(3):
        got = member_episode_seeds(seeds, ep, Rm)
        assert got.dtype == np.uint64 and got.shape == (len(seeds) * Rm,)
        for k, s in enumerate(seeds):
            # the solo run: one process, replica0 = 0, total_replicas = n_replicas (BatchedTrainer.start_episode)
            assert np.array_equal(got[k * Rm:(k + 1) * Rm], episode_seeds(s, ep, 0, Rm, max(Rm, Rm)))


def test_learner_rejections():
    from deeprl_signal_control_b200.agents.learner import check_population
    assert check_population(None, 5, 100, 1024, None) == [5]
    assert check_population([3, 4], 0, 512, 1024, None) == [3, 4]
    assert check_population([3], 0, 100, 1024, None) == [3]            # one member: the solo learner
    with pytest.raises(ValueError, match="multiple of 64"):
        check_population([3, 4], 0, 500, 1024, None)
    with pytest.raises(ValueError, match="chunk"):
        check_population([3, 4], 0, 640, 256, None)
    with pytest.raises(ValueError, match="distinct"):
        check_population([3, 3], 0, 512, 1024, None)
    with pytest.raises(ValueError, match="process group"):
        check_population([3, 4], 0, 512, 1024, object())


def _cfg(agent):
    c = configparser.ConfigParser()
    c.read_string(_ini(agent, 120, 240))
    return c


def test_driver_rejections(tmp_path):
    from deeprl_signal_control_b200.agents.train import train
    base = str(tmp_path / "b")
    with pytest.raises(ValueError, match="A2C agent"):
        train(_cfg("iqld"), base, n_replicas=64, seeds=[1, 2])
    with pytest.raises(ValueError, match="LSTM"):
        train(_cfg("ma2c"), base, n_replicas=64, policy="fc", seeds=[1, 2])
    with pytest.raises(ValueError, match="process_group"):
        train(_cfg("ma2c"), base, n_replicas=64, process_group=object(), seeds=[1, 2])
    with pytest.raises(ValueError, match="multiple of 64"):
        train(_cfg("ma2c"), base, n_replicas=100, seeds=[1, 2])
    with pytest.raises(ValueError, match="distinct"):
        train(_cfg("ma2c"), base, n_replicas=64, seeds=[1, 1])
    assert not os.path.exists(base)                                   # rejected before any directory is made


def test_models_reject_fc_population():
    from deeprl_signal_control_b200.agents.models import IA2C
    c = _cfg("ia2c")
    with pytest.raises(ValueError, match="LSTM"):
        IA2C([10], [2], [0], 0, c["MODEL_CONFIG"], n_replicas=64, policy="fc", seeds=[1, 2])
