"""CPU: the members driver builds the env and the learner before it makes any member directory, for A2C populations
and sweeps as for IQL members, so that a learner that refuses to build leaves nothing behind."""
import configparser
import os

import pytest

from tests.test_train_driver_gpu import _ini


def _cfg(lr_init=None):
    c = configparser.ConfigParser()
    c.read_string(_ini("ma2c", 120, 240))
    if lr_init is not None:
        c["MODEL_CONFIG"]["lr_init"] = lr_init
    return c


def test_a2c_learner_refusal_leaves_no_member_directory(tmp_path, monkeypatch):
    import torch
    from deeprl_signal_control_b200.agents.train import train_population, train_sweep
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    base = str(tmp_path / "b")
    with pytest.raises(RuntimeError, match="BatchedA2C needs a CUDA device"):
        train_population(_cfg(), base, [1, 2], n_replicas=64)
    assert not os.path.exists(base)
    with pytest.raises(RuntimeError, match="BatchedA2C needs a CUDA device"):
        train_sweep({"a": _cfg(), "b": _cfg("1e-3")}, base, n_replicas=64)
    assert not os.path.exists(base)
