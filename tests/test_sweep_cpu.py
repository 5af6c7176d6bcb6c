"""CPU: the host side of sweep training — which config keys the members may set for themselves and every refusal
(naming the key and both configs), member names and directories, each member's lr / entropy schedule against its solo
run's, the learner's sweep check, the `--sweep` CLI and the new native entry points."""
import configparser
import os

import pytest

from tests.test_train_driver_gpu import _ini

SWEEP_VALUES = {          # a value other than the base config's for every key a member may set
    ("ENV_CONFIG", "seed"): "13", ("ENV_CONFIG", "coop_gamma"): "0.75",
    ("MODEL_CONFIG", "lr_init"): "1e-3", ("MODEL_CONFIG", "lr_decay"): "linear", ("MODEL_CONFIG", "lr_min"): "1e-5",
    ("MODEL_CONFIG", "entropy_coef_init"): "0.02", ("MODEL_CONFIG", "entropy_decay"): "linear",
    ("MODEL_CONFIG", "entropy_coef_min"): "0.005", ("MODEL_CONFIG", "entropy_ratio"): "0.25",
    ("MODEL_CONFIG", "value_coef"): "0.25", ("MODEL_CONFIG", "max_grad_norm"): "20",
    ("MODEL_CONFIG", "rmsp_alpha"): "0.9", ("MODEL_CONFIG", "rmsp_epsilon"): "1e-4", ("MODEL_CONFIG", "gamma"): "0.95",
    ("MODEL_CONFIG", "reward_norm"): "3000.0", ("MODEL_CONFIG", "reward_clip"): "0"}


def _cfg(agent="ma2c", changes=None):
    c = configparser.ConfigParser()
    c.read_string(_ini(agent, 120, 240))
    for (sec, key), v in (changes or {}).items():
        c[sec][key] = v
    return c


def _write(tmp_path, name, cfg):
    p = tmp_path / ("%s.ini" % name)
    with open(p, "w") as f:
        cfg.write(f)
    return str(p)


def test_sweep_config_keys_are_the_issued_set():
    from deeprl_signal_control_b200.agents.train import SWEEP_CONFIG_KEYS
    assert {(s, k) for s, keys in SWEEP_CONFIG_KEYS.items() for k in keys} == set(SWEEP_VALUES)


@pytest.mark.parametrize("key", sorted(SWEEP_VALUES))
def test_each_sweep_key_may_differ(key):
    from deeprl_signal_control_b200.agents.train import sweep_members
    items = sweep_members({"a": _cfg(), "b": _cfg(changes={key: SWEEP_VALUES[key]})})
    assert [n for n, _, _ in items] == ["a", "b"]
    assert items[1][1][key[0]][key[1]] == SWEEP_VALUES[key]


@pytest.mark.parametrize("sec,key,value", [("MODEL_CONFIG", "num_lstm", "32"), ("MODEL_CONFIG", "batch_size", "60"),
                                           ("TRAIN_CONFIG", "total_step", "240"),
                                           ("ENV_CONFIG", "test_seeds", "10000"),
                                           ("ENV_CONFIG", "scenario", "real_net"),
                                           ("ENV_CONFIG", "peak_flow1", "1000")])
def test_other_keys_must_agree_and_the_error_names_key_and_files(tmp_path, sec, key, value):
    from deeprl_signal_control_b200.agents.train import sweep_members
    a, b = _write(tmp_path, "lr_a", _cfg()), _write(tmp_path, "lr_b", _cfg(changes={(sec, key): value}))
    with pytest.raises(ValueError, match=key) as e:
        sweep_members([a, b])
    assert a in str(e.value) and b in str(e.value)


def test_numbers_compare_by_value():
    from deeprl_signal_control_b200.agents.train import sweep_members
    sweep_members({"a": _cfg(changes={("MODEL_CONFIG", "num_lstm"): "64.0", ("MODEL_CONFIG", "lr_init"): "1e-3"}),
                   "b": _cfg()})


def test_refusals():
    from deeprl_signal_control_b200.agents.train import sweep_members
    with pytest.raises(ValueError, match="coop_gamma"):            # ia2c does not read coop_gamma
        sweep_members({"a": _cfg("ia2c"), "b": _cfg("ia2c", {("ENV_CONFIG", "coop_gamma"): "0.75"})})
    with pytest.raises(ValueError, match="identical"):
        sweep_members({"a": _cfg(), "b": _cfg(changes={("MODEL_CONFIG", "lr_init"): "1e-3"}), "c": _cfg()})
    with pytest.raises(ValueError, match="identical"):             # equal values written differently
        sweep_members({"a": _cfg(), "b": _cfg(changes={("MODEL_CONFIG", "lr_init"): "0.0005"})})
    with pytest.raises(ValueError, match="at least one"):
        sweep_members({})
    # the same seed twice is a sweep at one seed
    sweep_members({"a": _cfg(), "b": _cfg(changes={("MODEL_CONFIG", "gamma"): "0.9"})})


def test_duplicate_member_names_are_refused(tmp_path):
    from deeprl_signal_control_b200.agents.train import sweep_members
    (tmp_path / "x").mkdir()
    a = _write(tmp_path, "lr", _cfg())
    b = str(tmp_path / "x" / "lr.ini")
    with open(b, "w") as f:
        _cfg(changes={("MODEL_CONFIG", "lr_init"): "1e-3"}).write(f)
    with pytest.raises(ValueError, match="distinct"):
        sweep_members([a, b])


def test_driver_refusals_leave_no_directory(tmp_path):
    from deeprl_signal_control_b200.agents.train import train_sweep
    base = str(tmp_path / "b")
    two = lambda agent="ma2c": {"a": _cfg(agent), "b": _cfg(agent, {("MODEL_CONFIG", "lr_init"): "1e-3"})}
    with pytest.raises(ValueError, match="A2C agent"):
        train_sweep(two("iqld"), base, n_replicas=64)
    with pytest.raises(ValueError, match="LSTM"):
        train_sweep(two(), base, n_replicas=64, policy="fc")
    with pytest.raises(ValueError, match="process_group"):
        train_sweep(two(), base, n_replicas=64, process_group=object())
    with pytest.raises(ValueError, match="multiple of 64"):
        train_sweep(two(), base, n_replicas=100)
    with pytest.raises(ValueError, match="num_lstm"):
        train_sweep({"a": _cfg(), "b": _cfg(changes={("MODEL_CONFIG", "num_lstm"): "32"})}, base, n_replicas=64)
    with pytest.raises(ValueError, match="identical"):
        train_sweep({"a": _cfg(), "b": _cfg()}, base, n_replicas=64)
    with pytest.raises(ValueError, match="test_mode"):
        train_sweep(two(), base, "sometimes", n_replicas=64)
    assert not os.path.exists(base)


def test_sweep_dir():
    from deeprl_signal_control_b200.agents.train import sweep_dir
    assert sweep_dir("/x/base", "lr_hi", "ma2c") == os.path.join("/x/base", "lr_hi", "ma2c")


def test_learner_sweep_check():
    from deeprl_signal_control_b200.agents.learner import SWEEP_KEYS, check_population, check_sweep
    hp = lambda **kw: dict(dict(gamma=0.99, v_coef=0.5, max_grad_norm=40.0, alpha=0.99, eps=1e-5, reward_norm=2000.0,
                                reward_clip=2.0), **kw)
    seeds, hps = check_sweep([12, 12], [hp(), hp(gamma=0.9)], 512, 1024, None)       # seeds may repeat
    assert seeds == [12, 12] and hps[1]["gamma"] == 0.9 and set(hps[0]) == set(SWEEP_KEYS)
    assert check_sweep([12], [hp(reward_norm=None)], 100, 1024, None)[1][0]["reward_norm"] == 0.0   # one member: solo
    with pytest.raises(ValueError, match="multiple of 64"):
        check_sweep([1, 2], [hp(), hp()], 500, 1024, None)
    with pytest.raises(ValueError, match="chunk"):
        check_sweep([1, 2], [hp(), hp()], 640, 256, None)
    with pytest.raises(ValueError, match="process group"):
        check_sweep([1, 2], [hp(), hp()], 512, 1024, object())
    with pytest.raises(ValueError, match="one seed per member"):
        check_sweep([1], [hp(), hp()], 512, 1024, None)
    with pytest.raises(ValueError, match="exactly"):
        check_sweep([1, 2], [hp(), dict(hp(), lr=1e-3)], 512, 1024, None)
    with pytest.raises(ValueError, match="distinct"):                               # a population's seeds still are
        check_population([3, 3], 0, 512, 1024, None)


def test_member_schedules_equal_the_solo_schedulers():
    from deeprl_signal_control_b200.agents.models import a2c_hparams, a2c_schedulers
    from deeprl_signal_control_b200.agents.trainer import schedule_values
    from deeprl_signal_control_b200.agents.utils import Scheduler
    T, total = 120, 3600
    cfgs = [_cfg(), _cfg(changes={("MODEL_CONFIG", "lr_decay"): "linear", ("MODEL_CONFIG", "lr_min"): "1e-5",
                            ("MODEL_CONFIG", "lr_init"): "1e-3"}),
            _cfg(changes={("MODEL_CONFIG", "entropy_decay"): "linear", ("MODEL_CONFIG", "entropy_coef_init"): "0.05",
                    ("MODEL_CONFIG", "entropy_coef_min"): "0.001", ("MODEL_CONFIG", "entropy_ratio"): "0.25"})]
    lrs, betas = (list(s) for s in zip(*(a2c_schedulers(c["MODEL_CONFIG"], total) for c in cfgs)))
    # the solo runs' schedulers, written out as the reference's agents/models.py:53-69 builds them
    solo_lr = [Scheduler(5e-4, decay="constant"), Scheduler(1e-3, 1e-5, total, decay="linear"),
               Scheduler(5e-4, decay="constant")]
    solo_beta = [Scheduler(0.01, decay="constant"), Scheduler(0.01, decay="constant"),
                 Scheduler(0.05, 0.001, total * 0.25, decay="linear")]
    for _ in range(total // T + 2):
        assert schedule_values(lrs, T) == [s.get(T) for s in solo_lr]
        assert schedule_values(betas, T) == [s.get(T) for s in solo_beta]
    assert schedule_values(0.5, T) == 0.5 and schedule_values([0.5, 0.25], T) == [0.5, 0.25]
    assert a2c_hparams(cfgs[0]["MODEL_CONFIG"]) == dict(gamma=0.99, v_coef=0.5, max_grad_norm=40.0, alpha=0.99,
                                                          eps=1e-5, reward_norm=2000.0, reward_clip=2.0)


def _cli():
    import importlib.util
    spec = importlib.util.spec_from_file_location("train_cli", os.path.join(os.path.dirname(__file__), "..", "scripts",
                                                                           "train.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    return cli


def test_cli_parses_sweep_and_refuses_seeds_and_torchrun(monkeypatch):
    cli = _cli()
    a = cli.parse_args(["--base-dir", "b", "train", "--sweep", "x/a.ini, x/b.ini", "--replicas", "512"])
    assert a.sweep == ["x/a.ini", "x/b.ini"] and a.replicas == 512 and a.seeds is None
    assert cli.parse_args(["--base-dir", "b", "train"]).sweep is None
    with pytest.raises(SystemExit):
        cli.parse_args(["--base-dir", "b", "train", "--sweep", "a.ini,b.ini", "--seeds", "12,13"])
    with pytest.raises(SystemExit):
        cli.parse_args(["--base-dir", "b", "train", "--sweep", ","])
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit, match="torchrun"):
        cli.main(["--base-dir", "b", "train", "--sweep", "a.ini,b.ini", "--replicas", "64"])


def test_sweep_abi_is_exported():
    import ctypes as C
    from deeprl_signal_control_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build_native()
    lib = C.CDLL(_lib.LIB_PATH)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    headers = open(os.path.join(root, "include", "tsc.h")).read() + open(os.path.join(root, "include",
                                                                                       "tsc_learn.h")).read()
    for name in ("tsc_set_replica_coop_gamma", "tscl_returns_g", "tscl_device_transition_g"):
        assert hasattr(lib, name) and name in _lib.SYMBOLS and (name + "(") in headers
