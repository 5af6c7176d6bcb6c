"""Deterministic A2C training without a GPU: every refusal of `deterministic=True` (raised before any device work or
directory), the CLI flag passed through to each training entry point, and the new C entry point bound from the header."""
import configparser
import ctypes as C
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from layout_envelope import EDGES, net_tables, scenario_layout, synthetic_layout  # noqa: E402

from deeprl_signal_control_b200.agents import learner as lrn  # noqa: E402


def _grid_ma2c():
    return scenario_layout(net_tables("large_grid", "ma2c"), "ma2c")


def _refused(layout, match, **kw):
    with pytest.raises(ValueError, match=match):
        lrn.BatchedA2C(layout, 64, 4, chunk=64, deterministic=True, **kw)


def test_lean_layouts_are_accepted_by_the_check():
    for scen, agent, fw in (("large_grid", "ma2c", 128), ("large_grid", "ia2c", 128), ("real_net", "ma2c", 128),
                            ("real_net", "ia2c", 128)):
        lay = scenario_layout(net_tables(scen, agent), agent, fw=fw)
        assert lrn.deterministic_refusal(lrn.learner_paths(lay), True) is None


def test_use_tc_false_is_refused():
    _refused(_grid_ma2c(), "use_tc=False", use_tc=False)


def test_store_update_layout_is_refused():
    kw, _, update = EDGES["wave32_wait"]
    assert update == "store"
    _refused(synthetic_layout(**kw), "'store'")


def test_recompute_update_layout_is_refused():
    lay = scenario_layout(net_tables("large_grid", "ia2c"), "ia2c", fw=64)
    assert lrn.learner_paths(lay).update == "recompute"
    _refused(lay, "'recompute'")


def test_activation_store_off_is_refused():
    _refused(_grid_ma2c(), "activation store", store_acts=False)


def test_bptt_heads_off_is_refused(monkeypatch):
    monkeypatch.setenv("TSC_BPTT_HEADS", "0")
    _refused(_grid_ma2c(), "TSC_BPTT_HEADS=0")


def test_dx_library_is_refused(monkeypatch):
    monkeypatch.setenv("TSC_DX_LIBRARY", "1")
    _refused(_grid_ma2c(), "TSC_DX_LIBRARY=1")


MA2C_INI = """[ENV_CONFIG]
agent = ma2c
seed = 12
scenario = atsc_large_grid
[MODEL_CONFIG]
batch_size = 40
[TRAIN_CONFIG]
total_step = 720
test_interval = 720
log_interval = 720
"""


def test_fc_policy_is_refused_before_any_directory(tmp_path):
    from deeprl_signal_control_b200.agents import train as drv
    cp = configparser.ConfigParser()
    cp.read_string(MA2C_INI)
    with pytest.raises(ValueError, match="policy='fc'"):
        drv.train(cp, str(tmp_path / "run"), policy="fc", deterministic=True)
    with pytest.raises(ValueError, match="policy='fc'"):
        drv.train(cp, str(tmp_path / "pop"), policy="fc", seeds=[12, 13], deterministic=True)
    assert not os.listdir(tmp_path)


def test_fc_policy_model_is_refused():
    from deeprl_signal_control_b200.agents.models import IA2C
    cp = configparser.ConfigParser()
    cp.read_string(MA2C_INI)
    with pytest.raises(ValueError, match="policy='fc'"):
        IA2C([4], [2], [1], 0, cp["MODEL_CONFIG"], policy="fc", deterministic=True)


def _cli():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    import train as cli
    return cli


class _Out:
    final_step = episode_sets = env_samples = 0
    wall_sec = 0.0
    seeds, names, rank = [12, 13], ["a", "b"], 0


def test_cli_passes_deterministic_to_every_entry_point(monkeypatch):
    from deeprl_signal_control_b200.agents import train as drv
    cli = _cli()
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    seen = []
    monkeypatch.setattr(drv, "train", lambda *a, **kw: seen.append(("train", kw)) or _Out())
    monkeypatch.setattr(drv, "train_sweep", lambda *a, **kw: seen.append(("sweep", kw)) or _Out())
    base = ["--base-dir", "b", "train", "--replicas", "128"]
    assert cli.parse_args(base).deterministic is False
    cli.main(base + ["--deterministic", "--summaries"])
    cli.main(base + ["--deterministic", "--seeds", "12,13"])
    cli.main(base + ["--deterministic", "--sweep", "a.ini,b.ini"])
    cli.main(base)
    assert [(w, kw["deterministic"]) for w, kw in seen] == [("train", True), ("train", True), ("sweep", True),
                                                            ("train", False)]
    assert seen[0][1]["summaries"] and seen[1][1]["seeds"] == [12, 13]


def test_setter_is_bound_from_the_header():
    from deeprl_signal_control_b200 import _lib
    restype, argtypes = _lib._prototypes()["tscl_set_deterministic"]
    assert restype is C.c_int and argtypes == [C.c_void_p, C.c_int32, C.c_int32]
