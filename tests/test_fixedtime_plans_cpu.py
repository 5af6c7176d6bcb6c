"""CPU: the host side of fixed-time plan tuning (envs/fixedtime.py:write_tll, agents/tune_fixedtime.py).

- write_tll -> read_signal_programs -> program_tables gives back the tables, on the grid, Monaco, the small grid and
  the mini SUMO net and on random plans; on the mini SUMO net the env's green phase list (read_tls_programs) is kept.
- The search space on the four nets: the searched phases are the green ones, their bounds hold the shipped duration,
  and the transition phases keep theirs.
- The cross-entropy search on a synthetic separable objective: integer samples within bounds, offsets in [0, C_i),
  candidate 0 the incumbent, an incumbent that never gets worse, the same plans for the same rng_seed, an interior
  optimum of the small grid's plan reached within 30 generations of 128 candidates, and the circular mean across the
  0 / 1 wrap.
- Every refusal, before any device work, and the command line of scripts/tune_fixedtime.py.
"""
import configparser
import os
import sys

import numpy as np
import pytest

from tests.test_evaluate_agents_cpu import no_device  # noqa: F401
from tests.test_evaluator_cpu import GRID_INI
from tests.test_fixedtime_cpu import _nets_and_programs
from tests.test_pressure_cpu import _script

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "fixtures"))
NETS = ["grid", "monaco", "small", "mini_sumo"]


def _tables(net, programs):
    from deeprl_signal_control_b200.envs.fixedtime import program_tables
    return program_tables(net.node_names, [len(net.phases[n][0]) for n in net.node_names], programs)


def _same(a, b):
    for f in ("n_phases", "dur", "open", "major", "yellow", "offset"):
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f), err_msg=f)


def _random_plan(rng, programs):
    """the programs with random whole durations (1..40 s), random offsets and, for some ids, a phase dropped"""
    out = {}
    for tl, p in programs.items():
        phases = [[int(rng.integers(1, 41)), st] for _, st in p["phases"]]
        if len(phases) > 1 and rng.random() < 0.3:
            phases = phases[:-1]
        out[tl] = {"offset": int(rng.integers(-50, 200)), "phases": phases}
    return out


@pytest.mark.parametrize("scenario", NETS)
def test_write_tll_round_trips(scenario, tmp_path):
    from deeprl_signal_control_b200.envs.fixedtime import write_tll
    from deeprl_signal_control_b200.net.sumo_ingest import read_signal_programs, read_tls_programs
    net, programs = _nets_and_programs(tmp_path)[scenario]
    path = write_tll({k: {"offset": v.get("offset", 0), "phases": v["phases"]} for k, v in programs.items()},
                     str(tmp_path / "w.tll.xml"))
    back = read_signal_programs(path)
    assert list(back) == list(programs)
    assert {p["type"] for p in back.values()} == {"static"}
    _same(_tables(net, back), _tables(net, programs))
    rng = np.random.default_rng(len(scenario))
    for _ in range(3):
        plan = _random_plan(rng, programs)
        _same(_tables(net, read_signal_programs(write_tll(plan, str(tmp_path / "r.tll.xml")))), _tables(net, plan))
    if scenario == "mini_sumo":
        net_file = str(tmp_path / "mini.net.xml")                 # written by _nets_and_programs
        assert read_tls_programs(path) == read_tls_programs(net_file) and read_tls_programs(net_file)


def test_write_tll_refuses_what_it_cannot_write(tmp_path):
    from deeprl_signal_control_b200.envs.fixedtime import write_tll
    with pytest.raises(ValueError, match="tlLogic 'a': duration '2.5' is not a whole number"):
        write_tll({"a": {"offset": 0, "phases": [["2.5", "Gr"]]}}, str(tmp_path / "x.xml"))
    with pytest.raises(ValueError, match="tlLogic 'a': type 'actuated' is not static"):
        write_tll({"a": {"type": "actuated", "offset": 0, "phases": [[5, "Gr"]]}}, str(tmp_path / "x.xml"))


@pytest.mark.parametrize("scenario", NETS)
def test_search_space(scenario, tmp_path):
    from deeprl_signal_control_b200.agents.tune_fixedtime import search_space
    net, programs = _nets_and_programs(tmp_path)[scenario]
    prog = _tables(net, programs)
    sp = search_space(prog, 5, 60)
    searched = set(zip(sp.node.tolist(), sp.phase.tolist()))
    n_trans = 0
    for i, name in enumerate(net.node_names):
        for k, (d, st) in enumerate(programs[name]["phases"]):
            green = any(c in "Gg" for c in st) and "y" not in st
            assert ((i, k) in searched) == green, (name, k, st)
            n_trans += not green
    assert sp.n_green > 0 and n_trans > 0
    assert (sp.d0 == prog.dur[sp.node, sp.phase]).all()
    assert (sp.lo <= sp.d0).all() and (sp.d0 <= sp.hi).all()
    assert (sp.lo == np.minimum(5, sp.d0)).all() and (sp.hi == np.maximum(60, sp.d0)).all()
    # a plan changes the searched durations and the offsets, and nothing else
    rng = np.random.default_rng(1)
    g = rng.integers(sp.lo, sp.hi + 1)
    off = rng.integers(0, 50, sp.n_nodes)
    p = sp.program(g, off)
    trans = np.ones(prog.dur.shape, bool)
    trans[sp.node, sp.phase] = False
    assert (p.dur[trans] == prog.dur[trans]).all() and (p.dur[sp.node, sp.phase] == g).all()
    assert (p.offset == off).all() and (p.cycle == sp.cycles(g)).all()
    for f in ("n_phases", "open", "major", "yellow"):
        assert (getattr(p, f) == getattr(prog, f)).all()
    sp2 = search_space(prog, 1, 2)                              # bounds below the shipped durations still hold d0
    assert (sp2.hi == np.maximum(2, sp2.d0)).all() and (sp2.lo == np.minimum(1, sp2.d0)).all()


def _grid_space(min_green=5, max_green=60):
    from deeprl_signal_control_b200.agents.tune_fixedtime import search_space
    from deeprl_signal_control_b200.net import large_grid
    return search_space(_tables(large_grid.build_large_grid(agent="fixedtime"), large_grid.tls_programs()),
                        min_green, max_green)


def _separable(space, target_g, target_u):
    """a separable objective with its optimum at greens target_g and offset fractions target_u (of each candidate's own
    cycles, circular distance)"""
    def f(greens, offsets):
        c = np.stack([space.cycles(g) for g in greens])
        du = np.abs(np.mod(offsets / c - target_u + 0.5, 1.0) - 0.5)
        return -(((greens - target_g) ** 2).sum(axis=1) + 400.0 * (du ** 2).sum(axis=1))
    return f


def test_cem_samples_incumbent_and_determinism():
    from deeprl_signal_control_b200.agents.tune_fixedtime import cem
    sp = _grid_space()
    rng = np.random.default_rng(3)
    tg, tu = rng.integers(sp.lo + 3, sp.hi - 3), rng.random(sp.n_nodes)
    seen = []
    f = _separable(sp, tg, tu)

    def obj(g, o):
        seen.append((g.copy(), o.copy()))
        return f(g, o)
    res = cem(sp, obj, candidates=32, generations=6, elite_frac=0.25, rng_seed=5)
    inc = [r["incumbent_reward"] for r in res["rows"]]
    assert all(b >= a for a, b in zip(inc, inc[1:]))
    for gen, (g, o) in enumerate(seen):
        assert g.dtype == np.int64 and o.dtype == np.int64
        assert (g >= sp.lo).all() and (g <= sp.hi).all()
        c = np.stack([sp.cycles(x) for x in g])
        assert (o[1:] >= 0).all() and (o[1:] < c[1:]).all()
        if gen == 0:
            assert (g[0] == sp.d0).all() and (o[0] == sp.base.offset).all()
        else:                                                  # candidate 0 is the best plan so far
            best = int(np.argmax(res["scores"][gen - 1]))
            assert (g[0] == seen[gen - 1][0][best]).all() and (o[0] == seen[gen - 1][1][best]).all()
            assert res["scores"][gen][0] == inc[gen - 1]
    assert res["shipped_score"] == res["scores"][0][0]
    assert res["best_score"] == inc[-1] == max(s.max() for s in res["scores"])
    again = cem(sp, f, candidates=32, generations=6, elite_frac=0.25, rng_seed=5)
    other = cem(sp, f, candidates=32, generations=6, elite_frac=0.25, rng_seed=6)
    for a, b in zip(res["greens"] + res["offsets"], again["greens"] + again["offsets"]):
        np.testing.assert_array_equal(a, b)
    assert any(not np.array_equal(a, b) for a, b in zip(res["greens"], other["greens"]))


def test_cem_reaches_an_interior_optimum():
    """on the small grid's 13 greens and 6 offsets: the greens exactly and the offsets within 3% of a cycle after 30
    generations of 128 candidates"""
    from deeprl_signal_control_b200.agents.tune_fixedtime import cem, search_space
    from deeprl_signal_control_b200.net import small_grid
    sp = search_space(_tables(small_grid.build_small_grid(agent="fixedtime"), small_grid.tls_programs()), 5, 60)
    rng = np.random.default_rng(11)
    tg, tu = rng.integers(sp.lo + 5, sp.hi - 5), rng.random(sp.n_nodes)
    assert (tg != sp.d0).any() and sp.n_green == 13
    res = cem(sp, _separable(sp, tg, tu), candidates=128, generations=30, elite_frac=0.1, rng_seed=0)
    assert (res["best_greens"] == tg).all()
    c = sp.cycles(res["best_greens"])
    du = np.abs(np.mod(res["best_offsets"] / c - tu + 0.5, 1.0) - 0.5)
    assert du.max() < 0.03, du.max()


def test_cem_raises_when_the_incumbent_does_not_repeat():
    from deeprl_signal_control_b200.agents.tune_fixedtime import cem
    sp = _grid_space()
    calls = []

    def noisy(g, o):
        calls.append(1)
        return -np.abs(g - sp.d0).sum(axis=1).astype(np.float64) + 1e-9 * len(calls)
    with pytest.raises(RuntimeError, match="generation 1: the incumbent scored"):
        cem(sp, noisy, candidates=8, generations=3)


def test_elites_ties_and_circular_statistics():
    from deeprl_signal_control_b200.agents.tune_fixedtime import circular_mean_std, n_elites
    assert n_elites(512, 0.1) == 51 and n_elites(16, 0.1) == 2 and n_elites(10, 0.01) == 1 and n_elites(4, 1.0) == 4
    mean, std = circular_mean_std(np.array([[0.95], [0.05], [0.97], [0.03]]))
    assert abs(mean[0]) < 1e-12 or abs(mean[0] - 1) < 1e-12
    mean, std = circular_mean_std(np.array([[0.9], [0.0]]))
    assert abs(mean[0] - 0.95) < 1e-12
    a = 2 * np.pi * 0.05
    assert abs(std[0] - np.sqrt(-2 * np.log(np.cos(a))) / (2 * np.pi)) < 1e-12
    mean, std = circular_mean_std(np.array([[0.3], [0.3]]))
    assert abs(mean[0] - 0.3) < 1e-12 and std[0] < 1e-6
    # ties go to the lower index: elites and incumbent of equal scores
    from deeprl_signal_control_b200.agents.tune_fixedtime import cem
    sp = _grid_space()
    seen = []

    def flat(g, o):
        seen.append(g.copy())
        return np.zeros(len(g))
    res = cem(sp, flat, candidates=8, generations=2, elite_frac=0.25)
    assert (seen[1][0] == seen[0][0]).all() and (res["best_greens"] == sp.d0).all()


def _cfg(tmp_path, **env):
    cp = configparser.ConfigParser()
    cp.read_string(GRID_INI)
    for k, v in env.items():
        cp["ENV_CONFIG"][k] = v
    path = str(tmp_path / "config_greedy_large.ini")
    with open(path, "w") as f:
        cp.write(f)
    return path


@pytest.mark.parametrize("kw,match", [
    (dict(seeds=[1001, 20000]), r"tuning seeds \[20000\] are evaluation seeds"),
    (dict(seeds=[1001, 50000]), r"tuning seeds \[50000\] are evaluation seeds"),
    (dict(seeds=[1001, 777]), r"tuning seeds \[777\] are evaluation seeds"),
    (dict(seeds=[]), "no tuning seeds"),
    (dict(candidates=1), "candidates must be at least 2"),
    (dict(elite_frac=0.0), r"elite_frac must be in \(0, 1\]"),
    (dict(elite_frac=1.5), r"elite_frac must be in \(0, 1\]"),
    (dict(min_green=0), "need 1 <= min_green <= max_green"),
    (dict(min_green=30, max_green=20), "need 1 <= min_green <= max_green"),
    (dict(generations=-1), "generations must be at least 0"),
])
def test_refusals(kw, match, tmp_path, no_device):  # noqa: F811
    from deeprl_signal_control_b200.agents.tune_fixedtime import tune_fixedtime
    cfg = _cfg(tmp_path, test_seeds="777,888")
    args = dict(seeds=[1001, 1002])
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        tune_fixedtime(cfg, str(tmp_path / "out"), **args)
    assert not os.path.exists(str(tmp_path / "out"))


def test_refuses_an_existing_plan_and_a_scenario_without_programs(tmp_path, no_device, monkeypatch):  # noqa: F811
    import deeprl_signal_control_b200.envs.fixedtime as ft
    from deeprl_signal_control_b200.agents.tune_fixedtime import tune_fixedtime
    cfg = _cfg(tmp_path)
    os.makedirs(str(tmp_path / "out" / "fixedtime" / "data"))
    open(str(tmp_path / "out" / "fixedtime" / "data" / "tuned.tll.xml"), "w").close()
    with pytest.raises(ValueError, match="tuned.tll.xml exists"):
        tune_fixedtime(cfg, str(tmp_path / "out"), [1001])
    with pytest.raises(ValueError, match="no config"):
        tune_fixedtime(str(tmp_path / "none.ini"), str(tmp_path / "o2"), [1001])

    def none(env):
        raise ValueError("no fixed-time programs for scenario %r" % env.name)
    monkeypatch.setattr(ft, "scenario_programs", none)
    with pytest.raises(ValueError, match="scenario 'large_grid' has no fixed-time programs"):
        tune_fixedtime(cfg, str(tmp_path / "o3"), [1001])
    assert not os.path.exists(str(tmp_path / "o3"))


def test_command_line():
    tf = _script("tune_fixedtime")
    a = tf.parse_args(["--base-dir", "runs/tuned", "--config-dir", "config_greedy_large.ini", "--seeds",
                       "1001,1002,1003"])
    assert (a.base_dir, a.config_dir, a.seeds) == ("runs/tuned", "config_greedy_large.ini", [1001, 1002, 1003])
    assert (a.candidates, a.generations, a.elite_frac, a.min_green, a.max_green, a.rng_seed, a.device) == \
        (512, 30, 0.1, 5, 60, 0, 0)
    a = tf.parse_args(["--base-dir", "b", "--config-dir", "c.ini", "--seeds", "5", "--candidates", "16",
                       "--generations", "0", "--elite-frac", "0.5", "--min-green", "3", "--max-green", "90",
                       "--rng-seed", "7", "--device", "1"])
    assert (a.candidates, a.generations, a.elite_frac, a.min_green, a.max_green, a.rng_seed, a.device) == \
        (16, 0, 0.5, 3, 90, 7, 1)
    with pytest.raises(SystemExit):
        tf.parse_args(["--base-dir", "b", "--config-dir", "c.ini", "--seeds", "1,x"])
    with pytest.raises(SystemExit):
        tf.parse_args(["--base-dir", "b", "--seeds", "1"])
