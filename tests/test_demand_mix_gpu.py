"""GPU: one agent trained on a mixture of traffic demand levels (train(demand_mix=...), global replica g at level g mod L)
on 3 levels x 64 replicas and short episodes.

- Grid MA2C in deterministic mode, and iqld on Monaco `flow_rate` levels through the table cache: a mixture train() run
  leaves the checkpoint (weights and optimiser state), train_reward.csv and train_reward_demand.csv of a hand-wired
  BatchedTrainer / BatchedIQLTrainer loop on which the test sets the levels itself; each level's training row is the
  mean / std over that level's columns of the run's trace; each data/<label>/ is what scripts/evaluate.py writes for
  the config edited to that level.
- A one-level mixture at the config's own demand leaves the directory of a plain train() (deterministic A2C and IQL),
  plus demand_mix.json, train_reward_demand.csv and data/<label>/ (equal to data/'s CSVs).
- Two gloo ranks on one GPU against one process: the directory of the one-process run within the bounds of
  test_train_multirank_gpu.py, and each rank's replicas at the levels of their global indices.
"""
import configparser
import copy
import datetime
import glob
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import torch

from tests.test_demand_gpu import _cfg_text, _trip_rows, _write

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RB = 64                                                    # replicas per level
GRID_LEVELS = [{"peak_flow1": "660", "peak_flow2": "555"}, {"peak_flow1": "1100", "peak_flow2": "925"},
               {"peak_flow1": "1540", "peak_flow2": "1295"}]
MONACO_LEVELS = [{"flow_rate": "195"}, {"flow_rate": "325"}, {"flow_rate": "455"}]


def _label(lv):
    return "_".join("%s-%s" % kv for kv in lv.items())


def _config(agent, scenario):
    c = _cfg_text(agent)
    if scenario == "real_net":
        c["ENV_CONFIG"]["scenario"], c["ENV_CONFIG"]["flow_rate"] = "real_net", "325"
        c["ENV_CONFIG"]["data_path"] = "/nonexistent/"     # no Monaco net file: the shipped table cache
    return c


def _edited(c, lv):
    c = copy.deepcopy(c)
    for k, v in lv.items():
        c["ENV_CONFIG"][k] = v
    return c


def _ckpt(d, step):
    from deeprl_signal_control_b200.agents import checkpoint as ck
    return ck.load_npz(os.path.join(d, "model", "checkpoint-%d.npz" % step))


def _same_ckpt(a, b, step):
    (wa, ea), (wb, eb) = _ckpt(a, step), _ckpt(b, step)
    assert sorted(wa) == sorted(wb) and sorted(ea) == sorted(eb) and ea
    for x, y in ((wa, wb), (ea, eb)):
        for n in x:
            assert np.array_equal(x[n], y[n]), n


def _bytes(path):
    with open(path, "rb") as f:
        return f.read()


def _hand_wired(c, levels, R, out):
    """The run wired by hand: env, learner, trainer, the levels set on the simulator (replica r at level r mod L), one
    episode per set, the rows computed here and written as the driver writes them, the model saved."""
    from deeprl_signal_control_b200.agents.train import build_model
    from deeprl_signal_control_b200.envs import make_env
    env_cfg, mc = c["ENV_CONFIG"], c["MODEL_CONFIG"]
    agent, seed = env_cfg.get("agent"), env_cfg.getint("seed")
    total_step = int(c.getfloat("TRAIN_CONFIG", "total_step"))
    os.makedirs(os.path.join(out, "model"))
    env = make_env(env_cfg, R, out + "/", is_record=False)
    model = build_model(agent, env, mc, total_step, R, seed=seed, deterministic=True)
    sim = env._ensure_sim()
    nets = [make_env(_edited(c, lv)["ENV_CONFIG"], 1, "", is_record=False)._tables for lv in levels]
    L = len(levels)
    sim.set_replica_demand(nets, np.arange(R) % L)
    T = int(env.T)
    trace = torch.zeros(T, R, dtype=torch.float32, device=sim.device)
    if model.name == "iql":
        from deeprl_signal_control_b200.agents.learner_iql import BatchedIQLTrainer
        from deeprl_signal_control_b200.agents.models import iql_schedulers
        tr = BatchedIQLTrainer(sim, model, *iql_schedulers(mc, total_step), seed0=seed, greward_trace=trace)
    else:
        from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
        tr = BatchedTrainer(sim, model.batched, agent, model.lr_scheduler, model.beta_scheduler, seed0=seed,
                            greward_trace=trace)
    rows, lrows, step = [], [], 0
    while step < total_step:
        tr.run(T)
        step += T
        g = trace.cpu().numpy().astype(np.float64)
        rows.append({"agent": agent, "step": step, "test_id": -1, "avg_reward": float(tr.episode_rewards[-1]),
                     "std_reward": float(np.std(g))})
        for j, lv in enumerate(levels):
            x = g[:, np.arange(R) % L == j]
            lrows.append({"agent": agent, "step": step, "test_id": -1, "demand": _label(lv),
                          "avg_reward": float(x.mean(axis=0).mean()), "std_reward": float(np.std(x))})
    pd.DataFrame(rows).to_csv(os.path.join(out, "train_reward.csv"))
    pd.DataFrame(lrows).to_csv(os.path.join(out, "train_reward_demand.csv"))
    model.save(os.path.join(out, "model") + "/", step)
    torch.cuda.synchronize()
    return step


@pytest.mark.parametrize("agent,scenario,levels", [("ma2c", "large_grid", GRID_LEVELS),
                                                   ("iqld", "real_net", MONACO_LEVELS)])
def test_mixture_equals_the_hand_wired_loop_and_evaluate(tmp_path, monkeypatch, agent, scenario, levels):
    from deeprl_signal_control_b200.agents.train import train
    from deeprl_signal_control_b200.sim import BatchedSim
    c = _config(agent, scenario)
    path = _write(tmp_path / ("config_%s.ini" % agent), c)
    R, L = RB * len(levels), len(levels)
    rec = []
    step_fn = BatchedSim.step

    def recording_step(self, *a, **k):
        out = step_fn(self, *a, **k)
        rec.append(out[2].double().cpu().numpy().copy())
        return out
    monkeypatch.setattr(BatchedSim, "step", recording_step)
    base = str(tmp_path / "mix" / agent)
    out = train(path, base, "after_train_test", n_replicas=R, deterministic=True, demand_mix=levels)
    monkeypatch.undo()
    labels = [_label(lv) for lv in levels]
    assert json.load(open(os.path.join(base, "data", "demand_mix.json"))) == {"levels": levels, "labels": labels}
    hand = str(tmp_path / "hand")
    step = _hand_wired(c, levels, R, hand)
    assert step == out.final_step
    _same_ckpt(base, hand, step)
    for name in ("train_reward.csv", "train_reward_demand.csv"):
        assert _bytes(os.path.join(base, "data", name)) == _bytes(os.path.join(hand, name)), name
    # each level's training row: mean / std over that level's columns of the trace the run stepped
    df = pd.read_csv(os.path.join(base, "data", "train_reward_demand.csv"), index_col=0, float_precision="round_trip")
    T = len(rec) // out.episode_sets
    assert len(df) == L * out.episode_sets and list(df.demand) == labels * out.episode_sets
    for e in range(out.episode_sets):
        g = np.stack(rec[e * T:(e + 1) * T])
        for j in range(L):
            row, x = df.iloc[e * L + j], g[:, np.arange(R) % L == j]
            assert row.avg_reward == pytest.approx(np.mean(x), rel=1e-12) and row.std_reward == np.std(x), (e, j)
    live = [row.avg_reward for _, row in df.iloc[:L].iterrows()]
    assert len(set(live)) == L                                           # the levels do run at different demand
    # data/<label>/ is scripts/evaluate.py on the config edited to that level
    for lv, lab in zip(levels, labels):
        ref = str(tmp_path / "ref" / lab / agent)
        shutil.copytree(base, ref, ignore=shutil.ignore_patterns(*labels))
        for ini in glob.glob(os.path.join(ref, "data", "*.ini")):
            _write(ini, _edited(_read(ini), lv))
        r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", ref],
                           capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stdout + r.stderr
        got = {n: _bytes(os.path.join(base, "data", lab, n)) for n in os.listdir(os.path.join(base, "data", lab))}
        want = {n: _bytes(os.path.join(ref, "eva_data", n)) for n in got}
        assert sorted(got) == ["%s_%s_%s.csv" % (scenario, agent, k) for k in ("control", "traffic", "trip")]
        for n in got:
            if n.endswith("_trip.csv"):                  # arrivals of one second enter the log in atomic order
                assert _trip_rows(got[n]) == _trip_rows(want[n]), (lab, n)
            else:
                assert got[n] == want[n], (lab, n)
        summary = json.load(open(os.path.join(ref, "eva_data", "%s_summary.json" % agent)))
        mean, std = out.demand_post_test[labels.index(lab)]
        assert summary["episode_mean_reward"] == [float(x) for x in mean]
        assert summary["episode_std_reward"] == [float(x) for x in std]


def _read(ini):
    c = configparser.ConfigParser()
    c.read(ini)
    return c


def _listing(d):
    out = []
    for root, _, files in os.walk(d):
        for n in files:
            rel = os.path.relpath(os.path.join(root, n), d)
            out.append("<log>" if rel.endswith(".log") else "<events>" if "events." in rel else rel)
    return sorted(out)


@pytest.mark.parametrize("agent", ["ma2c", "iqll"])
def test_one_level_at_the_configured_demand_is_a_plain_run(tmp_path, agent):
    from deeprl_signal_control_b200.agents.train import train
    from tests.test_deterministic_gpu import _scalars
    c = _cfg_text(agent)
    T = 120 if agent == "ma2c" else 60
    c["TRAIN_CONFIG"]["total_step"], c["TRAIN_CONFIG"]["test_interval"] = str(2 * T), str(T)   # one in-training test
    path = _write(tmp_path / ("config_%s.ini" % agent), c)
    plain, mix = str(tmp_path / "plain" / agent), str(tmp_path / "mix" / agent)
    a = train(path, plain, "all_test", n_replicas=RB, summaries=True, deterministic=True)
    b = train(path, mix, "all_test", n_replicas=RB, summaries=True, deterministic=True,
              demand_mix=[{"peak_flow1": "1100"}])
    lab = "peak_flow1-1100"
    added = ["data/demand_mix.json", "data/train_reward_demand.csv"] + \
        ["data/%s/large_grid_%s_%s.csv" % (lab, agent, k) for k in ("control", "traffic", "trip")]
    assert _listing(mix) == sorted(_listing(plain) + added)
    assert a.final_step == b.final_step
    _same_ckpt(mix, plain, a.final_step)
    for n in os.listdir(os.path.join(plain, "data")):
        if n.endswith(".csv"):
            assert _bytes(os.path.join(mix, "data", n)) == _bytes(os.path.join(plain, "data", n)), n
            if n.startswith("large_grid_"):              # the level's post-training test is the config's own
                x, y = _bytes(os.path.join(mix, "data", lab, n)), _bytes(os.path.join(plain, "data", n))
                assert (_trip_rows(x) == _trip_rows(y)) if n.endswith("_trip.csv") else x == y, n
    assert _scalars(mix) == _scalars(plain)
    rows = pd.read_csv(os.path.join(plain, "data", "train_reward.csv"), index_col=0, float_precision="round_trip")
    lrows = pd.read_csv(os.path.join(mix, "data", "train_reward_demand.csv"), index_col=0, float_precision="round_trip")
    assert (lrows.demand == lab).all() and list(lrows.step) == list(rows.step)
    assert list(lrows.test_id) == list(rows.test_id) and (rows.test_id >= 0).any()
    tests = rows.test_id >= 0                             # the level's test rows are the config's own
    assert list(lrows.avg_reward[tests]) == list(rows.avg_reward[tests])
    assert list(lrows.std_reward) == list(rows.std_reward)
    assert np.allclose(lrows.avg_reward, rows.avg_reward, rtol=1e-6, atol=0)


# ---- two ranks -------------------------------------------------------------------------------------------------------
R2, WORLD = 48, 2


def _worker(rank, port, out):
    import torch.distributed as dist
    from deeprl_signal_control_b200.sim import BatchedSim
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=WORLD, timeout=datetime.timedelta(seconds=300))
    seen = []
    orig = BatchedSim.set_replica_demand

    def recording(self, levels=None, level_of=None):
        seen.append(np.asarray(level_of).copy())
        return orig(self, levels, level_of)
    BatchedSim.set_replica_demand = recording
    from deeprl_signal_control_b200.agents.train import train
    res = train(os.path.join(out, "config_ma2c.ini"), os.path.join(out, "ma2c"), "all_test", n_replicas=R2,
                process_group=dist.group.WORLD, demand_mix=GRID_LEVELS)
    BatchedSim.set_replica_demand = orig
    np.savez(os.path.join(out, "rank%d.npz" % rank), P=res.model.batched.P.cpu().numpy(),
             MS=res.model.batched.MS.cpu().numpy(), level_of=np.stack(seen))
    dist.destroy_process_group()


def test_two_ranks_leave_the_one_process_directory(tmp_path):
    import torch.multiprocessing as mp
    from deeprl_signal_control_b200.agents.train import train
    from tests.test_train_multirank_gpu import WEIGHT_BOUND, _free_port
    from tests.test_train_driver_gpu import _ini
    text = _ini("ma2c", 360, 240)
    w2, w1 = tmp_path / "w2", tmp_path / "w1"
    for d in (w2, w1):
        d.mkdir()
        (d / "config_ma2c.ini").write_text(text)
    mp.spawn(_worker, args=(_free_port(), str(w2)), nprocs=WORLD, join=True)
    one = train(str(w1 / "config_ma2c.ini"), str(w1 / "ma2c"), "all_test", n_replicas=R2, demand_mix=GRID_LEVELS)
    a, b = str(w2 / "ma2c"), str(w1 / "ma2c")
    assert _listing(a) == _listing(b)
    r = R2 // WORLD
    ranks = [dict(np.load(w2 / ("rank%d.npz" % k))) for k in range(WORLD)]
    for k, npz in enumerate(ranks):
        assert npz["level_of"].shape == (1, r)
        assert np.array_equal(npz["level_of"][0], (k * r + np.arange(r)) % 3), k
    assert np.array_equal(ranks[0]["P"], ranks[1]["P"]) and np.array_equal(ranks[0]["MS"], ranks[1]["MS"])
    err = float(np.abs(ranks[0]["P"] - one.model.batched.P.cpu().numpy()).max())
    print("\nmixture over 2 ranks: max |P_2 - P_1| = %.3g (bound %.0e)" % (err, WEIGHT_BOUND["ma2c"]))
    assert err <= WEIGHT_BOUND["ma2c"]
    for name, keys in (("train_reward.csv", ["step", "test_id"]), ("train_reward_demand.csv", ["step", "test_id", "demand"])):
        x, y = (pd.read_csv(os.path.join(d, "data", name), index_col=0, float_precision="round_trip") for d in (a, b))
        assert x[keys].equals(y[keys]), name
        first = x.step == x.step.iloc[0]                 # the first episode set plays the same episodes
        assert list(x.std_reward[first & (x.test_id == -1)]) == list(y.std_reward[first & (y.test_id == -1)]), name
    d2 = pd.read_csv(os.path.join(a, "data", "train_reward_demand.csv"), index_col=0, float_precision="round_trip")
    d1 = pd.read_csv(os.path.join(b, "data", "train_reward_demand.csv"), index_col=0, float_precision="round_trip")
    assert list(d2.avg_reward[:3]) == list(d1.avg_reward[:3])     # both from training_row over the same trace
