"""CPU: the training driver over several ranks (agents/train.py with a process group, dist.replica_range /
gather_traces) — world-size-2 gloo runs on CPU tensors of the trace gather, the pooled training row, the rank-0-only
rows, tests and CSV of the driver loop, and the rejection of bad arguments on every rank before any collective; and the
replica ranges of W ranks tiling [0, R_total)."""
import configparser
import datetime
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _global_trace(T, R_total, episode):
    g = torch.arange(T * R_total, dtype=torch.float64).reshape(T, R_total)
    return (-(((g * 7919) % 113) / 7.0) * episode).float()


class ShardTrainer:
    """One rank's share of a trainer: replicas [replica0, replica0 + r) of a deterministic global trace per episode."""

    def __init__(self, T, r, replica0, R_total):
        self.T_episode, self.r, self.replica0, self.R_total = T, r, replica0, R_total
        self.greward_trace = torch.zeros(T, r)
        self.episode_rewards = []
        self.episode = 0

    def run(self, n):
        assert n == self.T_episode
        self.episode += 1
        full = _global_trace(self.T_episode, self.R_total, self.episode)
        self.greward_trace.copy_(full[:, self.replica0:self.replica0 + self.r])
        self.episode_rewards.append(float(self.greward_trace.double().mean()))


class StubEvaluator:
    test_num = 2

    def __init__(self):
        self.calls = 0

    def perform_all(self):
        self.calls += 1
        return np.array([-1.0, -2.0]) * self.calls, np.array([0.5, 0.25]) * self.calls


COLLECTIVES = ("barrier", "gather", "all_gather", "all_reduce", "new_group", "broadcast")


def _forbid_collectives():
    """Any collective from here on fails the run: the argument checks must come before the first one."""
    def refuse(*a, **k):
        raise AssertionError("a collective ran before the arguments were checked")
    for name in COLLECTIVES:
        setattr(dist, name, refuse)


def _worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    sys.path.insert(0, ROOT)
    from deeprl_signal_control_b200.agents import train as drv
    from deeprl_signal_control_b200.dist import gather_traces, replica_range
    T, R_total = 6, 10
    replica0, r = replica_range(rank, world, R_total)

    # 1. the gather rebuilds [T, R_total] in global replica order on rank 0 only, and the row pools it
    full = _global_trace(T, R_total, 3)
    got = gather_traces(full[:, replica0:replica0 + r], group=None)
    if rank == 0:
        assert got.dtype == np.float32 and np.array_equal(got, full.numpy())
        avg, std = drv.training_row(got)
        one = full.double().numpy()
        assert std == np.std(one)                                       # the array a one-process run holds
        assert avg == float(np.mean(np.mean(one, axis=0)))
        np.testing.assert_allclose(avg, np.mean(one), rtol=1e-12)
    else:
        assert got is None

    # 2. the driver loop: every rank runs the schedule, rank 0 holds the rows, runs the tests and writes the CSV
    tr = ShardTrainer(T, r, replica0, R_total)
    ev = StubEvaluator() if rank == 0 else None
    path = os.path.join(out_dir, "rank%d" % rank) + os.sep
    os.makedirs(path)
    d = drv.Trainer(tr, ev, drv.Counter(3 * T, T, 100), "ma2c", True, path, group=dist.group.WORLD)
    d.run()
    assert d.n_episode_sets == 3 and tr.episode == 3
    if rank == 0:
        rows = [(x["step"], x["test_id"]) for x in d.data]
        assert rows == [(6, -1), (6, 0), (6, 1), (12, -1), (12, 0), (12, 1), (18, -1)]
        for e, x in enumerate([x for x in d.data if x["test_id"] == -1]):
            assert (x["avg_reward"], x["std_reward"]) == drv.training_row(_global_trace(T, R_total, e + 1).numpy())
        assert ev.calls == 2 and os.path.exists(path + "train_reward.csv")
    else:
        assert d.data == [] and os.listdir(path) == []

    # 3. bad arguments fail on every rank alike, before any collective (no rank is left waiting)
    cp = configparser.ConfigParser()
    for agent, n, match in (("ma2c", 7, "split evenly"), ("greedy", 8, "greedy"), ("a2c", 8, "a2c")):
        cp.read_string("[ENV_CONFIG]\nagent = %s\n[MODEL_CONFIG]\n[TRAIN_CONFIG]\n" % agent)
        dist.barrier()
        saved = {k: getattr(dist, k) for k in COLLECTIVES}
        _forbid_collectives()
        try:
            with pytest.raises(ValueError, match=match):
                drv.train(cp, os.path.join(out_dir, "bad_" + agent), n_replicas=n, process_group=dist.group.WORLD)
        finally:
            for k, v in saved.items():
                setattr(dist, k, v)
    open(os.path.join(out_dir, "ok%d" % rank), "w").write("1")
    dist.destroy_process_group()


def test_two_gloo_ranks_gather_pool_and_reject_alike(tmp_path):
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert (tmp_path / "ok0").exists() and (tmp_path / "ok1").exists()
    # an uneven split is refused before anything is written; greedy / a2c after rank 0 copied the config, as one
    # process does, and rank 1 wrote nothing
    assert not (tmp_path / "bad_ma2c").exists()
    for agent in ("greedy", "a2c"):
        base = tmp_path / ("bad_" + agent)
        assert sorted(os.listdir(base)) == ["data", "log", "model"]
        assert os.listdir(base / "data") == ["config.ini"] and os.listdir(base / "model") == []
        assert len(os.listdir(base / "log")) == 1


@pytest.mark.parametrize("world,total", [(1, 16), (2, 16), (4, 16), (3, 12), (8, 4096), (16, 16)])
def test_replica_ranges_tile_the_global_replicas(world, total):
    from deeprl_signal_control_b200.dist import replica_range
    ranges = [replica_range(k, world, total) for k in range(world)]
    assert ranges[0][0] == 0 and all(n == total // world for _, n in ranges)
    ids = np.concatenate([np.arange(r0, r0 + n) for r0, n in ranges])
    assert np.array_equal(ids, np.arange(total))


def test_replica_range_rejects_an_uneven_split_and_bad_ranks():
    from deeprl_signal_control_b200.dist import replica_range
    with pytest.raises(ValueError, match="split evenly"):
        replica_range(0, 3, 16)
    with pytest.raises(ValueError, match="not in a world"):
        replica_range(2, 2, 16)
    with pytest.raises(ValueError, match="not in a world"):
        replica_range(0, 0, 16)
