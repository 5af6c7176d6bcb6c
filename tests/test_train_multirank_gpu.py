"""GPU: one agent trained over two ranks by the training driver (agents/train.py with a process group), against the
one-process run with the same 16 replicas in all, on the grid config of test_train_driver_gpu.py (T = 120, 360 steps,
all_test).  Two gloo ranks share cuda:0 (torch.multiprocessing.spawn); the NCCL variant goes through torchrun and
scripts/train.py on two devices and is skipped with fewer.

Checked for ma2c, ia2c (FC policy), iqll and iqld: the directory is the one a one-process run leaves, all of it from rank
0; the first episode set plays the same episodes (A2C: the pooled std bit for bit, the mean to 1e-6; IQL: the first
backward's ring contents and its first round's replay indices); every row has the same step and test id; the final
weights agree with the one-process run within bounds set from the values observed on the H100, and the two ranks hold
bit-identical weights and optimiser state; a second IQL run repeats the first bit for bit; the post-training CSVs equal
scripts/evaluate.py on the run's own checkpoint."""
import datetime
import glob
import json
import os
import socket
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from tests.test_train_driver_gpu import R, SEEDS, _ini, _rows, _run, _weights

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORLD = 2
AGENTS = [("ma2c", "lstm"), ("ia2c", "fc"), ("iqll", "lstm"), ("iqld", "lstm")]
JOBS = [(a, a, p) for a, p in AGENTS] + [("iqld_again", "iqld", "lstm")]     # (tag, agent, policy)
# max |P_world2 - P_world1| after 360 steps: about 3x the worst of three runs on an H100 80GB HBM3 at 700 W (DESIGN.md
# §7: 1.49e-8, 2.98e-8, 2.98e-8, 9.79e-5).  IQL-DQN's Adam steps are about lr = 1e-4 wherever the gradient is tiny, so
# a last-bit difference in the summation order there moves a weight by up to lr.
WEIGHT_BOUND = {"ma2c": 5e-8, "ia2c": 1e-7, "iqll": 1e-7, "iqld": 3e-4}


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


class FirstIQLBackward:
    """Records, at the first BatchedIQL.backward that runs its rounds, the ring entries written so far and the replay
    indices of its first round."""

    def __init__(self):
        from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL
        self.cls, self.snap = BatchedIQL, None
        self.orig = BatchedIQL.backward, BatchedIQL.sample
        rec, (backward, sample) = self, self.orig

        def recording_backward(m, lr):
            if rec.snap is None and m.size >= m.batch_size:
                rec.snap = {k: getattr(m, k)[:m.size].cpu().numpy().copy() for k in ("s", "s1", "a", "r", "done")}
            return backward(m, lr)

        def recording_sample(m, rnd):
            idx = sample(m, rnd)
            if rec.snap is not None and "idx" not in rec.snap:
                rec.snap["idx"] = idx.cpu().numpy().copy()
            return idx
        BatchedIQL.backward, BatchedIQL.sample = recording_backward, recording_sample

    def restore(self):
        self.cls.backward, self.cls.sample = self.orig


def _state(model):
    if model.name == "iql":
        return {"P": model.P.cpu().numpy(), "M": model.M.cpu().numpy(), "V": model.V.cpu().numpy(),
                "t": np.int64(model.t)}
    return {"P": model.batched.P.cpu().numpy(), "MS": model.batched.MS.cpu().numpy()}


def _worker(rank, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=WORLD, timeout=datetime.timedelta(seconds=300))
    from deeprl_signal_control_b200.agents.train import train
    for tag, agent, policy in JOBS:
        rec = FirstIQLBackward()
        try:
            cfg = os.path.join(out, tag, "config_%s_large.ini" % agent)
            res = train(cfg, os.path.join(out, tag, agent), "all_test", n_replicas=R, policy=policy, device=0,
                        process_group=dist.group.WORLD)
        finally:
            rec.restore()
        snap = {"ring_" + k: v for k, v in (rec.snap or {}).items()}
        np.savez(os.path.join(out, "%s_rank%d.npz" % (tag, rank)), **_state(res.model), **snap,
                 meta=np.array(json.dumps({"world": res.world, "rank": res.rank, "env_samples": res.env_samples,
                                           "final_step": res.final_step, "data_none": res.data is None,
                                           "post_none": res.post_test is None,
                                           "post_test": None if res.post_test is None else
                                           [[float(x) for x in v] for v in res.post_test],
                                           "episode_rewards": res.trainer.episode_rewards})))
    np.save(os.path.join(out, "peak_rank%d.npy" % rank), np.int64(torch.cuda.max_memory_allocated()))
    dist.destroy_process_group()


@pytest.fixture(scope="module")
def world2(tmp_path_factory):
    """Every job trained over two gloo ranks on cuda:0, in one spawn: {tag: (base dir, [rank 0 npz, rank 1 npz])}"""
    import torch.multiprocessing as mp
    out = tmp_path_factory.mktemp("world2")
    for tag, agent, _ in JOBS:
        (out / tag).mkdir()
        (out / tag / ("config_%s_large.ini" % agent)).write_text(_ini(agent, 360, 240))
    t0 = time.time()
    mp.spawn(_worker, args=(_free_port(), str(out)), nprocs=WORLD, join=True)
    peaks = [int(np.load(out / ("peak_rank%d.npy" % k))) for k in range(WORLD)]
    print("\nworld-2 jobs: %.1f s wall, peak allocated per rank %s GB"
          % (time.time() - t0, [round(p / 1e9, 3) for p in peaks]))
    res = {}
    for tag, agent, _ in JOBS:
        res[tag] = (out / tag / agent, [dict(np.load(out / ("%s_rank%d.npz" % (tag, k)))) for k in range(WORLD)])
    return res


@pytest.fixture(scope="module")
def world1(tmp_path_factory):
    """The one-process run of every agent with the same R = 16: {agent: (base dir, namespace, IQL snapshot)}"""
    out = tmp_path_factory.mktemp("world1")
    res = {}
    for agent, policy in AGENTS:
        rec = FirstIQLBackward()
        try:
            base, ns = _run(out, agent, agent, "all_test", policy=policy)
        finally:
            rec.restore()
        res[agent] = (base, ns, rec.snap)
    print("\nworld-1 runs: peak allocated %.3f GB" % (torch.cuda.max_memory_allocated() / 1e9))
    return res


def _meta(npz):
    return json.loads(str(npz["meta"]))


def _layout(base):
    """The files the driver leaves under data/, model/ and log/, the log named by its kind rather than its time"""
    return sorted(("log/<time>.log" if d == "log" else "%s/%s" % (d, f)) for d in ("data", "model", "log")
                  for f in os.listdir(base / d))


@pytest.mark.parametrize("agent,policy", AGENTS)
def test_two_ranks_leave_the_one_process_directory(world2, world1, agent, policy):
    base2, (r0, r1) = world2[agent]
    base1, ns1, _ = world1[agent]
    files = _layout(base2)
    assert files == _layout(base1)
    assert [f for f in files if not f.startswith("data/")] == ["log/<time>.log", "model/checkpoint-360.npz"]
    assert (base2 / "data" / ("config_%s_large.ini" % agent)).read_text() == _ini(agent, 360, 240)
    logs = glob.glob(str(base2 / "log" / "*.log"))
    text = open(logs[0]).read()
    assert "Training: global step 240" in text and "over 2 ranks" in text and "[rank 1]" not in text
    m0, m1 = _meta(r0), _meta(r1)
    assert (m0["world"], m0["rank"], m1["world"], m1["rank"]) == (2, 0, 2, 1)
    assert m0["env_samples"] == m1["env_samples"] == 360 * R == ns1.env_samples
    assert (m0["data_none"], m0["post_none"], m1["data_none"], m1["post_none"]) == (False, False, True, True)


@pytest.mark.parametrize("agent,policy", AGENTS)
def test_two_ranks_play_the_one_process_episodes(world2, world1, agent, policy):
    base2, (r0, r1) = world2[agent]
    base1, ns1, snap1 = world1[agent]
    d2, d1 = _rows(base2), _rows(base1)
    assert list(zip(d2.step, d2.test_id)) == list(zip(d1.step, d1.test_id)) == \
        [(120, -1), (240, -1), (240, 0), (240, 1), (360, -1)]
    assert (d2.agent == agent).all()
    if agent in ("ma2c", "ia2c"):
        # the first update comes at the end of the first episode set (batch_size = T), so that set is the same play
        a, b = d2.iloc[0], d1.iloc[0]
        assert a.std_reward == b.std_reward
        assert abs(a.avg_reward - b.avg_reward) <= 1e-6 * abs(b.avg_reward)
    else:
        r = R // WORLD
        for k, npz in enumerate((r0, r1)):
            lo = k * r
            for key in ("s", "s1", "a", "r", "done"):
                assert np.array_equal(npz["ring_" + key], snap1[key][:, lo:lo + r]), (k, key)
            assert np.array_equal(npz["ring_idx"], snap1["idx"][:, lo:lo + r]), k


@pytest.mark.parametrize("agent,policy", AGENTS)
def test_two_ranks_train_one_model_close_to_the_one_process_run(world2, world1, agent, policy):
    _, (r0, r1) = world2[agent]
    _, ns1, _ = world1[agent]
    keys = [k for k in r0 if not k.startswith("ring_") and k != "meta"]
    for k in keys:
        assert np.array_equal(r0[k], r1[k]), k                         # one model, bit for bit on both ranks
    got, want = r0["P"], _weights(ns1.model).cpu().numpy()
    err = float(np.abs(got - want).max())
    print("\n%s: max |P_2 - P_1| = %.3g (bound %.0e), rows %s" % (agent, err, WEIGHT_BOUND[agent],
                                                                    _meta(r0)["episode_rewards"]))
    assert err <= WEIGHT_BOUND[agent]
    if agent.startswith("iq"):
        assert int(r0["t"]) == ns1.model.t > 0


def test_a_second_iql_run_repeats_the_first(world2):
    (b1, (a0, a1)), (b2, (c0, c1)) = world2["iqld"], world2["iqld_again"]
    for k in ("P", "M", "V", "t"):
        assert np.array_equal(a0[k], c0[k]) and np.array_equal(a1[k], c1[k]), k
    assert _rows(b1).equals(_rows(b2))
    assert _meta(a0)["episode_rewards"] == _meta(c0)["episode_rewards"]


@pytest.mark.parametrize("agent,policy", AGENTS)
def test_post_training_test_equals_evaluate_script(world2, agent, policy):
    base, (r0, _) = world2[agent]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "evaluate.py"), "--agent-dir", str(base),
                        "--evaluation-policy-type", "default", "--policy", policy], capture_output=True, text=True,
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    got = json.load(open(base / "eva_data" / ("%s_summary.json" % agent)))
    mean, std = _meta(r0)["post_test"]
    assert got["seeds"] == SEEDS
    assert got["episode_mean_reward"] == mean and got["episode_std_reward"] == std
    for kind in ("control", "traffic"):
        name = "large_grid_%s_%s.csv" % (agent, kind)
        assert (base / "data" / name).read_text() == (base / "eva_data" / name).read_text(), kind


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="the NCCL variant needs two visible GPUs")
def test_torchrun_nccl_two_devices(tmp_path, world1):
    cfg = tmp_path / "config_ma2c_large.ini"
    cfg.write_text(_ini("ma2c", 360, 240))
    base = tmp_path / "ma2c"
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", "2",
                        os.path.join(ROOT, "scripts", "train.py"), "--base-dir", str(base), "train", "--config-dir",
                        str(cfg), "--test-mode", "all_test", "--replicas", str(R), "--backend", "nccl"],
                       capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    line = json.loads(lines[0])
    assert (line["final_step"], line["env_samples"], line["world"]) == (360, 360 * R, 2)
    d2, d1 = _rows(base), _rows(world1["ma2c"][0])
    assert list(zip(d2.step, d2.test_id)) == list(zip(d1.step, d1.test_id))
    assert d2.iloc[0].std_reward == d1.iloc[0].std_reward
    assert _layout(base) == _layout(world1["ma2c"][0])
